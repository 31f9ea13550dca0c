"""Timing of whitening and log densities under N(x*, H) from the final L-BFGS approximation (DESIGN.md §8f), with the card's name and
power limit read in the same run.

- Large n (n = 1e7, c = 10, fp64, k in {1, 4, 16}): L' V, L^-1 V, L^-T V (one dots pass, the coefficients on the host, one combination
  pass: the sequence BFGSMat runs) and the log density (lbfgs_b200_hist_wt_dot_diff alone), each with GB/s on the traffic model,
  w = bytes per element:
      L', L^-T:     dots w n (c + k),          combination w n (2c + 2k)
      L^-1:         dots w n (2c + k),         combination w n (2c + 2k)
      log density:  dots w n (2c + k + 1),     no combination
  Also the S-only dots against hist_wt_dot_multi on the same V, and the log density against the route without it: B (X - mean) by
  the compact products (lbfgs_b200_axpy_out for the differences, hist_wt_dot_multi + hist_lincomb_multi), then a dot per point.
- Small batch (B = 65 536, n = 256 and B = 1024, n = 1016, m = 10): outputs per second of lbfgs_b200_small_hist_factor_apply for each op
  (k = 16 per problem) and of lbfgs_b200_small_hist_log_density (k = 16 points per problem).

Usage: python tools/hessian_whiten_bench.py [--reps R] [--out FILE]   (one JSON object on stdout; FILE also receives it)
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lbfgspp_b200 as lb  # noqa: E402
from tools.hessian_sample_bench import card, timed  # noqa: E402


class View:
    """n elements of a DeviceArray from element off on, for the per-vector calls of the route without wt_dot_diff."""

    def __init__(self, a, off, n):
        self.ptr, self.n, self.dtype, self.ct = C.c_void_p(a.ptr.value + off * a.dtype.itemsize), n, a.dtype, a.ct


def large_n(ctx, reps, n=10_000_000, m=10):
    w = 8
    rng = np.random.default_rng(1)
    h = lb.History(ctx, n, m)
    for _ in range(m):
        s = rng.standard_normal(n)
        y = s * (1.0 + rng.random(n))
        h.add(ctx.array(s), ctx.array(y))
    c = h.ncorr
    mean = ctx.array(rng.standard_normal(n))
    out = {}
    for k in (1, 4, 16):
        V = ctx.array(rng.standard_normal(k * n))
        OUT = ctx.empty(k * n)
        D = ctx.empty(k * n)
        coef = np.zeros((2 * c, k))

        def op_s():      # L' and L^-T: S'V, then the combination over W
            h.s_dot_multi(V, k, n)
            h.lincomb_multi(1.0, V, k, n, coef, OUT, n)

        def op_w():      # L^-1: W'V, then the combination (y coefficients zero)
            h.wt_dot_multi(V, k, n)
            h.lincomb_multi(1.0, V, k, n, coef, OUT, n)

        def density():
            h.wt_dot_diff(V, k, n, mean)

        def density_today():   # differences, B (x - mean), a dot per point
            for j in range(k):
                ctx.axpy_out(View(V, j * n, n), -1.0, mean, View(D, j * n, n))
            h.wt_dot_multi(D, k, n)
            h.lincomb_multi(1.0, D, k, n, coef, OUT, n)
            for j in range(k):
                ctx.dot(View(D, j * n, n), View(OUT, j * n, n))

        ts, tw, td = timed(ctx, op_s, reps), timed(ctx, op_w, reps), timed(ctx, density, reps)
        r = dict(LT_LINVT_ms=ts * 1e3, LT_LINVT_gb_s=w * n * (c + k + 2 * c + 2 * k) / ts / 1e9,
                 LINV_ms=tw * 1e3, LINV_gb_s=w * n * (2 * c + k + 2 * c + 2 * k) / tw / 1e9,
                 log_density_ms=td * 1e3, log_density_gb_s=w * n * (2 * c + k + 1) / td / 1e9)
        tt = timed(ctx, density_today, reps)
        r.update(log_density_via_products_ms=tt * 1e3, log_density_speedup=tt / td)
        tsd = timed(ctx, lambda: h.s_dot_multi(V, k, n), reps)
        twd = timed(ctx, lambda: h.wt_dot_multi(V, k, n), reps)
        r.update(s_dots_ms=tsd * 1e3, s_dots_gb_s=w * n * (c + k) / tsd / 1e9, wt_dots_ms=twd * 1e3,
                 wt_dots_gb_s=w * n * (2 * c + k) / twd / 1e9)
        out["k=%d" % k] = r
        del V, OUT, D
    return dict(n=n, c=c, dtype="f64", results=out)


def small_batch(ctx, reps, B, n, m=10, k=16):
    n = min(n, lb.small_max_n(m, lb.OBJ_ROSENBROCK_PAIRED))
    X0 = np.random.default_rng(2).uniform(-1.2, 1.2, (B, n))
    h = lb.SmallHistory(ctx, n, m, B)
    X = ctx.array(X0.reshape(-1))
    h.minimize(lb.OBJ_ROSENBROCK_PAIRED, X, lb.LBFGSParam(m=m, max_iterations=200))
    ctx.sync()
    res = dict(B=B, n=n, m=m, k=k, dtype="f64")
    V = ctx.array(np.random.default_rng(3).standard_normal(B * k * n))
    O = ctx.empty(B * k * n)
    for op in ("L", "LT", "LINV", "LINVT"):
        t = timed(ctx, lambda: h.factor_apply(op, 0, B, k, V, n, k * n, O, n, k * n), reps)
        res[op] = dict(ms=t * 1e3, outputs_per_s=B * k / t)
    t = timed(ctx, lambda: h.log_density(0, B, k, V, n, k * n, X, n), reps)
    res["log_density"] = dict(ms=t * 1e3, outputs_per_s=B * k / t)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    ctx = lb.Context()
    r = dict(card=name, power_limit=power, large_n=large_n(ctx, a.reps),
             small_batch=[small_batch(ctx, a.reps, 65536, 256), small_batch(ctx, a.reps, 1024, 1016)])
    s = json.dumps(r, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
