"""Timing of the sampler of N(x*, H) from the final L-BFGS approximation (DESIGN.md §8e), with the card's name and power limit read in the
same run.

- Large n (n = 1e7, c = 10, k in {1, 4, 16}): the fused sampler (lbfgs_b200_hist_wt_dot_normal + lbfgs_b200_hist_lincomb_normal, z generated
  inside both passes) against "generate z into memory, then the factor product" (lincomb_normal on a history with no pairs writes z, then
  lbfgs_b200_hist_wt_dot_multi + lbfgs_b200_hist_lincomb_multi read it), each with GB/s on the traffic model, w = bytes per element:
      fused:    w n 2c (dots) + w n (c + 1 + k) (combination: s columns, mean, k outputs)
      unfused:  w n k (write z) + w n (2c + k) (dots) + w n (2c + 2k) (combination: y and s columns, z, outputs)
  The host algebra between the passes is not part of either time's passes but is inside the measured call sequence.
- Small batch (B = 65 536, n = 256 and B = 1024, n = 1016, m = 10): draws per second of lbfgs_b200_small_hist_sample (k = 16 and k = 256
  per problem) and the time of lbfgs_b200_small_hist_logdet over all problems.

Usage: python tools/hessian_sample_bench.py [--reps R] [--out FILE]   (one JSON object on stdout; FILE also receives it)
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lbfgspp_b200 as lb  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power = [f.strip() for f in r.stdout.splitlines()[0].split(",")]
    return name, power


def timed(ctx, fn, reps):
    fn()
    ctx.sync()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    ctx.sync()
    return (time.perf_counter() - t0) / reps


def large_n(ctx, reps, n=10_000_000, m=10):
    w = 8
    rng = np.random.default_rng(1)
    h = lb.History(ctx, n, m)
    for _ in range(m):
        s = rng.standard_normal(n)
        y = s * (1.0 + rng.random(n))
        h.add(ctx.array(s), ctx.array(y))
    h0 = lb.History(ctx, n, m)          # no pairs: lincomb_normal writes a0 z, the generator alone
    c = h.ncorr
    mean = ctx.array(np.zeros(n))
    out = {}
    for k in (1, 4, 16):
        OUT = ctx.empty(k * n)
        Z = ctx.empty(k * n)
        coef = np.zeros((2 * c, k))

        def fused():
            h.wt_dot_normal(11, 0, 0, k)
            h.lincomb_normal(1.0, 11, 0, 0, k, mean, coef, OUT, n)

        def unfused():
            h0.lincomb_normal(1.0, 11, 0, 0, k, None, np.zeros((0, k)), Z, n)
            h.wt_dot_multi(Z, k, n)
            h.lincomb_multi(1.0, Z, k, n, coef, OUT, n)

        tf, tu = timed(ctx, fused, reps), timed(ctx, unfused, reps)
        bf = w * n * (2 * c + c + 1 + k)
        bu = w * n * (k + 2 * c + k + 2 * c + 2 * k)
        out["k=%d" % k] = dict(fused_ms=tf * 1e3, fused_gb_s=bf / tf / 1e9, unfused_ms=tu * 1e3, unfused_gb_s=bu / tu / 1e9,
                               speedup=tu / tf)
    # the two passes of the fused sampler alone, at k = 16
    tdots = timed(ctx, lambda: h.wt_dot_normal(11, 0, 0, 16), reps)
    OUT = ctx.empty(16 * n)
    tcomb = timed(ctx, lambda: h.lincomb_normal(1.0, 11, 0, 0, 16, mean, np.zeros((2 * c, 16)), OUT, n), reps)
    out["k=16 passes"] = dict(dots_ms=tdots * 1e3, dots_gb_s=w * n * 2 * c / tdots / 1e9, combination_ms=tcomb * 1e3,
                              combination_gb_s=w * n * (c + 1 + 16) / tcomb / 1e9)
    return dict(n=n, c=c, dtype="f64", results=out)


def small_batch(ctx, reps, B, n, m=10):
    n = min(n, lb.small_max_n(m, lb.OBJ_ROSENBROCK_PAIRED))
    X0 = np.random.default_rng(2).uniform(-1.2, 1.2, (B, n))
    h = lb.SmallHistory(ctx, n, m, B)
    X = ctx.array(X0.reshape(-1))
    h.minimize(lb.OBJ_ROSENBROCK_PAIRED, X, lb.LBFGSParam(m=m, max_iterations=200))
    ctx.sync()
    res = dict(B=B, n=n, m=m, dtype="f64")
    for k in (16, 256):
        if B * k * n > 600_000_000:
            continue
        O = ctx.empty(B * k * n)
        t = timed(ctx, lambda: h.sample(5, 0, 0, B, k, X, n, O, n, k * n), reps)
        res["k=%d" % k] = dict(ms=t * 1e3, draws_per_s=B * k / t, gb_s_outputs=8 * B * k * n / t / 1e9)
        del O
    t = timed(ctx, lambda: h.logdet(), reps)
    res["logdet_all"] = dict(ms=t * 1e3, problems_per_s=B / t)
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
