"""Throughput of the operator form of the final L-BFGS approximation on a C2-size ring (n = 1e7, m = c = 10, fp64).

For k in {1, 4, 8, 16} one product is the two k-vector passes over the history: lbfgs_b200_hist_wt_dot_multi ([Y S]'V, with its host
read-back) followed by lbfgs_b200_hist_lincomb_multi (the combination), i.e. what BFGSMat::hessian_times runs per group of vectors
minus the 2c x 2c host algebra.  Against it, in the same run and alternating with it: k separate lbfgs_b200_hist_apply_Hv calls (Gram
form).  Device time comes from CUDA events (lbfgs_b200_timer_start / stop) over enough calls to last at least a second, after warm-up.
Rates are algorithmic: 8 n (4c + 3k) bytes per product, 8 n (4c + 3) k bytes for k apply_Hv calls, against the 3.35 TB/s of the H100
SXM data sheet.  The card's name, power limit and SM clock are read in the same run.

  python tools/hessian_ops_bench.py [--n N] [--m M] [--min-seconds S] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lbfgspp_b200 as lb  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12   # H100 SXM HBM3, NVIDIA data sheet


class Column:
    """Column j of a device block, as the vector argument of History.apply_Hv (which only reads .ptr)"""

    def __init__(self, block, byte_offset):
        self.ptr = type(block.ptr)(block.ptr.value + byte_offset)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [s.strip() for s in q.split(",")]
        return dict(name=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
    except Exception as e:   # the measurement itself does not depend on it
        return dict(error=str(e))


def timed(ctx, fn, min_seconds):
    """ms per call of fn(): calls are batched until the batch lasts min_seconds of device time"""
    calls = 1
    while True:
        ctx.timer_start()
        for _ in range(calls):
            fn()
        ms = ctx.timer_stop()
        if ms >= 1e3 * min_seconds:
            return ms / calls
        calls = max(calls * 2, int(calls * 1.2e3 * min_seconds / max(ms, 1e-3)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--m", type=int, default=10)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the two variants per k")
    ap.add_argument("--out")
    args = ap.parse_args()
    n, m = args.n, args.m
    ctx = lb.Context(0)
    rng = np.random.default_rng(0)
    h = lb.History(ctx, n, m)
    for _ in range(m):
        s = rng.standard_normal(n)
        h.add(ctx.array(s), ctx.array(s + 0.1 * rng.standard_normal(n)))
    c = h.ncorr
    kmax = 16
    V = ctx.array(rng.standard_normal(kmax * n))
    OUT = ctx.empty(kmax * n)
    res = ctx.empty(n)
    cols = [Column(V, 8 * j * n) for j in range(kmax)]
    coef = {k: rng.standard_normal((2 * c, k)) for k in (1, 4, 8, 16)}

    def product(k):
        h.wt_dot_multi(V, k, n)
        h.lincomb_multi(0.5, V, k, n, coef[k], OUT, n)

    def separate(k):
        for j in range(k):
            h.apply_Hv(cols[j], 1.0, res, lb.HV_GRAM)

    rows = []
    for k in (1, 4, 8, 16):
        product(k), separate(k)   # warm-up
        t_multi, t_sep = [], []
        for _ in range(args.rounds):
            t_multi.append(timed(ctx, lambda: product(k), args.min_seconds))
            t_sep.append(timed(ctx, lambda: separate(k), args.min_seconds))
        bm, bs = 8.0 * n * (4 * c + 3 * k), 8.0 * n * (4 * c + 3) * k
        ms_m, ms_s = min(t_multi), min(t_sep)
        rows.append(dict(k=k, product_ms=ms_m, product_ms_all=t_multi, product_GBps=bm / ms_m / 1e6, product_peak_frac=bm / ms_m / 1e-3 / PEAK_BYTES_PER_S,
                         apply_Hv_x_k_ms=ms_s, apply_Hv_x_k_ms_all=t_sep, apply_Hv_x_k_GBps=bs / ms_s / 1e6,
                         apply_Hv_x_k_peak_frac=bs / ms_s / 1e-3 / PEAK_BYTES_PER_S, speedup=ms_s / ms_m,
                         words_per_coordinate=dict(product=4 * c + 3 * k, apply_Hv_x_k=(4 * c + 3) * k)))
    out = dict(n=n, m=m, c=c, dtype="fp64", card=card(), peak_bytes_per_s=PEAK_BYTES_PER_S, rows=rows)
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print("%-4s %12s %10s %8s | %14s %10s %8s | %7s" % ("k", "product ms", "GB/s", "of peak", "k x apply_Hv ms", "GB/s", "of peak", "speedup"))
    for r in rows:
        print("%-4d %12.3f %10.0f %7.1f%% | %14.3f %10.0f %7.1f%% | %6.2fx" % (r["k"], r["product_ms"], r["product_GBps"], 100 * r["product_peak_frac"],
                                                                             r["apply_Hv_x_k_ms"], r["apply_Hv_x_k_GBps"], 100 * r["apply_Hv_x_k_peak_frac"], r["speedup"]))


if __name__ == "__main__":
    main()
