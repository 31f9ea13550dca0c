"""Time the kept final approximations of the small-batch solve on the GPU (CUDA events, best of three).

    python tools/small_batch_hessian_bench.py [--out DIR]

Workloads (the small-batch solve's own): B = 65 536 problems of n = 256, m = 10, More-Thuente; B = 1024 at n = small_max_n(10) = 1016.
For each: the solve without and with keep_final_approx, alternating; the products with every problem's B and H at k = 1 and 16, as
problems/s and as GB/s of the w*n*(4c + 3k) bytes a problem's group needs (2c history columns read twice, V twice, OUT once) against the
H100 SXM data sheet's 3.35 TB/s; and the dense H of 1024 problems at n = 256 (V = I shared, k = n).  Prints one JSON line per number
and the card's name and power limit."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lbfgspp_b200 as lb  # noqa: E402

PEAK = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:   # the numbers still stand; say that the card could not be read
        return "unknown (%s)" % e


def timed(ctx, fn, reps=3):
    best = None
    for _ in range(reps):
        ctx.timer_start()
        fn()
        ms = ctx.timer_stop()
        best = ms if best is None else min(best, ms)
    return best


def run(ctx, B, n, m, emit):
    prm = lb.LBFGSParam(m=m, max_iterations=100)
    X0 = np.random.default_rng(0).uniform(-1.2, 1.2, (B, n))
    h = lb.SmallHistory(ctx, n, m, B)
    X = ctx.array(X0.reshape(-1))
    solve = {}
    for keep in (False, True, False, True, False, True):   # alternating
        ctx.check(ctx.lib.lbfgs_b200_memcpy_h2d(ctx.h, X.ptr, X0.ctypes.data_as(C.c_void_p), X0.nbytes))
        ms = timed(ctx, lambda: h.minimize(lb.OBJ_ROSENBROCK_PAIRED, X, prm, "MoreThuente", keep=keep), reps=1)
        solve[keep] = min(solve.get(keep, ms), ms)
    for keep in (False, True):
        emit(dict(what="solve", B=B, n=n, m=m, keep=keep, ms=solve[keep], problems_per_s=B / solve[keep] * 1e3))
    c_all, _ = h.info()
    c = float(c_all.mean())
    for k in (1, 16):
        V = ctx.array(np.random.default_rng(k).standard_normal(k * n))
        O = ctx.empty(B * k * n)
        for inverse in (0, 1):
            h.times(inverse, 0, B, k, V, n, 0, O, n, k * n)   # warm-up
            ms = timed(ctx, lambda: h.times(inverse, 0, B, k, V, n, 0, O, n, k * n))
            nbytes = B * 8 * n * (4 * c + 3 * k)
            emit(dict(what="products", op="H" if inverse else "B", B=B, n=n, m=m, k=k, mean_c=c, ms=ms, problems_per_s=B / ms * 1e3,
                      GB_per_s=nbytes / ms / 1e6, share_of_hbm_peak=nbytes / (ms * 1e-3) / PEAK))


def dense(ctx, emit):
    B, n, m = 1024, 256, 10
    prm = lb.LBFGSParam(m=m, max_iterations=100)
    h = lb.SmallHistory(ctx, n, m, B)
    X = ctx.array(np.random.default_rng(1).uniform(-1.2, 1.2, B * n))
    h.minimize(lb.OBJ_ROSENBROCK_PAIRED, X, prm, "MoreThuente")
    I = ctx.array(np.eye(n).reshape(-1))
    O = ctx.empty(B * n * n)
    h.times(1, 0, B, n, I, n, 0, O, n, n * n)
    ms = timed(ctx, lambda: h.times(1, 0, B, n, I, n, 0, O, n, n * n))
    emit(dict(what="dense H", B=B, n=n, m=m, ms=ms, matrices_per_s=B / ms * 1e3, GB_written_per_s=B * n * n * 8 / ms / 1e6))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also append the JSON lines to DIR/small_batch_hessian_bench.jsonl")
    ap.add_argument("--quick", action="store_true", help="small sizes (a check that the script runs, not a measurement)")
    args = ap.parse_args()
    lines = []

    def emit(d):
        lines.append(json.dumps(d))
        print(lines[-1], flush=True)
    emit(dict(card=card()))
    ctx = lb.Context(0)
    if args.quick:
        run(ctx, 256, 64, 10, emit)
    else:
        run(ctx, 65536, 256, 10, emit)
        run(ctx, 1024, lb.small_max_n(10, lb.OBJ_ROSENBROCK_PAIRED), 10, emit)
        dense(ctx, emit)
    ctx.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "small_batch_hessian_bench.jsonl"), "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
