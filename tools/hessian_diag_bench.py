"""Time the diagonals of the final L-BFGS approximation on the GPU (CUDA events over at least --min-seconds of device time per figure,
best of three).

    python tools/hessian_diag_bench.py [--min-seconds S] [--out DIR] [--quick]

Workloads:
  - large n: lbfgs_b200_hist_quad_diag on a full fp64 ring of n = 1e7 at m = c = 10, 20 and 64 -- the pass behind
    LBFGSSolver::final_approx_hessian_diagonal and final_approx_inverse_hessian_diagonal (both run the same pass; only the 2c x 2c
    host algebra that forms K differs, and it is not in these figures);
  - small batch: lbfgs_b200_small_hist_diag on B = 65 536 problems of n = 256 and on B = 1024 of n = small_max_n(10) = 1016, m = 10, after
    a kept More-Thuente solve, for B and H; and the only route there was before it, lbfgs_b200_small_hist_times with the columns of I
    (V shared, k = n) keeping entry i of product i, on a slice of problems whose n x n outputs fit in memory, per problem.
Each figure: ms, GB/s of the w*n*(2c + 1) bytes a diagonal needs (the 2c history columns read once, the result written once), and its
share of the bound that applies by the H100 SXM data sheet: 3.35 TB/s of HBM, or 2c^2 + 3c fp64 multiply-adds per element at 34 TFLOP/s
(17e12 fused multiply-adds/s).  The card's name, power limit and SM clock are read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lbfgspp_b200 as lb  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12   # H100 SXM HBM3, NVIDIA data sheet
PEAK_FMA_PER_S = 17e12       # H100 SXM FP64 (non-tensor) 34 TFLOP/s, NVIDIA data sheet


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [s.strip() for s in q.split(",")]
        return dict(name=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
    except Exception as e:   # the measurement itself does not depend on it
        return dict(error=str(e))


def timed(ctx, fn, min_seconds):
    """ms per call of fn(), best of three batches that each last at least min_seconds of device time"""
    fn()
    calls = 1
    while True:
        ctx.timer_start()
        for _ in range(calls):
            fn()
        ms = ctx.timer_stop()
        if ms >= 1e3 * min_seconds:
            break
        calls = max(calls * 2, int(calls * 1.2 * 1e3 * min_seconds / max(ms, 1e-3)))
    best = ms / calls
    for _ in range(2):
        ctx.timer_start()
        for _ in range(calls):
            fn()
        best = min(best, ctx.timer_stop() / calls)
    return best


def rates(n_elems, c, ms, w=8):
    nbytes = w * n_elems * (2 * c + 1)
    fmas = n_elems * (2 * c * c + 3 * c)
    t_bytes, t_fma = nbytes / PEAK_BYTES_PER_S, fmas / PEAK_FMA_PER_S
    bound = "hbm" if t_bytes >= t_fma else "fp64"
    return dict(GB_per_s=nbytes / ms / 1e6, bound=bound, share_of_bound=max(t_bytes, t_fma) / (ms * 1e-3))


def large(ctx, n, m, min_seconds, emit):
    h = lb.History(ctx, n, m)
    rng = np.random.default_rng(m)
    base = rng.standard_normal(n)
    for k in range(m):
        s = base * (1.0 + 0.01 * k) + 0.1 * rng.standard_normal(n)
        h.add(ctx.array(s), ctx.array(1.5 * s))
    c = h.ncorr
    A = rng.standard_normal((2 * c, 2 * c))
    out = ctx.empty(n)
    for label in ("B", "H"):
        K = (A + A.T) / 2
        ms = timed(ctx, lambda: h.quad_diag(1.0, K, out), min_seconds)
        emit(dict(what="large-n diagonal pass", op=label, n=n, m=m, c=c, ms=ms, **rates(n, c, ms)))
        A = rng.standard_normal((2 * c, 2 * c))


def small(ctx, B, n, m, slice_B, min_seconds, emit):
    prm = lb.LBFGSParam(m=m, max_iterations=100)
    h = lb.SmallHistory(ctx, n, m, B)
    X = ctx.array(np.random.default_rng(0).uniform(-1.2, 1.2, B * n))
    h.minimize(lb.OBJ_ROSENBROCK_PAIRED, X, prm, "MoreThuente")
    c_all, _ = h.info()
    c = float(c_all.mean())
    O = ctx.empty(B * n)
    I = ctx.array(np.eye(n).reshape(-1))
    OI = ctx.empty(slice_B * n * n)
    for inverse in (0, 1):
        op = "H" if inverse else "B"
        ms = timed(ctx, lambda: h.diagonal(inverse, 0, B, O, n), min_seconds)
        emit(dict(what="small-batch diagonal", op=op, B=B, n=n, m=m, mean_c=c, ms=ms, problems_per_s=B / ms * 1e3,
                  **rates(B * n, c, ms)))
        ms_old = timed(ctx, lambda: h.times(inverse, 0, slice_B, n, I, n, 0, OI, n, n * n), min_seconds)
        per_old, per_new = ms_old / slice_B, ms / B
        emit(dict(what="identity products (the route before)", op=op, problems=slice_B, n=n, m=m, ms=ms_old, ms_per_problem=per_old,
                  diagonal_ms_per_problem=per_new, speedup=per_old / per_new))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None, help="also append the JSON lines to DIR/hessian_diag_bench.jsonl")
    ap.add_argument("--quick", action="store_true", help="small sizes (a check that the script runs, not a measurement)")
    args = ap.parse_args()
    lines = []

    def emit(d):
        lines.append(json.dumps(d))
        print(lines[-1], flush=True)
    emit(dict(card=card()))
    ctx = lb.Context(0)
    if args.quick:
        large(ctx, 100_000, 10, 0.05, emit)
        small(ctx, 256, 64, 10, 16, 0.05, emit)
    else:
        for m in (10, 20, 64):
            large(ctx, 10_000_000, m, args.min_seconds, emit)
        small(ctx, 65536, 256, 10, 1024, args.min_seconds, emit)
        small(ctx, 1024, lb.small_max_n(10, lb.OBJ_ROSENBROCK_PAIRED), 10, 64, args.min_seconds, emit)
    emit(dict(card_after=card()))
    ctx.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "hessian_diag_bench.jsonl"), "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
