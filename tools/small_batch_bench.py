"""Throughput of the small-batch solve (LBFGSSmallBatchSolver: one thread block per problem) against the device-resident batch
(LBFGSBatchSolver: every pass of a problem spread over all SMs, B <= 4096) and the CPU checker on one core.

Workloads (paired Rosenbrock, fp64):
  selfcheck   the reference's self-checks: n = 2, 4, .., 24, 1024 random starts each, all four line searches, max_linesearch = 256
  n256        B = 65 536 random starts at n = 256, m = 10, More-Thuente (LBFGSBatchSolver: the first 4096)
  maxn        B = 1024 random starts at n = lbfgs_b200_small_max_n(m = 10), More-Thuente
For each: problems/s and iterations/s per path.  Device time comes from CUDA events (lbfgs_b200_timer_start / stop on the context's
stream) around each solve call, best of three runs that alternate the two GPU paths; the checker's time is its wall clock on a
subset of the problems.  The outputs are compared: status, iterations and the distance to x* = 1 of every path, and each GPU path's
fx against the checker's on the checked subset.  The card's name and power limit are read in the same run.

  python tools/small_batch_bench.py [--workloads selfcheck,n256,maxn] [--cpu-problems K] [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import lbfgspp_b200 as lb  # noqa: E402

LS = ["Backtracking", "Bracketing", "NocedalWright", "MoreThuente"]
MAXIT = 10000


class Param(C.Structure):   # lbfgs_b200_param
    _fields_ = [("m", C.c_int), ("epsilon", C.c_double), ("epsilon_rel", C.c_double), ("past", C.c_int), ("delta", C.c_double),
                ("max_iterations", C.c_int), ("linesearch", C.c_int), ("max_linesearch", C.c_int), ("min_step", C.c_double),
                ("max_step", C.c_double), ("ftol", C.c_double), ("wolfe", C.c_double)]


class Outcome(C.Structure):  # lbfgs_b200_outcome
    _fields_ = [("status", C.c_int), ("niter", C.c_int), ("nfev", C.c_longlong), ("fx", C.c_double), ("gnorm", C.c_double),
                ("rounds", C.c_longlong)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm_max = [s.strip() for s in q.split(",")]
        return dict(name=name, power_limit=power, sm_clock_max=sm_max)
    except Exception as e:   # the measurement itself does not depend on it
        return dict(error=str(e))


def summary(status, niter, X):
    ok = status == 0
    return dict(ok=int(ok.sum()), problems=int(len(status)), mean_niter=float(niter.mean()),
                max_err=float(np.max(np.abs(X[ok] - 1.0))) if ok.any() else None)


class GpuPaths:
    """Both GPU paths on one context, timed with CUDA events on its stream"""

    def __init__(self, ctx):
        self.ctx, self.lib = ctx, ctx.lib

    def small(self, X0, m, ls, max_linesearch):
        B, n = X0.shape
        p = Param(m, 1e-5, 1e-5, 0, 0.0, MAXIT, 3, max_linesearch, 1e-20, 1e20, 1e-4, 0.9)
        X = self.ctx.array(X0.reshape(-1))
        outs = (Outcome * B)()
        self.ctx.timer_start()
        self.ctx.check(self.lib.lbfgs_b200_small_minimize_f64(self.ctx.h, lb.OBJ_ROSENBROCK_PAIRED, None, None, 0, n, B, C.byref(p),
                                                              LS.index(ls), X.ptr, n, None, outs))
        ms = self.ctx.timer_stop()
        return ms, outs, X.get().reshape(B, n)

    def batch(self, X0, m, ls, max_linesearch):
        B, n = X0.shape
        p = Param(m, 1e-5, 1e-5, 0, 0.0, MAXIT, 3, max_linesearch, 1e-20, 1e20, 1e-4, 0.9)
        s = C.c_void_p()
        self.ctx.check(self.lib.lbfgs_b200_solver_create_batch(self.ctx.h, n, m, 8, B, C.byref(s)))
        try:
            X = self.ctx.array(X0.reshape(-1))
            outs = (Outcome * B)()
            self.ctx.timer_start()
            self.ctx.check(self.lib.lbfgs_b200_solver_minimize_batch_f64(s, lb.OBJ_ROSENBROCK_PAIRED, None, None, 0, C.byref(p),
                                                                        LS.index(ls), X.ptr, n, outs))
            ms = self.ctx.timer_stop()
            return ms, outs, X.get().reshape(B, n)
        finally:
            self.lib.lbfgs_b200_solver_destroy(s)


def arrays(outs):
    return (np.array([o.status for o in outs]), np.array([o.niter for o in outs]), np.array([o.fx for o in outs]))


def run_group(gpu, orc, groups, m, max_linesearch, cpu_problems, batch_cap=4096):
    """groups: list of (ls, X0).  Returns rates and checks of the three paths summed over the groups."""
    import pyoracle as po
    tot = {k: dict(ms=0.0, problems=0, iters=0) for k in ("small", "batch", "cpu")}
    checks = []
    for ls, X0 in groups:
        Xb0 = X0[:batch_cap]
        best = {"small": None, "batch": None}
        for _ in range(3):   # best of three, the two GPU paths alternating
            for key, fn, Xin in (("small", gpu.small, X0), ("batch", gpu.batch, Xb0)):
                r = fn(Xin, m, ls, max_linesearch)
                if best[key] is None or r[0] < best[key][0]:
                    best[key] = r
        (ms_s, outs_s, Xs), (ms_b, outs_b, Xb) = best["small"], best["batch"]
        st_s, it_s, fx_s = arrays(outs_s)
        st_b, it_b, fx_b = arrays(outs_b)
        tot["small"]["ms"] += ms_s; tot["small"]["problems"] += len(X0); tot["small"]["iters"] += int(it_s.sum())
        tot["batch"]["ms"] += ms_b; tot["batch"]["problems"] += len(Xb0); tot["batch"]["iters"] += int(it_b.sum())
        # the CPU checker, one core, on the first cpu_problems starts
        k = min(cpu_problems, len(X0))
        cprm = orc.default_param(m=m, max_linesearch=max_linesearch, max_iterations=MAXIT)
        t0 = time.perf_counter()
        cres = [orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, X0[b], LS.index(ls), cprm, trace_cap=1) for b in range(k)]
        tot["cpu"]["ms"] += 1e3 * (time.perf_counter() - t0); tot["cpu"]["problems"] += k
        tot["cpu"]["iters"] += sum(c["niter"] for c in cres)
        fx_c = np.array([c["fx"] for c in cres])
        it_c = np.array([c["niter"] for c in cres])
        kb = min(k, len(Xb0))
        checks.append(dict(ls=ls, n=X0.shape[1], small=summary(st_s, it_s, Xs), batch=summary(st_b, it_b, Xb),
                           cpu_ok=int(sum(c["status"] == "ok" for c in cres)), cpu_mean_niter=float(it_c.mean()),
                           small_vs_cpu_max_dfx=float(np.max(np.abs(fx_s[:k] - fx_c))),
                           batch_vs_cpu_max_dfx=float(np.max(np.abs(fx_b[:kb] - fx_c[:kb]))),
                           small_vs_batch_max_dx=float(np.max(np.abs(Xs[:len(Xb0)] - Xb))),
                           small_vs_batch_same_niter=float(np.mean(it_s[:len(Xb0)] == it_b))))
    rates = {k: dict(problems_per_s=v["problems"] / (v["ms"] / 1e3), iterations_per_s=v["iters"] / (v["ms"] / 1e3), ms=v["ms"],
                     problems=v["problems"]) for k, v in tot.items()}
    return dict(rates=rates, checks=checks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="selfcheck,n256,maxn")
    ap.add_argument("--cpu-problems", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import pyoracle as po
    orc = po.Oracle("orc")
    ctx = lb.Context(0)
    gpu = GpuPaths(ctx)
    out = dict(card=card(), workloads={})
    # warm-up of every kernel shape the timed runs use
    for ls in LS:
        gpu.small(np.zeros((4, 24)), 6, ls, 256)
        gpu.batch(np.zeros((4, 24)), 6, ls, 256)
    for w in a.workloads.split(","):
        if w == "selfcheck":
            groups = [(ls, np.random.default_rng(4000 + n).uniform(-1, 1, (1024, n))) for n in range(2, 25, 2) for ls in LS]
            out["workloads"][w] = run_group(gpu, orc, groups, 6, 256, a.cpu_problems)
        elif w == "n256":
            out["workloads"][w] = run_group(gpu, orc, [("MoreThuente", np.random.default_rng(7).uniform(-1, 1, (65536, 256)))], 10, 20,
                                            a.cpu_problems)
        elif w == "maxn":
            n = lb.small_max_n(10, lb.OBJ_ROSENBROCK_PAIRED)
            out["workloads"][w] = run_group(gpu, orc, [("MoreThuente", np.random.default_rng(8).uniform(-1, 1, (1024, n)))], 10, 20,
                                            a.cpu_problems)
            out["workloads"][w]["n"] = n
        print(json.dumps({w: out["workloads"][w]["rates"]}), flush=True)
    print(json.dumps(out["card"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
