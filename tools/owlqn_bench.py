"""OWL-QN throughput on one GPU: OWLQNSolver (F = f + lam |x|_1, fused projected trial) against LBFGSSolver's host-driven loop on the
same smooth f (lam = 0, Backtracking), in one process, the two arms alternating.  Workloads: the tridiagonal quadratic (the C3 data
model: d_i = exp(U[0, ln 1e3]), b = A x*, x* ~ N(0, 1)) and paired Rosenbrock, n = 1e7, m = 10, fp64; lam makes the tridiagonal solution
sparse but not empty (every pair of paired Rosenbrock is the same problem, so its solution is all zero or all nonzero: lam = 1 keeps
it nonzero).  Both arms run the same number of iterations (--iters, both must reach it).

  it/s       iterations over the time of synchronised minimize() calls alone (x0 and the data already in HBM), summed over a window
             of repeated calls lasting at least --window seconds
  per phase  a separate profiled call: device time of the trial kernels and of the direction (pair-forming dots, the curvature gate's
             host read-back, combination) from CUDA events on the context's stream (lbfgs_b200_profile_*), and GB/s on the
             words-per-coordinate model the library records with each span (DESIGN.md §8h)
Prints one JSON line per workload.

--weights unit: the arms are instead OWLQNSolver(param, lam, w = 1) and OWLQNSolver(param, lam), which take the same iteration path
bit for bit (checked), so the difference is the cost of the weight vector: one more word per coordinate in the trial (6 against 5)
and in the direction (4c + 11 against 4c + 9).

    python tools/owlqn_bench.py [--n N] [--iters K] [--window S] [--reps R] [--weights unit]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lbfgspp_b200 as lb  # noqa: E402

PH_APPLY_HV, PH_TRIAL = 0, 1


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def tridiag_data(n, kappa=1e3, seed=0):
    rng = np.random.default_rng(seed)
    d = np.exp(rng.uniform(0.0, np.log(kappa), n))
    xs = rng.standard_normal(n)
    b = (d + 1.0) * xs - 0.5 * (np.concatenate(([0.0], xs[:-1])) + np.concatenate((xs[1:], [0.0])))
    return d, b


def window(run, seconds):
    """(iterations, minimize() seconds, last result) over repeated calls lasting at least `seconds` of minimize() time"""
    its, t, r = 0, 0.0, None
    while t < seconds:
        r = run()
        assert r["status"] == "ok", r["msg"]
        its += r["niter"]
        t += r["seconds"]
    return its, t, r


def profiled(lib, h, run):
    """device ms and algorithmic bytes per phase of one call"""
    scratch = C.c_double(0)
    for ph in (PH_APPLY_HV, PH_TRIAL):
        lib.lbfgs_b200_profile_read(h, ph, None, None, 1)
        lib.lbfgs_b200_profile_bytes(h, ph, C.byref(scratch), 1)
    lib.lbfgs_b200_profile_enable(h, 1)
    r = run()
    out = {}
    for name, ph in (("trial", PH_TRIAL), ("direction", PH_APPLY_HV)):
        ms, calls, nbytes = C.c_double(0), C.c_uint64(0), C.c_double(0)
        lib.lbfgs_b200_profile_read(h, ph, C.byref(ms), C.byref(calls), 1)
        lib.lbfgs_b200_profile_bytes(h, ph, C.byref(nbytes), 1)
        out[name] = dict(ms_per_call=ms.value / max(calls.value, 1), calls=calls.value,
                         gb_per_s=nbytes.value / (ms.value * 1e6) if ms.value > 0 else None)
    lib.lbfgs_b200_profile_enable(h, 0)
    return out, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--weights", choices=["unit"], default=None)
    a = ap.parse_args()
    n = a.n
    d0, d1 = tridiag_data(n)
    work = {
        "quad_tridiag": (lb.OBJ_QUAD_TRIDIAG, 0.5, d0, d1, np.zeros(n)),
        "rosenbrock_paired": (lb.OBJ_ROSENBROCK_PAIRED, 1.0, None, None, np.full(n, -1.2)),
    }
    drv = lb.driver()
    abi = lb.abi()
    h = C.c_void_p(drv.lbfgsb200_drv_ctx(0))
    info = card()
    for name, (obj, lam, d0, d1, x0) in work.items():
        prm = lb.LBFGSParam(m=10, epsilon=1e-30, epsilon_rel=0.0, max_iterations=a.iters)
        owl = lb.OWLQNSolver(prm, lam)
        if a.weights:
            owl_w = lb.OWLQNSolver(prm, lam, weights=np.ones(n))
            arms = {"owlqn": lambda: owl.minimize(obj, x0, d0, d1), "owlqn_w1": lambda: owl_w.minimize(obj, x0, d0, d1)}
        else:
            ref = lb.LBFGSSolver(prm, "Backtracking", resident=False)
            arms = {"owlqn": lambda: owl.minimize(obj, x0, d0, d1), "lbfgs_lam0": lambda: ref.minimize(obj, x0, d0, d1)}
        other = "owlqn_w1" if a.weights else "lbfgs_lam0"
        last = {k: run() for k, run in arms.items()}             # warm-up of both arms
        if a.weights:
            assert last["owlqn"]["fx"] == last["owlqn_w1"]["fx"] and np.array_equal(last["owlqn"]["x"], last["owlqn_w1"]["x"])
        rates = {k: [] for k in arms}
        for _ in range(a.reps):
            for k, run in arms.items():
                its, t, last[k] = window(run, a.window)
                rates[k].append(its / t)
        assert last["owlqn"]["niter"] == last[other]["niter"] == a.iters, "both arms must run --iters iterations"
        phases = {k: profiled(abi, h, run)[0] for k, run in arms.items()}
        print(json.dumps(dict(workload=name, n=n, m=10, lam=lam, card=info, iterations=a.iters, nfev_owlqn=last["owlqn"]["nfev"],
                              **{"nfev_w1" if a.weights else "nfev_lbfgs": last[other]["nfev"]}, nonzeros=int(np.count_nonzero(last["owlqn"]["x"])),
                              it_s={k: sorted(v) for k, v in rates.items()}, phases=phases)))


if __name__ == "__main__":
    main()
