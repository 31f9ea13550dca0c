"""Generate tests/golden/c3_full.json, c4_full.json, c5_full.json: BASELINE configs 3, 4 and 5 at their stated sizes, run on
the CPU by the unmodified reference headers (oracle/_ref, built over minieigen: sequential sums) and by the restatement
(oracle/liboracle.so) under three summation orders (sequential = what _ref does, 8-lane partial sums = what an AVX-512 Eigen
redux does, and the Gram-form twin of apply_Hv with 8-lane sums = the GPU's re-association).  The spread BETWEEN the CPU
columns is what a different reduction order does to the reference itself; the GPU tests hold the H100 to these tables.

Run from the repo root (needs oracle/_ref: make -C oracle ref REF=<LBFGSpp checkout>):
    python tests/golden/make_fullsize.py [c3] [c4] [c5] [--procs 7]
C5 is 64 solves of 150-260 iterations at n = 1e6 in each of four CPU variants: about 15 minutes on 7 cores.
Floats are stored as hex strings.
"""
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import pyoracle as po  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
N = 1_000_000


def hx(v):
    return float(v).hex()


def summarize(r, xs=None, keep_trace=False):
    out = dict(status=r["status"], msg=r["msg"], niter=int(r["niter"]), nfev=int(r["nfev"]), fx=hx(r["fx"]), gnorm=hx(r["gnorm"]),
               seconds=r["seconds"], x_absmax=hx(np.max(np.abs(r["x"]))), x_sum=hx(np.sum(r["x"])))
    if xs is not None:
        out["x_err_inf"] = hx(np.max(np.abs(r["x"] - xs)))
    if keep_trace:
        out["trace"] = [hx(v) for v in r["trace"]]
    return out


def variants():
    """(name, library, kwargs) of the CPU columns."""
    return [("ref_headers", "ref", dict()),
            ("restatement_sequential", "orc", dict(sum_mode=po.SUM_SEQUENTIAL)),
            ("restatement_lanes8", "orc", dict(sum_mode=po.SUM_LANES8)),
            ("restatement_gram_lanes8", "orc", dict(sum_mode=po.SUM_LANES8, gram=True))]


# ----------------------------------------------------------------------------------------------------------------- C3
def c3_one(v):
    name, lib, kw = v
    orc = po.Oracle(lib)
    d, b, xs = po.quad_tridiag_data(N, kappa=1e3, seed=0)
    prm = orc.default_param(m=20)
    r = orc.lbfgs(po.OBJ_QUAD_TRIDIAG, np.zeros(N), po.LS_BRACKETING, prm, data0=d, data1=b, **kw)
    return name, summarize(r, xs, keep_trace=True)


def make_c3(pool):
    cols = dict(pool.map(c3_one, variants()))
    out = dict(config="C3: f = 1/2 x'Ax - b'x, A = diag(d) + 1/2 tridiag(-1,2,-1), d = exp(U[0,ln 1e3]) seed 0, x* ~ N(0,1) seed 0 "
                      "(pyoracle.quad_tridiag_data), n = 1e6, m = 20, LineSearchBracketing, x0 = 0, LBFGSParam defaults otherwise",
               n=N, m=20, linesearch="Bracketing", columns=cols)
    with open(os.path.join(GOLD, "c3_full.json"), "w") as fh:
        json.dump(out, fh, indent=1)
    for k, v in cols.items():
        print("C3", k, v["status"], v["niter"], v["nfev"], float.fromhex(v["fx"]), v["msg"])


# ----------------------------------------------------------------------------------------------------------------- C4
def c4_one(args):
    (name, lib, kw), kind, eps_rel = args
    if kw.get("gram"):
        return None
    orc = po.Oracle(lib)
    over = {} if eps_rel is None else dict(epsilon_rel=eps_rel)
    prm = orc.default_param(lbfgsb=True, **over)
    r = orc.lbfgsb(kind, np.full(N, 3.0), 2.0, 4.0, prm, sum_mode=kw.get("sum_mode", po.SUM_SEQUENTIAL))
    s = summarize(r, keep_trace=True)
    x = r["x"]
    s["n_at_lb"] = int(np.sum(x == 2.0))
    s["n_at_ub"] = int(np.sum(x == 4.0))
    s["x_head"] = [hx(v) for v in x[:8]]
    s["x_tail"] = [hx(v) for v in x[-8:]]
    return ("%s|%d|%s" % (name, kind, "default" if eps_rel is None else "epsrel0"), s)


def make_c4(pool):
    jobs = [(v, kind, e) for v in variants() for kind in (po.OBJ_ROSENBROCK_PAIRED, po.OBJ_ROSENBROCK_CHAINED) for e in (None, 0.0)]
    res = [r for r in pool.map(c4_one, jobs) if r is not None]
    runs = {}
    for key, s in res:
        name, kind, tag = key.split("|")
        runs.setdefault("paired" if int(kind) == po.OBJ_ROSENBROCK_PAIRED else "chained", {}).setdefault(tag, {})[name] = s
    out = dict(config="C4: Rosenbrock-box, both readings (SURVEY.md 8d): paired (README) and chained (example-rosenbrock-box.cpp) "
                      "objective, n = 1e6, lb = 2, ub = 4, x0 = 3, LBFGSBParam defaults; 'epsrel0' = the same with epsilon_rel = 0",
               n=N, runs=runs)
    with open(os.path.join(GOLD, "c4_full.json"), "w") as fh:
        json.dump(out, fh, indent=1)
    for obj, tags in runs.items():
        for tag, cols in tags.items():
            for k, v in cols.items():
                print("C4", obj, tag, k, v["status"], v["niter"], v["nfev"], float.fromhex(v["fx"]))


# ----------------------------------------------------------------------------------------------------------------- C5
def c5_one(args):
    (name, lib, kw), b = args
    orc = po.Oracle(lib)
    x0 = np.random.default_rng(1000 + b).uniform(-1, 1, N)
    r = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, po.LS_MORE_THUENTE, orc.default_param(m=10), **kw)
    s = summarize(r, np.ones(N))
    return name, b, s


def make_c5(pool, B=64):
    jobs = [(v, b) for b in range(B) for v in variants()]
    rows = {}
    for name, b, s in pool.imap_unordered(c5_one, jobs):
        rows.setdefault(b, {})[name] = s
        print("C5 seed", 1000 + b, name, s["status"], s["niter"], s["nfev"], float.fromhex(s["fx"]), flush=True)
    out = dict(config="C5: B = 64 independent paired Rosenbrock problems, n = 1e6, m = 10, LineSearchMoreThuente, "
                      "x0_b ~ U[-1,1] from numpy default_rng(1000 + b)", n=N, m=10, B=B,
               problems=[dict(seed=1000 + b, columns=rows[b]) for b in range(B)])
    with open(os.path.join(GOLD, "c5_full.json"), "w") as fh:
        json.dump(out, fh, indent=1)


if __name__ == "__main__":
    which = [a for a in sys.argv[1:] if a in ("c3", "c4", "c5")] or ["c3", "c4", "c5"]
    procs = int(sys.argv[sys.argv.index("--procs") + 1]) if "--procs" in sys.argv else 7
    with Pool(procs) as pool:
        if "c3" in which:
            make_c3(pool)
        if "c4" in which:
            make_c4(pool)
        if "c5" in which:
            make_c5(pool)
