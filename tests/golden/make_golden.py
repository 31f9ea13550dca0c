"""Generate tests/golden/lbfgs_ref.json from the UNMODIFIED reference headers (oracle/_ref, built over minieigen).

Needs oracle/_ref (make -C oracle ref REF=<LBFGSpp checkout>):   python tests/golden/make_golden.py
The reference ships no golden vectors of its own (SURVEY.md section 4); these freeze what its headers compute
(sequential summation, no FMA contraction) so that the travelling restatement can be checked on any machine.
Floats are stored as hex strings: comparisons are bit-exact.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import pyoracle as po  # noqa: E402

LS = {"Backtracking": 0, "Bracketing": 1, "NocedalWright": 2, "MoreThuente": 3}


def hx(a):
    return [float(v).hex() for v in np.atleast_1d(a)]


def main():
    ref = po.Oracle("ref")
    cases = []

    def lbfgs_case(name, objective, x0, ls, dtype="f64", data=None, **prm):
        p = ref.default_param(**prm)
        d0, d1 = (data if data else (None, None))
        r = ref.lbfgs(objective, x0, LS[ls], p, data0=d0, data1=d1, dtype=np.float64 if dtype == "f64" else np.float32)
        cases.append(dict(kind="lbfgs", name=name, objective=objective, ls=ls, dtype=dtype, x0=hx(x0), param=prm,
                          data=None if not data else [hx(d0), hx(d1)],
                          status=r["status"], msg=r["msg"], niter=r["niter"], nfev=r["nfev"], fx=float(r["fx"]).hex(),
                          gnorm=float(r["gnorm"]).hex(), trace=hx(r["trace"]), x=hx(r["x"]), grad=hx(r["grad"])))

    # config C1: example-rosenbrock.cpp with float -> double, default parameters, all four line searches
    for ls in LS:
        lbfgs_case("C1_rosenbrock_n10_" + ls, po.OBJ_ROSENBROCK_PAIRED, np.zeros(10), ls)
        lbfgs_case("C1f_rosenbrock_n10_f32_" + ls, po.OBJ_ROSENBROCK_PAIRED, np.zeros(10), ls, dtype="f32")
    # README parameters (epsilon 1e-6, max_iterations 100)
    lbfgs_case("readme_rosenbrock_n10", po.OBJ_ROSENBROCK_PAIRED, np.zeros(10), "NocedalWright", epsilon=1e-6, max_iterations=100)
    lbfgs_case("readme_rosenbrock_n10_epsrel0", po.OBJ_ROSENBROCK_PAIRED, np.zeros(10), "NocedalWright", epsilon=1e-6,
               epsilon_rel=0.0, max_iterations=100)
    # example-quadratic.cpp
    lbfgs_case("quadratic_n10", po.OBJ_QUAD_SHIFT, np.zeros(10), "NocedalWright")
    # random starts (the two self-checking examples' pattern), seeded here
    rng = np.random.default_rng(20260923)
    for n in (2, 6, 16, 24):
        for ls in LS:
            x0 = rng.uniform(-1, 1, n)
            lbfgs_case("rand_n%d_%s" % (n, ls), po.OBJ_ROSENBROCK_PAIRED, x0, ls, max_linesearch=256)
    # m = 10 MoreThuente at moderate n (config C2's shape), Armijo / Wolfe variants, past/delta, max_iterations
    lbfgs_case("C2small_rosenbrock_n1000_MT_m10", po.OBJ_ROSENBROCK_PAIRED, np.zeros(1000), "MoreThuente", m=10)
    lbfgs_case("armijo_BT", po.OBJ_ROSENBROCK_PAIRED, rng.uniform(-1, 1, 8), "Backtracking", linesearch=1, max_linesearch=64)
    lbfgs_case("wolfe_BR", po.OBJ_ROSENBROCK_PAIRED, rng.uniform(-1, 1, 8), "Bracketing", linesearch=2, max_linesearch=64)
    lbfgs_case("past_delta", po.OBJ_ROSENBROCK_PAIRED, np.zeros(12), "MoreThuente", past=3, delta=1e-6)
    lbfgs_case("maxiter5", po.OBJ_ROSENBROCK_PAIRED, np.zeros(12), "NocedalWright", max_iterations=5)
    # config C3's objective at small n
    d, b, _ = po.quad_tridiag_data(500, kappa=1e3, seed=0)
    lbfgs_case("C3small_quad_tridiag_n500_BR_m20", po.OBJ_QUAD_TRIDIAG, np.zeros(500), "Bracketing", data=(d, b), m=20)
    lbfgs_case("chained_rosenbrock_n50_MT", po.OBJ_ROSENBROCK_CHAINED, np.full(50, 3.0), "MoreThuente")
    # error paths
    lbfgs_case("err_bad_m", po.OBJ_ROSENBROCK_PAIRED, np.zeros(4), "NocedalWright", m=0)
    lbfgs_case("err_bad_ftol", po.OBJ_ROSENBROCK_PAIRED, np.zeros(4), "NocedalWright", ftol=0.6)
    lbfgs_case("err_nw_needs_strong_wolfe", po.OBJ_ROSENBROCK_PAIRED, np.zeros(4), "NocedalWright", linesearch=1)
    lbfgs_case("err_bt_budget", po.OBJ_ROSENBROCK_PAIRED, np.zeros(4), "Backtracking", max_linesearch=1)
    lbfgs_case("err_br_budget", po.OBJ_ROSENBROCK_PAIRED, np.zeros(4), "Bracketing", max_linesearch=1)
    lbfgs_case("mt_budget_returns_best", po.OBJ_ROSENBROCK_PAIRED, np.zeros(4), "MoreThuente", max_linesearch=1, max_iterations=3)
    lbfgs_case("nw_budget", po.OBJ_ROSENBROCK_PAIRED, np.zeros(4), "NocedalWright", max_linesearch=1, max_iterations=3)

    # BFGSMat::apply_Hv on explicit histories (ring wrap-around, c in {0,1,m-1,m})
    for n, m, npairs in ((7, 3, 0), (7, 3, 1), (7, 3, 2), (7, 3, 3), (7, 3, 8), (130, 6, 6), (130, 6, 17)):
        S = rng.standard_normal((npairs, n))
        Y = S + 0.1 * rng.standard_normal((npairs, n))
        v = rng.standard_normal(n)
        res, _, theta = ref.apply_Hv(S, Y, v, -1.0, m)
        cases.append(dict(kind="apply_Hv", name="hv_n%d_m%d_p%d" % (n, m, npairs), n=n, m=m, npairs=npairs, a=-1.0,
                          S=hx(S.ravel()), Y=hx(Y.ravel()), v=hx(v), res=hx(res), theta=float(theta).hex()))

    # LBFGSBSolver (config C4 shape, small n): example-rosenbrock-box.cpp and the README box example
    def lbfgsb_case(name, objective, x0, lb, ub, **prm):
        p = ref.default_param(lbfgsb=True, **prm)
        r = ref.lbfgsb(objective, x0, lb, ub, p)
        cases.append(dict(kind="lbfgsb", name=name, objective=objective, x0=hx(x0), lb=hx(np.broadcast_to(lb, x0.size)),
                          ub=hx(np.broadcast_to(ub, x0.size)), param=prm, status=r["status"], msg=r["msg"],
                          niter=r["niter"], nfev=r["nfev"], fx=float(r["fx"]).hex(), gnorm=float(r["gnorm"]).hex(),
                          trace=hx(r["trace"]), x=hx(r["x"]), grad=hx(r["grad"])))

    x0 = np.full(25, 3.0)
    x0[[0, 1]] = 2.0
    x0[[5, 7]] = 4.0
    lb = np.full(25, 2.0)
    ub = np.full(25, 4.0)
    lb[2], ub[2] = -np.inf, np.inf
    lbfgsb_case("box_example_chained_n25", po.OBJ_ROSENBROCK_CHAINED, x0, lb, ub)
    lbfgsb_case("box_readme_paired_n10", po.OBJ_ROSENBROCK_PAIRED, np.full(10, 3.0), 2.0, 4.0, epsilon=1e-6, max_iterations=100)
    lbfgsb_case("box_paired_n200", po.OBJ_ROSENBROCK_PAIRED, np.full(200, 3.0), 2.0, 4.0)
    lbfgsb_case("box_chained_n200", po.OBJ_ROSENBROCK_CHAINED, np.full(200, 3.0), 2.0, 4.0)
    lbfgsb_case("box_loose_paired_n40", po.OBJ_ROSENBROCK_PAIRED, rng.uniform(-1, 1, 40), -0.5, 0.8)

    out = os.path.join(HERE, "lbfgs_ref.json")
    with open(out, "w") as fh:
        json.dump(dict(generator="tests/golden/make_golden.py", source="oracle/_ref (unmodified reference headers @ ebef584 over oracle/minieigen)",
                       cases=cases), fh, indent=0)
    print("wrote", out, len(cases), "cases,", os.path.getsize(out) // 1024, "KiB")


if __name__ == "__main__":
    main()
