"""GPU parity tests for the bound-constrained solver (BASELINE config 4) against the reference headers' outputs:
the frozen golden vectors (tests/golden/lbfgs_ref.json, kind "lbfgsb"), and live runs of the restatement
(oracle/lbfgsb_oracle.hpp, pinned bit for bit to oracle/_ref by tests/test_oracle_cpu.py).  Parity: same iteration count, evaluation count within +-1 on the short runs (the
Cauchy sweep and the BOXCQP solves re-associate sums), |fx - fx_ref| <= 1e-9 max(1,|fx_ref|), |x - x_ref|_inf <= 1e-6."""
import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po
from util import golden_cases, unhex

pytestmark = pytest.mark.gpu


def check(g, c_status, c_niter, c_nfev, c_fx, c_x, iter_slack=0):
    assert g["status"] == c_status, (g["status"], g["msg"])
    assert abs(g["niter"] - c_niter) <= iter_slack, (g["niter"], c_niter)
    assert abs(g["nfev"] - c_nfev) <= iter_slack + 1, (g["nfev"], c_nfev)
    assert abs(g["fx"] - c_fx) <= 1e-9 * max(1.0, abs(c_fx)), (g["fx"], c_fx)
    assert np.max(np.abs(g["x"] - c_x)) <= 1e-6 * max(1.0, np.max(np.abs(c_x)))


@pytest.mark.parametrize("case", golden_cases("lbfgsb"), ids=lambda c: c["name"])
def test_lbfgsb_golden_vectors(case):
    prm = lb.LBFGSBParam(**case["param"])
    g = lb.LBFGSBSolver(prm).minimize(case["objective"], unhex(case["x0"]), unhex(case["lb"]), unhex(case["ub"]))
    check(g, case["status"], case["niter"], case["nfev"], float.fromhex(case["fx"]), unhex(case["x"]),
          iter_slack=0 if case["niter"] < 20 else 2)
    lbv, ubv = unhex(case["lb"]), unhex(case["ub"])
    assert np.all(g["x"] >= lbv) and np.all(g["x"] <= ubv)


@pytest.mark.parametrize("kind,n", [(lb.OBJ_ROSENBROCK_PAIRED, 1000), (lb.OBJ_ROSENBROCK_CHAINED, 1000),
                                    (lb.OBJ_ROSENBROCK_PAIRED, 100000), (lb.OBJ_ROSENBROCK_CHAINED, 100000)])
def test_config4_shape_box_2_4(orc, kind, n):
    """BASELINE config 4 (both readings of 'Rosenbrock-box', SURVEY.md 8d): lb = 2, ub = 4, x0 = 3."""
    x0 = np.full(n, 3.0)
    g = lb.LBFGSBSolver(lb.LBFGSBParam()).minimize(kind, x0, 2.0, 4.0)
    c = orc.lbfgsb(kind, x0, 2.0, 4.0, orc.default_param(lbfgsb=True))
    check(g, c["status"], c["niter"], c["nfev"], c["fx"], c["x"])


def test_box_random_interior_and_loose_bounds(orc):
    rng = np.random.default_rng(4)
    n = 5000
    x0 = rng.uniform(-1, 1, n)
    lbv = np.full(n, -0.5)
    ubv = np.full(n, 0.8)
    lbv[::7] = -np.inf
    ubv[::11] = np.inf
    g = lb.LBFGSBSolver(lb.LBFGSBParam()).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0, lbv, ubv)
    c = orc.lbfgsb(po.OBJ_ROSENBROCK_PAIRED, x0, lbv, ubv, orc.default_param(lbfgsb=True))
    assert g["status"] == c["status"] == "ok"
    assert abs(g["fx"] - c["fx"]) <= 1e-6 * max(1.0, abs(c["fx"]))
    assert np.all(g["x"] >= lbv) and np.all(g["x"] <= ubv)


def test_bounds_size_mismatch_is_invalid_argument():
    ctx_err = lb.LBFGSBSolver(lb.LBFGSBParam(m=0)).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.full(4, 3.0), 2.0, 4.0)
    assert ctx_err["status"] == "invalid_argument" and "'m' must be positive" in ctx_err["msg"]


# ---- kernel level: the parallel (sort + prefix-sum) Cauchy sweep against the reference's sequential sweep ------------------
def cauchy_sequential(S, Y, x0, g, lb, ub, m):
    """numpy restatement of Cauchy<Scalar>::get_cauchy_point (reference Cauchy.h:86-284) with a dense M; ring of size m."""
    S, Y = S[-m:], Y[-m:]
    c, n = S.shape[0], x0.size
    theta = 1.0
    W = np.zeros((n, 0))
    M = np.zeros((0, 0))
    if c:
        theta = float(Y[-1] @ Y[-1]) / float(S[-1] @ Y[-1])
        SY = S @ Y.T
        L = np.tril(SY, -1)                      # chronological order: row i newer than column j
        Minv = np.block([[-np.diag(np.diag(SY)), L.T], [L, theta * (S @ S.T)]])
        M = np.linalg.inv(Minv)
        W = np.hstack([Y.T, theta * S.T])
    brk = np.full(n, np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        brk = np.where(lb == ub, 0.0, np.where(g < 0, (x0 - ub) / g, np.where(g > 0, (x0 - lb) / g, np.inf)))
    d = np.where(brk == 0, 0.0, -g)
    free_inf = np.where(brk == np.inf)[0]
    ordv = np.where((brk != np.inf) & (brk != 0))[0]
    ordv = ordv[np.argsort(brk[ordv], kind="stable")]
    xcp = x0.copy()
    act = np.zeros(n, bool)
    if len(free_inf) == 0 and len(ordv) == 0:
        return xcp, act, np.zeros(2 * c)
    p = W.T @ d
    vc = np.zeros(2 * c)
    fp = -d @ d
    fpp = -theta * fp - p @ (M @ p)
    dtmin = -fp / fpp
    il, b = 0.0, 0
    iu = brk[ordv[0]] if len(ordv) else np.inf
    dt = iu - il
    crossed_all = False
    while dtmin >= dt:
        vc = vc + dt * p
        e = b
        while e < len(ordv) and brk[ordv[e]] <= iu:
            e += 1
        group = ordv[b:e]
        if len(free_inf) == 0 and e == len(ordv):
            xcp[group] = np.where(d[group] > 0, ub[group], lb[group])
            act[group] = True
            crossed_all = True
            break
        fp += dt * fpp
        for a in group:
            xcp[a] = ub[a] if d[a] > 0 else lb[a]
            z, ga = xcp[a] - x0[a], g[a]
            w = W[a]
            Mw = M @ w
            fp += ga * ga + theta * ga * z - ga * (Mw @ vc)
            fpp -= theta * ga * ga + 2 * ga * (Mw @ p) + ga * ga * (Mw @ w)
            p = p + ga * w
            d[a] = 0.0
            act[a] = True
        dtmin = -fp / fpp
        il, b = iu, e
        if b >= len(ordv):
            break
        iu = brk[ordv[b]]
        dt = iu - il
    if not crossed_all:
        if fpp < np.finfo(float).eps:
            dtmin = -fp / np.finfo(float).eps
        dtmin = max(dtmin, 0.0)
        vc = vc + dtmin * p
        tf = il + dtmin
        rest = np.concatenate([free_inf, ordv[b:]]).astype(int)
        xcp[rest] = x0[rest] + tf * d[rest]
    return xcp, act, vc


@pytest.mark.parametrize("n,m,npairs,seed", [(50, 4, 0, 0), (200, 4, 3, 1), (2000, 6, 6, 2), (5000, 6, 9, 3), (20000, 10, 10, 4),
                                              (3000, 20, 20, 5)])
def test_cauchy_point_against_sequential_sweep(n, m, npairs, seed):
    import ctypes as C
    rng = np.random.default_rng(seed)
    S = rng.standard_normal((npairs, n)) * 0.1
    Y = 2.0 * S + 0.02 * rng.standard_normal((npairs, n))          # curvature ~2: well-conditioned positive definite B
    lbv = rng.uniform(-1.0, -0.2, n)
    ubv = rng.uniform(0.2, 1.0, n)
    lbv[::13] = -np.inf
    ubv[::17] = np.inf
    x0 = np.clip(rng.uniform(-1.2, 1.2, n), lbv, ubv)
    g = rng.standard_normal(n) * rng.choice([0.01, 1.0, 30.0], n)   # widely spread breakpoints
    g[::29] = 0.0
    drv = lb.driver()
    dp = C.POINTER(C.c_double)
    P = lambda a: np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(dp)
    xcp = np.zeros(n)
    cls = np.zeros(n, dtype=np.uint8)
    vecc = np.zeros(2 * m)
    counts = (C.c_long * 2)()
    theta = C.c_double(0)
    err = C.create_string_buffer(256)
    Sc, Yc = np.ascontiguousarray(S), np.ascontiguousarray(Y)
    st = drv.lbfgsb200_drv_cauchy_f64(0, n, m, npairs, P(Sc) if npairs else None, P(Yc) if npairs else None, P(x0), P(g), P(lbv),
                                      P(ubv), P(xcp), cls.ctypes.data_as(C.POINTER(C.c_ubyte)), P(vecc), counts, C.byref(theta),
                                      err, 256)
    assert st == 0, err.value
    xr, act, vc = cauchy_sequential(S, Y, x0, g, lbv, ubv, m)
    c = min(npairs, m)
    assert np.max(np.abs(xcp - xr)) <= 1e-9 * max(1.0, np.max(np.abs(xr)))
    assert np.array_equal((cls & 2) != 0, act)
    assert counts[0] == act.sum()
    scale = max(1.0, np.max(np.abs(vc))) if c else 1.0
    # the driver orders W's columns newest pair first, the restatement oldest first
    if c:
        vy, vs = vecc[:c][::-1], vecc[c:2 * c][::-1]
        assert np.max(np.abs(np.concatenate([vy, vs]) - vc)) <= 1e-8 * scale
