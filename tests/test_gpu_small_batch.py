"""The small-batch solve (LBFGSSmallBatchSolver, include/LBFGSSmallBatch.h: one thread block per problem, the whole solve in shared
memory) against the CPU checker, the frozen outputs of the unmodified reference headers and LBFGSSolver.  Its decisions are the
device-resident solve's code and its sums are associated within one block, so it is held to the checker's parity bar, not to
bit-identity with LBFGSSolver; a problem's result must be bit-identical whatever the batch around it.  Every call sets a finite
max_iterations."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po
from test_gpu_solver import cpu_param
from util import LS, golden_cases, unhex

pytestmark = pytest.mark.gpu
LS_NAMES = ["Backtracking", "Bracketing", "NocedalWright", "MoreThuente"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAXIT = 5000


def small(X0, prm, ls, objective=lb.OBJ_ROSENBROCK_PAIRED, **kw):
    return lb.solve_small_batch(objective, np.atleast_2d(X0), prm, ls, **kw)


def near(g, gx, c, xtol):
    """The parity bar of check_parity without the trace (the small-batch solve keeps none): counts, fx, x."""
    assert (g["niter"], g["nfev"]) == (c["niter"], c["nfev"])
    assert abs(g["fx"] - c["fx"]) <= 1e-10 * max(1.0, abs(c["fx"]))
    assert np.max(np.abs(gx - c["x"])) <= xtol * max(1.0, np.max(np.abs(c["x"])))


@pytest.mark.parametrize("ls", LS_NAMES)
def test_reference_self_checks_full_size(orc, ls):
    """example-rosenbrock-comparison.cpp / -bracketing.cpp at their own size: 1024 random starts for every even n up to 24, one
    launch each.  Every start converges to |x - 1|_inf <= 1e-4.  The iteration counts are those of chaotic runs (up to ~150
    iterations), which move with the summation order: a problem's count must lie within the range that three orders give -- the
    checker's sequential and 8-lane sums and LBFGSBatchSolver's cross-CTA sums -- widened by 25 %, for at least 99 % of the starts."""
    prm = lb.LBFGSParam(max_linesearch=256, max_iterations=MAXIT)
    cprm = cpu_param(orc, prm)
    inside = total = 0
    worst = None
    for n in range(2, 25, 2):
        X0 = np.random.default_rng(4000 + n).uniform(-1, 1, (1024, n))
        res, X, _ = small(X0, prm, ls)
        assert all(r["status"] == "ok" for r in res), n
        assert np.max(np.abs(X - 1.0)) <= 1e-4, n
        bs = lb.BatchSession(lb.OBJ_ROSENBROCK_PAIRED, X0, prm, ls)
        rb, _, _ = bs.solve(return_x=False)
        bs.close()
        for b in range(len(X0)):
            c1 = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, X0[b], LS[ls], cprm, sum_mode=po.SUM_SEQUENTIAL, trace_cap=1)
            c2 = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, X0[b], LS[ls], cprm, sum_mode=po.SUM_LANES8, trace_cap=1)
            counts = (c1["niter"], c2["niter"], rb[b]["niter"])
            ok = 0.75 * min(counts) <= res[b]["niter"] <= 1.25 * max(counts)
            inside += ok
            total += 1
            if not ok and worst is None:
                worst = (n, b, res[b]["niter"], counts)
    print("%s: %d of %d starts inside the widened range; first outside: %s" % (ls, inside, total, worst))
    assert inside >= 0.99 * total, (inside, total, worst)


@pytest.mark.parametrize("case", [c for c in golden_cases("lbfgs") if c["dtype"] == "f64"], ids=lambda c: c["name"])
def test_small_batch_on_golden_cases(case):
    """Frozen outputs of the unmodified reference headers, each case as problem 0 of a batch of three (the other two: random starts
    of the same shape); the bar of test_resident_on_golden_cases without the trace.  Cases above max_n are refused."""
    prm = lb.LBFGSParam(**case["param"])
    if not prm.max_iterations:
        prm.max_iterations = MAXIT
    x0 = unhex(case["x0"])
    n = x0.size
    d0, d1 = (unhex(case["data"][0]), unhex(case["data"][1])) if case["data"] else (None, None)
    X0 = np.stack([x0] + [np.random.default_rng(s).uniform(-1, 1, n) for s in (1, 2)])
    max_n = lb.small_max_n(prm.m, case["objective"]) if prm.m >= 1 else 0
    if prm.m >= 1 and n > max_n:
        with pytest.raises(ValueError, match="exceeds %d" % max_n):
            small(X0, prm, case["ls"], case["objective"], data0=d0, data1=d1)
        return
    try:
        res, X, _ = small(X0, prm, case["ls"], case["objective"], data0=d0, data1=d1)
    except ValueError:
        assert case["status"] == "invalid_argument"   # refused before any solve, as LBFGSSolver's constructor refuses it
        return
    g = res[0]
    assert g["status"] == case["status"]
    if case["status"] != "ok":
        assert g["nfev"] == case["nfev"]
        return
    c = dict(niter=case["niter"], nfev=case["nfev"], fx=float.fromhex(case["fx"]), x=unhex(case["x"]))
    if case["niter"] > 60:  # chaotic regime: compare the optimum, not the path
        assert abs(g["fx"] - c["fx"]) <= 1e-9 * max(1.0, abs(c["fx"]))
    else:
        near(g, X[0], c, 1e-6)


@pytest.mark.parametrize("ls", LS_NAMES)
@pytest.mark.parametrize("n", [10, 1000])
def test_rosenbrock_from_zero_matches_checker(orc, ls, n):
    prm = lb.LBFGSParam(m=10 if n > 10 else 6, max_iterations=MAXIT)
    n = min(n, lb.small_max_n(prm.m, lb.OBJ_ROSENBROCK_PAIRED))
    res, X, _ = small(np.zeros((2, n)), prm, ls)
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, np.zeros(n), LS[ls], cpu_param(orc, prm), sum_mode=po.SUM_LANES8)
    for b in range(2):
        assert res[b]["status"] == c["status"] == "ok"
        near(res[b], X[b], c, 1e-7)


def test_other_objectives(orc):
    from test_gpu_resident_coupled import chained_grad, tridiag_grad
    # chained Rosenbrock: stored trials (x_lo / g_lo, RESTORE); odd n leaves a ragged last pack.  The gradient a problem returns is
    # the gradient expression at its x, bit for bit (no FMA contraction)
    prm = lb.LBFGSParam(max_iterations=MAXIT)
    for n in (300, 301):
        res, X, G = small(np.full((2, n), 1.3), prm, "NocedalWright", lb.OBJ_ROSENBROCK_CHAINED, want_grad=True)
        c = orc.lbfgs(po.OBJ_ROSENBROCK_CHAINED, np.full(n, 1.3), LS["NocedalWright"], cpu_param(orc, prm))
        for b in range(2):
            assert res[b]["status"] == c["status"] == "ok"
            near(res[b], X[b], c, 1e-6)
            assert np.array_equal(G[b], chained_grad(X[b]))
    # tridiagonal quadratic with per-problem data (ldd = n): every problem against the checker on its own d and b
    B = 3
    prm = lb.LBFGSParam(max_iterations=MAXIT)
    for n in (200, 201):
        data = [po.quad_tridiag_data(n, kappa=1e2, seed=10 + b) for b in range(B)]
        D = np.concatenate([d for d, _, _ in data])
        R = np.concatenate([r for _, r, _ in data])
        for ls in ("Bracketing", "MoreThuente"):
            res, X, G = small(np.zeros((B, n)), prm, ls, lb.OBJ_QUAD_TRIDIAG, data0=D, data1=R, ldd=n, want_grad=True)
            for b, (d, r, xs) in enumerate(data):
                c = orc.lbfgs(po.OBJ_QUAD_TRIDIAG, np.zeros(n), LS[ls], cpu_param(orc, prm), data0=d, data1=r)
                assert res[b]["status"] == c["status"] == "ok"
                near(res[b], X[b], c, 1e-6)
                assert np.max(np.abs(X[b] - xs)) <= 1e-3
                assert np.array_equal(G[b], tridiag_grad(X[b], d, r))
    # quadratic shift: 2 iterations, x = 0..9
    res, X, _ = small(np.zeros((2, 10)), lb.LBFGSParam(max_iterations=MAXIT), "NocedalWright", lb.OBJ_QUAD_SHIFT)
    assert all(r["niter"] == 2 for r in res) and np.allclose(X, np.arange(10.0), atol=1e-12)


def test_result_does_not_depend_on_the_batch():
    """One problem alone, then at positions 0, 17 and B-1 of a batch of B = 100 000 (beyond LBFGSBatchSolver's 4096): identical bits."""
    n, B = 10, 100000
    prm = lb.LBFGSParam(max_iterations=MAXIT)
    p = np.random.default_rng(99).uniform(-1, 1, n)
    alone, Xa, Ga = small(p[None, :], prm, "MoreThuente", want_grad=True)
    X0 = np.random.default_rng(100).uniform(-1, 1, (B, n))
    for pos in (0, 17, B - 1):
        X0[pos] = p
    res, X, G = small(X0, prm, "MoreThuente", want_grad=True)
    assert alone[0]["status"] == "ok"
    for pos in (0, 17, B - 1):
        assert res[pos] == alone[0]
        assert np.array_equal(X[pos], Xa[0]) and np.array_equal(G[pos], Ga[0])
    ok = np.array([r["status"] == "ok" for r in res])
    assert ok.mean() > 0.99 and np.max(np.abs(X[ok] - 1.0)) <= 5e-3


def test_stopping_rules_and_error_paths():
    """Every parameter set of test_resident_stopping_rules_and_error_paths as a batch of its own (x0 = 0 and an already optimal
    start): status and counts as LBFGSSolver returns or raises them on each problem alone."""
    sets = ((lb.LBFGSParam(max_iterations=5), "NocedalWright"), (lb.LBFGSParam(past=3, delta=1e-6), "MoreThuente"),
            (lb.LBFGSParam(max_linesearch=1), "Backtracking"), (lb.LBFGSParam(max_linesearch=1), "Bracketing"),
            (lb.LBFGSParam(max_linesearch=1, max_iterations=3), "MoreThuente"),
            (lb.LBFGSParam(max_linesearch=1, max_iterations=3), "NocedalWright"),
            (lb.LBFGSParam(linesearch=1), "NocedalWright"), (lb.LBFGSParam(linesearch=1, max_linesearch=64), "Backtracking"),
            (lb.LBFGSParam(linesearch=2, max_linesearch=64), "Bracketing"), (lb.LBFGSParam(m=0), "MoreThuente"),
            (lb.LBFGSParam(max_step=0.5), "MoreThuente"), (lb.LBFGSParam(min_step=10.0), "MoreThuente"))
    X0 = np.stack([np.zeros(12), np.ones(12)])
    for prm, ls in sets:
        if not prm.max_iterations:
            prm.max_iterations = MAXIT
        lone = [lb.LBFGSSolver(prm, ls, resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0) for x0 in X0]
        try:
            res, X, _ = small(X0, prm, ls)
        except ValueError:
            assert all(g["status"] == "invalid_argument" and g["nfev"] == 0 for g in lone), (prm.__dict__, ls)
            continue
        for g, r, x in zip(lone, res, X):
            assert r["status"] == g["status"] and r["nfev"] == g["nfev"], (prm.__dict__, ls, r, g["status"], g["nfev"])
            if g["status"] == "ok":
                assert r["niter"] == g["niter"]
                assert abs(r["fx"] - g["fx"]) <= 1e-10 * max(1.0, abs(g["fx"]))
                assert np.max(np.abs(x - g["x"])) <= 1e-6
    assert res[1]["niter"] == 1 and res[1]["nfev"] == 1


def test_float32(orc):
    prm = lb.LBFGSParam(max_iterations=MAXIT)
    res, X, G = small(np.zeros((3, 64)), prm, "NocedalWright", dtype=np.float32, want_grad=True)
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, np.zeros(64), LS["NocedalWright"], cpu_param(orc, prm), dtype=np.float32)
    assert X.dtype == np.float32 and G.dtype == np.float32
    for b in range(3):
        assert res[b]["status"] == "ok" and abs(res[b]["niter"] - c["niter"]) <= 3 and np.max(np.abs(X[b] - 1.0)) <= 1e-2
        assert np.array_equal(X[b], X[0]) and res[b] == res[0]
    # chained Rosenbrock: its last coordinates converge slowly, and in fp32 the stop rule gnorm <= 1e-5 |x| holds well before x = 1
    res, X, _ = small(np.full((2, 300), 1.3), prm, "MoreThuente", lb.OBJ_ROSENBROCK_CHAINED, dtype=np.float32)
    for r, x in zip(res, X):
        assert r["status"] == "ok" and r["gnorm"] <= 1e-5 * np.linalg.norm(x.astype(np.float64)) * 1.001 and r["fx"] <= 1e-3 * 182.0
    res, X, _ = small(np.zeros((2, 10)), prm, "NocedalWright", lb.OBJ_QUAD_SHIFT, dtype=np.float32)
    assert np.allclose(X, np.arange(10.0), atol=1e-5)


class _Param(C.Structure):   # lbfgs_b200_param
    _fields_ = [("m", C.c_int), ("epsilon", C.c_double), ("epsilon_rel", C.c_double), ("past", C.c_int), ("delta", C.c_double),
                ("max_iterations", C.c_int), ("linesearch", C.c_int), ("max_linesearch", C.c_int), ("min_step", C.c_double),
                ("max_step", C.c_double), ("ftol", C.c_double), ("wolfe", C.c_double)]


def test_misuse_is_refused(gpu_ctx):
    lib = gpu_ctx.lib
    max_n = lb.small_max_n(6, lb.OBJ_ROSENBROCK_PAIRED)
    X = gpu_ctx.array(np.zeros(4 * (max_n + 2)))
    outs = (C.c_byte * (64 * 4))()
    p = _Param(6, 1e-5, 1e-5, 0, 0.0, MAXIT, 3, 20, 1e-20, 1e20, 1e-4, 0.9)

    def call(n, B, ldx, obj=lb.OBJ_ROSENBROCK_PAIRED, prm=p):
        st = lib.lbfgs_b200_small_minimize_f64(gpu_ctx.h, obj, None, None, 0, n, B, C.byref(prm), 3, X.ptr, ldx, None, outs)
        return st, lib.lbfgs_b200_last_error(gpu_ctx.h).decode()

    st, msg = call(max_n + 2, 2, max_n + 2)
    assert st == 1 and str(max_n) in msg and "LBFGSBatchSolver" in msg
    assert call(10, 0, 10)[0] == 1
    assert call(10, 2, 8)[0] == 1
    assert call(11, 2, 11)[0] == 1                                   # paired Rosenbrock needs an even n
    assert call(10, 2, 10, prm=_Param(6, 1e-5, 1e-5, 65, 0.0, MAXIT, 3, 20, 1e-20, 1e20, 1e-4, 0.9))[0] == 1   # past > 64
    assert call(10, 2, 10)[0] == 0                                   # and the context still works
    with pytest.raises(ValueError, match="exceeds"):
        small(np.zeros((2, max_n + 2)), lb.LBFGSParam(max_iterations=MAXIT), "MoreThuente")


def test_line_search_comparison_batch_example():
    """examples/line_search_comparison_batch.cpp: the reference's self-checks at 1024 starts, one launch per (n, line search)."""
    lb.build_all()
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "examples")], check=True)
    r = subprocess.run([os.path.join(ROOT, "examples", "bin", "line_search_comparison_batch")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "FAILED" not in r.stdout and r.stdout.count("LineSearchMoreThuente") == 12
