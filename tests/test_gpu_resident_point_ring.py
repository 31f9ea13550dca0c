"""The device-resident solve's ring of iterates.

For objectives without neighbour coupling the ring holds the accepted iterates instead of the pairs: c chained pairs are c + 1
points, and every pass that reads a pair rebuilds s = x_end - x_start and y = grad f(x_end) - grad f(x_start) with the arithmetic that
formed it.  The library is built without FMA contraction, so the pairs -- and everything computed from them -- are the bits a stored
S|Y ring gave.  These tests hold the exported history to the explicit differences of the iterates, run rings that wrap several times
and chains that the curvature gate breaks, in fp64 and fp32, and hold batch members to their lone solves."""
import ctypes as C

import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po
from test_gpu_resident_exit_points import rosenbrock_grad
from test_gpu_resident_implied_grad import _plain_run, resident
from test_gpu_solver import check_parity, cpu_param
from util import LS

pytestmark = pytest.mark.gpu

DTYPES = pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])


def history(ctx, s, dtype, n):
    """The live columns (S, Y by age, newest first) of problem 0 of solver s, as lbfgs_b200_solver_history_of exports them."""
    lib = ctx.lib
    h = lib.lbfgs_b200_solver_history_of(s, 0)
    assert h, ctx.last_error() if hasattr(ctx, "last_error") else "history export failed"
    cols = []
    for age in range(lib.lbfgs_b200_hist_ncorr(h)):
        pair = []
        for get in (lib.lbfgs_b200_hist_s_col, lib.lbfgs_b200_hist_y_col):
            v = np.empty(n, dtype=dtype)
            ctx.check(lib.lbfgs_b200_memcpy_d2h(ctx.h, v.ctypes.data_as(C.c_void_p), C.c_void_p(get(h, age)), v.nbytes))
            pair.append(v)
        cols.append(pair)
    return cols


@DTYPES
@pytest.mark.parametrize("m", [3, 10])
def test_exported_history_is_the_iterates_differences(gpu_ctx, dtype, m):
    """After a solve capped at K iterations the exported columns are x_{k+1} - x_k and grad f(x_{k+1}) - grad f(x_k) of the
    iterates of the same solve capped at k = 0 .. K, bit for bit (m = 3: the ring of 2M = 8 points has wrapped twice)."""
    n = 2 ** 15 + 2 * 11          # a ragged last tile
    K = 18
    x0 = np.zeros(n, dtype=dtype)
    iterates = [x0]
    for k in range(1, K + 1):
        outs, X, G, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, lb.LBFGSParam(m=m, max_iterations=k), "MoreThuente")
        assert outs[0].status == 0
        if not np.array_equal(X[0], iterates[-1]):
            iterates.append(X[0])
    got = {}
    resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, lb.LBFGSParam(m=m, max_iterations=K), "MoreThuente",
             on_solver=lambda s: got.setdefault("cols", history(gpu_ctx, s, dtype, n)))
    cols = got["cols"]
    assert 1 <= len(cols) <= m and len(iterates) > m + 2
    diffs = [(iterates[k + 1] - iterates[k], rosenbrock_grad(iterates[k + 1]) - rosenbrock_grad(iterates[k])) for k in range(len(iterates) - 1)]
    # the newest pair is the one the last pair-forming pass accepted; with no rejections the ages run back one iteration each
    newest = next(k for k in range(len(diffs)) if np.array_equal(diffs[k][0], cols[0][0]))
    assert newest >= len(cols) - 1
    for age, (s, y) in enumerate(cols):
        ds, dy = diffs[newest - age]
        assert np.array_equal(s, ds) and np.array_equal(y, dy), age


@DTYPES
@pytest.mark.parametrize("m", [3, 12, 30])
def test_wrapping_ring_against_checker_and_front(gpu_ctx, orc, dtype, m):
    """A run of many more iterations than the ring has points, with a ragged last tile."""
    n = 2 ** 17 + 2 * 37
    prm = lb.LBFGSParam(m=m)
    outs, X, G, by_op = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n, dtype=dtype), prm, "MoreThuente")
    assert outs[0].status == 0 and by_op.get("dots_form", 0) >= 12
    if m == 3:   # the ring's 2M = 8 points have wrapped more than twice
        assert by_op["dots_form"] > 2 * 2 * (m + 1)
    assert np.array_equal(G[0], rosenbrock_grad(X[0]))
    if dtype == np.float64:
        g = lb.LBFGSSolver(prm, "MoreThuente", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n))
        assert np.array_equal(g["x"], X[0])
        c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, np.zeros(n), LS["MoreThuente"], cpu_param(orc, prm), sum_mode=po.SUM_LANES8)
        check_parity(g, c, xtol=1e-7)


@DTYPES
@pytest.mark.parametrize("m", [3, 8])
def test_broken_chains_single_batch_and_nan_padding(gpu_ctx, orc, dtype, m):
    """Pairs rejected by the curvature gate leave the live points in several runs of the ring.  The solve must match the CPU
    checker, batch members their lone solves, and a solve on pool blocks that held NaN (the padding of every vector and ring row
    then holds NaN) the same solve on fresh blocks, bit for bit."""
    n = 100002
    prm = lb.LBFGSParam(m=m, linesearch=lb.LBFGS_LINESEARCH_BACKTRACKING_ARMIJO, max_iterations=300, max_linesearch=60)
    x0, outs, X, G = _plain_run(gpu_ctx, n, prm, "Backtracking")
    x0 = x0.astype(dtype)
    outs, X, G, by_op = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "Backtracking")
    assert np.array_equal(G[0], rosenbrock_grad(X[0]))
    if dtype == np.float64:
        assert by_op.get("dots_plain", 0) > 0
        c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, LS["Backtracking"], cpu_param(orc, prm), sum_mode=po.SUM_LANES8)
        g = lb.LBFGSSolver(prm, "Backtracking", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0)
        check_parity(g, c, xtol=1e-7)
    X0 = np.stack([np.full(n, 0.5), x0, np.zeros(n)]).astype(dtype)
    bo, BX, BG, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "Backtracking")
    for b in range(len(X0)):
        lone, Xl, Gl, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0[b], prm, "Backtracking")
        assert (bo[b].status, bo[b].niter, bo[b].nfev, bo[b].fx) == (lone[0].status, lone[0].niter, lone[0].nfev, lone[0].fx)
        assert np.array_equal(BX[b], Xl[0]) and np.array_equal(BG[b], Gl[0])
    # NaN in blocks the pool hands out again
    junk = gpu_ctx.array(np.full(64 * n, np.nan, dtype=dtype))
    del junk
    again, Xa, Ga, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "Backtracking")
    assert (again[0].status, again[0].niter, again[0].nfev, again[0].fx) == (outs[0].status, outs[0].niter, outs[0].nfev, outs[0].fx)
    assert np.array_equal(Xa[0], X[0]) and np.array_equal(Ga[0], G[0])
