"""The combination pass of objectives without neighbour coupling.

Warps that own no unit of a tile form its direction and hand it, through slots and mbarriers of the pass, to the warps that own the
units, which store d and take the first trial.  How many warps form, in how many groups, and how many stages the ring keeps next to
the hand-off slots follow from the block length (32 to 512 units per tile) and from the number of staged point rows.  These tests run
CTAs that own a single ragged tile at every block length, and batches whose members stage different numbers of rows over many tiles
per CTA, in fp64 and fp32, and whole solves with three forming groups on a four-stage ring against the CPU checker."""
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


def block_length(m, dtype):
    """Elements per block of the tiled history (lbfgs_b200_solver_create_batch): the largest power of two up to 1024 for which two
    stages of 2m + 4 rows fit the kernel's 192 KB staging ring."""
    bt = 1024
    while bt > 32 and 2 * (2 * m + 4) * bt * np.dtype(dtype).itemsize > 196608:
        bt //= 2
    return bt


@DTYPES
@pytest.mark.parametrize("m", [3, 10, 30, 64])
def test_ctas_with_one_ragged_tile(gpu_ctx, dtype, m):
    """n = 5 blocks less 6 elements: five CTAs own one tile each, the last one ragged, and the others own none -- fewer tiles than
    stages and hand-off slots.  fp64: units per tile 512 (m = 3), 256, 64, 32.  Batch members are their lone solves, bit for bit."""
    n = 5 * block_length(m, dtype) - 6
    prm = lb.LBFGSParam(m=m, max_iterations=2 * m + 10)
    X0 = np.stack([np.random.default_rng(m).uniform(-1.5, 1.5, n), np.zeros(n), np.full(n, 0.5)]).astype(dtype)
    bo, BX, BG, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "MoreThuente")
    for b in range(len(X0)):
        lone, Xl, Gl, by_op = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0[b], prm, "MoreThuente")
        assert lone[0].status == 0 and by_op.get("combine_trial", 0) >= 10
        assert np.array_equal(Gl[0], rosenbrock_grad(Xl[0]))
        assert (bo[b].status, bo[b].niter, bo[b].nfev, bo[b].fx) == (lone[0].status, lone[0].niter, lone[0].nfev, lone[0].fx)
        assert np.array_equal(BX[b], Xl[0]) and np.array_equal(BG[b], Gl[0])


@DTYPES
def test_batch_members_staging_different_rows(gpu_ctx, dtype):
    """A batch whose members run the combination pass one after another in a round: one with chains the curvature gate broke (more
    staged point rows, so fewer stages), two with chained histories, over 14 or 15 tiles per CTA.  Each member is its lone solve,
    bit for bit."""
    n = 1000002
    prm = lb.LBFGSParam(m=8, linesearch=lb.LBFGS_LINESEARCH_BACKTRACKING_ARMIJO, max_iterations=300, max_linesearch=60)
    x0, _, _, _ = _plain_run(gpu_ctx, n, prm, "Backtracking")
    X0 = np.stack([x0, np.zeros(n), np.full(n, 0.5)]).astype(dtype)
    bo, BX, BG, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "Backtracking")
    for b in range(len(X0)):
        lone, Xl, Gl, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0[b], prm, "Backtracking")
        assert (bo[b].status, bo[b].niter, bo[b].nfev, bo[b].fx) == (lone[0].status, lone[0].niter, lone[0].nfev, lone[0].fx)
        assert np.array_equal(BX[b], Xl[0]) and np.array_equal(BG[b], Gl[0])


@pytest.mark.parametrize("m", [10, 11, 20])
def test_many_tiles_per_cta_against_checker(gpu_ctx, orc, m):
    """fp64 over 15 or 16 tiles per CTA: m = 10 has two forming groups of 8 warps on 256 units per tile; m = 11 and 20 have three
    groups of 4 warps on 128 units and a ring of four stages, so a stage's tiles are formed by different groups in turn.  The solve
    matches the CPU checker and the same solve through the C ABI, bit for bit."""
    n = 2 ** 19 + 2 * 37
    prm = lb.LBFGSParam(m=m)
    x0 = np.zeros(n)
    outs, X, G, by_op = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "MoreThuente")
    assert outs[0].status == 0 and by_op.get("combine_trial", 0) >= 10
    assert np.array_equal(G[0], rosenbrock_grad(X[0]))
    g = lb.LBFGSSolver(prm, "MoreThuente", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0)
    assert np.array_equal(g["x"], X[0])
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, LS["MoreThuente"], cpu_param(orc, prm), sum_mode=po.SUM_LANES8)
    check_parity(g, c, xtol=1e-7)
