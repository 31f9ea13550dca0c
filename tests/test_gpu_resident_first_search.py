"""The device-resident solve's first line search, whose direction is not stored.

For objectives without neighbour coupling the first search's direction d = -grad f(x0) is an element-wise function of x0, so FIRST
writes only x0 to the ring, and the passes that read d while k == 1 -- the trials, the last pass of a problem that stops on the ray,
and the first pair-forming pass -- evaluate it from x0 with FIRST's arithmetic (no FMA contraction, T(-1) * g exact).  Nor does
FIRST write g: a solve that stops right at FIRST (converged at x0, or the first search refuses to start) takes one MATERIALIZE
round like every other stop.  These runs end inside or right after the first search, at an n that gives every CTA several tiles and
leaves a ragged last pack, and are held to the CPU checker; the gradient they return must be grad f of the returned x bit for bit,
and batch members must match their lone solves bit for bit."""
import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po
from test_gpu_resident_exit_points import N, rosenbrock_grad
from test_gpu_resident_implied_grad import resident
from test_gpu_solver import check_parity, cpu_param
from util import LS

pytestmark = pytest.mark.gpu


def zeros(dt):
    return np.zeros(N, dtype=dt)


def near_minimum(dt):
    """x* = 1 with a few coordinates (one in the ragged last pack) off by 1/8: the first step 1/||g|| overshoots, so a search with
    one trial ends on its start point."""
    x = np.ones(N, dtype=dt)
    x[[3, 1000, 500001, N - 3, N - 1]] += dt(0.125)
    return x


# (id, start, parameters, status, rounds of MATERIALIZE / TRIAL): which way each run ends was found with the CPU checker
CASES = [
    ("converged_at_x0", zeros, dict(epsilon=1e4), "ok", 1, 0),
    ("max_step_after_first", zeros, dict(max_step=1e-4), "invalid_argument", 1, 0),
    ("cap_after_first_search", zeros, dict(max_iterations=1), "ok", 1, None),          # 18 trials, then the ray point
    ("cap_on_kept_trial", zeros, dict(max_linesearch=3, max_iterations=1), "ok", 1, 3),
    ("cap_on_start_point", near_minimum, dict(max_linesearch=1, max_iterations=1), "ok", 1, 1),
    ("on_after_start_point", near_minimum, dict(max_linesearch=1, max_iterations=3), "ok", 1, None),   # forms a pair at xp
]


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name,start,kw,status,n_mat,n_trial", CASES, ids=[c[0] for c in CASES])
def test_first_search_exit(gpu_ctx, orc, name, start, kw, status, n_mat, n_trial, dtype):
    prm = lb.LBFGSParam(**kw)
    x0 = start(dtype)
    outs, X, G, by_op = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "MoreThuente")
    assert (outs[0].status == 0) == (status == "ok"), (name, outs[0].status)
    assert np.array_equal(G[0], rosenbrock_grad(X[0]))
    assert by_op.get("materialize", 0) == n_mat and by_op.get("first", 0) == 1
    if n_trial is not None:
        assert by_op.get("trial", 0) == n_trial, by_op
    g = lb.LBFGSSolver(prm, "MoreThuente", dtype=dtype, resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0)
    assert np.array_equal(np.asarray(g["x"], dtype=dtype), X[0])
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, LS["MoreThuente"], cpu_param(orc, prm), dtype=dtype,
                  **({"sum_mode": po.SUM_LANES8} if dtype == np.float64 else {}))
    assert c["status"] == status, (c["status"], c["msg"])
    if dtype == np.float64:
        check_parity(g, c, xtol=1e-7)
        assert np.max(np.abs(g["x"] - c["x"])) <= 1e-7 * max(1.0, np.max(np.abs(c["x"])))
    else:   # fp32 sums in another order than the checker's: the bar of test_gpu_resident.py::test_resident_float32
        assert (g["status"], g["msg"]) == (c["status"], c["msg"])
        assert abs(g["niter"] - c["niter"]) <= 3
        assert np.max(np.abs(g["x"] - c["x"])) <= 1e-2 * max(1.0, np.max(np.abs(c["x"])))


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("kw", [dict(max_iterations=1), dict(max_linesearch=1, max_iterations=3), dict(epsilon=1e4),
                                dict(max_step=1e-4)], ids=["cap", "start_point", "converged", "max_step"])
def test_first_search_batch_matches_lone_solves(gpu_ctx, kw, dtype):
    """Members that stop in or after their first search (or go on) next to each other in one launch: each bit for bit its lone
    solve."""
    X0 = np.stack([zeros(dtype), near_minimum(dtype), np.full(N, 0.5, dtype=dtype)])
    prm = lb.LBFGSParam(**kw)
    outs, X, G, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "MoreThuente")
    for b in range(len(X0)):
        lone, Xl, Gl, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0[b], prm, "MoreThuente")
        assert (outs[b].status, outs[b].niter, outs[b].nfev, outs[b].fx) == (lone[0].status, lone[0].niter, lone[0].nfev, lone[0].fx)
        assert np.array_equal(X[b], Xl[0]) and np.array_equal(G[b], Gl[0])
        assert np.array_equal(G[b], rosenbrock_grad(X[b]))
