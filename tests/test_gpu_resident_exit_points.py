"""The point a device-resident solve returns, on every way a solve can end.

For objectives without neighbour coupling the line-search trials store nothing: a trial point is implied by its step on the ray
x = xp + step*d, the pair-forming pass rebuilds the accepted point, and a problem that stops while its point is still implied writes
it in one last pass.  These runs end in each way the loop can end -- convergence, the iteration cap, the past/delta stall, a search
that ends on its kept best trial or on its start point, a line-search error after a trial, an invalid step when a search is armed --
at an n that gives every CTA several tiles and leaves a ragged last pack, and hold the result to the CPU checker.  Independently of
the checker, the gradient a successful solve returns must be grad f(x) of the returned x bit for bit (element-wise objective, no
FMA contraction).
More-Thuente never raises the max_linesearch error here: out of budget it takes its best point (the kept-trial / start-point cases)."""
import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po
from test_gpu_solver import check_parity, cpu_param
from util import LS

pytestmark = pytest.mark.gpu
N = 2 ** 20 + 6

# (id, line search, parameters, status): which way each run ends was found with the CPU checker from x0 = 0
CASES = [
    ("converged", "MoreThuente", dict(), "ok"),
    ("iteration_cap", "MoreThuente", dict(max_iterations=7), "ok"),
    ("stall_on_start_point", "MoreThuente", dict(past=1, delta=1e-6, max_linesearch=2), "ok"),    # its last search ends on its start
    ("cap_on_kept_trial", "MoreThuente", dict(max_linesearch=3, max_iterations=2), "ok"),         # its last search ends on the kept trial
    ("cap_on_start_point", "MoreThuente", dict(max_linesearch=2, max_iterations=5), "ok"),
    ("max_linesearch_backtracking", "Backtracking", dict(max_linesearch=2, max_iterations=4), "runtime_error"),
    ("max_linesearch_bracketing", "Bracketing", dict(max_linesearch=2), "runtime_error"),
    ("step_max_when_armed", "MoreThuente", dict(max_step=0.5, max_iterations=4), "invalid_argument"),
    ("min_step_when_armed", "MoreThuente", dict(min_step=10.0), "invalid_argument"),
]


def rosenbrock_grad(x):
    """grad f of the paired Rosenbrock function, expression by expression as the kernels evaluate it (in x's dtype)."""
    g = np.empty_like(x)
    t1 = x.dtype.type(1) - x[0::2]
    t2 = x.dtype.type(10) * (x[1::2] - x[0::2] * x[0::2])
    g[1::2] = x.dtype.type(20) * t2
    g[0::2] = x.dtype.type(-2) * (x[0::2] * g[1::2] + t1)
    return g


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name,ls,kw,status", CASES, ids=[c[0] for c in CASES])
def test_resident_exit_point(orc, name, ls, kw, status, dtype):
    prm = lb.LBFGSParam(**kw)
    x0 = np.zeros(N, dtype=dtype)
    g = lb.LBFGSSolver(prm, ls, dtype=dtype, resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0)
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, LS[ls], cpu_param(orc, prm), dtype=dtype,
                  **({"sum_mode": po.SUM_LANES8} if dtype == np.float64 else {}))
    assert c["status"] == status, (c["status"], c["msg"])
    if status == "ok":   # (the front returns the final gradient and the launch count of a solve that did not throw)
        assert g["launches"] == 1
        assert np.array_equal(np.asarray(g["grad"], dtype=dtype), rosenbrock_grad(np.asarray(g["x"], dtype=dtype)))
    if dtype == np.float64:
        check_parity(g, c, xtol=1e-7)
        # on the error paths too: the point the solve stopped at (the failing trial, or the current point)
        assert np.max(np.abs(g["x"] - c["x"])) <= 1e-7 * max(1.0, np.max(np.abs(c["x"])))
        if status == "ok":
            assert np.max(np.abs(g["grad"] - c["grad"])) <= 1e-6 * max(1.0, np.max(np.abs(c["grad"])))
    else:   # fp32 sums in another order than the checker's: the bar of test_gpu_resident.py::test_resident_float32
        assert (g["status"], g["msg"]) == (c["status"], c["msg"])
        assert abs(g["niter"] - c["niter"]) <= 3
        assert np.max(np.abs(g["x"] - c["x"])) <= 1e-2 * max(1.0, np.max(np.abs(c["x"])))


def test_batch_members_finishing_in_different_rounds_match_lone_solves():
    """Problems of a batch stop in different rounds (a stopping problem writes its point while the others run other passes): each
    member is still bit-identical to its lone solve."""
    X0 = np.stack([np.zeros(N), np.full(N, 0.5), np.random.default_rng(7).uniform(-1, 1, N)])
    for kw in (dict(), dict(max_linesearch=2, max_iterations=5), dict(past=1, delta=1e-6, max_linesearch=2)):
        prm = lb.LBFGSParam(**kw)
        bs = lb.BatchSession(lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "MoreThuente")
        res, X, _ = bs.solve()
        bs.close()
        rounds = set()
        for b in range(len(X0)):
            lone = lb.LBFGSSolver(prm, "MoreThuente", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, X0[b])
            assert (res[b]["niter"], res[b]["nfev"], res[b]["fx"]) == (lone["niter"], lone["nfev"], lone["fx"])
            assert np.array_equal(X[b], lone["x"])
            rounds.add(res[b]["rounds"])
        if not kw:
            assert len(rounds) > 1   # the members did finish in different rounds
