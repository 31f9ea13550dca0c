"""The gradient a device-resident solve returns, now that its passes do not store it.

For objectives without neighbour coupling g = grad f(x) is an element-wise function of x, and the library is built without FMA
contraction, so the passes that need the gradient of a stored point evaluate it from that point instead of reading it: only FIRST
and the last pass of a problem (MATERIALIZE) write g.  Whatever way a solve ends -- on the ray, on its search's start point, on the
point already in x when arming a search fails, or with an error status -- the gradient it leaves (read through
lbfgs_b200_solver_final_grad(_of), which the front copies even for an error) must be grad f of the returned x, bit for bit.  The
pass that takes the dots without a new pair (after the curvature gate rejects one) evaluates g from x as well; a run that takes it
is held to the CPU checker, and batch members to their lone solves."""
import ctypes as C

import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po
from test_gpu_resident_exit_points import CASES, N, rosenbrock_grad
from test_gpu_solver import check_parity, cpu_param
from util import LS

pytestmark = pytest.mark.gpu


class _Param(C.Structure):      # lbfgs_b200_param
    _fields_ = [("m", C.c_int), ("epsilon", C.c_double), ("epsilon_rel", C.c_double), ("past", C.c_int), ("delta", C.c_double),
                ("max_iterations", C.c_int), ("linesearch", C.c_int), ("max_linesearch", C.c_int), ("min_step", C.c_double),
                ("max_step", C.c_double), ("ftol", C.c_double), ("wolfe", C.c_double)]


class _Outcome(C.Structure):    # lbfgs_b200_outcome
    _fields_ = [("status", C.c_int), ("niter", C.c_int), ("nfev", C.c_longlong), ("fx", C.c_double), ("gnorm", C.c_double),
                ("rounds", C.c_longlong)]


def resident(ctx, objective, X0, prm, ls, data0=None, data1=None, ldd=0, on_solver=None):
    """The rows of X0 solved by one launch of the device-resident solve through the C ABI (a single problem through
    lbfgs_b200_solver_minimize, several through the batch entry point): (outcomes, X, G, rounds by pass) with G the final gradients
    read through lbfgs_b200_solver_final_grad_of.  data0/data1: None, a host array (uploaded in X0's dtype) or a lb.DeviceArray
    (passed as it is), problem b's data at offset b*ldd (ldd = 0: shared).  on_solver(s): called with the solver after the solve."""
    X0 = np.atleast_2d(X0)
    dt = X0.dtype
    suf = "f64" if dt == np.float64 else "f32"
    B, n = X0.shape
    lib = ctx.lib
    data = [v if v is None or isinstance(v, lb.DeviceArray) else ctx.array(np.asarray(v, dtype=dt)) for v in (data0, data1)]
    d0, d1 = (None if v is None else v.ptr for v in data)
    s = C.c_void_p()
    if B == 1:
        ctx.check(lib.lbfgs_b200_solver_create(ctx.h, n, prm.m, dt.itemsize, C.byref(s)))
    else:
        ctx.check(lib.lbfgs_b200_solver_create_batch(ctx.h, n, prm.m, dt.itemsize, B, C.byref(s)))
    try:
        p = _Param(prm.m, prm.epsilon, prm.epsilon_rel, prm.past, prm.delta, prm.max_iterations, prm.linesearch, prm.max_linesearch,
                   prm.min_step, prm.max_step, prm.ftol, prm.wolfe)
        xd = ctx.array(X0.reshape(-1))
        outs = (_Outcome * B)()
        if B == 1:
            ctx.check(getattr(lib, "lbfgs_b200_solver_minimize_" + suf)(s, objective, d0, d1, C.byref(p), LS[ls], xd.ptr, None, 0, outs))
        else:
            ctx.check(getattr(lib, "lbfgs_b200_solver_minimize_batch_" + suf)(s, objective, d0, d1, ldd, C.byref(p), LS[ls], xd.ptr, n, outs))
        if on_solver is not None:
            on_solver(s)
        X = xd.get().reshape(B, n)
        G = np.empty((B, n), dtype=dt)
        for b in range(B):
            gp = lib.lbfgs_b200_solver_final_grad_of(s, b)
            ctx.check(lib.lbfgs_b200_memcpy_d2h(ctx.h, G[b].ctypes.data_as(C.c_void_p), C.c_void_p(gp), G[b].nbytes))
        ms, rounds, nbytes = (C.c_double * 10)(), (C.c_ulonglong * 10)(), (C.c_double * 10)()
        kms, sync = C.c_double(0), (C.c_double * 3)()
        ctx.check(lib.lbfgs_b200_solver_profile(s, C.byref(kms), ms, rounds, nbytes, sync))
        by_op = {lb.Session.OPS[k]: int(rounds[k]) for k in range(10) if rounds[k]}
        del xd
        return list(outs), X, G, by_op
    finally:
        lib.lbfgs_b200_solver_destroy(s)


def quad_shift_grad(x, gofs=0):
    """grad f of QuadShift, expression by expression as the kernels evaluate it: 2 (x_i - i), i the global index."""
    r = x - (np.arange(x.size, dtype=np.int64) + gofs).astype(x.dtype)
    return x.dtype.type(2) * r


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name,ls,kw,status", CASES, ids=[c[0] for c in CASES])
def test_every_exit_returns_grad_of_x(gpu_ctx, name, ls, kw, status, dtype):
    prm = lb.LBFGSParam(**kw)
    x0 = np.zeros(N, dtype=dtype)
    outs, X, G, by_op = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, prm, ls)
    assert (outs[0].status == 0) == (status == "ok"), (name, outs[0].status)
    assert np.array_equal(G[0], rosenbrock_grad(X[0]))
    # the same solve as the front's (which the existing tests hold to the CPU checker)
    f = lb.LBFGSSolver(prm, ls, dtype=dtype, resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0)
    assert f["status"] == status and f["nfev"] == outs[0].nfev
    if status == "ok":   # (the front reports no iteration count for a solve that threw)
        assert f["niter"] == outs[0].niter and np.array_equal(np.asarray(f["grad"], dtype=dtype), G[0])
    assert np.array_equal(np.asarray(f["x"], dtype=dtype), X[0])
    if name == "step_max_when_armed":   # the search that fails to arm follows a pair-forming pass: x is stored, g was not
        assert by_op.get("dots_form", 0) > 0 and by_op.get("materialize", 0) == 1


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_quad_shift_single_and_batch(gpu_ctx, orc, dtype):
    n = 3 * 2 ** 16 + 10
    prm = lb.LBFGSParam(m=6)
    X0 = np.stack([np.zeros(n), np.random.default_rng(3).uniform(-5, 5, n), np.full(n, 7.0)]).astype(dtype)
    outs, X, G, _ = resident(gpu_ctx, lb.OBJ_QUAD_SHIFT, X0, prm, "MoreThuente")
    for b in range(len(X0)):
        lone, Xl, Gl, _ = resident(gpu_ctx, lb.OBJ_QUAD_SHIFT, X0[b], prm, "MoreThuente")
        assert outs[b].status == 0 and (outs[b].niter, outs[b].nfev, outs[b].fx) == (lone[0].niter, lone[0].nfev, lone[0].fx)
        assert np.array_equal(X[b], Xl[0]) and np.array_equal(G[b], Gl[0])
        assert np.array_equal(G[b], quad_shift_grad(X[b]))
    if dtype == np.float64:
        c = orc.lbfgs(po.OBJ_QUAD_SHIFT, X0[0], LS["MoreThuente"], cpu_param(orc, prm), sum_mode=po.SUM_LANES8)
        assert (outs[0].niter, outs[0].nfev) == (c["niter"], c["nfev"])
        assert np.max(np.abs(X[0] - c["x"])) <= 1e-7 * max(1.0, np.max(np.abs(c["x"])))


def _plain_run(ctx, n, prm, ls):
    """A seeded random start whose resident solve takes at least one DOTS_PLAIN round (a pair rejected by the curvature gate).  The
    paired Rosenbrock function is a sum over independent pairs, so a start that repeats one random pair takes the decisions of that
    two-coordinate problem, whose Armijo steps do leave negative curvature now and then (a start with independent pairs averages
    the curvature over all of them and practically never does)."""
    for seed in range(40):
        x0 = np.tile(np.random.default_rng(seed).uniform(-2, 2, 2), n // 2)
        outs, X, G, by_op = resident(ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, prm, ls)
        if by_op.get("dots_plain", 0) > 0:
            return x0, outs, X, G
    pytest.fail("no seed gave a DOTS_PLAIN round")


def test_dots_plain_against_checker_and_lone_solves(gpu_ctx, orc):
    n = 100002
    prm = lb.LBFGSParam(m=8, linesearch=lb.LBFGS_LINESEARCH_BACKTRACKING_ARMIJO, max_iterations=300, max_linesearch=60)
    x0, outs, X, G = _plain_run(gpu_ctx, n, prm, "Backtracking")
    assert np.array_equal(G[0], rosenbrock_grad(X[0]))
    g = lb.LBFGSSolver(prm, "Backtracking", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0)
    assert np.array_equal(g["x"], X[0])
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, LS["Backtracking"], cpu_param(orc, prm), sum_mode=po.SUM_LANES8)
    check_parity(g, c, xtol=1e-7)
    # in a batch, next to problems that take other passes in the same rounds
    X0 = np.stack([np.zeros(n), x0, np.full(n, 0.5)])
    bo, BX, BG, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "Backtracking")
    for b in range(len(X0)):
        lone, Xl, Gl, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0[b], prm, "Backtracking")
        assert (bo[b].status, bo[b].niter, bo[b].nfev, bo[b].fx) == (lone[0].status, lone[0].niter, lone[0].nfev, lone[0].fx)
        assert np.array_equal(BX[b], Xl[0]) and np.array_equal(BG[b], Gl[0])


@pytest.mark.parametrize("m", [12, 30])
def test_ragged_tiles_and_long_histories(gpu_ctx, orc, m):
    """Every warp has a column at m = 12 and m = 30 (the warps of column 0 form the new pair), and n leaves a ragged last tile."""
    n = 2 ** 19 + 2 * 37
    prm = lb.LBFGSParam(m=m)
    outs, X, G, by_op = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n), prm, "MoreThuente")
    assert outs[0].status == 0 and by_op.get("dots_form", 0) >= 12   # (c = 3, 6 and 12 give every warp a column)
    assert np.array_equal(G[0], rosenbrock_grad(X[0]))
    g = lb.LBFGSSolver(prm, "MoreThuente", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n))
    assert np.array_equal(g["x"], X[0]) and np.array_equal(g["grad"], G[0])
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, np.zeros(n), LS["MoreThuente"], cpu_param(orc, prm), sum_mode=po.SUM_LANES8)
    check_parity(g, c, xtol=1e-7)
