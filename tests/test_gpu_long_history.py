"""Long histories, m = 25 to 64, in every solve path against float64 references.

Every entry point takes m <= 64, and several parts of the library run only past 24 or 32 pairs:
- the second lane set (entries 32..63) of the column-oriented coefficient recursion (gram_solve_in_smem) at c > 32;
- the third round of columns of the dots passes (k_gram_dots<T, 3>, k_persist<T, OBJ, 3>) at c > 48;
- the dynamic shared-memory opt-in of k_gram_combine (> 40 KB: fp64 c >= 50) and k_gram_fold (> 48 KB: fp64 c >= 54);
- the device-resident solve's 64-element (fp64) / 128-element (fp32) history blocks at m >= 47;
- rows 64..129 of its ring of 2M points (the second and third words of free_point's mask) after 64 accepted iterates at m >= 32;
- the small-batch solve with its 6M^2 Gram elements in shared memory at m > 32, at its own max_n.
Each test below asserts that its run reached the boundary it is about (the history's ncorr, the checker's iteration count or the
rounds by pass), so that a run that stops short fails instead of passing on short histories.  The iteration counts and caps were
chosen with the CPU checker: uncapped, the tridiagonal quadratic at kappa = 1e3 runs 105-200 iterations and paired Rosenbrock from
uniform(-2, 2) 123-240; caps are set where the checker's two summation orders still take the same decisions.

The opt-ins of k_gram_combine and k_gram_fold are reached by the fp64 apply_Hv cases at c >= 50 and c >= 54: the evidence that they
work is that those launches succeed and match the checker.

Not covered: free_point's search past a used row.  While no pair is rejected the live points form one cyclic run of rows ending at
the newest point, so the row after it is always free and the mask words are never consulted; at m >= 32 the live span wraps the whole
ring of 2M rows only if about m + 1 pairs are rejected within some 2m iterations, which none of these runs does."""
import ctypes as C

import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po
from test_gpu_resident_coupled import TRIDIAG, across_ctas, chained_grad, orders, spread_bar, tridiag_grad
from test_gpu_resident_exit_points import rosenbrock_grad
from test_gpu_resident_implied_grad import resident
from test_gpu_resident_point_ring import history
from test_gpu_solver import check_parity, cpu_param
from util import LS

pytestmark = pytest.mark.gpu

DTYPES = pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
HV_C = [24, 25, 32, 33, 48, 49, 50, 54, 64]


def seeded_pairs(npairs, n, seed, dtype=np.float64):
    rng = np.random.default_rng(seed)
    S = rng.standard_normal((npairs, n)).astype(dtype)
    Y = (S + 0.1 * rng.standard_normal((npairs, n))).astype(dtype)
    v = rng.standard_normal(n).astype(dtype)
    return S, Y, v


def filled(ctx, n, m, S, Y, dtype=np.float64):
    """A History of size m with the rows of S, Y appended back to back (every append after the first folds the one before it)."""
    h = lb.History(ctx, n, m, dtype)
    for s, y in zip(S, Y):
        h.add(ctx.array(s), ctx.array(y))
    return h


# ---- 1. the stand-alone apply_Hv ----------------------------------------------------------------------------------------------
HV_BUILDS = list(dict.fromkeys((c, m, npairs) for c in HV_C for (m, npairs) in ((c, c), (64, c), (c, 2 * c + 7))))   # (64, 64, 64) once


@pytest.mark.parametrize("c,m,npairs", HV_BUILDS, ids=["c%d-m%d-p%d" % b for b in HV_BUILDS])
def test_apply_Hv_long_history(gpu_ctx, orc, c, m, npairs):
    """c pairs held as m = c, as m = 64, and as a ring of m = c that wrapped; n: one partial tile, a ragged n that is not a multiple of
    the 2048-element tile, and the same n with v and res one element off alignment (the element-wise staging path)."""
    for n, off in ((1500, 0), (6151, 0), (6151, 1)):
        S, Y, v = seeded_pairs(npairs, n, seed=1000 * c + 10 * m + npairs + n)
        h = filled(gpu_ctx, n, m, S, Y)
        assert h.ncorr == c
        ref, _, theta_ref = orc.apply_Hv(S, Y, v, -1.0, m)
        scale = np.max(np.abs(ref))
        dv = lb.DeviceArray(gpu_ctx, v, offset_elems=off)
        for algo in (lb.HV_TWO_LOOP, lb.HV_AUTO):
            dres = lb.DeviceArray(gpu_ctx, None, np.float64, n, offset_elems=off)
            vdot = h.apply_Hv(dv, -1.0, dres, algo, want_dot=True)
            res = dres.get()
            assert np.max(np.abs(res - ref)) <= 1e-11 * scale, (n, off, algo, np.max(np.abs(res - ref)) / scale)
            assert abs(vdot - np.dot(v, res)) <= 4 * 64 * np.finfo(np.float64).eps * float(np.sum(np.abs(v * res)))
            h.apply_Hv(dv, -1.0, dres, algo)
            assert np.array_equal(dres.get(), res), "two calls gave different bits"
        theta, ys, _ = h.scalars()
        assert np.isclose(theta, theta_ref, rtol=1e-13)
        ys_ref = np.array([np.dot(S[npairs - 1 - a], Y[npairs - 1 - a]) for a in range(c)])
        sy_abs = np.array([np.sum(np.abs(S[npairs - 1 - a] * Y[npairs - 1 - a])) for a in range(c)])
        assert ys.shape == (c,) and np.all(np.abs(ys - ys_ref) <= 64 * np.finfo(np.float64).eps * sy_abs)


@pytest.mark.parametrize("c", [25, 33, 49, 64])
def test_apply_Hv_long_history_float32(gpu_ctx, orc, c):
    """fp32 histories (m = c, wrapped) against the float64 reference on the promoted fp32 inputs, at the bar of test_apply_Hv_float32."""
    n, m = 6151, c
    S, Y, v = seeded_pairs(c + 9, n, seed=c, dtype=np.float32)
    h = filled(gpu_ctx, n, m, S, Y, np.float32)
    assert h.ncorr == c
    ref, _, _ = orc.apply_Hv(S.astype(np.float64), Y.astype(np.float64), v.astype(np.float64), -1.0, m)
    for algo in (lb.HV_TWO_LOOP, lb.HV_AUTO):
        dres = gpu_ctx.empty(n, np.float32)
        h.apply_Hv(gpu_ctx.array(v), np.float32(-1.0), dres, algo)
        res = dres.get()
        assert np.max(np.abs(res - ref)) <= 2e-4 * np.max(np.abs(ref)), (algo, np.max(np.abs(res - ref)) / np.max(np.abs(ref)))
        h.apply_Hv(gpu_ctx.array(v), np.float32(-1.0), dres, algo)
        assert np.array_equal(dres.get(), res)


# Gram form against the separate calls / the two-loop recursion: 1e-11 in fp64 (test_fused_update_apply_Hv_matches_separate_calls),
# 2e-4 in fp32 (test_fused_update_apply_Hv_float32)
HV_RTOL = {np.float64: 1e-11, np.float32: 2e-4}


@DTYPES
@pytest.mark.parametrize("n", [6151, 3 * 2048])
@pytest.mark.parametrize("c,prior", [(33, 32), (49, 48), (64, 70)])
def test_fused_update_apply_Hv_long_history(gpu_ctx, n, c, prior, dtype):
    """lbfgs_b200_hist_update_apply_Hv at c = 33, 49 and 64 (a full ring: the new pair replaces the oldest) against the separate
    calls and against the literal two-loop recursion on the same history."""
    m = 64 if c == 64 else c + 5
    tol = HV_RTOL[dtype]
    a = dtype(-1.0)
    rng = np.random.default_rng(7 * n + c)
    ha, hb = lb.History(gpu_ctx, n, m, dtype), lb.History(gpu_ctx, n, m, dtype)
    for _ in range(prior):
        s = rng.standard_normal(n)
        ds, dy = gpu_ctx.array(s.astype(dtype)), gpu_ctx.array((s + 0.1 * rng.standard_normal(n)).astype(dtype))
        ha.add(ds, dy)
        hb.add(ds, dy)
    xp, gp = rng.standard_normal(n).astype(dtype), rng.standard_normal(n).astype(dtype)
    s = 0.3 * rng.standard_normal(n)
    x, g = (xp + s).astype(dtype), (gp + s + 0.1 * rng.standard_normal(n)).astype(dtype)
    dx, dxp, dg, dgp = (gpu_ctx.array(v) for v in (x, xp, g, gp))
    ra, rb_ = gpu_ctx.empty(n, dtype), gpu_ctx.empty(n, dtype)
    acc_a, _, _ = ha.update(dx, dxp, dg, dgp)
    dot_a = ha.apply_Hv(dg, a, ra, lb.HV_GRAM, want_dot=True)
    acc_b, dot_b = hb.update_apply_Hv(dx, dxp, dg, dgp, a, rb_, lb.HV_GRAM)
    assert acc_a and acc_b and ha.ncorr == hb.ncorr == c
    assert np.array_equal(hb.column("s", 0), x - xp) and np.array_equal(hb.column("y", 0), g - gp)
    assert np.array_equal(hb.column("s", c - 1), ha.column("s", c - 1))
    va, vb = ra.get(), rb_.get()
    assert np.max(np.abs(va - vb)) <= tol * np.max(np.abs(va))
    assert abs(dot_a - dot_b) <= tol * abs(dot_a)
    hb.apply_Hv(dg, a, ra, lb.HV_TWO_LOOP)
    assert np.max(np.abs(ra.get() - vb)) <= tol * np.max(np.abs(vb))


@DTYPES
def test_fused_update_rejected_pair_leaves_full_ring_untouched(gpu_ctx, dtype):
    """y = 0 fails the curvature gate with the ring full (c = m = 64): every column, theta and ys stay as they were, and the old
    history answers."""
    n, m = 6151, 64
    tol = HV_RTOL[dtype]
    a = dtype(-1.0)
    rng = np.random.default_rng(64)
    h = lb.History(gpu_ctx, n, m, dtype)
    for _ in range(m + 6):
        s = rng.standard_normal(n)
        h.add(gpu_ctx.array(s.astype(dtype)), gpu_ctx.array((s + 0.1 * rng.standard_normal(n)).astype(dtype)))
    assert h.ncorr == m
    ref = gpu_ctx.empty(n, dtype)
    xp, g = rng.standard_normal(n).astype(dtype), rng.standard_normal(n).astype(dtype)
    dg = gpu_ctx.array(g)
    h.apply_Hv(dg, a, ref, lb.HV_TWO_LOOP)   # folds the last appended pair
    before = [(h.column("s", k), h.column("y", k)) for k in range(m)]
    theta0, ys0, _ = h.scalars()
    res = gpu_ctx.empty(n, dtype)
    acc, dot = h.update_apply_Hv(gpu_ctx.array((xp + dtype(0.1)).astype(dtype)), gpu_ctx.array(xp), dg, dg, a, res, lb.HV_GRAM)
    assert not acc and h.ncorr == m
    assert all(np.array_equal(h.column("s", k), s) and np.array_equal(h.column("y", k), y) for k, (s, y) in enumerate(before))
    theta1, ys1, _ = h.scalars()
    assert theta1 == theta0 and np.array_equal(ys1, ys0)
    r = ref.get().astype(np.float64)
    assert np.max(np.abs(res.get() - r)) <= tol * np.max(np.abs(r))
    gr = float(np.dot(g.astype(np.float64), r))
    assert abs(dot - gr) <= 10 * tol * abs(gr)


# ---- 2. the host-driven loop --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hv", [lb.HV_AUTO, lb.HV_TWO_LOOP], ids=["gram", "two_loop"])
@pytest.mark.parametrize("ls", ["Bracketing", "MoreThuente"])
@pytest.mark.parametrize("m", [33, 49, 64])
def test_host_loop_tridiag(orc, m, ls, hv):
    """LBFGSSolver (not resident) on the tridiagonal quadratic, capped at 100 iterations: c = m for the last 100 - m of them.  (Uncapped,
    these runs take 187-192 iterations, and Bracketing ends some of them with its max_linesearch error in one summation order and not
    in the other; at the cap both orders take the same decisions.)"""
    n = 4099
    d, b, _ = po.quad_tridiag_data(n, kappa=1e3, seed=1)
    prm = lb.LBFGSParam(m=m, max_iterations=100)
    g = lb.LBFGSSolver(prm, ls, hv_algo=hv).minimize(lb.OBJ_QUAD_TRIDIAG, np.zeros(n), data0=d, data1=b)
    c = orc.lbfgs(po.OBJ_QUAD_TRIDIAG, np.zeros(n), LS[ls], cpu_param(orc, prm), data0=d, data1=b, sum_mode=po.SUM_LANES8)
    assert c["status"] == "ok" and c["niter"] > m
    check_parity(g, c, xtol=1e-7)


@pytest.mark.parametrize("ls", ["Bracketing", "MoreThuente"])
@pytest.mark.parametrize("m", [33, 49, 64])
def test_host_loop_tridiag_float32(orc, m, ls):
    """The fp32 host-driven loop, capped at m + 2 iterations (c = m for the last two; further on the fp32 checker's two summation
    orders part ways), against the fp32 checker: x within 32x the checker's own spread, or the fp32 bar of test_resident_exit_point."""
    n = 4099
    d, b, _ = (v.astype(np.float32) for v in po.quad_tridiag_data(n, kappa=1e3, seed=1))
    x0 = np.zeros(n, np.float32)
    prm = lb.LBFGSParam(m=m, max_iterations=m + 2)
    g = lb.LBFGSSolver(prm, ls, dtype=np.float32).minimize(lb.OBJ_QUAD_TRIDIAG, x0, data0=d, data1=b)
    c, c2 = orders(orc, lb.OBJ_QUAD_TRIDIAG, x0, d, b, ls, prm, np.float32)
    assert c["status"] == "ok" and c["niter"] == m + 2
    assert g["status"] == "ok" and g["niter"] == m + 2
    err = float(np.max(np.abs(np.asarray(g["x"], np.float64) - c["x"])))
    bar = max(spread_bar(c, c2), 1e-2 * max(1.0, float(np.max(np.abs(c["x"])))))
    assert err <= bar, (err, bar)


# ---- 3. the device-resident solve ---------------------------------------------------------------------------------------------
# neighbour-coupled: the S|Y ring.  Caps per m: (m + 2, about 2m) in fp64, m + 2 in fp32 (past it the fp32 checker's two orders part ways)
COUPLED_CAPS = {33: (35, 66), 49: (51, 98), 64: (66, 100)}


def capped_iterates(ctx, objective, x0, prm_kw, ls, first, last, **kw):
    """x of the solve capped at k = first .. last (the iterates; no pair is rejected in these runs).  x_0 is the start point
    (max_iterations = 0 would mean no cap)."""
    out = {0: x0} if first == 0 else {}
    for k in range(max(first, 1), last + 1):
        outs, X, _, _ = resident(ctx, objective, x0, lb.LBFGSParam(max_iterations=k, **prm_kw), ls, **kw)
        assert outs[0].status == 0 and outs[0].niter == k
        out[k] = X[0]
    return out


def held_to_checker_long(ctx, orc, objective, x0, d, b, prm, dtype):
    """A capped run against the checker: the front returns the C ABI's x and gradient, the gradient is grad f(x) bit for bit, the
    checker's two summation orders take the same decisions and the GPU takes them too (fp64), and x lies within 32x the checker's
    own spread between its orders -- or, in fp64, 1e-9 relative, where two orders happen to land closer than a third; in fp32
    within 1e-2 relative (the bar of test_resident_exit_point).  Returns the rounds by pass."""
    outs, X, G, by_op = resident(ctx, objective, x0, prm, "MoreThuente", data0=d, data1=b)
    g = lb.LBFGSSolver(prm, "MoreThuente", dtype=dtype, resident=True).minimize(objective, x0, data0=d, data1=b)
    assert np.array_equal(np.asarray(g["x"], dtype=dtype), X[0]) and np.array_equal(np.asarray(g["grad"], dtype=dtype), G[0])
    gref = tridiag_grad(X[0], d, b) if objective == TRIDIAG else rosenbrock_grad(X[0])
    assert np.array_equal(G[0], gref)
    c, c2 = orders(orc, objective, x0, d, b, "MoreThuente", prm, dtype)
    assert c["status"] == "ok" and outs[0].status == 0 and outs[0].niter == c["niter"] == prm.max_iterations
    xmax = max(1.0, float(np.max(np.abs(c["x"]))))
    err = float(np.max(np.abs(X[0].astype(np.float64) - c["x"])))
    if dtype == np.float64:
        assert (c["niter"], c["nfev"]) == (c2["niter"], c2["nfev"]) == (outs[0].niter, outs[0].nfev)
        bar = max(spread_bar(c, c2), 1e-9 * xmax)
        assert abs(outs[0].fx - c["fx"]) <= max(1e-10 * max(1.0, abs(c["fx"])), 32 * abs(c["fx"] - c2["fx"]))
    else:
        bar = max(spread_bar(c, c2), 1e-2 * xmax)
    assert err <= bar, (err, bar)
    return by_op


def exported(ctx, objective, x0, prm, ls, dtype, **kw):
    got = {}
    outs, X, G, by_op = resident(ctx, objective, x0, prm, ls, on_solver=lambda s: got.setdefault("cols", history(ctx, s, dtype, x0.size)), **kw)
    return got["cols"], by_op


def check_history_is_differences(cols, its, K, grad):
    """After a solve capped at K iterations (the last pair formed after iteration K - 1), the exported columns by age a are
    x_{K-1-a} - x_{K-2-a} and grad(x_{K-1-a}) - grad(x_{K-2-a}), bit for bit."""
    for age, (s, y) in enumerate(cols):
        xe, xs = its[K - 1 - age], its[K - 2 - age]
        assert np.array_equal(s, xe - xs), ("s", age)
        assert np.array_equal(y, grad(xe) - grad(xs)), ("y", age)


@DTYPES
@pytest.mark.parametrize("m", [33, 49, 64])
def test_resident_tridiag_long_history(gpu_ctx, orc, m, dtype):
    """n = 3 SMs BT + r, r odd: every CTA owns at least three history blocks (BT = 64 in fp64 and 128 in fp32 at m >= 47), the last one
    ragged.  The capped runs match the checker within 32x its own spread between two summation orders, return grad f(x) bit for
    bit, export S/Y columns that are the explicit differences of the iterates, and a batch with per-problem data at a padded stride
    (NaN between the problems) gives every member its lone solve's bits."""
    n, bt, sms, _ = across_ctas(gpu_ctx, m, dtype, 13)
    if m >= 47:
        assert bt == (64 if dtype == np.float64 else 128)
    d, b = (v.astype(dtype) for v in po.quad_tridiag_data(n, kappa=1e3, seed=1)[:2])
    x0 = np.zeros(n, dtype)
    K, K2 = COUPLED_CAPS[m]
    # against the checker at m + 2, where its two orders still agree to a few units in the last place (further on x drifts with the
    # summation order: at 2m the orders differ by 1e-8 .. 4e-4)
    by_op = held_to_checker_long(gpu_ctx, orc, TRIDIAG, x0, d, b, lb.LBFGSParam(m=m, max_iterations=K), dtype)
    assert by_op.get("dots_form", 0) >= K - 1, by_op   # c = m > 32, and > 48 at m = 49, 64: the third round of columns
    if dtype == np.float32:   # (fp32 runs stop at m + 2)
        K2 = K
    # at about 2m: the gradient, the front, and the history below
    outs, X, G, by_op = resident(gpu_ctx, TRIDIAG, x0, lb.LBFGSParam(m=m, max_iterations=K2), "MoreThuente", data0=d, data1=b)
    assert outs[0].status == 0 and outs[0].niter == K2 and by_op.get("dots_form", 0) >= K2 - 1
    assert np.array_equal(G[0], tridiag_grad(X[0], d, b))
    cols, _ = exported(gpu_ctx, TRIDIAG, x0, lb.LBFGSParam(m=m, max_iterations=K), "MoreThuente", dtype, data0=d, data1=b)
    assert len(cols) == m
    its = capped_iterates(gpu_ctx, TRIDIAG, x0, dict(m=m), "MoreThuente", K - m - 2, K - 1, data0=d, data1=b)
    check_history_is_differences(cols, its, K, lambda x: tridiag_grad(x, d, b))
    cols, _ = exported(gpu_ctx, TRIDIAG, x0, lb.LBFGSParam(m=m, max_iterations=K2), "MoreThuente", dtype, data0=d, data1=b)
    its = capped_iterates(gpu_ctx, TRIDIAG, x0, dict(m=m), "MoreThuente", K2 - m - 2, K2 - 1, data0=d, data1=b)
    check_history_is_differences(cols, its, K2, lambda x: tridiag_grad(x, d, b))
    # a batch with per-problem data, ldd > n a multiple of 16 bytes, NaN between and after the problems
    B, ldd = 3, n + (3 if dtype == np.float64 else 7)
    assert ldd * np.dtype(dtype).itemsize % 16 == 0
    size = (B - 1) * ldd + -(-n // 32) * 32
    D, R = np.full(size, np.nan, dtype), np.full(size, np.nan, dtype)
    data = [(d, b)] + [tuple(v.astype(dtype) for v in po.quad_tridiag_data(n, kappa=1e3, seed=30 + k)[:2]) for k in (1, 2)]
    for k, (dk, bk) in enumerate(data):
        D[k * ldd:k * ldd + n], R[k * ldd:k * ldd + n] = dk, bk
    prm = lb.LBFGSParam(m=m, max_iterations=K)
    X0 = np.stack([x0, np.random.default_rng(m).uniform(-1, 1, n), np.full(n, 0.5)]).astype(dtype)
    outs, X, G, _ = resident(gpu_ctx, TRIDIAG, X0, prm, "MoreThuente", data0=D, data1=R, ldd=ldd)
    for k, (dk, bk) in enumerate(data):
        lone, Xl, Gl, _ = resident(gpu_ctx, TRIDIAG, X0[k], prm, "MoreThuente", data0=dk, data1=bk)
        assert (outs[k].status, outs[k].niter, outs[k].nfev, outs[k].fx) == (lone[0].status, lone[0].niter, lone[0].nfev, lone[0].fx)
        assert outs[k].niter == K
        assert np.array_equal(X[k], Xl[0]) and np.array_equal(G[k], Gl[0])
        assert np.array_equal(G[k], tridiag_grad(X[k], dk, bk))


# without neighbour coupling: the ring of 2M points
RING_N = 2 ** 15 + 2 * 11     # a ragged last tile
RING_K = 80                   # > 2M = 68 at m = 33: the ring has wrapped; >= 64 accepted iterates at every m: rows 64.. are in use


def ring_start(m, dtype):
    return np.random.default_rng(m).uniform(-2, 2, RING_N).astype(dtype)


@DTYPES
@pytest.mark.parametrize("m", [33, 49, 64])
def test_resident_point_ring_long_history(gpu_ctx, orc, m, dtype):
    """Paired Rosenbrock from uniform(-2, 2), capped at K = 80 (uncapped the checker takes 168-212 iterations): the pair-forming pass
    has written 80 points to the 2M = 2m + 2 rows, rows 64 and up among them, and at m = 33 the ring has wrapped.  The exported
    history is the explicit differences of the iterates, the gradient is grad f(x), a batch member is its lone solve, and the run
    matches the checker."""
    x0 = ring_start(m, dtype)
    K = RING_K
    prm = lb.LBFGSParam(m=m, max_iterations=K)
    outs, X, G, by_op = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "MoreThuente")
    assert outs[0].status == 0 and outs[0].niter == K
    assert by_op.get("dots_form", 0) >= 66 and by_op.get("dots_plain", 0) == 0, by_op   # 66 points past the start: row 64 and up
    if m == 33:
        assert by_op["dots_form"] > 2 * (m + 1)                                          # and past 2M = 68 rows: wrapped
    assert np.array_equal(G[0], rosenbrock_grad(X[0]))
    cols, _ = exported(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "MoreThuente", dtype)
    assert len(cols) == m
    its = capped_iterates(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, dict(m=m), "MoreThuente", K - m - 2, K - 1)
    check_history_is_differences(cols, its, K, rosenbrock_grad)
    # as member 1 of a batch of three: its lone solve's bits
    X0 = np.stack([np.full(RING_N, 0.5), x0, ring_start(m + 1, dtype)]).astype(dtype)
    bo, BX, BG, _ = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "MoreThuente")
    assert (bo[1].status, bo[1].niter, bo[1].nfev, bo[1].fx) == (outs[0].status, outs[0].niter, outs[0].nfev, outs[0].fx)
    assert np.array_equal(BX[1], X[0]) and np.array_equal(BG[1], G[0])
    held_to_checker_long(gpu_ctx, orc, lb.OBJ_ROSENBROCK_PAIRED, x0, None, None, prm, dtype)


@DTYPES
def test_resident_short_history_in_long_blocks(gpu_ctx, orc, dtype):
    """m = 49 (BT = 64 in fp64) stopped at c <= 3: most warps of the dots pass are forming warps."""
    m, K = 49, 3
    n = 2 ** 17 + 2 * 37
    prm = lb.LBFGSParam(m=m, max_iterations=K)
    x0 = np.random.default_rng(5).uniform(-2, 2, n).astype(dtype)
    outs, X, G, by_op = resident(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "MoreThuente")
    assert outs[0].status == 0 and outs[0].niter == K and 1 <= by_op.get("dots_form", 0) <= 3, by_op
    assert np.array_equal(G[0], rosenbrock_grad(X[0]))
    cols, _ = exported(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "MoreThuente", dtype)
    its = capped_iterates(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, x0, dict(m=m), "MoreThuente", 1, K - 1)
    its[0] = x0
    assert len(cols) == K - 1
    check_history_is_differences(cols, its, K, rosenbrock_grad)
    if dtype == np.float64:
        g = lb.LBFGSSolver(prm, "MoreThuente", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0)
        assert np.array_equal(g["x"], X[0])
        c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, LS["MoreThuente"], cpu_param(orc, prm), sum_mode=po.SUM_LANES8)
        check_parity(g, c, xtol=1e-7)


# ---- 4. the small-batch solve -------------------------------------------------------------------------------------------------
SHAPES = [lb.OBJ_ROSENBROCK_PAIRED, lb.OBJ_ROSENBROCK_CHAINED, lb.OBJ_QUAD_TRIDIAG]
SHAPE_IDS = ["paired", "chained", "tridiag"]


def small_problem(objective, n, dtype, seed):
    """(x0, d, b): paired Rosenbrock from uniform(-2, 2), chained Rosenbrock from 1.3, the tridiagonal quadratic (kappa = 1e3) from 0."""
    if objective == lb.OBJ_ROSENBROCK_PAIRED:
        return np.random.default_rng(seed).uniform(-2, 2, n).astype(dtype), None, None
    if objective == lb.OBJ_ROSENBROCK_CHAINED:
        return np.full(n, 1.3, dtype), None, None
    d, b, _ = po.quad_tridiag_data(n, kappa=1e3, seed=seed)
    return np.zeros(n, dtype), d.astype(dtype), b.astype(dtype)


def small_grad(objective, x, d, b):
    return {lb.OBJ_ROSENBROCK_PAIRED: lambda: rosenbrock_grad(x), lb.OBJ_ROSENBROCK_CHAINED: lambda: chained_grad(x),
            lb.OBJ_QUAD_TRIDIAG: lambda: tridiag_grad(x, d, b)}[objective]()


def small_case(orc, objective, n, m, dtype, cap):
    """Problem 0 of a batch of three (the others: other starts, or other data), capped at `cap`, against the checker; the returned G
    is grad f(X) bit for bit, and the problem gives the same bits at position 2 of another batch."""
    x0, d, b = small_problem(objective, n, dtype, seed=1)
    prm = lb.LBFGSParam(m=m, max_iterations=cap)
    X0 = np.stack([x0, small_problem(objective, n, dtype, 2)[0], np.full(n, 0.5, dtype)])
    res, X, G = lb.solve_small_batch(objective, X0, prm, "MoreThuente", dtype=dtype, data0=d, data1=b, want_grad=True)
    for k in range(3):
        assert res[k]["status"] == "ok", res[k]
        assert np.array_equal(G[k], small_grad(objective, X[k], d, b))
    X1 = np.stack([np.full(n, 0.25, dtype), X0[1], x0])
    res1, Xp, Gp = lb.solve_small_batch(objective, X1, prm, "MoreThuente", dtype=dtype, data0=d, data1=b, want_grad=True)
    assert res1[2] == res[0] and np.array_equal(Xp[2], X[0]) and np.array_equal(Gp[2], G[0])
    kw = dict(data0=d, data1=b, dtype=dtype)
    c = orc.lbfgs(objective, x0, LS["MoreThuente"], cpu_param(orc, prm), sum_mode=po.SUM_LANES8, **kw)
    c2 = orc.lbfgs(objective, x0, LS["MoreThuente"], cpu_param(orc, prm), sum_mode=po.SUM_SEQUENTIAL, **kw)
    assert c["status"] == "ok"
    g = res[0]
    xmax = max(1.0, float(np.max(np.abs(c["x"]))))
    if dtype == np.float64:   # the parity bar, or 32x the checker's own spread where its two orders part (random-start Rosenbrock)
        assert (c["niter"], c["nfev"]) == (c2["niter"], c2["nfev"]) == (g["niter"], g["nfev"])
        assert abs(g["fx"] - c["fx"]) <= max(1e-10 * max(1.0, abs(c["fx"])), 32 * abs(c["fx"] - c2["fx"]))
        assert np.max(np.abs(X[0] - c["x"])) <= max(1e-7 * xmax, spread_bar(c, c2))
    else:     # fp32 sums in double within one block, the checker in fp32: the bar of test_resident_exit_point
        assert abs(g["niter"] - c["niter"]) <= 3
        assert np.max(np.abs(X[0] - c["x"])) <= max(1e-2 * xmax, spread_bar(c, c2))   # (random-start Rosenbrock: the orders part)
    return c


# (m, dtype, cap): fp64 m = 33 and 49, fp32 m = 64; at the cap c has reached m for paired Rosenbrock and the quadratic
SMALL = [(33, np.float64, 66), (49, np.float64, 51), (64, np.float32, 66)]


@pytest.mark.parametrize("objective", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("m,dtype,cap", SMALL, ids=["f64-m33", "f64-m49", "f32-m64"])
def test_small_batch_at_max_n(orc, m, dtype, cap, objective):
    """n = small_max_n(m, objective): the whole solve, with its 6M^2 Gram elements, fills one CTA's shared memory."""
    n = lb.small_max_n(m, objective, dtype)
    assert n >= 64
    c = small_case(orc, objective, n, m, dtype, cap)
    if objective != lb.OBJ_ROSENBROCK_CHAINED:   # (chained Rosenbrock from 1.3 converges in 19-20 iterations)
        assert c["niter"] == cap and cap > m
    with pytest.raises(ValueError, match="exceeds"):
        lb.solve_small_batch(objective, np.zeros((2, n + 2), dtype), lb.LBFGSParam(m=m, max_iterations=cap), "MoreThuente", dtype=dtype,
                             **({} if objective != lb.OBJ_QUAD_TRIDIAG else dict(data0=np.ones(n + 2), data1=np.ones(n + 2))))


@pytest.mark.parametrize("objective,n", [(lb.OBJ_ROSENBROCK_PAIRED, 128), (lb.OBJ_ROSENBROCK_PAIRED, 130), (lb.OBJ_QUAD_TRIDIAG, 128),
                                         (lb.OBJ_QUAD_TRIDIAG, 129), (lb.OBJ_ROSENBROCK_CHAINED, 129)])
def test_small_batch_thread_switch(orc, objective, n):
    """One warp per problem up to n = 128, four warps above, at m = 33 capped at 66 iterations."""
    c = small_case(orc, objective, n, 33, np.float64, 66)
    if objective != lb.OBJ_ROSENBROCK_CHAINED:
        assert c["niter"] == 66


# ---- 5. the final approximation at c = 64 -------------------------------------------------------------------------------------
def test_hessian_times_at_m64_against_textbook_update(gpu_ctx):
    """B V and H V of the operator form (the host's 2c x 2c algebra at c = 64, a ring that wrapped) against the textbook BFGS update
    applied pair by pair to theta I, and H V against apply_Hv on the same ring."""
    n, m, npairs = 400, 64, 70
    rng = np.random.default_rng(64)
    A = rng.standard_normal((n, n))
    A = A @ A.T / n + np.eye(n)
    S = rng.standard_normal((npairs, n))
    Y = S @ A
    Sk, Yk = S[-m:], Y[-m:]
    theta = float(Yk[-1] @ Yk[-1]) / float(Sk[-1] @ Yk[-1])
    Bd = theta * np.eye(n)
    for s, y in zip(Sk, Yk):
        Bs = Bd @ s
        Bd = Bd - np.outer(Bs, Bs) / (s @ Bs) + np.outer(y, y) / (y @ s)
    Hd = np.linalg.inv(Bd)
    V = rng.standard_normal((5, n))
    drv = lb.driver()
    dp = C.POINTER(C.c_double)
    BV, HV = np.zeros((5, n)), np.zeros((5, n))
    lb._checked("hist_times", lambda *err: drv.lbfgsb200_drv_hist_times_f64(0, n, m, npairs, S.ctypes.data_as(dp), Y.ctypes.data_as(dp),
                                                                           V.ctypes.data_as(dp), V.size, BV.ctypes.data_as(dp),
                                                                           HV.ctypes.data_as(dp), *err))
    cond = np.linalg.cond(Bd)
    assert np.max(np.abs(BV - V @ Bd)) <= 1e-9 * np.max(np.abs(V @ Bd))
    assert np.max(np.abs(HV - V @ Hd)) <= 1e-12 * cond * np.max(np.abs(V @ Hd))
    h = filled(gpu_ctx, n, m, S, Y)
    assert h.ncorr == m
    res = gpu_ctx.empty(n)
    for algo in (lb.HV_GRAM, lb.HV_TWO_LOOP):
        for j in range(5):
            h.apply_Hv(gpu_ctx.array(V[j]), 1.0, res, algo)
            assert np.max(np.abs(HV[j] - res.get())) <= 1e-11 * np.max(np.abs(HV[j]))


@pytest.mark.parametrize("resident", [False, True], ids=["host_loop", "resident"])
def test_hessian_times_after_m64_solve(resident):
    """An m = 64 solve that filled its history (paired Rosenbrock from uniform(-2, 2) at n = 140, past 64 iterations): B V and H V
    of the operator form against the library's own dense final_approx_hessian / final_approx_inverse_hessian.  A consistency check
    of the two forms after a real solve, not an independent reference: test_hessian_times_at_m64_against_textbook_update holds the
    operator form's 2c x 2c host algebra at c = 64 to the textbook update."""
    n = 140
    prm = lb.LBFGSParam(m=64)
    x0 = np.random.default_rng(140).uniform(-2, 2, n)
    niter, x, Bd, Hd = lb.solve_dense(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "MoreThuente", resident=resident)
    assert niter > 64
    niter2, x2, BV, HV, HBV = lb.solve_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, x0, np.eye(n), prm, "MoreThuente", resident=resident)
    assert niter2 == niter and np.array_equal(x2, x)
    assert np.max(np.abs(BV - Bd)) <= 1e-12 * np.max(np.abs(Bd))
    tol_h = 1e-12 * max(1.0, np.linalg.cond(Bd))
    assert np.max(np.abs(HV - Hd)) <= tol_h * np.max(np.abs(Hd))
    assert np.max(np.abs(HBV - np.eye(n))) <= tol_h
