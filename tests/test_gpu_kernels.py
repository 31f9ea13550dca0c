"""GPU parity tests, kernel level: every entry point of the C ABI against the CPU checker / numpy on the same inputs.
Tolerances: element-wise kernels must be bit-exact up to FMA contraction (<= 2 ulp); reductions over n terms are compared
with |err| <= 64*eps*sum|terms| (the GPU sums in a tree, the checker sequentially -- both are valid roundings)."""
import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po

pytestmark = pytest.mark.gpu

SIZES = [1, 2, 3, 4, 5, 31, 32, 33, 1000, 4097, (1 << 20) - 1, (1 << 20) + 1]


def red_tol(terms, dtype):
    return 64 * np.finfo(dtype).eps * float(np.sum(np.abs(terms.astype(np.float64)))) + 1e-300


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("n", SIZES)
def test_level1_kernels(gpu_ctx, n, dtype):
    rng = np.random.default_rng(n)
    a, b, c = (rng.standard_normal(n).astype(dtype) for _ in range(3))
    for off in (0, 1):  # off = 1: pointers not 32-byte aligned -> element-wise path
        da, db, dc = (lb.DeviceArray(gpu_ctx, v, offset_elems=off) for v in (a, b, c))
        out = lb.DeviceArray(gpu_ctx, None, dtype, n, offset_elems=off)
        assert abs(gpu_ctx.dot(da, db) - np.dot(a.astype(np.float64), b.astype(np.float64))) <= red_tol(a * b, dtype)
        d3 = gpu_ctx.dot3(da, db, dc)
        for got, terms in zip(d3, (a * b, a * a, c * c)):
            assert abs(got - np.sum(terms.astype(np.float64))) <= red_tol(terms, dtype)
        s = dtype(0.37)
        gpu_ctx.axpy_out(da, s, db, out)
        ref = a + s * b
        assert np.max(np.abs(out.get() - ref)) <= 2 * np.finfo(dtype).eps * np.max(np.abs(a) + np.abs(s * b))
        gpu_ctx.scale_out(dtype(-1.0), da, out)
        assert np.array_equal(out.get(), -a)
        gpu_ctx.axpy_out(da, s, db, da)  # in place
        assert np.max(np.abs(da.get() - ref)) <= 2 * np.finfo(dtype).eps * np.max(np.abs(a) + np.abs(s * b))


def test_reductions_are_deterministic(gpu_ctx):
    rng = np.random.default_rng(5)
    n = 3_000_001
    a, b = lb.DeviceArray(gpu_ctx, rng.standard_normal(n)), lb.DeviceArray(gpu_ctx, rng.standard_normal(n))
    vals = {gpu_ctx.dot(a, b) for _ in range(5)}
    assert len(vals) == 1


def objective_inputs(kind, n, rng):
    x = rng.uniform(-1.5, 1.5, n)
    if kind == lb.OBJ_QUAD_TRIDIAG:
        d, b, _ = po.quad_tridiag_data(n, seed=n)
        return x, d, b
    return x, None, None


def grad_expression(kind, x, d0, d1):
    """grad f of a built-in objective, expression by expression as the kernels evaluate it (in x's dtype)."""
    from test_gpu_resident_coupled import chained_grad, tridiag_grad
    from test_gpu_resident_exit_points import rosenbrock_grad
    from test_gpu_resident_implied_grad import quad_shift_grad
    return {lb.OBJ_ROSENBROCK_PAIRED: lambda: rosenbrock_grad(x), lb.OBJ_QUAD_SHIFT: lambda: quad_shift_grad(x),
            lb.OBJ_ROSENBROCK_CHAINED: lambda: chained_grad(x), lb.OBJ_QUAD_TRIDIAG: lambda: tridiag_grad(x, d0, d1)}[kind]()


# (objective, n): odd n for the objectives that allow it (the paired Rosenbrock function needs an even n)
OBJECTIVE_SIZES = [(kind, n) for n in (2, 3, 4, 5, 6, 10, 34, 1000, 1001, 4098, (1 << 18) + 2, (1 << 18) + 3)
                   for kind in (lb.OBJ_ROSENBROCK_PAIRED, lb.OBJ_QUAD_SHIFT, lb.OBJ_ROSENBROCK_CHAINED, lb.OBJ_QUAD_TRIDIAG)
                   if not (kind == lb.OBJ_ROSENBROCK_PAIRED and n % 2)]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kind,n", OBJECTIVE_SIZES)
def test_objective_and_fused_trial(gpu_ctx, orc, kind, n, dtype):
    rng = np.random.default_rng(100 * kind + n)
    xp, d0, d1 = objective_inputs(kind, n, rng)
    drt = rng.standard_normal(n)
    step = 0.173
    if dtype == np.float32:
        xp, drt = xp.astype(dtype), drt.astype(dtype)
        d0, d1 = (None if v is None else v.astype(dtype) for v in (d0, d1))
        step = dtype(step)
    x_ref = xp + step * drt
    eps = np.finfo(dtype).eps
    D0 = lb.DeviceArray(gpu_ctx, d0) if d0 is not None else None
    D1 = lb.DeviceArray(gpu_ctx, d1) if d1 is not None else None
    dxp, dd = lb.DeviceArray(gpu_ctx, xp), lb.DeviceArray(gpu_ctx, drt)
    dx, dg = gpu_ctx.empty(n, dtype), gpu_ctx.empty(n, dtype)
    f, gd, gg, xx = gpu_ctx.trial(kind, dxp, dd, step, dx, dg, D0, D1)
    x_gpu, g_gpu = dx.get(), dg.get()
    assert np.max(np.abs(x_gpu - x_ref)) <= 2 * eps * np.max(np.abs(xp) + np.abs(step * drt))
    # gradient at the GPU's own x (separates objective arithmetic from the axpy rounding)
    f_at, g_at = orc.objective(kind, x_gpu, d0, d1)
    if dtype == np.float64:
        scale = np.max(np.abs(g_at)) + 1.0
        assert np.max(np.abs(g_gpu - g_at)) <= 1e-13 * scale * 10
        assert abs(f - f_at) <= 1e-12 * max(1.0, abs(f_at))
        f_ref, _ = orc.objective(kind, x_ref, d0, d1)
        assert abs(f_ref - f) <= 1e-9 * max(1.0, abs(f_ref))
    else:   # fp32: the expression in fp32, bit for bit (no FMA contraction); f summed in fp32
        assert np.array_equal(g_gpu, grad_expression(kind, x_gpu, d0, d1))
        assert abs(f - f_at) <= 1e-4 * max(1.0, abs(f_at))
    g64 = g_at if dtype == np.float64 else g_gpu.astype(np.float64)
    assert abs(gd - np.dot(g64, drt)) <= red_tol(g64 * drt, dtype) * 4
    assert abs(gg - np.dot(g64, g64)) <= red_tol(g64 * g64, dtype) * 4
    assert abs(xx - np.dot(x_gpu.astype(np.float64), x_gpu)) <= red_tol(x_gpu.astype(np.float64) * x_gpu, dtype) * 4
    # plain evaluation entry point
    dg2 = gpu_ctx.empty(n, dtype)
    f2, _, gg2, xx2 = gpu_ctx.objective(kind, dx, dg2, D0, D1)
    assert np.array_equal(dg2.get(), g_gpu) and f2 == f and gg2 == gg and xx2 == xx


def test_paired_rosenbrock_rejects_odd_n(gpu_ctx):
    x, g = gpu_ctx.empty(7), gpu_ctx.empty(7)
    with pytest.raises(lb.LbfgsB200Error) as e:
        gpu_ctx.objective(lb.OBJ_ROSENBROCK_PAIRED, x, g)
    assert e.value.status == 1


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_history_update_and_gate(gpu_ctx, dtype):
    n, m = 1003, 3
    rng = np.random.default_rng(9)
    h = lb.History(gpu_ctx, n, m, dtype)
    xs = [rng.standard_normal(n).astype(dtype) for _ in range(6)]
    gs = [(2.0 * x + 0.05 * rng.standard_normal(n)).astype(dtype) for x in xs]
    for k in range(1, 6):
        x, xp, g, gp = (lb.DeviceArray(gpu_ctx, v) for v in (xs[k], xs[k - 1], gs[k], gs[k - 1]))
        ok, sy, yy = h.update(x, xp, g, gp)
        s, y = xs[k] - xs[k - 1], gs[k] - gs[k - 1]
        assert ok and h.ncorr == min(k, m)
        assert np.array_equal(h.column("s", 0), s) and np.array_equal(h.column("y", 0), y)   # bit exact
        assert abs(sy - np.dot(s.astype(np.float64), y.astype(np.float64))) <= red_tol(s * y, dtype)
        theta, ys, _ = h.scalars()
        assert np.isclose(theta, yy / sy, rtol=4 * np.finfo(dtype).eps) and ys[0] == dtype(sy)
        if k >= 2:  # older pairs stay where they were
            assert np.array_equal(h.column("s", 1), xs[k - 1] - xs[k - 2])
    # a pair with negative curvature is rejected and leaves the ring untouched, even when it is full
    before = [h.column("s", a) for a in range(m)]
    theta0 = h.scalars()[0]
    x, xp = lb.DeviceArray(gpu_ctx, xs[1]), lb.DeviceArray(gpu_ctx, xs[0])
    g, gp = lb.DeviceArray(gpu_ctx, gs[0]), lb.DeviceArray(gpu_ctx, gs[1])  # y = -(g1-g0)
    ok, sy, yy = h.update(x, xp, g, gp)
    assert not ok and sy < 0 and h.ncorr == m
    assert all(np.array_equal(h.column("s", a), before[a]) for a in range(m)) and h.scalars()[0] == theta0


HV_CASES = [(7, 3, 0), (7, 3, 1), (7, 3, 2), (7, 3, 3), (7, 3, 8), (130, 6, 17), (1001, 10, 10), (100003, 10, 25),
            (1 << 20, 6, 7), (4099, 20, 20)]


@pytest.mark.parametrize("algo", [lb.HV_TWO_LOOP, lb.HV_AUTO])
@pytest.mark.parametrize("n,m,npairs", HV_CASES)
def test_apply_Hv_against_checker(gpu_ctx, orc, n, m, npairs, algo):
    rng = np.random.default_rng(n + 31 * m + npairs)
    S = rng.standard_normal((npairs, n))
    Y = S + 0.1 * rng.standard_normal((npairs, n))
    v = rng.standard_normal(n)
    ref, ys_ref, theta_ref = orc.apply_Hv(S, Y, v, -1.0, m)
    h = lb.History(gpu_ctx, n, m)
    for k in range(npairs):
        h.add(lb.DeviceArray(gpu_ctx, S[k]), lb.DeviceArray(gpu_ctx, Y[k]))
    dv, dres = lb.DeviceArray(gpu_ctx, v), gpu_ctx.empty(n)
    vdot = h.apply_Hv(dv, -1.0, dres, algo, want_dot=True)
    res = dres.get()
    scale = np.max(np.abs(ref))
    assert np.max(np.abs(res - ref)) <= 1e-11 * scale
    assert abs(vdot - np.dot(v, res)) <= red_tol(v * res, np.float64) * 4
    if npairs:
        theta, ys, _ = h.scalars()
        assert np.isclose(theta, theta_ref, rtol=1e-13)
    # run-to-run determinism
    h.apply_Hv(dv, -1.0, dres, algo)
    assert np.array_equal(dres.get(), res)


def test_apply_Hv_golden_vectors(gpu_ctx):
    """The vectors frozen from the unmodified reference headers (tests/golden/make_golden.py)."""
    from util import golden_cases, unhex
    for c in golden_cases("apply_Hv"):
        n, npairs, m = c["n"], c["npairs"], c["m"]
        S, Y = unhex(c["S"]).reshape(npairs, n), unhex(c["Y"]).reshape(npairs, n)
        h = lb.History(gpu_ctx, n, m)
        for k in range(npairs):
            h.add(lb.DeviceArray(gpu_ctx, S[k]), lb.DeviceArray(gpu_ctx, Y[k]))
        dres = gpu_ctx.empty(n)
        h.apply_Hv(lb.DeviceArray(gpu_ctx, unhex(c["v"])), c["a"], dres, lb.HV_TWO_LOOP)
        ref = unhex(c["res"])
        assert np.max(np.abs(dres.get() - ref)) <= 1e-12 * np.max(np.abs(ref)), c["name"]


def test_apply_Hv_float32(gpu_ctx, orc):
    n, m, npairs = 5001, 5, 9
    rng = np.random.default_rng(2)
    S = rng.standard_normal((npairs, n)).astype(np.float32)
    Y = (S + 0.1 * rng.standard_normal((npairs, n))).astype(np.float32)
    v = rng.standard_normal(n).astype(np.float32)
    ref, _, _ = orc.apply_Hv(S.astype(np.float64), Y.astype(np.float64), v.astype(np.float64), -1.0, m)
    h = lb.History(gpu_ctx, n, m, np.float32)
    for k in range(npairs):
        h.add(lb.DeviceArray(gpu_ctx, S[k]), lb.DeviceArray(gpu_ctx, Y[k]))
    dres = gpu_ctx.empty(n, np.float32)
    h.apply_Hv(lb.DeviceArray(gpu_ctx, v), np.float32(-1.0), dres)
    assert np.max(np.abs(dres.get() - ref)) <= 2e-4 * np.max(np.abs(ref))


def test_bad_arguments_are_reported(gpu_ctx):
    with pytest.raises(lb.LbfgsB200Error) as e:
        lb.History(gpu_ctx, 10, 0)
    assert e.value.status == 1
    h = lb.History(gpu_ctx, 10, 3)
    v = gpu_ctx.empty(10)
    with pytest.raises(lb.LbfgsB200Error):
        h.apply_Hv(v, -1.0, v)  # aliasing
    h32 = lb.History(gpu_ctx, 10, 3, np.float32)
    with pytest.raises(lb.LbfgsB200Error):
        gpu_ctx.check(gpu_ctx.lib.lbfgs_b200_hist_apply_Hv_f64(h32.h, v.ptr, -1.0, gpu_ctx.empty(10).ptr, 0, None))


@pytest.mark.parametrize("n,m,npairs", [(6, 3, 0), (6, 3, 2), (12, 4, 4), (12, 4, 9), (40, 6, 6)])
def test_dense_hessian_approximations(n, m, npairs):
    """final_approx_hessian / final_approx_inverse_hessian (reference BFGSMat.h:150-271) against the textbook BFGS update applied
    pair by pair to B0 = theta*I (independent of the compact representation used on both sides)."""
    import ctypes as C
    rng = np.random.default_rng(n + npairs)
    S = rng.standard_normal((npairs, n))
    A = rng.standard_normal((n, n))
    A = A @ A.T / n + np.eye(n)                      # y = A s: consistent curvature
    Y = S @ A
    Sk, Yk = S[-m:], Y[-m:]
    theta = float(Yk[-1] @ Yk[-1]) / float(Sk[-1] @ Yk[-1]) if npairs else 1.0
    B = theta * np.eye(n)
    for s, y in zip(Sk, Yk):
        Bs = B @ s
        B = B - np.outer(Bs, Bs) / (s @ Bs) + np.outer(y, y) / (y @ s)
    drv = lb.driver()
    dp = C.POINTER(C.c_double)
    err = C.create_string_buffer(256)
    for inverse, ref in ((0, B), (1, np.linalg.inv(B))):
        out = np.zeros((n, n))
        Sc, Yc = np.ascontiguousarray(S), np.ascontiguousarray(Y)
        st = drv.lbfgsb200_drv_dense_f64(0, n, m, npairs, Sc.ctypes.data_as(dp) if npairs else None,
                                         Yc.ctypes.data_as(dp) if npairs else None, inverse, out.ctypes.data_as(dp), err, 256)
        assert st == 0, err.value
        assert np.max(np.abs(out - ref)) <= 1e-9 * np.max(np.abs(ref))


@pytest.mark.parametrize("n", [10, 2048, 2052, 100_003, (1 << 20) + 4])
@pytest.mark.parametrize("m,prior", [(4, 0), (4, 1), (4, 4), (4, 6), (10, 3), (20, 25)])
def test_fused_update_apply_Hv_matches_separate_calls(gpu_ctx, n, m, prior):
    """lbfgs_b200_hist_update_apply_Hv (pair formed inside the dots pass) == hist_update followed by apply_Hv."""
    rng = np.random.default_rng(1000 * m + prior + n)
    ha, hb = lb.History(gpu_ctx, n, m), lb.History(gpu_ctx, n, m)
    for _ in range(prior):
        s = rng.standard_normal(n)
        y = s + 0.1 * rng.standard_normal(n)
        ds, dy = gpu_ctx.array(s), gpu_ctx.array(y)
        ha.add(ds, dy)
        hb.add(ds, dy)
    xp, gp = rng.standard_normal(n), rng.standard_normal(n)
    s = 0.3 * rng.standard_normal(n)
    x, g = xp + s, gp + s + 0.1 * rng.standard_normal(n)
    dx, dxp, dg, dgp = (gpu_ctx.array(v) for v in (x, xp, g, gp))
    ra, rb_ = gpu_ctx.empty(n), gpu_ctx.empty(n)
    acc_a, _, _ = ha.update(dx, dxp, dg, dgp)
    dot_a = ha.apply_Hv(dg, -1.0, ra, lb.HV_GRAM, want_dot=True)
    acc_b, dot_b = hb.update_apply_Hv(dx, dxp, dg, dgp, -1.0, rb_, lb.HV_GRAM)
    assert acc_a and acc_b and ha.ncorr == hb.ncorr == min(prior + 1, m)
    assert np.array_equal(ha.column("s", 0), hb.column("s", 0)) and np.array_equal(ha.column("y", 0), hb.column("y", 0))
    assert np.array_equal(hb.column("s", 0), x - xp) and np.array_equal(hb.column("y", 0), g - gp)
    ta, ysa, _ = ha.scalars()
    tb, ysb, _ = hb.scalars()
    assert abs(ta - tb) <= 1e-13 * abs(ta) and np.max(np.abs(ysa - ysb)) <= 1e-13 * np.max(np.abs(ysa))
    va, vb = ra.get(), rb_.get()
    assert np.max(np.abs(va - vb)) <= 1e-11 * (np.max(np.abs(va)) + 1e-300)
    assert abs(dot_a - dot_b) <= 1e-11 * abs(dot_a)
    # a second round on top (exercises the fold of the pair committed by the fused call)
    x2 = x + 0.2 * rng.standard_normal(n)
    g2 = g + (x2 - x) + 0.05 * rng.standard_normal(n)
    dx2, dg2 = gpu_ctx.array(x2), gpu_ctx.array(g2)
    ha.update(dx2, dx, dg2, dg)
    dot_a = ha.apply_Hv(dg2, -1.0, ra, lb.HV_GRAM, want_dot=True)
    _, dot_b = hb.update_apply_Hv(dx2, dx, dg2, dg, -1.0, rb_, lb.HV_GRAM)
    va, vb = ra.get(), rb_.get()
    assert np.max(np.abs(va - vb)) <= 1e-10 * (np.max(np.abs(va)) + 1e-300)
    assert abs(dot_a - dot_b) <= 1e-10 * abs(dot_a)
    # literal two-loop on the history built by the fused calls: an independent algorithm on the same ring
    hb.apply_Hv(dg2, -1.0, ra, lb.HV_TWO_LOOP)
    assert np.max(np.abs(ra.get() - vb)) <= 1e-10 * (np.max(np.abs(vb)) + 1e-300)


@pytest.mark.parametrize("prior", [0, 2, 5])
def test_fused_update_apply_Hv_rejected_pair_leaves_history_untouched(gpu_ctx, prior):
    """y = 0 fails the curvature gate s'y > eps*y'y: the old history must answer (reference LBFGS.h:161-165)."""
    n, m = 50_000, 4
    rng = np.random.default_rng(prior)
    h = lb.History(gpu_ctx, n, m)
    for _ in range(prior):
        s = rng.standard_normal(n)
        ds, dy = gpu_ctx.array(s), gpu_ctx.array(s + 0.1 * rng.standard_normal(n))
        h.add(ds, dy)
    before = h.ncorr
    xp, g = rng.standard_normal(n), rng.standard_normal(n)
    dx, dxp, dg = gpu_ctx.array(xp + 0.1), gpu_ctx.array(xp), gpu_ctx.array(g)
    res, ref = gpu_ctx.empty(n), gpu_ctx.empty(n)
    acc, dot = h.update_apply_Hv(dx, dxp, dg, dg, -1.0, res, lb.HV_GRAM)
    assert not acc and h.ncorr == before
    h.apply_Hv(dg, -1.0, ref, lb.HV_TWO_LOOP)
    r = ref.get()
    assert np.max(np.abs(res.get() - r)) <= 1e-11 * np.max(np.abs(r))
    assert abs(dot - np.dot(g, r)) <= 1e-10 * abs(np.dot(g, r))
    # and the ring still accepts the next good pair
    x2, g2 = xp + 0.3 * rng.standard_normal(n), None
    g2 = g + (x2 - xp) * 1.5
    acc, _ = h.update_apply_Hv(gpu_ctx.array(x2), dxp, gpu_ctx.array(g2), dg, -1.0, res, lb.HV_GRAM)
    assert acc and h.ncorr == min(before + 1, m)


def test_fused_update_apply_Hv_unaligned_falls_back(gpu_ctx):
    n, m = 10_001, 3
    rng = np.random.default_rng(2)
    xp, gp = rng.standard_normal(n), rng.standard_normal(n)
    x, g = xp + 0.1 * rng.standard_normal(n), gp + 0.2 * rng.standard_normal(n)
    g = gp + (x - xp) * 2.0
    outs = []
    for off in (0, 1):
        h = lb.History(gpu_ctx, n, m)
        arrs = [lb.DeviceArray(gpu_ctx, v, offset_elems=off) for v in (x, xp, g, gp)]
        res = lb.DeviceArray(gpu_ctx, None, np.float64, n, offset_elems=off)
        acc, dot = h.update_apply_Hv(*arrs, -1.0, res, lb.HV_AUTO)
        assert acc
        outs.append((res.get(), dot))
    assert np.max(np.abs(outs[0][0] - outs[1][0])) <= 1e-12 * np.max(np.abs(outs[0][0]))
    assert abs(outs[0][1] - outs[1][1]) <= 1e-12 * abs(outs[0][1])


@pytest.mark.parametrize("n", [2048, 20_000, 300_001])
def test_fused_update_apply_Hv_float32(gpu_ctx, n):
    """The fp32 instantiation of the pair-forming dots pass (TMA tiles of 2048 floats) against the separate calls."""
    m, prior = 5, 7
    rng = np.random.default_rng(n)
    f32 = np.float32
    ha, hb = lb.History(gpu_ctx, n, m, f32), lb.History(gpu_ctx, n, m, f32)
    for _ in range(prior):
        s = rng.standard_normal(n).astype(f32)
        y = (s + 0.1 * rng.standard_normal(n)).astype(f32)
        ds, dy = gpu_ctx.array(s), gpu_ctx.array(y)
        ha.add(ds, dy)
        hb.add(ds, dy)
    xp, gp = rng.standard_normal(n).astype(f32), rng.standard_normal(n).astype(f32)
    s = (0.3 * rng.standard_normal(n)).astype(f32)
    x = (xp + s).astype(f32)
    g = (gp + s + 0.1 * rng.standard_normal(n)).astype(f32)
    dx, dxp, dg, dgp = (gpu_ctx.array(v) for v in (x, xp, g, gp))
    ra, rb_ = gpu_ctx.empty(n, f32), gpu_ctx.empty(n, f32)
    acc_a, _, _ = ha.update(dx, dxp, dg, dgp)
    dot_a = ha.apply_Hv(dg, f32(-1.0), ra, lb.HV_GRAM, want_dot=True)
    acc_b, dot_b = hb.update_apply_Hv(dx, dxp, dg, dgp, f32(-1.0), rb_, lb.HV_GRAM)
    assert acc_a and acc_b and ha.ncorr == hb.ncorr == m
    assert np.array_equal(hb.column("s", 0), x - xp) and np.array_equal(hb.column("y", 0), g - gp)
    va, vb = ra.get(), rb_.get()
    assert np.max(np.abs(va - vb)) <= 2e-4 * np.max(np.abs(va))
    assert abs(dot_a - dot_b) <= 2e-4 * abs(dot_a)


def test_device_memory_pool_hands_released_blocks_out_again():
    """Blocks released through the ABI stay with the context and come back on an exact size match (internal.cuh: pool_alloc), so the
    reference's reallocate-per-minimize() pattern costs no cudaMalloc / cudaFree; lbfgs_b200_trim returns them to the driver."""
    ctx = lb.Context(0)
    a = ctx.array(np.arange(5000.0))
    pa = a.base.value
    del a
    b = ctx.empty(5000)                      # same size: the same block
    assert b.base.value == pa
    c = ctx.empty(5000)                      # the pool is empty again: a fresh block
    assert c.base.value not in (pa, None)
    d = ctx.empty(7001)                      # another size never reuses it
    assert d.base.value not in (pa, c.base.value)
    # a recycled block starts with a cleared last line (ragged tails are read as whole 256-byte lines)
    e = ctx.array(np.full(5000 + 13, 7.0))
    pe = e.base.value
    del e
    f = ctx.empty(5000 + 13)
    assert f.base.value == pe
    tail = lb.DeviceArray(ctx, None, np.float64, 32, offset_elems=0)   # (only to keep the API exercised)
    del tail
    h = lb.History(ctx, 4096, 5)
    del h
    h2 = lb.History(ctx, 4096, 5)            # a history rebuilt from its own released blocks still works
    s = np.random.default_rng(0).standard_normal(4096)
    h2.add(ctx.array(s), ctx.array(s + 0.1))
    res = ctx.empty(4096)
    h2.apply_Hv(ctx.array(s), -1.0, res, lb.HV_AUTO)
    assert np.all(np.isfinite(res.get()))
    del b, c, d, f, h2, res
    ctx.trim()
    g = ctx.empty(5000)                      # after a trim the pool starts over
    assert g.base.value is not None
    del g
    ctx.close()

