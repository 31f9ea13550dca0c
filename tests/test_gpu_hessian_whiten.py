"""Whitening and log densities under N(x*, H) of the final L-BFGS approximation on the GPU: the large-n dots passes
(lbfgs_b200_hist_s_dot_multi / _wt_dot_diff) bit for bit against hist_wt_dot_multi, the front's L', L^-1, L^-T and log density against
the dense factor and scipy, whitening of the library's own draws, and the small-batch ops and log density
(lbfgs_b200_small_hist_factor_apply / _log_density) against dense references, with bit identity across positions, ranges and k."""
import numpy as np
import pytest

import lbfgspp_b200 as lb
from test_gpu_hessian_ops import seeded_ring
from test_gpu_hessian_sample import LINE_SEARCHES, normals, rel_err, run_factor
from test_gpu_small_batch_hessian import MAXIT, OBJECTIVES, kept, problem, solve_keep
from test_hessian_sample_cpu import bfgs_dense_inverse

pytestmark = pytest.mark.gpu
LOG2PI = np.log(2 * np.pi)


# ---- the large-n passes ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("m,npairs", [(3, 0), (3, 3), (10, 13), (64, 64)])
def test_large_n_dots_bit_identical(gpu_ctx, dtype, m, npairs):
    n, k = 20_001, 16
    h, Y, S = seeded_ring(gpu_ctx, n, m, npairs, dtype, seed=7 * m + npairs)
    c = h.ncorr
    rng = np.random.default_rng(m + npairs)
    X = rng.standard_normal((k, n)).astype(dtype)
    mean = rng.standard_normal(n).astype(dtype)
    Xd, md = gpu_ctx.array(X.reshape(-1)), gpu_ctx.array(mean)
    # S'V: the s rows of [Y S]'V, bit for bit
    SV = h.s_dot_multi(Xd, k, n)
    assert SV.shape == (c, k)
    if c:
        assert np.array_equal(SV, h.wt_dot_multi(Xd, k, n)[c:])
    # [Y S]'(X - mean) against [Y S]'V on V = X - mean formed by axpy_out, and the norms against float64
    Vh = np.zeros((k, n), dtype=dtype)
    one = gpu_ctx.array(np.zeros(n, dtype=dtype))
    for j in range(k):
        gpu_ctx.axpy_out(gpu_ctx.array(X[j]), dtype(-1), md, one)
        Vh[j] = one.get()
    assert np.array_equal(Vh, (X - mean).astype(dtype))
    R, nrm = h.wt_dot_diff(Xd, k, n, md)
    if c:
        assert np.array_equal(R.astype(dtype), h.wt_dot_multi(gpu_ctx.array(Vh.reshape(-1)), k, n))
    ref = np.sum(Vh.astype(np.float64) ** 2, axis=1)
    assert np.allclose(nrm, ref, rtol=1e-13, atol=0)
    # column j of a k = 16 call is the k = 1 call on that column
    for j in (0, 9, 15):
        Xj = gpu_ctx.array(X[j])
        if c:
            assert np.array_equal(h.s_dot_multi(Xj, 1, n)[:, 0], SV[:, j])
        Rj, nj = h.wt_dot_diff(Xj, 1, n, md)
        assert nj[0] == nrm[j]
        if c:
            assert np.array_equal(Rj[:, 0], R[:, j])


def test_large_n_error_paths(gpu_ctx):
    h, _, _ = seeded_ring(gpu_ctx, 100, 3, 3, np.float64, seed=1)
    V = gpu_ctx.array(np.zeros(17 * 100))
    for k, ld in ((0, 100), (17, 100), (1, 99)):
        with pytest.raises(lb.LbfgsB200Error):
            h.s_dot_multi(V, k, ld)
        with pytest.raises(lb.LbfgsB200Error):
            h.wt_dot_diff(V, k, ld, V)


# ---- the front, through the driver ---------------------------------------------------------------------------------------------------
def dense_factor(ls, resident, x0, prm):
    """L column by column from the existing factor product, and the solution."""
    n = x0.size
    _, x, L = lb.solve_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, x0, np.eye(n), "L", prm, ls, resident=resident)
    return x, L.T


@pytest.mark.parametrize("resident", [False, True], ids=["host_loop", "resident"])
@pytest.mark.parametrize("ls", LINE_SEARCHES)
def test_front_against_dense(resident, ls):
    stats = pytest.importorskip("scipy.stats")
    for n, m in ((2, 3), (18, 10), (300, 10), (300, 64)):
        prm = lb.LBFGSParam(m=m)
        x0 = np.linspace(-1, 1, n)
        x, L = dense_factor(ls, resident, x0, prm)
        cond = np.linalg.cond(L) ** 2
        tol = 1e-12 * min(max(1.0, cond), 1e3)
        V = np.random.default_rng(n + m).standard_normal((5, n))
        out = {}
        for op, want in (("LT", V @ L), ("LINV", np.linalg.solve(L, V.T).T), ("LINVT", np.linalg.solve(L.T, V.T).T)):
            _, x2, O = lb.solve_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, x0, V, op, prm, ls, resident=resident)
            assert np.array_equal(x2, x)
            assert rel_err(O, want) <= tol, (n, m, op, cond, rel_err(O, want))
            out[op] = O
        # round trips: L^-1 (L V) = V and L^-T (L' V) = V
        _, _, LV = lb.solve_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, x0, V, "L", prm, ls, resident=resident)
        _, _, back = lb.solve_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, x0, LV, "LINV", prm, ls, resident=resident)
        assert rel_err(back, V) <= tol
        _, _, backt = lb.solve_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, x0, out["LT"], "LINVT", prm, ls, resident=resident)
        assert rel_err(backt, V) <= tol
        # |L^-1 v|^2 = v'(B v), B v from the compact products (final_approx_hessian_times)
        H = L @ L.T
        _, _, BV, _, _ = lb.solve_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, x0, V, prm, ls, resident=resident)
        q = np.einsum("ij,ij->i", V, BV)
        assert np.allclose(np.sum(out["LINV"] ** 2, axis=1), q, rtol=tol, atol=0)
        # the log density against scipy at points around the solution
        P = x + 0.1 * V
        _, _, lp = lb.solve_hessian_log_density(lb.OBJ_ROSENBROCK_PAIRED, x0, P, None, prm, ls, resident=resident)
        want = stats.multivariate_normal(mean=x, cov=H, allow_singular=True).logpdf(P)
        assert np.allclose(lp, want, rtol=tol, atol=tol * n), (n, m, lp, want)


def test_whitening_the_library_draws():
    """L^-1 (draw - mean) returns the normals of the generator; their log densities are -|z|^2/2 - log det H/2 - n log(2 pi)/2."""
    n, m, seed, first, k = 200, 10, 99, 4, 6
    prm = lb.LBFGSParam(m=m)
    x0 = np.linspace(-1, 1, n)
    _, x, _, D, ld = lb.solve_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, x0, None, seed, first, k, prm, "MoreThuente")
    Z = np.stack([normals(seed, 0, first + j, n) for j in range(k)])
    _, _, Zb = lb.solve_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, x0, D - x, "LINV", prm, "MoreThuente")
    assert rel_err(Zb, Z) <= 1e-9
    _, _, lp = lb.solve_hessian_log_density(lb.OBJ_ROSENBROCK_PAIRED, x0, D, None, prm, "MoreThuente")
    want = -0.5 * np.sum(Z ** 2, axis=1) - 0.5 * ld - 0.5 * n * LOG2PI
    assert np.allclose(lp, want, rtol=1e-9, atol=1e-8 * n)


def test_front_batch_member_bit_identical():
    n, B = 1000, 3
    X0 = np.stack([np.random.default_rng(3000 + p).uniform(-1, 1, n) for p in range(B)])
    prm = lb.LBFGSParam(m=10)
    V = np.random.default_rng(6).standard_normal((3, n))
    for op in ("LT", "LINV", "LINVT"):
        _, O0 = lb.batch_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, X0, 0, V, op, prm, "MoreThuente")
        _, _, O1 = lb.solve_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, X0[0], V, op, prm, "MoreThuente", resident=True)
        assert np.array_equal(O0, O1), op
    X, lp0 = lb.batch_hessian_log_density(lb.OBJ_ROSENBROCK_PAIRED, X0, 0, X0[0] + 0.01 * V, None, prm, "MoreThuente")
    _, _, lp1 = lb.solve_hessian_log_density(lb.OBJ_ROSENBROCK_PAIRED, X0[0], X0[0] + 0.01 * V, None, prm, "MoreThuente", resident=True)
    assert np.array_equal(lp0, lp1)
    with pytest.raises(RuntimeError, match="problem index out of range"):
        lb.batch_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, X0, B, V, "LT", prm, "MoreThuente")


def test_log_density_at_n_1e6_against_a_float64_recomputation():
    """BFGSMat::log_density at n = 1e6: q = v'B v on an orthonormal basis Q of span [S Y] plus theta |(I - QQ')v|^2."""
    n, npairs, m = 1_000_000, 13, 10
    rng = np.random.default_rng(78)
    d = 1.0 + rng.random(n)
    S = rng.standard_normal((npairs, n))
    Y = S * d + 0.01 * rng.standard_normal((npairs, n))
    mean = rng.standard_normal(n)
    X = mean + 0.3 * rng.standard_normal((3, n))
    lp = lb.hist_hessian_log_density(S, Y, X, mean, m=m)
    _, _, ld = lb.hist_sample(S, Y, m=m, k=0)
    kS, kY = S[::-1][:m], Y[::-1][:m]
    c = kS.shape[0]
    theta = kY[0] @ kY[0] / (kS[0] @ kY[0])
    Q, _ = np.linalg.qr(np.concatenate([kS, kY]).T)
    s_, y_ = kS @ Q, kY @ Q
    Bt = theta * np.eye(2 * c)
    for s, y in zip(s_[::-1], y_[::-1]):
        Bs = Bt @ s
        Bt = Bt - np.outer(Bs, Bs) / (s @ Bs) + np.outer(y, y) / (y @ s)
    for j in range(3):
        v = X[j] - mean
        a = Q.T @ v
        q = a @ Bt @ a + theta * (v @ v - a @ a)
        want = -0.5 * q - 0.5 * ld - 0.5 * n * LOG2PI
        assert abs(lp[j] - want) <= 1e-9 * abs(want), (lp[j], want)


def test_hist_errors_and_zero_pairs():
    n = 50
    S = np.zeros((0, n))
    V = np.random.default_rng(2).standard_normal((2, n))
    # without pairs L^-1 = L^-T = sqrt(theta) I and L' = I / sqrt(theta)
    Li = lb.hist_hessian_factor(S, S, V, "LINV", m=3)
    sq = Li[0, 0] / V[0, 0]
    assert sq > 0 and np.allclose(Li, sq * V, rtol=1e-15, atol=0)
    assert np.allclose(lb.hist_hessian_factor(S, S, V, "LINVT", m=3), sq * V, rtol=1e-15, atol=0)
    assert np.allclose(lb.hist_hessian_factor(S, S, V, "LT", m=3), V / sq, rtol=1e-15, atol=0)
    lp = lb.hist_hessian_log_density(S, S, V, np.zeros(n), m=3)
    theta = sq * sq
    assert np.allclose(lp, -0.5 * theta * np.sum(V ** 2, axis=1) + 0.5 * n * np.log(theta) - 0.5 * n * LOG2PI, rtol=1e-13)
    with pytest.raises(RuntimeError, match="op must be"):
        lb.hist_hessian_factor(S, S, V, 4, m=3)
    with pytest.raises(RuntimeError, match="need a mean"):
        lb.hist_hessian_log_density(S, S, V, None, m=3)


# ---- the small batch -------------------------------------------------------------------------------------------------------------------
def run_op(ctx, h, op, b0, count, k, V):
    n = h.n
    O = ctx.array(np.full(count * k * n, np.nan, dtype=h.dtype))
    h.factor_apply(op, b0, count, k, ctx.array(V.reshape(-1)), n, k * n, O, n, k * n)
    return O.get().reshape(count, k, n)


def run_density(ctx, h, b0, count, k, X, MEAN):
    n = h.n
    return h.log_density(b0, count, k, ctx.array(X.reshape(-1)), n, k * n, ctx.array(MEAN.reshape(-1)), n)


def check_small(gpu_ctx, objective, n, m, dtype, B=3, its=MAXIT):
    X0, d0, d1, ldd = problem(objective, B, n, 700 + n + m, dtype)
    h, _, _, _ = solve_keep(gpu_ctx, objective, X0, lb.LBFGSParam(m=m, max_iterations=its), "MoreThuente", d0, d1, ldd)
    c_all, th = h.info()
    I = np.tile(np.eye(n, dtype=dtype), (B, 1, 1))
    L_all = run_factor(gpu_ctx, h, 0, B, n, I)
    # op L is factor_times, bit for bit
    assert np.array_equal(run_op(gpu_ctx, h, "L", 0, B, n, I), L_all)
    k = 5
    rng = np.random.default_rng(n * m)
    V = rng.standard_normal((B, k, n)).astype(dtype)
    MEAN = rng.standard_normal((B, n)).astype(dtype)
    P = (MEAN[:, None, :] + 0.5 * V).astype(dtype)
    outs = {op: run_op(gpu_ctx, h, op, 0, B, k, V) for op in ("LT", "LINV", "LINVT")}
    lp = run_density(gpu_ctx, h, 0, B, k, P, MEAN)
    ld = h.logdet()
    for b in range(B):
        L = L_all[b].T.astype(np.float64)
        S, Y, _, _, _, _, theta = kept(h, b)
        Hm = bfgs_dense_inverse(S, Y, theta)
        cond = np.linalg.cond(Hm)
        tol = 1e-12 * min(max(1.0, cond), 1e3) if dtype == np.float64 else 1e-4 * min(max(1.0, cond), 1e2)
        Vb = V[b].astype(np.float64)
        # the inverses are checked against solves with L as the factor product gave it, so that product's own error is amplified by
        # the solve too: in fp32 their bar's cap on cond(H) is that of fp64 (1e3), with histories of more pairs than coordinates
        tol_inv = tol if dtype == np.float64 else 1e-4 * min(max(1.0, cond), 1e3)
        for op, want, bar in (("LT", Vb @ L, tol), ("LINV", np.linalg.solve(L, Vb.T).T, tol_inv), ("LINVT", np.linalg.solve(L.T, Vb.T).T, tol_inv)):
            assert rel_err(outs[op][b].astype(np.float64), want) <= bar, (objective, n, m, b, op, int(c_all[b]), cond)
        Db = (P[b] - MEAN[b]).astype(np.float64)
        q = np.einsum("ij,ij->i", Db, np.linalg.solve(Hm, Db.T).T)
        want = -0.5 * q - 0.5 * ld[b] - 0.5 * n * LOG2PI
        assert np.allclose(lp[b], want, rtol=tol, atol=tol * max(1.0, np.max(np.abs(q)))), (objective, n, m, b, lp[b], want)
        # one problem alone, one vector at a time: the same bits
        for op in ("LT", "LINV", "LINVT"):
            assert np.array_equal(run_op(gpu_ctx, h, op, b, 1, 1, V[b, 2:3][None])[0, 0], outs[op][b, 2]), op
        assert np.array_equal(run_density(gpu_ctx, h, b, 1, 1, P[b, 2:3][None], MEAN[b:b + 1])[0, 0], lp[b, 2])
        if c_all[b] == 0:
            s = np.sqrt(float(th[b]))
            assert np.allclose(outs["LINV"][b], s * V[b], rtol=4 * np.finfo(dtype).eps, atol=0)
    return h


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("objective", OBJECTIVES)
def test_small_batch_against_dense(gpu_ctx, objective, dtype):
    for n, m in ((2, 3), (18, 10), (300, 10), (18, 20)):
        check_small(gpu_ctx, objective, n, m, dtype)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_small_batch_at_the_edge_of_the_budget(gpu_ctx, dtype):
    obj = lb.OBJ_ROSENBROCK_PAIRED
    check_small(gpu_ctx, obj, lb.small_max_n(10, obj, dtype), 10, dtype, B=2)
    m_big = max(m for m in range(1, 65) if lb.small_max_n(m, obj, dtype) >= 4)
    n_big = lb.small_max_n(m_big, obj, dtype)
    check_small(gpu_ctx, obj, n_big, m_big, dtype, B=2, its=max(2, n_big // 2))


def test_small_batch_positions_ranges_and_k(gpu_ctx):
    """A problem's outputs do not depend on its position, b0, count or k."""
    n, m, k = 40, 6, 20
    p = np.random.default_rng(11).uniform(-1.2, 1.2, n)
    others = np.random.default_rng(12).uniform(-1.2, 1.2, (40, n))
    prm = lb.LBFGSParam(m=m, max_iterations=MAXIT)
    V = np.random.default_rng(13).standard_normal((40, k, n))
    MEAN = np.random.default_rng(14).standard_normal((40, n))
    want = {}
    for pos in (0, 17, 39):
        X0 = others.copy()
        X0[pos] = p
        h, _, _, _ = solve_keep(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "MoreThuente")
        Vp, Mp = V.copy(), MEAN.copy()
        Vp[pos], Mp[pos] = V[0], MEAN[0]
        for op in ("LT", "LINV", "LINVT", "density"):
            full = run_density(gpu_ctx, h, 0, 40, k, Vp, Mp) if op == "density" else run_op(gpu_ctx, h, op, 0, 40, k, Vp)
            want.setdefault(op, full[pos])
            assert np.array_equal(full[pos], want[op]), (op, pos)
            for b0, count in ((pos, 1), (max(0, pos - 3), min(40, pos + 2) - max(0, pos - 3))):
                part = (run_density(gpu_ctx, h, b0, count, k, Vp[b0:b0 + count], Mp[b0:b0 + count]) if op == "density"
                        else run_op(gpu_ctx, h, op, b0, count, k, Vp[b0:b0 + count]))
                assert np.array_equal(part[pos - b0], want[op]), (op, pos, b0, count)
            one = (run_density(gpu_ctx, h, pos, 1, 2, Vp[pos, 13:15][None], Mp[pos:pos + 1]) if op == "density"
                   else run_op(gpu_ctx, h, op, pos, 1, 2, Vp[pos, 13:15][None]))
            assert np.array_equal(one[0], want[op][13:15]), (op, pos)


def test_small_batch_error_paths(gpu_ctx):
    h = lb.SmallHistory(gpu_ctx, 8, 3, 2)
    O = gpu_ctx.empty(16)
    with pytest.raises(lb.LbfgsB200Error):     # no solve has filled it
        h.factor_apply("LINV", 0, 1, 1, O, 8, 8, O, 8, 8)
    with pytest.raises(lb.LbfgsB200Error):
        h.log_density(0, 1, 1, O, 8, 8, O, 8)
    X0 = np.random.default_rng(1).uniform(-1, 1, (2, 8))
    h, _, _, _ = solve_keep(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, lb.LBFGSParam(m=3, max_iterations=20), "MoreThuente")
    V, O2 = gpu_ctx.array(np.ones(16)), gpu_ctx.empty(16)
    for args in ((4, 0, 1, 1, V, 8, 8, O2, 8, 8),          # op out of range
                 (-1, 0, 1, 1, V, 8, 8, O2, 8, 8),
                 ("LT", 0, 3, 1, V, 8, 8, O2, 8, 8),       # problems past B
                 ("LT", 0, 2, 0, V, 8, 8, O2, 8, 8),       # k = 0
                 ("LINV", 0, 1, 1, V, 7, 8, O2, 8, 8),     # ldv < n
                 ("LINVT", 0, 1, 1, V, 8, 8, O2, 7, 8)):   # ldo < n
        with pytest.raises(lb.LbfgsB200Error):
            h.factor_apply(*args)
    for args in ((0, 3, 1, V, 8, 8, V, 8),                 # problems past B
                 (0, 2, 0, V, 8, 8, V, 8),                 # k = 0
                 (0, 1, 1, V, 7, 8, V, 8),                 # ldx < n
                 (0, 2, 1, V, 8, -8, V, 8)):               # negative stride
        with pytest.raises(lb.LbfgsB200Error):
            h.log_density(*args)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_small_batch_front(dtype):
    """LBFGSSmallBatchSolver's all-problem forms through the driver, against the dense L of the factor product; a problem without pairs."""
    n, B, k = 24, 4, 3
    X0 = np.random.default_rng(9).uniform(-1.2, 1.2, (B, n)).astype(dtype)
    X0[1] = 1.0
    prm = lb.LBFGSParam(m=5, max_iterations=MAXIT)
    I = np.tile(np.eye(n, dtype=dtype), (B, 1, 1))
    _, X, LI = lb.small_batch_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, X0, I, "L", prm, dtype=dtype)
    V = np.random.default_rng(10).standard_normal((B, k, n)).astype(dtype)
    tol = 1e-12 if dtype == np.float64 else 1e-4
    res = {op: lb.small_batch_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, X0, V, op, prm, dtype=dtype)[2] for op in ("LT", "LINV", "LINVT")}
    P = (X[:, None, :] + 0.1 * V).astype(dtype)
    _, _, lp = lb.small_batch_hessian_log_density(lb.OBJ_ROSENBROCK_PAIRED, X0, P, None, prm, dtype=dtype)
    for b in range(B):
        L = LI[b].T.astype(np.float64)
        Vb = V[b].astype(np.float64)
        cap = min(max(1.0, np.linalg.cond(L) ** 2), 1e2)
        for op, want in (("LT", Vb @ L), ("LINV", np.linalg.solve(L, Vb.T).T), ("LINVT", np.linalg.solve(L.T, Vb.T).T)):
            assert rel_err(res[op][b].astype(np.float64), want) <= tol * cap, (b, op)
        Db = (P[b] - X[b]).astype(np.float64)
        H = L @ L.T
        q = np.einsum("ij,ij->i", Db, np.linalg.solve(H, Db.T).T)
        want = -0.5 * q - 0.5 * np.linalg.slogdet(H)[1] - 0.5 * n * LOG2PI
        assert np.allclose(lp[b], want, rtol=tol * cap, atol=tol * cap * n), b
    assert np.array_equal(res["LINV"][1], V[1])            # no pairs, theta = 1
    # the one-problem forms (b, ...): the same bits as that problem's rows of the all-problem forms
    for b in (0, 2):
        for op in ("LT", "LINV", "LINVT"):
            _, _, Ob = lb.small_batch_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, X0, V[b], op, prm, dtype=dtype, b=b)
            assert np.array_equal(Ob, res[op][b]), (b, op)
        _, _, lpb = lb.small_batch_hessian_log_density(lb.OBJ_ROSENBROCK_PAIRED, X0, P[b], None, prm, dtype=dtype, b=b)
        assert np.array_equal(lpb, lp[b]), b
        _, _, lpm = lb.small_batch_hessian_log_density(lb.OBJ_ROSENBROCK_PAIRED, X0, P[b], X[b], prm, dtype=dtype, b=b)
        assert np.array_equal(lpm, lp[b]), b
    with pytest.raises(ValueError, match="problem index out of range"):
        lb.small_batch_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, X0, V[0], "LT", prm, dtype=dtype, b=B)
    with pytest.raises(ValueError, match="op must be"):
        lb.small_batch_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, X0, V, 7, prm, dtype=dtype)
