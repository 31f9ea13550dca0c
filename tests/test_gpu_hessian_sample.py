"""Draws from N(x*, H) and log det H of the final L-BFGS approximation on the GPU: the sampler's large-n passes
(lbfgs_b200_hist_wt_dot_normal / lincomb_normal) against float64 numpy over the numpy restatement of the generator, and the small-batch
factor, sampler and log-determinant (lbfgs_b200_small_hist_factor_times / _sample / _logdet) against the dense H, slogdet, the
generator restatement and the sample covariance, with bit identity across draw groups, positions and ranges."""
import numpy as np
import pytest

import lbfgspp_b200 as lb
from test_gpu_hessian_ops import seeded_ring
from test_gpu_small_batch_hessian import MAXIT, OBJECTIVES, dense_ref, kept, problem, solve_keep
from test_hessian_sample_cpu import M0, M1, W0, W1, bfgs_dense_inverse

pytestmark = pytest.mark.gpu
MASK = np.uint64(0xFFFFFFFF)


def rel_err(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


def normals(seed, stream, j, n):
    """Vectorised restatement of csrc/philox.cuh: draw j of stream `stream`, coordinates 0..n-1, float64."""
    q = np.arange((n + 1) // 2, dtype=np.uint64)
    c0, c1 = q & MASK, q >> np.uint64(32)
    c2 = np.full_like(q, np.uint64(j))
    c3 = np.full_like(q, np.uint64(stream))
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    for _ in range(10):
        p0, p1 = np.uint64(M0) * c0, np.uint64(M1) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & MASK
        k0, k1 = (k0 + np.uint64(W0)) & MASK, (k1 + np.uint64(W1)) & MASK
    x0 = ((c1 << np.uint64(32)) | c0) >> np.uint64(11)
    x1 = ((c3 << np.uint64(32)) | c2) >> np.uint64(11)
    u0 = (x0 + np.uint64(1)).astype(np.float64) * 2.0 ** -53
    u1 = x1.astype(np.float64) * 2.0 ** -53
    r = np.sqrt(-2.0 * np.log(u0))
    z = np.empty(2 * q.size)
    z[0::2], z[1::2] = r * np.cos(2 * np.pi * u1), r * np.sin(2 * np.pi * u1)
    return z[:n]


# ---- the large-n passes ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("m,npairs", [(3, 0), (3, 3), (10, 13), (64, 64)])
def test_large_n_passes_against_float64(gpu_ctx, dtype, m, npairs):
    n, seed, stream, first, k = 20_001, 0x9E3779B97F4A7C15, 5, 11, 16
    h, Y, S = seeded_ring(gpu_ctx, n, m, npairs, dtype, seed=m + npairs)
    c = h.ncorr
    Z = np.stack([normals(seed, stream, first + j, n) for j in range(k)])
    Zt = Z.astype(dtype).astype(np.float64)
    W = np.concatenate([Y, S])
    tol = 1e-12 if dtype == np.float64 else 1e-5
    R = h.wt_dot_normal(seed, stream, first, k)
    if c:
        ref = W @ Zt.T
        assert np.all(np.abs(R - ref) <= tol * (np.abs(W) @ np.abs(Zt.T)) + 1e-300)
        # column j of a k = 16 call is bit-identical to the k = 1 call with first + j
        for j in (0, 7, 15):
            assert np.array_equal(h.wt_dot_normal(seed, stream, first + j, 1)[:, 0], R[:, j])
    coef = np.random.default_rng(3).standard_normal((2 * c, k)).astype(dtype)
    coef[:c] = np.nan                       # the y rows are not read
    mean = np.random.default_rng(4).standard_normal(n).astype(dtype)
    a0 = dtype(0.625)
    for mu in (mean, None):
        OUT = gpu_ctx.array(np.full(k * n, np.nan, dtype=dtype))
        h.lincomb_normal(a0, seed, stream, first, k, gpu_ctx.array(mu) if mu is not None else None, coef, OUT, n)
        got = OUT.get().reshape(k, n).astype(np.float64)
        ref = float(a0) * Zt + (coef[c:].astype(np.float64).T @ S if c else 0.0) + (mu.astype(np.float64) if mu is not None else 0.0)
        assert rel_err(got, ref) <= 10 * tol, rel_err(got, ref)
    # draws of a one-vector call with first + j are the same bits as column j of the 16-vector call
    one = gpu_ctx.array(np.zeros(n, dtype=dtype))
    h.lincomb_normal(a0, seed, stream, first + 9, 1, None, coef[:, 9:10].copy(), one, n)
    OUT = gpu_ctx.array(np.zeros(k * n, dtype=dtype))
    h.lincomb_normal(a0, seed, stream, first, k, None, coef, OUT, n)
    assert np.array_equal(one.get(), OUT.get().reshape(k, n)[9])


# ---- the small batch -------------------------------------------------------------------------------------------------------------------
def run_factor(ctx, h, b0, count, k, V):
    n = h.n
    Vd = ctx.array(V.reshape(-1))
    O = ctx.array(np.full(count * k * n, np.nan, dtype=h.dtype))
    h.factor_times(b0, count, k, Vd, n, k * n, O, n, k * n)
    return O.get().reshape(count, k, n)


def run_sample(ctx, h, seed, first, b0, count, k, MEAN=None):
    n = h.n
    O = ctx.array(np.full(count * k * n, np.nan, dtype=h.dtype))
    h.sample(seed, first, b0, count, k, ctx.array(MEAN.reshape(-1)) if MEAN is not None else None, n, O, n, k * n)
    return O.get().reshape(count, k, n)


def check_small(gpu_ctx, objective, n, m, dtype, B=3, its=MAXIT):
    X0, d0, d1, ldd = problem(objective, B, n, 500 + n + m, dtype)
    h, _, _, _ = solve_keep(gpu_ctx, objective, X0, lb.LBFGSParam(m=m, max_iterations=its), "MoreThuente", d0, d1, ldd)
    c_all, th = h.info()
    I = np.tile(np.eye(n, dtype=dtype), (B, 1, 1))
    L_all = run_factor(gpu_ctx, h, 0, B, n, I)          # row j: L e_j, i.e. column j of L
    ld = h.logdet()
    seed, first, k = 77, 3, 5
    MEAN = np.random.default_rng(n).standard_normal((B, n)).astype(dtype)
    D = run_sample(gpu_ctx, h, seed, first, 0, B, k, MEAN)
    for b in range(B):
        S, Y, _, _, _, _, theta = kept(h, b)
        _, Hm = dense_ref(S, Y, theta)
        L = L_all[b].T.astype(np.float64)
        # against the float64 BFGS recursion of the kept pairs; the scaling by cond(H) is capped (fp64 at 1e3, fp32 at 1e2) and the cond
        # seen is in the message
        Hm = bfgs_dense_inverse(S, Y, theta)
        cond = np.linalg.cond(Hm)
        tol = 1e-12 * min(max(1.0, cond), 1e3) if dtype == np.float64 else 1e-4 * min(max(1.0, cond), 1e2)
        assert rel_err(L @ L.T, Hm) <= tol, (objective, n, m, b, int(c_all[b]), cond, rel_err(L @ L.T, Hm))
        sign, want = np.linalg.slogdet(Hm)
        assert sign > 0 and abs(ld[b] - want) <= (1e-9 if dtype == np.float64 else 1e-3) * max(1.0, abs(want)), (b, ld[b], want)
        Z = np.stack([normals(seed, b, first + j, n) for j in range(k)]).astype(dtype).astype(np.float64)
        ref = MEAN[b].astype(np.float64) + Z @ L.T
        assert rel_err(D[b].astype(np.float64) - MEAN[b], ref - MEAN[b]) <= (1e-12 if dtype == np.float64 else 1e-4), b
        if c_all[b] == 0:
            assert np.allclose(L, np.eye(n) / np.sqrt(float(th[b])), rtol=4 * np.finfo(dtype).eps, atol=0)
        # one problem, one draw at a time: the same bits
        assert np.array_equal(run_sample(gpu_ctx, h, seed, first + 2, b, 1, 1, MEAN[b])[0, 0], D[b, 2])
        assert np.array_equal(h.logdet(b, 1), ld[b:b + 1])
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


def test_small_batch_positions_and_ranges(gpu_ctx):
    """A problem's draws and log det do not depend on its position, b0 or count, only on its stream b."""
    n, m, seed = 40, 6, 5
    p = np.random.default_rng(11).uniform(-1.2, 1.2, n)
    others = np.random.default_rng(12).uniform(-1.2, 1.2, (40, n))
    prm = lb.LBFGSParam(m=m, max_iterations=MAXIT)
    for pos in (0, 17, 39):
        X0 = others.copy()
        X0[pos] = p
        h, _, _, _ = solve_keep(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "MoreThuente")
        D = run_sample(gpu_ctx, h, seed, 0, 0, 40, 20)
        ld = h.logdet()
        if pos == 0:
            want_ld = ld[0]
        assert ld[pos] == want_ld
        for b0, count in ((pos, 1), (max(0, pos - 3), min(40, pos + 2) - max(0, pos - 3))):
            assert np.array_equal(run_sample(gpu_ctx, h, seed, 0, b0, count, 20)[pos - b0], D[pos])
            assert np.array_equal(h.logdet(b0, count)[pos - b0], ld[pos])
        # draw j does not depend on k or first
        assert np.array_equal(run_sample(gpu_ctx, h, seed, 13, pos, 1, 2)[0], D[pos, 13:15])
        # same history, stream pos: the draws are L (z of stream pos)
        L = run_factor(gpu_ctx, h, pos, 1, n, np.eye(n)[None])[0].T
        Z = np.stack([normals(seed, pos, j, n) for j in range(20)])
        assert rel_err(D[pos], Z @ L.T) <= 1e-12


def test_sample_covariance_matches_h(gpu_ctx):
    """At a fixed seed (deterministic): the covariance of 40 000 draws is H within 5 standard errors per entry."""
    n, k = 8, 40_000
    X0 = np.random.default_rng(21).uniform(-1.2, 1.2, (1, n))
    h, _, _, _ = solve_keep(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, lb.LBFGSParam(m=5, max_iterations=6), "MoreThuente")
    S, Y, _, _, _, _, theta = kept(h, 0)
    assert S.shape[0] > 0
    _, Hm = dense_ref(S, Y, theta)
    D = run_sample(gpu_ctx, h, 2024, 0, 0, 1, k)[0]
    cov = D.T @ D / k
    se = np.sqrt((Hm ** 2 + np.outer(np.diag(Hm), np.diag(Hm))) / k)
    assert np.all(np.abs(cov - Hm) <= 5 * se), np.max(np.abs(cov - Hm) / se)


def test_error_paths(gpu_ctx):
    h = lb.SmallHistory(gpu_ctx, 8, 3, 2)
    O = gpu_ctx.empty(16)
    with pytest.raises(lb.LbfgsB200Error):     # no solve has filled it
        h.sample(1, 0, 0, 1, 1, None, 8, O, 8, 8)
    with pytest.raises(lb.LbfgsB200Error):
        h.logdet()
    X0 = np.random.default_rng(1).uniform(-1, 1, (2, 8))
    h, _, _, _ = solve_keep(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, lb.LBFGSParam(m=3, max_iterations=20), "MoreThuente")
    for args in ((1, 0, 0, 3, 1, None, 8, O, 8, 8),       # problems past B
                 (1, 0, 0, 2, 0, None, 8, O, 8, 8),       # k = 0
                 (1, 0xFFFFFFFF, 0, 1, 2, None, 8, O, 8, 8),   # draws past 2^32
                 (1, 0, 0, 1, 1, None, 8, O, 7, 8),       # ldo < n
                 (1, 0, 0, 2, 1, None, 8, O, 8, 0),       # two problems on the same draws
                 (1, 0, 0, 2, 1, None, 8, O, 8, 4),       # problems' draws overlap (ldop < k * ldo)
                 (1, 0, 0, 1, 1, O, 8, O, 8, 8)):         # MEAN overlaps OUT
        with pytest.raises(lb.LbfgsB200Error):
            h.sample(*args)
    with pytest.raises(lb.LbfgsB200Error):
        h.logdet(1, 2)
    hist = lb.History(gpu_ctx, 100, 3)
    with pytest.raises(lb.LbfgsB200Error):
        hist.wt_dot_normal(1, 0, 0, 17)
    with pytest.raises(lb.LbfgsB200Error):
        hist.lincomb_normal(1.0, 1, 0, 0xFFFFFFF1, 16, None, np.zeros((0, 16)), O, 100)


def test_small_batch_without_pairs(gpu_ctx):
    """A problem started at the minimiser keeps no pair: L = I/sqrt(theta) = I (theta = 1), log det H = 0, draws = x + z."""
    n = 8
    X0 = np.random.default_rng(3).uniform(-1.2, 1.2, (3, n))
    X0[1] = 1.0
    h, _, _, _ = solve_keep(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, lb.LBFGSParam(m=4, max_iterations=MAXIT), "MoreThuente")
    c_all, th = h.info()
    assert c_all[1] == 0 and th[1] == 1.0 and c_all[0] > 0
    L = run_factor(gpu_ctx, h, 1, 1, n, np.eye(n)[None])[0]
    assert np.array_equal(L, np.eye(n))
    assert h.logdet(1, 1)[0] == 0.0
    MEAN = np.full((1, n), 0.5)
    D = run_sample(gpu_ctx, h, 8, 0, 1, 1, 3, MEAN)[0]
    Z = np.stack([normals(8, 1, j, n) for j in range(3)])
    assert rel_err(D - 0.5, Z) <= 1e-14


# ---- the front, through the driver ---------------------------------------------------------------------------------------------------
LINE_SEARCHES = ["Backtracking", "Bracketing", "NocedalWright", "MoreThuente"]


@pytest.mark.parametrize("resident", [False, True], ids=["host_loop", "resident"])
@pytest.mark.parametrize("ls", LINE_SEARCHES)
def test_front_factor_against_dense_h(resident, ls):
    for n, m in ((2, 3), (18, 10), (300, 10), (300, 64)):
        prm = lb.LBFGSParam(m=m)
        x0 = np.linspace(-1, 1, n)
        niter, x, Bd, Hd = lb.solve_dense(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, ls, resident=resident)
        seed, first, k = 31, 2, 18                     # two groups of draws
        niter2, x2, L, D, ld = lb.solve_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, x0, np.eye(n), seed, first, k, prm, ls, resident=resident)
        assert niter2 == niter and np.array_equal(x2, x)
        L = L.T
        cond = np.linalg.cond(Hd)
        err = rel_err(L @ L.T, Hd)
        assert err <= 1e-12 * min(max(1.0, cond), 1e3), (n, m, cond, err)
        # log det H = -log det B, B formed directly (not inverted); the scaling by cond(B) is capped at 1e3
        sign, logdet_b = np.linalg.slogdet(Bd)
        want, cb = -logdet_b, np.linalg.cond(Bd)
        assert sign > 0 and abs(ld - want) <= 1e-12 * min(max(1.0, cb), 1e3) * max(1.0, abs(want)), (n, m, ld, want, cb)
        Z = np.stack([normals(seed, 0, first + j, n) for j in range(k)])
        assert rel_err(D - x, Z @ L.T) <= 1e-12, (n, m)


def test_front_batch_member_streams():
    """Batch member 0 (stream 0) gives its lone solve's bits; member b's draws come from stream b."""
    n, B = 1000, 4
    X0 = np.stack([np.random.default_rng(2000 + p).uniform(-1, 1, n) for p in range(B)])
    prm = lb.LBFGSParam(m=10)
    V = np.random.default_rng(5).standard_normal((3, n))
    _, LV0, D0, ld0 = lb.batch_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, X0, 0, V, 9, 0, 17, prm, "MoreThuente")
    _, x, LV1, D1, ld1 = lb.solve_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, X0[0], V, 9, 0, 17, prm, "MoreThuente", resident=True)
    assert np.array_equal(LV0, LV1) and np.array_equal(D0, D1) and ld0 == ld1
    b = 2
    E = np.eye(n)[:64]
    X, LE, Db, _ = lb.batch_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, X0, b, E, 9, 0, 4, prm, "MoreThuente")
    # the first 64 columns of L_b against the draws' first 64 coordinates is not a full check: use L_b z through the factor product
    _, LZ, _, _ = lb.batch_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, X0, b, np.stack([normals(9, b, j, n) for j in range(4)]), 9, 0, 0, prm,
                                          "MoreThuente")
    assert rel_err(Db - X[b], LZ) <= 1e-12
    assert np.array_equal(LE, lb.batch_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, X0, b, E, 9, 0, 0, prm, "MoreThuente")[1])
    with pytest.raises(RuntimeError, match="problem index out of range"):
        lb.batch_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, X0, B, None, 9, 0, 1, prm, "MoreThuente")


def test_logdet_at_n_1e6_against_a_float64_recomputation():
    """BFGSMat::inverse_hessian_logdet at n = 1e6 against float64: the pairs projected on an orthonormal basis Q of span [S Y], the BFGS
    recursion run there, log det H = -((n - 2c) log theta + log det(Q'BQ))."""
    n, npairs, m = 1_000_000, 13, 10
    rng = np.random.default_rng(77)
    d = 1.0 + rng.random(n)
    S = rng.standard_normal((npairs, n))
    Y = S * d + 0.01 * rng.standard_normal((npairs, n))
    _, D, ld = lb.hist_sample(S, Y, m=m, seed=3, k=2)
    kS, kY = S[::-1][:m], Y[::-1][:m]
    c = kS.shape[0]
    theta = kY[0] @ kY[0] / (kS[0] @ kY[0])
    Q, _ = np.linalg.qr(np.concatenate([kS, kY]).T)
    s_, y_ = kS @ Q, kY @ Q
    Bt = theta * np.eye(2 * c)
    for s, y in zip(s_[::-1], y_[::-1]):
        Bs = Bt @ s
        Bt = Bt - np.outer(Bs, Bs) / (s @ Bs) + np.outer(y, y) / (y @ s)
    want = -((n - 2 * c) * np.log(theta) + np.linalg.slogdet(Bt)[1])
    assert abs(ld - want) <= 1e-9 * abs(want), (ld, want)
    assert np.all(np.isfinite(D))


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_small_batch_front(dtype):
    """LBFGSSmallBatchSolver's all-problem forms through the driver: L_b against H_b of the products with I, log det, draws around X_b."""
    n, B = 24, 4
    X0 = np.random.default_rng(9).uniform(-1.2, 1.2, (B, n)).astype(dtype)
    X0[1] = 1.0
    prm = lb.LBFGSParam(m=5, max_iterations=MAXIT)
    I = np.tile(np.eye(n, dtype=dtype), (B, 1, 1))
    _, X, LV, D, ld = lb.small_batch_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, X0, I, 4, 1, 3, prm, dtype=dtype)
    _, _, _, HV, _ = lb.small_batch_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, X0, I, prm, dtype=dtype)
    tol = 1e-12 if dtype == np.float64 else 1e-4
    for b in range(B):
        L = LV[b].T.astype(np.float64)
        H = HV[b].astype(np.float64)
        assert rel_err(L @ L.T, H) <= tol * min(max(1.0, np.linalg.cond(H)), 1e2), b
        assert abs(ld[b] - np.linalg.slogdet(H)[1]) <= (1e-9 if dtype == np.float64 else 1e-3) * max(1.0, abs(ld[b])), b
        Z = np.stack([normals(4, b, 1 + j, n) for j in range(3)]).astype(dtype).astype(np.float64)
        assert rel_err(D[b].astype(np.float64) - X[b], Z @ L.T) <= tol, b
    assert ld[1] == 0.0 and np.array_equal(LV[1], np.eye(n, dtype=dtype))
