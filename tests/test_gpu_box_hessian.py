"""The final approximation of a bound-constrained solve on the H100: the masked passes against their unmasked twins bit for bit, the
free-set classification kernel, LBFGSBSolver's free members after real solves against float64 dense references, and the free set at
n = 1e6."""
import numpy as np
import pytest

import lbfgspp_b200 as lb
from test_gpu_hessian_ops import padded_block, seeded_ring
from test_hessian_sample_cpu import normals

pytestmark = pytest.mark.gpu
FINAL = lb.CLS_FINAL
DT = [np.float64, np.float32]
IDS = ["f64", "f32"]


def ring_and_box(ctx, n, m, npairs, dtype, seed, cls):
    h, Y, S = seeded_ring(ctx, n, m, npairs, dtype, seed)
    box = lb.Box(h)
    box.set("cls", cls)
    return h, box, Y, S


@pytest.mark.parametrize("dtype", DT, ids=IDS)
@pytest.mark.parametrize("k", [1, 5, 16])
def test_masked_passes_with_every_row_are_their_twins(gpu_ctx, dtype, k):
    """With the mask holding every row, each masked pass is bit-identical to its unmasked twin (other class bits set at random)."""
    n, m = 50_003, 8
    rng = np.random.default_rng(k)
    h, box, Y, S = ring_and_box(gpu_ctx, n, m, 11, dtype, 5 + k, rng.integers(0, 64, n).astype(np.uint8) | FINAL)
    c = h.ncorr
    V = rng.standard_normal((k, n))
    ld = n + 3
    Vd = padded_block(gpu_ctx, V, ld, dtype)
    assert np.array_equal(h.wt_dot_multi_masked(box, FINAL, Vd, k, ld), h.wt_dot_multi(Vd, k, ld))
    mean = gpu_ctx.array(rng.standard_normal(n).astype(dtype))
    R1, n1 = h.wt_dot_diff_masked(box, FINAL, Vd, k, ld, mean)
    R0, n0 = h.wt_dot_diff(Vd, k, ld, mean)
    assert np.array_equal(R1, R0) and np.array_equal(n1, n0)
    assert np.array_equal(h.wt_dot_normal_masked(box, FINAL, 9, 2, 4, k), h.wt_dot_normal(9, 2, 4, k))
    Cc = rng.standard_normal((2 * c, k))
    O1, O0 = gpu_ctx.empty(k * n, dtype), gpu_ctx.empty(k * n, dtype)
    h.lincomb_multi_masked(box, FINAL, 0.7, Vd, k, ld, Cc, O1, n)
    h.lincomb_multi(0.7, Vd, k, ld, Cc, O0, n)
    assert np.array_equal(O1.get(), O0.get())
    Cs = Cc.copy()
    Cs[:c] = 0.0      # the unmasked sampler pass reads no y rows
    h.lincomb_normal_masked(box, FINAL, 0.7, 9, 2, 4, k, mean, Cs, O1, n)
    h.lincomb_normal(0.7, 9, 2, 4, k, mean, Cs, O0, n)
    assert np.array_equal(O1.get(), O0.get())
    K = rng.standard_normal((2 * c, 2 * c))
    K = K + K.T
    d1, d0 = gpu_ctx.empty(n, dtype), gpu_ctx.empty(n, dtype)
    h.quad_diag_masked(box, FINAL, 1.3, K, d1)
    h.quad_diag(1.3, K, d0)
    assert np.array_equal(d1.get(), d0.get())


@pytest.mark.parametrize("dtype", DT, ids=IDS)
def test_masked_passes_on_a_subset(gpu_ctx, dtype):
    """Rows outside the mask come out exactly 0 (mean_i for the draws), and the dots equal the twins on V with those rows zeroed."""
    n, m, k = 30_011, 6, 5
    rng = np.random.default_rng(1)
    cls = rng.integers(0, 64, n).astype(np.uint8)
    F = rng.random(n) < 0.4
    cls[F] |= FINAL
    h, box, Y, S = ring_and_box(gpu_ctx, n, m, 6, dtype, 3, cls)
    c = h.ncorr
    V = rng.standard_normal((k, n)).astype(dtype)
    Vd = gpu_ctx.array(V.reshape(-1))
    Vz = gpu_ctx.array(np.where(F, V, 0).astype(dtype).reshape(-1))
    assert np.array_equal(h.wt_dot_multi_masked(box, FINAL, Vd, k, n), h.wt_dot_multi(Vz, k, n))
    Cc = rng.standard_normal((2 * c, k))
    O = gpu_ctx.empty(k * n, dtype)
    h.lincomb_multi_masked(box, FINAL, 0.5, Vd, k, n, Cc, O, n)
    out = O.get().reshape(k, n)
    assert np.all(out[:, ~F] == 0.0)
    W = np.concatenate([Y, S])
    assert np.allclose(out[:, F], (0.5 * V.astype(np.float64) + Cc.T.astype(dtype).astype(np.float64) @ W)[:, F],
                       rtol=1e-5 if dtype == np.float32 else 1e-12, atol=1e-4 if dtype == np.float32 else 1e-11)
    mean = rng.standard_normal(n).astype(dtype)
    h.lincomb_normal_masked(box, FINAL, 0.5, 4, 0, 0, k, gpu_ctx.array(mean), Cc, O, n)
    assert np.all(O.get().reshape(k, n)[:, ~F] == mean[~F])
    d = gpu_ctx.empty(n, dtype)
    h.quad_diag_masked(box, FINAL, 2.0, np.eye(2 * c), d)
    assert np.all(d.get()[~F] == 0.0)


@pytest.mark.parametrize("dtype", DT, ids=IDS)
def test_final_classes_kernel(gpu_ctx, dtype):
    """The classification rule: exact bounds, one ulp inside, 16 eps inside, lb == ub and infinite bounds; other bits kept."""
    e = np.finfo(dtype).eps
    x = np.array([2, np.nextafter(dtype(2), dtype(3)), 2 + 32 * e, 4, np.nextafter(dtype(4), dtype(3)), 1, 1, -5, 0.5], dtype=dtype)
    lo = np.array([2, 2, 2, 2, 2, 1, -np.inf, -np.inf, 0], dtype=dtype)
    hi = np.array([4, 4, 4, 4, 4, 1, np.inf, np.inf, 1], dtype=dtype)
    h = lb.History(gpu_ctx, x.size, 2, dtype)
    box = lb.Box(h)
    box.set("cls", np.full(x.size, 5 | FINAL, dtype=np.uint8))
    nf = box.final_classes(gpu_ctx.array(x), gpu_ctx.array(lo), gpu_ctx.array(hi))
    cls = box.get("cls")
    assert nf == 4
    assert list((cls & FINAL) != 0) == [False, False, True, False, False, False, True, True, True]
    assert np.all(cls & 5 == 5)


def dense_free(Bd, F):
    return np.linalg.inv(Bd[np.ix_(F, F)])


BOUNDED = [("chained Rosenbrock in [2, 4]", lb.OBJ_ROSENBROCK_CHAINED, 200, 2.0, 4.0),
           ("paired Rosenbrock in [2, 4]", lb.OBJ_ROSENBROCK_PAIRED, 300, 2.0, 4.0),
           ("quadratic in [-0.5, 20.5]", lb.OBJ_QUAD_SHIFT, 256, -0.5, 20.5)]


@pytest.mark.parametrize("dtype", DT, ids=IDS)
@pytest.mark.parametrize("m", [5, 20])
@pytest.mark.parametrize("case", BOUNDED, ids=lambda c: c[0])
def test_free_members_after_real_solves(case, m, dtype):
    """LBFGSBSolver on the GPU: products, diagonals, log det, draws and log densities on the free set against B[F, F] of the dense B of
    the same solve, and H_F against the conditioning identity of the dense H."""
    stats = pytest.importorskip("scipy.stats")
    name, obj, n, lo, hi = case
    prm = lb.LBFGSBParam(m=m, max_iterations=200)
    x0 = np.full(n, 0.5 * (lo + hi)) + np.linspace(-0.2, 0.2, n)
    call = lambda op, **kw: lb.box_solve_hessian(obj, x0, lo, hi, op, param=prm, dtype=dtype, **kw)
    r = call("denseB", free=False)
    Bd, x = r["out"].astype(np.float64), r["x"]
    Hd = call("denseH", free=False)["out"].astype(np.float64)
    eps = 4 * np.finfo(dtype).eps
    fixed = (x <= lo + eps * max(1, abs(lo))) | (x >= hi - eps * max(1, abs(hi)))
    F, A = np.flatnonzero(~fixed), np.flatnonzero(fixed)
    assert 0 < F.size < n, (name, F.size)
    HF = dense_free(Bd, F)
    cond = np.linalg.cond(Bd[np.ix_(F, F)])
    tol = (1e-10 if dtype == np.float64 else 2e-3) * max(1.0, cond)
    assert np.linalg.norm(Hd[np.ix_(F, F)] - Hd[np.ix_(F, A)] @ np.linalg.solve(Hd[np.ix_(A, A)], Hd[np.ix_(A, F)]) - HF) <= \
        (1e-8 if dtype == np.float64 else 1e-2) * np.linalg.cond(Hd) * np.linalg.norm(HF)
    V = np.random.default_rng(n + m).standard_normal((6, n))
    for op, M in (("B", Bd[np.ix_(F, F)]), ("H", HF)):
        r = call(op, V=V)
        assert r["nfree"] == F.size and np.array_equal(r["x"], x)
        assert np.all(r["out"][:, A] == 0)
        got, want = r["out"][:, F].astype(np.float64), V[:, F] @ M.T
        assert np.linalg.norm(got - want) <= tol * np.linalg.norm(want), (name, op)
    d = call("diagH")["out"].astype(np.float64)
    assert np.all(d[A] == 0) and np.allclose(d[F], np.diag(HF), rtol=tol, atol=0)
    logdet = call("logdet")["logdet"]
    assert abs(logdet - np.linalg.slogdet(HF)[1]) <= tol * F.size
    mean = x.astype(np.float64)
    P = mean + 0.05 * V
    lp = call("log_density", V=P)["out"]
    want = stats.multivariate_normal(mean=mean[F], cov=HF).logpdf(P[:, F])
    assert np.allclose(lp, want, rtol=tol, atol=tol * F.size)
    k = 16
    draws = call("sample", k=k, seed=7, first=2)["out"].astype(np.float64)
    assert np.all(draws[:, A] == x[A])
    Z = np.stack([normals(7, 0, 2 + j, n) for j in range(k)]).astype(dtype).astype(np.float64)
    # L_F is the symmetric square root of H_F
    w, U = np.linalg.eigh(HF)
    LF = (U * np.sqrt(w)) @ U.T
    want = mean[F] + Z[:, F] @ LF
    assert np.linalg.norm(draws[:, F] - want) <= 10 * tol * np.linalg.norm(want - mean[F]), name


def numpy_free(S, Y, F):
    """float64 recomputation of theta, K_HF (raw [Y S] convention), log det H_F and the log-density quadratic form's M."""
    c = S.shape[0]
    theta = Y[0] @ Y[0] / (S[0] @ Y[0])
    SY, SS = S @ Y.T, S @ S.T
    Minv = np.zeros((2 * c, 2 * c))
    Minv[:c, :c] = -np.diag(np.diag(SY))
    L = np.triu(SY, 1)                  # L(a, b) = s_a'y_b for a newer than b (a < b by age)
    Minv[c:, :c] = L
    Minv[:c, c:] = L.T
    Minv[c:, c:] = theta * SS
    W = np.concatenate([Y, theta * S])[:, F]
    mid = Minv - (W @ W.T) / theta
    Dg = np.concatenate([np.ones(c), theta * np.ones(c)])
    KH = Dg[:, None] * np.linalg.inv(mid) * Dg[None, :] / theta ** 2
    nF = int(F.sum())
    logdet = -nF * np.log(theta) - np.linalg.slogdet(mid)[1] + np.linalg.slogdet(Minv)[1]
    return theta, KH, logdet, np.linalg.inv(Minv)


def test_free_set_at_n_1e6_explicit_history():
    """m = 20 random pairs at n = 1e6 and random class bytes: diag H_F, log det H_F and log densities against a float64 recomputation."""
    n, m = 1_000_000, 20
    rng = np.random.default_rng(2024)
    S = rng.standard_normal((m, n))
    Y = S * (1.0 + rng.random(n)) + 0.05 * rng.standard_normal((m, n))
    cls = rng.integers(0, 64, n).astype(np.uint8)
    F = rng.random(n) < 0.7
    cls[F] |= FINAL
    Sa, Ya = S[::-1], Y[::-1]          # by age
    theta, KH, logdet, M = numpy_free(Sa, Ya, F)
    r = lb.box_hist_hessian(S, Y, "diagH", cls=cls, m=m)
    assert r["nfree"] == F.sum()
    Wr = np.concatenate([Ya, Sa])
    want = np.zeros(n)
    Wf = Wr[:, F]
    want[F] = 1 / theta + np.sum(Wf * (KH @ Wf), axis=0)
    assert np.all(r["out"][~F] == 0) and np.allclose(r["out"], want, rtol=1e-9, atol=0)
    assert abs(r["logdet"] - logdet) <= 1e-9 * abs(logdet)
    mean = rng.standard_normal(n)
    X = mean + 0.01 * rng.standard_normal((3, n))
    lp = lb.box_hist_hessian(S, Y, "log_density", cls=cls, m=m, V=X, mean=mean)["out"]
    Wt = np.concatenate([Ya, theta * Sa])
    for j in range(3):
        v = np.where(F, X[j] - mean, 0.0)
        u = Wt @ v
        q = theta * v @ v - u @ M @ u
        want = -0.5 * q - 0.5 * logdet - 0.5 * F.sum() * np.log(2 * np.pi)
        assert abs(lp[j] - want) <= 1e-9 * abs(want), (j, lp[j], want)


def test_c4_shape_free_set():
    """Chained Rosenbrock in [2, 4] at n = 1e6: n_F equals the count of the rule on the returned x, diag H_F is finite and positive on F."""
    n = 1_000_000
    prm = lb.LBFGSBParam(m=10, max_iterations=60)
    r = lb.box_solve_hessian(lb.OBJ_ROSENBROCK_CHAINED, np.full(n, 3.0), 2.0, 4.0, "diagH", param=prm)
    x, d = r["x"], r["out"]
    eps = 4 * np.finfo(np.float64).eps
    F = ~((x <= 2.0 + eps * 2.0) | (x >= 4.0 - eps * 4.0))
    assert r["nfree"] == F.sum() and 0 < r["nfree"] < n
    assert np.all(np.isfinite(d[F])) and np.all(d[F] > 0) and np.all(d[~F] == 0)
