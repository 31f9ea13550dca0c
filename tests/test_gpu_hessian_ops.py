"""The operator form of the final L-BFGS approximation on the GPU: the two k-vector passes over the S/Y history
(lbfgs_b200_hist_wt_dot_multi / lbfgs_b200_hist_lincomb_multi) against float64 numpy, the front's B V / H V
(LBFGSSolver / LBFGSBatchSolver::final_approx_*_times) against the dense matrices and apply_Hv, at C2 / C5 scale, and the error paths."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- kernels ------------------------------------------------------------------------------------------------------------------
def seeded_ring(ctx, n, m, npairs, dtype, seed):
    """A History with npairs seeded pairs (wrapped when npairs > m) and its columns by age as float64 (c, n) arrays."""
    rng = np.random.default_rng(seed)
    h = lb.History(ctx, n, m, dtype)
    for _ in range(npairs):
        s = rng.standard_normal(n).astype(dtype)
        y = (s + 0.3 * rng.standard_normal(n)).astype(dtype)
        h.add(ctx.array(s), ctx.array(y))
    c = h.ncorr
    Y = np.array([h.column("y", a) for a in range(c)], dtype=np.float64).reshape(c, n)
    S = np.array([h.column("s", a) for a in range(c)], dtype=np.float64).reshape(c, n)
    return h, Y, S


def padded_block(ctx, A, ld, dtype):
    """The rows of A (k, n) as k device columns with leading dimension ld (padding filled with NaN: it must never be read)."""
    k, n = A.shape
    host = np.full((k, ld), np.nan)
    host[:, :n] = A
    return ctx.array(host.reshape(-1).astype(dtype))


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("m", [6, 10, 20, 64])
@pytest.mark.parametrize("cwant", ["0", "1", "5", "m"])
def test_kernels_against_float64(gpu_ctx, dtype, m, cwant):
    n = 100_003                      # ragged: the ring's ld is padded, and so are V's and OUT's
    npairs = {"0": 0, "1": 1, "5": 5, "m": m + 3}[cwant]   # c = m: a wrapped ring
    h, Y, S = seeded_ring(gpu_ctx, n, m, npairs, dtype, seed=m * 10 + npairs)
    c = h.ncorr
    assert c == min(npairs, m)
    W = np.concatenate([Y, S])       # rows y by age, then s by age
    tol = 1e-12 if dtype == np.float64 else 1e-5
    rng = np.random.default_rng(7 + m + npairs)
    for k in (1, 3, 16):
        V = rng.standard_normal((k, n)).astype(dtype).astype(np.float64)
        ldv, ldo = n + 5, n + 3
        Vd = padded_block(gpu_ctx, V, ldv, dtype)
        R = h.wt_dot_multi(Vd, k, ldv)
        assert R.shape == (2 * c, k)
        ref = W @ V.T
        assert np.all(np.abs(R - ref) <= tol * (np.abs(W) @ np.abs(V).T) + 1e-300), (k, np.max(np.abs(R - ref)))
        Cc = rng.standard_normal((2 * c, k))
        a0 = 0.75
        OUTd = padded_block(gpu_ctx, np.zeros((k, n)), ldo, dtype)
        h.lincomb_multi(a0, Vd, k, ldv, Cc, OUTd, ldo)
        out = OUTd.get().reshape(k, ldo)
        Cq = Cc.astype(dtype).astype(np.float64)
        ref = a0 * V + Cq.T @ W
        bound = abs(a0) * np.abs(V) + np.abs(Cq).T @ np.abs(W)
        assert np.all(np.abs(out[:, :n] - ref) <= tol * bound + 1e-300), k
        assert np.all(np.isnan(out[:, n:])), "the padding of OUT was written"
        if k == 16:   # column j of a k = 16 call is bit-identical to the k = 1 call on that column alone
            for j in (0, 5, 15):
                Vj = padded_block(gpu_ctx, V[j:j + 1], n, dtype)
                assert np.array_equal(h.wt_dot_multi(Vj, 1, n)[:, 0], R[:, j]), j
                Oj = gpu_ctx.empty(n, dtype)
                h.lincomb_multi(a0, Vj, 1, n, Cc[:, j:j + 1], Oj, n)
                assert np.array_equal(Oj.get(), out[j, :n]), j


def test_abi_rejects_bad_arguments(gpu_ctx):
    h, _, _ = seeded_ring(gpu_ctx, 64, 4, 2, np.float64, seed=1)
    V = gpu_ctx.empty(64 * 17)
    for k in (0, 17):
        with pytest.raises(lb.LbfgsB200Error, match="k must be in 1..16"):
            h.wt_dot_multi(V, k, 64)
        with pytest.raises(lb.LbfgsB200Error, match="k must be in 1..16"):
            h.lincomb_multi(1.0, V, k, 64, np.zeros((4, max(k, 1))), V, 64)
    with pytest.raises(lb.LbfgsB200Error, match="leading dimension 63 is smaller than n = 64"):
        h.wt_dot_multi(V, 1, 63)


# ---- the front: B V and H V against the dense matrices and apply_Hv ---------------------------------------------------------------
def rel_err(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


@pytest.mark.parametrize("resident", [False, True], ids=["host_loop", "resident"])
@pytest.mark.parametrize("n", [10, 1000])
def test_identity_blocks_reproduce_the_dense_matrices(resident, n):
    prm = lb.LBFGSParam(m=8)
    x0 = np.linspace(-1, 1, n)
    niter, x, Bd, Hd = lb.solve_dense(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "MoreThuente", resident=resident)
    niter2, x2, BV, HV, HBV = lb.solve_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, x0, np.eye(n), prm, "MoreThuente", resident=resident)
    assert niter2 == niter and np.array_equal(x2, x)
    assert rel_err(BV, Bd) <= 1e-12, rel_err(BV, Bd)          # row j = B e_j = column j of the symmetric B
    # the dense H inverts a B that is exact only to rounding: the comparison with it is good to cond(B) times that
    tol_h = 1e-12 * max(1.0, np.linalg.cond(Bd))
    assert rel_err(HV, Hd) <= tol_h, (rel_err(HV, Hd), tol_h)
    assert rel_err(HBV, np.eye(n)) <= tol_h, rel_err(HBV, np.eye(n))


@pytest.mark.parametrize("m,npairs", [(6, 3), (6, 9), (20, 20)])
@pytest.mark.parametrize("n", [10, 1000])
def test_inverse_equals_apply_Hv(gpu_ctx, n, m, npairs):
    """H v of the operator form against lbfgs_b200_hist_apply_Hv(v, a = 1) with both algorithms on the same ring: 1e-11 relative,
    the bar between the Gram form and the literal recursion."""
    rng = np.random.default_rng(n + m + npairs)
    A = np.linspace(1.0, 50.0, n)      # pairs of a diagonal quadratic: y = A s
    S = rng.standard_normal((npairs, n))
    Y = S * A
    V = rng.standard_normal((5, n))
    drv = lb.driver()
    dp = C.POINTER(C.c_double)
    BV, HV = np.zeros((5, n)), np.zeros((5, n))
    lb._checked("hist_times", lambda *err: drv.lbfgsb200_drv_hist_times_f64(0, n, m, npairs, S.ctypes.data_as(dp), Y.ctypes.data_as(dp),
                                                                           V.ctypes.data_as(dp), V.size, BV.ctypes.data_as(dp),
                                                                           HV.ctypes.data_as(dp), *err))
    h = lb.History(gpu_ctx, n, m)
    for k in range(npairs):
        h.add(gpu_ctx.array(S[k]), gpu_ctx.array(Y[k]))
    res = gpu_ctx.empty(n)
    for algo in (lb.HV_GRAM, lb.HV_TWO_LOOP):
        for j in range(5):
            h.apply_Hv(gpu_ctx.array(V[j]), 1.0, res, algo)
            assert rel_err(HV[j], res.get()) <= 1e-11, (algo, j, rel_err(HV[j], res.get()))
    for j in range(5):   # B is positive definite on these vectors
        assert np.dot(V[j], BV[j]) > 0


# ---- at scale ---------------------------------------------------------------------------------------------------------------------
def check_products(V, BV, HV, HBV):
    assert np.max(np.abs(HBV - V)) <= 1e-8 * np.max(np.abs(V)), np.max(np.abs(HBV - V))
    for j in range(V.shape[0]):
        assert np.dot(V[j], BV[j]) > 0 and np.dot(V[j], HV[j]) > 0, j


def test_c2_shaped_solve():
    n, k = 10_000_000, 8
    V = np.random.default_rng(2).standard_normal((k, n))
    _, _, BV, HV, HBV = lb.solve_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n), V, lb.LBFGSParam(m=10), "MoreThuente", resident=True)
    check_products(V, BV, HV, HBV)


def test_c5_batch_member_equals_its_lone_solve():
    n, B, b, k = 1_000_000, 4, 2, 8
    X0 = np.stack([np.random.default_rng(1000 + p).uniform(-1, 1, n) for p in range(B)])
    V = np.random.default_rng(3).standard_normal((k, n))
    prm = lb.LBFGSParam(m=10)
    BV, HV, HBV = lb.batch_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, X0, b, V, prm, "MoreThuente")
    check_products(V, BV, HV, HBV)
    _, _, BV1, HV1, HBV1 = lb.solve_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, X0[b], V, prm, "MoreThuente", resident=True)
    assert np.array_equal(BV, BV1) and np.array_equal(HV, HV1) and np.array_equal(HBV, HBV1)


# ---- error paths (argument validation only) ---------------------------------------------------------------------------------------
def test_error_paths_on_the_gpu(tmp_path):
    from test_hessian_ops_cpu import check_error_lines, run_errors_program
    libdir = os.path.join(ROOT, "lbfgspp_b200")
    out = run_errors_program(tmp_path, ["-L", libdir, "-l:liblbfgs_b200.so", "-Wl,-rpath," + libdir], args=["resident"])
    check_error_lines(out)
    assert out["batch before minimize"] == "logic_error: LBFGSBatchSolver: no history yet (minimize() has not run)"
    assert out["batch problem 2 of 2"] == "invalid_argument: LBFGSBatchSolver: problem index out of range"
    assert out["batch size mismatch"] == "invalid_argument: V.size() must be a positive multiple of n"
    assert out["batch two vectors"] == "ok"
