"""The diagonals of the final L-BFGS approximation on the GPU: the large-n pass (lbfgs_b200_hist_quad_diag) against float64 numpy, the
front's diag B / diag H (LBFGSSolver / LBFGSBatchSolver::final_approx_*_diagonal) against the dense matrices and the products, at C2 / C5
scale, the small-batch diagonals (lbfgs_b200_small_hist_diag) against the dense matrices and numpy over the kept columns, and the error
paths."""
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb
from test_gpu_hessian_ops import seeded_ring
from test_gpu_small_batch_hessian import MAXIT, OBJECTIVES, dense_ref, kept, problem, solve_keep

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel_err(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


# ---- the large-n pass ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("m", [6, 10, 20, 64])
@pytest.mark.parametrize("cwant", ["0", "1", "5", "m"])
def test_kernel_against_float64(gpu_ctx, dtype, m, cwant):
    n = 100_003
    npairs = {"0": 0, "1": 1, "5": 5, "m": m + 3}[cwant]   # c = m: a wrapped ring
    h, Y, S = seeded_ring(gpu_ctx, n, m, npairs, dtype, seed=m * 10 + npairs + 1)
    c = h.ncorr
    W = np.concatenate([Y, S])       # rows y by age, then s by age
    rng = np.random.default_rng(5 + m + npairs)
    A = rng.standard_normal((2 * c, 2 * c))
    K = ((A + A.T) / 2).astype(dtype)
    Kl = K.copy()
    Kl[np.tril_indices(2 * c, -1)] = np.nan     # only the upper triangle may be read
    a0 = 0.75
    out = gpu_ctx.array(np.full(n + 7, np.nan, dtype=dtype))
    h.quad_diag(a0, Kl, out)
    got = out.get()
    assert np.all(np.isnan(got[n:])), "entries past n were written"
    Kd = K.astype(np.float64)
    ref = a0 + np.einsum("pi,pq,qi->i", W, Kd, W)
    bound = abs(a0) + np.einsum("pi,pq,qi->i", np.abs(W), np.abs(Kd), np.abs(W))
    tol = 1e-12 if dtype == np.float64 else 1e-5
    assert np.all(np.abs(got[:n] - ref) <= tol * bound), np.max(np.abs(got[:n] - ref) / bound)
    if c == 0:
        assert np.all(got[:n] == dtype(a0))


# ---- the front -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("resident", [False, True], ids=["host_loop", "resident"])
@pytest.mark.parametrize("n", [10, 1000])
def test_front_against_the_dense_matrices_and_the_products(resident, n):
    prm = lb.LBFGSParam(m=8)
    x0 = np.linspace(-1, 1, n)
    niter, x, Bd, Hd = lb.solve_dense(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "MoreThuente", resident=resident)
    niter2, x2, dB, dH = lb.solve_hessian_diagonal(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, "MoreThuente", resident=resident)
    assert niter2 == niter and np.array_equal(x2, x)
    tol_h = 1e-12 * max(1.0, np.linalg.cond(Bd))
    assert rel_err(dB, np.diag(Bd)) <= 1e-12, rel_err(dB, np.diag(Bd))
    assert rel_err(dH, np.diag(Hd)) <= tol_h, (rel_err(dH, np.diag(Hd)), tol_h)
    _, _, BV, HV, _ = lb.solve_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, x0, np.eye(n), prm, "MoreThuente", resident=resident)
    assert rel_err(dB, np.diag(BV)) <= 1e-12 and rel_err(dH, np.diag(HV)) <= 1e-12


def test_c2_shaped_solve():
    n = 10_000_000
    prm = lb.LBFGSParam(m=10)
    _, _, dB, dH = lb.solve_hessian_diagonal(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n), prm, "MoreThuente", resident=True)
    assert np.all(np.isfinite(dB)) and np.all(dB > 0) and np.all(np.isfinite(dH)) and np.all(dH > 0)
    idx = np.sort(np.random.default_rng(32).choice(n, 32, replace=False))
    E = np.zeros((32, n))
    E[np.arange(32), idx] = 1.0
    _, _, BV, HV, _ = lb.solve_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n), E, prm, "MoreThuente", resident=True)
    assert rel_err(dB[idx], BV[np.arange(32), idx]) <= 1e-12
    assert rel_err(dH[idx], HV[np.arange(32), idx]) <= 1e-12


def test_c5_batch_member_equals_its_lone_solve():
    n, B, b = 1_000_000, 4, 2
    X0 = np.stack([np.random.default_rng(1000 + p).uniform(-1, 1, n) for p in range(B)])
    prm = lb.LBFGSParam(m=10)
    dB, dH = lb.batch_hessian_diagonal(lb.OBJ_ROSENBROCK_PAIRED, X0, b, prm, "MoreThuente")
    _, _, dB1, dH1 = lb.solve_hessian_diagonal(lb.OBJ_ROSENBROCK_PAIRED, X0[b], prm, "MoreThuente", resident=True)
    assert np.array_equal(dB, dB1) and np.array_equal(dH, dH1)
    assert np.all(dB > 0) and np.all(dH > 0)


# ---- the small batch -------------------------------------------------------------------------------------------------------------------
def diagonals(ctx, h, inverse, b0=0, count=None, ldo=None):
    count = h.B - b0 if count is None else count
    ldo = h.n if ldo is None else ldo
    O = ctx.array(np.full(count * ldo, np.nan, dtype=h.dtype))
    h.diagonal(inverse, b0, count, O, ldo)
    out = O.get().reshape(count, ldo)
    assert np.all(np.isnan(out[:, h.n:])), "the padding of OUT was written"
    return out[:, :h.n]


def check_small(gpu_ctx, objective, n, m, dtype, B=3, its=MAXIT):
    X0, d0, d1, ldd = problem(objective, B, n, 300 + n + m, dtype)
    h, _, _, _ = solve_keep(gpu_ctx, objective, X0, lb.LBFGSParam(m=m, max_iterations=its), "MoreThuente", d0, d1, ldd)
    c_all, th = h.info()
    eps = np.finfo(dtype).eps
    dB_all, dH_all = diagonals(gpu_ctx, h, 0, ldo=n + 3), diagonals(gpu_ctx, h, 1)
    for b in range(B):
        S, Y, _, _, _, _, theta = kept(h, b)
        Bm, Hm = dense_ref(S, Y, theta)
        tol = 1e-10 if dtype == np.float64 else max(1e-3, 100 * eps * np.linalg.cond(Bm))
        assert rel_err(dB_all[b].astype(np.float64), np.diag(Bm)) <= tol, (objective, n, m, b, int(c_all[b]))
        assert rel_err(dH_all[b].astype(np.float64), np.diag(Hm)) <= tol, (objective, n, m, b, int(c_all[b]))
        # one problem per call gives the same bits as all of them in one call
        assert np.array_equal(diagonals(gpu_ctx, h, 0, b, 1)[0], dB_all[b]) and np.array_equal(diagonals(gpu_ctx, h, 1, b, 1)[0], dH_all[b])
        if c_all[b] == 0:
            assert np.all(dB_all[b] == th[b]) and np.all(dH_all[b] == dtype(1) / th[b])
    return h, dB_all, dH_all


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("objective", OBJECTIVES)
def test_small_batch_against_the_reference(gpu_ctx, objective, dtype):
    for m in (1, 3, 10):
        check_small(gpu_ctx, objective, 30, m, dtype)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_small_batch_front_against_dense(dtype):
    """The driver entry (LBFGSSmallBatchSolver::final_approx_*_diagonal, all problems) against np.diag of the front's dense matrices."""
    n, B = 24, 4
    X0 = np.random.default_rng(9).uniform(-1.2, 1.2, (B, n)).astype(dtype)
    X0[1] = 1.0                      # the minimiser: stops with c = 0, theta = 1
    prm = lb.LBFGSParam(m=5, max_iterations=MAXIT)
    res, X, dB, dH = lb.small_batch_hessian_diagonal(lb.OBJ_ROSENBROCK_PAIRED, X0, prm, dtype=dtype)
    _, Xs, _ = lb.solve_small_batch(lb.OBJ_ROSENBROCK_PAIRED, X0, prm, dtype=dtype)
    assert np.array_equal(X, Xs)
    assert np.all(dB[1] == 1) and np.all(dH[1] == 1)
    I = np.eye(n, dtype=dtype)
    _, _, BV, HV, _ = lb.small_batch_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, X0, I, prm, dtype=dtype)
    tol = 1e-12 if dtype == np.float64 else 1e-4
    for b in range(B):   # row j of the products with I is column j of B_b / H_b: its diagonal is entry j of row j
        assert rel_err(dB[b].astype(np.float64), np.diag(BV[b]).astype(np.float64)) <= tol, b
        assert rel_err(dH[b].astype(np.float64), np.diag(HV[b]).astype(np.float64)) <= tol, b


def test_small_batch_positions_and_ranges(gpu_ctx):
    """A problem's diagonal does not depend on its position in the batch, b0 or count."""
    n, m = 40, 6
    p = np.random.default_rng(11).uniform(-1.2, 1.2, n)
    others = np.random.default_rng(12).uniform(-1.2, 1.2, (40, n))
    prm = lb.LBFGSParam(m=m, max_iterations=MAXIT)
    ha, _, _, _ = solve_keep(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, p[None, :], prm, "MoreThuente")
    want = [diagonals(gpu_ctx, ha, inv)[0] for inv in (0, 1)]
    for pos in (0, 17, 39):
        X0 = others.copy()
        X0[pos] = p
        h, _, _, _ = solve_keep(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "MoreThuente")
        for inv in (0, 1):
            assert np.array_equal(diagonals(gpu_ctx, h, inv)[pos], want[inv]), (pos, inv)
            for b0, count in ((pos, 1), (max(0, pos - 3), min(40, pos + 2) - max(0, pos - 3))):
                assert np.array_equal(diagonals(gpu_ctx, h, inv, b0, count)[pos - b0], want[inv]), (pos, inv, b0, count)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_small_batch_at_the_edges_of_the_budget(gpu_ctx, dtype):
    """n = small_max_n at m = 10, and the largest m whose products (and so the diagonal's algebra) fit."""
    obj = lb.OBJ_ROSENBROCK_PAIRED
    check_small(gpu_ctx, obj, lb.small_max_n(10, obj, dtype), 10, dtype, B=2)
    m_big = max(m for m in range(1, 65) if lb.small_max_n(m, obj, dtype) >= 4)
    n_big = lb.small_max_n(m_big, obj, dtype)
    check_small(gpu_ctx, obj, n_big, m_big, dtype, B=2, its=max(2, n_big // 2))


# ---- error paths (argument validation only) -------------------------------------------------------------------------------------------
def test_error_paths_on_the_gpu(tmp_path):
    from test_hessian_diag_cpu import CXX, EXPECTED
    libdir = os.path.join(ROOT, "lbfgspp_b200")
    exe = str(tmp_path / "hessian_diag_errors")
    subprocess.run(CXX + ["-o", exe, os.path.join(ROOT, "tests", "cpp", "hessian_diag_errors.cpp"), "-L", libdir, "-l:liblbfgs_b200.so",
                          "-Wl,-rpath," + libdir, "-pthread"], check=True)
    r = subprocess.run([exe, "gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.endswith("hessian diag errors done\n"), r.stdout + r.stderr
    out = dict(line.split(": ", 1) for line in r.stdout.splitlines()[:-1])
    for case, want in EXPECTED.items():
        assert out[case] == want, (case, out[case])
    no_hist = "logic_error: LBFGSSmallBatchSolver: no final approximation kept (call keep_final_approx(true) before minimize())"
    want = {
        "batch before minimize": "logic_error: LBFGSBatchSolver: no history yet (minimize() has not run)",
        "batch problem 2 of 2": "invalid_argument: LBFGSBatchSolver: problem index out of range",
        "batch problem -1": "invalid_argument: LBFGSBatchSolver: problem index out of range",
        "batch problem 1": "ok",
        "small before minimize": no_hist,
        "small not kept": no_hist,
        "small problem 3 of 3": "invalid_argument: LBFGSSmallBatchSolver: problem index out of range",
        "small problem 2": "ok",
        "small all": "ok",
        "small_hist_diag unfilled": "ERR_INVALID: small_hist_diag: no solve has filled the history",
        "small_hist_diag range": "ERR_INVALID: small_hist_diag: problems [2, 4) are not within the 3 of the history",
        "small_hist_diag b0<0": "ERR_INVALID: small_hist_diag: problems [-1, 0) are not within the 3 of the history",
        "small_hist_diag count=0": "ERR_INVALID: small_hist_diag: problems [0, 0) are not within the 3 of the history",
        "small_hist_diag NULL": "ERR_INVALID: small_hist_diag: NULL argument",
        "small_hist_diag ldo<n": "ERR_INVALID: small_hist_diag: leading dimension ldo = 7 must be at least n = 8",
        "small_hist_diag fp32": "ERR_INVALID: small_hist_diag: the history holds fp64 values",
        "small_hist_diag ok": "OK: ",
    }
    for case, w in want.items():
        assert out[case] == w, (case, out[case])
