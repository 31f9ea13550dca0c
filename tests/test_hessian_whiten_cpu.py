"""Whitening and log densities under N(mu, H) of the final L-BFGS approximation on a CPU: the transpose and the inverses of the
square-root factor and the quadratic form of include/LBFGSpp/CompactForm.h (compact_factor_upper / compact_factor_t_coef /
compact_factor_inv_coef / compact_factor_invt_coef / compact_factor_quad, compiled by g++ as BFGSMat uses them) against a float64 dense
BFGS recursion and scipy's multivariate normal, and a -Werror compile of every new member of the front."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = ["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas"]


@pytest.fixture(scope="module")
def whiten(tmp_path_factory):
    d = tmp_path_factory.mktemp("whiten")
    src = d / "w.cpp"
    src.write_text("""
#include <cmath>
#include <vector>
#include <LBFGSpp/CompactForm.h>
using namespace LBFGSpp;
// op 0: L Z, 1: L' Z, 2: L^-1 Z, 3: L^-T Z for k vectors (columns of Z, n x k row-major) from W = [Y S] by age (n x 2c row-major) and
// its Gram blocks by age; q[j] = Z_j' B Z_j.  Returns compact_factor_setup's status.
extern "C" int factor_apply(int op, int n, int c, int k, const double* W, const double* SY, const double* SS, const double* YY, double theta,
                            const double* Z, double* OUT, double* q, double* logsum)
{
    std::vector<double> beta((size_t)(2 * c * c + 1)), Tm((size_t)(c * c + 1)), wv((size_t)(2 * c + 1)), C((size_t)(2 * c + 1)),
        z((size_t)(c + 1));
    const int st = compact_factor_setup(c, SY, SS, YY, c, theta, beta.data(), Tm.data(), logsum);
    if (st) return st;
    if (op >= 2) compact_factor_upper(c, SY, c, Tm.data());
    const double rsq = 1.0 / std::sqrt(theta), sq = std::sqrt(theta);
    for (int j = 0; j < k; j++)
    {
        double vv = 0.0;
        for (int i = 0; i < n; i++) vv += Z[i * k + j] * Z[i * k + j];
        for (int r = 0; r < 2 * c; r++)
        {
            double acc = 0.0;
            for (int i = 0; i < n; i++) acc += W[i * 2 * c + r] * Z[i * k + j];
            wv[(size_t)r] = acc;
        }
        if (op == 0) compact_factor_coef(c, beta.data(), Tm.data(), rsq, wv.data(), 1, C.data(), 1);
        if (op == 1) compact_factor_t_coef(c, beta.data(), Tm.data(), rsq, wv.data() + c, 1, z.data(), C.data(), 1);
        if (op == 2) compact_factor_inv_coef(c, beta.data(), Tm.data(), sq, wv.data(), 1, z.data(), C.data(), 1);
        if (op == 3) compact_factor_invt_coef(c, beta.data(), Tm.data(), sq, wv.data() + c, 1, z.data(), C.data(), 1);
        if (op >= 2) q[j] = compact_factor_quad(c, beta.data(), Tm.data(), SS, c, theta, wv.data(), 1, vv, z.data());
        const double a0 = op <= 1 ? rsq : sq;
        for (int i = 0; i < n; i++)
        {
            double acc = a0 * Z[i * k + j];
            for (int r = 0; r < 2 * c; r++) acc += C[(size_t)r] * W[i * 2 * c + r];
            OUT[i * k + j] = acc;
        }
    }
    return 0;
}
""")
    so = str(d / "w.so")
    subprocess.run(CXX + ["-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-o", so, str(src)], check=True)
    lib = C.CDLL(so)
    dp = C.POINTER(C.c_double)
    lib.factor_apply.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, dp, dp, dp, dp, C.c_double, dp, dp, dp, dp]
    return lib


def _p(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def bfgs_dense_inverse(S, Y, theta):
    """H by the BFGS recursion from I/theta, pairs applied oldest first; S, Y by age (row 0 newest)."""
    n = S.shape[1]
    H = np.eye(n) / theta
    for s, y in zip(S[::-1], Y[::-1]):
        rho = 1.0 / (y @ s)
        V = np.eye(n) - rho * np.outer(y, s)
        H = V.T @ H @ V + rho * np.outer(s, s)
    return H


def history(n, c, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n)) / np.sqrt(n)
    A = A @ A.T + 0.5 * np.eye(n)
    S = rng.standard_normal((c, n))
    Y = S @ A.T
    theta = (Y[0] @ Y[0] / (S[0] @ Y[0])) if c else 1.7
    return S, Y, theta


def run(lib, op, S, Y, theta, Z):
    c, n = S.shape
    k = Z.shape[1]
    W = np.ascontiguousarray(np.concatenate([Y, S]).T) if c else np.zeros((n, 1))
    SY, SS, YY = [np.ascontiguousarray(a) if c else np.zeros(1) for a in (S @ Y.T, S @ S.T, Y @ Y.T)]
    Zc = np.ascontiguousarray(Z)
    OUT = np.zeros((n, k))
    q = np.zeros(k)
    ls = C.c_double(0.0)
    st = lib.factor_apply(op, n, c, k, _p(W), _p(SY), _p(SS), _p(YY), theta, _p(Zc), _p(OUT), _p(q), C.byref(ls))
    return st, OUT, q, ls.value


SHAPES = [(7, 0), (7, 3), (5, 5), (40, 10), (80, 25), (200, 20), (150, 64)]


@pytest.mark.parametrize("n,c", SHAPES)
def test_transpose_and_inverses_match_dense(whiten, n, c):
    S, Y, theta = history(n, c, 300 + n + c)
    Z = np.random.default_rng(n + c).standard_normal((n, 6))
    st, L, _, _ = run(whiten, 0, S, Y, theta, np.eye(n))
    assert st == 0
    H = bfgs_dense_inverse(S, Y, theta)
    assert np.linalg.norm(L @ L.T - H) <= 1e-12 * np.linalg.norm(H)
    cond = np.linalg.cond(L)
    for op, want in ((1, L.T @ Z), (2, np.linalg.solve(L, Z)), (3, np.linalg.solve(L.T, Z))):
        st, got, _, _ = run(whiten, op, S, Y, theta, Z)
        assert st == 0
        assert np.linalg.norm(got - want) <= 1e-13 * cond * np.linalg.norm(want), op


@pytest.mark.parametrize("n,c", SHAPES)
def test_quadratic_form_is_v_b_v(whiten, n, c):
    S, Y, theta = history(n, c, 500 + n + c)
    V = np.random.default_rng(7 + n).standard_normal((n, 5))
    H = bfgs_dense_inverse(S, Y, theta)
    want = np.einsum("ij,ij->j", V, np.linalg.solve(H, V))
    for op in (2, 3):
        st, LiV, q, _ = run(whiten, op, S, Y, theta, V)
        assert st == 0
        assert np.allclose(q, want, rtol=1e-9 * np.linalg.cond(H), atol=0)
    _, LiV, _, _ = run(whiten, 2, S, Y, theta, V)
    assert np.allclose(np.sum(LiV ** 2, axis=0), q, rtol=1e-9 * np.linalg.cond(H), atol=0)


@pytest.mark.parametrize("n,c", [(6, 0), (6, 4), (12, 12), (30, 9)])
def test_log_density_matches_scipy(whiten, n, c):
    stats = pytest.importorskip("scipy.stats")
    S, Y, theta = history(n, c, 900 + n + c)
    rng = np.random.default_rng(n * 31 + c)
    mu = rng.standard_normal(n)
    X = mu[:, None] + rng.standard_normal((n, 4))
    st, _, q, ls = run(whiten, 2, S, Y, theta, X - mu[:, None])
    assert st == 0
    logdet = -n * np.log(theta) + ls
    got = -0.5 * q - 0.5 * logdet - 0.5 * n * np.log(2 * np.pi)
    want = stats.multivariate_normal(mean=mu, cov=bfgs_dense_inverse(S, Y, theta)).logpdf(X.T)
    assert np.allclose(got, want, rtol=1e-10, atol=1e-9)


def test_no_pairs_is_a_scaled_identity(whiten):
    n, theta = 9, 2.5
    S = Y = np.zeros((0, n))
    V = np.random.default_rng(1).standard_normal((n, 3))
    for op, scale in ((1, 1 / np.sqrt(theta)), (2, np.sqrt(theta)), (3, np.sqrt(theta))):
        st, got, q, _ = run(whiten, op, S, Y, theta, V)
        assert st == 0
        assert np.allclose(got, scale * V, rtol=1e-15, atol=0)
        if op >= 2:
            assert np.allclose(q, theta * np.sum(V ** 2, axis=0), rtol=1e-15, atol=0)


def test_refuses_nonpositive_curvature(whiten):
    S, Y, theta = history(10, 3, 5)
    Y = Y.copy()
    Y[1] = -Y[1]
    st, _, _, _ = run(whiten, 2, S, Y, theta, np.eye(10))
    assert st == 2


def test_front_members_compile_with_werror(tmp_path):
    """Every new member of the front, in both precisions, compiles with -Werror."""
    src = tmp_path / "front.cpp"
    src.write_text("""
#include <LBFGSSmallBatch.h>
using namespace LBFGSpp;
template <class S> void f(LBFGSSolver<S>& s, LBFGSBatchSolver<S>& b, LBFGSSmallBatchSolver<S>& sb, BFGSMat<S>& m, DeviceVector<S>& V,
                          DeviceVector<S>& O)
{
    s.final_approx_inverse_hessian_factor_transpose_times(V, O); s.final_approx_inverse_hessian_factor_solve(V, O);
    s.final_approx_inverse_hessian_factor_transpose_solve(V, O); (void)s.final_approx_log_density(V, O);
    b.final_approx_inverse_hessian_factor_transpose_times(0, V, O); b.final_approx_inverse_hessian_factor_solve(0, V, O);
    b.final_approx_inverse_hessian_factor_transpose_solve(0, V, O); (void)b.final_approx_log_density(0, V, O);
    sb.final_approx_inverse_hessian_factor_transpose_times(V, O); sb.final_approx_inverse_hessian_factor_solve(V, O);
    sb.final_approx_inverse_hessian_factor_transpose_solve(V, O); (void)sb.final_approx_log_density(V, O);
    sb.final_approx_inverse_hessian_factor_transpose_times(0L, V, O); sb.final_approx_inverse_hessian_factor_solve(0L, V, O);
    sb.final_approx_inverse_hessian_factor_transpose_solve(0L, V, O); (void)sb.final_approx_log_density(0L, V, O);
    m.inverse_hessian_factor_transpose_times(V, 1, O); m.inverse_hessian_factor_solve(V, 1, O);
    m.inverse_hessian_factor_transpose_solve(V, 1, O); (void)m.log_density(V, O, 1);
}
template void f<double>(LBFGSSolver<double>&, LBFGSBatchSolver<double>&, LBFGSSmallBatchSolver<double>&, BFGSMat<double>&,
                        DeviceVector<double>&, DeviceVector<double>&);
template void f<float>(LBFGSSolver<float>&, LBFGSBatchSolver<float>&, LBFGSSmallBatchSolver<float>&, BFGSMat<float>&,
                       DeviceVector<float>&, DeviceVector<float>&);
""")
    subprocess.run(CXX + ["-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", "-o", str(tmp_path / "front.o"), str(src)], check=True)


# ---- the front and the driver on the test double -------------------------------------------------------------------------------------
import lbfgspp_b200 as lb   # noqa: E402

MOCK = os.path.join(ROOT, "tests", "cpp", "mock_abi_hessian_whiten.cpp")
DRIVER_FLAGS = ["-fPIC", "-shared", "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic"]


def driver_on(tmp_path_factory, mock, name):
    so = str(tmp_path_factory.mktemp(name) / (name + ".so"))
    subprocess.run(CXX + DRIVER_FLAGS + ["-o", so] + [os.path.join(ROOT, "lbfgspp_b200", "csrc", u) for u in lb.build.DRIVER_UNITS]
                   + [mock, "-pthread"], check=True)
    return C.CDLL(so)


@pytest.fixture(scope="module")
def front(tmp_path_factory):
    return driver_on(tmp_path_factory, MOCK, "front_on_whiten_mock")


def rel_err(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


# no pair, fewer pairs than m, a full ring that has wrapped
CASES = [("c=0", 10, dict(m=6), np.ones(10)),
         ("c<m", 64, dict(m=20, max_iterations=5), np.zeros(64)),
         ("c=m", 10, dict(m=3), np.full(10, -0.7)),
         ("c=m, n=64", 64, dict(m=6), np.linspace(-1, 1, 64))]


@pytest.mark.parametrize("ls", ["Backtracking", "Bracketing", "NocedalWright", "MoreThuente"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_front_matches_the_dense_matrices(front, ls, case):
    """The host-driven loop on the test double: L' V, L^-1 V, L^-T V against the dense B and H of the same solve (L L' = H, L^-1 V
    from L, |L^-1 v|^2 = v'B v with B formed directly), and the log density against scipy with covariance H."""
    stats = pytest.importorskip("scipy.stats")
    name, n, kw, x0 = case
    prm = lb.LBFGSParam(**kw)
    niter, x, Bd, Hd = lb.solve_dense(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, ls, resident=False, lib=front)
    _, _, L = lb.solve_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, x0, np.eye(n), "L", prm, ls, resident=False, lib=front)
    L = L.T
    tol = 1e-12 * max(1.0, np.linalg.cond(Hd))
    assert rel_err(L @ L.T, Hd) <= tol, (name, ls)
    V = np.random.default_rng(n).standard_normal((5, n))
    out = {}
    for op, want in (("LT", V @ L), ("LINV", np.linalg.solve(L, V.T).T), ("LINVT", np.linalg.solve(L.T, V.T).T)):
        niter2, x2, O = lb.solve_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, x0, V, op, prm, ls, resident=False, lib=front)
        assert niter2 == niter and np.array_equal(x2, x), (name, ls, op)
        assert rel_err(O, want) <= tol, (name, ls, op, rel_err(O, want))
        out[op] = O
    q = np.einsum("ij,ij->i", V, V @ Bd.T)
    assert np.allclose(np.sum(out["LINV"] ** 2, axis=1), q, rtol=tol, atol=0), (name, ls)
    P = x + 0.1 * V
    _, _, lp = lb.solve_hessian_log_density(lb.OBJ_ROSENBROCK_PAIRED, x0, P, None, prm, ls, resident=False, lib=front)
    want = stats.multivariate_normal(mean=x, cov=Hd).logpdf(P)
    assert np.allclose(lp, want, rtol=tol, atol=tol * n), (name, ls, lp, want)
    if name == "c=0":   # theta = 1 after a reset: every op is the identity
        assert all(np.array_equal(O, V) for O in out.values())


@pytest.mark.parametrize("npairs, m", [(0, 4), (3, 5), (9, 4), (20, 20)])
def test_explicit_history_matches_the_recursion(front, npairs, m):
    """BFGSMat on an explicit ring against the float64 dense BFGS recursion of the kept pairs, with 20 vectors (two groups of 16)."""
    stats = pytest.importorskip("scipy.stats")
    rng = np.random.default_rng(11 * npairs + m)
    n = 50
    S = rng.standard_normal((npairs, n))
    Y = S * (1.0 + rng.random(n)) + 0.01 * rng.standard_normal((npairs, n))
    kS, kY = S[::-1][:m], Y[::-1][:m]
    theta = (kY[0] @ kY[0] / (kS[0] @ kY[0])) if npairs else 1.0
    H = bfgs_dense_inverse(kS, kY, theta)
    L = lb.hist_hessian_factor(S, Y, np.eye(n), "L", m=m, lib=front).T
    cond = np.linalg.cond(H)
    assert rel_err(L @ L.T, H) <= 1e-12 * cond
    V = rng.standard_normal((20, n))
    for op, want in (("LT", V @ L), ("LINV", np.linalg.solve(L, V.T).T), ("LINVT", np.linalg.solve(L.T, V.T).T)):
        assert rel_err(lb.hist_hessian_factor(S, Y, V, op, m=m, lib=front), want) <= 1e-12 * cond, op
    mean = rng.standard_normal(n)
    X = mean + 0.3 * V
    lp = lb.hist_hessian_log_density(S, Y, X, mean, m=m, lib=front)
    assert np.allclose(lp, stats.multivariate_normal(mean=mean, cov=H).logpdf(X), rtol=1e-12 * cond, atol=1e-12 * cond * n)


EXPECTED_ERRORS = {
    "solver before minimize, LT": "logic_error", "solver before minimize, LINV": "logic_error",
    "solver before minimize, LINVT": "logic_error", "solver before minimize, log density": "logic_error",
    "solver after minimize, LT": "ok", "solver after minimize, log density": "ok",
    "solver, V of n + 1": "invalid_argument", "solver, X of n + 1": "invalid_argument", "solver, mean of n - 1": "invalid_argument",
    "batch before minimize, LT": "logic_error", "batch before minimize, LINV": "logic_error",
    "batch before minimize, LINVT": "logic_error", "batch before minimize, log density": "logic_error",
    "s_dot_multi, k = 1": "OK", "s_dot_multi, k = 0": "ERR_INVALID", "s_dot_multi, k = 17": "ERR_INVALID",
    "s_dot_multi, ldv < n": "ERR_INVALID", "s_dot_multi, NULL R": "ERR_INVALID",
    "wt_dot_diff, k = 1": "OK", "wt_dot_diff, k = 0": "ERR_INVALID", "wt_dot_diff, k = 17": "ERR_INVALID",
    "wt_dot_diff, ldx < n": "ERR_INVALID", "wt_dot_diff, NULL mean": "ERR_INVALID", "wt_dot_diff, NULL norms": "ERR_INVALID",
}


def test_error_paths_on_the_test_double(tmp_path):
    """std::logic_error before a solve, std::invalid_argument for bad sizes, ERR_INVALID from the passes for bad k, leading dimensions
    and NULL arguments."""
    exe = str(tmp_path / "hessian_whiten_errors")
    subprocess.run(CXX + ["-o", exe, os.path.join(ROOT, "tests", "cpp", "hessian_whiten_errors.cpp"), MOCK, "-pthread"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.endswith("hessian whiten errors done\n"), r.stdout + r.stderr
    assert dict(line.split(": ", 1) for line in r.stdout.splitlines()[:-1]) == EXPECTED_ERRORS


def test_driver_error_paths(front):
    V = np.eye(4)
    with pytest.raises(RuntimeError, match="op must be"):
        lb.solve_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(4), V, 4, resident=False, lib=front)
    with pytest.raises(RuntimeError, match="op must be"):
        lb.hist_hessian_factor(np.ones((1, 4)), np.ones((1, 4)), V, -1, lib=front)
    with pytest.raises(ValueError, match="op must be"):
        lb.small_batch_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, np.zeros((2, 4)), np.zeros((2, 1, 4)), 7, lib=front)
    with pytest.raises(RuntimeError, match="need a mean"):
        lb.hist_hessian_log_density(np.ones((1, 4)), np.ones((1, 4)), V, None, lib=front)
    Yneg = -np.ones((1, 4))                               # y's < 0: no positive definite H
    for op in ("LT", "LINV", "LINVT"):
        with pytest.raises(RuntimeError, match="positive definite"):
            lb.hist_hessian_factor(np.ones((1, 4)), Yneg, V, op, lib=front)
    assert np.all(np.isnan(lb.hist_hessian_log_density(np.ones((1, 4)), Yneg, V, np.zeros(4), lib=front)))


def test_driver_reports_the_missing_entry_points(tmp_path_factory):
    """Against the test double without the whitening passes, the driver library still loads and says what is missing; against any
    test double (none has a small-batch history) the small-batch entry points name theirs."""
    lib = driver_on(tmp_path_factory, os.path.join(ROOT, "tests", "cpp", "mock_abi_hessian_sample.cpp"), "drv_on_sample_mock")
    for call in (lambda: lb.solve_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(4), np.eye(4), "LT", resident=False, lib=lib),
                 lambda: lb.solve_hessian_log_density(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(4), np.eye(4), resident=False, lib=lib),
                 lambda: lb.batch_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, np.zeros((2, 4)), 0, np.eye(4), "LINV", lib=lib),
                 lambda: lb.hist_hessian_factor(np.ones((1, 4)), np.ones((1, 4)), np.eye(4), "LINVT", lib=lib)):
        with pytest.raises(RuntimeError, match="lbfgs_b200_hist_s_dot_multi_"):
            call()
    for dt in (np.float64, np.float32):
        with pytest.raises(RuntimeError, match="lbfgs_b200_small_hist_factor_apply_"):
            lb.small_batch_hessian_factor(lb.OBJ_ROSENBROCK_PAIRED, np.zeros((2, 4)), np.zeros((2, 1, 4)), "LT", dtype=dt, lib=lib)
        with pytest.raises(RuntimeError, match="lbfgs_b200_small_hist_log_density_"):
            lb.small_batch_hessian_log_density(lb.OBJ_ROSENBROCK_PAIRED, np.zeros((2, 4)), np.zeros((2, 1, 4)), dtype=dt, lib=lib)
