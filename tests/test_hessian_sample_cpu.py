"""Draws from N(x*, H) and log det H of the final L-BFGS approximation on a CPU: the square-root factor of
include/LBFGSpp/CompactForm.h (compact_factor_setup / compact_factor_coef, compiled by g++ as BFGSMat uses them) against a float64 dense
BFGS recursion, a numpy restatement of the counter-based normal generator of lbfgspp_b200/csrc/philox.cuh against its known-answer
vectors, a -Werror compile of every new member of the front, and the front and the driver compiled against
tests/cpp/mock_abi_hessian_sample.cpp (the host test double of the C ABI with the sampler's passes) against the dense inverse of the same
solve across the four line searches, with their error paths."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = ["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas"]


# ---- the factor ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def factor(tmp_path_factory):
    d = tmp_path_factory.mktemp("factor")
    src = d / "f.cpp"
    src.write_text("""
#include <cmath>
#include <vector>
#include <LBFGSpp/CompactForm.h>
using namespace LBFGSpp;
// L Z for k vectors (columns of Z, n x k row-major) from W = [Y S] by age (W n x 2c row-major) and its Gram blocks by age
extern "C" int factor_times(int n, int c, int k, const double* W, const double* SY, const double* SS, const double* YY, double theta,
                            const double* Z, double* OUT, double* logsum)
{
    std::vector<double> beta((size_t)(2 * c * c + 1)), Tm((size_t)(c * c + 1)), wv((size_t)(2 * c + 1)), C((size_t)(2 * c + 1));
    const int st = compact_factor_setup(c, SY, SS, YY, c, theta, beta.data(), Tm.data(), logsum);
    if (st) return st;
    const double rsq = 1.0 / std::sqrt(theta);
    for (int j = 0; j < k; j++)
    {
        for (int r = 0; r < 2 * c; r++)
        {
            double acc = 0.0;
            for (int i = 0; i < n; i++) acc += W[i * 2 * c + r] * Z[i * k + j];
            wv[(size_t)r] = acc;
        }
        compact_factor_coef(c, beta.data(), Tm.data(), rsq, wv.data(), 1, C.data(), 1);
        for (int i = 0; i < n; i++)
        {
            double acc = rsq * Z[i * k + j];
            for (int r = 0; r < 2 * c; r++) acc += C[(size_t)r] * W[i * 2 * c + r];
            OUT[i * k + j] = acc;
        }
    }
    return 0;
}
""")
    so = str(d / "f.so")
    subprocess.run(CXX + ["-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-o", so, str(src)], check=True)
    lib = C.CDLL(so)
    dp = C.POINTER(C.c_double)
    lib.factor_times.argtypes = [C.c_int, C.c_int, C.c_int, dp, dp, dp, dp, C.c_double, dp, dp, dp]
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


def run_factor(lib, S, Y, theta, Z):
    c, n = S.shape
    k = Z.shape[1]
    W = np.ascontiguousarray(np.concatenate([Y, S]).T) if c else np.zeros((n, 1))
    SY, SS, YY = [np.ascontiguousarray(a) if c else np.zeros(1) for a in (S @ Y.T, S @ S.T, Y @ Y.T)]
    Zc = np.ascontiguousarray(Z)
    OUT = np.zeros((n, k))
    ls = C.c_double(0.0)
    st = lib.factor_times(n, c, k, _p(W), _p(SY), _p(SS), _p(YY), theta, _p(Zc), _p(OUT), C.byref(ls))
    return st, OUT, ls.value


@pytest.mark.parametrize("n,c", [(7, 0), (7, 3), (5, 5), (40, 10), (80, 25), (200, 20), (150, 64)])
def test_factor_matches_dense_bfgs(factor, n, c):
    S, Y, theta = history(n, c, 100 + n + c)
    st, L, ls = run_factor(factor, S, Y, theta, np.eye(n))
    assert st == 0
    H = bfgs_dense_inverse(S, Y, theta)
    assert np.linalg.norm(L @ L.T - H) <= 1e-12 * np.linalg.norm(H)
    sign, logdet = np.linalg.slogdet(H)
    assert sign > 0
    assert abs(-n * np.log(theta) + ls - logdet) <= 1e-10 * max(1.0, abs(logdet))


def test_factor_is_linear_in_z(factor):
    S, Y, theta = history(30, 6, 3)
    Z = np.random.default_rng(4).standard_normal((30, 5))
    _, L, _ = run_factor(factor, S, Y, theta, np.eye(30))
    _, LZ, _ = run_factor(factor, S, Y, theta, Z)
    assert np.allclose(LZ, L @ Z, rtol=1e-12, atol=1e-12)


def test_factor_refuses_nonpositive_curvature(factor):
    S, Y, theta = history(10, 3, 5)
    Y[1] = -Y[1]   # y's < 0 for the middle pair
    st, _, _ = run_factor(factor, S, Y, theta, np.eye(10))
    assert st == 2


# ---- the generator -------------------------------------------------------------------------------------------------------------------
M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for r in range(10):
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & MASK, p1 & MASK, ((p0 >> 32) ^ c3 ^ k1) & MASK, p0 & MASK
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return c0, c1, c2, c3


def uniforms(seed, stream, j, q):
    w = philox4x32_10((q & MASK, q >> 32, j, stream), (seed & MASK, seed >> 32))
    x0 = ((w[1] << 32) | w[0]) >> 11
    x1 = ((w[3] << 32) | w[2]) >> 11
    return (x0 + 1) * 2.0 ** -53, x1 * 2.0 ** -53


def normals(seed, stream, j, n):
    """Draw j of stream `stream`, coordinates 0..n-1, as the device makes it (to the rounding of log, sqrt and sincospi)."""
    z = np.empty(n + 1)
    for q in range((n + 1) // 2):
        u0, u1 = uniforms(seed, stream, j, q)
        r = np.sqrt(-2.0 * np.log(u0))
        z[2 * q], z[2 * q + 1] = r * np.cos(2 * np.pi * u1), r * np.sin(2 * np.pi * u1)
    return z[:n]


@pytest.mark.parametrize("ctr,key,out", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((MASK,) * 4, (MASK, MASK), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, out):
    assert philox4x32_10(ctr, key) == out


def test_uniforms_and_normals_of_the_counter_layout():
    # the key is the seed, the counter (q low, q high, draw, stream); the uniforms lie in (0, 1]
    seed = 0x0123456789ABCDEF
    w = philox4x32_10((5, 0, 7, 3), (0x89ABCDEF, 0x01234567))
    u0, u1 = uniforms(seed, 3, 7, 5)
    assert u0 == (((((w[1] << 32) | w[0]) >> 11) + 1) * 2.0 ** -53)
    assert 0.0 < u0 <= 1.0 and 0.0 <= u1 < 1.0
    z = normals(seed, 3, 7, 12)
    r = np.sqrt(-2 * np.log(u0))
    assert z[10] == r * np.cos(2 * np.pi * u1) and z[11] == r * np.sin(2 * np.pi * u1)
    # a draw depends on (seed, stream, j, i) only, and different streams / draws differ
    assert np.array_equal(normals(seed, 3, 7, 11), z[:11])
    assert not np.array_equal(normals(seed, 4, 7, 12), z)
    big = np.concatenate([normals(11, 0, j, 1000) for j in range(20)])
    assert abs(big.mean()) < 0.05 and abs(big.std() - 1) < 0.05


# ---- the front compiles cleanly ------------------------------------------------------------------------------------------------------
def test_front_members_compile_with_werror(tmp_path):
    src = tmp_path / "front.cpp"
    src.write_text("""
#include <LBFGS.h>
#include <LBFGSBatch.h>
#include <LBFGSSmallBatch.h>
using namespace LBFGSpp;
template <class S> void use(LBFGSSolver<S>& s, LBFGSBatchSolver<S>& bs, LBFGSSmallBatchSolver<S>& sb, BFGSMat<S>& m, DeviceVector<S>& V,
                            DeviceVector<S>& OUT)
{
    m.inverse_hessian_factor_times(V, 1, OUT);
    m.sample(&V, 7ull, 0u, 0u, 3, OUT);
    double d = m.inverse_hessian_logdet();
    s.final_approx_inverse_hessian_factor_times(V, OUT);
    s.final_approx_sample(V, 7ull, 0u, 4, OUT);
    d += s.final_approx_inverse_hessian_logdet();
    bs.final_approx_inverse_hessian_factor_times(0, V, OUT);
    bs.final_approx_sample(0, V, 7ull, 0u, 4, OUT);
    d += bs.final_approx_inverse_hessian_logdet(0);
    sb.final_approx_inverse_hessian_factor_times(V, OUT);
    sb.final_approx_inverse_hessian_factor_times(1, V, OUT);
    sb.final_approx_sample(V, 7ull, 0u, 4, OUT);
    sb.final_approx_sample(1, V, 7ull, 0u, 4, OUT);
    std::vector<double> all = sb.final_approx_inverse_hessian_logdet();
    d += sb.final_approx_inverse_hessian_logdet(1) + all[0];
    (void)d;
}
template void use<double>(LBFGSSolver<double>&, LBFGSBatchSolver<double>&, LBFGSSmallBatchSolver<double>&, BFGSMat<double>&,
                          DeviceVector<double>&, DeviceVector<double>&);
template void use<float>(LBFGSSolver<float>&, LBFGSBatchSolver<float>&, LBFGSSmallBatchSolver<float>&, BFGSMat<float>&,
                         DeviceVector<float>&, DeviceVector<float>&);
""")
    subprocess.run(CXX + ["-Werror", "-Wextra", "-c", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "front.o"), str(src)],
                   check=True)


# ---- the front and the driver on the test double -------------------------------------------------------------------------------------
import lbfgspp_b200 as lb   # noqa: E402

MOCK = os.path.join(ROOT, "tests", "cpp", "mock_abi_hessian_sample.cpp")


@pytest.fixture(scope="module")
def front(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hessian_sample") / "front_on_mock.so")
    subprocess.run(CXX + ["-march=x86-64-v3", "-fPIC", "-shared", "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic",
                          "-o", so] + [os.path.join(ROOT, "lbfgspp_b200", "csrc", u) for u in lb.build.DRIVER_UNITS] + [MOCK, "-pthread"], check=True)
    return C.CDLL(so)


def rel_err(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


# no pair, fewer pairs than m, a full ring that has wrapped
CASES = [("c=0", 10, dict(m=6), np.ones(10)),
         ("c<m", 64, dict(m=20, max_iterations=5), np.zeros(64)),
         ("c=m", 10, dict(m=3), np.full(10, -0.7)),
         ("c=m, n=64", 64, dict(m=6), np.linspace(-1, 1, 64))]


@pytest.mark.parametrize("ls", ["Backtracking", "Bracketing", "NocedalWright", "MoreThuente"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_front_matches_the_dense_inverse(front, ls, case):
    name, n, kw, x0 = case
    prm = lb.LBFGSParam(**kw)
    niter, x, _, Hd = lb.solve_dense(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, ls, resident=False, lib=front)
    seed, first, k = 123, 4, 3
    niter2, x2, L, D, ld = lb.solve_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, x0, np.eye(n), seed, first, k, prm, ls, resident=False, lib=front)
    assert niter2 == niter and np.array_equal(x2, x), (name, ls)
    L = L.T                                               # row j of the output is L e_j
    tol = 1e-12 * max(1.0, np.linalg.cond(Hd))            # the dense H inverts a B exact only to rounding
    assert rel_err(L @ L.T, Hd) <= tol, (name, ls, rel_err(L @ L.T, Hd))
    sign, want = np.linalg.slogdet(Hd)
    assert sign > 0 and abs(ld - want) <= 1e-10 * max(1.0, abs(want)), (name, ls, ld, want)
    Z = np.stack([normals(seed, 0, first + j, n) for j in range(k)])
    assert rel_err(D - x, Z @ L.T) <= 1e-12, (name, ls)
    if name == "c=0":   # theta = 1 after a reset: L = I, log det H = 0
        assert np.array_equal(L, np.eye(n)) and ld == 0.0


@pytest.mark.parametrize("npairs, m", [(0, 4), (3, 5), (9, 4)])
def test_explicit_history_matches_the_recursion(front, npairs, m):
    rng = np.random.default_rng(7 * npairs + m)
    n = 50
    S = rng.standard_normal((npairs, n))
    Y = S * (1.0 + rng.random(n)) + 0.01 * rng.standard_normal((npairs, n))
    mean = rng.standard_normal(n)
    L, D, ld = lb.hist_sample(S, Y, m=m, V=np.eye(n), mean=mean, seed=9, stream=6, first=0, k=20, lib=front)
    L = L.T
    kS, kY = S[::-1][:m], Y[::-1][:m]                     # by age, the newest m pairs
    theta = (kY[0] @ kY[0] / (kS[0] @ kY[0])) if npairs else 1.0
    H = bfgs_dense_inverse(kS, kY, theta)
    assert rel_err(L @ L.T, H) <= 1e-12 * np.linalg.cond(H)
    assert abs(ld - np.linalg.slogdet(H)[1]) <= 1e-10 * max(1.0, abs(ld))
    Z = np.stack([normals(9, 6, j, n) for j in range(20)])
    assert rel_err(D - mean, Z @ L.T) <= 1e-12


def test_driver_error_paths(front):
    with pytest.raises(RuntimeError, match="first \\+ k"):
        lb.solve_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(4), seed=1, first=0xFFFFFFFF, k=2, resident=False, lib=front)
    Yneg = -np.ones((1, 4))                               # y's < 0: no positive definite H
    with pytest.raises(RuntimeError, match="positive definite"):
        lb.hist_sample(np.ones((1, 4)), Yneg, k=1, lib=front)
    assert np.isnan(lb.hist_sample(np.ones((1, 4)), Yneg, lib=front)[2])


def test_driver_reports_the_missing_entry_points(tmp_path):
    """Against the test double without the sampler's passes, the driver library still loads and says what is missing."""
    so = str(tmp_path / "drv_on_diag_mock.so")
    subprocess.run(CXX + ["-fPIC", "-shared", "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic", "-o", so]
                   + [os.path.join(ROOT, "lbfgspp_b200", "csrc", u) for u in lb.build.DRIVER_UNITS]
                   + [os.path.join(ROOT, "tests", "cpp", "mock_abi_hessian_diag.cpp"), "-pthread"], check=True)
    lib = C.CDLL(so)
    with pytest.raises(RuntimeError, match="lbfgs_b200_hist_wt_dot_normal_"):
        lb.solve_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(4), k=1, resident=False, lib=lib)
    with pytest.raises(RuntimeError, match="lbfgs_b200_hist_wt_dot_normal_"):
        lb.hist_sample(np.ones((1, 4)), np.ones((1, 4)), lib=lib)
    for dt in (np.float64, np.float32):
        with pytest.raises(RuntimeError, match="lbfgs_b200_small_hist_sample_"):
            lb.small_batch_hessian_sample(lb.OBJ_ROSENBROCK_PAIRED, np.zeros((2, 4)), k=1, dtype=dt, lib=lib)
