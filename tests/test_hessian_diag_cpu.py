"""The diagonals of the final L-BFGS approximation (final_approx_hessian_diagonal / final_approx_inverse_hessian_diagonal) on a CPU: the
middle matrices K_B and K_H of include/LBFGSpp/CompactForm.h (compiled by g++, as BFGSMat uses them) against numpy, the header-only
front and the driver's units compiled against tests/cpp/mock_abi_hessian_diag.cpp (the host test double of the C ABI with the diagonal
pass) against the dense matrices of the same solve, and the error paths."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOCK = os.path.join(ROOT, "tests", "cpp", "mock_abi_hessian_diag.cpp")
CXX = ["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas"]


# ---- the K matrices ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kmats(tmp_path_factory):
    d = tmp_path_factory.mktemp("kmats")
    src = d / "k.cpp"
    src.write_text("""
#include <vector>
#include <LBFGSpp/CompactForm.h>
using namespace LBFGSpp;
// K_B as BFGSMat forms it: Minv -> BK factor -> M by unit columns -> compact_kb, then symmetrised
extern "C" void k_b(int c, const double* SY, const double* SS, double theta, double* K)
{
    const int w = 2 * c;
    std::vector<double> F((size_t)(w * w)), M((size_t)(w * w)), z((size_t)w), unit((size_t)(2 * w - 1), 0.0);
    std::vector<int> order((size_t)w);
    std::vector<unsigned char> tag((size_t)w);
    unit[(size_t)(w - 1)] = 1.0;
    compact_minv(c, SY, SS, c, theta, F.data());
    bk_factor(F.data(), w, order.data(), tag.data());
    for (int j = 0; j < w; j++)
    {
        for (int i = 0; i < w; i++) M[size_t(i * w + j)] = i == j ? 1.0 : 0.0;
        bk_solve(F.data(), w, order.data(), tag.data(), M.data() + j, w, z.data());
    }
    compact_kb(c, M.data(), theta, unit.data(), 0, 1, K);
    compact_k_symmetrise(w, K, 0, 1);
}
// K_H: R and Y'Y in chronological order -> compact_kh, two threads' worth of columns, then symmetrised by rows in two strides
extern "C" void k_h(int c, const double* SY, const double* YY, double theta, double* K)
{
    const int w = 2 * c;
    std::vector<double> R((size_t)(c * c)), YYc((size_t)(c * c)), scr((size_t)(2 * w)), unit((size_t)(2 * w - 1), 0.0);
    unit[(size_t)(w - 1)] = 1.0;
    compact_h_setup(c, SY, YY, c, R.data(), YYc.data());
    compact_kh(c, R.data(), YYc.data(), theta, unit.data(), 0, 2, scr.data(), 2, K);
    compact_kh(c, R.data(), YYc.data(), theta, unit.data(), 1, 2, scr.data() + 1, 2, K);
    compact_k_symmetrise(w, K, 1, 2);
    compact_k_symmetrise(w, K, 0, 2);
}
""")
    so = str(d / "k.so")
    subprocess.run(CXX + ["-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-o", so, str(src)], check=True)
    lib = C.CDLL(so)
    dp = C.POINTER(C.c_double)
    for name in ("k_b", "k_h"):
        getattr(lib, name).argtypes = [C.c_int, dp, dp, C.c_double, dp]
    return lib


def _p(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def bfgs_dense(S, Y):
    """B by the BFGS recursion from theta I (theta = y'y / s'y of the newest pair), pairs applied oldest first; S, Y by age (row 0 newest)."""
    n = S.shape[1]
    theta = Y[0] @ Y[0] / (S[0] @ Y[0])
    B = theta * np.eye(n)
    for s, y in zip(S[::-1], Y[::-1]):
        Bs = B @ s
        B = B - np.outer(Bs, Bs) / (s @ Bs) + np.outer(y, y) / (y @ s)
    return B, theta


@pytest.mark.parametrize("c", [1, 2, 5, 10, 20, 64])
def test_k_matrices_give_the_compact_form(kmats, c):
    rng = np.random.default_rng(100 + c)
    n = 2 * c + 40
    A = np.diag(1.0 + rng.random(n))                     # a well-conditioned curvature: y = A s keeps every pair positive
    S = rng.standard_normal((c, n))
    Y = S @ A.T + 0.01 * rng.standard_normal((c, n))
    SY, SS, YY = S @ Y.T, S @ S.T, Y @ Y.T               # by age: SY[a, b] = s_a'y_b
    B, theta = bfgs_dense(S, Y)
    W = np.hstack([Y.T, S.T])                            # [Y S], columns by age
    KB, KH = np.zeros((2 * c, 2 * c)), np.zeros((2 * c, 2 * c))
    kmats.k_b(c, _p(np.ascontiguousarray(SY)), _p(np.ascontiguousarray(SS)), theta, _p(KB))
    kmats.k_h(c, _p(np.ascontiguousarray(SY)), _p(np.ascontiguousarray(YY)), theta, _p(KH))
    assert np.array_equal(KB, KB.T) and np.array_equal(KH, KH.T)
    Bk = theta * np.eye(n) + W @ KB @ W.T
    Hk = np.eye(n) / theta + W @ KH @ W.T
    tol = 1e-12 * np.linalg.cond(B)
    assert np.max(np.abs(Bk - B)) <= tol * np.max(np.abs(B)), c
    H = np.linalg.inv(B)
    assert np.max(np.abs(Hk - H)) <= tol * np.max(np.abs(H)), c
    assert np.max(np.abs(KH[:c, :c])) == 0.0   # the y-y block of K_H is zero


# ---- the front and the driver on the test double -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def front(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hessian_diag") / "front_on_mock.so")
    subprocess.run(CXX + ["-march=x86-64-v3", "-fPIC", "-shared", "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic",
                          "-o", so] + [os.path.join(ROOT, "lbfgspp_b200", "csrc", u) for u in lb.build.DRIVER_UNITS] + [MOCK, "-pthread"], check=True)
    return C.CDLL(so)


def rel_err(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


# the cases of the operator form's tests: no pair, fewer pairs than m, a full ring that has wrapped
CASES = [("c=0", 10, dict(m=6), np.ones(10)),
         ("c<m", 64, dict(m=20, max_iterations=5), np.zeros(64)),
         ("c=m", 10, dict(m=3), np.full(10, -0.7)),
         ("c=m, n=64", 64, dict(m=6), np.linspace(-1, 1, 64))]


@pytest.mark.parametrize("ls", ["Backtracking", "Bracketing", "NocedalWright", "MoreThuente"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_diagonals_match_the_dense_matrices(front, ls, case):
    name, n, kw, x0 = case
    prm = lb.LBFGSParam(**kw)
    niter, x, Bd, Hd = lb.solve_dense(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, ls, resident=False, lib=front)
    niter2, x2, dB, dH = lb.solve_hessian_diagonal(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, ls, resident=False, lib=front)
    assert niter2 == niter and np.array_equal(x2, x), (name, ls)
    tol_h = 1e-12 * max(1.0, np.linalg.cond(Bd))   # the dense H inverts a B exact only to rounding (see test_hessian_ops_cpu.py)
    assert rel_err(dB, np.diag(Bd)) <= 1e-12, (name, ls, rel_err(dB, np.diag(Bd)))
    assert rel_err(dH, np.diag(Hd)) <= tol_h, (name, ls, rel_err(dH, np.diag(Hd)), tol_h)
    if name == "c=0":   # B = theta I and H = I / theta with theta = 1 after a reset
        assert np.array_equal(dB, np.ones(n)) and np.array_equal(dH, np.ones(n))


@pytest.mark.parametrize("npairs, m", [(0, 4), (3, 5), (9, 4)])
def test_explicit_history_matches_the_bfgs_recursion(front, npairs, m):
    rng = np.random.default_rng(7 * npairs + m)
    n = 50
    S = rng.standard_normal((npairs, n))
    Y = S * (1.0 + rng.random(n)) + 0.01 * rng.standard_normal((npairs, n))
    dB, dH = lb.hist_diagonal(S, Y, m=m, lib=front)
    if npairs == 0:
        assert np.array_equal(dB, np.ones(n)) and np.array_equal(dH, np.ones(n))
        return
    kept_S, kept_Y = S[::-1][:m], Y[::-1][:m]           # by age, the newest m pairs
    B, _ = bfgs_dense(kept_S, kept_Y)
    tol = 1e-12 * np.linalg.cond(B)
    assert rel_err(dB, np.diag(B)) <= tol
    assert rel_err(dH, np.diag(np.linalg.inv(B))) <= tol


EXPECTED = {
    "before minimize, B": "logic_error: BFGSMat: no history yet (minimize() has not run)",
    "before minimize, H": "logic_error: BFGSMat: no history yet (minimize() has not run)",
    "after minimize, B": "ok",
    "after minimize, H": "ok",
    "quad_diag NULL out": "ERR_INVALID: hist_quad_diag: NULL argument",
    "quad_diag NULL K": "ERR_INVALID: hist_quad_diag: NULL argument",
    "quad_diag ok": "OK: ",
}


def test_error_paths_on_the_test_double(tmp_path):
    exe = str(tmp_path / "hessian_diag_errors")
    subprocess.run(CXX + ["-o", exe, os.path.join(ROOT, "tests", "cpp", "hessian_diag_errors.cpp"), MOCK, "-pthread"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.endswith("hessian diag errors done\n"), r.stdout + r.stderr
    out = dict(line.split(": ", 1) for line in r.stdout.splitlines()[:-1])
    assert out == EXPECTED


def test_driver_reports_the_missing_entry_points(tmp_path):
    """Against the test double without the diagonal pass, the driver library still loads and says what is missing."""
    so = str(tmp_path / "drv_on_ops_mock.so")
    subprocess.run(CXX + ["-fPIC", "-shared", "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic", "-o", so]
                   + [os.path.join(ROOT, "lbfgspp_b200", "csrc", u) for u in lb.build.DRIVER_UNITS]
                   + [os.path.join(ROOT, "tests", "cpp", "mock_abi_hessian_ops.cpp"), "-pthread"], check=True)
    lib = C.CDLL(so)
    with pytest.raises(RuntimeError, match="lbfgs_b200_hist_quad_diag_"):
        lb.solve_hessian_diagonal(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(4), lb.LBFGSParam(), resident=False, lib=lib)
    with pytest.raises(RuntimeError, match="lbfgs_b200_hist_quad_diag_"):
        lb.hist_diagonal(np.ones((1, 4)), np.ones((1, 4)), lib=lib)
    for dt in (np.float64, np.float32):
        with pytest.raises(RuntimeError, match="lbfgs_b200_small_hist_diag_"):
            lb.small_batch_hessian_diagonal(lb.OBJ_ROSENBROCK_PAIRED, np.zeros((2, 4)), dtype=dt, lib=lib)


def test_front_members_compile(tmp_path):
    src = tmp_path / "tu.cpp"
    src.write_text("""
#include <LBFGS.h>
#include <LBFGSBatch.h>
#include <LBFGSSmallBatch.h>
using namespace LBFGSpp;
template <class S> void use(LBFGSSolver<S, LineSearchMoreThuente>& s, LBFGSBatchSolver<S, LineSearchMoreThuente>& b,
                            LBFGSSmallBatchSolver<S, LineSearchMoreThuente>& sb, BFGSMat<S>& mat, DeviceVector<S>& O)
{
    s.final_approx_hessian_diagonal(O);
    s.final_approx_inverse_hessian_diagonal(O);
    b.final_approx_hessian_diagonal(1, O);
    b.final_approx_inverse_hessian_diagonal(1, O);
    sb.final_approx_hessian_diagonal(O);
    sb.final_approx_inverse_hessian_diagonal(O);
    sb.final_approx_hessian_diagonal(1L, O);
    sb.final_approx_inverse_hessian_diagonal(1L, O);
    mat.hessian_diagonal(O);
    mat.inverse_hessian_diagonal(O);
}
template void use<double>(LBFGSSolver<double, LineSearchMoreThuente>&, LBFGSBatchSolver<double, LineSearchMoreThuente>&,
                          LBFGSSmallBatchSolver<double, LineSearchMoreThuente>&, BFGSMat<double>&, DeviceVector<double>&);
template void use<float>(LBFGSSolver<float, LineSearchMoreThuente>&, LBFGSBatchSolver<float, LineSearchMoreThuente>&,
                         LBFGSSmallBatchSolver<float, LineSearchMoreThuente>&, BFGSMat<float>&, DeviceVector<float>&);
""")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o",
                    str(tmp_path / "tu.o")], check=True)
