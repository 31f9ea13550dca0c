"""The operator form of the final L-BFGS approximation (LBFGSSolver::final_approx_hessian_times / final_approx_inverse_hessian_times,
include/LBFGSpp/BFGSMat.h) on a CPU: the header-only front and the driver's units compiled against tests/cpp/mock_abi_hessian_ops.cpp,
the host-memory test double of the C ABI with the two k-vector passes.  The products must agree with the dense matrices of final_approx_hessian() /
final_approx_inverse_hessian() of the same solve, H must undo B, and misuse must raise the documented exceptions."""
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the test double of the C ABI (tests/cpp/mock_abi.cpp) with host versions of the two k-vector passes
MOCK = os.path.join(ROOT, "tests", "cpp", "mock_abi_hessian_ops.cpp")
CXX = ["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas"]


@pytest.fixture(scope="module")
def front(tmp_path_factory):
    import ctypes as C
    so = str(tmp_path_factory.mktemp("hessian_ops") / "front_on_mock.so")
    subprocess.run(CXX + ["-march=x86-64-v3", "-fPIC", "-shared", "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic",
                          "-o", so] + [os.path.join(ROOT, "lbfgspp_b200", "csrc", u) for u in lb.build.DRIVER_UNITS] + [MOCK, "-pthread"], check=True)
    return C.CDLL(so)


def rel_err(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


# (name, n, param, x0): no pair (the start is the minimiser), fewer pairs than m, a full ring that has wrapped
CASES = [("c=0", 10, dict(m=6), np.ones(10)),
         ("c<m", 64, dict(m=20, max_iterations=5), np.zeros(64)),
         ("c=m", 10, dict(m=3), np.full(10, -0.7)),
         ("c=m, n=64", 64, dict(m=6), np.linspace(-1, 1, 64))]


@pytest.mark.parametrize("ls", ["Backtracking", "Bracketing", "NocedalWright", "MoreThuente"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_products_match_the_dense_matrices(front, ls, case):
    name, n, kw, x0 = case
    prm = lb.LBFGSParam(**kw)
    niter, x, Bd, Hd = lb.solve_dense(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, ls, resident=False, lib=front)
    # H is compared with the inverse of a B that is itself exact only to rounding (its products agree to 1e-12): inverting amplifies
    # that by up to cond(B) (1e3 - 1e4 on these solves), so the bar of everything that involves H scales with it
    tol_h = 1e-12 * max(1.0, np.linalg.cond(Bd))
    rng = np.random.default_rng(n + len(name))
    for k in (1, 3, 17):   # 17: two groups of vectors per pass (16 + 1)
        V = rng.standard_normal((k, n))
        niter2, x2, BV, HV, HBV = lb.solve_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, x0, V, prm, ls, resident=False, lib=front)
        assert niter2 == niter and np.array_equal(x2, x), (name, ls)
        assert rel_err(BV, V @ Bd.T) <= 1e-12, (name, ls, k, rel_err(BV, V @ Bd.T))
        assert rel_err(HV, V @ Hd.T) <= tol_h, (name, ls, k, rel_err(HV, V @ Hd.T), tol_h)
        assert rel_err(HBV, V) <= tol_h, (name, ls, k, rel_err(HBV, V), tol_h)
    if name == "c=0":   # B = theta I and H = I / theta with theta = 1 after a reset
        assert np.array_equal(BV, V) and np.array_equal(HV, V)


def test_driver_reports_a_size_mismatch(front):
    with pytest.raises(RuntimeError, match="^solve_hessian_times failed: V.size\\(\\) must be a positive multiple of n$"):
        lb.solve_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(10), np.zeros(15), lb.LBFGSParam(), resident=False, lib=front)


def run_errors_program(tmp_path, link, args=()):
    exe = str(tmp_path / "hessian_ops_errors")
    subprocess.run(CXX + ["-o", exe, os.path.join(ROOT, "tests", "cpp", "hessian_ops_errors.cpp")] + link + ["-pthread"], check=True)
    r = subprocess.run([exe] + list(args), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.endswith("hessian ops errors done\n"), r.stdout + r.stderr
    return dict(line.split(": ", 1) for line in r.stdout.splitlines()[:-1])


EXPECTED = {
    "before minimize, B": "logic_error: BFGSMat: no history yet (minimize() has not run)",
    "before minimize, H": "logic_error: BFGSMat: no history yet (minimize() has not run)",
    "size mismatch, B": "invalid_argument: V.size() must be a positive multiple of n",
    "size mismatch, H": "invalid_argument: V.size() must be a positive multiple of n",
    "empty V": "invalid_argument: V.size() must be a positive multiple of n",
    "two vectors": "ok",
}
ABI_EXPECTED = {
    "wt_dot_multi k=0": "ERR_INVALID: hist_wt_dot_multi: k must be in 1..16",
    "wt_dot_multi k=17": "ERR_INVALID: hist_wt_dot_multi: k must be in 1..16",
    "wt_dot_multi ldv<n": "ERR_INVALID: hist_wt_dot_multi: leading dimension",
    "wt_dot_multi NULL": "ERR_INVALID: hist_wt_dot_multi: NULL argument",
    "lincomb_multi k=0": "ERR_INVALID: hist_lincomb_multi: k must be in 1..16",
    "lincomb_multi k=17": "ERR_INVALID: hist_lincomb_multi: k must be in 1..16",
    "lincomb_multi ldo<n": "ERR_INVALID: hist_lincomb_multi: leading dimension",
    "lincomb_multi NULL": "ERR_INVALID: hist_lincomb_multi: NULL argument",
}


def check_error_lines(out):
    for case, want in EXPECTED.items():
        assert out[case] == want, (case, out[case])
    for case, want in ABI_EXPECTED.items():
        assert out[case].startswith(want), (case, out[case])


def test_error_paths_on_the_test_double(tmp_path):
    check_error_lines(run_errors_program(tmp_path, [MOCK]))
