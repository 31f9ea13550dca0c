"""CPU checks of the kept small-batch approximations: the driver still loads against a C ABI without them and says what is missing,
the C++ front's new members compile, and the compact-form algebra of include/LBFGSpp/CompactForm.h (compiled by g++, as BFGSMat uses
it) agrees with numpy on random pairs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CXX = ["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas"]


def test_driver_reports_the_missing_entry_points(tmp_path):
    so = str(tmp_path / "drv_on_mock.so")
    subprocess.run(CXX + ["-fPIC", "-shared", "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic", "-o", so]
                   + [os.path.join(ROOT, "lbfgspp_b200", "csrc", u) for u in lb.build.DRIVER_UNITS]
                   + [os.path.join(ROOT, "tests", "cpp", "mock_abi_hessian_ops.cpp"), "-pthread"], check=True)
    drv = lb.driver(C.CDLL(so))
    for suf, dt in (("f64", np.float64), ("f32", np.float32)):
        err = C.create_string_buffer(256)
        X0, V, out = np.zeros(4, dt), np.zeros(4, dt), np.zeros(4, dt)
        items = (lb._SmallItem * 1)()
        r = getattr(drv, "lbfgsb200_drv_small_batch_hessian_times_" + suf)(
            0, 0, 4, 1, lb._ptr(X0), None, None, 0, 3, C.byref(lb.LBFGSParam()._c()), lb._ptr(V), 1, 1, lb._ptr(out), lb._ptr(out),
            lb._ptr(out), lb._ptr(out), items, err, len(err))
        assert r == -2 and "lbfgs_b200_small_minimize_keep_" in err.value.decode()


def test_front_members_compile(tmp_path):
    src = tmp_path / "tu.cpp"
    src.write_text("""
#include <LBFGSSmallBatch.h>
using namespace LBFGSpp;
template <class S> void use(LBFGSSmallBatchSolver<S, LineSearchMoreThuente>& s, DeviceVector<S>& V, DeviceVector<S>& O)
{
    s.keep_final_approx(true);
    s.final_approx_hessian_times(V, O);
    s.final_approx_inverse_hessian_times(V, O);
    s.final_approx_hessian_times(1L, V, O);
    s.final_approx_inverse_hessian_times(1L, V, O);
    SmallMatrix<S> B = s.final_approx_hessian(0), H = s.final_approx_inverse_hessian(0);
    (void)B; (void)H;
}
template void use<double>(LBFGSSmallBatchSolver<double, LineSearchMoreThuente>&, DeviceVector<double>&, DeviceVector<double>&);
template void use<float>(LBFGSSmallBatchSolver<float, LineSearchMoreThuente>&, DeviceVector<float>&, DeviceVector<float>&);
""")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o",
                    str(tmp_path / "tu.o")], check=True)


@pytest.fixture(scope="module")
def algebra(tmp_path_factory):
    d = tmp_path_factory.mktemp("compact")
    src = d / "compact.cpp"
    src.write_text("""
#include <vector>
#include <LBFGSpp/CompactForm.h>
using namespace LBFGSpp;
// B coefficients through Minv -> BK factor -> M by unit columns -> compact_b_coef, as BFGSMat does it
extern "C" void b_coef(int c, const double* SY, const double* SS, double theta, const double* wv, double* C)
{
    const int w = 2 * c;
    std::vector<double> F((size_t)(w * w)), M((size_t)(w * w)), z((size_t)w);
    std::vector<int> order((size_t)w);
    std::vector<unsigned char> tag((size_t)w);
    compact_minv(c, SY, SS, c, theta, F.data());
    bk_factor(F.data(), w, order.data(), tag.data());
    for (int j = 0; j < w; j++)
    {
        for (int i = 0; i < w; i++) M[size_t(i * w + j)] = i == j ? 1.0 : 0.0;
        bk_solve(F.data(), w, order.data(), tag.data(), M.data() + j, w, z.data());
    }
    compact_b_coef(c, M.data(), theta, wv, 1, C, 1);
}
extern "C" void h_coef(int c, const double* SY, const double* YY, double theta, const double* wv, double* C)
{
    std::vector<double> R((size_t)(c * c)), Y((size_t)(c * c)), w((size_t)c), us((size_t)c);
    compact_h_setup(c, SY, YY, c, R.data(), Y.data());
    compact_h_coef(c, R.data(), Y.data(), theta, wv, 1, w.data(), us.data(), 1, C, 1);
}
""")
    so = str(d / "compact.so")
    subprocess.run(CXX + ["-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-o", so, str(src)], check=True)
    return C.CDLL(so)


@pytest.mark.parametrize("c", [1, 2, 5, 10, 20])
def test_compact_algebra_matches_numpy(algebra, c):
    rng = np.random.default_rng(c)
    n = 3 * c + 4
    S = rng.standard_normal((c, n))
    Y = S + 0.3 * rng.standard_normal((c, n))   # s'y > 0 on the diagonal
    theta = float(Y[0] @ Y[0] / (S[0] @ Y[0]))
    v = rng.standard_normal(n)
    SY, SS, YY = S @ Y.T, S @ S.T, Y @ Y.T
    wv = np.concatenate([Y @ v, S @ v])
    dp = C.POINTER(C.c_double)
    ptr = lambda a: np.ascontiguousarray(a).ctypes.data_as(dp)  # noqa: E731
    Cb, Ch = np.zeros(2 * c), np.zeros(2 * c)
    algebra.b_coef(c, ptr(SY), ptr(SS), C.c_double(theta), ptr(wv), ptr(Cb))
    algebra.h_coef(c, ptr(SY), ptr(YY), C.c_double(theta), ptr(wv), ptr(Ch))
    # numpy: the same matrices from the pairs
    W = np.hstack([Y.T, theta * S.T])
    L = np.triu(SY, 1)
    Minv = np.block([[-np.diag(np.diag(SY)), L.T], [L, theta * SS]])
    Bv = theta * v - W @ np.linalg.solve(Minv, W.T @ v)
    Sc, Yc = S[::-1], Y[::-1]
    R = np.triu(Sc @ Yc.T)
    wr = np.linalg.solve(R, Sc @ v)
    us = np.linalg.solve(R.T, (np.diag(np.diag(R)) + Yc @ Yc.T / theta) @ wr - Yc @ v / theta)
    Hv = v / theta + Sc.T @ us - Yc.T @ wr / theta
    got_B = theta * v + Y.T @ Cb[:c] + S.T @ Cb[c:]
    got_H = v / theta + Y.T @ Ch[:c] + S.T @ Ch[c:]
    cond = np.linalg.cond(Minv)
    assert np.max(np.abs(got_B - Bv)) <= 1e-12 * cond * np.max(np.abs(Bv))
    assert np.max(np.abs(got_H - Hv)) <= 1e-12 * np.linalg.cond(R) ** 2 * np.max(np.abs(Hv))
