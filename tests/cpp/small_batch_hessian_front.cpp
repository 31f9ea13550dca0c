// small_batch_hessian_front.cpp -- the kept final approximations of LBFGSSmallBatchSolver through the C++ front and the C ABI: every
// refused call with its exception or status, and the dense matrices of final_approx_hessian(b) / final_approx_inverse_hessian(b).
// Prints one line per case: "<case>: <exception type>: <message>", "<case>: <status>: <last error>" or "<case>: <value>".
// Linked against liblbfgs_b200.so (GPU).
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "../../include/LBFGSSmallBatch.h"

using namespace LBFGSpp;
typedef DeviceVector<double> Vector;

template <class F> void report(const char* what, F f)
{
    try { f(); std::printf("%s: ok\n", what); }
    catch (const std::invalid_argument& e) { std::printf("%s: invalid_argument: %s\n", what, e.what()); }
    catch (const std::logic_error& e) { std::printf("%s: logic_error: %s\n", what, e.what()); }
    catch (const std::exception& e) { std::printf("%s: other: %s\n", what, e.what()); }
}

// largest |A - A'| / max |A|, and largest |B H - I|
static double asym(const SmallMatrix<double>& A)
{
    double d = 0, s = 0;
    for (int i = 0; i < A.rows(); i++)
        for (int j = 0; j < A.cols(); j++) { d = std::fmax(d, std::fabs(A(i, j) - A(j, i))); s = std::fmax(s, std::fabs(A(i, j))); }
    return d / s;
}
static double inv_err(const SmallMatrix<double>& B, const SmallMatrix<double>& H)
{
    double e = 0;
    const int n = B.rows();
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++)
        {
            double acc = 0;
            for (int q = 0; q < n; q++) acc += B(i, q) * H(q, j);
            e = std::fmax(e, std::fabs(acc - (i == j ? 1.0 : 0.0)));
        }
    return e;
}

int main()
{
    Device& dev = Device::get_default();
    LBFGSParam<double> prm;
    prm.m = 4;
    prm.max_iterations = 30;
    const long n = 8, B = 3;
    BuiltinObjective<double> obj(LBFGS_B200_OBJ_ROSENBROCK_PAIRED);
    Vector V(dev, B * 2 * n), OUT(dev), one(dev, 2 * n);
    V.setZero();
    one.setZero();
    LBFGSSmallBatchSolver<double, LineSearchMoreThuente> solver(prm);
    report("before minimize, all", [&]() { solver.final_approx_hessian_times(V, OUT); });
    report("before minimize, one", [&]() { solver.final_approx_inverse_hessian_times(0, one, OUT); });
    report("before minimize, dense", [&]() { solver.final_approx_hessian(0); });
    Vector X(dev, B * n);
    std::vector<double> x0(size_t(B * n), 0.0);
    for (long i = 0; i < n; i++) x0[size_t(2 * n + i)] = 1.0;   // problem 2 starts at the minimiser: no pair
    X.copy_from_host(x0.data(), B * n);
    solver.minimize(obj, X, B);
    report("not kept", [&]() { solver.final_approx_hessian_times(V, OUT); });
    solver.keep_final_approx(true);
    X.copy_from_host(x0.data(), B * n);
    solver.minimize(obj, X, B);
    Vector bad(dev, n + 3), empty(dev);
    bad.setZero();
    report("kept, all", [&]() { solver.final_approx_hessian_times(V, OUT); });
    report("all, not whole", [&]() { solver.final_approx_hessian_times(bad, OUT); });
    report("all, empty", [&]() { solver.final_approx_inverse_hessian_times(empty, OUT); });
    report("one, b = -1", [&]() { solver.final_approx_hessian_times(-1, one, OUT); });
    report("one, b = B", [&]() { solver.final_approx_inverse_hessian_times(B, one, OUT); });
    report("one, not whole", [&]() { solver.final_approx_hessian_times(0, bad, OUT); });
    report("dense, b = B", [&]() { solver.final_approx_inverse_hessian(B); });
    report("kept, one", [&]() { solver.final_approx_inverse_hessian_times(1, one, OUT); });
    for (long b = 0; b < B; b++)
    {
        const SmallMatrix<double> Bd = solver.final_approx_hessian(b), Hd = solver.final_approx_inverse_hessian(b);
        std::printf("dense %ld asym B: %.3e\n", b, asym(Bd));
        std::printf("dense %ld asym H: %.3e\n", b, asym(Hd));
        std::printf("dense %ld BH - I: %.3e\n", b, inv_err(Bd, Hd));
        if (b == 2)   // no pair: exactly theta I and I / theta, theta = 1
        {
            bool exact = true;
            for (int i = 0; i < n; i++)
                for (int j = 0; j < n; j++) exact = exact && Bd(i, j) == (i == j ? 1.0 : 0.0) && Hd(i, j) == (i == j ? 1.0 : 0.0);
            std::printf("dense 2 exact: %d\n", int(exact));
        }
    }

    // the C ABI
    auto abi = [&](const char* what, lbfgs_b200_status st) {
        std::printf("%s: %s: %s\n", what, st == LBFGS_B200_ERR_INVALID ? "ERR_INVALID" : st == LBFGS_B200_OK ? "OK" : "other",
                    st == LBFGS_B200_OK ? "" : lbfgs_b200_last_error(dev.ctx()));
    };
    lbfgs_b200_small_hist* h = nullptr;
    dev.check(lbfgs_b200_small_hist_create(dev.ctx(), n, 4, 8, B, &h));
    abi("times before a solve", lbfgs_b200_small_hist_times_f64(h, 0, 0, B, 1, V.data(), n, n, OUT.data(), n, n));
    const lbfgs_b200_param p = detail::abi_param(prm);
    std::vector<lbfgs_b200_outcome> outs(size_t(B + 1));
    Vector X4(dev, (B + 1) * n), Vn(dev, 40 * n), O2(dev, 40 * n);
    X4.setZero();
    Vn.setZero();
    lbfgs_b200_param p5 = p;
    p5.m = 5;
    abi("keep, B differs", lbfgs_b200_small_minimize_keep_f64(dev.ctx(), 0, nullptr, nullptr, 0, n, B + 1, &p, 3, X4.data(), n, nullptr, outs.data(), h));
    abi("keep, n differs", lbfgs_b200_small_minimize_keep_f64(dev.ctx(), 0, nullptr, nullptr, 0, n + 2, B, &p, 3, X4.data(), n + 2, nullptr, outs.data(), h));
    abi("keep, m differs", lbfgs_b200_small_minimize_keep_f64(dev.ctx(), 0, nullptr, nullptr, 0, n, B, &p5, 3, X4.data(), n, nullptr, outs.data(), h));
    abi("keep, precision differs", lbfgs_b200_small_minimize_keep_f32(dev.ctx(), 0, nullptr, nullptr, 0, n, B, &p, 3, reinterpret_cast<float*>(X4.data()),
                                                                      n, nullptr, outs.data(), h));
    abi("keep, NULL history", lbfgs_b200_small_minimize_keep_f64(dev.ctx(), 0, nullptr, nullptr, 0, n, B, &p, 3, X4.data(), n, nullptr, outs.data(), nullptr));
    abi("keep", lbfgs_b200_small_minimize_keep_f64(dev.ctx(), 0, nullptr, nullptr, 0, n, B, &p, 3, X4.data(), n, nullptr, outs.data(), h));
    abi("times k=0", lbfgs_b200_small_hist_times_f64(h, 0, 0, B, 0, Vn.data(), n, 0, O2.data(), n, n));
    abi("times ldv<n", lbfgs_b200_small_hist_times_f64(h, 0, 0, 1, 1, Vn.data(), n - 1, 0, O2.data(), n, 0));
    abi("times ldo<n", lbfgs_b200_small_hist_times_f64(h, 1, 0, 1, 1, Vn.data(), n, 0, O2.data(), n - 1, 0));
    abi("times b0<0", lbfgs_b200_small_hist_times_f64(h, 0, -1, 1, 1, Vn.data(), n, 0, O2.data(), n, 0));
    abi("times past B", lbfgs_b200_small_hist_times_f64(h, 0, 1, B, 1, Vn.data(), n, 0, O2.data(), n, n));
    abi("times count=0", lbfgs_b200_small_hist_times_f64(h, 0, 0, 0, 1, Vn.data(), n, 0, O2.data(), n, n));
    abi("times NULL V", lbfgs_b200_small_hist_times_f64(h, 0, 0, 1, 1, nullptr, n, 0, O2.data(), n, 0));
    abi("times NULL OUT", lbfgs_b200_small_hist_times_f64(h, 0, 0, 1, 1, Vn.data(), n, 0, nullptr, n, 0));
    abi("times OUT=V other layout", lbfgs_b200_small_hist_times_f64(h, 0, 0, 1, 2, Vn.data(), n, 0, Vn.data(), n + 1, 0));
    abi("times OUT=V shared", lbfgs_b200_small_hist_times_f64(h, 0, 0, 2, 1, Vn.data(), n, 0, Vn.data(), n, 0));
    abi("times OUT=V same layout", lbfgs_b200_small_hist_times_f64(h, 0, 0, B, 2, Vn.data(), n, 2 * n, Vn.data(), n, 2 * n));
    abi("times wrong precision", lbfgs_b200_small_hist_times_f32(h, 0, 0, 1, 1, reinterpret_cast<float*>(Vn.data()), n, 0,
                                                                 reinterpret_cast<float*>(O2.data()), n, 0));
    abi("times", lbfgs_b200_small_hist_times_f64(h, 1, 0, B, 40, Vn.data(), n, 0, O2.data(), n, 40 * n));
    lbfgs_b200_small_hist* h2 = nullptr;
    abi("create m=0", lbfgs_b200_small_hist_create(dev.ctx(), n, 0, 8, B, &h2));
    abi("create B=0", lbfgs_b200_small_hist_create(dev.ctx(), n, 4, 8, 0, &h2));
    abi("create NULL out", lbfgs_b200_small_hist_create(dev.ctx(), n, 4, 8, B, nullptr));
    abi("sync", lbfgs_b200_sync(dev.ctx()));
    lbfgs_b200_small_hist_destroy(h);
    std::printf("small batch hessian front done\n");
    return 0;
}
