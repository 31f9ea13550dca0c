// hessian_ops_errors.cpp -- the error paths of the operator form of the final approximation (LBFGSSolver /
// LBFGSBatchSolver::final_approx_*_times and the two k-vector entry points of the C ABI).  Prints one line per case:
// "<case>: <exception type>: <message>" or "<case>: <status>: <last error>".  Linked against tests/cpp/mock_abi_hessian_ops.cpp (CPU) or
// liblbfgs_b200.so (GPU); with the argument "resident" it also covers the device-resident solve and the batch solver.
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>

#include "../../include/LBFGS.h"
#include "../../include/LBFGSBatch.h"
#include "../../include/LBFGSpp/DeviceObjectives.h"

using namespace LBFGSpp;
typedef DeviceVector<double> Vector;

template <class F> void report(const char* what, F f)
{
    try { f(); std::printf("%s: ok\n", what); }
    catch (const std::invalid_argument& e) { std::printf("%s: invalid_argument: %s\n", what, e.what()); }
    catch (const std::logic_error& e) { std::printf("%s: logic_error: %s\n", what, e.what()); }
    catch (const std::exception& e) { std::printf("%s: other: %s\n", what, e.what()); }
}

int main(int argc, char** argv)
{
    const bool resident = argc > 1 && std::strcmp(argv[1], "resident") == 0;
    Device& dev = Device::get_default();
    LBFGSParam<double> prm;
    const long n = 8;
    Vector V(dev, 2 * n), OUT(dev);
    V.setZero();
    {
        LBFGSSolver<double, LineSearchMoreThuente> solver(prm);
        report("before minimize, B", [&]() { solver.final_approx_hessian_times(V, OUT); });
        report("before minimize, H", [&]() { solver.final_approx_inverse_hessian_times(V, OUT); });
        solver.set_device_resident(resident);
        BuiltinObjective<double> obj(LBFGS_B200_OBJ_ROSENBROCK_PAIRED);
        Vector x(dev, n);
        x.setZero();
        double fx = 0;
        solver.minimize(obj, x, fx);
        Vector bad(dev, n + 3), empty(dev);
        bad.setZero();
        report("size mismatch, B", [&]() { solver.final_approx_hessian_times(bad, OUT); });
        report("size mismatch, H", [&]() { solver.final_approx_inverse_hessian_times(bad, OUT); });
        report("empty V", [&]() { solver.final_approx_hessian_times(empty, OUT); });
        report("two vectors", [&]() { solver.final_approx_hessian_times(V, OUT); });
        // the ABI on a ring of this size: k outside 1..16, a leading dimension below n, NULL pointers
        lbfgs_b200_hist* h = nullptr;
        dev.check(lbfgs_b200_hist_create(dev.ctx(), &h, n, 4, 8));
        double R[2 * 4 * 17] = {0}, C[2 * 4 * 17] = {0};
        auto abi = [&](const char* what, lbfgs_b200_status st) {
            std::printf("%s: %s: %s\n", what, st == LBFGS_B200_ERR_INVALID ? "ERR_INVALID" : st == LBFGS_B200_OK ? "OK" : "other",
                        st == LBFGS_B200_OK ? "" : lbfgs_b200_last_error(dev.ctx()));
        };
        abi("wt_dot_multi k=0", lbfgs_b200_hist_wt_dot_multi_f64(h, 0, V.data(), n, R));
        abi("wt_dot_multi k=17", lbfgs_b200_hist_wt_dot_multi_f64(h, 17, V.data(), n, R));
        abi("wt_dot_multi ldv<n", lbfgs_b200_hist_wt_dot_multi_f64(h, 1, V.data(), n - 1, R));
        abi("wt_dot_multi NULL", lbfgs_b200_hist_wt_dot_multi_f64(h, 1, nullptr, n, R));
        abi("lincomb_multi k=0", lbfgs_b200_hist_lincomb_multi_f64(h, 1.0, 0, V.data(), n, C, OUT.data(), n));
        abi("lincomb_multi k=17", lbfgs_b200_hist_lincomb_multi_f64(h, 1.0, 17, V.data(), n, C, OUT.data(), n));
        abi("lincomb_multi ldo<n", lbfgs_b200_hist_lincomb_multi_f64(h, 1.0, 1, V.data(), n, C, OUT.data(), n - 1));
        abi("lincomb_multi NULL", lbfgs_b200_hist_lincomb_multi_f64(h, 1.0, 1, V.data(), n, C, nullptr, n));
        lbfgs_b200_hist_destroy(h);
    }
    if (resident)
    {
        LBFGSBatchSolver<double, LineSearchMoreThuente> batch(prm);
        report("batch before minimize", [&]() { batch.final_approx_hessian_times(0, V, OUT); });
        BuiltinObjective<double> obj(LBFGS_B200_OBJ_ROSENBROCK_PAIRED);
        Vector X(dev, 2 * n);
        X.setZero();
        batch.minimize(obj, X, 2);
        report("batch problem 2 of 2", [&]() { batch.final_approx_hessian_times(2, V, OUT); });
        Vector bad(dev, n + 3);
        bad.setZero();
        report("batch size mismatch", [&]() { batch.final_approx_inverse_hessian_times(1, bad, OUT); });
        report("batch two vectors", [&]() { batch.final_approx_inverse_hessian_times(1, V, OUT); });
    }
    std::printf("hessian ops errors done\n");
    return 0;
}
