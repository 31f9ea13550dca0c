// hessian_whiten_errors.cpp -- the error paths of whitening and log densities under N(x*, H) (LBFGSSolver / LBFGSBatchSolver::
// final_approx_inverse_hessian_factor_transpose_times / _solve / _transpose_solve / final_approx_log_density and the two whitening
// passes of the C ABI).  Prints one line per case: "<case>: <exception type>" or "<case>: <status>".  Linked against
// tests/cpp/mock_abi_hessian_whiten.cpp.
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "../../include/LBFGS.h"
#include "../../include/LBFGSBatch.h"
#include "../../include/LBFGSpp/DeviceObjectives.h"

using namespace LBFGSpp;
typedef DeviceVector<double> Vector;

template <class F> void report(const char* what, F f)
{
    try { f(); std::printf("%s: ok\n", what); }
    catch (const std::invalid_argument&) { std::printf("%s: invalid_argument\n", what); }
    catch (const std::logic_error&) { std::printf("%s: logic_error\n", what); }
    catch (const std::runtime_error&) { std::printf("%s: runtime_error\n", what); }
    catch (const std::exception&) { std::printf("%s: other\n", what); }
}

int main()
{
    Device& dev = Device::get_default();
    LBFGSParam<double> prm;
    const long n = 8;
    Vector V(dev, n), X(dev, 2 * n), mean(dev, n), OUT(dev), odd(dev, n + 1), shortmean(dev, n - 1);
    V.setZero();
    X.setZero();
    mean.setZero();
    odd.setZero();
    shortmean.setZero();
    {
        LBFGSSolver<double, LineSearchMoreThuente> solver(prm);
        report("solver before minimize, LT", [&]() { solver.final_approx_inverse_hessian_factor_transpose_times(V, OUT); });
        report("solver before minimize, LINV", [&]() { solver.final_approx_inverse_hessian_factor_solve(V, OUT); });
        report("solver before minimize, LINVT", [&]() { solver.final_approx_inverse_hessian_factor_transpose_solve(V, OUT); });
        report("solver before minimize, log density", [&]() { solver.final_approx_log_density(mean, X); });
        solver.set_device_resident(false);
        BuiltinObjective<double> obj(LBFGS_B200_OBJ_ROSENBROCK_PAIRED);
        Vector x(dev, n);
        x.setZero();
        double fx = 0;
        solver.minimize(obj, x, fx);
        report("solver after minimize, LT", [&]() { solver.final_approx_inverse_hessian_factor_transpose_times(V, OUT); });
        report("solver after minimize, log density", [&]() { solver.final_approx_log_density(x, X); });
        report("solver, V of n + 1", [&]() { solver.final_approx_inverse_hessian_factor_solve(odd, OUT); });
        report("solver, X of n + 1", [&]() { solver.final_approx_log_density(x, odd); });
        report("solver, mean of n - 1", [&]() { solver.final_approx_log_density(shortmean, X); });
    }
    {
        LBFGSBatchSolver<double, LineSearchMoreThuente> batch(prm);
        report("batch before minimize, LT", [&]() { batch.final_approx_inverse_hessian_factor_transpose_times(0, V, OUT); });
        report("batch before minimize, LINV", [&]() { batch.final_approx_inverse_hessian_factor_solve(0, V, OUT); });
        report("batch before minimize, LINVT", [&]() { batch.final_approx_inverse_hessian_factor_transpose_solve(0, V, OUT); });
        report("batch before minimize, log density", [&]() { batch.final_approx_log_density(0, mean, X); });
    }
    {
        // the two passes on a ring with one pair: k out of 1..16, a leading dimension below n, NULL arguments
        lbfgs_b200_hist* h = nullptr;
        dev.check(lbfgs_b200_hist_create(dev.ctx(), &h, n, 4, 8));
        Vector s(dev), y(dev);
        const std::vector<double> ones(size_t(n), 1.0), twos(size_t(n), 2.0);
        s.copy_from_host(ones.data(), n);
        y.copy_from_host(twos.data(), n);
        dev.check(lbfgs_b200_hist_add_f64(h, s.data(), y.data()));
        std::vector<double> R(2 * 17), nrm(17);
        auto abi = [&](const char* what, lbfgs_b200_status st) {
            std::printf("%s: %s\n", what, st == LBFGS_B200_ERR_INVALID ? "ERR_INVALID" : st == LBFGS_B200_OK ? "OK" : "other");
        };
        abi("s_dot_multi, k = 1", lbfgs_b200_hist_s_dot_multi_f64(h, 1, V.data(), n, R.data()));
        abi("s_dot_multi, k = 0", lbfgs_b200_hist_s_dot_multi_f64(h, 0, V.data(), n, R.data()));
        abi("s_dot_multi, k = 17", lbfgs_b200_hist_s_dot_multi_f64(h, 17, V.data(), n, R.data()));
        abi("s_dot_multi, ldv < n", lbfgs_b200_hist_s_dot_multi_f64(h, 1, V.data(), n - 1, R.data()));
        abi("s_dot_multi, NULL R", lbfgs_b200_hist_s_dot_multi_f64(h, 1, V.data(), n, nullptr));
        abi("wt_dot_diff, k = 1", lbfgs_b200_hist_wt_dot_diff_f64(h, 1, X.data(), n, mean.data(), R.data(), nrm.data()));
        abi("wt_dot_diff, k = 0", lbfgs_b200_hist_wt_dot_diff_f64(h, 0, X.data(), n, mean.data(), R.data(), nrm.data()));
        abi("wt_dot_diff, k = 17", lbfgs_b200_hist_wt_dot_diff_f64(h, 17, X.data(), n, mean.data(), R.data(), nrm.data()));
        abi("wt_dot_diff, ldx < n", lbfgs_b200_hist_wt_dot_diff_f64(h, 1, X.data(), n - 1, mean.data(), R.data(), nrm.data()));
        abi("wt_dot_diff, NULL mean", lbfgs_b200_hist_wt_dot_diff_f64(h, 1, X.data(), n, nullptr, R.data(), nrm.data()));
        abi("wt_dot_diff, NULL norms", lbfgs_b200_hist_wt_dot_diff_f64(h, 1, X.data(), n, mean.data(), R.data(), nullptr));
        lbfgs_b200_hist_destroy(h);
    }
    std::printf("hessian whiten errors done\n");
    return 0;
}
