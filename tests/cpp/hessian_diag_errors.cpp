// hessian_diag_errors.cpp -- the error paths of the diagonals of the final approximation (LBFGSSolver / LBFGSBatchSolver /
// LBFGSSmallBatchSolver::final_approx_*_diagonal and the two diagonal entry points of the C ABI).  Prints one line per case:
// "<case>: <exception type>: <message>" or "<case>: <status>: <last error>".  Linked against tests/cpp/mock_abi_hessian_diag.cpp (CPU)
// or liblbfgs_b200.so (GPU); with the argument "gpu" it also covers the batch solver, the small-batch solver and its entry point.
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/LBFGS.h"
#include "../../include/LBFGSBatch.h"
#include "../../include/LBFGSSmallBatch.h"
#include "../../include/LBFGSpp/DeviceObjectives.h"

// the small-batch part of the C ABI, which the test double lacks: only called with "gpu"
#pragma weak lbfgs_b200_small_minimize_f64
#pragma weak lbfgs_b200_small_minimize_keep_f64
#pragma weak lbfgs_b200_small_hist_create
#pragma weak lbfgs_b200_small_hist_destroy
#pragma weak lbfgs_b200_small_hist_diag_f64
#pragma weak lbfgs_b200_small_hist_diag_f32

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
    const bool gpu = argc > 1 && std::strcmp(argv[1], "gpu") == 0;
    Device& dev = Device::get_default();
    LBFGSParam<double> prm;
    const long n = 8;
    Vector OUT(dev);
    auto abi = [&](const char* what, lbfgs_b200_status st) {
        std::printf("%s: %s: %s\n", what, st == LBFGS_B200_ERR_INVALID ? "ERR_INVALID" : st == LBFGS_B200_OK ? "OK" : "other",
                    st == LBFGS_B200_OK ? "" : lbfgs_b200_last_error(dev.ctx()));
    };
    {
        LBFGSSolver<double, LineSearchMoreThuente> solver(prm);
        report("before minimize, B", [&]() { solver.final_approx_hessian_diagonal(OUT); });
        report("before minimize, H", [&]() { solver.final_approx_inverse_hessian_diagonal(OUT); });
        solver.set_device_resident(gpu);
        BuiltinObjective<double> obj(LBFGS_B200_OBJ_ROSENBROCK_PAIRED);
        Vector x(dev, n);
        x.setZero();
        double fx = 0;
        solver.minimize(obj, x, fx);
        report("after minimize, B", [&]() { solver.final_approx_hessian_diagonal(OUT); });
        report("after minimize, H", [&]() { solver.final_approx_inverse_hessian_diagonal(OUT); });
        // the ABI on a ring with one pair: NULL out, NULL K
        lbfgs_b200_hist* h = nullptr;
        dev.check(lbfgs_b200_hist_create(dev.ctx(), &h, n, 4, 8));
        Vector s(dev), y(dev);
        const std::vector<double> ones(size_t(n), 1.0), twos(size_t(n), 2.0);
        s.copy_from_host(ones.data(), n);
        y.copy_from_host(twos.data(), n);
        dev.check(lbfgs_b200_hist_add_f64(h, s.data(), y.data()));
        double K[4] = {1, 0, 0, 1};
        OUT.resize(n);
        abi("quad_diag NULL out", lbfgs_b200_hist_quad_diag_f64(h, 1.0, K, nullptr));
        abi("quad_diag NULL K", lbfgs_b200_hist_quad_diag_f64(h, 1.0, nullptr, OUT.data()));
        abi("quad_diag ok", lbfgs_b200_hist_quad_diag_f64(h, 1.0, K, OUT.data()));
        lbfgs_b200_hist_destroy(h);
    }
    if (gpu)
    {
        LBFGSBatchSolver<double, LineSearchMoreThuente> batch(prm);
        report("batch before minimize", [&]() { batch.final_approx_hessian_diagonal(0, OUT); });
        BuiltinObjective<double> obj(LBFGS_B200_OBJ_ROSENBROCK_PAIRED);
        Vector X(dev, 2 * n);
        X.setZero();
        batch.minimize(obj, X, 2);
        report("batch problem 2 of 2", [&]() { batch.final_approx_hessian_diagonal(2, OUT); });
        report("batch problem -1", [&]() { batch.final_approx_inverse_hessian_diagonal(-1, OUT); });
        report("batch problem 1", [&]() { batch.final_approx_inverse_hessian_diagonal(1, OUT); });

        LBFGSSmallBatchSolver<double, LineSearchMoreThuente> small(prm);
        report("small before minimize", [&]() { small.final_approx_hessian_diagonal(OUT); });
        Vector XS(dev, 3 * n);
        XS.setZero();
        small.minimize(obj, XS, 3);
        report("small not kept", [&]() { small.final_approx_inverse_hessian_diagonal(0L, OUT); });
        small.keep_final_approx(true);
        XS.setZero();
        small.minimize(obj, XS, 3);
        report("small problem 3 of 3", [&]() { small.final_approx_hessian_diagonal(3L, OUT); });
        report("small problem 2", [&]() { small.final_approx_hessian_diagonal(2L, OUT); });
        report("small all", [&]() { small.final_approx_inverse_hessian_diagonal(OUT); });

        lbfgs_b200_small_hist* sh = nullptr;
        dev.check(lbfgs_b200_small_hist_create(dev.ctx(), n, 4, 8, 3, &sh));
        OUT.resize(3 * n);
        abi("small_hist_diag unfilled", lbfgs_b200_small_hist_diag_f64(sh, 0, 0, 1, OUT.data(), n));
        lbfgs_b200_param p{};
        p.m = 4; p.epsilon = 1e-5; p.epsilon_rel = 1e-5; p.past = 0; p.delta = 0; p.max_iterations = 0; p.max_linesearch = 20;
        p.min_step = 1e-20; p.max_step = 1e20; p.ftol = 1e-4; p.wolfe = 0.9; p.linesearch = 1;
        lbfgs_b200_outcome outs[3];
        XS.setZero();
        dev.check(lbfgs_b200_small_minimize_keep_f64(dev.ctx(), LBFGS_B200_OBJ_ROSENBROCK_PAIRED, nullptr, nullptr, 0, n, 3, &p,
                                                     LBFGS_B200_LS_MORE_THUENTE, XS.data(), n, nullptr, outs, sh));
        abi("small_hist_diag range", lbfgs_b200_small_hist_diag_f64(sh, 0, 2, 2, OUT.data(), n));
        abi("small_hist_diag b0<0", lbfgs_b200_small_hist_diag_f64(sh, 0, -1, 1, OUT.data(), n));
        abi("small_hist_diag count=0", lbfgs_b200_small_hist_diag_f64(sh, 1, 0, 0, OUT.data(), n));
        abi("small_hist_diag NULL", lbfgs_b200_small_hist_diag_f64(sh, 0, 0, 3, nullptr, n));
        abi("small_hist_diag ldo<n", lbfgs_b200_small_hist_diag_f64(sh, 1, 0, 3, OUT.data(), n - 1));
        abi("small_hist_diag fp32", lbfgs_b200_small_hist_diag_f32(sh, 1, 0, 3, reinterpret_cast<float*>(OUT.data()), n));
        abi("small_hist_diag ok", lbfgs_b200_small_hist_diag_f64(sh, 1, 0, 3, OUT.data(), n));
        dev.check(lbfgs_b200_sync(dev.ctx()));
        lbfgs_b200_small_hist_destroy(sh);
    }
    std::printf("hessian diag errors done\n");
    return 0;
}
