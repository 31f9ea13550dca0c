// driver_owlqn.cpp -- host-buffer entry point of the L1-regularised solve (include/OWLQN.h) in liblbfgs_b200_driver.so: the caller
// hands over x0 (and the objective's data) in host memory, the entry uploads them, runs OWLQNSolver<Scalar>::minimize() on the GPU and
// downloads x and grad f(x).  A unit of its own, which refers to the OWL-QN entries of the C ABI weakly: the driver library still loads
// against a library (or test double) that exports the C ABI without them, and this entry point then names the missing one.
#include <chrono>
#include <cstring>
#include <stdexcept>
#include <string>

#include "../../include/OWLQN.h"
#include "../../include/LBFGSpp/DeviceObjectives.h"
#include "driver_common.h"

#pragma weak lbfgs_b200_owlqn_trial_f64
#pragma weak lbfgs_b200_owlqn_trial_f32
#pragma weak lbfgs_b200_owlqn_project_f64
#pragma weak lbfgs_b200_owlqn_project_f32
#pragma weak lbfgs_b200_owlqn_sums_f64
#pragma weak lbfgs_b200_owlqn_sums_f32
#pragma weak lbfgs_b200_owlqn_update_dir_f64
#pragma weak lbfgs_b200_owlqn_update_dir_f32
#pragma weak lbfgs_b200_owlqn_weighted_trial_f64
#pragma weak lbfgs_b200_owlqn_weighted_trial_f32
#pragma weak lbfgs_b200_owlqn_weighted_project_f64
#pragma weak lbfgs_b200_owlqn_weighted_project_f32
#pragma weak lbfgs_b200_owlqn_weighted_sums_f64
#pragma weak lbfgs_b200_owlqn_weighted_sums_f32
#pragma weak lbfgs_b200_owlqn_weighted_update_dir_f64
#pragma weak lbfgs_b200_owlqn_weighted_update_dir_f32

using namespace LBFGSpp;
using namespace lbfgsb200_drv;

#pragma GCC visibility push(default)
extern "C" {

typedef struct
{
    int status;   // 0 ok, 1 invalid_argument, 2 logic_error, 3 runtime_error, 4 other
    char msg[200];
    int niter;
    long nfev;
    double fx;    // F(x) = f(x) + lambda |x|_1 (weighted: f(x) + lambda sum_i w_i |x_i|)
    double gnorm; // ||pg||_2 at x
    double seconds;  // minimize() alone, operands already in HBM (host wall clock around a synchronised call)
} drv_owlqn_result;

}  // extern "C"

namespace {

// std::runtime_error naming the first OWL-QN entry the library in use lacks (the weighted ones too when the solve is weighted)
template <class Scalar> void require_entries(bool weighted)
{
    const bool d = sizeof(Scalar) == 8;
    const char* names[8] = {"lbfgs_b200_owlqn_trial", "lbfgs_b200_owlqn_project", "lbfgs_b200_owlqn_sums", "lbfgs_b200_owlqn_update_dir",
                            "lbfgs_b200_owlqn_weighted_trial", "lbfgs_b200_owlqn_weighted_project", "lbfgs_b200_owlqn_weighted_sums",
                            "lbfgs_b200_owlqn_weighted_update_dir"};
    const bool have[8] = {d ? bool(lbfgs_b200_owlqn_trial_f64) : bool(lbfgs_b200_owlqn_trial_f32),
                          d ? bool(lbfgs_b200_owlqn_project_f64) : bool(lbfgs_b200_owlqn_project_f32),
                          d ? bool(lbfgs_b200_owlqn_sums_f64) : bool(lbfgs_b200_owlqn_sums_f32),
                          d ? bool(lbfgs_b200_owlqn_update_dir_f64) : bool(lbfgs_b200_owlqn_update_dir_f32),
                          d ? bool(lbfgs_b200_owlqn_weighted_trial_f64) : bool(lbfgs_b200_owlqn_weighted_trial_f32),
                          d ? bool(lbfgs_b200_owlqn_weighted_project_f64) : bool(lbfgs_b200_owlqn_weighted_project_f32),
                          d ? bool(lbfgs_b200_owlqn_weighted_sums_f64) : bool(lbfgs_b200_owlqn_weighted_sums_f32),
                          d ? bool(lbfgs_b200_owlqn_weighted_update_dir_f64) : bool(lbfgs_b200_owlqn_weighted_update_dir_f32)};
    for (int k = 0; k < (weighted ? 8 : 4); k++)
        if (!have[k]) throw std::runtime_error(std::string("the C ABI in use lacks ") + names[k] + (d ? "_f64" : "_f32"));
}

template <class Scalar>
int owlqn_any(int dev_ordinal, int objective, const Scalar* data0_host, const Scalar* data1_host, long n, const drv_param* q, double lam,
              const Scalar* w_host, int fused, Scalar* x_host, Scalar* grad_host, drv_owlqn_result* out)
{
    std::memset(out, 0, sizeof(*out));
    auto fail = [&](int code, const char* what) {
        out->status = code;
        std::strncpy(out->msg, what, sizeof(out->msg) - 1);
        out->msg[sizeof(out->msg) - 1] = 0;
    };
    try
    {
        const LBFGSParam<Scalar> prm = to_param<Scalar>(q);
        OWLQNSolver<Scalar> plain_solver(prm, Scalar(lam));   // checks param and lambda before any device work
        require_entries<Scalar>(w_host != nullptr);
        Device& dev = device(dev_ordinal);
        DeviceVector<Scalar> d0(dev), d1(dev), x(dev), w(dev);
        if (data0_host) d0.copy_from_host(data0_host, n);
        if (data1_host) d1.copy_from_host(data1_host, n);
        if (w_host) w.copy_from_host(w_host, n);
        x.copy_from_host(x_host, n);
        OWLQNSolver<Scalar> weighted_solver(prm, Scalar(lam), w);
        OWLQNSolver<Scalar>& solver = w_host ? weighted_solver : plain_solver;
        Scalar fx = Scalar(0);
        dev.synchronize();
        const auto t0 = std::chrono::steady_clock::now();
        try
        {
            if (fused)
            {
                BuiltinObjective<Scalar> obj(objective, d0.data(), d1.data());
                out->niter = solver.minimize(obj, x, fx);
            }
            else
            {
                PlainObjective<Scalar> obj(objective, d0.data(), d1.data());
                out->niter = solver.minimize(obj, x, fx);
            }
        }
        catch (...)
        {
            out->nfev = solver.num_evaluations();
            throw;
        }
        dev.synchronize();
        out->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        out->nfev = solver.num_evaluations();
        out->fx = double(fx);
        out->gnorm = double(solver.final_grad_norm());
        x.copy_to_host(x_host);
        if (grad_host) solver.final_grad().copy_to_host(grad_host);
    }
    catch (const std::invalid_argument& e) { fail(1, e.what()); }
    catch (const std::logic_error& e) { fail(2, e.what()); }
    catch (const std::runtime_error& e) { fail(3, e.what()); }
    catch (const std::exception& e) { fail(4, e.what()); }
    return out->status;
}

}  // namespace

extern "C" {

// OWLQNSolver<Scalar>(param, lam).minimize(f, x, fx) on device `dev`, or with w_host != NULL (n weights)
// OWLQNSolver<Scalar>(param, lam, w).minimize(f, x, fx), F = f + lam sum_i w_i |x_i|; fused != 0: the built-in objective with its fused projected trial,
// fused = 0: the same objective as a plain device functor (the unfused route).  x_host: start point in, solution out; grad_host
// (optional): grad f at the solution.  Returns out->status.
int lbfgsb200_drv_owlqn_f64(int dev, int objective, const double* data0, const double* data1, long n, const drv_param* q, double lam,
                            const double* w_host, int fused, double* x_host, double* grad_host, drv_owlqn_result* out)
{
    return owlqn_any<double>(dev, objective, data0, data1, n, q, lam, w_host, fused, x_host, grad_host, out);
}
int lbfgsb200_drv_owlqn_f32(int dev, int objective, const float* data0, const float* data1, long n, const drv_param* q, double lam,
                            const float* w_host, int fused, float* x_host, float* grad_host, drv_owlqn_result* out)
{
    return owlqn_any<float>(dev, objective, data0, data1, n, q, lam, w_host, fused, x_host, grad_host, out);
}

}  // extern "C"
