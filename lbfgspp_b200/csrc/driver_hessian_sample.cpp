// driver_hessian_sample.cpp -- host-buffer entry points of N(x*, H) from the final approximation (LBFGSSolver / LBFGSBatchSolver /
// LBFGSSmallBatchSolver::final_approx_inverse_hessian_factor_times / final_approx_sample / final_approx_inverse_hessian_logdet), built
// into lbfgspp_b200/liblbfgs_b200_driver.so next to driver.cpp.  A unit of its own, which refers to the sampler's passes of the C ABI
// (lbfgs_b200_hist_*_normal_*, lbfgs_b200_small_hist_factor_times_* / _sample_* / _logdet_*) weakly: the driver library still loads
// against a library (or test double) that exports the C ABI without them, and these entry points then report which one is missing.
#include "driver_small_batch.h"

#include <cstdio>

#pragma weak lbfgs_b200_hist_wt_dot_normal_f64
#pragma weak lbfgs_b200_hist_wt_dot_normal_f32
#pragma weak lbfgs_b200_hist_lincomb_normal_f64
#pragma weak lbfgs_b200_hist_lincomb_normal_f32
#pragma weak lbfgs_b200_small_hist_factor_times_f64
#pragma weak lbfgs_b200_small_hist_factor_times_f32
#pragma weak lbfgs_b200_small_hist_sample_f64
#pragma weak lbfgs_b200_small_hist_sample_f32
#pragma weak lbfgs_b200_small_hist_logdet_f64
#pragma weak lbfgs_b200_small_hist_logdet_f32

using namespace LBFGSpp;
using namespace lbfgsb200_drv;

#pragma GCC visibility push(default)

namespace {

void require_normal_passes()
{
    if (!lbfgs_b200_hist_wt_dot_normal_f64 || !lbfgs_b200_hist_lincomb_normal_f64)
        throw std::runtime_error("the C ABI library in use has no sampler passes (lbfgs_b200_hist_wt_dot_normal_*, lbfgs_b200_hist_lincomb_normal_*)");
}

// L V (kv vectors of V_host, into LV_out), kd draws first .. first+kd-1 around the solution (into draws_out) and log det H (into
// *logdet_out), each only when its output is given.  f(V, OUT) is the factor product, s(first, k, OUT) the sampler, l() the log-det.
template <class F, class S, class L>
void factor_outputs(Device& dev, long n, int kv, const double* V_host, double* LV_out, int kd, double* draws_out, double* logdet_out, F f, S s, L l)
{
    DeviceVector<double> out(dev);
    if (LV_out && kv > 0)
    {
        DeviceVector<double> V(dev);
        V.copy_from_host(V_host, std::ptrdiff_t(kv) * n);
        f(V, out);
        out.copy_to_host(LV_out);
    }
    if (draws_out && kd > 0)
    {
        s(kd, out);
        out.copy_to_host(draws_out);
    }
    if (logdet_out) *logdet_out = l();
}

}  // namespace

// minimize() on a built-in objective (resident = 1: the device-resident solve, 0: the host-driven loop), then L V, draws
// x* + L z_j (j = first .. first+kd-1, stream 0) and log det H of the final approximation.
extern "C" int lbfgsb200_drv_solve_hessian_sample_f64(int device_ordinal, int objective, long n, int ls, const drv_param* q, int resident,
                                                      double* x_host, int kv, const double* V_host, double* LV_out, unsigned long long seed,
                                                      unsigned first, int kd, double* draws_out, double* logdet_out, int* niter_out, char* err,
                                                      int errlen)
{
    return reported(err, errlen, 1, [&]() {
        require_normal_passes();
        Device& dev = device(device_ordinal);
        const LBFGSParam<double> prm = to_param<double>(q);
        BuiltinObjective<double> obj(objective);
        DeviceVector<double> x(dev);
        x.copy_from_host(x_host, n);
        double fx = 0;
        int niter = 0;
        with_line_search(ls, [&](auto tag) {
            typename decltype(tag)::template Solver<double> solver(prm);
            solver.set_device_resident(resident != 0);
            niter = solver.minimize(obj, x, fx);
            factor_outputs(dev, n, kv, V_host, LV_out, kd, draws_out, logdet_out,
                           [&](const DeviceVector<double>& V, DeviceVector<double>& O) { solver.final_approx_inverse_hessian_factor_times(V, O); },
                           [&](int k, DeviceVector<double>& O) { solver.final_approx_sample(x, seed, first, k, O); },
                           [&]() { return solver.final_approx_inverse_hessian_logdet(); });
        });
        x.copy_to_host(x_host);
        if (niter_out) *niter_out = niter;
        return 0;
    });
}

// The same for problem b of a batch of B problems (rows of x0s_host) minimised by LBFGSBatchSolver: its draws are from stream b.
// xs_out (optional) receives the solutions.
extern "C" int lbfgsb200_drv_batch_hessian_sample_f64(int device_ordinal, int objective, long n, int B, const double* x0s_host, int ls,
                                                      const drv_param* q, int b, int kv, const double* V_host, double* LV_out,
                                                      unsigned long long seed, unsigned first, int kd, double* draws_out, double* logdet_out,
                                                      double* xs_out, char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
        require_normal_passes();
        Device& dev = device(device_ordinal);
        const LBFGSParam<double> prm = to_param<double>(q);
        BuiltinObjective<double> obj(objective);
        DeviceVector<double> X(dev), xb(dev);
        X.copy_from_host(x0s_host, std::ptrdiff_t(n) * B);
        with_line_search(ls, [&](auto tag) {
            typename decltype(tag)::template BatchSolver<double> solver(prm);
            solver.minimize(obj, X, B);
            std::vector<double> xs(size_t(n) * size_t(B));
            X.copy_to_host(xs.data());
            if (xs_out) std::copy(xs.begin(), xs.end(), xs_out);
            if (b >= 0 && b < B) xb.copy_from_host(xs.data() + size_t(b) * size_t(n), n);
            factor_outputs(dev, n, kv, V_host, LV_out, kd, draws_out, logdet_out,
                           [&](const DeviceVector<double>& V, DeviceVector<double>& O) { solver.final_approx_inverse_hessian_factor_times(b, V, O); },
                           [&](int k, DeviceVector<double>& O) { solver.final_approx_sample(b, xb, seed, first, k, O); },
                           [&]() { return solver.final_approx_inverse_hessian_logdet(b); });
        });
        return 0;
    });
}

// The same for an explicit history: the pairs (S_host[k], Y_host[k]) added in order to a ring of size m (test hook for BFGSMat's
// inverse_hessian_factor_times / sample / inverse_hessian_logdet, stream `stream`, mean_host: n values or NULL)
extern "C" int lbfgsb200_drv_hist_sample_f64(int device_ordinal, long n, int m, int npairs, const double* S_host, const double* Y_host, int kv,
                                             const double* V_host, double* LV_out, const double* mean_host, unsigned long long seed,
                                             unsigned stream, unsigned first, int kd, double* draws_out, double* logdet_out, char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
        require_normal_passes();
        Device& dev = device(device_ordinal);
        BFGSMat<double> mat;
        mat.reset(dev, n, m);
        DeviceVector<double> s(dev), y(dev), mean(dev);
        for (int k = 0; k < npairs; k++)
        {
            s.copy_from_host(S_host + size_t(k) * n, n);
            y.copy_from_host(Y_host + size_t(k) * n, n);
            mat.add_correction(s, y);
        }
        if (mean_host) mean.copy_from_host(mean_host, n);
        factor_outputs(dev, n, kv, V_host, LV_out, kd, draws_out, logdet_out,
                       [&](const DeviceVector<double>& V, DeviceVector<double>& O) { mat.inverse_hessian_factor_times(V, kv, O); },
                       [&](int k, DeviceVector<double>& O) { mat.sample(mean_host ? &mean : nullptr, seed, stream, first, k, O); },
                       [&]() { return mat.inverse_hessian_logdet(); });
        return 0;
    });
}

namespace {

// small_batch with the final approximations kept, then for every problem: L_b V (V_host: B*kv vectors, problem b's at b*kv*n), kd
// draws X_b + L_b z_j around the solutions from stream b (B*kd vectors) and log det H_b (B values), one launch each
template <class Scalar>
int small_batch_hessian_sample(int device_ordinal, int objective, long n, long B, const Scalar* x0s_host, const Scalar* data0_host,
                               const Scalar* data1_host, long ldd, int ls, const drv_param* q, Scalar* xs_out, int kv, const Scalar* V_host,
                               Scalar* LV_out, unsigned long long seed, unsigned first, int kd, Scalar* draws_out, double* logdet_out,
                               drv_small_item* items, char* err, int errlen)
{
    if (!lbfgs_b200_small_hist_create || !lbfgs_b200_small_hist_destroy ||
        (sizeof(Scalar) == 8 ? !lbfgs_b200_small_minimize_keep_f64 || !lbfgs_b200_small_hist_sample_f64
                             : !lbfgs_b200_small_minimize_keep_f32 || !lbfgs_b200_small_hist_sample_f32))
    {
        std::snprintf(err, size_t(errlen), "the C ABI library in use has no small-batch sampler (lbfgs_b200_small_minimize_keep_*, "
                                           "lbfgs_b200_small_hist_sample_*)");
        return -2;
    }
    return small_batch<Scalar>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, nullptr, items, err, errlen,
                               true, [&](auto& solver, Device& dev, DeviceVector<Scalar>& X) {
        DeviceVector<Scalar> out(dev);
        if (LV_out && kv > 0)
        {
            DeviceVector<Scalar> V(dev);
            V.copy_from_host(V_host, std::ptrdiff_t(kv) * n * B);
            solver.final_approx_inverse_hessian_factor_times(V, out);
            out.copy_to_host(LV_out);
        }
        if (draws_out && kd > 0)
        {
            solver.final_approx_sample(X, seed, first, kd, out);   // around the solutions
            out.copy_to_host(draws_out);
        }
        if (logdet_out)
        {
            const std::vector<double> ld = solver.final_approx_inverse_hessian_logdet();
            std::copy(ld.begin(), ld.end(), logdet_out);
        }
    });
}

}  // namespace

extern "C" int lbfgsb200_drv_small_batch_hessian_sample_f64(int device_ordinal, int objective, long n, long B, const double* x0s_host,
                                                            const double* data0_host, const double* data1_host, long ldd, int ls,
                                                            const drv_param* q, double* xs_out, int kv, const double* V_host, double* LV_out,
                                                            unsigned long long seed, unsigned first, int kd, double* draws_out,
                                                            double* logdet_out, drv_small_item* items, char* err, int errlen)
{
    return small_batch_hessian_sample<double>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, kv, V_host,
                                              LV_out, seed, first, kd, draws_out, logdet_out, items, err, errlen);
}

extern "C" int lbfgsb200_drv_small_batch_hessian_sample_f32(int device_ordinal, int objective, long n, long B, const float* x0s_host,
                                                            const float* data0_host, const float* data1_host, long ldd, int ls,
                                                            const drv_param* q, float* xs_out, int kv, const float* V_host, float* LV_out,
                                                            unsigned long long seed, unsigned first, int kd, float* draws_out,
                                                            double* logdet_out, drv_small_item* items, char* err, int errlen)
{
    return small_batch_hessian_sample<float>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, kv, V_host,
                                             LV_out, seed, first, kd, draws_out, logdet_out, items, err, errlen);
}

#pragma GCC visibility pop
