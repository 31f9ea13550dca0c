// driver_small_batch.cpp -- host-buffer entry points of the small-batch solve (LBFGSSmallBatchSolver, include/LBFGSSmallBatch.h),
// built into lbfgspp_b200/liblbfgs_b200_driver.so next to driver.cpp.  A unit of its own, which refers to the small-batch part of
// the C ABI weakly: the driver library still loads against a library (or test double) that exports the C ABI without it, and these
// entry points then report that instead.
#include "driver_small_batch.h"

#include <algorithm>
#include <cstdio>
#include <type_traits>

using namespace LBFGSpp;
using namespace lbfgsb200_drv;

#pragma GCC visibility push(default)

namespace {

// small_batch with the final approximations kept, then B_b V_b, H_b V_b and H_b (B_b V_b) for every problem b.  V_host: k vectors
// of n shared by all problems (shared != 0) or B*k of them, problem b's at [(b*k + j)*n, ...); BV/HV/HBV: B*k*n each.
template <class Scalar>
int small_batch_hessian_times(int device_ordinal, int objective, long n, long B, const Scalar* x0s_host, const Scalar* data0_host,
                              const Scalar* data1_host, long ldd, int ls, const drv_param* q, const Scalar* V_host, long k, int shared,
                              Scalar* xs_out, Scalar* BV, Scalar* HV, Scalar* HBV, drv_small_item* items, char* err, int errlen)
{
    if (!lbfgs_b200_small_hist_create || !lbfgs_b200_small_hist_destroy ||
        (sizeof(Scalar) == 8 ? !lbfgs_b200_small_minimize_keep_f64 || !lbfgs_b200_small_hist_times_f64
                             : !lbfgs_b200_small_minimize_keep_f32 || !lbfgs_b200_small_hist_times_f32))
    {
        std::snprintf(err, size_t(errlen), "the C ABI library in use has no kept small-batch approximations (lbfgs_b200_small_minimize_keep_*, "
                                           "lbfgs_b200_small_hist_*)");
        return -2;
    }
    return small_batch<Scalar>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, nullptr, items, err, errlen,
                               true, [&](auto& solver, Device& dev) {
        const size_t total = size_t(B) * size_t(k) * size_t(n);
        std::vector<Scalar> v(total);
        for (long b = 0; b < B; b++)
            std::copy(V_host + (shared ? 0 : size_t(b) * size_t(k) * size_t(n)), V_host + (shared ? 0 : size_t(b) * size_t(k) * size_t(n)) + size_t(k) * size_t(n),
                      v.begin() + std::ptrdiff_t(size_t(b) * size_t(k) * size_t(n)));
        DeviceVector<Scalar> Vd(dev), Bd(dev), Hd(dev), HBd(dev);
        Vd.copy_from_host(v.data(), std::ptrdiff_t(total));
        solver.final_approx_hessian_times(Vd, Bd);
        solver.final_approx_inverse_hessian_times(Vd, Hd);
        solver.final_approx_inverse_hessian_times(Bd, HBd);
        Bd.copy_to_host(BV);
        Hd.copy_to_host(HV);
        HBd.copy_to_host(HBV);
    });
}

}  // namespace

extern "C" int lbfgsb200_drv_small_batch_hessian_times_f64(int device_ordinal, int objective, long n, long B, const double* x0s_host,
                                                           const double* data0_host, const double* data1_host, long ldd, int ls, const drv_param* q,
                                                           const double* V_host, long k, int shared, double* xs_out, double* BV, double* HV,
                                                           double* HBV, drv_small_item* items, char* err, int errlen)
{
    return small_batch_hessian_times<double>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, V_host, k, shared, xs_out,
                                             BV, HV, HBV, items, err, errlen);
}

extern "C" int lbfgsb200_drv_small_batch_hessian_times_f32(int device_ordinal, int objective, long n, long B, const float* x0s_host,
                                                           const float* data0_host, const float* data1_host, long ldd, int ls, const drv_param* q,
                                                           const float* V_host, long k, int shared, float* xs_out, float* BV, float* HV,
                                                           float* HBV, drv_small_item* items, char* err, int errlen)
{
    return small_batch_hessian_times<float>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, V_host, k, shared, xs_out,
                                            BV, HV, HBV, items, err, errlen);
}

extern "C" int lbfgsb200_drv_small_batch_f64(int device_ordinal, int objective, long n, long B, const double* x0s_host, const double* data0_host,
                                             const double* data1_host, long ldd, int ls, const drv_param* q, double* xs_out, double* gs_out,
                                             drv_small_item* items, char* err, int errlen)
{
    return small_batch<double>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, gs_out, items, err, errlen);
}

extern "C" int lbfgsb200_drv_small_batch_f32(int device_ordinal, int objective, long n, long B, const float* x0s_host, const float* data0_host,
                                             const float* data1_host, long ldd, int ls, const drv_param* q, float* xs_out, float* gs_out,
                                             drv_small_item* items, char* err, int errlen)
{
    return small_batch<float>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, gs_out, items, err, errlen);
}

#pragma GCC visibility pop
