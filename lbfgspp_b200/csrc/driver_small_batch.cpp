// driver_small_batch.cpp -- host-buffer entry points of the small-batch solve (LBFGSSmallBatchSolver, include/LBFGSSmallBatch.h),
// built into lbfgspp_b200/liblbfgs_b200_driver.so next to driver.cpp.  A unit of its own, which refers to the small-batch part of
// the C ABI weakly: the driver library still loads against a library (or test double) that exports the C ABI without it, and these
// entry points then report that instead.
#include "../../include/LBFGSpp/DeviceObjectives.h"
#include "driver_common.h"

#pragma weak lbfgs_b200_small_minimize_f64
#pragma weak lbfgs_b200_small_minimize_f32

using namespace LBFGSpp;
using namespace lbfgsb200_drv;

#pragma GCC visibility push(default)

extern "C" {

typedef struct
{
    int code;           // 0, or the LineSearchError code of the exception LBFGSSolver would have thrown (LBFGSpp/LineSearchCore.h)
    int kind;           // 0 ok, 1 invalid_argument, 2 logic_error, 3 runtime_error (ls_error_kind)
    int niter;
    long nfev;
    double fx, gnorm;
    long rounds;
} drv_small_item;

}  // extern "C"

namespace {

// B problems (rows of x0s_host, n each) minimised by LBFGSSmallBatchSolver; data0/data1 (optional, host) per problem at data + b*ldd
// (ldd = 0: shared).  xs_out / gs_out (optional): solutions and final gradients.  Returns the number of problems that did not end
// cleanly, -1 (err holds the message) when the call was refused as an invalid argument, -2 on any other failure.
template <class Scalar>
int small_batch(int device_ordinal, int objective, long n, long B, const Scalar* x0s_host, const Scalar* data0_host, const Scalar* data1_host,
                long ldd, int ls, const drv_param* q, Scalar* xs_out, Scalar* gs_out, drv_small_item* items, char* err, int errlen)
{
    int invalid = 0;
    const int r = reported(err, errlen, -2, [&]() {
        try
        {
            if (sizeof(Scalar) == 8 ? !lbfgs_b200_small_minimize_f64 : !lbfgs_b200_small_minimize_f32)
                throw std::runtime_error("the C ABI library in use has no small-batch solve (lbfgs_b200_small_minimize_*)");
            Device& dev = device(device_ordinal);
            const LBFGSParam<Scalar> prm = to_param<Scalar>(q);
            DeviceVector<Scalar> X(dev), D0(dev), D1(dev);
            X.copy_from_host(x0s_host, std::ptrdiff_t(n) * B);
            const std::ptrdiff_t dlen = ldd ? std::ptrdiff_t(ldd) * (B - 1) + n : n;
            if (data0_host) D0.copy_from_host(data0_host, dlen);
            if (data1_host) D1.copy_from_host(data1_host, dlen);
            BuiltinObjective<Scalar> obj(objective, data0_host ? D0.data() : nullptr, data1_host ? D1.data() : nullptr);
            int bad = 0;
            with_line_search(ls, [&](auto tag) {
                typename decltype(tag)::template SmallBatchSolver<Scalar> solver(prm);
                const std::vector<BatchOutcome<Scalar> > out = solver.minimize(obj, X, B, ldd);
                for (long b = 0; b < B; b++)
                {
                    const BatchOutcome<Scalar>& o = out[size_t(b)];
                    items[b].code = o.status;
                    items[b].kind = o.status == 0 ? 0 : ls_error_kind(o.status);
                    items[b].niter = o.niter; items[b].nfev = o.nfev; items[b].fx = double(o.fx); items[b].gnorm = double(o.gnorm);
                    items[b].rounds = o.rounds;
                    bad += o.status != 0;
                }
                if (gs_out)
                    dev.check(lbfgs_b200_memcpy_d2h(dev.ctx(), gs_out, solver.final_grad(0), sizeof(Scalar) * size_t(n) * size_t(B)));
            });
            if (xs_out) X.copy_to_host(xs_out);
            return bad;
        }
        catch (const std::invalid_argument&)
        {
            invalid = 1;
            throw;
        }
    });
    return (r == -2 && invalid) ? -1 : r;
}

}  // namespace

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
