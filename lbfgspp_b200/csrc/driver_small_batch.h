// driver_small_batch.h -- the small-batch solve behind the host-buffer entry points of csrc/driver_small_batch.cpp and
// csrc/driver_hessian_diag.cpp.  The small-batch part of the C ABI is referred to weakly: the driver library still loads against a
// library (or test double) that exports the C ABI without it, and the entry points then report that instead.
#ifndef LBFGSPP_B200_DRIVER_SMALL_BATCH_H
#define LBFGSPP_B200_DRIVER_SMALL_BATCH_H

#include "../../include/LBFGSpp/DeviceObjectives.h"
#include "driver_common.h"

#include <type_traits>

#pragma weak lbfgs_b200_small_minimize_f64
#pragma weak lbfgs_b200_small_minimize_f32
#pragma weak lbfgs_b200_small_minimize_keep_f64
#pragma weak lbfgs_b200_small_minimize_keep_f32
#pragma weak lbfgs_b200_small_hist_create
#pragma weak lbfgs_b200_small_hist_destroy
#pragma weak lbfgs_b200_small_hist_times_f64
#pragma weak lbfgs_b200_small_hist_times_f32

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

namespace lbfgsb200_drv {

// B problems (rows of x0s_host, n each) minimised by LBFGSSmallBatchSolver; data0/data1 (optional, host) per problem at data + b*ldd
// (ldd = 0: shared).  xs_out / gs_out (optional): solutions and final gradients.  Returns the number of problems that did not end
// cleanly, -1 (err holds the message) when the call was refused as an invalid argument, -2 on any other failure.
// `after(solver, dev)` or `after(solver, dev, X)` (optional, X: the solutions on the device) runs on the solver once minimize() has returned; `keep`: minimize() keeps the final approximations
template <class Scalar, class After = std::nullptr_t>
int small_batch(int device_ordinal, int objective, long n, long B, const Scalar* x0s_host, const Scalar* data0_host, const Scalar* data1_host,
                long ldd, int ls, const drv_param* q, Scalar* xs_out, Scalar* gs_out, drv_small_item* items, char* err, int errlen,
                bool keep = false, After after = nullptr)
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
                solver.keep_final_approx(keep);
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
                if constexpr (std::is_invocable_v<After&, decltype(solver)&, Device&, DeviceVector<Scalar>&>) after(solver, dev, X);
                else if constexpr (!std::is_same_v<After, std::nullptr_t>) after(solver, dev);
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

}  // namespace lbfgsb200_drv

#endif  // LBFGSPP_B200_DRIVER_SMALL_BATCH_H
