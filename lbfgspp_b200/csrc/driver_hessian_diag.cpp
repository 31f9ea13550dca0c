// driver_hessian_diag.cpp -- host-buffer entry points of the diagonals of the final approximation
// (LBFGSSolver / LBFGSBatchSolver / LBFGSSmallBatchSolver::final_approx_hessian_diagonal / final_approx_inverse_hessian_diagonal),
// built into lbfgspp_b200/liblbfgs_b200_driver.so next to driver.cpp.  A unit of its own, which refers to the diagonal passes of the
// C ABI (lbfgs_b200_hist_quad_diag_*, lbfgs_b200_small_hist_diag_*) weakly: the driver library still loads against a library (or test
// double) that exports the C ABI without them, and these entry points then report which one is missing.
#include "driver_small_batch.h"

#include <cstdio>

#pragma weak lbfgs_b200_hist_quad_diag_f64
#pragma weak lbfgs_b200_hist_quad_diag_f32
#pragma weak lbfgs_b200_small_hist_diag_f64
#pragma weak lbfgs_b200_small_hist_diag_f32

using namespace LBFGSpp;
using namespace lbfgsb200_drv;

#pragma GCC visibility push(default)

namespace {

void require_quad_diag()
{
    if (!lbfgs_b200_hist_quad_diag_f64)
        throw std::runtime_error("the C ABI library in use has no diagonal pass (lbfgs_b200_hist_quad_diag_*)");
}

// diag(B) and diag(H) of a final approximation into the host buffers that are given.  diag(out, inverse) is
// final_approx_{inverse_,}hessian_diagonal.
template <class Diag>
void diagonals(Device& dev, Diag diag, double* dB_out, double* dH_out)
{
    DeviceVector<double> d(dev);
    if (dB_out)
    {
        diag(d, false);
        d.copy_to_host(dB_out);
    }
    if (dH_out)
    {
        diag(d, true);
        d.copy_to_host(dH_out);
    }
}

}  // namespace

// minimize() on a built-in objective (resident = 1: the device-resident solve, 0: the host-driven loop), then the diagonals of
// final_approx_hessian() / final_approx_inverse_hessian() (LBFGSSolver::final_approx_*_diagonal), n values each.
extern "C" int lbfgsb200_drv_solve_hessian_diag_f64(int device_ordinal, int objective, long n, int ls, const drv_param* q, int resident,
                                                    double* x_host, double* dB_out, double* dH_out, int* niter_out, char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
        require_quad_diag();
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
            diagonals(dev, [&](DeviceVector<double>& out, bool inverse) {
                if (inverse) solver.final_approx_inverse_hessian_diagonal(out);
                else solver.final_approx_hessian_diagonal(out);
            }, dB_out, dH_out);
        });
        x.copy_to_host(x_host);
        if (niter_out) *niter_out = niter;
        return 0;
    });
}

// The same for problem b of a batch of B problems (rows of x0s_host) minimised by LBFGSBatchSolver (one persistent kernel launch).
extern "C" int lbfgsb200_drv_batch_hessian_diag_f64(int device_ordinal, int objective, long n, int B, const double* x0s_host, int ls,
                                                    const drv_param* q, int b, double* dB_out, double* dH_out, char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
        require_quad_diag();
        Device& dev = device(device_ordinal);
        const LBFGSParam<double> prm = to_param<double>(q);
        BuiltinObjective<double> obj(objective);
        DeviceVector<double> X(dev);
        X.copy_from_host(x0s_host, std::ptrdiff_t(n) * B);
        with_line_search(ls, [&](auto tag) {
            typename decltype(tag)::template BatchSolver<double> solver(prm);
            solver.minimize(obj, X, B);
            diagonals(dev, [&](DeviceVector<double>& out, bool inverse) {
                if (inverse) solver.final_approx_inverse_hessian_diagonal(b, out);
                else solver.final_approx_hessian_diagonal(b, out);
            }, dB_out, dH_out);
        });
        return 0;
    });
}

// diag(B) and diag(H) of an explicit history (test hook for BFGSMat::hessian_diagonal / inverse_hessian_diagonal)
extern "C" int lbfgsb200_drv_hist_diag_f64(int device_ordinal, long n, int m, int npairs, const double* S_host, const double* Y_host,
                                           double* dB_out, double* dH_out, char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
        require_quad_diag();
        Device& dev = device(device_ordinal);
        BFGSMat<double> mat;
        mat.reset(dev, n, m);
        DeviceVector<double> s(dev), y(dev);
        for (int k = 0; k < npairs; k++)
        {
            s.copy_from_host(S_host + size_t(k) * n, n);
            y.copy_from_host(Y_host + size_t(k) * n, n);
            mat.add_correction(s, y);
        }
        diagonals(dev, [&](DeviceVector<double>& out, bool inverse) {
            if (inverse) mat.inverse_hessian_diagonal(out);
            else mat.hessian_diagonal(out);
        }, dB_out, dH_out);
        return 0;
    });
}

namespace {

// small_batch with the final approximations kept, then every problem's diag(B_b) and diag(H_b) (B*n values each, problem b's at b*n)
// from one launch each
template <class Scalar>
int small_batch_hessian_diag(int device_ordinal, int objective, long n, long B, const Scalar* x0s_host, const Scalar* data0_host,
                             const Scalar* data1_host, long ldd, int ls, const drv_param* q, Scalar* xs_out, Scalar* dB_out, Scalar* dH_out,
                             drv_small_item* items, char* err, int errlen)
{
    if (!lbfgs_b200_small_hist_create || !lbfgs_b200_small_hist_destroy ||
        (sizeof(Scalar) == 8 ? !lbfgs_b200_small_minimize_keep_f64 || !lbfgs_b200_small_hist_diag_f64
                             : !lbfgs_b200_small_minimize_keep_f32 || !lbfgs_b200_small_hist_diag_f32))
    {
        std::snprintf(err, size_t(errlen), "the C ABI library in use has no small-batch diagonals (lbfgs_b200_small_minimize_keep_*, "
                                           "lbfgs_b200_small_hist_diag_*)");
        return -2;
    }
    return small_batch<Scalar>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, nullptr, items, err, errlen,
                               true, [&](auto& solver, Device& dev) {
        DeviceVector<Scalar> d(dev);
        if (dB_out)
        {
            solver.final_approx_hessian_diagonal(d);
            d.copy_to_host(dB_out);
        }
        if (dH_out)
        {
            solver.final_approx_inverse_hessian_diagonal(d);
            d.copy_to_host(dH_out);
        }
    });
}

}  // namespace

extern "C" int lbfgsb200_drv_small_batch_hessian_diag_f64(int device_ordinal, int objective, long n, long B, const double* x0s_host,
                                                          const double* data0_host, const double* data1_host, long ldd, int ls, const drv_param* q,
                                                          double* xs_out, double* dB_out, double* dH_out, drv_small_item* items, char* err,
                                                          int errlen)
{
    return small_batch_hessian_diag<double>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, dB_out, dH_out,
                                            items, err, errlen);
}

extern "C" int lbfgsb200_drv_small_batch_hessian_diag_f32(int device_ordinal, int objective, long n, long B, const float* x0s_host,
                                                          const float* data0_host, const float* data1_host, long ldd, int ls, const drv_param* q,
                                                          float* xs_out, float* dB_out, float* dH_out, drv_small_item* items, char* err,
                                                          int errlen)
{
    return small_batch_hessian_diag<float>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, dB_out, dH_out,
                                           items, err, errlen);
}

#pragma GCC visibility pop
