// driver_hessian_ops.cpp -- host-buffer entry points of the operator form of the final approximation
// (LBFGSSolver / LBFGSBatchSolver::final_approx_hessian_times / final_approx_inverse_hessian_times), built into
// lbfgspp_b200/liblbfgs_b200_driver.so next to driver.cpp.  A unit of its own: the other entry points link against any library that
// exports the C ABI without the k-vector passes (lbfgs_b200_hist_wt_dot_multi / lbfgs_b200_hist_lincomb_multi).
#include "../../include/LBFGSpp/DeviceObjectives.h"
#include "driver_common.h"

using namespace LBFGSpp;
using namespace lbfgsb200_drv;

#pragma GCC visibility push(default)

namespace {

// Products of a final approximation with the v_len / n vectors of V_host (back to back): BV_out = B V, HV_out = H V,
// HBV_out = H (B V), each when its buffer is given.  apply(V, OUT, inverse) is final_approx_{inverse_,}hessian_times.
template <class Apply>
void hessian_products(Device& dev, Apply apply, const double* V_host, long v_len, double* BV_out, double* HV_out, double* HBV_out)
{
    if (!V_host && v_len > 0) throw std::invalid_argument("V is NULL");
    DeviceVector<double> V(dev), BV(dev), OUT(dev);
    V.copy_from_host(V_host, v_len);
    if (BV_out || HBV_out)
    {
        apply(V, BV, false);
        if (BV_out) BV.copy_to_host(BV_out);
    }
    if (HV_out)
    {
        apply(V, OUT, true);
        OUT.copy_to_host(HV_out);
    }
    if (HBV_out)
    {
        apply(BV, OUT, true);
        OUT.copy_to_host(HBV_out);
    }
}

}  // namespace

// minimize() on a built-in objective (resident = 1: the device-resident solve, 0: the host-driven loop), then the operator form of
// final_approx_hessian() / final_approx_inverse_hessian() (LBFGSSolver::final_approx_*_times) on the v_len / n vectors of V_host.
extern "C" int lbfgsb200_drv_solve_hessian_times_f64(int device_ordinal, int objective, long n, int ls, const drv_param* q, int resident,
                                                     double* x_host, const double* V_host, long v_len, double* BV_out, double* HV_out,
                                                     double* HBV_out, int* niter_out, char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
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
            hessian_products(dev, [&](const DeviceVector<double>& V, DeviceVector<double>& OUT, bool inverse) {
                if (inverse) solver.final_approx_inverse_hessian_times(V, OUT);
                else solver.final_approx_hessian_times(V, OUT);
            }, V_host, v_len, BV_out, HV_out, HBV_out);
        });
        x.copy_to_host(x_host);
        if (niter_out) *niter_out = niter;
        return 0;
    });
}

// The same for problem b of a batch of B problems (rows of x0s_host) minimised by LBFGSBatchSolver (one persistent kernel launch).
extern "C" int lbfgsb200_drv_batch_hessian_times_f64(int device_ordinal, int objective, long n, int B, const double* x0s_host, int ls,
                                                     const drv_param* q, int b, const double* V_host, long v_len, double* BV_out,
                                                     double* HV_out, double* HBV_out, char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
        Device& dev = device(device_ordinal);
        const LBFGSParam<double> prm = to_param<double>(q);
        BuiltinObjective<double> obj(objective);
        DeviceVector<double> X(dev);
        X.copy_from_host(x0s_host, std::ptrdiff_t(n) * B);
        with_line_search(ls, [&](auto tag) {
            typename decltype(tag)::template BatchSolver<double> solver(prm);
            solver.minimize(obj, X, B);
            hessian_products(dev, [&](const DeviceVector<double>& V, DeviceVector<double>& OUT, bool inverse) {
                if (inverse) solver.final_approx_inverse_hessian_times(b, V, OUT);
                else solver.final_approx_hessian_times(b, V, OUT);
            }, V_host, v_len, BV_out, HV_out, HBV_out);
        });
        return 0;
    });
}

// B V and H V of an explicit history (test hook for BFGSMat::hessian_times / inverse_hessian_times, the operator form of the above)
extern "C" int lbfgsb200_drv_hist_times_f64(int device_ordinal, long n, int m, int npairs, const double* S_host, const double* Y_host,
                                            const double* V_host, long v_len, double* BV_out, double* HV_out, char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
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
        const int k = BFGSMat<double>::block_count(v_len, n);
        hessian_products(dev, [&](const DeviceVector<double>& V, DeviceVector<double>& OUT, bool inverse) {
            if (inverse) mat.inverse_hessian_times(V, k, OUT);
            else mat.hessian_times(V, k, OUT);
        }, V_host, v_len, BV_out, HV_out, nullptr);
        return 0;
    });
}

#pragma GCC visibility pop
