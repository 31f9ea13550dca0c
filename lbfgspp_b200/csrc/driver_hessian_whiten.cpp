// driver_hessian_whiten.cpp -- host-buffer entry points of whitening and log densities under N(x*, H) from the final approximation
// (LBFGSSolver / LBFGSBatchSolver / LBFGSSmallBatchSolver::final_approx_inverse_hessian_factor_transpose_times / _solve /
// _transpose_solve / final_approx_log_density), built into lbfgspp_b200/liblbfgs_b200_driver.so next to driver.cpp.  A unit of its
// own, which refers to the passes it needs of the C ABI (lbfgs_b200_hist_s_dot_multi_* / _wt_dot_diff_*,
// lbfgs_b200_small_hist_factor_apply_* / _log_density_*) weakly: the driver library still loads against a library (or test double)
// that exports the C ABI without them, and these entry points then report which one is missing.
//
// op (LBFGS_B200_FACTOR_*): L, L', L^-1 or L^-T, with H = L L'.  Each entry point applies op to the kv vectors of V_host (into
// OV_out) and evaluates log N(x_j; mean, H) at the kx points of X_host (into logp_out), each only when its output is given.
#include "driver_small_batch.h"

#include <cstdio>

#pragma weak lbfgs_b200_hist_wt_dot_normal_f64   // op L shares BFGSMat's code with the sampler
#pragma weak lbfgs_b200_hist_wt_dot_normal_f32
#pragma weak lbfgs_b200_hist_lincomb_normal_f64
#pragma weak lbfgs_b200_hist_lincomb_normal_f32
#pragma weak lbfgs_b200_hist_s_dot_multi_f64
#pragma weak lbfgs_b200_hist_s_dot_multi_f32
#pragma weak lbfgs_b200_hist_wt_dot_diff_f64
#pragma weak lbfgs_b200_hist_wt_dot_diff_f32
#pragma weak lbfgs_b200_small_hist_factor_times_f64
#pragma weak lbfgs_b200_small_hist_factor_times_f32
#pragma weak lbfgs_b200_small_hist_factor_apply_f64
#pragma weak lbfgs_b200_small_hist_factor_apply_f32
#pragma weak lbfgs_b200_small_hist_log_density_f64
#pragma weak lbfgs_b200_small_hist_log_density_f32

using namespace LBFGSpp;
using namespace lbfgsb200_drv;

#pragma GCC visibility push(default)

namespace {

void require_whiten_passes()
{
    if (!lbfgs_b200_hist_s_dot_multi_f64 || !lbfgs_b200_hist_wt_dot_diff_f64)
        throw std::runtime_error("the C ABI library in use has no whitening passes (lbfgs_b200_hist_s_dot_multi_*, lbfgs_b200_hist_wt_dot_diff_*)");
}

void require_op(int op)
{
    if (op < LBFGS_B200_FACTOR_L || op > LBFGS_B200_FACTOR_LINVT) throw std::invalid_argument("op must be one of LBFGS_B200_FACTOR_*");
}

// op applied to the kv vectors of V_host (into OV_out) and the log densities of the kx points of X_host around mean (into logp_out).
// f(op, V, OUT) applies op, l(mean, X) returns the densities.
template <class F, class L>
void whiten_outputs(Device& dev, long n, int op, int kv, const double* V_host, double* OV_out, int kx, const double* X_host,
                    const DeviceVector<double>& mean, double* logp_out, F f, L l)
{
    if (OV_out && kv > 0)
    {
        DeviceVector<double> V(dev), out(dev);
        V.copy_from_host(V_host, std::ptrdiff_t(kv) * n);
        f(op, V, out);
        out.copy_to_host(OV_out);
    }
    if (logp_out && kx > 0)
    {
        DeviceVector<double> X(dev);
        X.copy_from_host(X_host, std::ptrdiff_t(kx) * n);
        const std::vector<double> lp = l(mean, X);
        std::copy(lp.begin(), lp.end(), logp_out);
    }
}

// the op of a solver, problem index first when it has one
template <class Solver, class Vec, class... B>
void apply_op(Solver& s, int op, const Vec& V, Vec& O, B... b)
{
    if (op == LBFGS_B200_FACTOR_L) s.final_approx_inverse_hessian_factor_times(b..., V, O);
    else if (op == LBFGS_B200_FACTOR_LT) s.final_approx_inverse_hessian_factor_transpose_times(b..., V, O);
    else if (op == LBFGS_B200_FACTOR_LINV) s.final_approx_inverse_hessian_factor_solve(b..., V, O);
    else s.final_approx_inverse_hessian_factor_transpose_solve(b..., V, O);
}

}  // namespace

// minimize() on a built-in objective (resident = 1: the device-resident solve, 0: the host-driven loop), then op(L) V and the log
// densities of N(mean, H) at the points of X (mean_host NULL: the solution).
extern "C" int lbfgsb200_drv_solve_hessian_whiten_f64(int device_ordinal, int objective, long n, int ls, const drv_param* q, int resident,
                                                      double* x_host, int op, int kv, const double* V_host, double* OV_out, int kx,
                                                      const double* X_host, const double* mean_host, double* logp_out, int* niter_out,
                                                      char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
        require_whiten_passes();
        require_op(op);
        Device& dev = device(device_ordinal);
        const LBFGSParam<double> prm = to_param<double>(q);
        BuiltinObjective<double> obj(objective);
        DeviceVector<double> x(dev), mean(dev);
        x.copy_from_host(x_host, n);
        double fx = 0;
        int niter = 0;
        with_line_search(ls, [&](auto tag) {
            typename decltype(tag)::template Solver<double> solver(prm);
            solver.set_device_resident(resident != 0);
            niter = solver.minimize(obj, x, fx);
            if (mean_host) mean.copy_from_host(mean_host, n);
            whiten_outputs(dev, n, op, kv, V_host, OV_out, kx, X_host, mean_host ? mean : x, logp_out,
                           [&](int o, const DeviceVector<double>& V, DeviceVector<double>& O) { apply_op(solver, o, V, O); },
                           [&](const DeviceVector<double>& mu, const DeviceVector<double>& X) { return solver.final_approx_log_density(mu, X); });
        });
        x.copy_to_host(x_host);
        if (niter_out) *niter_out = niter;
        return 0;
    });
}

// The same for problem b of a batch of B problems (rows of x0s_host) minimised by LBFGSBatchSolver (mean_host NULL: its solution).
// xs_out (optional) receives the solutions.
extern "C" int lbfgsb200_drv_batch_hessian_whiten_f64(int device_ordinal, int objective, long n, int B, const double* x0s_host, int ls,
                                                      const drv_param* q, int b, int op, int kv, const double* V_host, double* OV_out, int kx,
                                                      const double* X_host, const double* mean_host, double* logp_out, double* xs_out,
                                                      char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
        require_whiten_passes();
        require_op(op);
        Device& dev = device(device_ordinal);
        const LBFGSParam<double> prm = to_param<double>(q);
        BuiltinObjective<double> obj(objective);
        DeviceVector<double> X(dev), mean(dev);
        X.copy_from_host(x0s_host, std::ptrdiff_t(n) * B);
        with_line_search(ls, [&](auto tag) {
            typename decltype(tag)::template BatchSolver<double> solver(prm);
            solver.minimize(obj, X, B);
            std::vector<double> xs(size_t(n) * size_t(B));
            X.copy_to_host(xs.data());
            if (xs_out) std::copy(xs.begin(), xs.end(), xs_out);
            if (mean_host) mean.copy_from_host(mean_host, n);
            else if (b >= 0 && b < B) mean.copy_from_host(xs.data() + size_t(b) * size_t(n), n);
            whiten_outputs(dev, n, op, kv, V_host, OV_out, kx, X_host, mean, logp_out,
                           [&](int o, const DeviceVector<double>& V, DeviceVector<double>& O) { apply_op(solver, o, V, O, b); },
                           [&](const DeviceVector<double>& mu, const DeviceVector<double>& P) { return solver.final_approx_log_density(b, mu, P); });
        });
        return 0;
    });
}

// The same for an explicit history: the pairs (S_host[k], Y_host[k]) added in order to a ring of size m (test hook for BFGSMat's
// inverse_hessian_factor_* and log_density; mean_host: n values, required for the log densities)
extern "C" int lbfgsb200_drv_hist_whiten_f64(int device_ordinal, long n, int m, int npairs, const double* S_host, const double* Y_host, int op,
                                             int kv, const double* V_host, double* OV_out, int kx, const double* X_host, const double* mean_host,
                                             double* logp_out, char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
        require_whiten_passes();
        require_op(op);
        if (logp_out && kx > 0 && !mean_host) throw std::invalid_argument("the log densities need a mean");
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
        whiten_outputs(dev, n, op, kv, V_host, OV_out, kx, X_host, mean, logp_out,
                       [&](int o, const DeviceVector<double>& V, DeviceVector<double>& O) {
                           if (o == LBFGS_B200_FACTOR_L) mat.inverse_hessian_factor_times(V, kv, O);
                           else if (o == LBFGS_B200_FACTOR_LT) mat.inverse_hessian_factor_transpose_times(V, kv, O);
                           else if (o == LBFGS_B200_FACTOR_LINV) mat.inverse_hessian_factor_solve(V, kv, O);
                           else mat.inverse_hessian_factor_transpose_solve(V, kv, O);
                       },
                       [&](const DeviceVector<double>& mu, const DeviceVector<double>& X) { return mat.log_density(mu, X, kx); });
        return 0;
    });
}

namespace {

// small_batch with the final approximations kept, then for every problem: op(L_b) V (V_host: B*kv vectors, problem b's at b*kv*n) and
// the log densities of N(mean_b, H_b) at B*kx points (problem b's at b*kx*n; means_host: B means, NULL: the solutions), one launch
// each; logp_out[b*kx + j].  one >= 0: problem `one` alone through the one-problem forms (V_host kv vectors, X_host kx points,
// means_host one mean or NULL: its solution).
template <class Scalar>
int small_batch_hessian_whiten(int device_ordinal, int objective, long n, long B, const Scalar* x0s_host, const Scalar* data0_host,
                               const Scalar* data1_host, long ldd, int ls, const drv_param* q, Scalar* xs_out, int op, int kv, const Scalar* V_host,
                               Scalar* OV_out, int kx, const Scalar* X_host, const Scalar* means_host, double* logp_out, long one,
                               drv_small_item* items, char* err, int errlen)
{
    if (op < LBFGS_B200_FACTOR_L || op > LBFGS_B200_FACTOR_LINVT)
    {
        std::snprintf(err, size_t(errlen), "op must be one of LBFGS_B200_FACTOR_*");
        return -1;
    }
    if (!lbfgs_b200_small_hist_create || !lbfgs_b200_small_hist_destroy ||
        (sizeof(Scalar) == 8 ? !lbfgs_b200_small_minimize_keep_f64 || !lbfgs_b200_small_hist_factor_times_f64 ||
                                   !lbfgs_b200_small_hist_factor_apply_f64 || !lbfgs_b200_small_hist_log_density_f64
                             : !lbfgs_b200_small_minimize_keep_f32 || !lbfgs_b200_small_hist_factor_times_f32 ||
                                   !lbfgs_b200_small_hist_factor_apply_f32 || !lbfgs_b200_small_hist_log_density_f32))
    {
        std::snprintf(err, size_t(errlen), "the C ABI library in use has no small-batch whitening (lbfgs_b200_small_minimize_keep_*, "
                                           "lbfgs_b200_small_hist_factor_apply_*, lbfgs_b200_small_hist_log_density_*)");
        return -2;
    }
    return small_batch<Scalar>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, nullptr, items, err, errlen,
                               true, [&](auto& solver, Device& dev, DeviceVector<Scalar>& X) {
        const long per = one >= 0 ? 1 : B;   // problems whose vectors and points are given
        if (OV_out && kv > 0)
        {
            DeviceVector<Scalar> V(dev), out(dev);
            V.copy_from_host(V_host, std::ptrdiff_t(kv) * n * per);
            if (one >= 0) apply_op(solver, op, V, out, one);
            else apply_op(solver, op, V, out);
            out.copy_to_host(OV_out);
        }
        if (logp_out && kx > 0)
        {
            DeviceVector<Scalar> P(dev), M(dev);
            P.copy_from_host(X_host, std::ptrdiff_t(kx) * n * per);
            if (means_host) M.copy_from_host(means_host, std::ptrdiff_t(n) * per);
            else if (one >= 0 && one < B)   // problem one's solution
            {
                std::vector<Scalar> xs(size_t(n) * size_t(B));
                X.copy_to_host(xs.data());
                M.copy_from_host(xs.data() + size_t(one) * size_t(n), n);
            }
            const std::vector<double> lp = one >= 0 ? solver.final_approx_log_density(one, M, P)
                                                    : solver.final_approx_log_density(means_host ? M : X, P);
            std::copy(lp.begin(), lp.end(), logp_out);
        }
    });
}

}  // namespace

extern "C" int lbfgsb200_drv_small_batch_hessian_whiten_f64(int device_ordinal, int objective, long n, long B, const double* x0s_host,
                                                            const double* data0_host, const double* data1_host, long ldd, int ls,
                                                            const drv_param* q, double* xs_out, int op, int kv, const double* V_host,
                                                            double* OV_out, int kx, const double* X_host, const double* means_host,
                                                            double* logp_out, long one, drv_small_item* items, char* err,
                                                            int errlen)
{
    return small_batch_hessian_whiten<double>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, op, kv, V_host,
                                              OV_out, kx, X_host, means_host, logp_out, one, items, err, errlen);
}

extern "C" int lbfgsb200_drv_small_batch_hessian_whiten_f32(int device_ordinal, int objective, long n, long B, const float* x0s_host,
                                                            const float* data0_host, const float* data1_host, long ldd, int ls,
                                                            const drv_param* q, float* xs_out, int op, int kv, const float* V_host,
                                                            float* OV_out, int kx, const float* X_host, const float* means_host,
                                                            double* logp_out, long one, drv_small_item* items, char* err,
                                                            int errlen)
{
    return small_batch_hessian_whiten<float>(device_ordinal, objective, n, B, x0s_host, data0_host, data1_host, ldd, ls, q, xs_out, op, kv, V_host,
                                             OV_out, kx, X_host, means_host, logp_out, one, items, err, errlen);
}

#pragma GCC visibility pop
