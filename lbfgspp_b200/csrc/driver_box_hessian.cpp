// driver_box_hessian.cpp -- host-buffer entry points of the final approximation of a bound-constrained solve (LBFGSBSolver::
// final_approx_* over the whole space and final_approx_free_* on the free variables at the solution), built into
// lbfgspp_b200/liblbfgs_b200_driver.so next to driver.cpp.  A unit of its own, which refers to every pass it needs of the C ABI weakly:
// the driver library still loads against a library (or test double) that exports the C ABI without them, and these entry points then
// report which one is missing.
//
// op (DRV_BOXH_*) is one operation on the approximation; `free` chooses B_F / H_F on the free set (1) or B / H over the whole space
// (0).  Outputs go to out (vectors: kv*n products or draws, n for a diagonal, n*n for a dense matrix) and dout (kv log densities);
// logdet_out (optional) always receives log det H or log det H_F.
#include "driver_common.h"
#include "../../include/LBFGSB.h"

#pragma weak lbfgs_b200_hist_wt_dot_multi_f64
#pragma weak lbfgs_b200_hist_wt_dot_multi_f32
#pragma weak lbfgs_b200_hist_lincomb_multi_f64
#pragma weak lbfgs_b200_hist_lincomb_multi_f32
#pragma weak lbfgs_b200_hist_quad_diag_f64
#pragma weak lbfgs_b200_hist_quad_diag_f32
#pragma weak lbfgs_b200_hist_wt_dot_normal_f64
#pragma weak lbfgs_b200_hist_wt_dot_normal_f32
#pragma weak lbfgs_b200_hist_lincomb_normal_f64
#pragma weak lbfgs_b200_hist_lincomb_normal_f32
#pragma weak lbfgs_b200_hist_s_dot_multi_f64
#pragma weak lbfgs_b200_hist_s_dot_multi_f32
#pragma weak lbfgs_b200_hist_wt_dot_diff_f64
#pragma weak lbfgs_b200_hist_wt_dot_diff_f32
#pragma weak lbfgs_b200_hist_wt_dot_multi_masked_f64
#pragma weak lbfgs_b200_hist_wt_dot_multi_masked_f32
#pragma weak lbfgs_b200_hist_wt_dot_diff_masked_f64
#pragma weak lbfgs_b200_hist_wt_dot_diff_masked_f32
#pragma weak lbfgs_b200_hist_wt_dot_normal_masked_f64
#pragma weak lbfgs_b200_hist_wt_dot_normal_masked_f32
#pragma weak lbfgs_b200_hist_lincomb_multi_masked_f64
#pragma weak lbfgs_b200_hist_lincomb_multi_masked_f32
#pragma weak lbfgs_b200_hist_lincomb_normal_masked_f64
#pragma weak lbfgs_b200_hist_lincomb_normal_masked_f32
#pragma weak lbfgs_b200_hist_quad_diag_masked_f64
#pragma weak lbfgs_b200_hist_quad_diag_masked_f32
#pragma weak lbfgs_b200_box_final_classes_f64
#pragma weak lbfgs_b200_box_final_classes_f32

using namespace LBFGSpp;
using namespace lbfgsb200_drv;

extern "C" {
enum { DRV_BOXH_B_TIMES = 0, DRV_BOXH_H_TIMES = 1, DRV_BOXH_B_DIAG = 2, DRV_BOXH_H_DIAG = 3, DRV_BOXH_SAMPLE = 4, DRV_BOXH_LOG_DENSITY = 5,
       DRV_BOXH_LOGDET = 6, DRV_BOXH_L = 7, DRV_BOXH_LT = 8, DRV_BOXH_LINV = 9, DRV_BOXH_LINVT = 10, DRV_BOXH_DENSE_B = 11,
       DRV_BOXH_DENSE_H = 12 };
}

#pragma GCC visibility push(default)

namespace {

// the passes an operation needs, named when the library in use lacks one
template <class Scalar> void require_passes(int op, bool free)
{
    const bool d = sizeof(Scalar) == 8;
    auto need = [](bool have, const char* what) {
        if (!have) throw std::runtime_error(std::string("the C ABI library in use has no ") + what);
    };
    if (op < DRV_BOXH_B_TIMES || op > DRV_BOXH_DENSE_H) throw std::invalid_argument("op must be one of DRV_BOXH_*");
    if (free)
    {
        if (op >= DRV_BOXH_L) throw std::invalid_argument("the free set has no factor products and no dense matrices");
        need(d ? lbfgs_b200_box_final_classes_f64 && lbfgs_b200_hist_wt_dot_multi_masked_f64 && lbfgs_b200_hist_wt_dot_diff_masked_f64 &&
                     lbfgs_b200_hist_wt_dot_normal_masked_f64 && lbfgs_b200_hist_lincomb_multi_masked_f64 &&
                     lbfgs_b200_hist_lincomb_normal_masked_f64 && lbfgs_b200_hist_quad_diag_masked_f64
               : lbfgs_b200_box_final_classes_f32 && lbfgs_b200_hist_wt_dot_multi_masked_f32 && lbfgs_b200_hist_wt_dot_diff_masked_f32 &&
                     lbfgs_b200_hist_wt_dot_normal_masked_f32 && lbfgs_b200_hist_lincomb_multi_masked_f32 &&
                     lbfgs_b200_hist_lincomb_normal_masked_f32 && lbfgs_b200_hist_quad_diag_masked_f32,
             "free-set passes (lbfgs_b200_box_final_classes_*, lbfgs_b200_hist_*_masked_*)");
        return;
    }
    need(d ? lbfgs_b200_hist_wt_dot_multi_f64 && lbfgs_b200_hist_lincomb_multi_f64 : lbfgs_b200_hist_wt_dot_multi_f32 && lbfgs_b200_hist_lincomb_multi_f32,
         "k-vector passes (lbfgs_b200_hist_wt_dot_multi_*, lbfgs_b200_hist_lincomb_multi_*)");
    if (op == DRV_BOXH_B_DIAG || op == DRV_BOXH_H_DIAG)
        need(d ? lbfgs_b200_hist_quad_diag_f64 != nullptr : lbfgs_b200_hist_quad_diag_f32 != nullptr, "diagonal pass (lbfgs_b200_hist_quad_diag_*)");
    if (op == DRV_BOXH_SAMPLE || op == DRV_BOXH_L)
        need(d ? lbfgs_b200_hist_wt_dot_normal_f64 && lbfgs_b200_hist_lincomb_normal_f64 : lbfgs_b200_hist_wt_dot_normal_f32 && lbfgs_b200_hist_lincomb_normal_f32,
             "sampler passes (lbfgs_b200_hist_wt_dot_normal_*, lbfgs_b200_hist_lincomb_normal_*)");
    if (op == DRV_BOXH_LOG_DENSITY || op >= DRV_BOXH_LT)
        need(d ? lbfgs_b200_hist_s_dot_multi_f64 && lbfgs_b200_hist_wt_dot_diff_f64 : lbfgs_b200_hist_s_dot_multi_f32 && lbfgs_b200_hist_wt_dot_diff_f32,
             "whitening passes (lbfgs_b200_hist_s_dot_multi_*, lbfgs_b200_hist_wt_dot_diff_*)");
}

// op on an approximation A (LBFGSBSolver, or BFGSMat through BoxMat below); V_host: kv vectors (products, factor ops) or points (log
// density); mean: the draws' and densities' mean
template <class Scalar, class A>
void box_op(Device& dev, A& a, long n, bool free, int op, int kv, const Scalar* V_host, const DeviceVector<Scalar>& mean, unsigned long long seed,
            unsigned first, Scalar* out, double* dout, double* logdet_out)
{
    typedef DeviceVector<Scalar> Vector;
    Vector V(dev), O(dev);
    if (V_host && kv > 0) V.copy_from_host(V_host, std::ptrdiff_t(kv) * n);
    switch (op)
    {
    case DRV_BOXH_B_TIMES: free ? a.final_approx_free_hessian_times(V, O) : a.final_approx_hessian_times(V, O); break;
    case DRV_BOXH_H_TIMES: free ? a.final_approx_free_inverse_hessian_times(V, O) : a.final_approx_inverse_hessian_times(V, O); break;
    case DRV_BOXH_B_DIAG: free ? a.final_approx_free_hessian_diagonal(O) : a.final_approx_hessian_diagonal(O); break;
    case DRV_BOXH_H_DIAG: free ? a.final_approx_free_inverse_hessian_diagonal(O) : a.final_approx_inverse_hessian_diagonal(O); break;
    case DRV_BOXH_SAMPLE: free ? a.final_approx_free_sample(mean, seed, first, kv, O) : a.final_approx_sample(mean, seed, first, kv, O); break;
    case DRV_BOXH_LOG_DENSITY:
    {
        const std::vector<double> lp = free ? a.final_approx_free_log_density(mean, V) : a.final_approx_log_density(mean, V);
        if (dout) std::copy(lp.begin(), lp.end(), dout);
        break;
    }
    case DRV_BOXH_L: a.final_approx_inverse_hessian_factor_times(V, O); break;
    case DRV_BOXH_LT: a.final_approx_inverse_hessian_factor_transpose_times(V, O); break;
    case DRV_BOXH_LINV: a.final_approx_inverse_hessian_factor_solve(V, O); break;
    case DRV_BOXH_LINVT: a.final_approx_inverse_hessian_factor_transpose_solve(V, O); break;
    case DRV_BOXH_DENSE_B:
    case DRV_BOXH_DENSE_H:
    {
        const SmallMatrix<Scalar> D = op == DRV_BOXH_DENSE_B ? a.final_approx_hessian() : a.final_approx_inverse_hessian();
        if (out) std::copy(D.data(), D.data() + size_t(n) * size_t(n), out);
        break;
    }
    default: break;
    }
    if (out && O.size() > 0) O.copy_to_host(out);
    if (logdet_out) *logdet_out = free ? a.final_approx_free_inverse_hessian_logdet() : a.final_approx_inverse_hessian_logdet();
}

// LBFGSBSolver's members over an explicit history (test hook): the same names on a BFGSMat whose pairs were added one by one
template <class Scalar>
struct BoxMat
{
    typedef DeviceVector<Scalar> Vector;
    BFGSMat<Scalar, true> m;
    int k(const Vector& V) { return BFGSMat<Scalar, true>::block_count(V.size(), m.dim()); }
    void final_approx_hessian_times(const Vector& V, Vector& O) { m.hessian_times(V, k(V), O); }
    void final_approx_inverse_hessian_times(const Vector& V, Vector& O) { m.inverse_hessian_times(V, k(V), O); }
    void final_approx_hessian_diagonal(Vector& O) { m.hessian_diagonal(O); }
    void final_approx_inverse_hessian_diagonal(Vector& O) { m.inverse_hessian_diagonal(O); }
    void final_approx_sample(const Vector& mu, unsigned long long seed, unsigned first, int kv, Vector& O) { m.sample(&mu, seed, 0u, first, kv, O); }
    std::vector<double> final_approx_log_density(const Vector& mu, const Vector& X) { return m.log_density(mu, X, k(X)); }
    double final_approx_inverse_hessian_logdet() { return m.inverse_hessian_logdet(); }
    void final_approx_inverse_hessian_factor_times(const Vector& V, Vector& O) { m.inverse_hessian_factor_times(V, k(V), O); }
    void final_approx_inverse_hessian_factor_transpose_times(const Vector& V, Vector& O) { m.inverse_hessian_factor_transpose_times(V, k(V), O); }
    void final_approx_inverse_hessian_factor_solve(const Vector& V, Vector& O) { m.inverse_hessian_factor_solve(V, k(V), O); }
    void final_approx_inverse_hessian_factor_transpose_solve(const Vector& V, Vector& O) { m.inverse_hessian_factor_transpose_solve(V, k(V), O); }
    SmallMatrix<Scalar> final_approx_hessian() { return m.dense(false); }
    SmallMatrix<Scalar> final_approx_inverse_hessian() { return m.dense(true); }
    void final_approx_free_hessian_times(const Vector& V, Vector& O) { m.free_hessian_times(V, k(V), O); }
    void final_approx_free_inverse_hessian_times(const Vector& V, Vector& O) { m.free_inverse_hessian_times(V, k(V), O); }
    void final_approx_free_hessian_diagonal(Vector& O) { m.free_hessian_diagonal(O); }
    void final_approx_free_inverse_hessian_diagonal(Vector& O) { m.free_inverse_hessian_diagonal(O); }
    void final_approx_free_sample(const Vector& mu, unsigned long long seed, unsigned first, int kv, Vector& O) { m.free_sample(&mu, seed, 0u, first, kv, O); }
    std::vector<double> final_approx_free_log_density(const Vector& mu, const Vector& X) { return m.free_log_density(mu, X, k(X)); }
    double final_approx_free_inverse_hessian_logdet() { return m.free_inverse_hessian_logdet(); }
};

// LBFGSBSolver<Scalar>::minimize on a built-in objective, then op (tol < 0: the default tolerance of final_approx_free_set)
template <class Scalar>
int box_hessian(int device_ordinal, int objective, long n, const drv_param* q, Scalar* x_host, const Scalar* lb_host, const Scalar* ub_host,
                int free, double tol, int op, int kv, const Scalar* V_host, const Scalar* mean_host, unsigned long long seed, unsigned first,
                Scalar* out, double* dout, double* logdet_out, long* nfree_out, int* niter_out, char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
        require_passes<Scalar>(op, free != 0);
        Device& dev = device(device_ordinal);
        typedef DeviceVector<Scalar> Vector;
        Vector x(dev), lb(dev), ub(dev), mean(dev);
        x.copy_from_host(x_host, n);
        lb.copy_from_host(lb_host, n);
        ub.copy_from_host(ub_host, n);
        LBFGSBParam<Scalar> prm;
        prm.m = q->m; prm.epsilon = Scalar(q->epsilon); prm.epsilon_rel = Scalar(q->epsilon_rel); prm.past = q->past; prm.delta = Scalar(q->delta);
        prm.max_iterations = q->max_iterations; prm.max_submin = q->max_submin; prm.max_linesearch = q->max_linesearch;
        prm.min_step = Scalar(q->min_step); prm.max_step = Scalar(q->max_step); prm.ftol = Scalar(q->ftol); prm.wolfe = Scalar(q->wolfe);
        LBFGSBSolver<Scalar> solver(prm);
        BuiltinObjective<Scalar> obj(objective);
        Scalar fx = 0;
        const int niter = solver.minimize(obj, x, fx, lb, ub);
        if (free)
        {
            const long nf = tol < 0 ? solver.final_approx_free_set(x, lb, ub) : solver.final_approx_free_set(x, lb, ub, Scalar(tol));
            if (nfree_out) *nfree_out = nf;
        }
        if (mean_host) mean.copy_from_host(mean_host, n);
        box_op<Scalar>(dev, solver, n, free != 0, op, kv, V_host, mean_host ? mean : x, seed, first, out, dout, logdet_out);
        x.copy_to_host(x_host);
        if (niter_out) *niter_out = niter;
        return 0;
    });
}

}  // namespace

extern "C" int lbfgsb200_drv_box_hessian_f64(int device_ordinal, int objective, long n, const drv_param* q, double* x_host, const double* lb_host,
                                             const double* ub_host, int free, double tol, int op, int kv, const double* V_host,
                                             const double* mean_host, unsigned long long seed, unsigned first, double* out, double* dout,
                                             double* logdet_out, long* nfree_out, int* niter_out, char* err, int errlen)
{
    return box_hessian<double>(device_ordinal, objective, n, q, x_host, lb_host, ub_host, free, tol, op, kv, V_host, mean_host, seed, first, out,
                               dout, logdet_out, nfree_out, niter_out, err, errlen);
}

extern "C" int lbfgsb200_drv_box_hessian_f32(int device_ordinal, int objective, long n, const drv_param* q, float* x_host, const float* lb_host,
                                             const float* ub_host, int free, double tol, int op, int kv, const float* V_host,
                                             const float* mean_host, unsigned long long seed, unsigned first, float* out, double* dout,
                                             double* logdet_out, long* nfree_out, int* niter_out, char* err, int errlen)
{
    return box_hessian<float>(device_ordinal, objective, n, q, x_host, lb_host, ub_host, free, tol, op, kv, V_host, mean_host, seed, first, out,
                              dout, logdet_out, nfree_out, niter_out, err, errlen);
}

// The same on an explicit history: the pairs (S_host[k], Y_host[k]) added in order to a ring of size m <= 20, the free set taken from
// the LBFGS_B200_CLS_FINAL bits of cls_host (n bytes; required when free).  mean_host: n values (required for draws and densities).
extern "C" int lbfgsb200_drv_box_hist_hessian_f64(int device_ordinal, long n, int m, int npairs, const double* S_host, const double* Y_host,
                                                  int free, const unsigned char* cls_host, int op, int kv, const double* V_host,
                                                  const double* mean_host, unsigned long long seed, unsigned first, double* out, double* dout,
                                                  double* logdet_out, long* nfree_out, char* err, int errlen)
{
    return reported(err, errlen, 1, [&]() {
        require_passes<double>(op, free != 0);
        if (free && !cls_host) throw std::invalid_argument("the free set needs class bytes");
        if ((op == DRV_BOXH_SAMPLE || op == DRV_BOXH_LOG_DENSITY) && !mean_host) throw std::invalid_argument("draws and densities need a mean");
        Device& dev = device(device_ordinal);
        BoxMat<double> a;
        a.m.reset(dev, n, m);
        DeviceVector<double> s(dev), y(dev), mean(dev);
        for (int k = 0; k < npairs; k++)
        {
            s.copy_from_host(S_host + size_t(k) * n, n);
            y.copy_from_host(Y_host + size_t(k) * n, n);
            a.m.add_correction(s, y);
        }
        a.m.refresh_middle();
        if (free)
        {
            const long nf = long(a.m.free_set_classes(cls_host));
            if (nfree_out) *nfree_out = nf;
        }
        if (mean_host) mean.copy_from_host(mean_host, n);
        box_op<double>(dev, a, n, free != 0, op, kv, V_host, mean, seed, first, out, dout, logdet_out);
        return 0;
    });
}

#pragma GCC visibility pop
