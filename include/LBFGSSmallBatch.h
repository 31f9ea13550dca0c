// LBFGSSmallBatch.h -- LBFGSSmallBatchSolver<Scalar, LineSearch>: many independent small unconstrained problems of a built-in
// objective minimised by ONE ordinary kernel launch, one thread block per problem, the whole solve in that block's shared memory.
//
// LBFGSBatchSolver (LBFGSBatch.h) spreads every pass of a problem over all SMs, which pays off at large n; at n of a few to a few
// hundred coordinates there is nothing to spread.  This solver gives each problem a thread block of its own instead (C ABI:
// lbfgs_b200_small_minimize_*), so B is limited only by device memory and n by one block's shared memory (max_n()).  Same
// parameters, line-search policies, stopping rules and per-problem outcomes as LBFGSBatchSolver.  A problem's result does not depend
// on B or on its position in the batch; it equals LBFGSSolver's to rounding (its sums are associated within one block), not bit for bit.
#ifndef LBFGSPP_B200_LBFGS_SMALL_BATCH_H
#define LBFGSPP_B200_LBFGS_SMALL_BATCH_H

#include <limits>
#include <stdexcept>
#include <vector>

#include "LBFGSBatch.h"

namespace LBFGSpp {

namespace detail {
template <class S> struct small_batch_abi;
template <> struct small_batch_abi<double>
{
    static lbfgs_b200_status minimize(lbfgs_b200_ctx* c, int obj, const double* d0, const double* d1, int64_t ldd, int64_t n, int64_t B,
                                      const lbfgs_b200_param* p, int ls, double* X, int64_t ldx, double* G, lbfgs_b200_outcome* o)
    { return lbfgs_b200_small_minimize_f64(c, obj, d0, d1, ldd, n, B, p, ls, X, ldx, G, o); }
    static lbfgs_b200_status minimize_keep(lbfgs_b200_ctx* c, int obj, const double* d0, const double* d1, int64_t ldd, int64_t n, int64_t B,
                                           const lbfgs_b200_param* p, int ls, double* X, int64_t ldx, double* G, lbfgs_b200_outcome* o,
                                           lbfgs_b200_small_hist* h)
    { return lbfgs_b200_small_minimize_keep_f64(c, obj, d0, d1, ldd, n, B, p, ls, X, ldx, G, o, h); }
    static lbfgs_b200_status times(lbfgs_b200_small_hist* h, int inv, int64_t b0, int64_t count, int k, const double* V, int64_t ldv,
                                   int64_t ldvp, double* OUT, int64_t ldo, int64_t ldop)
    { return lbfgs_b200_small_hist_times_f64(h, inv, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop); }
    static lbfgs_b200_status diag(lbfgs_b200_small_hist* h, int inv, int64_t b0, int64_t count, double* OUT, int64_t ldo)
    { return lbfgs_b200_small_hist_diag_f64(h, inv, b0, count, OUT, ldo); }
    static lbfgs_b200_status factor_times(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, int k, const double* V, int64_t ldv, int64_t ldvp,
                                          double* OUT, int64_t ldo, int64_t ldop)
    { return lbfgs_b200_small_hist_factor_times_f64(h, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop); }
    static lbfgs_b200_status sample(lbfgs_b200_small_hist* h, uint64_t seed, uint32_t first, int64_t b0, int64_t count, int k, const double* M,
                                    int64_t ldm, double* OUT, int64_t ldo, int64_t ldop)
    { return lbfgs_b200_small_hist_sample_f64(h, seed, first, b0, count, k, M, ldm, OUT, ldo, ldop); }
    static lbfgs_b200_status logdet(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, double* out)
    { return lbfgs_b200_small_hist_logdet_f64(h, b0, count, out); }
    static lbfgs_b200_status factor_apply(lbfgs_b200_small_hist* h, int op, int64_t b0, int64_t count, int k, const double* V, int64_t ldv,
                                          int64_t ldvp, double* OUT, int64_t ldo, int64_t ldop)
    { return lbfgs_b200_small_hist_factor_apply_f64(h, op, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop); }
    static lbfgs_b200_status log_density(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, int k, const double* X, int64_t ldx, int64_t ldxp,
                                         const double* M, int64_t ldm, double* out)
    { return lbfgs_b200_small_hist_log_density_f64(h, b0, count, k, X, ldx, ldxp, M, ldm, out); }
};
template <> struct small_batch_abi<float>
{
    static lbfgs_b200_status minimize(lbfgs_b200_ctx* c, int obj, const float* d0, const float* d1, int64_t ldd, int64_t n, int64_t B,
                                      const lbfgs_b200_param* p, int ls, float* X, int64_t ldx, float* G, lbfgs_b200_outcome* o)
    { return lbfgs_b200_small_minimize_f32(c, obj, d0, d1, ldd, n, B, p, ls, X, ldx, G, o); }
    static lbfgs_b200_status minimize_keep(lbfgs_b200_ctx* c, int obj, const float* d0, const float* d1, int64_t ldd, int64_t n, int64_t B,
                                           const lbfgs_b200_param* p, int ls, float* X, int64_t ldx, float* G, lbfgs_b200_outcome* o,
                                           lbfgs_b200_small_hist* h)
    { return lbfgs_b200_small_minimize_keep_f32(c, obj, d0, d1, ldd, n, B, p, ls, X, ldx, G, o, h); }
    static lbfgs_b200_status times(lbfgs_b200_small_hist* h, int inv, int64_t b0, int64_t count, int k, const float* V, int64_t ldv,
                                   int64_t ldvp, float* OUT, int64_t ldo, int64_t ldop)
    { return lbfgs_b200_small_hist_times_f32(h, inv, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop); }
    static lbfgs_b200_status diag(lbfgs_b200_small_hist* h, int inv, int64_t b0, int64_t count, float* OUT, int64_t ldo)
    { return lbfgs_b200_small_hist_diag_f32(h, inv, b0, count, OUT, ldo); }
    static lbfgs_b200_status factor_times(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, int k, const float* V, int64_t ldv, int64_t ldvp,
                                          float* OUT, int64_t ldo, int64_t ldop)
    { return lbfgs_b200_small_hist_factor_times_f32(h, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop); }
    static lbfgs_b200_status sample(lbfgs_b200_small_hist* h, uint64_t seed, uint32_t first, int64_t b0, int64_t count, int k, const float* M,
                                    int64_t ldm, float* OUT, int64_t ldo, int64_t ldop)
    { return lbfgs_b200_small_hist_sample_f32(h, seed, first, b0, count, k, M, ldm, OUT, ldo, ldop); }
    static lbfgs_b200_status logdet(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, double* out)
    { return lbfgs_b200_small_hist_logdet_f32(h, b0, count, out); }
    static lbfgs_b200_status factor_apply(lbfgs_b200_small_hist* h, int op, int64_t b0, int64_t count, int k, const float* V, int64_t ldv,
                                          int64_t ldvp, float* OUT, int64_t ldo, int64_t ldop)
    { return lbfgs_b200_small_hist_factor_apply_f32(h, op, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop); }
    static lbfgs_b200_status log_density(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, int k, const float* X, int64_t ldx, int64_t ldxp,
                                         const float* M, int64_t ldm, double* out)
    { return lbfgs_b200_small_hist_log_density_f32(h, b0, count, k, X, ldx, ldxp, M, ldm, out); }
};
}  // namespace detail

template <typename Scalar, template <class> class LineSearch = LineSearchNocedalWright>
class LBFGSSmallBatchSolver
{
public:
    typedef DeviceVector<Scalar> Vector;

private:
    const LBFGSParam<Scalar>& m_param;
    Vector m_grad;          // B*n final gradients
    std::ptrdiff_t m_n;
    long m_B;
    bool m_keep;                    // keep_final_approx()
    lbfgs_b200_small_hist* m_hist;  // the final approximations of the last minimize(), when it kept them
    Device* m_dev;
    bool m_kept;                    // the last minimize() filled m_hist

    LBFGSSmallBatchSolver(const LBFGSSmallBatchSolver&);
    LBFGSSmallBatchSolver& operator=(const LBFGSSmallBatchSolver&);

public:
    LBFGSSmallBatchSolver(const LBFGSParam<Scalar>& param)
        : m_param(param), m_n(0), m_B(0), m_keep(false), m_hist(nullptr), m_dev(nullptr), m_kept(false)
    {
        m_param.check_param();
    }
    ~LBFGSSmallBatchSolver()
    {
        if (m_hist) lbfgs_b200_small_hist_destroy(m_hist);
    }

    // Keep every problem's final L-BFGS approximation on the device in the next minimize() calls (off by default): B*(2m*n + m + 3m^2
    // + 2) elements of device memory, see lbfgs_b200_small_hist_create.  Off, minimize() allocates nothing for it.
    void keep_final_approx(bool on) { m_keep = on; }

    // largest n a problem may have for history size m and built-in objective `objective` (LBFGS_B200_OBJ_*); 0 if none
    static std::ptrdiff_t max_n(int m, int objective) { return std::ptrdiff_t(lbfgs_b200_small_max_n(m, int(sizeof(Scalar)), objective)); }

    // X holds the B start points back to back (problem b at [b*n, (b+1)*n)) and receives the solutions.  f describes the built-in
    // objective; problem b's data vectors (if the objective has any) start at data + b*ldd (ldd = 0: shared by all problems).  Adds
    // every problem's evaluations to f's call count.
    std::vector<BatchOutcome<Scalar> > minimize(BuiltinObjective<Scalar>& f, Vector& X, long B, std::ptrdiff_t ldd = 0)
    {
        if (B < 1 || X.size() % B != 0) throw std::invalid_argument("LBFGSSmallBatchSolver: X must hold B vectors of equal length");
        Device& dev = X.device();
        const std::ptrdiff_t n = X.size() / B;
        m_grad = Vector(dev, X.size());
        m_n = n;
        m_B = B;
        m_kept = false;
        const lbfgs_b200_param p = detail::abi_param(m_param);
        std::vector<lbfgs_b200_outcome> raw((size_t)B);
        if (m_keep)
        {
            if (m_hist && (m_dev != &dev || !same_shape(n, B)))
            {
                lbfgs_b200_small_hist_destroy(m_hist);
                m_hist = nullptr;
            }
            if (!m_hist) dev.check(lbfgs_b200_small_hist_create(dev.ctx(), int64_t(n), m_param.m, int(sizeof(Scalar)), int64_t(B), &m_hist));
            m_dev = &dev;
            m_hist_n = n; m_hist_B = B; m_hist_m = m_param.m;
            dev.check(detail::small_batch_abi<Scalar>::minimize_keep(dev.ctx(), f.builtin_kind(), f.builtin_data0(), f.builtin_data1(), int64_t(ldd),
                                                                     int64_t(n), int64_t(B), &p, detail::line_search_id<LineSearch>::value, X.data(),
                                                                     int64_t(n), m_grad.data(), raw.data(), m_hist));
            m_kept = true;
        }
        else
            dev.check(detail::small_batch_abi<Scalar>::minimize(dev.ctx(), f.builtin_kind(), f.builtin_data0(), f.builtin_data1(), int64_t(ldd), int64_t(n),
                                                                int64_t(B), &p, detail::line_search_id<LineSearch>::value, X.data(), int64_t(n),
                                                                m_grad.data(), raw.data()));
        std::vector<BatchOutcome<Scalar> > out((size_t)B);
        for (size_t b = 0; b < size_t(B); b++)
        {
            out[b].status = raw[b].status; out[b].niter = raw[b].niter; out[b].nfev = long(raw[b].nfev);
            out[b].fx = Scalar(raw[b].fx); out[b].gnorm = Scalar(raw[b].gnorm); out[b].rounds = long(raw[b].rounds);
            f.add_calls(long(raw[b].nfev));
        }
        return out;
    }
    // gradient of problem b at its solution (device pointer into the solver's own B*n buffer, valid until the next minimize())
    const Scalar* final_grad(long b) const { return m_grad.data() + std::ptrdiff_t(b) * m_n; }

    // The final approximations of the last minimize() (keep_final_approx(true)) as operators, every problem in one launch: V holds
    // B*k vectors back to back, problem b's vector j at [(b*k + j)*n, ...); OUT (resized to match) receives B_b or H_b times each.
    void final_approx_hessian_times(const Vector& V, Vector& OUT) { all_times(V, OUT, false); }
    void final_approx_inverse_hessian_times(const Vector& V, Vector& OUT) { all_times(V, OUT, true); }
    // One problem b: OUT = B_b V or H_b V, V holding k = V.size()/n vectors back to back (the signatures of LBFGSBatchSolver).
    void final_approx_hessian_times(long b, const Vector& V, Vector& OUT) { one_times(b, V, OUT, false); }
    void final_approx_inverse_hessian_times(long b, const Vector& V, Vector& OUT) { one_times(b, V, OUT, true); }
    // The dense n x n matrices of problem b (LBFGSSolver::final_approx_hessian / final_approx_inverse_hessian), formed on the device
    // as the products with the columns of I.
    SmallMatrix<Scalar> final_approx_hessian(long b) { return dense(b, false); }
    SmallMatrix<Scalar> final_approx_inverse_hessian(long b) { return dense(b, true); }
    // Their diagonals, formed on the device with no products (lbfgs_b200_small_hist_diag): every problem in one launch, OUT resized
    // to B*n with problem b's at [b*n, (b + 1)*n), or problem b alone, OUT resized to n.  A problem's diagonal is the same either way.
    void final_approx_hessian_diagonal(Vector& OUT) { diagonal(0, m_B, OUT, false); }
    void final_approx_inverse_hessian_diagonal(Vector& OUT) { diagonal(0, m_B, OUT, true); }
    void final_approx_hessian_diagonal(long b, Vector& OUT) { one_diagonal(b, OUT, false); }
    void final_approx_inverse_hessian_diagonal(long b, Vector& OUT) { one_diagonal(b, OUT, true); }

    // N(x_b, H_b) for every kept problem without forming H_b (lbfgs_b200_small_hist_factor_times / _sample / _logdet, H_b = L_b L_b'):
    // OUT = L_b V in the layouts of final_approx_inverse_hessian_times; OUT = X_b + L_b z_j for the k draws first .. first+k-1 of
    // stream b (X holds the B means back to back; OUT is resized to B*k vectors, problem b's draw j at [(b*k + j)*n, ...)); log det H_b.
    // One problem b alone: the same values.  A problem whose pairs fail the positive-curvature check gets NaN.
    void final_approx_inverse_hessian_factor_times(const Vector& V, Vector& OUT)
    {
        require_kept();
        const int k = all_count(V);
        OUT.resize(V.size());
        m_dev->check(detail::small_batch_abi<Scalar>::factor_times(m_hist, 0, int64_t(m_B), k, V.data(), int64_t(m_n), int64_t(k) * m_n, OUT.data(),
                                                                   int64_t(m_n), int64_t(k) * m_n));
    }
    void final_approx_inverse_hessian_factor_times(long b, const Vector& V, Vector& OUT)
    {
        require_one(b);
        const int k = BFGSMat<Scalar>::block_count(V.size(), m_n);
        OUT.resize(V.size());
        m_dev->check(detail::small_batch_abi<Scalar>::factor_times(m_hist, int64_t(b), 1, k, V.data(), int64_t(m_n), 0, OUT.data(), int64_t(m_n), 0));
    }
    void final_approx_sample(const Vector& X, unsigned long long seed, uint32_t first, int k, Vector& OUT)
    {
        require_kept();
        if (X.size() != m_n * std::ptrdiff_t(m_B)) throw std::invalid_argument("X must hold B * n values");
        draws(0, m_B, X.data(), seed, first, k, OUT);
    }
    void final_approx_sample(long b, const Vector& mean, unsigned long long seed, uint32_t first, int k, Vector& OUT)
    {
        require_one(b);
        if (mean.size() != m_n) throw std::invalid_argument("mean must hold n values");
        draws(b, 1, mean.data(), seed, first, k, OUT);
    }
    std::vector<double> final_approx_inverse_hessian_logdet()
    {
        require_kept();
        std::vector<double> out(static_cast<size_t>(m_B));
        m_dev->check(detail::small_batch_abi<Scalar>::logdet(m_hist, 0, int64_t(m_B), out.data()));
        return out;
    }
    double final_approx_inverse_hessian_logdet(long b)
    {
        require_one(b);
        double out = 0.0;
        m_dev->check(detail::small_batch_abi<Scalar>::logdet(m_hist, int64_t(b), 1, &out));
        return out;
    }

    // Whitening and log densities under N(x_b, H_b) for every kept problem (lbfgs_b200_small_hist_factor_apply / _log_density):
    // OUT = L_b' V, L_b^-1 V or L_b^-T V in the layouts of final_approx_inverse_hessian_factor_times; log N(x; MEAN_b, H_b) for the k
    // points of each problem, X holding B*k points (problem b's point j at [(b*k + j)*n, ...)) and MEANS the B means back to back,
    // out[b*k + j].  One problem b alone: the same values.  A problem whose pairs fail the positive-curvature check gets NaN.
    void final_approx_inverse_hessian_factor_transpose_times(const Vector& V, Vector& OUT) { all_factor(LBFGS_B200_FACTOR_LT, V, OUT); }
    void final_approx_inverse_hessian_factor_solve(const Vector& V, Vector& OUT) { all_factor(LBFGS_B200_FACTOR_LINV, V, OUT); }
    void final_approx_inverse_hessian_factor_transpose_solve(const Vector& V, Vector& OUT) { all_factor(LBFGS_B200_FACTOR_LINVT, V, OUT); }
    void final_approx_inverse_hessian_factor_transpose_times(long b, const Vector& V, Vector& OUT) { one_factor(b, LBFGS_B200_FACTOR_LT, V, OUT); }
    void final_approx_inverse_hessian_factor_solve(long b, const Vector& V, Vector& OUT) { one_factor(b, LBFGS_B200_FACTOR_LINV, V, OUT); }
    void final_approx_inverse_hessian_factor_transpose_solve(long b, const Vector& V, Vector& OUT) { one_factor(b, LBFGS_B200_FACTOR_LINVT, V, OUT); }
    std::vector<double> final_approx_log_density(const Vector& MEANS, const Vector& X)
    {
        require_kept();
        if (MEANS.size() != m_n * std::ptrdiff_t(m_B)) throw std::invalid_argument("MEANS must hold B * n values");
        const int k = all_count(X);
        std::vector<double> out(static_cast<size_t>(k) * static_cast<size_t>(m_B));
        m_dev->check(detail::small_batch_abi<Scalar>::log_density(m_hist, 0, int64_t(m_B), k, X.data(), int64_t(m_n), int64_t(k) * m_n, MEANS.data(),
                                                                  int64_t(m_n), out.data()));
        return out;
    }
    std::vector<double> final_approx_log_density(long b, const Vector& mean, const Vector& X)
    {
        require_one(b);
        if (mean.size() != m_n) throw std::invalid_argument("mean must hold n values");
        const int k = BFGSMat<Scalar>::block_count(X.size(), m_n);
        std::vector<double> out(static_cast<size_t>(k));
        m_dev->check(detail::small_batch_abi<Scalar>::log_density(m_hist, int64_t(b), 1, k, X.data(), int64_t(m_n), 0, mean.data(), 0, out.data()));
        return out;
    }

private:
    void all_factor(int op, const Vector& V, Vector& OUT)
    {
        require_kept();
        const int k = all_count(V);
        OUT.resize(V.size());
        m_dev->check(detail::small_batch_abi<Scalar>::factor_apply(m_hist, op, 0, int64_t(m_B), k, V.data(), int64_t(m_n), int64_t(k) * m_n,
                                                                   OUT.data(), int64_t(m_n), int64_t(k) * m_n));
    }
    void one_factor(long b, int op, const Vector& V, Vector& OUT)
    {
        require_one(b);
        const int k = BFGSMat<Scalar>::block_count(V.size(), m_n);
        OUT.resize(V.size());
        m_dev->check(detail::small_batch_abi<Scalar>::factor_apply(m_hist, op, int64_t(b), 1, k, V.data(), int64_t(m_n), 0, OUT.data(), int64_t(m_n), 0));
    }

    std::ptrdiff_t m_hist_n = 0;
    long m_hist_B = 0;
    int m_hist_m = 0;
    bool same_shape(std::ptrdiff_t n, long B) const { return m_hist_n == n && m_hist_B == B && m_hist_m == m_param.m; }

    void require_kept() const
    {
        if (!m_kept) throw std::logic_error("LBFGSSmallBatchSolver: no final approximation kept (call keep_final_approx(true) before minimize())");
    }
    void require_one(long b) const
    {
        require_kept();
        if (b < 0 || b >= m_B) throw std::invalid_argument("LBFGSSmallBatchSolver: problem index out of range");
    }
    int all_count(const Vector& V) const
    {
        const std::ptrdiff_t per = m_n * std::ptrdiff_t(m_B);
        if (V.size() < 1 || V.size() % per != 0 || V.size() / per > std::numeric_limits<int>::max())
            throw std::invalid_argument("V.size() must be a positive multiple of B * n");
        return int(V.size() / per);
    }
    void draws(long b0, long count, const Scalar* mean, unsigned long long seed, uint32_t first, int k, Vector& OUT)
    {
        if (k < 1 || uint64_t(first) + uint64_t(k) > (uint64_t(1) << 32)) throw std::invalid_argument("need k >= 1 and first + k <= 2^32");
        OUT.resize(m_n * std::ptrdiff_t(k) * std::ptrdiff_t(count));
        m_dev->check(detail::small_batch_abi<Scalar>::sample(m_hist, seed, first, int64_t(b0), int64_t(count), k, mean, int64_t(m_n), OUT.data(),
                                                             int64_t(m_n), int64_t(k) * m_n));
    }
    void all_times(const Vector& V, Vector& OUT, bool inverse)
    {
        require_kept();
        const std::ptrdiff_t per = m_n * std::ptrdiff_t(m_B);
        if (V.size() < 1 || V.size() % per != 0 || V.size() / per > std::numeric_limits<int>::max())
            throw std::invalid_argument("V.size() must be a positive multiple of B * n");
        const int k = int(V.size() / per);
        OUT.resize(V.size());
        m_dev->check(detail::small_batch_abi<Scalar>::times(m_hist, inverse, 0, int64_t(m_B), k, V.data(), int64_t(m_n), int64_t(k) * m_n,
                                                            OUT.data(), int64_t(m_n), int64_t(k) * m_n));
    }
    void one_times(long b, const Vector& V, Vector& OUT, bool inverse)
    {
        require_kept();
        if (b < 0 || b >= m_B) throw std::invalid_argument("LBFGSSmallBatchSolver: problem index out of range");
        const int k = BFGSMat<Scalar>::block_count(V.size(), m_n);
        OUT.resize(V.size());
        m_dev->check(detail::small_batch_abi<Scalar>::times(m_hist, inverse, int64_t(b), 1, k, V.data(), int64_t(m_n), 0, OUT.data(),
                                                            int64_t(m_n), 0));
    }
    void diagonal(long b0, long count, Vector& OUT, bool inverse)
    {
        require_kept();
        OUT.resize(m_n * std::ptrdiff_t(count));
        m_dev->check(detail::small_batch_abi<Scalar>::diag(m_hist, inverse, int64_t(b0), int64_t(count), OUT.data(), int64_t(m_n)));
    }
    void one_diagonal(long b, Vector& OUT, bool inverse)
    {
        require_kept();
        if (b < 0 || b >= m_B) throw std::invalid_argument("LBFGSSmallBatchSolver: problem index out of range");
        diagonal(b, 1, OUT, inverse);
    }
    SmallMatrix<Scalar> dense(long b, bool inverse)
    {
        require_kept();
        if (b < 0 || b >= m_B) throw std::invalid_argument("LBFGSSmallBatchSolver: problem index out of range");
        const int n = int(m_n);
        std::vector<Scalar> eye(size_t(n) * size_t(n), Scalar(0));
        for (int i = 0; i < n; i++) eye[size_t(i) * size_t(n) + size_t(i)] = Scalar(1);
        Vector I(*m_dev), OUT(*m_dev);
        I.copy_from_host(eye.data(), std::ptrdiff_t(n) * n);
        one_times(b, I, OUT, inverse);
        OUT.copy_to_host(eye.data());
        SmallMatrix<Scalar> A(n, n);
        for (int j = 0; j < n; j++)   // column j of A is the product with e_j
            for (int i = 0; i < n; i++) A(i, j) = eye[size_t(j) * size_t(n) + size_t(i)];
        return A;
    }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_LBFGS_SMALL_BATCH_H
