// lbfgs_oracle.hpp -- TEST INFRASTRUCTURE ONLY.  CPU restatement of the LBFGSpp hot path.
//
// This file is a checker, never a product path: only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / "--impl reference" legs may execute it.
//
// What it restates (reference @ ebef584, paths relative to the reference checkout):
//   History<T>::reset/add/apply_Hv   include/LBFGSpp/BFGSMat.h:61-97, 276-302
//   ls_backtracking                  include/LBFGSpp/LineSearchBacktracking.h:44-121
//   ls_bracketing                    include/LBFGSpp/LineSearchBracketing.h:48-128
//   ls_nocedal_wright (+quad_interp) include/LBFGSpp/LineSearchNocedalWright.h:30-60, 84-279
//   ls_more_thuente (+helpers)       include/LBFGSpp/LineSearchMoreThuente.h:34-189, 213-615
//   check_lbfgs_param                include/LBFGSpp/Param.h:191-218
//   lbfgs_minimize                   include/LBFGS.h:78-173
//
// Pinning: the reference cannot be built as-is (Eigen is absent from this image), but its
// UNMODIFIED headers do compile over oracle/minieigen; tests/test_oracle_pin.py checks that
// this restatement (ORC_SUM_SEQUENTIAL, -ffp-contract=off) reproduces that build BIT FOR BIT
// (niter, nfev, every fx of the trace, final x) and tests/golden/*.json freezes its outputs.
// The reference itself ships no golden vectors (SURVEY.md section 4).  The arithmetic of real
// Eigen (SIMD-interleaved partial sums) differs from both at rounding level; ORC_SUM_LANES8
// mimics an 8-lane Eigen redux so that sensitivity to summation order can be measured.
#ifndef LBFGS_ORACLE_HPP
#define LBFGS_ORACLE_HPP

#include <algorithm>
#include <cmath>
#include <limits>
#include <stdexcept>
#include <vector>

#include "oracle_api.h"

#ifdef _OPENMP
#include <omp.h>
#endif

namespace orc {

// ---------------------------------------------------------------------------
// level-1 kernels with a selectable summation order
// ---------------------------------------------------------------------------
template <class T>
struct Blas1
{
    int mode;     // ORC_SUM_*
    int threads;  // used by ORC_SUM_LANES8_OMP only

    explicit Blas1(int mode_ = ORC_SUM_SEQUENTIAL, int threads_ = 1) : mode(mode_), threads(threads_ < 1 ? 1 : threads_) {}

    static T dot_seq(const T* a, const T* b, long n)
    {
        T acc = T(0);
        for (long i = 0; i < n; i++) acc += a[i] * b[i];
        return acc;
    }
    // eight interleaved partial sums (what an AVX-512 double / AVX float redux does), fixed combine tree
    static T dot_lanes(const T* a, const T* b, long n)
    {
        T l[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const long nb = n & ~7L;
        for (long i = 0; i < nb; i += 8)
            for (int k = 0; k < 8; k++) l[k] += a[i + k] * b[i + k];
        T acc = ((l[0] + l[4]) + (l[2] + l[6])) + ((l[1] + l[5]) + (l[3] + l[7]));
        for (long i = nb; i < n; i++) acc += a[i] * b[i];
        return acc;
    }
    T dot(const T* a, const T* b, long n) const
    {
        if (mode == ORC_SUM_SEQUENTIAL) return dot_seq(a, b, n);
        if (mode == ORC_SUM_LANES8 || threads == 1) return dot_lanes(a, b, n);
        // contiguous chunks, one per thread slot, partials added in slot order: deterministic for a given `threads`
        std::vector<T> part(threads, T(0));
        const long chunk = ((n + threads - 1) / threads + 7) & ~7L;
#pragma omp parallel for num_threads(threads) schedule(static, 1)
        for (int t = 0; t < threads; t++)
        {
            const long lo = std::min(n, t * chunk), hi = std::min(n, lo + chunk);
            part[t] = dot_lanes(a + lo, b + lo, hi - lo);
        }
        T acc = T(0);
        for (int t = 0; t < threads; t++) acc += part[t];
        return acc;
    }
    T sqnorm(const T* a, long n) const { return dot(a, a, n); }
    T norm(const T* a, long n) const { return std::sqrt(sqnorm(a, n)); }

    // out = a + s*b   (out may alias a)
    void add_scaled(T* out, const T* a, T s, const T* b, long n) const
    {
        if (mode == ORC_SUM_LANES8_OMP && threads > 1)
        {
#pragma omp parallel for num_threads(threads) schedule(static)
            for (long i = 0; i < n; i++) out[i] = a[i] + s * b[i];
        }
        else
            for (long i = 0; i < n; i++) out[i] = a[i] + s * b[i];
    }
    // out -= s*b
    void sub_scaled(T* out, T s, const T* b, long n) const
    {
        if (mode == ORC_SUM_LANES8_OMP && threads > 1)
        {
#pragma omp parallel for num_threads(threads) schedule(static)
            for (long i = 0; i < n; i++) out[i] -= s * b[i];
        }
        else
            for (long i = 0; i < n; i++) out[i] -= s * b[i];
    }
    void scale_to(T* out, T s, const T* a, long n) const
    {
        if (mode == ORC_SUM_LANES8_OMP && threads > 1)
        {
#pragma omp parallel for num_threads(threads) schedule(static)
            for (long i = 0; i < n; i++) out[i] = s * a[i];
        }
        else
            for (long i = 0; i < n; i++) out[i] = s * a[i];
    }
    void divide(T* out, T s, long n) const
    {
        if (mode == ORC_SUM_LANES8_OMP && threads > 1)
        {
#pragma omp parallel for num_threads(threads) schedule(static)
            for (long i = 0; i < n; i++) out[i] /= s;
        }
        else
            for (long i = 0; i < n; i++) out[i] /= s;
    }
    void diff(T* out, const T* a, const T* b, long n) const
    {
        if (mode == ORC_SUM_LANES8_OMP && threads > 1)
        {
#pragma omp parallel for num_threads(threads) schedule(static)
            for (long i = 0; i < n; i++) out[i] = a[i] - b[i];
        }
        else
            for (long i = 0; i < n; i++) out[i] = a[i] - b[i];
    }
    void copy(T* out, const T* a, long n) const
    {
        if (mode == ORC_SUM_LANES8_OMP && threads > 1)
        {
#pragma omp parallel for num_threads(threads) schedule(static)
            for (long i = 0; i < n; i++) out[i] = a[i];
        }
        else
            std::copy(a, a + n, out);
    }
};

// ---------------------------------------------------------------------------
// parameters (Param.h) -- one struct for both solvers, validated like check_param()
// ---------------------------------------------------------------------------
inline void check_lbfgs_param(const orc_param& p, bool lbfgsb)
{
    if (p.m <= 0) throw std::invalid_argument("'m' must be positive");
    if (p.epsilon < 0) throw std::invalid_argument("'epsilon' must be non-negative");
    if (p.epsilon_rel < 0) throw std::invalid_argument("'epsilon_rel' must be non-negative");
    if (p.past < 0) throw std::invalid_argument("'past' must be non-negative");
    if (p.delta < 0) throw std::invalid_argument("'delta' must be non-negative");
    if (p.max_iterations < 0) throw std::invalid_argument("'max_iterations' must be non-negative");
    if (lbfgsb)
    {
        if (p.max_submin < 0) throw std::invalid_argument("'max_submin' must be non-negative");
    }
    else if (p.linesearch < 1 || p.linesearch > 3)
        throw std::invalid_argument("unsupported line search termination condition");
    if (p.max_linesearch <= 0) throw std::invalid_argument("'max_linesearch' must be positive");
    if (p.min_step < 0) throw std::invalid_argument("'min_step' must be positive");
    if (p.max_step < p.min_step) throw std::invalid_argument("'max_step' must be greater than 'min_step'");
    if (p.ftol <= 0 || p.ftol >= 0.5) throw std::invalid_argument("'ftol' must satisfy 0 < ftol < 0.5");
    if (p.wolfe <= p.ftol || p.wolfe >= 1) throw std::invalid_argument("'wolfe' must satisfy ftol < wolfe < 1");
}

inline void default_param(orc_param& p, bool lbfgsb)
{
    p.m = 6;
    p.epsilon = 1e-5;
    p.epsilon_rel = 1e-5;
    p.past = lbfgsb ? 1 : 0;
    p.delta = lbfgsb ? 1e-10 : 0.0;
    p.max_iterations = 0;
    p.linesearch = 3;
    p.max_submin = 10;
    p.max_linesearch = 20;
    p.min_step = 1e-20;
    p.max_step = 1e+20;
    p.ftol = 1e-4;
    p.wolfe = 0.9;
}

// ---------------------------------------------------------------------------
// the S/Y ring (BFGSMat, L-BFGS part)
// ---------------------------------------------------------------------------
template <class T>
struct History
{
    long n;
    int m, ncorr, ptr;
    T theta;
    std::vector<T> S, Y;  // n x m, column j at offset j*n
    std::vector<T> ys, alpha;
    Blas1<T> la;
    // Gram-form study (NOT in the reference): SY(i,j) = s_i'y_j, YY(i,j) = y_i'y_j by physical slot
    bool gram;
    std::vector<T> SY, YY;

    explicit History(const Blas1<T>& la_, bool gram_ = false) :
        n(0), m(0), ncorr(0), ptr(0), theta(1), la(la_), gram(gram_) {}

    T* s_col(int j) { return &S[size_t(j) * n]; }
    T* y_col(int j) { return &Y[size_t(j) * n]; }

    void reset(long n_, int m_)  // BFGSMat.h:61-78
    {
        n = n_;
        m = m_;
        theta = T(1);
        S.assign(size_t(n) * m, T(0));
        Y.assign(size_t(n) * m, T(0));
        ys.assign(m, T(0));
        alpha.assign(m, T(0));
        ncorr = 0;
        ptr = m;
        if (gram)
        {
            SY.assign(size_t(m) * m, T(0));
            YY.assign(size_t(m) * m, T(0));
        }
    }

    void add(const T* s, const T* y)  // BFGSMat.h:81-97
    {
        const int loc = ptr % m;
        la.copy(s_col(loc), s, n);
        la.copy(y_col(loc), y, n);
        const T sy = la.dot(s_col(loc), y_col(loc), n);
        ys[loc] = sy;
        theta = la.sqnorm(y_col(loc), n) / sy;
        if (ncorr < m) ncorr++;
        ptr = loc + 1;
        if (gram)
        {
            // slots 0..ncorr-1 are the valid ones (the ring fills 0,1,.. before it wraps)
            for (int j = 0; j < ncorr; j++)
            {
                SY[j * m + loc] = la.dot(s_col(j), y_col(loc), n);
                SY[loc * m + j] = la.dot(s_col(loc), y_col(j), n);
                YY[j * m + loc] = YY[loc * m + j] = la.dot(y_col(j), y_col(loc), n);
            }
        }
    }

    // Vector-free two-loop: the same recursion as apply_Hv() carried out on 2c coefficients, with every
    // inner product s_j'q / y_j'r expanded over the Gram matrices.  Two passes over S,Y instead of four.
    void apply_Hv_gram(const T* v, T a, T* res)
    {
        std::vector<T> bs(m, T(0)), by(m, T(0)), cs(m, T(0)), cy(m, T(0));
        std::vector<int> order;  // newest -> oldest
        int j = ptr % m;
        for (int i = 0; i < ncorr; i++)
        {
            j = (j + m - 1) % m;
            order.push_back(j);
            bs[j] = la.dot(s_col(j), v, n);
            by[j] = la.dot(y_col(j), v, n);
        }
        for (int i = 0; i < ncorr; i++)
        {
            const int jj = order[i];
            T sq = a * bs[jj];
            for (int t = 0; t < i; t++) sq -= alpha[order[t]] * SY[jj * m + order[t]];
            alpha[jj] = sq / ys[jj];
        }
        for (int i = ncorr - 1; i >= 0; i--)
        {
            const int jj = order[i];
            T yq = a * by[jj];
            for (int t = 0; t < ncorr; t++) yq -= alpha[order[t]] * YY[jj * m + order[t]];
            T yr = yq / theta;
            for (int t = ncorr - 1; t > i; t--) yr += cs[order[t]] * SY[order[t] * m + jj];
            const T beta = yr / ys[jj];
            cs[jj] = alpha[jj] - beta;
            cy[jj] = -(alpha[jj] / theta);
        }
        const T cv = a / theta;
        for (long e = 0; e < n; e++)
        {
            T acc = cv * v[e];
            for (int i = 0; i < ncorr; i++) acc += cy[order[i]] * Y[size_t(order[i]) * n + e];
            for (int i = ncorr - 1; i >= 0; i--) acc += cs[order[i]] * S[size_t(order[i]) * n + e];
            res[e] = acc;
        }
    }

    void apply_Hv(const T* v, T a, T* res)  // BFGSMat.h:276-302
    {
        la.scale_to(res, a, v, n);
        int j = ptr % m;
        for (int i = 0; i < ncorr; i++)
        {
            j = (j + m - 1) % m;
            alpha[j] = la.dot(s_col(j), res, n) / ys[j];
            la.sub_scaled(res, alpha[j], y_col(j), n);
        }
        la.divide(res, theta, n);
        for (int i = 0; i < ncorr; i++)
        {
            const T beta = la.dot(y_col(j), res, n) / ys[j];
            la.add_scaled(res, res, alpha[j] - beta, s_col(j), n);
            j = (j + 1) % m;
        }
    }
};

// ---------------------------------------------------------------------------
// line searches.  Common signature (mirrors the reference's static LineSearch()):
//   f(x_ptr, grad_ptr) -> fx;  vectors are std::vector so that snapshots swap in O(1).
// ---------------------------------------------------------------------------
template <class T> using Vec = std::vector<T>;

template <class T, class F>
void ls_backtracking(F& f, const orc_param& prm, const Blas1<T>& la, const Vec<T>& xp, const Vec<T>& drt, T /*step_max*/,
                     T& step, T& fx, Vec<T>& grad, T& dg, Vec<T>& x)
{
    const long n = long(xp.size());
    const T dec = T(0.5), inc = T(2.1);
    if (step <= T(0)) throw std::invalid_argument("'step' must be positive");
    const T fx_init = fx;
    const T dg_init = la.dot(grad.data(), drt.data(), n);
    if (dg_init > 0) throw std::logic_error("the moving direction increases the objective function value");
    const T test_decr = T(prm.ftol) * dg_init;
    T width;
    int iter;
    for (iter = 0; iter < prm.max_linesearch; iter++)
    {
        la.add_scaled(x.data(), xp.data(), step, drt.data(), n);
        fx = f(x.data(), grad.data());
        if (fx > fx_init + step * test_decr || (fx != fx))
            width = dec;
        else
        {
            dg = la.dot(grad.data(), drt.data(), n);
            if (prm.linesearch == 1) break;  // Armijo
            if (dg < T(prm.wolfe) * dg_init)
                width = inc;
            else
            {
                if (prm.linesearch == 2) break;  // regular Wolfe
                if (dg > -T(prm.wolfe) * dg_init)
                    width = dec;
                else
                    break;  // strong Wolfe
            }
        }
        if (step < T(prm.min_step)) throw std::runtime_error("the line search step became smaller than the minimum value allowed");
        if (step > T(prm.max_step)) throw std::runtime_error("the line search step became larger than the maximum value allowed");
        step *= width;
    }
    if (iter >= prm.max_linesearch) throw std::runtime_error("the line search routine reached the maximum number of iterations");
}

template <class T, class F>
void ls_bracketing(F& f, const orc_param& prm, const Blas1<T>& la, const Vec<T>& xp, const Vec<T>& drt, T /*step_max*/,
                   T& step, T& fx, Vec<T>& grad, T& dg, Vec<T>& x)
{
    const long n = long(xp.size());
    if (step <= T(0)) throw std::invalid_argument("'step' must be positive");
    const T fx_init = fx;
    const T dg_init = la.dot(grad.data(), drt.data(), n);
    if (dg_init > 0) throw std::logic_error("the moving direction increases the objective function value");
    const T test_decr = T(prm.ftol) * dg_init;
    T step_lo = 0, step_hi = std::numeric_limits<T>::infinity();
    int iter;
    for (iter = 0; iter < prm.max_linesearch; iter++)
    {
        la.add_scaled(x.data(), xp.data(), step, drt.data(), n);
        fx = f(x.data(), grad.data());
        if (fx > fx_init + step * test_decr || !std::isfinite(fx))
            step_hi = step;
        else
        {
            dg = la.dot(grad.data(), drt.data(), n);
            if (prm.linesearch == 1) break;
            if (dg < T(prm.wolfe) * dg_init)
                step_lo = step;
            else
            {
                if (prm.linesearch == 2) break;
                if (dg > -T(prm.wolfe) * dg_init)
                    step_hi = step;
                else
                    break;
            }
        }
        if (step_lo > step_hi) throw std::runtime_error("the lower bound of the bracketing interval becomes larger than the upper bound");
        if (step < T(prm.min_step)) throw std::runtime_error("the line search step became smaller than the minimum value allowed");
        if (step > T(prm.max_step)) throw std::runtime_error("the line search step became larger than the maximum value allowed");
        step = std::isinf(step_hi) ? 2 * step : step_lo / 2 + step_hi / 2;
    }
    if (iter >= prm.max_linesearch) throw std::runtime_error("the line search routine reached the maximum number of iterations");
}

template <class T>
T nw_quad_interp(T step_lo, T step_hi, T fx_lo, T fx_hi, T dg_lo)  // NocedalWright.h:30-60
{
    const T fdiff = fx_hi - fx_lo;
    const T sdiff = step_hi - step_lo;
    const T smid = (step_hi + step_lo) / T(2);
    T cand = fdiff * step_lo - smid * sdiff * dg_lo;
    cand = cand / (fdiff - sdiff * dg_lo);
    const bool bad = !std::isfinite(cand);
    const T end_dist = std::min(std::abs(cand - step_lo), std::abs(cand - step_hi));
    const bool near_end = end_dist < T(0.01) * std::abs(sdiff);
    const bool bisect = bad || (cand <= std::min(step_lo, step_hi)) || (cand >= std::max(step_lo, step_hi)) || near_end;
    return bisect ? smid : cand;
}

template <class T, class F>
void ls_nocedal_wright(F& f, const orc_param& prm, const Blas1<T>& la, const Vec<T>& xp, const Vec<T>& drt, T /*step_max*/,
                       T& step, T& fx, Vec<T>& grad, T& dg, Vec<T>& x)
{
    const long n = long(xp.size());
    if (step <= T(0)) throw std::invalid_argument("'step' must be positive");
    if (prm.linesearch != 3)
        throw std::invalid_argument("'param.linesearch' must be 'LBFGS_LINESEARCH_BACKTRACKING_STRONG_WOLFE' for LineSearchNocedalWright");
    const T expansion = T(2);
    const T fx_init = fx, dg_init = dg;
    if (dg_init > T(0)) throw std::logic_error("the moving direction increases the objective function value");
    const T test_decr = T(prm.ftol) * dg_init, test_curv = -T(prm.wolfe) * dg_init;
    T step_hi, fx_hi;
    T step_lo = T(0), fx_lo = fx_init, dg_lo = dg_init;
    Vec<T> x_lo(xp), grad_lo(grad);
    int iter = 0;
    for (;;)  // bracketing phase
    {
        la.add_scaled(x.data(), xp.data(), step, drt.data(), n);
        fx = f(x.data(), grad.data());
        dg = la.dot(grad.data(), drt.data(), n);
        if (fx - fx_init > step * test_decr || (T(0) < step_lo && fx >= fx_lo))
        {
            step_hi = step;
            fx_hi = fx;
            break;
        }
        if (std::abs(dg) <= test_curv) return;
        step_hi = step_lo;
        fx_hi = fx_lo;
        step_lo = step;
        fx_lo = fx;
        dg_lo = dg;
        x_lo.swap(x);
        grad_lo.swap(grad);
        if (dg >= T(0)) break;
        iter++;
        if (iter >= prm.max_linesearch)
        {
            x.swap(x_lo);
            grad.swap(grad_lo);
            return;
        }
        step *= expansion;
    }
    for (;;)  // zoom phase
    {
        step = nw_quad_interp(step_lo, step_hi, fx_lo, fx_hi, dg_lo);
        la.add_scaled(x.data(), xp.data(), step, drt.data(), n);
        fx = f(x.data(), grad.data());
        dg = la.dot(grad.data(), drt.data(), n);
        if (fx - fx_init > step * test_decr || fx >= fx_lo)
        {
            if (step == step_hi)
                throw std::runtime_error("the line search routine failed, possibly due to insufficient numeric precision");
            step_hi = step;
            fx_hi = fx;
        }
        else
        {
            if (std::abs(dg) <= test_curv) return;
            if (dg * (step_hi - step_lo) >= T(0))
            {
                step_hi = step_lo;
                fx_hi = fx_lo;
            }
            if (step == step_lo)
                throw std::runtime_error("the line search routine failed, possibly due to insufficient numeric precision");
            step_lo = step;
            fx_lo = fx;
            dg_lo = dg;
            x_lo.swap(x);
            grad_lo.swap(grad);
        }
        iter++;
        if (iter >= prm.max_linesearch)
        {
            if (step_lo <= T(0))
                throw std::runtime_error("the line search routine failed, unable to sufficiently decrease the function value");
            step = step_lo;
            fx = fx_lo;
            dg = dg_lo;
            x.swap(x_lo);
            grad.swap(grad_lo);
            return;
        }
    }
}

// --- More-Thuente helpers (MoreThuente.h:34-189) ---
template <class T>
T mt_quadmin_fg(T a, T b, T fa, T ga, T fb)
{
    const T ba = b - a;
    const T w = T(0.5) * ba * ga / (fa - fb + ba * ga);
    return a + w * ba;
}
template <class T>
T mt_quadmin_gg(T a, T b, T ga, T gb)
{
    const T w = ga / (ga - gb);
    return a + w * (b - a);
}
template <class T>
T mt_cubicmin(T a, T b, T fa, T fb, T ga, T gb, bool& exists)
{
    using std::abs;
    using std::sqrt;
    const T apb = a + b;
    const T ba = b - a;
    const T ba2 = ba * ba;
    const T fba = fb - fa;
    const T gba = gb - ga;
    const T z3 = (ga + gb) * ba - T(2) * fba;
    const T z2 = T(0.5) * (gba * ba2 - T(3) * apb * z3);
    const T z1 = fba * ba2 - apb * z2 - (a * apb + b * b) * z3;
    const T eps = std::numeric_limits<T>::epsilon();
    if (abs(z3) < eps * abs(z2) || abs(z3) < eps * abs(z1))
    {
        exists = (z2 * ba > T(0));
        return exists ? (-T(0.5) * z1 / z2) : b;
    }
    const T u = z2 / (T(3) * z3), v = z1 / z2;
    const T vu = v / u;
    exists = (vu <= T(1));
    if (!exists) return b;
    T r1 = T(0), r2 = T(0);
    if (abs(u) >= abs(v))
    {
        const T w = T(1) + sqrt(T(1) - vu);
        r1 = -u * w;
        r2 = -v / w;
    }
    else
    {
        const T sqrtd = sqrt(abs(u)) * sqrt(abs(v)) * sqrt(1 - u / v);
        r1 = -u - sqrtd;
        r2 = -u + sqrtd;
    }
    return (z3 * ba > T(0)) ? (std::max)(r1, r2) : (std::min)(r1, r2);
}
template <class T>
T mt_step_selection(T al, T au, T at, T fl, T fu, T ft, T gl, T gu, T gt)
{
    using std::abs;
    if (al == au) return al;
    if (!std::isfinite(ft) || !std::isfinite(gt)) return (al + at) / T(2);
    bool ac_exists;
    const T ac = mt_cubicmin(al, at, fl, ft, gl, gt, ac_exists);
    const T aq = mt_quadmin_fg(al, at, fl, gl, ft);
    if (ft > fl)  // case 1
    {
        if (!ac_exists) return aq;
        return (abs(ac - al) < abs(aq - al)) ? ac : ((aq + ac) / T(2));
    }
    const T as = mt_quadmin_gg(al, at, gl, gt);
    if (gt * gl < T(0))  // case 2
        return (abs(ac - at) >= abs(as - at)) ? ac : as;
    const T deltal = T(1.1), deltau = T(0.66);
    if (abs(gt) < abs(gl))  // case 3
    {
        const T res = (ac_exists && (ac - at) * (at - al) > T(0) && abs(ac - at) < abs(as - at)) ? ac : as;
        return (at > al) ? (std::min)(at + deltau * (au - at), res) : (std::max)(at + deltau * (au - at), res);
    }
    if (!std::isfinite(au) || !std::isfinite(fu) || !std::isfinite(gu)) return at + deltal * (at - al);  // case 4
    bool ae_exists;
    const T ae = mt_cubicmin(at, au, ft, fu, gt, gu, ae_exists);
    return (at > al) ? (std::min)(at + deltau * (au - at), ae) : (std::max)(at + deltau * (au - at), ae);
}

template <class T, class F>
void ls_more_thuente(F& f, const orc_param& prm, const Blas1<T>& la, const Vec<T>& xp, const Vec<T>& drt, T step_max,
                     T& step, T& fx, Vec<T>& grad, T& dg, Vec<T>& x)
{
    using std::abs;
    const long n = long(xp.size());
    const T step_min = T(prm.min_step);
    if (step <= T(0)) throw std::invalid_argument("'step' must be positive");
    if (step < step_min) throw std::invalid_argument("'step' is smaller than 'param.min_step'");
    if (step > step_max) throw std::invalid_argument("'step' exceeds 'step_max'");
    const T fx_init = fx, dg_init = dg;
    if (dg_init >= T(0)) throw std::logic_error("the moving direction does not decrease the objective function value");
    const T test_decr = T(prm.ftol) * dg_init, test_curv = -T(prm.wolfe) * dg_init;
    const T Inf = std::numeric_limits<T>::infinity();
    T I_lo = T(0), I_hi = Inf;
    T fI_lo = T(0), fI_hi = Inf;
    T gI_lo = (T(1) - T(prm.ftol)) * dg_init, gI_hi = Inf;
    T psiI_lo = fI_lo;
    Vec<T> x_lo(xp), grad_lo(grad);
    T fx_lo = fx_init, dg_lo = dg_init;
    bool bracketed = false;
    const bool f_is_psi = true;  // the reference's stage switch is commented out (MoreThuente.h:455-462)
    bool use_step_min_safeguard = (step_min > T(0));
    T I_width = Inf, I_width_prev = Inf;
    int I_shrink_fail_count = 0;
    const T delta_max = T(1.1), delta_min = T(7) / T(12), shrink = T(0.66);
    int iter;
    for (iter = 0; iter < prm.max_linesearch; iter++)
    {
        la.add_scaled(x.data(), xp.data(), step, drt.data(), n);
        fx = f(x.data(), grad.data());
        dg = la.dot(grad.data(), drt.data(), n);
        const T psit = fx - fx_init - step * test_decr;
        const T dpsit = dg - test_decr;
        if (psit <= T(0) && abs(dg) <= test_curv) return;
        if (step <= step_min && (psit > T(0) || dpsit >= T(0))) return;
        if (step >= step_max && (psit <= T(0) && dpsit < T(0))) return;
        const T ft = f_is_psi ? psit : fx;
        const T gt = f_is_psi ? dpsit : dg;
        if (use_step_min_safeguard && (psit <= T(0) && dpsit < T(0))) use_step_min_safeguard = false;
        T new_step;
        const bool in_case_2 = (psit <= psiI_lo) && (dpsit * (I_lo - step) > T(0));
        if (in_case_2)
            new_step = (std::min)(step_max, step + delta_max * (step - I_lo));
        else
        {
            new_step = mt_step_selection(I_lo, I_hi, step, fI_lo, fI_hi, ft, gI_lo, gI_hi, gt);
            new_step = (std::max)(new_step, step_min);
            new_step = (std::min)(new_step, step_max);
            if (use_step_min_safeguard)
            {
                const T lower = step_min;
                const T upper = (std::max)(step_min, delta_min * step);
                new_step = (std::max)(new_step, lower);
                new_step = (std::min)(new_step, upper);
            }
        }
        if (psit > psiI_lo)
        {
            I_hi = step;
            fI_hi = ft;
            gI_hi = gt;
        }
        else
        {
            if (!in_case_2)
            {
                I_hi = I_lo;
                fI_hi = fI_lo;
                gI_hi = gI_lo;
            }
            I_lo = step;
            fI_lo = ft;
            gI_lo = gt;
            psiI_lo = psit;
            x_lo.swap(x);
            grad_lo.swap(grad);
            fx_lo = fx;
            dg_lo = dg;
        }
        if (!bracketed && !in_case_2)
        {
            const T I_left = (std::min)(I_lo, I_hi), I_right = (std::max)(I_lo, I_hi);
            bracketed = (I_left >= step_min && I_right <= step_max);
        }
        if (bracketed)
        {
            I_width_prev = I_width;
            I_width = abs(I_hi - I_lo);
            if (I_width_prev < Inf && I_width > shrink * I_width_prev)
                I_shrink_fail_count += 1;
            else
                I_shrink_fail_count = 0;
            if (I_shrink_fail_count >= 2)
            {
                new_step = (I_lo + I_hi) / T(2);
                I_shrink_fail_count = 0;
            }
        }
        step = new_step;
    }
    if (iter >= prm.max_linesearch)
    {
        step = I_lo;
        fx = fx_lo;
        dg = dg_lo;
        x.swap(x_lo);
        grad.swap(grad_lo);
    }
}

// ---------------------------------------------------------------------------
// the unconstrained solver (LBFGS.h:78-173)
// ---------------------------------------------------------------------------
template <class T>
struct LbfgsOutcome
{
    int niter;
    T fx, gnorm;
    Vec<T> grad;
};

template <class T, class F>
LbfgsOutcome<T> lbfgs_minimize(F& f, const orc_param& prm, int ls, const Blas1<T>& la, Vec<T>& x, bool gram = false)
{
    using std::abs;
    check_lbfgs_param(prm, false);
    const long n = long(x.size());
    History<T> hist(la, gram);
    hist.reset(n, prm.m);
    Vec<T> xp(n), grad(n), gradp(n), drt(n), fxs(prm.past > 0 ? prm.past : 0);
    LbfgsOutcome<T> out;
    const int fpast = prm.past;

    T fx = f(x.data(), grad.data());
    T gnorm = la.norm(grad.data(), n);
    if (fpast > 0) fxs[0] = fx;
    auto finish = [&](int k) {
        out.niter = k;
        out.fx = fx;
        out.gnorm = gnorm;
        out.grad.swap(grad);
        return out;
    };
    if (gnorm <= T(prm.epsilon) || gnorm <= T(prm.epsilon_rel) * la.norm(x.data(), n)) return finish(1);

    la.scale_to(drt.data(), T(-1), grad.data(), n);  // drt = -grad (exact, same bits as unary minus)
    T step = T(1) / la.norm(drt.data(), n);
    const T eps = std::numeric_limits<T>::epsilon();
    Vec<T> s(n), y(n);

    int k = 1;
    for (;;)
    {
        la.copy(xp.data(), x.data(), n);
        la.copy(gradp.data(), grad.data(), n);
        T dg = la.dot(grad.data(), drt.data(), n);
        const T step_max = T(prm.max_step);
        switch (ls)
        {
        case ORC_LS_BACKTRACKING: ls_backtracking(f, prm, la, xp, drt, step_max, step, fx, grad, dg, x); break;
        case ORC_LS_BRACKETING: ls_bracketing(f, prm, la, xp, drt, step_max, step, fx, grad, dg, x); break;
        case ORC_LS_NOCEDAL_WRIGHT: ls_nocedal_wright(f, prm, la, xp, drt, step_max, step, fx, grad, dg, x); break;
        case ORC_LS_MORE_THUENTE: ls_more_thuente(f, prm, la, xp, drt, step_max, step, fx, grad, dg, x); break;
        default: throw std::invalid_argument("unknown line search id");
        }
        gnorm = la.norm(grad.data(), n);
        if (gnorm <= T(prm.epsilon) || gnorm <= T(prm.epsilon_rel) * la.norm(x.data(), n)) return finish(k);
        if (fpast > 0)
        {
            const T fxd = fxs[k % fpast];
            if (k >= fpast && abs(fxd - fx) <= T(prm.delta) * std::max(std::max(abs(fx), abs(fxd)), T(1))) return finish(k);
            fxs[k % fpast] = fx;
        }
        if (prm.max_iterations != 0 && k >= prm.max_iterations) return finish(k);

        la.diff(s.data(), x.data(), xp.data(), n);
        la.diff(y.data(), grad.data(), gradp.data(), n);
        if (la.dot(s.data(), y.data(), n) > eps * la.sqnorm(y.data(), n)) hist.add(s.data(), y.data());
        if (gram)
            hist.apply_Hv_gram(grad.data(), -T(1), drt.data());
        else
            hist.apply_Hv(grad.data(), -T(1), drt.data());
        step = T(1);
        k++;
    }
}

template <class T, class F>
LbfgsOutcome<T> lbfgs_minimize_gram(F& f, const orc_param& prm, int ls, const Blas1<T>& la, Vec<T>& x)
{
    return lbfgs_minimize<T>(f, prm, ls, la, x, true);
}

}  // namespace orc
#endif
