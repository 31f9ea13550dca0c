// owlqn_oracle_weighted.hpp -- CPU checker of OWLQNSolver(param, lambda, w) (include/OWLQN.h): OWL-QN for F(x) = f(x) + lam sum_i w_i |x_i|,
// the loop of owlqn_oracle.hpp restated with per-coordinate weights.  TEST INFRASTRUCTURE ONLY; it shares no code with the product's
// front.
//
//   weights    lam_i = lam * w_i; a w_i < 0, not finite, or with lam * w_i not finite is refused after the first evaluation
//   start      f, g at x0; F0 = f + lam sum w_i |x0_i|; d = -pg (pg with lam_i); dg = -pg.pg; step = 1/||pg||
//   search     where lam_i > 0, x_i = pi(xp_i + step d_i; xi_i) as in owlqn_oracle.hpp; where lam_i == 0, x_i = xp_i + step d_i
//   direction  d = -H pg (two-loop recursion); d_i = 0 where lam_i > 0 and d_i pg_i >= 0; dg = pg.d < 0
#ifndef LBFGSPP_B200_TESTS_OWLQN_ORACLE_WEIGHTED_HPP
#define LBFGSPP_B200_TESTS_OWLQN_ORACLE_WEIGHTED_HPP

#include "owlqn_oracle.hpp"

namespace orc_owlqn {

// x: start point in, solution out (the last iterate when it throws); g: grad f at x; w: n weights.  nfev counts the evaluations, also
// on a throw.
template <class T>
Outcome minimize_weighted(int objective, const T* d0, const T* d1, long n, const orc_param& p, T lam, const T* w, const orc::Blas1<T>& la,
                          T* x, T* g, long& nfev)
{
    if (!(lam > T(0)) || !(lam <= std::numeric_limits<T>::max())) throw std::invalid_argument("'lambda' must be positive and finite");
    std::vector<T> xp(n), gp(n), d(n), pg(n), pgp(n), dx(n), ax(n), lw(n), s(n), y(n);
    for (long i = 0; i < n; i++) lw[i] = lam * w[i];
    orc::History<T> H(la);
    H.reset(n, p.m);
    auto l1 = [&](const T* v) { for (long i = 0; i < n; i++) ax[i] = std::fabs(v[i]); return la.dot(ax.data(), w, n); };
    auto form_pg = [&](const T* xv, const T* gv, T* out) { for (long i = 0; i < n; i++) out[i] = pseudo_grad(xv[i], gv[i], lw[i]); };
    auto converged = [&](T gnorm) { return gnorm <= T(p.epsilon) || gnorm <= T(p.epsilon_rel) * std::sqrt(la.sqnorm(x, n)); };
    std::vector<T> fpast(p.past > 0 ? p.past : 0);

    const T f0 = orc::evaluate<T>(objective, d0, d1, n, x, g);
    nfev = 1;
    for (long i = 0; i < n; i++)
        if (!(w[i] >= T(0)) || !(w[i] <= std::numeric_limits<T>::max()) || !(std::fabs(lw[i]) <= std::numeric_limits<T>::max()))
            throw std::invalid_argument("a weight is negative, not finite, or makes lambda * w overflow");
    T F = f0 + lam * l1(x);
    form_pg(x, g, pg.data());
    T pgpg = la.sqnorm(pg.data(), n);
    T gnorm = std::sqrt(pgpg);
    if (p.past > 0) fpast[0] = F;
    if (converged(gnorm)) return Outcome{1, nfev, double(F), double(gnorm)};
    for (long i = 0; i < n; i++) d[i] = -pg[i];
    T step = T(1) / gnorm, dg = -pgpg;

    for (int k = 1;; k++)
    {
        if (step <= T(0)) throw std::invalid_argument("'step' must be positive");
        if (dg > T(0)) throw std::logic_error("the moving direction increases the objective function value");
        std::memcpy(xp.data(), x, sizeof(T) * n);
        std::memcpy(gp.data(), g, sizeof(T) * n);
        const T Fp = F;
        form_pg(xp.data(), gp.data(), pgp.data());
        for (int trials = 0;;)
        {
            for (long i = 0; i < n; i++)
            {
                const T xi = xp[i] != T(0) ? (xp[i] > T(0) ? T(1) : T(-1)) : (pgp[i] < T(0) ? T(1) : pgp[i] > T(0) ? T(-1) : T(0));
                const T z = xp[i] + step * d[i];
                x[i] = (lw[i] == T(0) || z * xi > T(0)) ? z : T(0);
                dx[i] = x[i] - xp[i];
            }
            const T f = orc::evaluate<T>(objective, d0, d1, n, x, g);
            nfev++;
            F = f + lam * l1(x);
            const T dirder = la.dot(pgp.data(), dx.data(), n);
            if (F <= Fp + T(p.ftol) * dirder) break;   // false for a NaN F: the step shrinks
            if (step < T(p.min_step)) throw std::runtime_error("the line search step became smaller than the minimum value allowed");
            if (step > T(p.max_step)) throw std::runtime_error("the line search step became larger than the maximum value allowed");
            step *= T(0.5);
            if (++trials >= p.max_linesearch) throw std::runtime_error("the line search routine reached the maximum number of iterations");
        }
        form_pg(x, g, pg.data());
        gnorm = std::sqrt(la.sqnorm(pg.data(), n));
        if (converged(gnorm)) return Outcome{k, nfev, double(F), double(gnorm)};
        if (p.past > 0)
        {
            const T old = fpast[k % p.past];
            if (k >= p.past && std::fabs(old - F) <= T(p.delta) * std::max(std::max(std::fabs(F), std::fabs(old)), T(1)))
                return Outcome{k, nfev, double(F), double(gnorm)};
            fpast[k % p.past] = F;
        }
        if (p.max_iterations != 0 && k >= p.max_iterations) return Outcome{k, nfev, double(F), double(gnorm)};

        la.diff(s.data(), x, xp.data(), n);
        la.diff(y.data(), g, gp.data(), n);
        if (la.dot(s.data(), y.data(), n) > std::numeric_limits<T>::epsilon() * la.sqnorm(y.data(), n)) H.add(s.data(), y.data());
        H.apply_Hv(pg.data(), T(-1), d.data());
        for (long i = 0; i < n; i++)
            if (lw[i] != T(0) && d[i] * pg[i] >= T(0)) d[i] = T(0);
        dg = la.dot(pg.data(), d.data(), n);
        if (!(dg < T(0))) throw std::logic_error("the moving direction increases the objective function value");
        step = T(1);
    }
}

}  // namespace orc_owlqn

#endif
