// owlqn_oracle.hpp -- CPU checker of OWLQNSolver (include/OWLQN.h): OWL-QN (Andrew & Gao, "Scalable training of L1-regularized
// log-linear models", ICML 2007) for F(x) = f(x) + lam |x|_1, written from the paper as a plain loop over the built-in objectives of
// oracle/objectives.hpp and the history and level-1 sums of oracle/lbfgs_oracle.hpp, with their summation modes (ORC_SUM_*).
// TEST INFRASTRUCTURE ONLY.  It shares no code with the product's front: the pseudo-gradient, the orthant, the projection, the search
// and the stopping rules are restated here.
//
//   start      f, g at x0; F0 = f + lam |x0|_1; d = -pg; dg = -pg.pg; step = 1/||pg||
//   search     x = pi(xp + step d; xi), xi = sign(xp) or sign(-pgp) at xp = 0; accept F <= F(xp) + ftol pgp.(x - xp); else step /= 2
//              with LineSearchBacktracking's min_step / max_step / max_linesearch failures; the last trial is the result
//   stop       ||pg|| <= max(epsilon, epsilon_rel ||x||), |F - F_past| <= delta max(|F|, |F_past|, 1), max_iterations
//   direction  pair (x - xp, g - gp) if s'y > eps y'y; d = -H pg (two-loop recursion); d_i = 0 where d_i pg_i >= 0; dg = pg.d < 0
#ifndef LBFGSPP_B200_TESTS_OWLQN_ORACLE_HPP
#define LBFGSPP_B200_TESTS_OWLQN_ORACLE_HPP

#include <cmath>
#include <cstring>
#include <limits>
#include <stdexcept>
#include <vector>

#include "../../oracle/lbfgs_oracle.hpp"
#include "../../oracle/objectives.hpp"

namespace orc_owlqn {

template <class T> T pseudo_grad(T x, T g, T lam)
{
    if (x > T(0)) return g + lam;
    if (x < T(0)) return g - lam;
    if (g + lam < T(0)) return g + lam;
    if (g - lam > T(0)) return g - lam;
    return T(0);
}

struct Outcome
{
    int niter;
    long nfev;
    double fx, gnorm;
};

// x: start point in, solution out (the last iterate when it throws); g: grad f at x.  nfev counts the evaluations, also on a throw.
template <class T>
Outcome minimize(int objective, const T* d0, const T* d1, long n, const orc_param& p, T lam, const orc::Blas1<T>& la, T* x, T* g, long& nfev)
{
    if (!(lam > T(0)) || !(lam <= std::numeric_limits<T>::max())) throw std::invalid_argument("'lambda' must be positive and finite");
    std::vector<T> xp(n), gp(n), d(n), pg(n), pgp(n), dx(n), ax(n), one(n, T(1)), s(n), y(n);
    orc::History<T> H(la);
    H.reset(n, p.m);
    auto l1 = [&](const T* v) { for (long i = 0; i < n; i++) ax[i] = std::fabs(v[i]); return la.dot(ax.data(), one.data(), n); };
    auto form_pg = [&](const T* xv, const T* gv, T* out) { for (long i = 0; i < n; i++) out[i] = pseudo_grad(xv[i], gv[i], lam); };
    auto converged = [&](T gnorm) { return gnorm <= T(p.epsilon) || gnorm <= T(p.epsilon_rel) * std::sqrt(la.sqnorm(x, n)); };
    std::vector<T> fpast(p.past > 0 ? p.past : 0);

    T F = orc::evaluate<T>(objective, d0, d1, n, x, g) + lam * l1(x);
    nfev = 1;
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
                x[i] = (z * xi > T(0)) ? z : T(0);
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
            if (d[i] * pg[i] >= T(0)) d[i] = T(0);
        dg = la.dot(pg.data(), d.data(), n);
        if (!(dg < T(0))) throw std::logic_error("the moving direction increases the objective function value");
        step = T(1);
    }
}

}  // namespace orc_owlqn

#endif
