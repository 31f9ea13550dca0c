// LBFGSpp/OWLQNCore.h -- the element-wise expressions and the scalar line-search core of OWL-QN (Andrew & Gao, "Scalable training of
// L1-regularized log-linear models", ICML 2007), for F(x) = f(x) + lambda |x|_1.  Compiled by g++ (the front, include/OWLQN.h) and by
// nvcc (the kernels of csrc/lbfgs_b200.cu and two_loop_gram.cuh), so that every pass that needs the pseudo-gradient forms it from x and
// g = grad f(x) with the same expression instead of storing it.  With -fmad=false on the device both sides compute the same bits.
#ifndef LBFGSPP_B200_OWLQN_CORE_H
#define LBFGSPP_B200_OWLQN_CORE_H

#include "LineSearchCore.h"

namespace LBFGSpp {

// the pseudo-gradient of F at x (paper, section 3.2): g_i + lambda sign(x_i) off zero; at x_i = 0 the one-sided derivative that
// descends, or 0 when neither does
template <typename T>
LBFGS_HD inline T owlqn_pg(T x, T g, T lam)
{
    if (x > T(0)) return g + lam;
    if (x < T(0)) return g - lam;
    const T right = g + lam;
    if (right < T(0)) return right;
    const T left = g - lam;
    if (left > T(0)) return left;
    return T(0);
}

// the orthant a search stays in (xi of the paper): sign(xp_i), or sign(-pgp_i) at xp_i = 0
template <typename T>
LBFGS_HD inline int owlqn_orthant(T xp, T pgp)
{
    if (xp > T(0)) return 1;
    if (xp < T(0)) return -1;
    return (pgp < T(0)) ? 1 : (pgp > T(0)) ? -1 : 0;
}

// pi(z; xi): z where it lies in the orthant, exactly 0 elsewhere
template <typename T>
LBFGS_HD inline T owlqn_project(T z, int xi)
{
    return ((xi > 0 && z > T(0)) || (xi < 0 && z < T(0))) ? z : T(0);
}

// one coordinate of the trial point x = pi(xp + step d; xi(xp, pgp))
template <typename T>
LBFGS_HD inline T owlqn_point(T xp, T d, T gp, T step, T lam)
{
    return owlqn_project(xp + step * d, owlqn_orthant(xp, owlqn_pg(xp, gp, lam)));
}

// the orthant constraint on a direction (paper, section 3.2): d_i = 0 where it does not oppose pg_i
template <typename T>
LBFGS_HD inline T owlqn_constrain(T d, T pg)
{
    return (d * pg >= T(0)) ? T(0) : d;
}

// Per-coordinate weights, F = f + lambda sum_i w_i |x_i|: coordinate i carries lam_i = lambda * w_i, rounded once in T
// (owlqn_lam_i).  Where lam_i > 0 the expressions above apply with lam_i in place of lambda; where lam_i == 0 (w_i = 0, or a w_i so
// small that lambda * w_i underflows) the coordinate is smooth: pg_i = g_i (owlqn_pg at lam = 0), the trial coordinate is not
// projected and the direction is not constrained.
template <typename T>
LBFGS_HD inline T owlqn_lam_i(T lam, T w)
{
    return lam * w;
}

// one coordinate of the weighted trial point: pi(xp + step d; xi) where lam_i > 0, xp + step d where lam_i == 0
template <typename T>
LBFGS_HD inline T owlqn_point_w(T xp, T d, T gp, T step, T lam_i)
{
    return lam_i > T(0) ? owlqn_point(xp, d, gp, step, lam_i) : xp + step * d;
}

// the weighted direction constraint: owlqn_constrain where lam_i > 0, d unchanged where lam_i == 0
template <typename T>
LBFGS_HD inline T owlqn_constrain_w(T d, T pg, T lam_i)
{
    return lam_i > T(0) ? owlqn_constrain(d, pg) : d;
}

// a weight the solver accepts: w >= 0, finite, and lambda * w finite (v - v is 0 exactly for a finite v, NaN otherwise)
template <typename T>
LBFGS_HD inline bool owlqn_weight_ok(T lam, T w)
{
    const T lw = owlqn_lam_i(lam, w);
    return w >= T(0) && w - w == T(0) && lw - lw == T(0);
}

// The projected backtracking search of OWL-QN as a resumable core (the shape of the four cores of LineSearchCore.h):
//     int init(opts, F0, dg0, step0)   dg0 = pg(xp).d; returns 0 or an error code
//     int advance(F, dirder)           F = F(x) at the trial, dirder = pg(xp).(x - xp); LSC_EVALUATE at the new `step`,
//                                      LSC_ACCEPT, or an error code
// Acceptance is the orthant-wise Armijo test F(x) <= F(xp) + ftol pg(xp).(x - xp); a failed trial halves the step.  The step and
// trial-count rules, and the error codes, are those of BacktrackingCore.  The accepted point is always the last trial.
template <typename Scalar>
struct OrthantBacktrackingCore
{
    Scalar step;
    LineSearchOptions<Scalar> prm;
    Scalar f0;
    int trials;

    LBFGS_HD int init(const LineSearchOptions<Scalar>& p, Scalar fx_init, Scalar dg_init, Scalar step0)
    {
        prm = p; f0 = fx_init; step = step0; trials = 0;
        if (step0 <= Scalar(0)) return LSE_STEP_NOT_POSITIVE;
        if (dg_init > Scalar(0)) return LSE_NOT_DESCENT;
        return 0;
    }
    LBFGS_HD int advance(Scalar fx, Scalar dirder)
    {
        if (!((fx > f0 + prm.ftol * dirder) || (fx != fx))) return LSC_ACCEPT;
        if (step < prm.min_step) return LSE_STEP_TOO_SMALL;
        if (step > prm.max_step) return LSE_STEP_TOO_LARGE;
        step *= Scalar(0.5);
        if (++trials >= prm.max_linesearch) return LSE_MAX_TRIALS;
        return LSC_EVALUATE;
    }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_OWLQN_CORE_H
