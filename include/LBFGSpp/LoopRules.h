// LBFGSpp/LoopRules.h -- the stopping rules and the curvature gate of the L-BFGS loop (reference LBFGS.h:137-162, LBFGSB.h:206-238),
// written once for the host loops (LBFGS.h, LBFGSB.h), the device-resident solve (persist.cuh) and the pair-commit kernel of the
// host-driven loop (lbfgs_b200.cu).  Compiled by g++ and nvcc alike: with -ffp-contract=off / -fmad=false both take the same decisions.
#ifndef LBFGSPP_B200_LOOP_RULES_H
#define LBFGSPP_B200_LOOP_RULES_H

#include "LineSearchCore.h"

namespace LBFGSpp {

// LBFGS.h:137-140: the gradient is small in absolute terms or relative to ||x|| (xx = x.x).  gnorm is the norm the loop tests: ||g||_2
// for LBFGSSolver, the projected gradient's infinity norm for LBFGSBSolver.
template <typename Scalar>
LBFGS_HD inline bool gradient_converged(Scalar gnorm, Scalar xx, Scalar epsilon, Scalar epsilon_rel)
{
    return gnorm <= epsilon || gnorm <= epsilon_rel * std::sqrt(xx);
}

// LBFGS.h:142-149: f has moved by at most delta (relative) over the last `past` iterations.  fx_hist is the caller's ring of the past
// f values (`past` slots, fx_hist[0] = f at the start point); iteration k's fx enters it unless the test stops the loop.
template <typename Scalar>
LBFGS_HD inline bool stalled(Scalar* fx_hist, int past, int k, Scalar fx, Scalar delta)
{
    using namespace lsdetail;
    if (past <= 0) return false;
    const Scalar fxd = fx_hist[k % past];
    if (k >= past && tabs(fxd - fx) <= delta * tmax(tmax(tabs(fx), tabs(fxd)), Scalar(1))) return true;
    fx_hist[k % past] = fx;
    return false;
}

// LBFGS.h:151-154 (max_iterations = 0: no cap)
LBFGS_HD inline bool iteration_cap(int k, int max_iterations) { return max_iterations != 0 && k >= max_iterations; }

// LBFGS.h:161: the pair (s, y) enters the history only when s'y > eps * y'y (eps: the machine epsilon of Scalar)
template <typename Scalar> LBFGS_HD inline bool curvature_ok(Scalar sy, Scalar yy, Scalar eps) { return sy > eps * yy; }

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_LOOP_RULES_H
