// LBFGSpp/LineSearchBacktracking.h -- backtracking line search as a resumable state machine.
//
// Same decisions as the reference's LineSearchBacktracking<Scalar>::LineSearch
// (reference include/LBFGSpp/LineSearchBacktracking.h:44-121): shrink the step by 0.5 when the Armijo test
// fails (or f is NaN), grow it by 2.1 when the curvature is still too negative, stop according to
// param.linesearch.  The vector work of each trial lives in LineSearchDriver.h.
#ifndef LBFGSPP_B200_LINE_SEARCH_BACKTRACKING_H
#define LBFGSPP_B200_LINE_SEARCH_BACKTRACKING_H

#include <stdexcept>

#include "LineSearchCore.h"
#include "LineSearchDriver.h"
#include "Param.h"

namespace LBFGSpp {

template <typename Scalar>
class LineSearchBacktracking
{
public:
    typedef DeviceVector<Scalar> Vector;

    // The decisions live in BacktrackingCore<Scalar> (LineSearchCore.h, shared with the device-resident solve); Machine is that core, armed by a
    // constructor that throws like the reference.
    typedef CoreMachine<Scalar, BacktrackingCore> Machine;

    // Reference-compatible entry point.  `grad` holds the gradient at xp on entry and at x on return;
    // `dg` is an output only (the reference recomputes grad.dot(drt) itself, LineSearchBacktracking.h:60).
    template <typename Foo>
    static void LineSearch(Foo& f, const LBFGSParam<Scalar>& param, const Vector& xp, const Vector& drt, const Scalar& step_max,
                           Scalar& step, Scalar& fx, Vector& grad, Scalar& dg, Vector& x)
    {
        LineSearchWorkspace<Scalar> ws(xp.device());
        const Vector gradp(grad);
        dg = gradp.dot(drt);
        Machine search(param, fx, dg, step, step_max);
        run_line_search(search, f, xp, gradp, drt, step, fx, dg, x, grad, ws);
    }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_LINE_SEARCH_BACKTRACKING_H
