// LBFGSpp/LineSearchBracketing.h -- bisection/doubling bracketing line search as a resumable state machine.
//
// Same decisions as the reference's LineSearchBracketing<Scalar>::LineSearch
// (reference include/LBFGSpp/LineSearchBracketing.h:48-128): keep an interval [lo, hi]; a failed Armijo
// test (or a non-finite f) lowers hi, a too-negative slope raises lo, a too-positive slope lowers hi; the next
// trial is 2*step while hi is infinite and the midpoint afterwards.
#ifndef LBFGSPP_B200_LINE_SEARCH_BRACKETING_H
#define LBFGSPP_B200_LINE_SEARCH_BRACKETING_H

#include <cmath>
#include <limits>
#include <stdexcept>

#include "LineSearchCore.h"
#include "LineSearchDriver.h"
#include "Param.h"

namespace LBFGSpp {

template <typename Scalar>
class LineSearchBracketing
{
public:
    typedef DeviceVector<Scalar> Vector;

    // The decisions live in BracketingCore<Scalar> (LineSearchCore.h, shared with the device-resident solve); Machine is that core, armed by a
    // constructor that throws like the reference.
    typedef CoreMachine<Scalar, BracketingCore> Machine;

    // Reference-compatible entry point (`dg` is an output only, LineSearchBracketing.h:60).
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

#endif  // LBFGSPP_B200_LINE_SEARCH_BRACKETING_H
