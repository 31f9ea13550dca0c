// LBFGSpp/LineSearchNocedalWright.h -- strong-Wolfe bracket + zoom search as a resumable state machine.
//
// Same decisions as the reference's LineSearchNocedalWright<Scalar>::LineSearch
// (reference include/LBFGSpp/LineSearchNocedalWright.h:84-279, interpolation helper :30-60): a bracketing phase
// that doubles the step until the minimum is bracketed, then a zoom phase that interpolates quadratically
// between the low point (value + slope) and the high point (value).  Ignores step_max / min_step / max_step
// exactly like the reference does.
#ifndef LBFGSPP_B200_LINE_SEARCH_NOCEDAL_WRIGHT_H
#define LBFGSPP_B200_LINE_SEARCH_NOCEDAL_WRIGHT_H

#include <algorithm>
#include <cmath>
#include <stdexcept>

#include "LineSearchCore.h"
#include "LineSearchDriver.h"
#include "Param.h"

namespace LBFGSpp {

template <typename Scalar>
class LineSearchNocedalWright
{
public:
    typedef DeviceVector<Scalar> Vector;

    // The decisions live in NocedalWrightCore<Scalar> (LineSearchCore.h, shared with the device-resident solve); Machine is that core, armed by a
    // constructor that throws like the reference.
    typedef CoreMachine<Scalar, NocedalWrightCore> Machine;

    // Reference-compatible entry point: `grad`/`dg` hold the gradient / slope at xp on entry.
    template <typename Foo>
    static void LineSearch(Foo& f, const LBFGSParam<Scalar>& param, const Vector& xp, const Vector& drt, const Scalar& step_max,
                           Scalar& step, Scalar& fx, Vector& grad, Scalar& dg, Vector& x)
    {
        LineSearchWorkspace<Scalar> ws(xp.device());
        const Vector gradp(grad);
        Machine search(param, fx, dg, step, step_max);
        run_line_search(search, f, xp, gradp, drt, step, fx, dg, x, grad, ws);
    }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_LINE_SEARCH_NOCEDAL_WRIGHT_H
