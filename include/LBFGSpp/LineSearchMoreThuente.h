// LBFGSpp/LineSearchMoreThuente.h -- More-Thuente strong-Wolfe search as a resumable state machine.
//
// Same decisions as the reference's LineSearchMoreThuente<Scalar>::LineSearch
// (reference include/LBFGSpp/LineSearchMoreThuente.h:213-615) including its simplifications: the search works on
// the auxiliary function psi(a) = f(a) - f(0) - a*ftol*f'(0) throughout (the switch to f itself is commented out
// in the reference, :455-462), trial values are chosen by the safeguarded cubic/quadratic rules of
// step_selection (:116-189), an un-bracketed interval is extrapolated by 1.1, a bracketed one that fails to
// shrink by 0.66 twice in a row is bisected, and while no acceptable-decrease point has been seen the next
// step is capped at 7/12 of the current one ("step_min safeguard").
// All arithmetic below is host scalar work; the vector work of each trial lives in LineSearchDriver.h.
#ifndef LBFGSPP_B200_LINE_SEARCH_MORE_THUENTE_H
#define LBFGSPP_B200_LINE_SEARCH_MORE_THUENTE_H

#include <algorithm>
#include <cmath>
#include <limits>
#include <stdexcept>

#include "LineSearchCore.h"
#include "LineSearchDriver.h"
#include "Param.h"

namespace LBFGSpp {

template <typename Scalar>
class LineSearchMoreThuente
{
public:
    typedef DeviceVector<Scalar> Vector;

    // The decisions (interval update, safeguarded cubic/quadratic step selection) live in MoreThuenteCore<Scalar>
    // (LineSearchCore.h, shared with the device-resident solve); Machine is that core, armed by a constructor that throws like the reference.
    typedef CoreMachine<Scalar, MoreThuenteCore> Machine;

    // Reference-compatible entry point (generic over the parameter struct so that LBFGSBSolver can use it):
    // `grad`/`dg` hold the gradient / slope at xp on entry.
    template <typename Foo, typename SolverParam>
    static void LineSearch(Foo& f, const SolverParam& param, const Vector& xp, const Vector& drt, const Scalar& step_max,
                           Scalar& step, Scalar& fx, Vector& grad, Scalar& dg, Vector& x)
    {
        LineSearchWorkspace<Scalar> ws(xp.device());
        const Vector gradp(grad);
        Machine search(param, fx, dg, step, step_max);
        run_line_search(search, f, xp, gradp, drt, step, fx, dg, x, grad, ws);
    }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_LINE_SEARCH_MORE_THUENTE_H
