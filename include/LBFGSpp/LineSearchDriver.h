// LBFGSpp/LineSearchDriver.h -- the device side of every line search, shared by the four policies.
//
// In the reference each LineSearch*.h interleaves three Eigen expressions per trial
//     x = xp + step * drt;  fx = f(x, grad);  dg = grad.dot(drt);         (e.g. LineSearchMoreThuente.h:412-414)
// with the scalar logic that picks the next step.  Here the scalar logic is a resumable core and the bookkeeping
// around one search is a SearchRecord (LineSearchCore.h, the same code the device-resident solve runs); this file
// owns the three expressions:
//   * for an objective that offers `fused_trial()` (the built-in device objectives) a trial is ONE kernel that
//     also returns g.g and x.x, so the solver never launches separate norm kernels (LBFGS.h:130,137);
//   * for any other functor it is axpy kernel -> user functor -> one 3-way reduction kernel.
// Snapshots of the best point (the reference's x_lo / grad_lo, LineSearchMoreThuente.h:393) are preallocated
// buffers exchanged by pointer swap; the initial copy `x_lo = xp, grad_lo = grad` is never made: if a search
// ends on the initial point, xp and the saved gradient are copied back instead (same values, 4n words saved
// per call in the common case).
#ifndef LBFGSPP_B200_LINE_SEARCH_DRIVER_H
#define LBFGSPP_B200_LINE_SEARCH_DRIVER_H

#include <type_traits>
#include <utility>

#include "DeviceVector.h"
#include "LineSearchCore.h"

namespace LBFGSpp {

template <typename Scalar>
struct TrialValues
{
    Scalar fx;  // f(x)
    Scalar dg;  // grad . drt
    Scalar gg;  // grad . grad
    Scalar xx;  // x . x
};

namespace detail {

// Detects `void Foo::fused_trial(const Vector& xp, const Vector& drt, Scalar step, Vector& x, Vector& grad, Scalar* out4)`
template <class Foo, class Vector, class Scalar>
class has_fused_trial
{
    template <class F>
    static auto probe(int) -> decltype(std::declval<F&>().fused_trial(std::declval<const Vector&>(), std::declval<const Vector&>(),
                                                                       Scalar(0), std::declval<Vector&>(), std::declval<Vector&>(),
                                                                       static_cast<Scalar*>(nullptr)),
                                       std::true_type());
    template <class> static std::false_type probe(...);
public:
    static const bool value = decltype(probe<Foo>(0))::value;
};

// Detects `Scalar Foo::fused_value(const Vector& x, Vector& grad, Scalar* out4)`: f, grad and the norms in one kernel
template <class Foo, class Vector, class Scalar>
class has_fused_value
{
    template <class F>
    static auto probe(int) -> decltype(std::declval<F&>().fused_value(std::declval<const Vector&>(), std::declval<Vector&>(),
                                                                       static_cast<Scalar*>(nullptr)),
                                       std::true_type());
    template <class> static std::false_type probe(...);
public:
    static const bool value = decltype(probe<Foo>(0))::value;
};

template <class Foo, class Scalar>
typename std::enable_if<has_fused_trial<Foo, DeviceVector<Scalar>, Scalar>::value, TrialValues<Scalar> >::type
evaluate_trial(Foo& f, const DeviceVector<Scalar>& xp, const DeviceVector<Scalar>& drt, Scalar step,
               DeviceVector<Scalar>& x, DeviceVector<Scalar>& grad)
{
    Scalar out[4];
    f.fused_trial(xp, drt, step, x, grad, out);
    return TrialValues<Scalar>{out[0], out[1], out[2], out[3]};
}

template <class Foo, class Scalar>
typename std::enable_if<!has_fused_trial<Foo, DeviceVector<Scalar>, Scalar>::value, TrialValues<Scalar> >::type
evaluate_trial(Foo& f, const DeviceVector<Scalar>& xp, const DeviceVector<Scalar>& drt, Scalar step,
               DeviceVector<Scalar>& x, DeviceVector<Scalar>& grad)
{
    Device& dev = xp.device();
    const std::ptrdiff_t n = xp.size();
    dev.check(Abi<Scalar>::axpy_out(dev.ctx(), n, xp.data(), step, drt.data(), x.data()));
    TrialValues<Scalar> t;
    t.fx = f(static_cast<const DeviceVector<Scalar>&>(x), grad);
    Scalar out[3];
    dev.check(Abi<Scalar>::dot3(dev.ctx(), n, grad.data(), drt.data(), x.data(), out));
    t.dg = out[0];
    t.gg = out[1];
    t.xx = out[2];
    return t;
}

// f, grad and both squared norms at a given x (first evaluation of minimize(), LBFGS.h:91-92,100)
template <class Foo, class Scalar>
typename std::enable_if<has_fused_value<Foo, DeviceVector<Scalar>, Scalar>::value, TrialValues<Scalar> >::type
evaluate_point(Foo& f, const DeviceVector<Scalar>& x, DeviceVector<Scalar>& grad)
{
    Scalar out[4];
    f.fused_value(x, grad, out);
    return TrialValues<Scalar>{out[0], Scalar(0), out[2], out[3]};
}
template <class Foo, class Scalar>
typename std::enable_if<!has_fused_value<Foo, DeviceVector<Scalar>, Scalar>::value, TrialValues<Scalar> >::type
evaluate_point(Foo& f, const DeviceVector<Scalar>& x, DeviceVector<Scalar>& grad)
{
    TrialValues<Scalar> t;
    t.fx = f(x, grad);
    Device& dev = x.device();
    Scalar out[3];
    dev.check(Abi<Scalar>::dot3(dev.ctx(), x.size(), grad.data(), grad.data(), x.data(), out));
    t.dg = Scalar(0);
    t.gg = out[1];
    t.xx = out[2];
    return t;
}

}  // namespace detail

// Scratch owned by the solver and lent to every line-search call.
template <typename Scalar>
struct LineSearchWorkspace
{
    DeviceVector<Scalar> x_lo, grad_lo;
    Scalar gg;        // in: g.g at the start point; out: g.g at the returned point
    Scalar xx;        // in: x.x at the start point; out: x.x at the returned point
    long evaluations; // trials performed by the last call
    LineSearchWorkspace() : gg(0), xx(0), evaluations(0) {}
    explicit LineSearchWorkspace(Device& dev) : x_lo(dev), grad_lo(dev), gg(0), xx(0), evaluations(0) {}
};

// Runs `search` (a policy's Machine, constructed -- and so validated -- by the caller with step, fx, dg) to completion.
//   xp, gradp : start point and its gradient (read only)
//   x, grad   : receive the accepted point and gradient (their previous contents are irrelevant)
//   step, fx, dg : in = initial step, f(xp), gradp.drt ; out = accepted step, f(x), grad.drt
template <class Machine, class Foo, class Scalar>
void run_line_search(Machine& search, Foo& f, const DeviceVector<Scalar>& xp, const DeviceVector<Scalar>& gradp,
                     const DeviceVector<Scalar>& drt, Scalar& step, Scalar& fx, Scalar& dg,
                     DeviceVector<Scalar>& x, DeviceVector<Scalar>& grad, LineSearchWorkspace<Scalar>& ws)
{
    const std::ptrdiff_t n = xp.size();
    x.resize(n);
    grad.resize(n);
    SearchRecord<Scalar> rec = {fx, dg, ws.gg, ws.xx, Scalar(0), Scalar(0), 0};   // the start point, nothing kept yet
    ws.evaluations = 0;
    for (;;)
    {
        const TrialValues<Scalar> t = detail::evaluate_trial(f, xp, drt, search.step, x, grad);
        ws.evaluations++;
        bool keep = false;
        const int action = search.advance(t.fx, t.dg, keep);
        const int next = rec.digest(action, keep, t.fx, t.dg, t.gg, t.xx, search.best_fx, search.best_dg);
        if (next >= LSE_STEP_NOT_POSITIVE) ls_throw(next);
        if (keep) { ws.x_lo.resize(n); ws.grad_lo.resize(n); ws.x_lo.swap(x); ws.grad_lo.swap(grad); }
        if (next == SEARCH_EVALUATE) continue;
        if (next == SEARCH_TAKE_KEPT)
        {
            x.swap(ws.x_lo);
            grad.swap(ws.grad_lo);
        }
        else if (next == SEARCH_TAKE_START)
        {
            x = xp;       // device copies; only when no trial ever improved on the start point
            grad = gradp;
        }
        step = search.step; fx = rec.fx; dg = rec.dg; ws.gg = rec.gg; ws.xx = rec.xx;
        return;
    }
}

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_LINE_SEARCH_DRIVER_H
