// LBFGSpp/DeviceObjectives.h -- objective functors whose f/grad run on the GPU.
//
// The reference's users write `Scalar operator()(const Vector& x, Vector& grad)` over host vectors
// (reference LBFGS.h:69-71; examples/example-rosenbrock.cpp:15-27).  On the GPU front x and grad are device
// vectors, so an objective is a functor that launches kernels.  BuiltinObjective wraps the four objective kernels
// compiled into liblbfgs_b200 (the reference's example functions + the SPD quadratic of the benchmark configs) and
// exposes, besides operator(), the two fused entry points LineSearchDriver.h looks for:
//   fused_trial(xp, drt, step, x, grad, out4)  x = xp + step*drt; grad = f'(x); out4 = {f, grad.drt, grad.grad, x.x}
//   fused_value(x, grad, out4)                 grad = f'(x); out4 = {f, -, grad.grad, x.x}
// A user-written device objective only needs operator(); PlainObjective below shows that path (and tests use it to
// exercise the unfused axpy -> functor -> dot3 route).
#ifndef LBFGSPP_B200_DEVICE_OBJECTIVES_H
#define LBFGSPP_B200_DEVICE_OBJECTIVES_H

#include "DeviceVector.h"

namespace LBFGSpp {

template <typename Scalar>
class BuiltinObjective
{
    typedef DeviceVector<Scalar> Vector;
    int m_kind;
    const Scalar* m_data0;
    const Scalar* m_data1;
    long m_ncalls;

public:
    // kind: LBFGS_B200_OBJ_*; data0/data1: device pointers some kinds need (QUAD_TRIDIAG: diagonal, right-hand side)
    explicit BuiltinObjective(int kind, const Scalar* data0 = nullptr, const Scalar* data1 = nullptr) :
        m_kind(kind), m_data0(data0), m_data1(data1), m_ncalls(0) {}

    long ncalls() const { return m_ncalls; }
    // descriptor used by the device-resident solve (LBFGSSolver picks it when these members exist)
    int builtin_kind() const { return m_kind; }
    const Scalar* builtin_data0() const { return m_data0; }
    const Scalar* builtin_data1() const { return m_data1; }
    void add_calls(long k) { m_ncalls += k; }

    Scalar operator()(const Vector& x, Vector& grad)
    {
        Scalar out[4];
        fused_value(x, grad, out);
        return out[0];
    }
    void fused_value(const Vector& x, Vector& grad, Scalar* out4)
    {
        grad.resize(x.size());
        Device& dev = x.device();
        dev.check(detail::Abi<Scalar>::objective(dev.ctx(), m_kind, m_data0, m_data1, x.size(), x.data(), grad.data(), out4));
        m_ncalls++;
    }
    void fused_trial(const Vector& xp, const Vector& drt, Scalar step, Vector& x, Vector& grad, Scalar* out4)
    {
        Device& dev = xp.device();
        dev.check(detail::Abi<Scalar>::trial(dev.ctx(), m_kind, m_data0, m_data1, xp.size(), xp.data(), drt.data(), step,
                                             x.data(), grad.data(), out4));
        m_ncalls++;
    }
};

// The same objectives without the fused hooks: what a user-supplied device functor looks like to the solver.
template <typename Scalar>
class PlainObjective
{
    typedef DeviceVector<Scalar> Vector;
    int m_kind;
    const Scalar* m_data0;
    const Scalar* m_data1;
    long m_ncalls;

public:
    explicit PlainObjective(int kind, const Scalar* data0 = nullptr, const Scalar* data1 = nullptr) :
        m_kind(kind), m_data0(data0), m_data1(data1), m_ncalls(0) {}
    long ncalls() const { return m_ncalls; }
    Scalar operator()(const Vector& x, Vector& grad)
    {
        grad.resize(x.size());
        Device& dev = x.device();
        Scalar out[4];
        dev.check(detail::Abi<Scalar>::objective(dev.ctx(), m_kind, m_data0, m_data1, x.size(), x.data(), grad.data(), out));
        m_ncalls++;
        return out[0];
    }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_DEVICE_OBJECTIVES_H
