// LBFGSB.h -- LBFGSBSolver<Scalar, LineSearch>: bound-constrained L-BFGS-B with every n-vector in H100 HBM.
//
// Drop-in for the reference's include/LBFGSB.h (reference LBFGSB.h:116-262): same class template, constructor, minimize(f, x,
// fx, lb, ub) / final_grad() / final_grad_norm(), same convergence tests (projected-gradient infinity norm against epsilon and
// epsilon_rel*||x||_2, past/delta), same BFGS reset when the subspace direction is not a descent direction or has no room
// (reference :188-197).  Vector = LBFGSpp::DeviceVector<Scalar>.  Per iteration:
//   dir_info kernel (g.d and the largest feasible step)      reference :176-179, 68-86
//   More-Thuente line search, one fused kernel per trial      reference :203
//   proj_grad_norm kernel                                     reference :206, 62-65
//   update kernel + Gram fold + host 2c x 2c refresh          reference :235-238, BFGSMat.h:99-146
//   clamp kernel, Cauchy (LBFGSpp/Cauchy.h), SubspaceMin (LBFGSpp/SubspaceMin.h)   reference :240-250
// The bound-constrained path runs replicated per GPU (no n-sharding) and supports m <= 20.
#ifndef LBFGSPP_B200_LBFGSB_H
#define LBFGSPP_B200_LBFGSB_H

#include <algorithm>
#include <cmath>
#include <stdexcept>
#include <vector>

#include "LBFGSpp/BFGSMat.h"
#include "LBFGSpp/Cauchy.h"
#include "LBFGSpp/DeviceVector.h"
#include "LBFGSpp/LineSearchDriver.h"
#include "LBFGSpp/LineSearchMoreThuente.h"
#include "LBFGSpp/Param.h"
#include "LBFGSpp/PhaseClock.h"
#include "LBFGSpp/SubspaceMin.h"

namespace LBFGSpp {

template <typename Scalar, template <class> class LineSearch = LineSearchMoreThuente>
class LBFGSBSolver
{
public:
    typedef DeviceVector<Scalar> Vector;

private:
    const LBFGSBParam<Scalar>& m_param;
    BFGSMat<Scalar, true> m_bfgs;
    std::vector<Scalar> m_fx;
    Vector m_xp, m_grad, m_gradp, m_drt;
    LineSearchWorkspace<Scalar> m_ws;
    Scalar m_projgnorm;
    long m_nfev;

    Scalar proj_grad_norm(Device& dev, const Vector& x, const Vector& g, const Vector& lb, const Vector& ub)
    {
        Scalar v = Scalar(0);
        dev.check(detail::BoxAbi<Scalar>::proj_grad_norm(dev.ctx(), x.size(), x.data(), g.data(), lb.data(), ub.data(), &v));
        return v;
    }
    // drt = xcp - x
    void cauchy_direction(Device& dev, const Vector& x)
    {
        const Scalar* xcp = static_cast<const Scalar*>(lbfgs_b200_box_xcp(m_bfgs.box()));
        dev.check(detail::Abi<Scalar>::axpy_out(dev.ctx(), x.size(), xcp, Scalar(-1), x.data(), m_drt.data()));
    }

public:
    LBFGSBSolver(const LBFGSBParam<Scalar>& param) : m_param(param), m_projgnorm(0), m_nfev(0) { m_param.check_param(); }

    template <typename Foo>
    inline int minimize(Foo& f, Vector& x, Scalar& fx, const Vector& lb, const Vector& ub)
    {
        using std::abs;
        Device& dev = x.device();
        const std::ptrdiff_t n = x.size();
        if (lb.size() != n || ub.size() != n) throw std::invalid_argument("'lb' and 'ub' must have the same size as 'x'");
        const int fpast = m_param.past;

        dev.check(detail::BoxAbi<Scalar>::clamp(dev.ctx(), n, x.data(), lb.data(), ub.data()));   // force_bounds, :128
        m_bfgs.reset(dev, n, m_param.m);
        m_bfgs.refresh_middle();
        for (Vector* v : {&m_xp, &m_grad, &m_gradp, &m_drt, &m_ws.x_lo, &m_ws.grad_lo})
        {
            if (!v->is_bound_to(dev)) *v = Vector(dev);
            v->resize(n);
        }
        if (fpast > 0) m_fx.assign(size_t(fpast), Scalar(0));
        m_nfev = 0;

        TrialValues<Scalar> at = detail::evaluate_point(f, static_cast<const Vector&>(x), m_grad);
        m_nfev++;
        fx = at.fx;
        m_projgnorm = proj_grad_norm(dev, x, m_grad, lb, ub);
        if (fpast > 0) m_fx[0] = fx;
        if (m_projgnorm <= m_param.epsilon || m_projgnorm <= m_param.epsilon_rel * std::sqrt(at.xx)) return 1;
        m_ws.gg = at.gg;
        m_ws.xx = at.xx;

        CauchyResult<Scalar> cp = Cauchy<Scalar>::get_cauchy_point(m_bfgs, x, m_grad, lb, ub);
        cauchy_direction(dev, x);                                                   // m_drt = xcp - x, :163
        {
            const Scalar nrm = m_drt.norm();                                        // m_drt.normalize(), :164
            if (nrm > Scalar(0)) dev.check(detail::Abi<Scalar>::scale_out(dev.ctx(), n, Scalar(1) / nrm, m_drt.data(), m_drt.data()));
        }

        int k = 1;
        for (;;)
        {
            m_xp.swap(x);            // current point -> "previous" (pointer rotation instead of :174-175)
            m_gradp.swap(m_grad);

            Scalar info[2];
            {
                PhaseClock::Scope ph(dev, "dir_info");
                dev.check(detail::BoxAbi<Scalar>::dir_info(dev.ctx(), n, m_xp.data(), m_drt.data(), m_gradp.data(), lb.data(), ub.data(), info));
            }
            Scalar dg = info[0], step_max = info[1];
            if (dg >= Scalar(0) || step_max <= m_param.min_step)                    // :188-197
            {
                cauchy_direction(dev, m_xp);
                m_bfgs.reset(dev, n, m_param.m);
                m_bfgs.refresh_middle();
                dev.check(detail::BoxAbi<Scalar>::dir_info(dev.ctx(), n, m_xp.data(), m_drt.data(), m_gradp.data(), lb.data(), ub.data(), info));
                dg = info[0];
                step_max = info[1];
            }
            step_max = std::min(m_param.max_step, step_max);
            Scalar step = std::min(Scalar(1), step_max);

            {
                PhaseClock::Scope ph(dev, "line_search");
                run_line_search<typename LineSearch<Scalar>::Machine>(f, m_param, m_xp, m_gradp, m_drt, step_max, step, fx, dg, x, m_grad, m_ws);
            }
            m_nfev += m_ws.evaluations;

            m_projgnorm = proj_grad_norm(dev, x, m_grad, lb, ub);                   // :206
            if (m_projgnorm <= m_param.epsilon || m_projgnorm <= m_param.epsilon_rel * std::sqrt(m_ws.xx)) return k;
            if (fpast > 0)
            {
                const Scalar fxd = m_fx[size_t(k % fpast)];
                if (k >= fpast && abs(fxd - fx) <= m_param.delta * std::max(std::max(abs(fx), abs(fxd)), Scalar(1))) return k;
                m_fx[size_t(k % fpast)] = fx;
            }
            if (m_param.max_iterations != 0 && k >= m_param.max_iterations) return k;

            {
                PhaseClock::Scope ph(dev, "update+middle_matrix");
                if (m_bfgs.update(x, m_xp, m_grad, m_gradp)) m_bfgs.refresh_middle();   // :235-238 (+ BFGSMat.h:99-146)
            }

            dev.check(detail::BoxAbi<Scalar>::clamp(dev.ctx(), n, x.data(), lb.data(), ub.data()));   // :240
            cp = Cauchy<Scalar>::get_cauchy_point(m_bfgs, x, m_grad, lb, ub);                          // :241
            {
                PhaseClock::Scope ph(dev, "subspace_min");
                SubspaceMin<Scalar>::subspace_minimize(m_bfgs, x, m_grad, lb, ub, cp, m_param.max_submin, m_drt);   // :249-250
            }
            k++;
        }
        return k;
    }

    const Vector& final_grad() const { return m_grad; }
    Scalar final_grad_norm() const { return m_projgnorm; }
    long num_evaluations() const { return m_nfev; }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_LBFGSB_H
