// OWLQN.h -- OWLQNSolver<Scalar>: L1-regularised L-BFGS (OWL-QN; Andrew & Gao, "Scalable training of L1-regularized log-linear models",
// ICML 2007) with every n-vector in H100 HBM.  Minimises F(x) = f(x) + lambda |x|_1 for a smooth f and a scalar lambda > 0 that
// applies to every coordinate: lasso, sparse logistic regression, compressed sensing, feature selection.
//
// The loop is LBFGSSolver's host-driven loop (LBFGS.h) with the paper's three changes, all element-wise and all inside the kernels:
//   steepest-descent start       d = -pg, step = 1/||pg||                   lbfgs_b200_owlqn_sums (d written)
//   projected line search        x = pi(xp + step d; xi), orthant-wise       lbfgs_b200_owlqn_trial (built-in objectives, one kernel)
//                                Armijo F(x) <= F(xp) + ftol pgp.(x - xp),   or lbfgs_b200_owlqn_project -> f -> lbfgs_b200_owlqn_sums
//                                step halved on failure                      (any other device functor)
//   constrained direction        d = -H pg, d_i = 0 where d_i pg_i >= 0     lbfgs_b200_owlqn_update_dir (pair-forming dots + combination)
// pg is the pseudo-gradient of F (LBFGSpp/OWLQNCore.h).  It is never stored: each pass forms it from x and g = grad f(x).  The pairs
// s = x - xp, y = g - gp use the smooth gradients, behind LBFGSSolver's curvature gate.  The stopping rules are LBFGSSolver's
// (LoopRules.h) on ||pg||_2 and on the ring of past F values.
//
// Per-coordinate weights (OWLQNSolver(param, lambda, w)): F(x) = f(x) + lambda sum_i w_i |x_i|, w_i >= 0.  Coordinate i carries
// lambda * w_i rounded once; where that is 0 (w_i = 0, or so small that the product underflows) the coordinate is smooth and
// unpenalised: an intercept, a random effect, any block left out of the penalty.  The same passes read w as one more word per
// coordinate.
//
// From LBFGSParam it uses m, epsilon, epsilon_rel, past, delta, max_iterations, max_linesearch, min_step, max_step and ftol; `linesearch`
// and `wolfe` do not apply (the projected search tests sufficient decrease only).  One GPU: the vectors cannot be sharded.
#ifndef LBFGSPP_B200_OWLQN_H
#define LBFGSPP_B200_OWLQN_H

#include <cmath>
#include <limits>
#include <stdexcept>
#include <type_traits>
#include <vector>

#include "LBFGS.h"
#include "LBFGSpp/BFGSMat.h"
#include "LBFGSpp/DeviceVector.h"
#include "LBFGSpp/LineSearchCore.h"
#include "LBFGSpp/LoopRules.h"
#include "LBFGSpp/OWLQNCore.h"
#include "LBFGSpp/Param.h"

namespace LBFGSpp {

namespace detail {
template <class S> struct OwlqnAbi;
#define LBFGSPP_B200_OWLQNABI(T, SUF)                                                                                                   \
    template <> struct OwlqnAbi<T>                                                                                                      \
    {                                                                                                                                   \
        static lbfgs_b200_status trial(lbfgs_b200_ctx* c, int obj, const T* d0, const T* d1, int64_t n, const T* xp, const T* d,        \
                                       const T* gp, T step, T lam, T* x, T* g, T* o5)                                                   \
        { return lbfgs_b200_owlqn_trial_##SUF(c, obj, d0, d1, n, xp, d, gp, step, lam, x, g, o5); }                                     \
        static lbfgs_b200_status project(lbfgs_b200_ctx* c, int64_t n, const T* xp, const T* d, const T* gp, T step, T lam, T* x, T* o2) \
        { return lbfgs_b200_owlqn_project_##SUF(c, n, xp, d, gp, step, lam, x, o2); }                                                   \
        static lbfgs_b200_status sums(lbfgs_b200_ctx* c, int64_t n, const T* x, const T* g, T lam, T* d, T* o3)                         \
        { return lbfgs_b200_owlqn_sums_##SUF(c, n, x, g, lam, d, o3); }                                                                 \
        static lbfgs_b200_status update_dir(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, T eps, T lam, T* d,   \
                                            int* acc, T* dg)                                                                           \
        { return lbfgs_b200_owlqn_update_dir_##SUF(h, x, xp, g, gp, eps, lam, d, acc, dg); }                                            \
        static lbfgs_b200_status trial(lbfgs_b200_ctx* c, int obj, const T* d0, const T* d1, int64_t n, const T* xp, const T* d,        \
                                       const T* gp, T step, T lam, const T* w, T* x, T* g, T* o5)                                       \
        { return lbfgs_b200_owlqn_weighted_trial_##SUF(c, obj, d0, d1, n, xp, d, gp, step, lam, w, x, g, o5); }                         \
        static lbfgs_b200_status project(lbfgs_b200_ctx* c, int64_t n, const T* xp, const T* d, const T* gp, T step, T lam,           \
                                         const T* w, T* x, T* o2)                                                                       \
        { return lbfgs_b200_owlqn_weighted_project_##SUF(c, n, xp, d, gp, step, lam, w, x, o2); }                                       \
        static lbfgs_b200_status sums(lbfgs_b200_ctx* c, int64_t n, const T* x, const T* g, T lam, const T* w, T* d, T* o3)             \
        { return lbfgs_b200_owlqn_weighted_sums_##SUF(c, n, x, g, lam, w, d, o3); }                                                     \
        static lbfgs_b200_status update_dir(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, T eps, T lam,         \
                                            const T* w, T* d, int* acc, T* dg)                                                         \
        { return lbfgs_b200_owlqn_weighted_update_dir_##SUF(h, x, xp, g, gp, eps, lam, w, d, acc, dg); }                                \
    };
LBFGSPP_B200_OWLQNABI(double, f64)
LBFGSPP_B200_OWLQNABI(float, f32)
#undef LBFGSPP_B200_OWLQNABI

}  // namespace detail

template <typename Scalar>
class OWLQNSolver
{
public:
    typedef DeviceVector<Scalar> Vector;

private:
    const LBFGSParam<Scalar>& m_param;  // held by reference, like LBFGSSolver
    const Scalar m_lambda;
    const Vector* m_weights;            // nullptr: every coordinate weighs 1 (held by reference, like the param)
    BFGSMat<Scalar> m_bfgs;
    std::vector<Scalar> m_fx;           // ring of past values of F
    Vector m_xp, m_grad, m_gradp, m_drt;
    Scalar m_gnorm;
    long m_nfev;

    // what one trial returns: F(x), pgp.(x - xp), pg.pg, x.x
    struct Trial { Scalar F, dirder, pgpg, xx; };

    // x = pi(xp + step d; xi) with f and g at x, through one fused kernel for the built-in objectives (LBFGS.h, is_builtin_objective)...
    template <typename Foo>
    typename std::enable_if<detail::is_builtin_objective<Foo>::value, Trial>::type trial(Foo& f, Scalar step, Vector& x)
    {
        Device& dev = x.device();
        Scalar o[5];
        if (m_weights)
            dev.check(detail::OwlqnAbi<Scalar>::trial(dev.ctx(), f.builtin_kind(), f.builtin_data0(), f.builtin_data1(), x.size(),
                                                      m_xp.data(), m_drt.data(), m_gradp.data(), step, m_lambda, m_weights->data(), x.data(),
                                                      m_grad.data(), o));
        else
            dev.check(detail::OwlqnAbi<Scalar>::trial(dev.ctx(), f.builtin_kind(), f.builtin_data0(), f.builtin_data1(), x.size(),
                                                      m_xp.data(), m_drt.data(), m_gradp.data(), step, m_lambda, x.data(), m_grad.data(), o));
        f.add_calls(1);
        return Trial{o[0] + m_lambda * o[1], o[2], o[3], o[4]};
    }
    // ...or the projection, the user's functor and the sums
    template <typename Foo>
    typename std::enable_if<!detail::is_builtin_objective<Foo>::value, Trial>::type trial(Foo& f, Scalar step, Vector& x)
    {
        Device& dev = x.device();
        const std::ptrdiff_t n = x.size();
        Scalar p[2], s[3];
        if (m_weights)
            dev.check(detail::OwlqnAbi<Scalar>::project(dev.ctx(), n, m_xp.data(), m_drt.data(), m_gradp.data(), step, m_lambda,
                                                        m_weights->data(), x.data(), p));
        else
            dev.check(detail::OwlqnAbi<Scalar>::project(dev.ctx(), n, m_xp.data(), m_drt.data(), m_gradp.data(), step, m_lambda, x.data(), p));
        const Scalar fx = f(static_cast<const Vector&>(x), m_grad);
        sums(dev, x, nullptr, s);
        return Trial{fx + m_lambda * p[0], p[1], s[1], s[2]};
    }
    // {|x|_1 (weighted: sum w_i |x_i|), pg.pg, x.x} at (x, m_grad), and d = -pg when d is given; the weighted entry refuses bad weights
    void sums(Device& dev, const Vector& x, Scalar* d, Scalar* s)
    {
        if (m_weights)
            dev.check(detail::OwlqnAbi<Scalar>::sums(dev.ctx(), x.size(), x.data(), m_grad.data(), m_lambda, m_weights->data(), d, s));
        else
            dev.check(detail::OwlqnAbi<Scalar>::sums(dev.ctx(), x.size(), x.data(), m_grad.data(), m_lambda, d, s));
    }

public:
    // lambda: the weight of |x|_1; std::invalid_argument unless it is positive and finite
    OWLQNSolver(const LBFGSParam<Scalar>& param, Scalar lambda) : m_param(param), m_lambda(lambda), m_weights(nullptr), m_gnorm(0), m_nfev(0)
    {
        m_param.check_param();
        if (!(lambda > Scalar(0)) || !(lambda <= std::numeric_limits<Scalar>::max()))
            throw std::invalid_argument("'lambda' must be positive and finite");
    }
    // F = f + lambda sum_i w_i |x_i|: weights is a device vector held by reference (it must outlive the solver and keep its storage).
    // minimize() throws std::invalid_argument when its size or device differs from x's, or when a w_i is negative or not finite or
    // makes lambda * w_i overflow (checked by the first sums pass, before any trial).
    OWLQNSolver(const LBFGSParam<Scalar>& param, Scalar lambda, const Vector& weights) : OWLQNSolver(param, lambda)
    {
        m_weights = &weights;
    }

    // Minimise F = f + lambda |x|_1 from x (device vector, updated in place; its storage may be exchanged with an internal buffer).
    // f is any device functor `Scalar f(const Vector& x, Vector& grad)` returning the smooth part and its gradient; built-in objectives
    // (BuiltinObjective) take the fused projected trial.  fx receives F(x).  Returns the number of iterations; throws what
    // LineSearchBacktracking throws when the search fails, and std::logic_error when a direction does not descend.
    template <typename Foo>
    int minimize(Foo& f, Vector& x, Scalar& fx)
    {
        Device& dev = x.device();
        const std::ptrdiff_t n = x.size();
        const int fpast = m_param.past;
        const LineSearchOptions<Scalar> opts = line_search_options<Scalar>(m_param, LSK_BACKTRACKING);

        if (m_weights && (m_weights->size() != n || !m_weights->is_bound_to(dev)))
            throw std::invalid_argument("OWLQNSolver: the weights must have x's size and live on x's device");
        m_bfgs.reset(dev, n, m_param.m);
        for (Vector* v : {&m_xp, &m_grad, &m_gradp, &m_drt})
        {
            if (!v->is_bound_to(dev)) *v = Vector(dev);
            v->resize(n);
        }
        if (fpast > 0) m_fx.assign(size_t(fpast), Scalar(0));
        m_nfev = 0;

        // first evaluation, F0, d = -pg and the early exit (LBFGS.h:91-108 with pg in place of g)
        const Scalar f0 = f(static_cast<const Vector&>(x), m_grad);
        m_nfev++;
        Scalar s[3];
        sums(dev, x, m_drt.data(), s);
        fx = f0 + m_lambda * s[0];
        if (fpast > 0) m_fx[0] = fx;
        m_gnorm = std::sqrt(s[1]);
        if (gradient_converged(m_gnorm, s[2], m_param.epsilon, m_param.epsilon_rel)) return 1;
        Scalar step = Scalar(1) / m_gnorm;
        Scalar dg = -s[1];

        int k = 1;
        for (;;)
        {
            OrthantBacktrackingCore<Scalar> search;
            if (const int rc = search.init(opts, fx, dg, step)) ls_throw(rc);
            m_xp.swap(x);
            m_gradp.swap(m_grad);
            Trial t;
            for (;;)
            {
                t = trial(f, search.step, x);
                m_nfev++;
                const int action = search.advance(t.F, t.dirder);
                if (action >= LSE_STEP_NOT_POSITIVE) ls_throw(action);
                if (action == LSC_ACCEPT) break;
            }
            fx = t.F;
            m_gnorm = std::sqrt(t.pgpg);
            if (gradient_converged(m_gnorm, t.xx, m_param.epsilon, m_param.epsilon_rel) || stalled(m_fx.data(), fpast, k, fx, m_param.delta) ||
                iteration_cap(k, m_param.max_iterations))
                return k;

            int accepted = 0;
            if (m_weights)
                dev.check(detail::OwlqnAbi<Scalar>::update_dir(m_bfgs.handle(), x.data(), m_xp.data(), m_grad.data(), m_gradp.data(),
                                                               std::numeric_limits<Scalar>::epsilon(), m_lambda, m_weights->data(),
                                                               m_drt.data(), &accepted, &dg));
            else
                dev.check(detail::OwlqnAbi<Scalar>::update_dir(m_bfgs.handle(), x.data(), m_xp.data(), m_grad.data(), m_gradp.data(),
                                                               std::numeric_limits<Scalar>::epsilon(), m_lambda, m_drt.data(), &accepted, &dg));
            if (!(dg < Scalar(0))) ls_throw(LSE_NOT_DESCENT);
            step = Scalar(1);
            k++;
        }
        return k;
    }

    // grad f at the solution (the smooth part), ||pg||_2 there (pg under the weights), and the evaluations of f in the last minimize()
    const Vector& final_grad() const { return m_grad; }
    Scalar final_grad_norm() const { return m_gnorm; }
    long num_evaluations() const { return m_nfev; }
    Scalar lambda() const { return m_lambda; }
    // the per-coordinate weights, or nullptr when every coordinate weighs 1
    const Vector* weights() const { return m_weights; }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_OWLQN_H
