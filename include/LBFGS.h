// LBFGS.h -- LBFGSSolver<Scalar, LineSearch>: unconstrained L-BFGS with every n-vector in H100 HBM.
//
// Drop-in for the reference's include/LBFGS.h: same class template, same constructor / minimize() /
// final_grad() / final_grad_norm() surface, same convergence rules and return values (reference LBFGS.h:78-173).
// What changes is the Vector type (LBFGSpp::DeviceVector<Scalar>, device memory) and where the arithmetic runs:
// every Eigen expression of the reference's loop body is a call into liblbfgs_b200 (include/lbfgs_b200.h).
//
//   reference (per iteration)                         here
//   m_xp = x; m_gradp = m_grad        LBFGS.h:121-122  O(1) pointer rotation, no copy
//   dg = m_grad.dot(m_drt)            LBFGS.h:123      comes out of the tail of apply_Hv (v.res)
//   line search trials                LBFGS.h:127      one fused kernel per trial (built-in objectives)
//   m_grad.norm(), x.norm()           LBFGS.h:130,137  by-products of the accepted trial's kernel
//   s, y, gate, add_correction        LBFGS.h:159-162  formed inside the first apply_Hv pass, straight into the ring slot
//   apply_Hv(m_grad, -1, m_drt)       LBFGS.h:165      Gram form: pair-forming dots + combination (2 kernels); or the
//                                                      literal 2c+1 stage kernels; or the device-resident graph
//
// The objective is any callable `Scalar f(const Vector& x, Vector& grad)` working on device vectors (taken by
// non-const reference, called once per trial, exactly like the reference).  Objectives that additionally offer
// fused_trial()/fused_value() (see LBFGSpp/DeviceObjectives.h) get the single-kernel trial.
#ifndef LBFGSPP_B200_LBFGS_H
#define LBFGSPP_B200_LBFGS_H

#include <algorithm>
#include <cmath>
#include <type_traits>
#include <vector>

#include "LBFGSpp/BFGSMat.h"
#include "LBFGSpp/DeviceVector.h"
#include "LBFGSpp/LineSearchBacktracking.h"
#include "LBFGSpp/LineSearchBracketing.h"
#include "LBFGSpp/LineSearchDriver.h"
#include "LBFGSpp/LineSearchMoreThuente.h"
#include "LBFGSpp/LineSearchNocedalWright.h"
#include "LBFGSpp/Param.h"

namespace LBFGSpp {

// A minimal host vector for code that has no Eigen: contiguous storage + the few members user functors rely on.
template <typename Scalar>
class HostVector
{
    std::vector<Scalar> m_v;

public:
    HostVector() {}
    explicit HostVector(std::ptrdiff_t n, Scalar fill = Scalar(0)) : m_v(size_t(n), fill) {}
    std::ptrdiff_t size() const { return std::ptrdiff_t(m_v.size()); }
    void resize(std::ptrdiff_t n) { m_v.resize(size_t(n)); }
    Scalar* data() { return m_v.data(); }
    const Scalar* data() const { return m_v.data(); }
    Scalar& operator[](std::ptrdiff_t i) { return m_v[size_t(i)]; }
    const Scalar& operator[](std::ptrdiff_t i) const { return m_v[size_t(i)]; }
    static HostVector Zero(std::ptrdiff_t n) { return HostVector(n, Scalar(0)); }
    static HostVector Constant(std::ptrdiff_t n, Scalar v) { return HostVector(n, v); }
};

// Wraps a host functor `Scalar f(const HostVec& x, HostVec& grad)` as a device functor (see LBFGSSolver::minimize below).
template <typename Foo, typename HostVec>
class HostFunctorAdapter
{
    Foo& m_f;
    HostVec m_x, m_g;

public:
    HostFunctorAdapter(Foo& f, std::ptrdiff_t n) : m_f(f), m_x(n), m_g(n) {}
    template <typename Scalar>
    Scalar operator()(const DeviceVector<Scalar>& x, DeviceVector<Scalar>& grad)
    {
        x.copy_to_host(m_x.data());
        const Scalar fx = m_f(static_cast<const HostVec&>(m_x), m_g);
        grad.copy_from_host(m_g.data(), x.size());
        return fx;
    }
};

namespace detail {
// objectives that can be run by the device-resident solve: they describe themselves as one of the library's kernels
template <class Foo>
class is_builtin_objective
{
    template <class F> static auto probe(int) -> decltype(std::declval<F&>().builtin_kind(), std::true_type());
    template <class> static std::false_type probe(...);
public:
    static const bool value = decltype(probe<Foo>(0))::value;
};
template <template <class> class LS> struct line_search_id;
template <> struct line_search_id<LineSearchBacktracking> { static const int value = LBFGS_B200_LS_BACKTRACKING; };
template <> struct line_search_id<LineSearchBracketing> { static const int value = LBFGS_B200_LS_BRACKETING; };
template <> struct line_search_id<LineSearchNocedalWright> { static const int value = LBFGS_B200_LS_NOCEDAL_WRIGHT; };
template <> struct line_search_id<LineSearchMoreThuente> { static const int value = LBFGS_B200_LS_MORE_THUENTE; };
template <class S> struct resident_abi;
template <> struct resident_abi<double>
{
    static lbfgs_b200_status minimize(lbfgs_b200_solver* s, int obj, const double* d0, const double* d1, const lbfgs_b200_param* p, int ls,
                                      double* x, double* tr, long long cap, lbfgs_b200_outcome* o)
    { return lbfgs_b200_solver_minimize_f64(s, obj, d0, d1, p, ls, x, tr, cap, o); }
};
template <> struct resident_abi<float>
{
    static lbfgs_b200_status minimize(lbfgs_b200_solver* s, int obj, const float* d0, const float* d1, const lbfgs_b200_param* p, int ls,
                                      float* x, double* tr, long long cap, lbfgs_b200_outcome* o)
    { return lbfgs_b200_solver_minimize_f32(s, obj, d0, d1, p, ls, x, tr, cap, o); }
};
}  // namespace detail

template <typename Scalar, template <class> class LineSearch = LineSearchNocedalWright>
class LBFGSSolver
{
public:
    typedef DeviceVector<Scalar> Vector;

private:
    const LBFGSParam<Scalar>& m_param;  // held by reference, like the reference (LBFGS.h:29)
    BFGSMat<Scalar> m_bfgs;
    std::vector<Scalar> m_fx;           // ring of past objective values (host scalars)
    Vector m_xp, m_grad, m_gradp, m_drt;
    LineSearchWorkspace<Scalar> m_ws;
    Scalar m_gnorm;
    long m_nfev;
    // device-resident solve (built-in objectives): the whole minimize() is one persistent kernel launch
    int m_resident;   // -1 automatic, 0 host-driven loop, 1 device-resident solve
    lbfgs_b200_solver* m_rsolver;
    Device* m_rdev;
    std::ptrdiff_t m_rn;
    int m_rm;
    bool m_resident_last;   // the last minimize() ran on the device-resident solver: its ring (not m_bfgs's) holds the final approximation
    double* m_trace;
    long m_trace_cap;

    template <typename Foo>
    int minimize_resident(Foo& f, Vector& x, Scalar& fx)
    {
        Device& dev = x.device();
        const std::ptrdiff_t n = x.size();
        if (m_rsolver && (m_rdev != &dev || m_rn != n || m_rm != m_param.m))
        {
            lbfgs_b200_solver_destroy(m_rsolver);
            m_rsolver = nullptr;
        }
        if (!m_rsolver)
        {
            dev.check(lbfgs_b200_solver_create(dev.ctx(), n, m_param.m, int(sizeof(Scalar)), &m_rsolver));
            m_rdev = &dev; m_rn = n; m_rm = m_param.m;
        }
        lbfgs_b200_param p;
        p.m = m_param.m; p.epsilon = m_param.epsilon; p.epsilon_rel = m_param.epsilon_rel; p.past = m_param.past; p.delta = m_param.delta;
        p.max_iterations = m_param.max_iterations; p.linesearch = m_param.linesearch; p.max_linesearch = m_param.max_linesearch;
        p.min_step = m_param.min_step; p.max_step = m_param.max_step; p.ftol = m_param.ftol; p.wolfe = m_param.wolfe;
        lbfgs_b200_outcome out;
        dev.check(detail::resident_abi<Scalar>::minimize(m_rsolver, f.builtin_kind(), f.builtin_data0(), f.builtin_data1(), &p,
                                                         detail::line_search_id<LineSearch>::value, x.data(), m_trace, m_trace_cap, &out));
        m_resident_last = true;   // final_approx_hessian() asks the solver for this solve's ring on demand
        f.add_calls(long(out.nfev));
        m_nfev = long(out.nfev);
        if (!m_grad.is_bound_to(dev)) m_grad = Vector(dev);
        m_grad.resize(n);
        dev.check(lbfgs_b200_memcpy_d2d(dev.ctx(), m_grad.data(), lbfgs_b200_solver_final_grad(m_rsolver), sizeof(Scalar) * size_t(n)));
        if (out.status != 0) ls_throw(out.status);   // the exception the line search would have thrown on the host
        fx = Scalar(out.fx);
        m_gnorm = Scalar(out.gnorm);
        return out.niter;
    }
    template <typename Foo>
    typename std::enable_if<detail::is_builtin_objective<Foo>::value, bool>::type try_resident(Foo& f, Vector& x, Scalar& fx, int& niter)
    {
        // automatic: built-in objectives run as ONE persistent kernel launch (no host round trip per trial, pair update and first
        // trial fused into the two apply_Hv passes) unless the caller pinned another apply_Hv algorithm (the literal two-loop
        // recursion or the unfused Gram form exist only in the host-driven loop)
        const int algo = m_bfgs.algorithm();
        const bool algo_ok = algo == LBFGS_B200_HV_AUTO || algo == LBFGS_B200_HV_GRAM;
        const bool want = (m_resident == 1) || (m_resident == -1 && algo_ok);
        if (!want || m_param.past > 64) return false;
        niter = minimize_resident(f, x, fx);
        return true;
    }
    template <typename Foo>
    typename std::enable_if<!detail::is_builtin_objective<Foo>::value, bool>::type try_resident(Foo&, Vector&, Scalar&, int&) { return false; }

    bool small_gradient(Scalar gg, Scalar xx)
    {
        m_gnorm = std::sqrt(gg);
        return m_gnorm <= m_param.epsilon || m_gnorm <= m_param.epsilon_rel * std::sqrt(xx);
    }

public:
    LBFGSSolver(const LBFGSParam<Scalar>& param) :
        m_param(param), m_gnorm(0), m_nfev(0), m_resident(-1), m_rsolver(nullptr), m_rdev(nullptr), m_rn(0), m_rm(0), m_resident_last(false), m_trace(nullptr),
        m_trace_cap(0)
    {
        m_param.check_param();
    }
    ~LBFGSSolver() { lbfgs_b200_solver_destroy(m_rsolver); }

    // Built-in objectives can be minimised by the device-resident solve (one persistent kernel launch, no host round trips; same
    // decisions as the host-driven loop below, sums re-associated).  Default: automatic (resident whenever the objective is built in).
    void set_device_resident(bool on) { m_resident = on ? 1 : 0; }
    void set_device_resident_auto() { m_resident = -1; }
    // resident solve only: record f of every evaluation into a host buffer (tests)
    void set_trace_buffer(double* host, long cap) { m_trace = host; m_trace_cap = cap; }
    // the device-resident solver behind the last minimize() of a built-in objective (nullptr before the first one): accounting via
    // lbfgs_b200_solver_profile()
    lbfgs_b200_solver* resident_handle() const { return m_rsolver; }

    // apply_Hv implementation selector (LBFGS_B200_HV_*); not part of the reference API
    void set_hv_algorithm(int algo) { m_bfgs.set_algorithm(algo); }

    // Minimise f starting from x (device vector, updated in place; its storage may be exchanged with an internal
    // buffer).  Returns the number of iterations; throws what the reference throws.
    template <typename Foo>
    inline int minimize(Foo& f, Vector& x, Scalar& fx)
    {
        using std::abs;
        Device& dev = x.device();
        const std::ptrdiff_t n = x.size();
        const int fpast = m_param.past;
        {
            int niter_resident = 0;
            if (try_resident(f, x, fx, niter_resident)) return niter_resident;
        }

        m_resident_last = false;
        m_bfgs.reset(dev, n, m_param.m);
        for (Vector* v : {&m_xp, &m_grad, &m_gradp, &m_drt, &m_ws.x_lo, &m_ws.grad_lo})
        {
            if (!v->is_bound_to(dev)) *v = Vector(dev);
            v->resize(n);
        }
        if (fpast > 0) m_fx.assign(size_t(fpast), Scalar(0));
        m_nfev = 0;

        // first evaluation and early exit (LBFGS.h:91-103)
        TrialValues<Scalar> at = detail::evaluate_point(f, static_cast<const Vector&>(x), m_grad);
        m_nfev++;
        fx = at.fx;
        if (fpast > 0) m_fx[0] = fx;
        if (small_gradient(at.gg, at.xx)) return 1;

        // steepest-descent start: drt = -grad, first step 1/||drt||  (LBFGS.h:106-108)
        dev.check(detail::Abi<Scalar>::scale_out(dev.ctx(), n, Scalar(-1), m_grad.data(), m_drt.data()));
        Scalar step = Scalar(1) / m_gnorm;
        Scalar dg = -at.gg;  // grad . (-grad): the same products as g.g, negated
        m_ws.gg = at.gg;
        m_ws.xx = at.xx;

        int k = 1;
        for (;;)
        {
            // the line search validates its inputs before it touches x (the reference throws from LineSearch() with x still the
            // current point): run that validation before the buffers rotate
            { typename LineSearch<Scalar>::Machine probe(m_param, fx, dg, step, m_param.max_step); (void)probe; }
            // the current point becomes the "previous" one: rotate buffers instead of copying
            m_xp.swap(x);
            m_gradp.swap(m_grad);

            const Scalar step_max = m_param.max_step;
            run_line_search<typename LineSearch<Scalar>::Machine>(f, m_param, m_xp, m_gradp, m_drt, step_max, step, fx, dg,
                                                                  x, m_grad, m_ws);
            m_nfev += m_ws.evaluations;

            if (small_gradient(m_ws.gg, m_ws.xx)) return k;                 // LBFGS.h:137-140
            if (fpast > 0)                                                   // LBFGS.h:142-149
            {
                const Scalar fxd = m_fx[size_t(k % fpast)];
                if (k >= fpast && abs(fxd - fx) <= m_param.delta * std::max(std::max(abs(fx), abs(fxd)), Scalar(1))) return k;
                m_fx[size_t(k % fpast)] = fx;
            }
            if (m_param.max_iterations != 0 && k >= m_param.max_iterations) return k;  // LBFGS.h:151-154

            // LBFGS.h:159-162 (s, y, curvature gate, add_correction) + :165 (apply_Hv) + :123 of the next pass (dg), fused
            dg = m_bfgs.update_apply_Hv_dot(x, m_xp, m_grad, m_gradp, -Scalar(1), m_drt);
            step = Scalar(1);
            k++;
        }
        return k;
    }

    // ----- host-vector compatibility mode ---------------------------------------------------------------------------
    // Existing LBFGSpp code passes host vectors (Eigen::VectorXd) and a functor over host vectors.  Any `HostVec` with
    // data() / size() / resize() (Eigen::VectorXd, LBFGSpp::HostVector<Scalar>, ...) is accepted here: x is uploaded once, every
    // objective evaluation copies x to the host, calls `f(x_host, grad_host)` and uploads grad (2n words over PCIe per call --
    // meant for small problems and for porting; the vector work of the solver itself still runs on the GPU), and the
    // solution is copied back into x.
    template <typename Foo, typename HostVec>
    typename std::enable_if<!std::is_same<HostVec, Vector>::value, int>::type minimize(Foo& f, HostVec& x, Scalar& fx)
    {
        Device& dev = Device::get_default();
        const std::ptrdiff_t n = std::ptrdiff_t(x.size());
        HostFunctorAdapter<Foo, HostVec> adapter(f, n);
        Vector xd(dev);
        xd.copy_from_host(x.data(), n);
        const int niter = minimize(adapter, xd, fx);
        xd.copy_to_host(x.data());
        return niter;
    }

    const Vector& final_grad() const { return m_grad; }
    Scalar final_grad_norm() const { return m_gnorm; }
    // final_approx_hessian() / final_approx_inverse_hessian() of the reference (LBFGS.h:192-197 -> BFGSMat.h:150-271): explicit
    // n x n matrices, only sensible for small n; returned row-major on the host.
    SmallMatrix<Scalar> final_approx_hessian() { sync_history(); return m_bfgs.dense(false); }
    SmallMatrix<Scalar> final_approx_inverse_hessian() { sync_history(); return m_bfgs.dense(true); }

private:
    // after a device-resident solve the S/Y ring lives in the solver (tiled layout): fetch a column-major copy and let m_bfgs look at it
    void sync_history()
    {
        if (!m_resident_last || !m_rsolver) return;
        lbfgs_b200_hist* h = lbfgs_b200_solver_history(m_rsolver);
        if (!h) m_rdev->check(LBFGS_B200_ERR_CUDA);
        m_bfgs.borrow(*m_rdev, h, m_rn, m_rm);
    }

public:
    // number of objective evaluations of the last minimize() call (not in the reference; used by tests/bench)
    long num_evaluations() const { return m_nfev; }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_LBFGS_H
