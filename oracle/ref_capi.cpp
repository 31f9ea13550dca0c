// ref_capi.cpp -- TEST INFRASTRUCTURE ONLY.
//
// C-ABI wrapper ("ref_" prefix of oracle_api.h) around the UNMODIFIED reference headers.
// Compiled ONLY when a reference checkout is named (make -C oracle ref REF=<LBFGSpp checkout>):
//     g++ -I oracle/minieigen -I $(REF)/include ... -o oracle/_ref/libref_lbfgspp.so
// No reference source is copied: <LBFGS.h>/<LBFGSB.h> are included from where they lie.
// Arithmetic comes from oracle/minieigen (strictly sequential sums), control flow is the
// reference's own.  Used to (1) pin the restatement bit-for-bit and (2) generate
// tests/golden/*.json (tests/golden/make_golden.py).
#include <chrono>
#include <cstring>
#include <stdexcept>

#include <Eigen/Core>
#include <LBFGS.h>
#include <LBFGSB.h>

#include "objectives.hpp"
#include "oracle_api.h"

namespace {

template <class T>
struct Functor
{
    typedef Eigen::Matrix<T, Eigen::Dynamic, 1> Vec;
    int objective;
    const T* d0;
    const T* d1;
    long n;
    long nfev;
    double* trace;
    long cap;
    Functor(int o, const T* a, const T* b, long n_, double* tr, long cap_) :
        objective(o), d0(a), d1(b), n(n_), nfev(0), trace(tr), cap(cap_) {}
    T operator()(const Vec& x, Vec& g)
    {
        const T fx = orc::evaluate<T>(objective, d0, d1, n, x, g);
        if (trace && nfev < cap) trace[nfev] = double(fx);
        nfev++;
        return fx;
    }
};

template <class T, class P>
void fill_common(P& p, const orc_param* q)
{
    p.m = q->m;
    p.epsilon = T(q->epsilon);
    p.epsilon_rel = T(q->epsilon_rel);
    p.past = q->past;
    p.delta = T(q->delta);
    p.max_iterations = q->max_iterations;
    p.max_linesearch = q->max_linesearch;
    p.min_step = T(q->min_step);
    p.max_step = T(q->max_step);
    p.ftol = T(q->ftol);
    p.wolfe = T(q->wolfe);
}

void set_error(orc_result* out, int code, const char* what)
{
    out->status = code;
    std::strncpy(out->msg, what, sizeof(out->msg) - 1);
    out->msg[sizeof(out->msg) - 1] = 0;
}

template <class Body>
int guarded(orc_result* out, Body body)
{
    std::memset(out, 0, sizeof(*out));
    try { body(); }
    catch (const std::invalid_argument& e) { set_error(out, ORC_INVALID_ARGUMENT, e.what()); }
    catch (const std::logic_error& e) { set_error(out, ORC_LOGIC_ERROR, e.what()); }
    catch (const std::runtime_error& e) { set_error(out, ORC_RUNTIME_ERROR, e.what()); }
    catch (const std::exception& e) { set_error(out, ORC_OTHER_ERROR, e.what()); }
    return out->status;
}

template <class T, template <class> class LS>
void run_lbfgs(Functor<T>& f, const orc_param* q, long n, T* x, T* grad_out, orc_result* out)
{
    typedef Eigen::Matrix<T, Eigen::Dynamic, 1> Vec;
    LBFGSpp::LBFGSParam<T> p;
    fill_common<T>(p, q);
    p.linesearch = q->linesearch;
    LBFGSpp::LBFGSSolver<T, LS> solver(p);
    Vec xv(n);
    for (long i = 0; i < n; i++) xv[i] = x[i];
    T fx = T(0);
    const auto t0 = std::chrono::steady_clock::now();
    int niter = 0;
    try { niter = solver.minimize(f, xv, fx); }
    catch (...)
    {
        out->nfev = f.nfev;
        out->trace_len = f.nfev < f.cap ? f.nfev : f.cap;
        for (long i = 0; i < n; i++) x[i] = xv[i];
        throw;
    }
    out->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    out->niter = niter;
    out->fx = double(fx);
    out->gnorm = double(solver.final_grad_norm());
    for (long i = 0; i < n; i++) x[i] = xv[i];
    if (grad_out)
        for (long i = 0; i < n; i++) grad_out[i] = solver.final_grad()[i];
    out->nfev = f.nfev;
    out->trace_len = f.nfev < f.cap ? f.nfev : f.cap;
}

template <class T>
int lbfgs_any(int objective, const T* d0, const T* d1, long n, int ls, const orc_param* q, T* x, T* grad_out,
              double* trace, long cap, orc_result* out)
{
    return guarded(out, [&]() {
        Functor<T> f(objective, d0, d1, n, trace, cap);
        switch (ls)
        {
        case ORC_LS_BACKTRACKING: run_lbfgs<T, LBFGSpp::LineSearchBacktracking>(f, q, n, x, grad_out, out); break;
        case ORC_LS_BRACKETING: run_lbfgs<T, LBFGSpp::LineSearchBracketing>(f, q, n, x, grad_out, out); break;
        case ORC_LS_NOCEDAL_WRIGHT: run_lbfgs<T, LBFGSpp::LineSearchNocedalWright>(f, q, n, x, grad_out, out); break;
        case ORC_LS_MORE_THUENTE: run_lbfgs<T, LBFGSpp::LineSearchMoreThuente>(f, q, n, x, grad_out, out); break;
        default: throw std::invalid_argument("unknown line search id");
        }
    });
}

}  // namespace

extern "C" {

void ref_default_param(orc_param* p, int lbfgsb)
{
    std::memset(p, 0, sizeof(*p));
    if (lbfgsb)
    {
        LBFGSpp::LBFGSBParam<double> d;
        p->m = d.m; p->epsilon = d.epsilon; p->epsilon_rel = d.epsilon_rel; p->past = d.past; p->delta = d.delta;
        p->max_iterations = d.max_iterations; p->max_submin = d.max_submin; p->max_linesearch = d.max_linesearch;
        p->min_step = d.min_step; p->max_step = d.max_step; p->ftol = d.ftol; p->wolfe = d.wolfe;
        p->linesearch = LBFGSpp::LBFGS_LINESEARCH_BACKTRACKING_STRONG_WOLFE;
    }
    else
    {
        LBFGSpp::LBFGSParam<double> d;
        p->m = d.m; p->epsilon = d.epsilon; p->epsilon_rel = d.epsilon_rel; p->past = d.past; p->delta = d.delta;
        p->max_iterations = d.max_iterations; p->linesearch = d.linesearch; p->max_linesearch = d.max_linesearch;
        p->min_step = d.min_step; p->max_step = d.max_step; p->ftol = d.ftol; p->wolfe = d.wolfe;
        p->max_submin = 10;
    }
}

int ref_lbfgs_f64(int objective, const double* d0, const double* d1, long n, int ls, const orc_param* q, int,
                  double* x, double* grad_out, double* trace, long cap, orc_result* out)
{
    return lbfgs_any<double>(objective, d0, d1, n, ls, q, x, grad_out, trace, cap, out);
}

int ref_lbfgs_f32(int objective, const float* d0, const float* d1, long n, int ls, const orc_param* q, int,
                  float* x, float* grad_out, double* trace, long cap, orc_result* out)
{
    return lbfgs_any<float>(objective, d0, d1, n, ls, q, x, grad_out, trace, cap, out);
}

int ref_lbfgsb_f64(int objective, const double* d0, const double* d1, long n, const orc_param* q, int, double* x,
                   const double* lb, const double* ub, double* grad_out, double* trace, long cap, orc_result* out)
{
    typedef Eigen::Matrix<double, Eigen::Dynamic, 1> Vec;
    return guarded(out, [&]() {
        Functor<double> f(objective, d0, d1, n, trace, cap);
        LBFGSpp::LBFGSBParam<double> p;
        fill_common<double>(p, q);
        p.max_submin = q->max_submin;
        LBFGSpp::LBFGSBSolver<double> solver(p);
        Vec xv(n), lbv(n), ubv(n);
        for (long i = 0; i < n; i++) { xv[i] = x[i]; lbv[i] = lb[i]; ubv[i] = ub[i]; }
        double fx = 0;
        const auto t0 = std::chrono::steady_clock::now();
        int niter = 0;
        try { niter = solver.minimize(f, xv, fx, lbv, ubv); }
        catch (...)
        {
            out->nfev = f.nfev;
            out->trace_len = f.nfev < f.cap ? f.nfev : f.cap;
            throw;
        }
        out->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        out->niter = niter;
        out->fx = fx;
        out->gnorm = solver.final_grad_norm();
        for (long i = 0; i < n; i++) x[i] = xv[i];
        if (grad_out)
            for (long i = 0; i < n; i++) grad_out[i] = solver.final_grad()[i];
        out->nfev = f.nfev;
        out->trace_len = f.nfev < f.cap ? f.nfev : f.cap;
    });
}

int ref_bfgs_apply_Hv_f64(long n, int m, int npairs, const double* S, const double* Y, const double* v, double a,
                          int, double* res, double* ys_out, double* theta_out)
{
    typedef Eigen::Matrix<double, Eigen::Dynamic, 1> Vec;
    LBFGSpp::BFGSMat<double> mat;
    mat.reset(int(n), m);
    Vec s(n), y(n);
    for (int k = 0; k < npairs; k++)
    {
        for (long i = 0; i < n; i++) { s[i] = S[i + long(k) * n]; y[i] = Y[i + long(k) * n]; }
        mat.add_correction(s, y);
    }
    Vec vv(n), out;
    for (long i = 0; i < n; i++) vv[i] = v[i];
    mat.apply_Hv(vv, a, out);
    for (long i = 0; i < n; i++) res[i] = out[i];
    if (theta_out) *theta_out = mat.theta();
    (void)ys_out;  // m_ys is private in the reference; only the restatement reports it
    return 0;
}

double ref_objective_f64(int objective, const double* d0, const double* d1, long n, const double* x, double* grad)
{
    return orc::evaluate<double>(objective, d0, d1, n, x, grad);
}

}  // extern "C"
