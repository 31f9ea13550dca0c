// LBFGSpp/LineSearchCore.h -- the scalar decision logic of the four line searches as plain structs that compile both for
// the host (g++, used by the header-only front) and for the device (nvcc, used by the device-resident solve).
//
// A core is a resumable state machine over scalars only:
//     int init(params, fx0, dg0, step0, step_max)    validates like the reference; returns 0 or an error code
//     int advance(fx, dg, bool& keep)                digests the trial at `step`; returns LSC_EVALUATE / LSC_ACCEPT /
//                                                    LSC_TAKE_BEST or an error code; `keep` = remember this trial as the best
//     step, best_fx, best_dg                         the next trial step; f and g.d of the best trial kept so far
// Error codes map one-to-one to the reference's exceptions (type + message, see ls_error_message / ls_error_kind).
// The host loop runs a typed core, the device-resident solve a RunTimeCore (the same four, chosen by kind); both build the options
// with line_search_options() and do the bookkeeping around one search with a SearchRecord.
// Decisions follow the reference line by line in meaning:
//   BacktrackingCore   reference include/LBFGSpp/LineSearchBacktracking.h:44-121
//   BracketingCore     reference include/LBFGSpp/LineSearchBracketing.h:48-128
//   NocedalWrightCore  reference include/LBFGSpp/LineSearchNocedalWright.h:30-60, 84-279
//   MoreThuenteCore    reference include/LBFGSpp/LineSearchMoreThuente.h:34-189, 213-615
#ifndef LBFGSPP_B200_LINE_SEARCH_CORE_H
#define LBFGSPP_B200_LINE_SEARCH_CORE_H

#include <cfloat>
#include <cmath>

#if defined(__CUDACC__)
#define LBFGS_HD __host__ __device__
#else
#define LBFGS_HD
#endif

namespace LBFGSpp {

// what a core asks for after a trial: evaluate at `step`, accept the trial, or (out of budget) take the best point seen so far
enum { LSC_EVALUATE = 0, LSC_ACCEPT = 1, LSC_TAKE_BEST = 2 };

// error codes: >= 16
enum LineSearchError
{
    LSE_STEP_NOT_POSITIVE = 16,      // invalid_argument "'step' must be positive"
    LSE_STEP_BELOW_MIN = 17,         // invalid_argument "'step' is smaller than 'param.min_step'"
    LSE_STEP_ABOVE_MAX = 18,         // invalid_argument "'step' exceeds 'step_max'"
    LSE_NW_NEEDS_STRONG_WOLFE = 19,  // invalid_argument (NocedalWright with another termination condition)
    LSE_NOT_DESCENT_STRICT = 20,     // logic_error "the moving direction does not decrease the objective function value"
    LSE_NOT_DESCENT = 21,            // logic_error "the moving direction increases the objective function value"
    LSE_STEP_TOO_SMALL = 22,         // runtime_error "the line search step became smaller than the minimum value allowed"
    LSE_STEP_TOO_LARGE = 23,         // runtime_error "the line search step became larger than the maximum value allowed"
    LSE_MAX_TRIALS = 24,             // runtime_error "the line search routine reached the maximum number of iterations"
    LSE_BRACKET_INVERTED = 25,       // runtime_error "the lower bound of the bracketing interval becomes larger than the upper bound"
    LSE_PRECISION = 26,              // runtime_error "the line search routine failed, possibly due to insufficient numeric precision"
    LSE_NO_DECREASE = 27             // runtime_error "the line search routine failed, unable to sufficiently decrease the function value"
};

// 1 = std::invalid_argument, 2 = std::logic_error, 3 = std::runtime_error
inline int ls_error_kind(int code)
{
    if (code >= LSE_STEP_NOT_POSITIVE && code <= LSE_NW_NEEDS_STRONG_WOLFE) return 1;
    if (code == LSE_NOT_DESCENT_STRICT || code == LSE_NOT_DESCENT) return 2;
    return 3;
}
inline const char* ls_error_message(int code)
{
    switch (code)
    {
    case LSE_STEP_NOT_POSITIVE: return "'step' must be positive";
    case LSE_STEP_BELOW_MIN: return "'step' is smaller than 'param.min_step'";
    case LSE_STEP_ABOVE_MAX: return "'step' exceeds 'step_max'";
    case LSE_NW_NEEDS_STRONG_WOLFE: return "'param.linesearch' must be 'LBFGS_LINESEARCH_BACKTRACKING_STRONG_WOLFE' for LineSearchNocedalWright";
    case LSE_NOT_DESCENT_STRICT: return "the moving direction does not decrease the objective function value";
    case LSE_NOT_DESCENT: return "the moving direction increases the objective function value";
    case LSE_STEP_TOO_SMALL: return "the line search step became smaller than the minimum value allowed";
    case LSE_STEP_TOO_LARGE: return "the line search step became larger than the maximum value allowed";
    case LSE_MAX_TRIALS: return "the line search routine reached the maximum number of iterations";
    case LSE_BRACKET_INVERTED: return "the lower bound of the bracketing interval becomes larger than the upper bound";
    case LSE_PRECISION: return "the line search routine failed, possibly due to insufficient numeric precision";
    case LSE_NO_DECREASE: return "the line search routine failed, unable to sufficiently decrease the function value";
    }
    return "unknown line search error";
}

// which core: the same ids as LBFGS_B200_LS_* of include/lbfgs_b200.h
enum LineSearchKind { LSK_BACKTRACKING = 0, LSK_BRACKETING = 1, LSK_NOCEDAL_WRIGHT = 2, LSK_MORE_THUENTE = 3 };

// the line-search relevant fields of LBFGSParam / LBFGSBParam
template <typename Scalar>
struct LineSearchOptions
{
    int linesearch;      // 1 Armijo, 2 Wolfe, 3 strong Wolfe
    int max_linesearch;
    Scalar min_step, max_step, ftol, wolfe;
};

// param.linesearch; LBFGSBParam has none (L-BFGS-B runs More-Thuente)
template <class Param> inline auto linesearch_of(const Param& p, int) -> decltype(int(p.linesearch)) { return p.linesearch; }
template <class Param> inline int linesearch_of(const Param&, long) { return 3; }

// The options of a search of the given kind from LBFGSParam, LBFGSBParam or lbfgs_b200_param.  More-Thuente always tests the strong
// Wolfe conditions, whatever param.linesearch says.
template <typename Scalar, class Param>
inline LineSearchOptions<Scalar> line_search_options(const Param& p, int kind)
{
    const LineSearchOptions<Scalar> o = {(kind == LSK_MORE_THUENTE) ? 3 : linesearch_of(p, 0), p.max_linesearch, Scalar(p.min_step),
                                         Scalar(p.max_step), Scalar(p.ftol), Scalar(p.wolfe)};
    return o;
}

namespace lsdetail {
template <typename T> LBFGS_HD inline T inf_of();
template <> LBFGS_HD inline double inf_of<double>() { return HUGE_VAL; }
template <> LBFGS_HD inline float inf_of<float>() { return HUGE_VALF; }
template <typename T> LBFGS_HD inline T eps_of();
template <> LBFGS_HD inline double eps_of<double>() { return DBL_EPSILON; }
template <> LBFGS_HD inline float eps_of<float>() { return FLT_EPSILON; }
template <typename T> LBFGS_HD inline T tmin(T a, T b) { return (b < a) ? b : a; }   // std::min(a, b)
template <typename T> LBFGS_HD inline T tmax(T a, T b) { return (a < b) ? b : a; }   // std::max(a, b)
template <typename T> LBFGS_HD inline T tabs(T a) { return a < T(0) ? -a : a; }
template <typename T> LBFGS_HD inline bool finite(T a) { return (a == a) && (a != inf_of<T>()) && (a != -inf_of<T>()); }
}  // namespace lsdetail

// ---------------------------------------------------------------------------------------------------- Backtracking
template <typename Scalar>
struct BacktrackingCore
{
    static const int kind = LSK_BACKTRACKING;
    Scalar step, best_fx, best_dg;
    LineSearchOptions<Scalar> prm;
    Scalar f0, slope0, armijo_slope;
    int trials;

    LBFGS_HD int init(const LineSearchOptions<Scalar>& p, Scalar fx_init, Scalar dg_init, Scalar step0, Scalar /*step_max*/)
    {
        prm = p; f0 = fx_init; slope0 = dg_init; armijo_slope = p.ftol * dg_init; step = step0;
        best_fx = fx_init; best_dg = dg_init; trials = 0;
        if (step0 <= Scalar(0)) return LSE_STEP_NOT_POSITIVE;
        if (dg_init > Scalar(0)) return LSE_NOT_DESCENT;
        return 0;
    }
    LBFGS_HD int advance(Scalar fx, Scalar dg, bool& /*keep*/)
    {
        const Scalar shrink = Scalar(0.5), grow = Scalar(2.1);
        Scalar factor;
        if ((fx > f0 + step * armijo_slope) || (fx != fx))
            factor = shrink;
        else
        {
            if (prm.linesearch == 1) return LSC_ACCEPT;
            if (dg < prm.wolfe * slope0)
                factor = grow;
            else
            {
                if (prm.linesearch == 2) return LSC_ACCEPT;
                if (dg > -prm.wolfe * slope0)
                    factor = shrink;
                else
                    return LSC_ACCEPT;
            }
        }
        if (step < prm.min_step) return LSE_STEP_TOO_SMALL;
        if (step > prm.max_step) return LSE_STEP_TOO_LARGE;
        step *= factor;
        if (++trials >= prm.max_linesearch) return LSE_MAX_TRIALS;
        return LSC_EVALUATE;
    }
};

// ---------------------------------------------------------------------------------------------------- Bracketing
template <typename Scalar>
struct BracketingCore
{
    static const int kind = LSK_BRACKETING;
    Scalar step, best_fx, best_dg;
    LineSearchOptions<Scalar> prm;
    Scalar f0, slope0, armijo_slope, lo, hi;
    int trials;

    LBFGS_HD int init(const LineSearchOptions<Scalar>& p, Scalar fx_init, Scalar dg_init, Scalar step0, Scalar /*step_max*/)
    {
        prm = p; f0 = fx_init; slope0 = dg_init; armijo_slope = p.ftol * dg_init; lo = Scalar(0);
        hi = lsdetail::inf_of<Scalar>(); step = step0; best_fx = fx_init; best_dg = dg_init; trials = 0;
        if (step0 <= Scalar(0)) return LSE_STEP_NOT_POSITIVE;
        if (dg_init > Scalar(0)) return LSE_NOT_DESCENT;
        return 0;
    }
    LBFGS_HD int advance(Scalar fx, Scalar dg, bool& /*keep*/)
    {
        if (fx > f0 + step * armijo_slope || !lsdetail::finite(fx))
            hi = step;
        else
        {
            if (prm.linesearch == 1) return LSC_ACCEPT;
            if (dg < prm.wolfe * slope0)
                lo = step;
            else
            {
                if (prm.linesearch == 2) return LSC_ACCEPT;
                if (dg > -prm.wolfe * slope0)
                    hi = step;
                else
                    return LSC_ACCEPT;
            }
        }
        if (lo > hi) return LSE_BRACKET_INVERTED;
        if (step < prm.min_step) return LSE_STEP_TOO_SMALL;
        if (step > prm.max_step) return LSE_STEP_TOO_LARGE;
        step = (hi == lsdetail::inf_of<Scalar>()) ? 2 * step : lo / 2 + hi / 2;
        if (++trials >= prm.max_linesearch) return LSE_MAX_TRIALS;
        return LSC_EVALUATE;
    }
};

// ---------------------------------------------------------------------------------------------------- Nocedal-Wright
template <typename Scalar>
struct NocedalWrightCore
{
    static const int kind = LSK_NOCEDAL_WRIGHT;
    Scalar step, best_fx, best_dg;
    LineSearchOptions<Scalar> prm;
    Scalar f0, decrease_slope, curvature_bound, lo, hi, f_lo, f_hi, slope_lo;
    int zoom, budget_used;

    // minimiser of the parabola through (lo, f_lo) with slope slope_lo and (hi, f_hi); bisect when it is not finite,
    // outside the interval or within 1% of an end point
    LBFGS_HD Scalar interpolate() const
    {
        using namespace lsdetail;
        const Scalar df = f_hi - f_lo, ds = hi - lo, mid = (hi + lo) / Scalar(2);
        Scalar cand = df * lo - mid * ds * slope_lo;
        cand = cand / (df - ds * slope_lo);
        const bool useless = !finite(cand);
        const Scalar margin = tmin(tabs(cand - lo), tabs(cand - hi));
        const bool hugging = margin < Scalar(0.01) * tabs(ds);
        const bool bisect = useless || cand <= tmin(lo, hi) || cand >= tmax(lo, hi) || hugging;
        return bisect ? mid : cand;
    }
    LBFGS_HD void remember(Scalar fx, Scalar dg, bool& keep)
    {
        lo = step; f_lo = fx; slope_lo = dg; best_fx = fx; best_dg = dg; keep = true;
    }
    LBFGS_HD int init(const LineSearchOptions<Scalar>& p, Scalar fx_init, Scalar dg_init, Scalar step0, Scalar /*step_max*/)
    {
        prm = p; f0 = fx_init; decrease_slope = p.ftol * dg_init; curvature_bound = -p.wolfe * dg_init;
        lo = Scalar(0); hi = Scalar(0); f_lo = fx_init; f_hi = Scalar(0); slope_lo = dg_init; zoom = 0; budget_used = 0;
        step = step0; best_fx = fx_init; best_dg = dg_init;
        if (step0 <= Scalar(0)) return LSE_STEP_NOT_POSITIVE;
        if (p.linesearch != 3) return LSE_NW_NEEDS_STRONG_WOLFE;
        if (dg_init > Scalar(0)) return LSE_NOT_DESCENT;
        return 0;
    }
    LBFGS_HD int advance(Scalar fx, Scalar dg, bool& keep)
    {
        using namespace lsdetail;
        const bool too_high = fx - f0 > step * decrease_slope;
        if (!zoom)
        {
            if (too_high || (Scalar(0) < lo && fx >= f_lo))
            {
                hi = step; f_hi = fx; zoom = 1; step = interpolate();
                return LSC_EVALUATE;
            }
            if (tabs(dg) <= curvature_bound) return LSC_ACCEPT;
            hi = lo;
            f_hi = f_lo;
            remember(fx, dg, keep);
            if (dg >= Scalar(0))
            {
                zoom = 1; step = interpolate();
                return LSC_EVALUATE;
            }
            if (++budget_used >= prm.max_linesearch) return LSC_TAKE_BEST;  // best == the trial just kept
            step *= Scalar(2);
            return LSC_EVALUATE;
        }
        if (too_high || fx >= f_lo)
        {
            if (step == hi) return LSE_PRECISION;
            hi = step;
            f_hi = fx;
        }
        else
        {
            if (tabs(dg) <= curvature_bound) return LSC_ACCEPT;
            if (dg * (hi - lo) >= Scalar(0))
            {
                hi = lo;
                f_hi = f_lo;
            }
            if (step == lo) return LSE_PRECISION;
            remember(fx, dg, keep);
        }
        if (++budget_used >= prm.max_linesearch)
        {
            if (lo <= Scalar(0)) return LSE_NO_DECREASE;
            step = lo;
            return LSC_TAKE_BEST;
        }
        step = interpolate();
        return LSC_EVALUATE;
    }
};

// ---------------------------------------------------------------------------------------------------- More-Thuente
template <typename Scalar>
struct MoreThuenteCore
{
    struct Sample { Scalar at, f, g; };   // abscissa, psi value, psi slope

    static const int kind = LSK_MORE_THUENTE;
    Scalar step, best_fx, best_dg;
    Scalar smin, smax, f0, decrease_slope, curvature_bound, psi_lo, width, width_before;
    Sample lo, hi;
    int bracketed, cap_next_step, stalls, trials, budget;

    // interpolating polynomials through two samples (reference :34-114)
    LBFGS_HD static Scalar quadratic_from_values(const Sample& p, const Sample& q)
    {
        const Scalar span = q.at - p.at;
        const Scalar w = Scalar(0.5) * span * p.g / (p.f - q.f + span * p.g);
        return p.at + w * span;
    }
    LBFGS_HD static Scalar quadratic_from_slopes(const Sample& p, const Sample& q)
    {
        const Scalar w = p.g / (p.g - q.g);
        return p.at + w * (q.at - p.at);
    }
    LBFGS_HD static Scalar cubic(const Sample& p, const Sample& q, bool& found)
    {
        using namespace lsdetail;
        const Scalar a = p.at, b = q.at;
        const Scalar sum = a + b, span = b - a, span2 = span * span;
        const Scalar df = q.f - p.f, dgr = q.g - p.g;
        const Scalar c3 = (p.g + q.g) * span - Scalar(2) * df;
        const Scalar c2 = Scalar(0.5) * (dgr * span2 - Scalar(3) * sum * c3);
        const Scalar c1 = df * span2 - sum * c2 - (a * sum + b * b) * c3;
        const Scalar tiny = eps_of<Scalar>();
        if (tabs(c3) < tiny * tabs(c2) || tabs(c3) < tiny * tabs(c1))
        {
            found = (c2 * span > Scalar(0));
            return found ? (-Scalar(0.5) * c1 / c2) : b;
        }
        const Scalar u = c2 / (Scalar(3) * c3), v = c1 / c2;
        const Scalar ratio = v / u;
        found = (ratio <= Scalar(1));
        if (!found) return b;
        Scalar root_a, root_b;
        if (tabs(u) >= tabs(v))
        {
            const Scalar w = Scalar(1) + std::sqrt(Scalar(1) - ratio);
            root_a = -u * w;
            root_b = -v / w;
        }
        else
        {
            const Scalar disc = std::sqrt(tabs(u)) * std::sqrt(tabs(v)) * std::sqrt(1 - u / v);
            root_a = -u - disc;
            root_b = -u + disc;
        }
        return (c3 * span > Scalar(0)) ? tmax(root_a, root_b) : tmin(root_a, root_b);
    }
    // safeguarded choice of the next trial given the trial sample t (reference :116-189)
    LBFGS_HD static Scalar select_step(const Sample& lo, const Sample& hi, const Sample& t)
    {
        using namespace lsdetail;
        if (lo.at == hi.at) return lo.at;
        if (!finite(t.f) || !finite(t.g)) return (lo.at + t.at) / Scalar(2);
        bool cubic_ok;
        const Scalar ac = cubic(lo, t, cubic_ok);
        const Scalar aq = quadratic_from_values(lo, t);
        if (t.f > lo.f)
        {
            if (!cubic_ok) return aq;
            return (tabs(ac - lo.at) < tabs(aq - lo.at)) ? ac : ((aq + ac) / Scalar(2));
        }
        const Scalar as = quadratic_from_slopes(lo, t);
        if (t.g * lo.g < Scalar(0)) return (tabs(ac - t.at) >= tabs(as - t.at)) ? ac : as;
        const Scalar extrapolate = Scalar(1.1), toward_hi = Scalar(0.66);
        if (tabs(t.g) < tabs(lo.g))
        {
            const bool use_cubic = cubic_ok && (ac - t.at) * (t.at - lo.at) > Scalar(0) && tabs(ac - t.at) < tabs(as - t.at);
            const Scalar pick = use_cubic ? ac : as;
            const Scalar limit = t.at + toward_hi * (hi.at - t.at);
            return (t.at > lo.at) ? tmin(limit, pick) : tmax(limit, pick);
        }
        if (!finite(hi.at) || !finite(hi.f) || !finite(hi.g)) return t.at + extrapolate * (t.at - lo.at);
        bool unused;
        const Scalar ae = cubic(t, hi, unused);
        const Scalar limit = t.at + toward_hi * (hi.at - t.at);
        return (t.at > lo.at) ? tmin(limit, ae) : tmax(limit, ae);
    }

    LBFGS_HD int init(const LineSearchOptions<Scalar>& p, Scalar fx_init, Scalar dg_init, Scalar step0, Scalar step_max)
    {
        using namespace lsdetail;
        const Scalar inf = inf_of<Scalar>();
        smin = p.min_step; smax = step_max; f0 = fx_init; decrease_slope = p.ftol * dg_init; curvature_bound = -p.wolfe * dg_init;
        psi_lo = Scalar(0); bracketed = 0; cap_next_step = (p.min_step > Scalar(0)) ? 1 : 0; width = inf; width_before = inf;
        stalls = 0; trials = 0; budget = p.max_linesearch; step = step0; best_fx = fx_init; best_dg = dg_init;
        lo.at = Scalar(0); lo.f = Scalar(0); lo.g = (Scalar(1) - p.ftol) * dg_init;
        hi.at = inf; hi.f = inf; hi.g = inf;
        if (step0 <= Scalar(0)) return LSE_STEP_NOT_POSITIVE;
        if (step0 < smin) return LSE_STEP_BELOW_MIN;
        if (step0 > smax) return LSE_STEP_ABOVE_MAX;
        if (dg_init >= Scalar(0)) return LSE_NOT_DESCENT_STRICT;
        return 0;
    }
    LBFGS_HD int advance(Scalar fx, Scalar dg, bool& keep)
    {
        using namespace lsdetail;
        const Scalar inf = inf_of<Scalar>();
        const Scalar psi = fx - f0 - step * decrease_slope;
        const Scalar dpsi = dg - decrease_slope;
        if (psi <= Scalar(0) && tabs(dg) <= curvature_bound) return LSC_ACCEPT;
        if (step <= smin && (psi > Scalar(0) || dpsi >= Scalar(0))) return LSC_ACCEPT;
        if (step >= smax && (psi <= Scalar(0) && dpsi < Scalar(0))) return LSC_ACCEPT;

        const Sample t = {step, psi, dpsi};
        if (cap_next_step && psi <= Scalar(0) && dpsi < Scalar(0)) cap_next_step = 0;
        const bool marching = (psi <= psi_lo) && (dpsi * (lo.at - step) > Scalar(0));
        Scalar next;
        if (marching)
            next = tmin(smax, step + Scalar(1.1) * (step - lo.at));
        else
        {
            next = select_step(lo, hi, t);
            next = tmax(next, smin);
            next = tmin(next, smax);
            if (cap_next_step)
            {
                const Scalar ceiling = tmax(smin, (Scalar(7) / Scalar(12)) * step);
                next = tmax(next, smin);
                next = tmin(next, ceiling);
            }
        }
        if (psi > psi_lo)
            hi = t;
        else
        {
            if (!marching) hi = lo;
            lo = t;
            psi_lo = psi;
            best_fx = fx;
            best_dg = dg;
            keep = true;
        }
        if (!bracketed && !marching)
        {
            const Scalar left = tmin(lo.at, hi.at), right = tmax(lo.at, hi.at);
            bracketed = (left >= smin && right <= smax) ? 1 : 0;
        }
        if (bracketed)
        {
            width_before = width;
            width = tabs(hi.at - lo.at);
            if (width_before < inf && width > Scalar(0.66) * width_before)
                stalls += 1;
            else
                stalls = 0;
            if (stalls >= 2)
            {
                next = (lo.at + hi.at) / Scalar(2);
                stalls = 0;
            }
        }
        step = next;
        if (++trials >= budget)
        {
            step = lo.at;
            return LSC_TAKE_BEST;
        }
        return LSC_EVALUATE;
    }
};

// ---------------------------------------------------------------------------------------------------- chosen at run time
// One of the four cores, picked by `kind` (LSK_*).  The cores begin with the same members (step, best_fx, best_dg), so those are
// read without a dispatch.
template <typename Scalar>
struct RunTimeCore
{
    int kind;
    union
    {
        BacktrackingCore<Scalar> bt;
        BracketingCore<Scalar> br;
        NocedalWrightCore<Scalar> nw;
        MoreThuenteCore<Scalar> mt;
    };

    LBFGS_HD int init(const LineSearchOptions<Scalar>& p, Scalar fx_init, Scalar dg_init, Scalar step0, Scalar step_max)
    {
        switch (kind)
        {
        case LSK_BACKTRACKING: return bt.init(p, fx_init, dg_init, step0, step_max);
        case LSK_BRACKETING: return br.init(p, fx_init, dg_init, step0, step_max);
        case LSK_NOCEDAL_WRIGHT: return nw.init(p, fx_init, dg_init, step0, step_max);
        default: return mt.init(p, fx_init, dg_init, step0, step_max);
        }
    }
    LBFGS_HD int advance(Scalar fx, Scalar dg, bool& keep)
    {
        switch (kind)
        {
        case LSK_BACKTRACKING: return bt.advance(fx, dg, keep);
        case LSK_BRACKETING: return br.advance(fx, dg, keep);
        case LSK_NOCEDAL_WRIGHT: return nw.advance(fx, dg, keep);
        default: return mt.advance(fx, dg, keep);
        }
    }
    LBFGS_HD Scalar step() const { return bt.step; }
    LBFGS_HD Scalar best_fx() const { return bt.best_fx; }
    LBFGS_HD Scalar best_dg() const { return bt.best_dg; }
};

// ---------------------------------------------------------------------------------------------------- one search's bookkeeping
// What a driver does after a core has digested a trial
enum SearchStep
{
    SEARCH_EVALUATE = 0,     // evaluate the objective at the core's step
    SEARCH_ACCEPT = 1,       // the trial just evaluated is the result
    SEARCH_TAKE_KEPT = 2,    // the best trial kept so far is the result: bring x_lo, g_lo back
    SEARCH_TAKE_START = 3    // no trial improved on the start point, which is the result: copy xp, gp back
};

// The values of the current point of the loop and their bookkeeping during one search.  Between searches {fx, dg, gg, xx} describe the
// current point; during a search they still describe its start point, and the search's result replaces them.  A trial the core
// keeps (`keep`) moves into the driver's x_lo / g_lo buffers; its g.g and x.x are remembered here, its f and g.d by the core.
template <typename Scalar>
struct SearchRecord
{
    Scalar fx, dg, gg, xx;   // f, g.d, g.g, x.x
    Scalar lo_gg, lo_xx;     // g.g, x.x of the kept trial
    int have_lo;             // a trial has been kept

    LBFGS_HD void begin() { have_lo = 0; }
    // the core's (action, keep) on the trial {tfx, tdg, tgg, txx}: returns a SearchStep, or the core's error code (then nothing is
    // recorded and no trial is kept)
    LBFGS_HD int digest(int action, bool keep, Scalar tfx, Scalar tdg, Scalar tgg, Scalar txx, Scalar best_fx, Scalar best_dg)
    {
        if (action >= LSE_STEP_NOT_POSITIVE) return action;
        if (keep) { have_lo = 1; lo_gg = tgg; lo_xx = txx; }
        if (action == LSC_EVALUATE) return SEARCH_EVALUATE;
        if (action == LSC_ACCEPT) { fx = tfx; dg = tdg; gg = tgg; xx = txx; return SEARCH_ACCEPT; }
        fx = best_fx;   // LSC_TAKE_BEST
        dg = best_dg;
        if (!have_lo) return SEARCH_TAKE_START;   // gg, xx are the start point's already
        gg = lo_gg; xx = lo_xx;
        return SEARCH_TAKE_KEPT;
    }
};

#if !defined(__CUDACC__)
}  // namespace LBFGSpp
#include <stdexcept>
namespace LBFGSpp {
// host side: turn an error code into the exception the reference throws at that point
inline void ls_throw(int code)
{
    switch (ls_error_kind(code))
    {
    case 1: throw std::invalid_argument(ls_error_message(code));
    case 2: throw std::logic_error(ls_error_message(code));
    default: throw std::runtime_error(ls_error_message(code));
    }
}

// A policy's Machine (LineSearch*.h): the core, armed by a constructor that validates the search's inputs and throws like the
// reference.
template <typename Scalar, template <class> class Core>
struct CoreMachine : Core<Scalar>
{
    template <class Param>
    CoreMachine(const Param& param, Scalar fx_init, Scalar dg_init, Scalar step0, Scalar step_max)
    {
        const int rc = this->init(line_search_options<Scalar>(param, Core<Scalar>::kind), fx_init, dg_init, step0, step_max);
        if (rc != 0) ls_throw(rc);
    }
};
#endif

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_LINE_SEARCH_CORE_H
