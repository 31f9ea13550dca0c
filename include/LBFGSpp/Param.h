// LBFGSpp/Param.h -- solver options of the H100 L-BFGS / L-BFGS-B front.
//
// Drop-in for the reference's include/LBFGSpp/Param.h: same struct names, same public fields, same
// defaults (reference Param.h:171-182 and :330-341), same enum values (:23-62) and the same
// std::invalid_argument messages from check_param() (:191-218, :350-376).  No device work happens here.
//
// One difference in range, not in meaning: the reference accepts any positive m; the device history holds at most m = 64 pairs
// (LBFGSSolver) / m = 20 (LBFGSBSolver).  check_param() keeps the reference's messages, so a larger m is reported by minimize() when
// the history is created (std::invalid_argument: "hist_create: need n >= 1 and 1 <= m <= 64", "the bound-constrained path supports
// m <= 20").
#ifndef LBFGSPP_B200_PARAM_H
#define LBFGSPP_B200_PARAM_H

#include <stdexcept>

namespace LBFGSpp {

// Which condition ends a Backtracking / Bracketing line search (the other two line searches always use
// the strong Wolfe conditions).  Values are the reference's.
enum LINE_SEARCH_TERMINATION_CONDITION
{
    LBFGS_LINESEARCH_BACKTRACKING_ARMIJO = 1,        // sufficient decrease only
    LBFGS_LINESEARCH_BACKTRACKING = 2,               // alias of the regular Wolfe condition
    LBFGS_LINESEARCH_BACKTRACKING_WOLFE = 2,         // sufficient decrease + curvature
    LBFGS_LINESEARCH_BACKTRACKING_STRONG_WOLFE = 3   // sufficient decrease + |curvature|
};

namespace detail {

// Checks shared by both option structs; `P` only needs the common fields.
template <class P>
inline void validate_common_options(const P& p)
{
    struct Rule { bool violated; const char* message; };
    const Rule head[] = {
        {p.m <= 0, "'m' must be positive"},
        {p.epsilon < 0, "'epsilon' must be non-negative"},
        {p.epsilon_rel < 0, "'epsilon_rel' must be non-negative"},
        {p.past < 0, "'past' must be non-negative"},
        {p.delta < 0, "'delta' must be non-negative"},
        {p.max_iterations < 0, "'max_iterations' must be non-negative"},
    };
    for (const Rule& r : head)
        if (r.violated) throw std::invalid_argument(r.message);
}

template <class P>
inline void validate_step_options(const P& p)
{
    struct Rule { bool violated; const char* message; };
    const Rule tail[] = {
        {p.max_linesearch <= 0, "'max_linesearch' must be positive"},
        {p.min_step < 0, "'min_step' must be positive"},
        {p.max_step < p.min_step, "'max_step' must be greater than 'min_step'"},
        {p.ftol <= 0 || p.ftol >= 0.5, "'ftol' must satisfy 0 < ftol < 0.5"},
        {p.wolfe <= p.ftol || p.wolfe >= 1, "'wolfe' must satisfy ftol < wolfe < 1"},
    };
    for (const Rule& r : tail)
        if (r.violated) throw std::invalid_argument(r.message);
}

}  // namespace detail

// Options of LBFGSSolver.
template <typename Scalar = double>
class LBFGSParam
{
public:
    int m = 6;                         // history length (columns of S and Y kept in HBM)
    Scalar epsilon = Scalar(1e-5);     // stop when ||g|| <= epsilon
    Scalar epsilon_rel = Scalar(1e-5); // ... or ||g|| <= epsilon_rel * ||x||
    int past = 0;                      // compare f with its value `past` iterations ago (0 = off)
    Scalar delta = Scalar(0);          // relative decrease threshold for that test
    int max_iterations = 0;            // 0 = unlimited
    int linesearch = LBFGS_LINESEARCH_BACKTRACKING_STRONG_WOLFE;
    int max_linesearch = 20;           // trials per line search
    Scalar min_step = Scalar(1e-20);
    Scalar max_step = Scalar(1e+20);
    Scalar ftol = Scalar(1e-4);        // sufficient-decrease constant
    Scalar wolfe = Scalar(0.9);        // curvature constant

    inline void check_param() const
    {
        detail::validate_common_options(*this);
        if (linesearch < LBFGS_LINESEARCH_BACKTRACKING_ARMIJO || linesearch > LBFGS_LINESEARCH_BACKTRACKING_STRONG_WOLFE)
            throw std::invalid_argument("unsupported line search termination condition");
        detail::validate_step_options(*this);
    }
};

// Options of LBFGSBSolver.
template <typename Scalar = double>
class LBFGSBParam
{
public:
    int m = 6;
    Scalar epsilon = Scalar(1e-5);     // on the projected-gradient infinity norm
    Scalar epsilon_rel = Scalar(1e-5);
    int past = 1;
    Scalar delta = Scalar(1e-10);
    int max_iterations = 0;
    int max_submin = 10;               // subspace-minimisation sweeps
    int max_linesearch = 20;
    Scalar min_step = Scalar(1e-20);
    Scalar max_step = Scalar(1e+20);
    Scalar ftol = Scalar(1e-4);
    Scalar wolfe = Scalar(0.9);

    inline void check_param() const
    {
        detail::validate_common_options(*this);
        if (max_submin < 0) throw std::invalid_argument("'max_submin' must be non-negative");
        detail::validate_step_options(*this);
    }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_PARAM_H
