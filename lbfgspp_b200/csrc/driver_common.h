// driver_common.h -- what the translation units of liblbfgs_b200_driver.so share: the parameter struct of the host-buffer entry
// points, the Device of each GPU ordinal, the line-search dispatch and the error reporting through a caller's text buffer.
#ifndef LBFGSPP_B200_DRIVER_COMMON_H
#define LBFGSPP_B200_DRIVER_COMMON_H

#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>

#include "../../include/LBFGS.h"
#include "../../include/LBFGSBatch.h"
#include "../../include/LBFGSSmallBatch.h"

extern "C" {

typedef struct
{
    int m;
    double epsilon, epsilon_rel;
    int past;
    double delta;
    int max_iterations;
    int linesearch;
    int max_submin;
    int max_linesearch;
    double min_step, max_step, ftol, wolfe;
} drv_param;

enum { DRV_LS_BACKTRACKING = 0, DRV_LS_BRACKETING = 1, DRV_LS_NOCEDAL_WRIGHT = 2, DRV_LS_MORE_THUENTE = 3 };

}  // extern "C"

namespace lbfgsb200_drv {

using namespace LBFGSpp;

// one Device (context + stream) per GPU ordinal for the whole library
inline std::map<int, std::shared_ptr<Device> >& devices()
{
    static std::map<int, std::shared_ptr<Device> > m;
    return m;
}
inline Device& device(int ordinal)
{
    std::shared_ptr<Device>& d = devices()[ordinal];
    if (!d) d = std::make_shared<Device>(ordinal);
    return *d;
}

// The solver types of one line-search policy; with_line_search() hands one of these to its callback.
template <template <class> class LS>
struct LineSearchTag
{
    template <class Scalar> using Solver = LBFGSSolver<Scalar, LS>;
    template <class Scalar> using BatchSolver = LBFGSBatchSolver<Scalar, LS>;
    template <class Scalar> using SmallBatchSolver = LBFGSSmallBatchSolver<Scalar, LS>;
};

// f(LineSearchTag<LS>()) for the policy of a DRV_LS_* id: the one place a line-search id becomes a type.
template <class F>
auto with_line_search(int ls, F f) -> decltype(f(LineSearchTag<LineSearchMoreThuente>()))
{
    switch (ls)
    {
    case DRV_LS_BACKTRACKING: return f(LineSearchTag<LineSearchBacktracking>());
    case DRV_LS_BRACKETING: return f(LineSearchTag<LineSearchBracketing>());
    case DRV_LS_NOCEDAL_WRIGHT: return f(LineSearchTag<LineSearchNocedalWright>());
    case DRV_LS_MORE_THUENTE: return f(LineSearchTag<LineSearchMoreThuente>());
    default: throw std::invalid_argument("unknown line search id");
    }
}

// The entry points that report through a caller's text buffer: body()'s result, or `failed` with the exception's message in
// err (errlen bytes, NUL-terminated).
template <class R, class Body>
R reported(char* err, int errlen, R failed, Body body)
{
    try { return body(); }
    catch (const std::exception& e)
    {
        if (err && errlen > 0) { std::strncpy(err, e.what(), size_t(errlen) - 1); err[errlen - 1] = 0; }
        return failed;
    }
}

template <class Scalar>
LBFGSParam<Scalar> to_param(const drv_param* q)
{
    LBFGSParam<Scalar> p;
    p.m = q->m;
    p.epsilon = Scalar(q->epsilon);
    p.epsilon_rel = Scalar(q->epsilon_rel);
    p.past = q->past;
    p.delta = Scalar(q->delta);
    p.max_iterations = q->max_iterations;
    p.linesearch = q->linesearch;
    p.max_linesearch = q->max_linesearch;
    p.min_step = Scalar(q->min_step);
    p.max_step = Scalar(q->max_step);
    p.ftol = Scalar(q->ftol);
    p.wolfe = Scalar(q->wolfe);
    return p;
}

}  // namespace lbfgsb200_drv

#endif  // LBFGSPP_B200_DRIVER_COMMON_H
