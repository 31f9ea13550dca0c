// LBFGSSmallBatch.h -- LBFGSSmallBatchSolver<Scalar, LineSearch>: many independent small unconstrained problems of a built-in
// objective minimised by ONE ordinary kernel launch, one thread block per problem, the whole solve in that block's shared memory.
//
// LBFGSBatchSolver (LBFGSBatch.h) spreads every pass of a problem over all SMs, which pays off at large n; at n of a few to a few
// hundred coordinates there is nothing to spread.  This solver gives each problem a thread block of its own instead (C ABI:
// lbfgs_b200_small_minimize_*), so B is limited only by device memory and n by one block's shared memory (max_n()).  Same
// parameters, line-search policies, stopping rules and per-problem outcomes as LBFGSBatchSolver.  A problem's result does not depend
// on B or on its position in the batch; it equals LBFGSSolver's to rounding (its sums are associated within one block), not bit for bit.
#ifndef LBFGSPP_B200_LBFGS_SMALL_BATCH_H
#define LBFGSPP_B200_LBFGS_SMALL_BATCH_H

#include <vector>

#include "LBFGSBatch.h"

namespace LBFGSpp {

namespace detail {
template <class S> struct small_batch_abi;
template <> struct small_batch_abi<double>
{
    static lbfgs_b200_status minimize(lbfgs_b200_ctx* c, int obj, const double* d0, const double* d1, int64_t ldd, int64_t n, int64_t B,
                                      const lbfgs_b200_param* p, int ls, double* X, int64_t ldx, double* G, lbfgs_b200_outcome* o)
    { return lbfgs_b200_small_minimize_f64(c, obj, d0, d1, ldd, n, B, p, ls, X, ldx, G, o); }
};
template <> struct small_batch_abi<float>
{
    static lbfgs_b200_status minimize(lbfgs_b200_ctx* c, int obj, const float* d0, const float* d1, int64_t ldd, int64_t n, int64_t B,
                                      const lbfgs_b200_param* p, int ls, float* X, int64_t ldx, float* G, lbfgs_b200_outcome* o)
    { return lbfgs_b200_small_minimize_f32(c, obj, d0, d1, ldd, n, B, p, ls, X, ldx, G, o); }
};
}  // namespace detail

template <typename Scalar, template <class> class LineSearch = LineSearchNocedalWright>
class LBFGSSmallBatchSolver
{
public:
    typedef DeviceVector<Scalar> Vector;

private:
    const LBFGSParam<Scalar>& m_param;
    Vector m_grad;          // B*n final gradients
    std::ptrdiff_t m_n;

    LBFGSSmallBatchSolver(const LBFGSSmallBatchSolver&);
    LBFGSSmallBatchSolver& operator=(const LBFGSSmallBatchSolver&);

public:
    LBFGSSmallBatchSolver(const LBFGSParam<Scalar>& param) : m_param(param), m_n(0) { m_param.check_param(); }

    // largest n a problem may have for history size m and built-in objective `objective` (LBFGS_B200_OBJ_*); 0 if none
    static std::ptrdiff_t max_n(int m, int objective) { return std::ptrdiff_t(lbfgs_b200_small_max_n(m, int(sizeof(Scalar)), objective)); }

    // X holds the B start points back to back (problem b at [b*n, (b+1)*n)) and receives the solutions.  f describes the built-in
    // objective; problem b's data vectors (if the objective has any) start at data + b*ldd (ldd = 0: shared by all problems).  Adds
    // every problem's evaluations to f's call count.
    std::vector<BatchOutcome<Scalar> > minimize(BuiltinObjective<Scalar>& f, Vector& X, long B, std::ptrdiff_t ldd = 0)
    {
        if (B < 1 || X.size() % B != 0) throw std::invalid_argument("LBFGSSmallBatchSolver: X must hold B vectors of equal length");
        Device& dev = X.device();
        const std::ptrdiff_t n = X.size() / B;
        m_grad = Vector(dev, X.size());
        m_n = n;
        const lbfgs_b200_param p = detail::abi_param(m_param);
        std::vector<lbfgs_b200_outcome> raw((size_t)B);
        dev.check(detail::small_batch_abi<Scalar>::minimize(dev.ctx(), f.builtin_kind(), f.builtin_data0(), f.builtin_data1(), int64_t(ldd), int64_t(n),
                                                            int64_t(B), &p, detail::line_search_id<LineSearch>::value, X.data(), int64_t(n),
                                                            m_grad.data(), raw.data()));
        std::vector<BatchOutcome<Scalar> > out((size_t)B);
        for (size_t b = 0; b < size_t(B); b++)
        {
            out[b].status = raw[b].status; out[b].niter = raw[b].niter; out[b].nfev = long(raw[b].nfev);
            out[b].fx = Scalar(raw[b].fx); out[b].gnorm = Scalar(raw[b].gnorm); out[b].rounds = long(raw[b].rounds);
            f.add_calls(long(raw[b].nfev));
        }
        return out;
    }
    // gradient of problem b at its solution (device pointer into the solver's own B*n buffer, valid until the next minimize())
    const Scalar* final_grad(long b) const { return m_grad.data() + std::ptrdiff_t(b) * m_n; }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_LBFGS_SMALL_BATCH_H
