// LBFGSBatch.h -- LBFGSBatchSolver<Scalar, LineSearch>: B independent unconstrained problems of the same shape minimised by ONE
// persistent kernel launch (BASELINE config 5).
//
// The reference has no batch interface: a user loops over `LBFGSSolver::minimize()` calls (reference LBFGS.h:78-173).  On the GPU
// B separate solves of n = 1e6 are latency-bound, so the device-resident solve (include/lbfgs_b200.h, "device-resident solve")
// accepts a batch: in every round each running problem executes the one streaming pass its own state asks for, problems leave as
// they converge, and every problem's result is bit-identical to what LBFGSSolver::minimize() returns for it alone.  With n sharded
// over ranks (lbfgs_b200_comm_p2p_*), one exchange per round carries the partial sums of all running problems.
// Same parameters, same line-search policies, same exceptions as LBFGSSolver -- reported per problem instead of thrown.
#ifndef LBFGSPP_B200_LBFGS_BATCH_H
#define LBFGSPP_B200_LBFGS_BATCH_H

#include <vector>

#include "LBFGS.h"
#include "LBFGSpp/DeviceObjectives.h"

namespace LBFGSpp {

template <typename Scalar>
struct BatchOutcome
{
    int status;      // 0, or a LineSearchError code (LBFGSpp/LineSearchCore.h): the exception LBFGSSolver would have thrown
    int niter;       // what minimize() would have returned
    long nfev;       // objective evaluations
    Scalar fx, gnorm;
    long rounds;     // streaming passes the problem took part in
};

namespace detail {
template <class S> struct batch_abi;
template <> struct batch_abi<double>
{
    static lbfgs_b200_status minimize(lbfgs_b200_solver* s, int obj, const double* d0, const double* d1, int64_t ldd, const lbfgs_b200_param* p,
                                      int ls, double* x, int64_t ldx, lbfgs_b200_outcome* o)
    { return lbfgs_b200_solver_minimize_batch_f64(s, obj, d0, d1, ldd, p, ls, x, ldx, o); }
};
template <> struct batch_abi<float>
{
    static lbfgs_b200_status minimize(lbfgs_b200_solver* s, int obj, const float* d0, const float* d1, int64_t ldd, const lbfgs_b200_param* p,
                                      int ls, float* x, int64_t ldx, lbfgs_b200_outcome* o)
    { return lbfgs_b200_solver_minimize_batch_f32(s, obj, d0, d1, ldd, p, ls, x, ldx, o); }
};
}  // namespace detail

template <typename Scalar, template <class> class LineSearch = LineSearchNocedalWright>
class LBFGSBatchSolver
{
public:
    typedef DeviceVector<Scalar> Vector;

private:
    const LBFGSParam<Scalar>& m_param;
    lbfgs_b200_solver* m_solver;
    Device* m_dev;
    std::ptrdiff_t m_n;
    int m_B, m_m;

    LBFGSBatchSolver(const LBFGSBatchSolver&);
    LBFGSBatchSolver& operator=(const LBFGSBatchSolver&);

public:
    LBFGSBatchSolver(const LBFGSParam<Scalar>& param) : m_param(param), m_solver(nullptr), m_dev(nullptr), m_n(0), m_B(0), m_m(0)
    {
        m_param.check_param();
    }
    ~LBFGSBatchSolver() { lbfgs_b200_solver_destroy(m_solver); }

    // X holds the B start points back to back (problem b at [b*n, (b+1)*n)) and receives the solutions.  f describes the built-in
    // objective; its data vectors (if any) are shared by all problems.
    std::vector<BatchOutcome<Scalar> > minimize(BuiltinObjective<Scalar>& f, Vector& X, int B)
    {
        if (B < 1 || X.size() % B != 0) throw std::invalid_argument("LBFGSBatchSolver: X must hold B vectors of equal length");
        Device& dev = X.device();
        const std::ptrdiff_t n = X.size() / B;
        if (m_solver && (m_dev != &dev || m_n != n || m_B != B || m_m != m_param.m))
        {
            lbfgs_b200_solver_destroy(m_solver);
            m_solver = nullptr;
        }
        if (!m_solver)
        {
            dev.check(lbfgs_b200_solver_create_batch(dev.ctx(), n, m_param.m, int(sizeof(Scalar)), B, &m_solver));
            m_dev = &dev; m_n = n; m_B = B; m_m = m_param.m;
        }
        const lbfgs_b200_param p = detail::abi_param(m_param);
        std::vector<lbfgs_b200_outcome> raw((size_t)B);
        dev.check(detail::batch_abi<Scalar>::minimize(m_solver, f.builtin_kind(), f.builtin_data0(), f.builtin_data1(), 0, &p,
                                                      detail::line_search_id<LineSearch>::value, X.data(), int64_t(n), raw.data()));
        std::vector<BatchOutcome<Scalar> > out((size_t)B);
        for (int b = 0; b < B; b++)
        {
            out[size_t(b)].status = raw[size_t(b)].status; out[size_t(b)].niter = raw[size_t(b)].niter; out[size_t(b)].nfev = long(raw[size_t(b)].nfev);
            out[size_t(b)].fx = Scalar(raw[size_t(b)].fx); out[size_t(b)].gnorm = Scalar(raw[size_t(b)].gnorm); out[size_t(b)].rounds = long(raw[size_t(b)].rounds);
            f.add_calls(long(raw[size_t(b)].nfev));
        }
        return out;
    }
    // gradient of problem b at its solution (device pointer into the solver's storage, valid until the next minimize())
    const Scalar* final_grad(int b) const { return static_cast<const Scalar*>(lbfgs_b200_solver_final_grad_of(m_solver, b)); }
    // the solver object behind the last minimize() (nullptr before the first one): accounting via lbfgs_b200_solver_profile()
    lbfgs_b200_solver* solver_handle() const { return m_solver; }

    // LBFGSSolver::final_approx_hessian_times / final_approx_inverse_hessian_times for problem b of the last minimize(): OUT = B_b V
    // or H_b V, V holding k = V.size()/n vectors back to back.  The products are those of the same problem solved alone.
    void final_approx_hessian_times(int b, const Vector& V, Vector& OUT) { approx_times(b, V, OUT, false); }
    void final_approx_inverse_hessian_times(int b, const Vector& V, Vector& OUT) { approx_times(b, V, OUT, true); }
    // LBFGSSolver::final_approx_hessian_diagonal / final_approx_inverse_hessian_diagonal for problem b: bit-identical to the same
    // problem's diagonal solved alone.
    void final_approx_hessian_diagonal(int b, Vector& out) { approx_diagonal(b, out, false); }
    void final_approx_inverse_hessian_diagonal(int b, Vector& out) { approx_diagonal(b, out, true); }

    // LBFGSSolver::final_approx_inverse_hessian_factor_times / final_approx_sample / final_approx_inverse_hessian_logdet for problem
    // b, its draws from stream b: the same values as problem b solved alone with stream b.
    void final_approx_inverse_hessian_factor_times(int b, const Vector& V, Vector& OUT)
    {
        BFGSMat<Scalar> mat;
        borrow(b, mat);
        mat.inverse_hessian_factor_times(V, BFGSMat<Scalar>::block_count(V.size(), m_n), OUT);
    }
    void final_approx_sample(int b, const Vector& mean, unsigned long long seed, uint32_t first, int k, Vector& OUT)
    {
        BFGSMat<Scalar> mat;
        borrow(b, mat);
        mat.sample(&mean, seed, uint32_t(b), first, k, OUT);
    }
    double final_approx_inverse_hessian_logdet(int b)
    {
        BFGSMat<Scalar> mat;
        borrow(b, mat);
        return mat.inverse_hessian_logdet();
    }

    // LBFGSSolver::final_approx_inverse_hessian_factor_transpose_times / _solve / _transpose_solve / final_approx_log_density for
    // problem b: the same values as problem b solved alone.
    void final_approx_inverse_hessian_factor_transpose_times(int b, const Vector& V, Vector& OUT) { factor_op(b, LBFGS_B200_FACTOR_LT, V, OUT); }
    void final_approx_inverse_hessian_factor_solve(int b, const Vector& V, Vector& OUT) { factor_op(b, LBFGS_B200_FACTOR_LINV, V, OUT); }
    void final_approx_inverse_hessian_factor_transpose_solve(int b, const Vector& V, Vector& OUT) { factor_op(b, LBFGS_B200_FACTOR_LINVT, V, OUT); }
    std::vector<double> final_approx_log_density(int b, const Vector& mean, const Vector& X)
    {
        BFGSMat<Scalar> mat;
        borrow(b, mat);
        return mat.log_density(mean, X, BFGSMat<Scalar>::block_count(X.size(), m_n));
    }

private:
    void factor_op(int b, int op, const Vector& V, Vector& OUT)
    {
        BFGSMat<Scalar> mat;
        borrow(b, mat);
        const int k = BFGSMat<Scalar>::block_count(V.size(), m_n);
        if (op == LBFGS_B200_FACTOR_LT) mat.inverse_hessian_factor_transpose_times(V, k, OUT);
        else if (op == LBFGS_B200_FACTOR_LINV) mat.inverse_hessian_factor_solve(V, k, OUT);
        else mat.inverse_hessian_factor_transpose_solve(V, k, OUT);
    }

    void borrow(int b, BFGSMat<Scalar>& mat)
    {
        if (!m_solver) throw std::logic_error("LBFGSBatchSolver: no history yet (minimize() has not run)");
        if (b < 0 || b >= m_B) throw std::invalid_argument("LBFGSBatchSolver: problem index out of range");
        lbfgs_b200_hist* h = lbfgs_b200_solver_history_of(m_solver, b);   // column-major copy of problem b's ring
        if (!h) m_dev->check(LBFGS_B200_ERR_CUDA);
        mat.borrow(*m_dev, h, m_n, m_m);
    }

    void approx_diagonal(int b, Vector& out, bool inverse)
    {
        if (!m_solver) throw std::logic_error("LBFGSBatchSolver: no history yet (minimize() has not run)");
        if (b < 0 || b >= m_B) throw std::invalid_argument("LBFGSBatchSolver: problem index out of range");
        lbfgs_b200_hist* h = lbfgs_b200_solver_history_of(m_solver, b);   // column-major copy of problem b's ring
        if (!h) m_dev->check(LBFGS_B200_ERR_CUDA);
        BFGSMat<Scalar> mat;
        mat.borrow(*m_dev, h, m_n, m_m);
        if (inverse) mat.inverse_hessian_diagonal(out);
        else mat.hessian_diagonal(out);
    }

    void approx_times(int b, const Vector& V, Vector& OUT, bool inverse)
    {
        if (!m_solver) throw std::logic_error("LBFGSBatchSolver: no history yet (minimize() has not run)");
        if (b < 0 || b >= m_B) throw std::invalid_argument("LBFGSBatchSolver: problem index out of range");
        const int k = BFGSMat<Scalar>::block_count(V.size(), m_n);
        lbfgs_b200_hist* h = lbfgs_b200_solver_history_of(m_solver, b);   // column-major copy of problem b's ring
        if (!h) m_dev->check(LBFGS_B200_ERR_CUDA);
        BFGSMat<Scalar> mat;
        mat.borrow(*m_dev, h, m_n, m_m);
        if (inverse) mat.inverse_hessian_times(V, k, OUT);
        else mat.hessian_times(V, k, OUT);
    }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_LBFGS_BATCH_H
