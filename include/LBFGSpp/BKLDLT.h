// LBFGSpp/BKLDLT.h -- Bunch-Kaufman LDL' factorisation of the small symmetric indefinite "middle" matrices of L-BFGS-B.
//
// Role and interface of the reference's BKLDLT<Scalar> (reference include/LBFGSpp/BKLDLT.h:30-530): compute(mat, uplo),
// solve_inplace / solve, info(); std::invalid_argument for a non-square matrix (:395-396), std::logic_error when a solve is
// requested before compute() (:446-447), info() == NUMERICAL_ISSUE when a pivot block is singular.  The matrices are at
// most 2m x 2m (40 x 40 for m = 20), live on the host, and are factorised once per accepted correction pair, so this is
// scalar host code by design (SURVEY.md 8a row B5: "negligible").
//
// Own implementation: a dense square work array (not the reference's packed columns), an explicit global permutation, and a
// per-position block tag.   P A P' = L D L',  L unit lower triangular, D block diagonal with 1x1 and 2x2 blocks.
// Pivoting is the classical partial (Bunch-Kaufman 1977, "algorithm A") rule with alpha = (1 + sqrt(17)) / 8; the swap test
// uses |a(r,r)| >= alpha*sigma as published (the reference tests |a(k,k)| there, BKLDLT.h:252), so the two factorizations may
// pick different pivots on the same matrix; the solves agree to rounding (tests/test_front_cpu.py).
#ifndef LBFGSPP_B200_BKLDLT_H
#define LBFGSPP_B200_BKLDLT_H

#include <stdexcept>
#include <vector>

#include "CompactForm.h"
#include "SmallDense.h"

namespace LBFGSpp {

enum BKLDLT_UPLO { Lower = 0, Upper = 1 };

template <typename Scalar>
class BKLDLT
{
    int m_n;
    SmallMatrix<Scalar> m_w;              // strictly lower part: L;  diagonal (and sub-diagonal inside a pair): D
    std::vector<int> m_order;             // m_order[i] = original index now at position i
    std::vector<unsigned char> m_tag;     // BK_SINGLE / BK_PAIR_HEAD / BK_PAIR_TAIL
    int m_info;

public:
    BKLDLT() : m_n(0), m_info(NOT_COMPUTED) {}
    explicit BKLDLT(const SmallMatrix<Scalar>& mat, int uplo = Lower) : m_n(0), m_info(NOT_COMPUTED) { compute(mat, uplo); }

    // Only the `uplo` triangle of `mat` is read.  The factorisation itself is bk_factor (CompactForm.h).
    void compute(const SmallMatrix<Scalar>& mat, int uplo = Lower)
    {
        if (mat.rows() != mat.cols()) throw std::invalid_argument("BKLDLT: matrix must be square");
        const int n = m_n = mat.rows();
        m_w = SmallMatrix<Scalar>(n, n);
        for (int i = 0; i < n; i++)
            for (int j = 0; j <= i; j++) m_w(i, j) = m_w(j, i) = (uplo == Lower) ? mat(i, j) : mat(j, i);
        m_order.resize(size_t(n));
        m_tag.assign(size_t(n), (unsigned char)BK_SINGLE);
        m_info = bk_factor(m_w.data(), n, m_order.data(), m_tag.data()) == 0 ? SUCCESSFUL : NUMERICAL_ISSUE;
    }

    void solve_inplace(std::vector<Scalar>& b) const
    {
        if (m_info == NOT_COMPUTED) throw std::logic_error("BKLDLT: need to call compute() first");
        std::vector<Scalar> z(static_cast<size_t>(m_n));
        bk_solve(m_w.data(), m_n, m_order.data(), m_tag.data(), b.data(), 1, z.data());
    }
    std::vector<Scalar> solve(std::vector<Scalar> b) const
    {
        solve_inplace(b);
        return b;
    }
    int info() const { return m_info; }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_BKLDLT_H
