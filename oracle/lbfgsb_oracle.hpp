// lbfgsb_oracle.hpp -- TEST INFRASTRUCTURE ONLY.  CPU restatement of the bound-constrained solver of LBFGSpp.
//
// What it restates (reference @ ebef584, paths relative to the reference's include/):
//   PackedLDLT<T>                    LBFGSpp/BKLDLT.h:30-530     (Bunch-Kaufman LDL' of the 2m x 2m middle matrices)
//   BoxHistory<T>                    LBFGSpp/BFGSMat.h:81-146, 307-615  (BFGSMat<Scalar, true>)
//   cauchy_point                     LBFGSpp/Cauchy.h:31-50, 86-284
//   subspace_minimize                LBFGSpp/SubspaceMin.h:122-302
//   lbfgsb_minimize                  LBFGSB.h:55-86, 116-262
// Pinning: tests/test_oracle_cpu.py::test_pin_lbfgsb_* demand bit-for-bit equality with the unmodified reference headers
// compiled over oracle/minieigen (every sum strictly left to right, no FMA contraction, the same std::sort); to get there the
// expressions below are evaluated in the order minieigen evaluates the reference's (e.g. `theta * S' * v` scales S first).
#ifndef LBFGSB_ORACLE_HPP
#define LBFGSB_ORACLE_HPP

#include <algorithm>
#include <cmath>
#include <limits>
#include <stdexcept>
#include <utility>
#include <vector>

#include "lbfgs_oracle.hpp"

namespace orc {

// ---------------------------------------------------------------------------------------------------------------------
// Bunch-Kaufman LDL' on a packed lower triangle (column j holds rows j..n-1), BKLDLT.h
// ---------------------------------------------------------------------------------------------------------------------
template <class T>
class PackedLDLT
{
    long n_;
    std::vector<T> data_;
    std::vector<long> colstart_;                 // offset of column j in data_
    std::vector<long> perm_;                     // >= 0: 1x1 pivot swapped with perm; < 0: part of a 2x2 pivot, -perm-1
    std::vector<std::pair<long, long> > swaps_;  // compressed permutation
    bool computed_;
    int info_;  // 0 ok, 1 not computed, 2 numerical issue

    T& at(long i, long j) { return data_[colstart_[j] + (i - j)]; }
    const T& at(long i, long j) const { return data_[colstart_[j] + (i - j)]; }
    T* col(long j) { return &data_[colstart_[j]]; }

    // largest |a(i,k)|, i > k (BKLDLT.h:179-197)
    T below_diag_max(long k, long& r)
    {
        const T* head = col(k);
        const T* end = col(k) + (n_ - k);
        r = k + 1;
        T lambda = std::abs(head[1]);
        for (const T* p = head + 2; p < end; p++)
        {
            const T a = std::abs(*p);
            if (lambda < a)
            {
                lambda = a;
                r = k + (p - head);
            }
        }
        return lambda;
    }
    // largest off-diagonal magnitude in row/column r of the trailing block (BKLDLT.h:203-222)
    T row_col_max(long k, long r, long& p)
    {
        T sigma = T(-1);
        if (r < n_ - 1) sigma = below_diag_max(r, p);
        for (long j = k; j < r; j++)
        {
            const T a = std::abs(at(r, j));
            if (sigma < a)
            {
                sigma = a;
                p = j;
            }
        }
        return sigma;
    }
    void swap_1x1(long k, long r)  // BKLDLT.h:118-142
    {
        if (k == r)
        {
            perm_[k] = r;
            return;
        }
        std::swap(at(k, k), at(r, r));
        std::swap_ranges(&at(r + 1, k), col(k) + (n_ - k), &at(r + 1, r));
        T* src = &at(k + 1, k);
        for (long j = k + 1; j < r; j++, src++) std::swap(*src, at(r, j));
        perm_[k] = r;
    }
    void swap_2x2(long k, long r, long p)  // BKLDLT.h:150-164
    {
        swap_1x1(k, p);
        swap_1x1(k + 1, r);
        std::swap(at(k + 1, k), at(r, k));
        perm_[k] = -perm_[k] - 1;
        perm_[k + 1] = -perm_[k + 1] - 1;
    }
    void swap_rows(long r1, long r2, long c1, long c2)  // BKLDLT.h:167-176
    {
        if (r1 == r2) return;
        for (long j = c1; j <= c2; j++) std::swap(at(r1, j), at(r2, j));
    }
    // choose the pivot for step k; true = 1x1 (BKLDLT.h:230-285)
    bool choose_pivot(long k, T alpha)
    {
        long r = k, p = k;
        const T lambda = below_diag_max(k, r);
        if (lambda > T(0))
        {
            const T akk = std::abs(at(k, k));
            if (akk < alpha * lambda)
            {
                const T sigma = row_col_max(k, r, p);
                if (sigma * akk < alpha * lambda * lambda)
                {
                    if (akk >= alpha * sigma)
                    {
                        swap_1x1(k, r);
                        swap_rows(k, r, 0, k - 1);
                        return true;
                    }
                    p = k;
                    swap_2x2(k, r, p);
                    swap_rows(k, p, 0, k - 1);
                    swap_rows(k + 1, r, 0, k - 1);
                    return false;
                }
            }
        }
        return true;
    }
    int eliminate_1x1(long k)  // BKLDLT.h:300-326
    {
        const T akk = at(k, k);
        if (akk == T(0)) return 2;
        at(k, k) = T(1) / akk;
        T* l = col(k) + 1;
        const long ldim = n_ - k - 1;
        for (long j = 0; j < ldim; j++)
        {
            T* dst = col(j + k + 1);
            const T f = l[j] / akk;
            for (long i = 0; i < ldim - j; i++) dst[i] -= f * l[j + i];
        }
        for (long i = 0; i < ldim; i++) l[i] /= akk;
        return 0;
    }
    int eliminate_2x2(long k)  // BKLDLT.h:329-364
    {
        T& e11 = at(k, k);
        T& e21 = at(k + 1, k);
        T& e22 = at(k + 1, k + 1);
        if (e11 * e22 - e21 * e21 == T(0)) return 2;
        {
            const T delta = e11 * e22 - e21 * e21;  // in-place inverse of the 2x2 block (BKLDLT.h:288-295)
            std::swap(e11, e22);
            e11 /= delta;
            e22 /= delta;
            e21 = -e21 / delta;
        }
        T* l1 = &at(k + 2, k);
        T* l2 = &at(k + 2, k + 1);
        const long ldim = n_ - k - 2;
        std::vector<T> x0(ldim), x1(ldim);
        for (long i = 0; i < ldim; i++) x0[i] = l1[i] * e11 + l2[i] * e21;
        for (long i = 0; i < ldim; i++) x1[i] = l1[i] * e21 + l2[i] * e22;
        for (long j = 0; j < ldim; j++)
        {
            T* dst = col(j + k + 2);
            for (long i = 0; i < ldim - j; i++) dst[i] -= (x0[j + i] * l1[j] + x1[j + i] * l2[j]);
        }
        for (long i = 0; i < ldim; i++) l1[i] = x0[i];
        for (long i = 0; i < ldim; i++) l2[i] = x1[i];
        return 0;
    }

public:
    PackedLDLT() : n_(0), computed_(false), info_(1) {}

    // `a` is column-major with leading dimension lda; only the lower triangle is read (BKLDLT.h:390-441)
    void compute(const T* a, long n, long lda)
    {
        n_ = n;
        perm_.resize(n);
        if (n == 1) perm_[0] = 0;  // setLinSpaced(1, 0, 0) yields `high`
        else for (long i = 0; i < n; i++) perm_[i] = 0 + i * ((n - 1) - 0) / (n - 1);
        swaps_.clear();
        data_.assign(size_t(n * (n + 1) / 2), T(0));
        colstart_.resize(n);
        long off = 0;
        for (long j = 0; j < n; j++)
        {
            colstart_[j] = off;
            off += n - j;
        }
        for (long j = 0; j < n; j++)
            for (long i = j; i < n; i++) at(i, j) = a[i + j * lda];
        const T alpha = T((1.0 + std::sqrt(17.0)) / 8.0);
        info_ = 1;
        long k = 0;
        for (k = 0; k < n - 1; k++)
        {
            const bool one = choose_pivot(k, alpha);
            if (one)
                info_ = eliminate_1x1(k);
            else
            {
                info_ = eliminate_2x2(k);
                k++;
            }
            if (info_ != 0) break;
        }
        if (k == n - 1)
        {
            const T akk = at(k, k);
            if (akk == T(0)) info_ = 2;
            at(k, k) = T(1) / at(k, k);
        }
        for (long i = 0; i < n; i++)
        {
            const long p = (perm_[i] >= 0) ? perm_[i] : (-perm_[i] - 1);
            if (p != i) swaps_.push_back(std::make_pair(i, p));
        }
        computed_ = true;
    }

    void solve_inplace(T* x) const  // BKLDLT.h:444-520
    {
        if (!computed_) throw std::logic_error("BKLDLT: need to call compute() first");
        const long np = long(swaps_.size());
        for (long i = 0; i < np; i++) std::swap(x[swaps_[i].first], x[swaps_[i].second]);
        const long end = (perm_[n_ - 1] < 0) ? (n_ - 3) : (n_ - 2);
        for (long i = 0; i <= end; i++)
        {
            const long b1 = n_ - i - 1, b2 = b1 - 1;
            if (perm_[i] >= 0)
            {
                const T* l = &at(i + 1, i);
                for (long t = 0; t < b1; t++) x[i + 1 + t] -= l[t] * x[i];
            }
            else
            {
                const T* l1 = &at(i + 2, i);
                const T* l2 = &at(i + 2, i + 1);
                for (long t = 0; t < b2; t++) x[i + 2 + t] -= (l1[t] * x[i] + l2[t] * x[i + 1]);
                i++;
            }
        }
        for (long i = 0; i < n_; i++)
        {
            const T e11 = at(i, i);
            if (perm_[i] >= 0)
                x[i] *= e11;
            else
            {
                const T e21 = at(i + 1, i), e22 = at(i + 1, i + 1);
                const T wi = x[i] * e11 + x[i + 1] * e21;
                x[i + 1] = x[i] * e21 + x[i + 1] * e22;
                x[i] = wi;
                i++;
            }
        }
        long i = (perm_[n_ - 1] < 0) ? (n_ - 3) : (n_ - 2);
        for (; i >= 0; i--)
        {
            const long ldim = n_ - i - 1;
            const T* l = &at(i + 1, i);
            T acc = T(0);
            for (long t = 0; t < ldim; t++) acc += x[i + 1 + t] * l[t];
            x[i] -= acc;
            if (perm_[i] < 0)
            {
                const T* l2 = &at(i + 1, i - 1);
                T acc2 = T(0);
                for (long t = 0; t < ldim; t++) acc2 += x[i + 1 + t] * l2[t];
                x[i - 1] -= acc2;
                i--;
            }
        }
        for (i = np - 1; i >= 0; i--) std::swap(x[swaps_[i].first], x[swaps_[i].second]);
    }
    int info() const { return info_; }
};

// ---------------------------------------------------------------------------------------------------------------------
// BFGSMat<Scalar, true>
// ---------------------------------------------------------------------------------------------------------------------
template <class T>
struct BoxHistory
{
    typedef std::vector<T> V;
    typedef std::vector<int> IndexSet;
    long n;
    int m, ncorr, ptr;
    T theta;
    V S, Y;        // n x m column-major
    V ys;
    V Minv;        // permuted M inverse, 2m x 2m column-major
    PackedLDLT<T> Msolver;

    T* s_col(int j) { return &S[size_t(j) * n]; }
    T* y_col(int j) { return &Y[size_t(j) * n]; }
    const T* s_col(int j) const { return &S[size_t(j) * n]; }
    const T* y_col(int j) const { return &Y[size_t(j) * n]; }
    T& mi(int i, int j) { return Minv[size_t(i) + size_t(j) * 2 * m]; }
    const T& mi(int i, int j) const { return Minv[size_t(i) + size_t(j) * 2 * m]; }

    void reset(long n_, int m_)  // BFGSMat.h:61-78
    {
        n = n_;
        m = m_;
        theta = T(1);
        S.assign(size_t(n) * m, T(0));
        Y.assign(size_t(n) * m, T(0));
        ys.assign(m, T(0));
        ncorr = 0;
        ptr = m;
        Minv.assign(size_t(4) * m * m, T(0));
        for (int i = 0; i < 2 * m; i++) mi(i, i) = T(1);
    }

    static T dot(const T* a, const T* b, long len)
    {
        T acc = T(0);
        for (long i = 0; i < len; i++) acc += a[i] * b[i];
        return acc;
    }

    void add(const T* s, const T* y)  // BFGSMat.h:81-146
    {
        const int loc = ptr % m;
        std::copy(s, s + n, s_col(loc));
        std::copy(y, y + n, y_col(loc));
        const T sy = dot(s_col(loc), y_col(loc), n);
        ys[loc] = sy;
        theta = dot(y_col(loc), y_col(loc), n) / sy;
        if (ncorr < m) ncorr++;
        ptr = loc + 1;

        mi(loc, loc) = -sy;
        V Ss(ncorr);
        for (int i = 0; i < ncorr; i++) Ss[i] = dot(s_col(i), s_col(loc), n);
        for (int i = 0; i < ncorr; i++) mi(m + loc, m + i) = Ss[i];
        for (int i = 0; i < ncorr; i++) mi(m + i, m + loc) = Ss[i];
        const int len = ncorr - 1;
        if (ncorr >= m)
            for (int i = 0; i < m; i++) mi(m + i, loc) = T(0);
        int yloc = (loc + m - 1) % m;
        for (int i = 0; i < len; i++)
        {
            mi(m + loc, yloc) = dot(s_col(loc), y_col(yloc), n);
            yloc = (yloc + m - 1) % m;
        }
        for (int j = 0; j < m; j++)
            for (int i = 0; i < m; i++) mi(m + i, m + j) *= theta;
        Msolver.compute(Minv.data(), 2 * m, 2 * m);
        for (int j = 0; j < m; j++)
            for (int i = 0; i < m; i++) mi(m + i, m + j) /= theta;
    }

    // res = [Y'v ; theta*S'v] (BFGSMat.h:315-320; theta scales S before the product, as minieigen evaluates it)
    void apply_Wtv(const V& v, V& res) const
    {
        res.assign(size_t(2 * ncorr), T(0));
        for (int i = 0; i < ncorr; i++) res[i] = dot(y_col(i), v.data(), n);
        for (int i = 0; i < ncorr; i++)
        {
            T acc = T(0);
            const T* sc = s_col(i);
            for (long k = 0; k < n; k++) acc += (theta * sc[k]) * v[k];
            res[ncorr + i] = acc;
        }
    }
    V Wb(int b) const  // BFGSMat.h:325-335
    {
        V res(static_cast<size_t>(2 * ncorr));
        for (int j = 0; j < ncorr; j++)
        {
            res[j] = y_col(j)[b];
            res[ncorr + j] = s_col(j)[b];
        }
        for (int j = 0; j < ncorr; j++) res[ncorr + j] *= theta;
        return res;
    }
    // rows of [Y S] (no theta), nb x 2c column-major (BFGSMat.h:338-358)
    V Wb(const IndexSet& b) const
    {
        const long nb = long(b.size());
        V res(static_cast<size_t>(nb) * 2 * ncorr);
        for (int j = 0; j < ncorr; j++)
            for (long i = 0; i < nb; i++)
            {
                res[size_t(j) * nb + i] = y_col(j)[b[i]];
                res[size_t(ncorr + j) * nb + i] = s_col(j)[b[i]];
            }
        return res;
    }
    void apply_Mv(const V& v, V& res) const  // BFGSMat.h:361-378
    {
        res.assign(size_t(2 * ncorr), T(0));
        if (ncorr < 1) return;
        V pad(static_cast<size_t>(2 * m), T(0));
        for (int i = 0; i < ncorr; i++) pad[i] = v[i];
        for (int i = 0; i < ncorr; i++) pad[m + i] = v[ncorr + i];
        Msolver.solve_inplace(pad.data());
        for (int i = 0; i < ncorr; i++) res[i] = pad[i];
        for (int i = 0; i < ncorr; i++) res[ncorr + i] = pad[m + i];
    }
    bool apply_WtPv(const IndexSet& P, const V& v, V& res, bool test_zero = false) const  // BFGSMat.h:382-433
    {
        const int* Pp = P.data();
        const T* vp = v.data();
        long nP = long(P.size());
        IndexSet Pr;
        V vr;
        if (test_zero)
        {
            Pr.reserve(nP);
            for (long i = 0; i < nP; i++)
                if (vp[i] != T(0))
                {
                    Pr.push_back(Pp[i]);
                    vr.push_back(vp[i]);
                }
            Pp = Pr.data();
            vp = vr.data();
            nP = long(Pr.size());
        }
        res.assign(size_t(2 * ncorr), T(0));
        if (ncorr < 1 || nP < 1) return false;
        for (int j = 0; j < ncorr; j++)
        {
            T ry = T(0), rs = T(0);
            const T* yp = y_col(j);
            const T* sp = s_col(j);
            for (long i = 0; i < nP; i++)
            {
                const int row = Pp[i];
                ry += yp[row] * vp[i];
                rs += sp[row] * vp[i];
            }
            res[j] = ry;
            res[ncorr + j] = rs;
        }
        for (int j = 0; j < ncorr; j++) res[ncorr + j] *= theta;
        return true;
    }
    bool apply_PtWMv(const IndexSet& P, const V& v, V& res, T scale) const  // BFGSMat.h:435-460
    {
        const long nP = long(P.size());
        res.assign(size_t(nP), T(0));
        if (ncorr < 1 || nP < 1) return false;
        V Mv;
        apply_Mv(v, Mv);
        for (int j = 0; j < ncorr; j++) Mv[ncorr + j] *= theta;
        for (int j = 0; j < ncorr; j++)
        {
            const T* yp = y_col(j);
            const T* sp = s_col(j);
            const T my = Mv[j], ms = Mv[ncorr + j];
            for (long i = 0; i < nP; i++) res[i] += my * yp[P[i]] + ms * sp[P[i]];
        }
        for (long i = 0; i < nP; i++) res[i] *= scale;
        return true;
    }
    bool apply_PtWMv(const V& WP, long nP, const V& v, V& res, T scale) const  // BFGSMat.h:462-478
    {
        res.assign(size_t(nP), T(0));
        if (ncorr < 1 || nP < 1) return false;
        V Mv;
        apply_Mv(v, Mv);
        for (int j = 0; j < ncorr; j++) Mv[ncorr + j] *= theta;
        for (long i = 0; i < nP; i++)
        {
            T acc = T(0);
            for (int k = 0; k < 2 * ncorr; k++) acc += WP[size_t(k) * nP + i] * Mv[k];
            res[i] = scale * acc;
        }
        return true;
    }
    void compute_FtBAb(const V& WF, const IndexSet& fv, const IndexSet& act, const V& Wd, const V& drt, V& res) const  // :486-522
    {
        const long nact = long(act.size()), nfree = long(fv.size());
        res.assign(size_t(nfree), T(0));
        if (ncorr < 1 || nact < 1 || nfree < 1) return;
        V rhs(static_cast<size_t>(2 * ncorr));
        if (nact <= nfree)
        {
            V Ad(static_cast<size_t>(nfree), T(0));
            for (long i = 0; i < nact; i++) Ad[i] = drt[act[i]];
            apply_WtPv(act, Ad, rhs);
        }
        else
        {
            V Fd(static_cast<size_t>(nfree));
            for (long i = 0; i < nfree; i++) Fd[i] = drt[fv[i]];
            for (int j = 0; j < 2 * ncorr; j++)
            {
                T acc = T(0);
                for (long k = 0; k < nfree; k++) acc += WF[size_t(j) * nfree + k] * Fd[k];
                rhs[j] = acc;
            }
            for (int j = 0; j < ncorr; j++) rhs[ncorr + j] *= theta;
            for (int j = 0; j < 2 * ncorr; j++) rhs[j] = Wd[j] - rhs[j];
        }
        apply_PtWMv(WF, nfree, rhs, res, T(-1));
    }
    void solve_PtBP(const V& WP, long nP, const V& v, V& res) const  // BFGSMat.h:529-565
    {
        res.assign(size_t(nP), T(0));
        if (ncorr < 1 || nP < 1)
        {
            for (long i = 0; i < nP; i++) res[i] = v[i] / theta;
            return;
        }
        const int c = ncorr, w = 2 * ncorr;
        V mid(static_cast<size_t>(w) * w, T(0));
        auto wp = [&](long k, int col) -> const T& { return WP[size_t(col) * nP + k]; };
        auto dotcols = [&](int a, int b) {
            T acc = T(0);
            for (long k = 0; k < nP; k++) acc += wp(k, a) * wp(k, b);
            return acc;
        };
        for (int j = 0; j < c; j++)
            for (int i = 0; i < c - j; i++) mid[size_t(j + i) + size_t(j) * w] = mi(j + i, j) - dotcols(j + i, j) / theta;
        for (int b = 0; b < c; b++)
            for (int a = 0; a < c; a++) mid[size_t(c + a) + size_t(b) * w] = mi(m + a, b) - dotcols(c + a, b);
        for (int j = 0; j < c; j++)
            for (int i = 0; i < c - j; i++)
                mid[size_t(c + j + i) + size_t(c + j) * w] = theta * (mi(m + j + i, m + j) - dotcols(c + j + i, c + j));
        PackedLDLT<T> midsolver;
        midsolver.compute(mid.data(), w, w);
        V WPv(static_cast<size_t>(w));
        for (int j = 0; j < w; j++)
        {
            T acc = T(0);
            for (long k = 0; k < nP; k++) acc += wp(k, j) * v[k];
            WPv[j] = acc;
        }
        for (int j = 0; j < c; j++) WPv[c + j] *= theta;
        midsolver.solve_inplace(WPv.data());
        for (int j = 0; j < c; j++) WPv[c + j] *= theta;
        for (long i = 0; i < nP; i++)
        {
            T acc = T(0);
            for (int k = 0; k < w; k++) acc += wp(i, k) * WPv[k];
            res[i] = v[i] / theta + acc / (theta * theta);
        }
    }
    bool apply_PtBQv(const V& WP, long nP, const IndexSet& Q, const V& v, V& res, bool test_zero = false) const  // :570-594
    {
        const long nQ = long(Q.size());
        res.assign(size_t(nP), T(0));
        if (ncorr < 1 || nP < 1 || nQ < 1) return false;
        V WQtv;
        if (!apply_WtPv(Q, v, WQtv, test_zero)) return false;
        V MWQtv;
        apply_Mv(WQtv, MWQtv);
        for (int j = 0; j < ncorr; j++) MWQtv[ncorr + j] *= theta;
        for (long i = 0; i < nP; i++)
        {
            T acc = T(0);
            for (int k = 0; k < 2 * ncorr; k++) acc += (-WP[size_t(k) * nP + i]) * MWQtv[k];
            res[i] = acc;
        }
        return true;
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// generalized Cauchy point (Cauchy.h:86-284)
// ---------------------------------------------------------------------------------------------------------------------
template <class T>
void cauchy_point(const BoxHistory<T>& bfgs, const std::vector<T>& x0, const std::vector<T>& g, const std::vector<T>& lb,
                  const std::vector<T>& ub, std::vector<T>& xcp, std::vector<T>& vecc, std::vector<int>& newact, std::vector<int>& fv)
{
    typedef std::vector<T> V;
    const long n = long(x0.size());
    xcp = x0;
    vecc.assign(size_t(2 * bfgs.ncorr), T(0));
    newact.clear();
    fv.clear();
    V brk(n), d(n);
    std::vector<int> ord;
    const T inf = std::numeric_limits<T>::infinity();
    for (long i = 0; i < n; i++)
    {
        if (lb[i] == ub[i]) brk[i] = T(0);
        else if (g[i] < T(0)) brk[i] = (x0[i] - ub[i]) / g[i];
        else if (g[i] > T(0)) brk[i] = (x0[i] - lb[i]) / g[i];
        else brk[i] = inf;
        const bool zero = (brk[i] == T(0));
        d[i] = zero ? T(0) : -g[i];
        if (brk[i] == inf) fv.push_back(int(i));
        else if (!zero) ord.push_back(int(i));
    }
    const T* values = brk.data();
    std::sort(ord.begin(), ord.end(), [values](int a, int b) { return values[a] < values[b]; });
    const long nord = long(ord.size()), nfree = long(fv.size());
    if (nfree < 1 && nord < 1) return;

    V p;
    bfgs.apply_Wtv(d, p);
    T fp = T(0);
    for (long i = 0; i < n; i++) fp += d[i] * d[i];
    fp = -fp;
    V cache;
    bfgs.apply_Mv(p, cache);
    T pc = T(0);
    for (size_t k = 0; k < p.size(); k++) pc += p[k] * cache[k];
    T fpp = -bfgs.theta * fp - pc;
    T dtmin = -fp / fpp;
    T il = T(0);
    long b = 0;
    T iu = (nord < 1) ? inf : brk[ord[b]];
    T dt = iu - il;
    bool crossed_all = false;
    const int c = bfgs.ncorr;
    V wact(static_cast<size_t>(2 * c));
    while (dtmin >= dt)
    {
        for (int k = 0; k < 2 * c; k++) vecc[k] += dt * p[k];
        const long act_begin = b;
        long e = b;
        for (; e < nord; e++)
            if (brk[ord[e]] > iu) break;
        const long act_end = e - 1;
        if (nfree == 0 && act_end == nord - 1)
        {
            for (long i = act_begin; i <= act_end; i++)
            {
                const int a = ord[i];
                xcp[a] = (d[a] > T(0)) ? ub[a] : lb[a];
                newact.push_back(a);
            }
            crossed_all = true;
            break;
        }
        fp += dt * fpp;
        for (long i = act_begin; i <= act_end; i++)
        {
            const int a = ord[i];
            xcp[a] = (d[a] > T(0)) ? ub[a] : lb[a];
            const T zact = xcp[a] - x0[a];
            const T gact = g[a];
            const T ggact = gact * gact;
            wact = bfgs.Wb(a);
            bfgs.apply_Mv(wact, cache);
            T cvc = T(0), cvp = T(0), cvw = T(0);
            for (int k = 0; k < 2 * c; k++) cvc += cache[k] * vecc[k];
            for (int k = 0; k < 2 * c; k++) cvp += cache[k] * p[k];
            for (int k = 0; k < 2 * c; k++) cvw += cache[k] * wact[k];
            fp += ggact + bfgs.theta * gact * zact - gact * cvc;
            fpp -= (bfgs.theta * ggact + 2 * gact * cvp + ggact * cvw);
            for (int k = 0; k < 2 * c; k++) p[k] += gact * wact[k];
            d[a] = T(0);
            newact.push_back(a);
        }
        dtmin = -fp / fpp;
        il = iu;
        b = act_end + 1;
        if (b >= nord) break;
        iu = brk[ord[b]];
        dt = iu - il;
    }
    const T eps = std::numeric_limits<T>::epsilon();
    if (fpp < eps) dtmin = -fp / eps;
    if (!crossed_all)
    {
        dtmin = std::max(dtmin, T(0));
        for (int k = 0; k < 2 * c; k++) vecc[k] += dtmin * p[k];
        const T tfinal = il + dtmin;
        for (long i = 0; i < nfree; i++)
        {
            const int co = fv[i];
            xcp[co] = x0[co] + tfinal * d[co];
        }
        for (long i = b; i < nord; i++)
        {
            const int co = ord[i];
            xcp[co] = x0[co] + tfinal * d[co];
            fv.push_back(co);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// subspace minimisation (SubspaceMin.h:122-302)
// ---------------------------------------------------------------------------------------------------------------------
template <class T>
void subspace_minimize(const BoxHistory<T>& bfgs, const std::vector<T>& x0, const std::vector<T>& xcp, const std::vector<T>& g,
                       const std::vector<T>& lb, const std::vector<T>& ub, const std::vector<T>& Wd, const std::vector<int>& newact,
                       const std::vector<int>& fv, int maxit, std::vector<T>& drt)
{
    typedef std::vector<T> V;
    typedef std::vector<int> IndexSet;
    const long n = long(x0.size());
    drt.resize(n);
    for (long i = 0; i < n; i++) drt[i] = xcp[i] - x0[i];
    const long nfree = long(fv.size());
    if (nfree < 1) return;
    const V WF = bfgs.Wb(fv);
    V vecc;
    bfgs.compute_FtBAb(WF, fv, newact, Wd, drt, vecc);
    V vecl(nfree), vecu(nfree);
    for (long i = 0; i < nfree; i++)
    {
        const int co = fv[i];
        vecl[i] = lb[co] - x0[co];
        vecu[i] = ub[co] - x0[co];
        vecc[i] += g[co];
    }
    V negc(nfree);
    for (long i = 0; i < nfree; i++) negc[i] = -vecc[i];
    V vecy;
    bfgs.solve_PtBP(WF, nfree, negc, vecy);
    bool inside = true;
    for (long i = 0; i < nfree; i++)
        if (vecy[i] < vecl[i] || vecy[i] > vecu[i])
        {
            inside = false;
            break;
        }
    auto assign_free = [&](const V& v) {
        for (long i = 0; i < nfree; i++) drt[fv[i]] = v[i];
    };
    if (inside)
    {
        assign_free(vecy);
        return;
    }
    const V yfallback = vecy;
    V lambda(nfree, T(0)), mu(nfree, T(0));
    IndexSet L, U, P, yL, yU, yP;
    auto subvec = [](const V& v, const IndexSet& ind) {
        V r(ind.size());
        for (size_t i = 0; i < ind.size(); i++) r[i] = v[ind[i]];
        return r;
    };
    int k;
    for (k = 0; k < maxit; k++)
    {
        L.clear(); U.clear(); P.clear(); yL.clear(); yU.clear(); yP.clear();
        for (long i = 0; i < nfree; i++)
        {
            const int co = fv[i];
            const T li = vecl[i], ui = vecu[i];
            if ((vecy[i] < li) || (vecy[i] == li && lambda[i] >= T(0)))
            {
                L.push_back(co); yL.push_back(int(i)); vecy[i] = li; mu[i] = T(0);
            }
            else if ((vecy[i] > ui) || (vecy[i] == ui && mu[i] >= T(0)))
            {
                U.push_back(co); yU.push_back(int(i)); vecy[i] = ui; lambda[i] = T(0);
            }
            else
            {
                P.push_back(co); yP.push_back(int(i)); lambda[i] = T(0); mu[i] = T(0);
            }
        }
        const V WP = bfgs.Wb(P);
        const long nP = long(P.size());
        if (nP > 0)
        {
            V rhs = subvec(vecc, yP);
            const V lL = subvec(vecl, yL), uU = subvec(vecu, yU);
            V tmp;
            if (bfgs.apply_PtBQv(WP, nP, L, lL, tmp, true))
                for (long i = 0; i < nP; i++) rhs[i] += tmp[i];
            if (bfgs.apply_PtBQv(WP, nP, U, uU, tmp, true))
                for (long i = 0; i < nP; i++) rhs[i] += tmp[i];
            V negrhs(nP);
            for (long i = 0; i < nP; i++) negrhs[i] = -rhs[i];
            bfgs.solve_PtBP(WP, nP, negrhs, tmp);
            for (long i = 0; i < nP; i++) vecy[yP[i]] = tmp[i];
        }
        const long nL = long(L.size()), nU = long(U.size());
        V Fy;
        if (nL > 0 || nU > 0) bfgs.apply_WtPv(fv, vecy, Fy);
        if (nL > 0)
        {
            V res;
            bfgs.apply_PtWMv(L, Fy, res, T(-1));
            const V cL = subvec(vecc, yL), yLv = subvec(vecy, yL);
            for (long i = 0; i < nL; i++) res[i] += cL[i] + bfgs.theta * yLv[i];
            for (long i = 0; i < nL; i++) lambda[yL[i]] = res[i];
        }
        if (nU > 0)
        {
            V neg;
            bfgs.apply_PtWMv(U, Fy, neg, T(-1));
            const V cU = subvec(vecc, yU), yUv = subvec(vecy, yU);
            for (long i = 0; i < nU; i++) neg[i] += cU[i] + bfgs.theta * yUv[i];
            for (long i = 0; i < nU; i++) mu[yU[i]] = -neg[i];
        }
        bool okL = true, okU = true, okP = true;
        for (size_t i = 0; i < yL.size(); i++)
            if (lambda[yL[i]] < T(0)) { okL = false; break; }
        for (size_t i = 0; i < yU.size(); i++)
            if (mu[yU[i]] < T(0)) { okU = false; break; }
        for (size_t i = 0; i < yP.size(); i++)
        {
            const int co = yP[i];
            if (vecy[co] < vecl[co] || vecy[co] > vecu[co]) { okP = false; break; }
        }
        if (okL && okU && okP) break;
    }
    if (k >= maxit)
    {
        auto project = [&](const V& v) {
            V r(nfree);
            for (long i = 0; i < nfree; i++) r[i] = std::min(std::max(v[i], vecl[i]), vecu[i]);
            return r;
        };
        auto dirderiv = [&]() {
            T acc = T(0);
            for (long i = 0; i < n; i++) acc += drt[i] * g[i];
            return acc;
        };
        const T eps = std::numeric_limits<T>::epsilon();
        vecy = project(vecy);
        assign_free(vecy);
        if (dirderiv() <= -eps) return;
        vecy = project(yfallback);
        assign_free(vecy);
        if (dirderiv() <= -eps) return;
        assign_free(yfallback);
        return;
    }
    assign_free(vecy);
}

// ---------------------------------------------------------------------------------------------------------------------
// LBFGSBSolver<Scalar, LineSearchMoreThuente>::minimize (LBFGSB.h:116-262)
// ---------------------------------------------------------------------------------------------------------------------
template <class T, class F>
LbfgsOutcome<T> lbfgsb_minimize(F& f, const orc_param& prm, const Blas1<T>& la, Vec<T>& x, const Vec<T>& lb, const Vec<T>& ub)
{
    using std::abs;
    check_lbfgs_param(prm, true);
    const long n = long(x.size());
    if (long(lb.size()) != n || long(ub.size()) != n) throw std::invalid_argument("'lb' and 'ub' must have the same size as 'x'");
    auto force_bounds = [&](Vec<T>& v) {
        for (long i = 0; i < n; i++) v[i] = std::min(std::max(v[i], lb[i]), ub[i]);
    };
    auto proj_grad_norm = [&](const Vec<T>& xv, const Vec<T>& gv) {
        T best = T(0);
        for (long i = 0; i < n; i++)
        {
            const T p = abs(std::min(std::max(xv[i] - gv[i], lb[i]), ub[i]) - xv[i]);
            if (i == 0 || p > best) best = p;
        }
        return best;
    };
    auto max_step_size = [&](const Vec<T>& x0, const Vec<T>& d) {
        T step = std::numeric_limits<T>::infinity();
        for (long i = 0; i < n; i++)
        {
            if (d[i] > T(0)) step = std::min(step, (ub[i] - x0[i]) / d[i]);
            else if (d[i] < T(0)) step = std::min(step, (lb[i] - x0[i]) / d[i]);
        }
        return step;
    };

    force_bounds(x);
    BoxHistory<T> bfgs;
    bfgs.reset(n, prm.m);
    Vec<T> xp(n), grad(n), gradp(n), drt(n), fxs(prm.past > 0 ? prm.past : 0);
    const int fpast = prm.past;
    LbfgsOutcome<T> out;
    T fx = f(x.data(), grad.data());
    T pg = proj_grad_norm(x, grad);
    if (fpast > 0) fxs[0] = fx;
    auto finish = [&](int k) {
        out.niter = k;
        out.fx = fx;
        out.gnorm = pg;
        out.grad.swap(grad);
        return out;
    };
    if (pg <= T(prm.epsilon) || pg <= T(prm.epsilon_rel) * la.norm(x.data(), n)) return finish(1);

    Vec<T> xcp(n), vecc;
    std::vector<int> newact, fv;
    cauchy_point(bfgs, x, grad, lb, ub, xcp, vecc, newact, fv);
    for (long i = 0; i < n; i++) drt[i] = xcp[i] - x[i];
    {
        const T z = la.sqnorm(drt.data(), n);
        if (z > T(0))
        {
            const T nrm = std::sqrt(z);
            for (long i = 0; i < n; i++) drt[i] /= nrm;
        }
    }
    const T eps = std::numeric_limits<T>::epsilon();
    Vec<T> s(n), y(n);
    int k = 1;
    for (;;)
    {
        xp = x;
        gradp = grad;
        T dg = la.dot(grad.data(), drt.data(), n);
        T step_max = max_step_size(x, drt);
        if (dg >= T(0) || step_max <= T(prm.min_step))
        {
            for (long i = 0; i < n; i++) drt[i] = xcp[i] - x[i];
            bfgs.reset(n, prm.m);
            dg = la.dot(grad.data(), drt.data(), n);
            step_max = max_step_size(x, drt);
        }
        step_max = std::min(T(prm.max_step), step_max);
        T step = T(1);
        step = std::min(step, step_max);
        ls_more_thuente(f, prm, la, xp, drt, step_max, step, fx, grad, dg, x);
        pg = proj_grad_norm(x, grad);
        if (pg <= T(prm.epsilon) || pg <= T(prm.epsilon_rel) * la.norm(x.data(), n)) return finish(k);
        if (fpast > 0)
        {
            const T fxd = fxs[k % fpast];
            if (k >= fpast && abs(fxd - fx) <= T(prm.delta) * std::max(std::max(abs(fx), abs(fxd)), T(1))) return finish(k);
            fxs[k % fpast] = fx;
        }
        if (prm.max_iterations != 0 && k >= prm.max_iterations) return finish(k);
        la.diff(s.data(), x.data(), xp.data(), n);
        la.diff(y.data(), grad.data(), gradp.data(), n);
        if (la.dot(s.data(), y.data(), n) > eps * la.sqnorm(y.data(), n)) bfgs.add(s.data(), y.data());
        force_bounds(x);
        cauchy_point(bfgs, x, grad, lb, ub, xcp, vecc, newact, fv);
        subspace_minimize(bfgs, x, xcp, grad, lb, ub, vecc, newact, fv, prm.max_submin, drt);
        k++;
    }
}

}  // namespace orc
#endif
