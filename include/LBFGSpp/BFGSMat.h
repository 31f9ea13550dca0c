// LBFGSpp/BFGSMat.h -- the limited-memory quasi-Newton matrix, resident in HBM.
//
// Front for the S/Y ring kept by liblbfgs_b200 (lbfgs_b200_hist).  It offers the members of the reference's
// BFGSMat<Scalar> that the unconstrained solver uses (reference include/LBFGSpp/BFGSMat.h): reset(n, m) :61-78,
// add_correction(s, y) :81-97 and apply_Hv(v, a, res) :276-302, plus one fused entry the reference spells as four
// Eigen expressions: update(x, xp, g, gp) == { s = x - xp; y = g - gp; if (s'y > eps*y'y) add_correction(s, y) }
// (reference LBFGS.h:159-162).  The n x m matrices never visit the host.
#ifndef LBFGSPP_B200_BFGS_MAT_H
#define LBFGSPP_B200_BFGS_MAT_H

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <limits>
#include <stdexcept>

#include <vector>

#include "DeviceVector.h"
#include "BKLDLT.h"
#include "CompactForm.h"
#include "SmallDense.h"

namespace LBFGSpp {

template <typename Scalar, bool LBFGSB = false>
class BFGSMat
{
    typedef DeviceVector<Scalar> Vector;

    Device* m_dev;
    lbfgs_b200_hist* m_hist;
    bool m_owned;      // false: m_hist belongs to a device-resident solver (borrow())
    std::ptrdiff_t m_n;
    int m_m;
    int m_algo;  // LBFGS_B200_HV_*

    BFGSMat(const BFGSMat&);
    BFGSMat& operator=(const BFGSMat&);

public:
    BFGSMat() : m_dev(nullptr), m_hist(nullptr), m_owned(true), m_n(0), m_m(0), m_algo(LBFGS_B200_HV_AUTO), m_theta_host(1), m_c_host(0), m_box(nullptr), m_nfree(-1) {}
    ~BFGSMat()
    {
        lbfgs_b200_box_destroy(m_box);
        if (m_owned) lbfgs_b200_hist_destroy(m_hist);
    }

    // Which apply_Hv implementation to run (LBFGS_B200_HV_AUTO picks by problem size).
    void set_algorithm(int algo) { m_algo = algo; }
    int algorithm() const { return m_algo; }

    // Forget all pairs.  Unlike the reference, storage is kept when (n, m) did not change, so calling
    // minimize() repeatedly does not reallocate 2*n*m words each time.
    void reset(Device& dev, std::ptrdiff_t n, int m)
    {
        if (m_hist && (!m_owned || m_dev != &dev || m_n != n || m_m != m))
        {
            lbfgs_b200_box_destroy(m_box);
            m_box = nullptr;
            if (m_owned) lbfgs_b200_hist_destroy(m_hist);
            m_hist = nullptr;
            m_owned = true;
        }
        m_dev = &dev;
        m_n = n;
        m_m = m;
        mark_free(-1);
        if (!m_hist)
            dev.check(lbfgs_b200_hist_create(dev.ctx(), &m_hist, n, m, int(sizeof(Scalar))));
        else
            dev.check(lbfgs_b200_hist_reset(m_hist));
    }
    void reset(std::ptrdiff_t n, int m) { reset(Device::get_default(), n, m); }

    // Look at a ring that somebody else owns (the device-resident solver's, after its minimize()): dense() and the Gram accessors
    // then describe that solve's final approximation.  The ring must outlive this object's use of it.
    void borrow(Device& dev, lbfgs_b200_hist* hist, std::ptrdiff_t n, int m)
    {
        lbfgs_b200_box_destroy(m_box);
        m_box = nullptr;
        if (m_owned) lbfgs_b200_hist_destroy(m_hist);
        m_hist = hist;
        m_owned = false;
        mark_free(-1);
        m_dev = &dev;
        m_n = n;
        m_m = m;
    }
    void require_history() const
    {
        if (!m_hist || !m_dev) throw std::logic_error("BFGSMat: no history yet (minimize() has not run)");
    }

    int num_corrections() const { return lbfgs_b200_hist_ncorr(m_hist); }

    // BFGSMat.h:81-97
    void add_correction(const Vector& s, const Vector& y)
    {
        m_free.level = 0;
        m_dev->check(detail::Abi<Scalar>::hist_add(m_hist, s.data(), y.data()));
    }

    // LBFGS.h:159-162 in one kernel; returns whether the pair passed the curvature gate
    bool update(const Vector& x, const Vector& xp, const Vector& g, const Vector& gp)
    {
        m_free.level = 0;
        int accepted = 0;
        m_dev->check(detail::Abi<Scalar>::hist_update(m_hist, x.data(), xp.data(), g.data(), gp.data(),
                                                      std::numeric_limits<Scalar>::epsilon(), &accepted, nullptr));
        return accepted != 0;
    }

    // res = a * H * v  (BFGSMat.h:276-302)
    void apply_Hv(const Vector& v, const Scalar& a, Vector& res)
    {
        res.resize(v.size());
        m_dev->check(detail::Abi<Scalar>::hist_apply_Hv(m_hist, v.data(), a, res.data(), m_algo, nullptr));
    }
    // Same, and also returns v.res from the tail of the last kernel: with v = grad, a = -1 this is the
    // directional derivative `dg = m_grad.dot(m_drt)` of LBFGS.h:123 at no extra memory traffic.
    Scalar apply_Hv_dot(const Vector& v, const Scalar& a, Vector& res)
    {
        res.resize(v.size());
        Scalar vr = Scalar(0);
        m_dev->check(detail::Abi<Scalar>::hist_apply_Hv(m_hist, v.data(), a, res.data(), m_algo, &vr));
        return vr;
    }

    // update(x, xp, g, gp) followed by apply_Hv_dot(g, a, res) as ONE device pass over x, xp, g, gp (LBFGS.h:159-165): the
    // correction pair is formed inside the Gram-dots kernel.  Returns g.res; `accepted` tells whether the pair passed the gate.
    Scalar update_apply_Hv_dot(const Vector& x, const Vector& xp, const Vector& g, const Vector& gp, const Scalar& a, Vector& res,
                               bool* accepted = nullptr)
    {
        m_free.level = 0;
        res.resize(g.size());
        int acc = 0;
        Scalar vr = Scalar(0);
        m_dev->check(detail::Abi<Scalar>::hist_update_apply_Hv(m_hist, x.data(), xp.data(), g.data(), gp.data(),
                                                               std::numeric_limits<Scalar>::epsilon(), a, res.data(), m_algo, &acc, &vr));
        if (accepted) *accepted = acc != 0;
        return vr;
    }

    //========== L-BFGS-B part (reference BFGSMat.h:99-146, 307-615) ==========//
    // B = theta*I - W M W' with W = [Y, theta*S] (n x 2c, columns ordered newest pair first) and M = inv(Minv),
    //   Minv = [ -D   L' ]   D = diag(s_a'y_a),  L(a,b) = s_a'y_b when pair a is newer than pair b, else 0.
    //          [  L  theta*S'S ]
    // The c x c Gram blocks are kept on the device (folded pair by pair by the same pass that serves apply_Hv) and
    // downloaded here; the 2c x 2c algebra is host work like in the reference.  W itself is never formed: products with
    // W are masked passes over the S/Y columns (Wt_dot, lincomb, masked_gram).
private:
    Scalar m_theta_host;
    int m_c_host;
    SmallMatrix<Scalar> m_Minv, m_M, m_SS, m_SY;
    BKLDLT<Scalar> m_Msolver;  // Minv is symmetric indefinite (reference BFGSMat.h:47,134-146)
    lbfgs_b200_box* m_box;
    int64_t m_nfree;           // size of the free set marked by free_set(); -1: none since the last reset()
    // the free-set setup kept between calls (free_setup): level 0 none, 1 K_B, 2 also K_HF, E and log det H_F; b_ok / h_ok: whether B_F /
    // H_F could be formed
    struct FreeSetup
    {
        int level = 0, c = 0;
        bool b_ok = false, h_ok = false;
        double theta = 1.0, logdet = 0.0;
        std::vector<double> SY, SS, Minv, KB, KH, E;
    };
    FreeSetup m_free;

public:
    lbfgs_b200_hist* handle() const { return m_hist; }
    Device& device() const { return *m_dev; }
    Scalar theta() const { return m_theta_host; }
    int ncorr() const { return m_c_host; }
    const SmallMatrix<Scalar>& Minv() const { return m_Minv; }
    const SmallMatrix<Scalar>& Mmat() const { return m_M; }

    // Download the Gram blocks and rebuild Minv / M.  Call after reset() and after every accepted update().
    void refresh_middle()
    {
        require_history();
        const int c = num_corrections();
        m_c_host = c;
        m_theta_host = Scalar(1);
        if (c == 0)
        {
            m_dev->check(detail::BoxAbi<Scalar>::hist_gram(m_hist, nullptr, nullptr, nullptr, nullptr, &m_theta_host));
            m_Minv = SmallMatrix<Scalar>();
            m_M = SmallMatrix<Scalar>();
            return;
        }
        m_SY = SmallMatrix<Scalar>(c, c);
        m_SS = SmallMatrix<Scalar>(c, c);
        m_dev->check(detail::BoxAbi<Scalar>::hist_gram(m_hist, m_SY.data(), m_SS.data(), nullptr, nullptr, &m_theta_host));
        m_Minv = SmallMatrix<Scalar>(2 * c, 2 * c);
        compact_minv(c, m_SY.data(), m_SS.data(), c, m_theta_host, m_Minv.data());
        m_Msolver.compute(m_Minv);
        m_M = SmallMatrix<Scalar>(2 * c, 2 * c);
        std::vector<Scalar> e(size_t(2 * c));
        for (int j = 0; j < 2 * c; j++)
        {
            std::fill(e.begin(), e.end(), Scalar(0));
            e[size_t(j)] = Scalar(1);
            m_Msolver.solve_inplace(e);
            for (int i = 0; i < 2 * c; i++) m_M(i, j) = e[size_t(i)];
        }
    }

    // res = M v   (apply_Mv, BFGSMat.h:361-378)
    std::vector<Scalar> apply_Mv(const std::vector<Scalar>& v) const
    {
        if (m_c_host < 1) return std::vector<Scalar>();
        return m_Msolver.solve(v);
    }

    // W'v for a device vector v (already zero outside the index set of interest): [Y'v ; theta*S'v]
    // (apply_Wtv / apply_WtPv, BFGSMat.h:315-320, 382-433)
    std::vector<Scalar> Wt_dot(const Scalar* v_dev)
    {
        const int c = m_c_host;
        std::vector<Scalar> raw(size_t(2 * c), Scalar(0));
        if (c > 0)
        {
            m_dev->check(detail::BoxAbi<Scalar>::hist_wt_dot(m_hist, v_dev, raw.data()));
            for (int a = 0; a < c; a++) raw[size_t(c + a)] *= m_theta_host;
        }
        return raw;
    }

    // out_i = a0*v0_i + sum_a cy_a*y_a[i] + cs_a*s_a[i] on rows whose class byte intersects `mask`
    void lincomb(Scalar a0, const Scalar* v0_dev, const std::vector<Scalar>& coef, int mask, Scalar* out_dev)
    {
        m_dev->check(detail::BoxAbi<Scalar>::hist_lincomb(m_hist, box(), a0, v0_dev, coef.empty() ? nullptr : coef.data(),
                                                          lbfgs_b200_box_classes(box()), mask, out_dev));
    }

    // inv(P'BP) v on the rows of `mask`; v_dev must be zero outside the mask  (solve_PtBP, BFGSMat.h:529-565)
    void solve_PtBP(int mask, const Scalar* v_dev, Scalar* out_dev)
    {
        const int c = m_c_host;
        const Scalar theta = m_theta_host;
        if (c < 1)
        {
            lincomb(Scalar(1) / theta, v_dev, std::vector<Scalar>(), mask, out_dev);
            return;
        }
        SmallMatrix<Scalar> G(2 * c, 2 * c);
        m_dev->check(detail::BoxAbi<Scalar>::hist_masked_gram(m_hist, box(), lbfgs_b200_box_classes(box()), mask, G.data()));
        SmallMatrix<Scalar> mid(2 * c, 2 * c);
        compact_free_mid(c, m_Minv.data(), m_SS.data(), c, G.data(), theta, mid.data());
        BKLDLT<Scalar> midsolver(mid);  // reference BFGSMat.h:551
        std::vector<Scalar> z = Wt_dot(v_dev);      // [Y_P'v ; theta*S_P'v]
        midsolver.solve_inplace(z);
        std::vector<Scalar> coef(size_t(2 * c));
        const Scalar t2 = theta * theta;
        for (int a = 0; a < c; a++)
        {
            coef[size_t(a)] = z[size_t(a)] / t2;
            coef[size_t(c + a)] = theta * z[size_t(c + a)] / t2;
        }
        lincomb(Scalar(1) / theta, v_dev, coef, mask, out_dev);
    }

    // out = -W_rows * (M u) on the rows of `mask`, u a host 2c-vector in W's [Y ; theta*S] convention
    // (apply_PtWMv with scale -1 / apply_PtBQv, BFGSMat.h:435-478, 570-615)
    void minus_W_M(const std::vector<Scalar>& u, int mask, Scalar* out_dev)
    {
        const int c = m_c_host;
        std::vector<Scalar> coef(size_t(2 * c), Scalar(0));
        if (c > 0)
        {
            const std::vector<Scalar> Mu = apply_Mv(u);
            for (int a = 0; a < c; a++)
            {
                coef[size_t(a)] = -Mu[size_t(a)];
                coef[size_t(c + a)] = -m_theta_host * Mu[size_t(c + a)];
            }
        }
        lincomb(Scalar(0), nullptr, coef, mask, out_dev);
    }

    //========== the final approximation on the free variables F of a bound-constrained solve ==========
    // B_F = Z'BZ and H_F = (Z'BZ)^-1 (CompactForm.h, compact_free_mid / compact_free_kh / compact_free_sqrt; the 2c x 2c algebra in fp64
    // whatever Scalar is), F the coordinates whose class byte carries LBFGS_B200_CLS_FINAL.  free_set marks F at a point x (see
    // lbfgs_b200_box_final_classes) and returns n_F; free_set_classes takes F from n class bytes on the host instead.  Every other member
    // works on the rows of F through the masked passes (lbfgs_b200_hist_*_masked), in groups of 16 vectors, with the rows outside F
    // written as 0 (products, diagonals) or mean_i (draws):
    //   free_hessian_times / free_inverse_hessian_times: OUT = B_F V or H_F V (V's rows outside F are not read);
    //   free_hessian_diagonal / free_inverse_hessian_diagonal: diag B_F = diag B on F, diag H_F;
    //   free_inverse_hessian_logdet: log det H_F = -n_F log theta + sum_i log(1 + sigma_i);
    //   free_sample: mean + L_F z_j on F for the k draws first .. first+k-1 of stream `stream`, L_F the symmetric square root of H_F;
    //   free_log_density: log N(x_F; mean_F, H_F) of the k points of X, from the masked dots of x_j - mean alone.
    // The setup (K_B; for H_F also the masked Gram pass, K_HF, the square root and log det H_F) is formed on first use and kept until the
    // free set or the history changes.  std::logic_error before free_set / free_set_classes (after a reset()).  When H_F cannot be formed
    // (a singular middle matrix, or some 1 + sigma_i not positive and finite): std::runtime_error from the H_F products, diag H_F and the
    // sampler, NaN from the log-determinant and the densities; when M itself cannot be formed, the B_F members throw as well.
    int64_t free_set(const Vector& x, const Vector& lb, const Vector& ub, Scalar tol)
    {
        require_history();
        if (x.size() != m_n || lb.size() != m_n || ub.size() != m_n) throw std::invalid_argument("x, lb and ub must hold n values");
        int64_t nf = 0;
        m_dev->check(detail::BoxAbi<Scalar>::final_classes(box(), x.data(), lb.data(), ub.data(), tol, &nf));
        mark_free(nf);
        return nf;
    }
    int64_t free_set_classes(const unsigned char* cls_host)
    {
        require_history();
        m_dev->check(lbfgs_b200_memcpy_h2d(m_dev->ctx(), const_cast<unsigned char*>(lbfgs_b200_box_classes(box())), cls_host, size_t(m_n)));
        int64_t nf = 0;
        for (std::ptrdiff_t i = 0; i < m_n; i++) nf += (cls_host[i] & LBFGS_B200_CLS_FINAL) ? 1 : 0;
        mark_free(nf);
        return nf;
    }
    int64_t free_count() const { return m_nfree; }

    void free_hessian_times(const Vector& V, int k, Vector& OUT) { free_times(V, k, OUT, false); }
    void free_inverse_hessian_times(const Vector& V, int k, Vector& OUT) { free_times(V, k, OUT, true); }
    void free_hessian_diagonal(Vector& out) { free_diagonal(out, false); }
    void free_inverse_hessian_diagonal(Vector& out) { free_diagonal(out, true); }
    double free_inverse_hessian_logdet() { return free_setup(true).logdet; }
    void free_sample(const Vector* mean, unsigned long long seed, uint32_t stream, uint32_t first, int k, Vector& OUT)
    {
        require_free();
        if (mean && mean->size() != m_n) throw std::invalid_argument("mean must hold n values");
        if (k < 1 || uint64_t(first) + uint64_t(k) > (uint64_t(1) << 32)) throw std::invalid_argument("need k >= 1 and first + k <= 2^32");
        const FreeSetup& f = free_setup(true);
        if (!f.h_ok) throw std::runtime_error("BFGSMat: the kept pairs do not define a positive definite H_F");
        const int c = f.c, w = 2 * c, kGroup = 16;
        const double rsq = 1.0 / std::sqrt(f.theta);
        OUT.resize(std::ptrdiff_t(k) * m_n);
        std::vector<Scalar> Wv, C;
        for (int j0 = 0; j0 < k; j0 += kGroup)
        {
            const int kk = std::min(kGroup, k - j0);
            C.assign(size_t(std::max(1, w * kk)), Scalar(0));
            if (c > 0)
            {
                Wv.assign(size_t(w * kk), Scalar(0));
                m_dev->check(detail::BoxAbi<Scalar>::hist_wt_dot_normal_masked(m_hist, box(), classes(), LBFGS_B200_CLS_FINAL, seed, stream,
                                                                                first + uint32_t(j0), kk, Wv.data()));
                coef_times(w, kk, f.E.data(), rsq, Wv.data(), C.data());
            }
            m_dev->check(detail::BoxAbi<Scalar>::hist_lincomb_normal_masked(m_hist, box(), classes(), LBFGS_B200_CLS_FINAL, Scalar(rsq), seed,
                                                                             stream, first + uint32_t(j0), kk, mean ? mean->data() : nullptr,
                                                                             c > 0 ? C.data() : nullptr, OUT.data() + std::ptrdiff_t(j0) * m_n, m_n));
        }
    }
    std::vector<double> free_log_density(const Vector& mean, const Vector& X, int k)
    {
        require_free();
        if (mean.size() != m_n) throw std::invalid_argument("mean must hold n values");
        if (block_count(X.size(), m_n) != k) throw std::invalid_argument("X.size() must be k * n");
        const FreeSetup& f = free_setup(true);
        std::vector<double> out(static_cast<size_t>(k), std::numeric_limits<double>::quiet_NaN());
        if (!f.h_ok) return out;
        const int w = 2 * f.c, kGroup = 16;
        std::vector<double> Wv, nrm;
        for (int j0 = 0; j0 < k; j0 += kGroup)
        {
            const int kk = std::min(kGroup, k - j0);
            Wv.assign(size_t(std::max(1, w * kk)), 0.0);
            nrm.assign(size_t(kk), 0.0);
            m_dev->check(detail::BoxAbi<Scalar>::hist_wt_dot_diff_masked(m_hist, box(), classes(), LBFGS_B200_CLS_FINAL, kk,
                                                                          X.data() + std::ptrdiff_t(j0) * m_n, m_n, mean.data(), Wv.data(), nrm.data()));
            for (int j = 0; j < kk; j++)
            {
                double q = f.theta * nrm[size_t(j)];   // v_F'B_F v_F = theta |v_F|^2 + r'K_B r, r = W_F'v
                for (int p = 0; p < w; p++)
                {
                    double kr = 0.0;
                    for (int r = 0; r < w; r++) kr += f.KB[size_t(p * w + r)] * Wv[size_t(r * kk + j)];
                    q += Wv[size_t(p * kk + j)] * kr;
                }
                out[size_t(j0 + j)] = compact_log_density(q, f.logdet, double(m_nfree));
            }
        }
        return out;
    }

private:
    const unsigned char* classes() { return lbfgs_b200_box_classes(box()); }
    void require_free() const
    {
        require_history();
        if (m_nfree < 0) throw std::logic_error("BFGSMat: no free set marked since the last minimize() (call final_approx_free_set)");
    }
    void mark_free(int64_t nf)
    {
        m_nfree = nf;
        m_free.level = 0;
    }

    // C[p][j] = a * sum_q K[p][q] R[q][j] for kk vectors (K w x w in double, R and C [w][kk])
    template <class TR>
    static void coef_times(int w, int kk, const double* K, double a, const TR* R, Scalar* C)
    {
        for (int p = 0; p < w; p++)
            for (int j = 0; j < kk; j++)
            {
                double acc = 0.0;
                for (int q = 0; q < w; q++) acc += K[p * w + q] * double(R[q * kk + j]);
                C[p * kk + j] = Scalar(a * acc);
            }
    }

    // The kept setup, at level 1 (K_B) or 2 (also K_HF, E and log det H_F, which need the masked Gram pass); formed on first use.
    const FreeSetup& free_setup(bool h)
    {
        require_free();
        FreeSetup& f = m_free;
        if (f.level >= (h ? 2 : 1)) return f;
        refresh_middle();
        const int c = m_c_host, w = 2 * c;
        const size_t ww = size_t(std::max(1, w * w)), cc = static_cast<size_t>(c * c), ws = static_cast<size_t>(w);
        if (f.level == 0)
        {
            f.c = c;
            f.theta = double(m_theta_host);
            f.KB.assign(ww, 0.0);
            f.SY.assign(std::max<size_t>(1, cc), 0.0);
            f.SS.assign(std::max<size_t>(1, cc), 0.0);
            f.Minv.assign(ww, 0.0);
            f.b_ok = true;
            if (c > 0)
            {
                std::vector<double> M(ww), z(ws), unit(2 * ws - 1, 0.0);
                for (size_t e = 0; e < cc; e++) { f.SY[e] = double(m_SY.data()[e]); f.SS[e] = double(m_SS.data()[e]); }
                compact_minv(c, f.SY.data(), f.SS.data(), c, f.theta, f.Minv.data());
                std::vector<int> order(ws);
                std::vector<unsigned char> tag(ws);
                std::vector<double> fac(f.Minv);
                f.b_ok = bk_factor(fac.data(), w, order.data(), tag.data()) == 0;
                if (f.b_ok)
                {
                    for (int r = 0; r < w; r++)
                    {
                        for (int i = 0; i < w; i++) M[size_t(i * w + r)] = i == r ? 1.0 : 0.0;
                        bk_solve(fac.data(), w, order.data(), tag.data(), M.data() + r, w, z.data());
                    }
                    unit[ws - 1] = 1.0;
                    compact_kb(c, M.data(), f.theta, unit.data(), 0, 1, f.KB.data());
                    compact_k_symmetrise(w, f.KB.data(), 0, 1);
                    for (size_t e = 0; e < ww; e++) f.b_ok = f.b_ok && std::isfinite(f.KB[e]);
                }
            }
            f.level = 1;
        }
        if (h)
        {
            f.KH.assign(ww, 0.0);
            f.E.assign(ww, 0.0);
            f.h_ok = f.b_ok;
            double ls = 0.0;
            if (c > 0 && f.h_ok)
            {
                std::vector<double> G(ww), mid(ww), z(ws), scratch(size_t(5 * w * w + 3 * w));
                std::vector<int> order(ws);
                std::vector<unsigned char> tag(ws);
                std::vector<Scalar> Gs(ww);
                m_dev->check(detail::BoxAbi<Scalar>::hist_masked_gram(m_hist, box(), classes(), LBFGS_B200_CLS_FINAL, Gs.data()));
                for (size_t e = 0; e < ww; e++) G[e] = double(Gs[e]);
                compact_free_mid(c, f.Minv.data(), f.SS.data(), c, G.data(), f.theta, mid.data());
                f.h_ok = compact_free_kh(c, mid.data(), f.theta, order.data(), tag.data(), z.data(), f.KH.data()) == 0 &&
                         compact_free_sqrt(w, G.data(), f.KH.data(), f.theta, f.E.data(), &ls, scratch.data()) == 0;
            }
            f.logdet = -double(m_nfree) * std::log(f.theta) + ls;
            f.h_ok = f.h_ok && std::isfinite(f.logdet);
            for (size_t e = 0; e < ww && f.h_ok; e++) f.h_ok = std::isfinite(f.KH[e]) && std::isfinite(f.E[e]);
            if (!f.h_ok) f.logdet = std::numeric_limits<double>::quiet_NaN();
            f.level = 2;
        }
        return f;
    }

    const FreeSetup& checked_setup(bool inverse)
    {
        const FreeSetup& f = free_setup(inverse);
        if (inverse ? !f.h_ok : !f.b_ok)
            throw std::runtime_error(inverse ? "BFGSMat: the kept pairs do not define a positive definite H_F" : "BFGSMat: singular middle matrix");
        return f;
    }

    void free_diagonal(Vector& out, bool inverse)
    {
        const FreeSetup& f = checked_setup(inverse);
        const int w = 2 * f.c;
        std::vector<Scalar> K(size_t(std::max(1, w * w)));
        for (int e = 0; e < w * w; e++) K[size_t(e)] = Scalar(inverse ? f.KH[size_t(e)] : f.KB[size_t(e)]);
        out.resize(m_n);
        m_dev->check(detail::BoxAbi<Scalar>::hist_quad_diag_masked(m_hist, box(), classes(), LBFGS_B200_CLS_FINAL,
                                                                    Scalar(inverse ? 1.0 / f.theta : f.theta), w > 0 ? K.data() : nullptr, out.data()));
    }

    void free_times(const Vector& V, int k, Vector& OUT, bool inverse)
    {
        require_free();
        if (block_count(V.size(), m_n) != k) throw std::invalid_argument("V.size() must be k * n");
        const FreeSetup& f = checked_setup(inverse);
        const int c = f.c, w = 2 * c, kGroup = 16;
        OUT.resize(V.size());
        std::vector<Scalar> Wv, C;
        for (int j0 = 0; j0 < k; j0 += kGroup)
        {
            const int kk = std::min(kGroup, k - j0);
            const Scalar* v = V.data() + std::ptrdiff_t(j0) * m_n;
            C.assign(size_t(std::max(1, w * kk)), Scalar(0));
            if (c > 0)
            {
                Wv.assign(size_t(w * kk), Scalar(0));
                m_dev->check(detail::BoxAbi<Scalar>::hist_wt_dot_multi_masked(m_hist, box(), classes(), LBFGS_B200_CLS_FINAL, kk, v, m_n, Wv.data()));
                coef_times(w, kk, inverse ? f.KH.data() : f.KB.data(), 1.0, Wv.data(), C.data());
            }
            m_dev->check(detail::BoxAbi<Scalar>::hist_lincomb_multi_masked(m_hist, box(), classes(), LBFGS_B200_CLS_FINAL,
                                                                            Scalar(inverse ? 1.0 / f.theta : f.theta), kk, v, m_n,
                                                                            c > 0 ? C.data() : nullptr, OUT.data() + std::ptrdiff_t(j0) * m_n, m_n));
        }
    }

public:
    // Explicit n x n approximations for small n (final_approx_hessian / final_approx_inverse_hessian of the reference,
    // BFGSMat.h:150-271), through the compact representation:
    //   B = theta*I - W M W'                with the Minv above,
    //   H = I/theta + Z N Z',  Z = [Y/theta, S],  N = [ 0, -R^-1 ; -R^-T, R^-T (D + Y'Y/theta) R^-1 ],  R = triu(S'Y) in
    //   chronological order.  H is formed as inv(B) here (same matrix; n is small by contract).
    SmallMatrix<Scalar> dense(bool inverse)
    {
        refresh_middle();
        const int n = int(m_n), c = m_c_host;
        if (n > 4096) throw std::invalid_argument("dense Hessian approximations are only formed for n <= 4096");
        SmallMatrix<Scalar> B(n, n);
        for (int i = 0; i < n; i++) B(i, i) = m_theta_host;
        if (c > 0)
        {
            // rows of W = [Y, theta*S] by age, downloaded column by column
            SmallMatrix<Scalar> W(n, 2 * c);
            std::vector<Scalar> col(static_cast<size_t>(n));
            for (int a = 0; a < c; a++)
            {
                m_dev->check(lbfgs_b200_memcpy_d2h(m_dev->ctx(), col.data(), lbfgs_b200_hist_y_col(m_hist, a), sizeof(Scalar) * size_t(n)));
                for (int i = 0; i < n; i++) W(i, a) = col[size_t(i)];
                m_dev->check(lbfgs_b200_memcpy_d2h(m_dev->ctx(), col.data(), lbfgs_b200_hist_s_col(m_hist, a), sizeof(Scalar) * size_t(n)));
                for (int i = 0; i < n; i++) W(i, c + a) = m_theta_host * col[size_t(i)];
            }
            for (int i = 0; i < n; i++)
            {
                std::vector<Scalar> wi(size_t(2 * c));
                for (int q = 0; q < 2 * c; q++) wi[size_t(q)] = W(i, q);
                const std::vector<Scalar> Mw = m_M.times(wi);
                for (int j = 0; j < n; j++)
                {
                    Scalar acc = Scalar(0);
                    for (int q = 0; q < 2 * c; q++) acc += W(j, q) * Mw[size_t(q)];
                    B(j, i) -= acc;
                }
            }
        }
        if (!inverse) return B;
        SmallSolver<Scalar> lu(B);
        SmallMatrix<Scalar> H(n, n);
        std::vector<Scalar> e(static_cast<size_t>(n));
        for (int j = 0; j < n; j++)
        {
            std::fill(e.begin(), e.end(), Scalar(0));
            e[size_t(j)] = Scalar(1);
            lu.solve_inplace(e);
            for (int i = 0; i < n; i++) H(i, j) = e[size_t(i)];
        }
        return H;
    }

    // The operator form of the same two matrices, at any n: OUT = B V or H V for k vectors stored back to back in V (OUT is resized
    // to match), in groups of 16 vectors.  Per group one pass over the history for W'V (lbfgs_b200_hist_wt_dot_multi), the 2c x 2c
    // algebra of CompactForm.h on the host, and one pass for the combination (lbfgs_b200_hist_lincomb_multi):
    //   B v = theta v - W M W'v                  C = -M W'v in W's [Y ; theta S] convention, a0 = theta
    //   H v = v/theta + S u_s + Y u_y/theta      u_y = -R^-1 S'v,  u_s = R^-T ((D + Y'Y/theta) R^-1 S'v - Y'v/theta),  a0 = 1/theta
    // (the compact form of H above, with triangular solves per vector; B is never inverted).  With c = 0: B = theta I, H = I/theta.
    void hessian_times(const Vector& V, int k, Vector& OUT) { times(V, k, OUT, false); }
    void inverse_hessian_times(const Vector& V, int k, Vector& OUT) { times(V, k, OUT, true); }

    // k = size / n for a block of whole n-vectors (the LBFGSBatchSolver convention)
    static int block_count(std::ptrdiff_t size, std::ptrdiff_t n)
    {
        if (n < 1 || size < 1 || size % n != 0 || size / n > std::numeric_limits<int>::max())
            throw std::invalid_argument("V.size() must be a positive multiple of n");
        return int(size / n);
    }
    std::ptrdiff_t dim() const { return m_n; }

    // The diagonals of the same two matrices at any n, with no products: written over the raw columns W = [Y S] as
    // B = theta I + W K_B W' and H = I/theta + W K_H W' (CompactForm.h, compact_kb / compact_kh, K formed here on the host), entry i is
    // a0 + r_i' K r_i with r_i row i of W: one pass over the history (lbfgs_b200_hist_quad_diag).  out is resized to n.  With c = 0:
    // theta and 1/theta.
    void hessian_diagonal(Vector& out) { diagonal(out, false); }
    void inverse_hessian_diagonal(Vector& out) { diagonal(out, true); }

    // A square-root factor of H and its log-determinant (CompactForm.h, compact_factor_setup / compact_factor_coef): H = L L' with
    //   L = (I + s_{c-1} b_{c-1}') ... (I + s_0 b_0') / sqrt(theta),   log det H = -n log theta + sum_t log(rho_t s_t'B_t s_t)
    // formed from the Gram blocks alone.  inverse_hessian_factor_times: OUT = L V for k vectors back to back, in groups of 16 through
    // the k-vector passes (W'V, the algebra on the host, then the combination).  sample: OUT = mean + L z_j for the k draws
    // first .. first+k-1 of stream `stream` (mean == nullptr: zero), z_j generated inside both passes and never stored
    // (lbfgs_b200_hist_wt_dot_normal / lincomb_normal).  With c = 0: L = I/sqrt(theta).  Pairs without positive curvature
    // (impossible after a solve, whose curvature gate refuses them): std::runtime_error, and NaN from inverse_hessian_logdet.
    void inverse_hessian_factor_times(const Vector& V, int k, Vector& OUT) { factor<LBFGS_B200_FACTOR_L>(&V, nullptr, 0, 0, 0, k, OUT); }
    void sample(const Vector* mean, unsigned long long seed, uint32_t stream, uint32_t first, int k, Vector& OUT)
    {
        if (mean && mean->size() != m_n) throw std::invalid_argument("mean must hold n values");
        factor<LBFGS_B200_FACTOR_L>(nullptr, mean, seed, stream, first, k, OUT);
    }
    double inverse_hessian_logdet()
    {
        require_history();
        const FactorSetup f = factor_setup(false);
        return f.logdet;
    }

    // Whitening and log densities under N(mean, H) with the same factor (CompactForm.h, compact_factor_t_coef / _inv_coef /
    // _invt_coef / compact_factor_quad): OUT = L' V, L^-1 V or L^-T V for k vectors back to back, in groups of 16, each one dots
    // pass and one combination pass (L' and L^-T read only S for their dots: lbfgs_b200_hist_s_dot_multi).  log_density: log N(x_j;
    // mean, H) for the k points of X, from W'(x_j - mean) and |x_j - mean|^2 alone (lbfgs_b200_hist_wt_dot_diff; no combination
    // pass).  With c = 0: L' = I/sqrt(theta), L^-1 = L^-T = sqrt(theta) I.  Pairs without positive curvature: std::runtime_error from
    // the products, NaN from log_density.
    void inverse_hessian_factor_transpose_times(const Vector& V, int k, Vector& OUT) { factor<LBFGS_B200_FACTOR_LT>(&V, nullptr, 0, 0, 0, k, OUT); }
    void inverse_hessian_factor_solve(const Vector& V, int k, Vector& OUT) { factor<LBFGS_B200_FACTOR_LINV>(&V, nullptr, 0, 0, 0, k, OUT); }
    void inverse_hessian_factor_transpose_solve(const Vector& V, int k, Vector& OUT) { factor<LBFGS_B200_FACTOR_LINVT>(&V, nullptr, 0, 0, 0, k, OUT); }
    std::vector<double> log_density(const Vector& mean, const Vector& X, int k)
    {
        require_history();
        if (mean.size() != m_n) throw std::invalid_argument("mean must hold n values");
        if (block_count(X.size(), m_n) != k) throw std::invalid_argument("X.size() must be k * n");
        const FactorSetup f = factor_setup(true);
        std::vector<double> out(static_cast<size_t>(k), std::numeric_limits<double>::quiet_NaN());
        if (std::isnan(f.logdet)) return out;
        const int c = lbfgs_b200_hist_ncorr(m_hist), kGroup = 16;
        std::vector<double> Wv, nrm, z(size_t(c > 0 ? c : 1));   // the dots as summed (fp64): q cancels when v lies mostly in span S
        for (int j0 = 0; j0 < k; j0 += kGroup)
        {
            const int kk = std::min(kGroup, k - j0);
            Wv.assign(size_t(std::max(1, 2 * c * kk)), 0.0);
            nrm.assign(size_t(kk), 0.0);
            m_dev->check(detail::BoxAbi<Scalar>::hist_wt_dot_diff(m_hist, kk, X.data() + std::ptrdiff_t(j0) * m_n, m_n, mean.data(), Wv.data(),
                                                                  nrm.data()));
            for (int j = 0; j < kk; j++)
            {
                const double q = compact_factor_quad(c, f.beta.data(), f.Tm.data(), f.SS.data(), c, f.theta, Wv.data() + j, kk, nrm[size_t(j)], z.data());
                out[size_t(j0 + j)] = compact_log_density(q, f.logdet, double(m_n));
            }
        }
        return out;
    }

private:
    // compact_factor_setup from the history's Gram blocks (and compact_factor_upper when `upper`, for the inverses); logdet = log det H,
    // NaN when the setup's check fails
    struct FactorSetup
    {
        std::vector<double> beta, Tm;
        std::vector<Scalar> SY, SS;
        Scalar theta = Scalar(1);
        double logdet = 0.0;
    };
    FactorSetup factor_setup(bool upper)
    {
        FactorSetup f;
        const int c = lbfgs_b200_hist_ncorr(m_hist);
        const size_t cs = size_t(c > 0 ? c : 1);
        std::vector<Scalar> YY(cs * cs);
        f.SY.assign(cs * cs, Scalar(0));
        f.SS.assign(cs * cs, Scalar(0));
        m_dev->check(detail::BoxAbi<Scalar>::hist_gram(m_hist, f.SY.data(), f.SS.data(), YY.data(), nullptr, &f.theta));
        f.beta.assign(2 * cs * cs, 0.0);
        f.Tm.assign(cs * cs, 0.0);
        double ls = 0.0;
        if (compact_factor_setup(c, f.SY.data(), f.SS.data(), YY.data(), c, f.theta, f.beta.data(), f.Tm.data(), &ls) != 0)
            f.logdet = std::numeric_limits<double>::quiet_NaN();
        else
        {
            f.logdet = -double(m_n) * std::log(double(f.theta)) + ls;
            if (upper) compact_factor_upper(c, f.SY.data(), c, f.Tm.data());
        }
        return f;
    }

    // OUT = OP(L) V (V given) or the draws mean + L z_j (V == nullptr, OP L), OP one of LBFGS_B200_FACTOR_*.  A template argument, so
    // that the factor and the sampler refer to no pass they do not use.
    template <int OP>
    void factor(const Vector* V, const Vector* mean, unsigned long long seed, uint32_t stream, uint32_t first, int k, Vector& OUT)
    {
        require_history();
        if (V && block_count(V->size(), m_n) != k) throw std::invalid_argument("V.size() must be k * n");
        if (!V && (k < 1 || uint64_t(first) + uint64_t(k) > (uint64_t(1) << 32))) throw std::invalid_argument("need k >= 1 and first + k <= 2^32");
        constexpr bool inv = OP == LBFGS_B200_FACTOR_LINV || OP == LBFGS_B200_FACTOR_LINVT;
        constexpr bool sdots = OP == LBFGS_B200_FACTOR_LT || OP == LBFGS_B200_FACTOR_LINVT;   // S'V suffices
        const FactorSetup f = factor_setup(inv);
        if (std::isnan(f.logdet)) throw std::runtime_error("BFGSMat: the kept pairs do not define a positive definite H");
        const int c = lbfgs_b200_hist_ncorr(m_hist);
        const double rsq = 1.0 / std::sqrt(double(f.theta)), sq = std::sqrt(double(f.theta));
        const Scalar a0 = inv ? Scalar(sq) : Scalar(rsq);
        OUT.resize(std::ptrdiff_t(k) * m_n);
        const int kGroup = 16;
        std::vector<Scalar> Wv, C;
        std::vector<double> z(size_t(c > 0 ? c : 1));
        for (int j0 = 0; j0 < k; j0 += kGroup)
        {
            const int kk = std::min(kGroup, k - j0);
            const Scalar* v = V ? V->data() + std::ptrdiff_t(j0) * m_n : nullptr;
            C.assign(size_t(2 * c * kk), Scalar(0));
            if (c > 0)
            {
                Wv.assign(size_t((sdots ? 1 : 2) * c * kk), Scalar(0));
                if (!V) m_dev->check(detail::BoxAbi<Scalar>::hist_wt_dot_normal(m_hist, seed, stream, first + uint32_t(j0), kk, Wv.data()));
                else if constexpr (sdots) m_dev->check(detail::BoxAbi<Scalar>::hist_s_dot_multi(m_hist, kk, v, m_n, Wv.data()));
                else m_dev->check(detail::BoxAbi<Scalar>::hist_wt_dot_multi(m_hist, kk, v, m_n, Wv.data()));
                for (int j = 0; j < kk; j++)
                {
                    const double* beta = f.beta.data();
                    const double* Tm = f.Tm.data();
                    if constexpr (OP == LBFGS_B200_FACTOR_LT) compact_factor_t_coef(c, beta, Tm, rsq, Wv.data() + j, kk, z.data(), C.data() + j, kk);
                    else if constexpr (OP == LBFGS_B200_FACTOR_LINV) compact_factor_inv_coef(c, beta, Tm, sq, Wv.data() + j, kk, z.data(), C.data() + j, kk);
                    else if constexpr (OP == LBFGS_B200_FACTOR_LINVT) compact_factor_invt_coef(c, beta, Tm, sq, Wv.data() + j, kk, z.data(), C.data() + j, kk);
                    else compact_factor_coef(c, beta, Tm, rsq, Wv.data() + j, kk, C.data() + j, kk);
                }
            }
            Scalar* out = OUT.data() + std::ptrdiff_t(j0) * m_n;
            if (V) m_dev->check(detail::BoxAbi<Scalar>::hist_lincomb_multi(m_hist, a0, kk, v, m_n, c > 0 ? C.data() : nullptr, out, m_n));
            else m_dev->check(detail::BoxAbi<Scalar>::hist_lincomb_normal(m_hist, a0, seed, stream, first + uint32_t(j0), kk,
                                                                          mean ? mean->data() : nullptr, c > 0 ? C.data() : nullptr, out, m_n));
        }
    }

    void diagonal(Vector& out, bool inverse)
    {
        require_history();
        refresh_middle();
        const int c = m_c_host, w = 2 * c;
        const Scalar theta = m_theta_host;
        std::vector<Scalar> K(size_t(w) * size_t(w));
        if (c > 0)
        {
            std::vector<Scalar> unit(size_t(2 * w - 1), Scalar(0));
            unit[size_t(w - 1)] = Scalar(1);
            if (inverse)
            {
                SmallMatrix<Scalar> YYage(c, c), R(c, c), YY(c, c);
                m_dev->check(detail::BoxAbi<Scalar>::hist_gram(m_hist, nullptr, nullptr, YYage.data(), nullptr, nullptr));
                compact_h_setup(c, m_SY.data(), YYage.data(), c, R.data(), YY.data());
                std::vector<Scalar> scr(static_cast<size_t>(w));
                compact_kh(c, R.data(), YY.data(), theta, unit.data(), 0, 1, scr.data(), 1, K.data());
            }
            else
                compact_kb(c, m_M.data(), theta, unit.data(), 0, 1, K.data());
            compact_k_symmetrise(w, K.data(), 0, 1);
        }
        out.resize(m_n);
        m_dev->check(detail::BoxAbi<Scalar>::hist_quad_diag(m_hist, inverse ? Scalar(1) / theta : theta, c > 0 ? K.data() : nullptr, out.data()));
    }

    void times(const Vector& V, int k, Vector& OUT, bool inverse)
    {
        require_history();
        if (block_count(V.size(), m_n) != k) throw std::invalid_argument("V.size() must be k * n");
        refresh_middle();
        const int c = m_c_host;
        const Scalar theta = m_theta_host;
        // H: R and Y'Y in chronological order (compact_h_setup)
        SmallMatrix<Scalar> R(c, c), YY(c, c);
        if (inverse && c > 0)
        {
            SmallMatrix<Scalar> YYage(c, c);
            m_dev->check(detail::BoxAbi<Scalar>::hist_gram(m_hist, nullptr, nullptr, YYage.data(), nullptr, nullptr));
            compact_h_setup(c, m_SY.data(), YYage.data(), c, R.data(), YY.data());
        }
        OUT.resize(V.size());
        const int kGroup = 16;
        const size_t cs = static_cast<size_t>(c);
        std::vector<Scalar> Wv, C, w(cs), us(cs);
        for (int j0 = 0; j0 < k; j0 += kGroup)
        {
            const int kk = std::min(kGroup, k - j0);
            const Scalar* v = V.data() + std::ptrdiff_t(j0) * m_n;
            C.assign(size_t(2 * c * kk), Scalar(0));
            if (c > 0)
            {
                Wv.assign(size_t(2 * c * kk), Scalar(0));
                m_dev->check(detail::BoxAbi<Scalar>::hist_wt_dot_multi(m_hist, kk, v, m_n, Wv.data()));
            }
            for (int j = 0; j < kk && c > 0; j++)
            {
                if (inverse) compact_h_coef(c, R.data(), YY.data(), theta, Wv.data() + j, kk, w.data(), us.data(), 1, C.data() + j, kk);
                else compact_b_coef(c, m_M.data(), theta, Wv.data() + j, kk, C.data() + j, kk);
            }
            m_dev->check(detail::BoxAbi<Scalar>::hist_lincomb_multi(m_hist, inverse ? Scalar(1) / theta : theta, kk, v, m_n,
                                                                    c > 0 ? C.data() : nullptr, OUT.data() + std::ptrdiff_t(j0) * m_n, m_n));
        }
    }

public:
    // the n-sized scratch of Cauchy / SubspaceMin, created on first use and tied to the history
    lbfgs_b200_box* box()
    {
        if (!m_box) m_dev->check(lbfgs_b200_box_create(m_hist, &m_box));
        return m_box;
    }
    void drop_box()
    {
        lbfgs_b200_box_destroy(m_box);
        m_box = nullptr;
    }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_BFGS_MAT_H
