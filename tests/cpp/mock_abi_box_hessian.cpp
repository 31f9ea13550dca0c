// mock_abi_box_hessian.cpp -- the host-memory TEST DOUBLE of the C ABI with the whitening passes (mock_abi_hessian_whiten.cpp, included
// whole) plus host versions of the masked passes and of the free-set classification (lbfgs_b200_hist_*_masked,
// lbfgs_b200_box_final_classes), so that LBFGSBSolver's final_approx_free_* members run on a CPU.  TEST INFRASTRUCTURE ONLY.
// Each masked pass is its unmasked twin of the test double on the vectors with the rows outside the mask zeroed (for the differences:
// x_i replaced by mean_i), followed by writing 0 (or mean_i for the draws) to the output rows outside the mask.
#include "mock_abi_hessian_whiten.cpp"

namespace {

template <class T> lbfgs_b200_status check_mask(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, const char* what)
{
    if (!b || b->h != h || !cls) return fail(h->ctx, LBFGS_B200_ERR_INVALID, (std::string(what) + ": NULL argument or a box of another history").c_str());
    return LBFGS_B200_OK;
}

template <class T> std::vector<T> masked_copy(const unsigned char* cls, int mask, long n, int k, const T* V, int64_t ldv, const T* fill)
{
    std::vector<T> out(size_t(n) * size_t(k));
    for (int j = 0; j < k; j++)
        for (long i = 0; i < n; i++) out[size_t(j) * n + i] = (cls[i] & mask) ? V[j * ldv + i] : (fill ? fill[i] : T(0));
    return out;
}

template <class T>
lbfgs_b200_status do_wt_dot_multi_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, int k, const T* V,
                                         int64_t ldv, T* R)
{
    if (auto st = check_multi<T>(h, k, ldv, "hist_wt_dot_multi_masked")) return st;
    if (auto st = check_mask<T>(h, b, cls, "hist_wt_dot_multi_masked")) return st;
    if (!V || !R) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_wt_dot_multi_masked: NULL argument");
    const long n = h->get<T>().n;
    const std::vector<T> Vm = masked_copy<T>(cls, mask, n, k, V, ldv, nullptr);
    return do_wt_dot_multi<T>(h, k, Vm.data(), n, R);
}

template <class T>
lbfgs_b200_status do_wt_dot_diff_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, int k, const T* X,
                                        int64_t ldx, const T* mean, double* R, double* nrm)
{
    if (auto st = check_multi<T>(h, k, ldx, "hist_wt_dot_diff_masked")) return st;
    if (auto st = check_mask<T>(h, b, cls, "hist_wt_dot_diff_masked")) return st;
    if (!X || !mean || !R || !nrm) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_wt_dot_diff_masked: NULL argument");
    const long n = h->get<T>().n;
    const std::vector<T> Xm = masked_copy<T>(cls, mask, n, k, X, ldx, mean);
    return do_wt_dot_diff<T>(h, k, Xm.data(), n, mean, R, nrm);
}

template <class T>
lbfgs_b200_status do_wt_dot_normal_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, uint64_t seed,
                                          uint32_t stream, uint32_t first, int k, T* R)
{
    if (auto st = check_multi<T>(h, k, h ? h->get<T>().n : 0, "hist_wt_dot_normal_masked")) return st;
    if (auto st = check_mask<T>(h, b, cls, "hist_wt_dot_normal_masked")) return st;
    if (uint64_t(first) + uint64_t(k) > (uint64_t(1) << 32)) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_wt_dot_normal_masked: draws past 2^32");
    if (!R) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_wt_dot_normal_masked: NULL argument");
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr;
    for (int r = 0; r < 2 * c; r++)
    {
        const T* col = static_cast<const T*>(column<T>(h, r >= c, r < c ? r : r - c));
        for (int j = 0; j < k; j++)
        {
            double acc = 0.0;
            for (long i = 0; i < H.n; i++)
                if (cls[i] & mask) acc += double(col[i]) * mock_normal<T>(seed, stream, first + uint32_t(j), i);
            R[r * k + j] = T(acc);
        }
    }
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_lincomb_multi_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, T a0, int k, const T* V,
                                          int64_t ldv, const T* C, T* OUT, int64_t ldo)
{
    if (auto st = check_multi<T>(h, k, ldv, "hist_lincomb_multi_masked")) return st;
    if (auto st = check_mask<T>(h, b, cls, "hist_lincomb_multi_masked")) return st;
    if (auto st = do_lincomb_multi<T>(h, a0, k, V, ldv, C, OUT, ldo)) return st;
    for (int j = 0; j < k; j++)
        for (long i = 0; i < h->get<T>().n; i++)
            if (!(cls[i] & mask)) OUT[j * ldo + i] = T(0);
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_lincomb_normal_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, T a0, uint64_t seed,
                                           uint32_t stream, uint32_t first, int k, const T* mean, const T* Cf, T* OUT, int64_t ldo)
{
    if (auto st = check_multi<T>(h, k, h ? h->get<T>().n : 0, "hist_lincomb_normal_masked")) return st;
    if (auto st = check_mask<T>(h, b, cls, "hist_lincomb_normal_masked")) return st;
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr;
    if (uint64_t(first) + uint64_t(k) > (uint64_t(1) << 32)) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_lincomb_normal_masked: draws past 2^32");
    if (!OUT || (c > 0 && !Cf)) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_lincomb_normal_masked: NULL argument");
    if (ldo < H.n) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_lincomb_normal_masked: leading dimension is smaller than n");
    for (int j = 0; j < k; j++)
        for (long i = 0; i < H.n; i++)
        {
            const T m = mean ? mean[i] : T(0);
            if (!(cls[i] & mask)) { OUT[j * ldo + i] = m; continue; }
            T r = a0 * T(mock_normal<T>(seed, stream, first + uint32_t(j), i));
            if (mean) r = m + r;
            for (int a = 0; a < c; a++) r += Cf[a * k + j] * static_cast<const T*>(column<T>(h, false, a))[i];
            for (int a = 0; a < c; a++) r += Cf[(c + a) * k + j] * static_cast<const T*>(column<T>(h, true, a))[i];
            OUT[j * ldo + i] = r;
        }
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_quad_diag_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, T a0, const T* K, T* out)
{
    if (auto st = check_hist<T>(h)) return st;
    if (auto st = check_mask<T>(h, b, cls, "hist_quad_diag_masked")) return st;
    if (auto st = do_quad_diag<T>(h, a0, K, out)) return st;
    for (long i = 0; i < h->get<T>().n; i++)
        if (!(cls[i] & mask)) out[i] = T(0);
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_final_classes(lbfgs_b200_box* b, const T* x, const T* lb, const T* ub, T tol, int64_t* nfree)
{
    if (auto st = check_box<T>(b)) return st;
    if (!x || !lb || !ub || !nfree || !(tol >= T(0))) return fail(b->h->ctx, LBFGS_B200_ERR_INVALID, "box_final_classes: bad arguments");
    const T inf = std::numeric_limits<T>::infinity();
    int64_t nf = 0;
    for (int64_t i = 0; i < b->n; i++)
    {
        const bool fixed = lb[i] == ub[i] || (lb[i] > -inf && x[i] <= lb[i] + tol * std::max(T(1), std::fabs(lb[i]))) ||
                           (ub[i] < inf && x[i] >= ub[i] - tol * std::max(T(1), std::fabs(ub[i])));
        b->cls[size_t(i)] = fixed ? (unsigned char)(b->cls[size_t(i)] & ~LBFGS_B200_CLS_FINAL) : (unsigned char)(b->cls[size_t(i)] | LBFGS_B200_CLS_FINAL);
        nf += fixed ? 0 : 1;
    }
    *nfree = nf;
    return LBFGS_B200_OK;
}

}  // namespace

extern "C" {

#define MOCK_BOX_HESSIAN(T, SUF)                                                                                                     \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_multi_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, \
                                                                int k, const T* V, int64_t ldv, T* R)                                \
    { return do_wt_dot_multi_masked<T>(h, b, cls, mask, k, V, ldv, R); }                                                             \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_diff_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask,  \
                                                               int k, const T* X, int64_t ldx, const T* mean, double* R, double* nrm) \
    { return do_wt_dot_diff_masked<T>(h, b, cls, mask, k, X, ldx, mean, R, nrm); }                                                   \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_normal_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, \
                                                                 uint64_t seed, uint32_t stream, uint32_t first, int k, T* R)       \
    { return do_wt_dot_normal_masked<T>(h, b, cls, mask, seed, stream, first, k, R); }                                               \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_multi_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, \
                                                                 T a0, int k, const T* V, int64_t ldv, const T* C, T* OUT, int64_t ldo) \
    { return do_lincomb_multi_masked<T>(h, b, cls, mask, a0, k, V, ldv, C, OUT, ldo); }                                              \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_normal_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, \
                                                                  T a0, uint64_t seed, uint32_t stream, uint32_t first, int k,       \
                                                                  const T* mean, const T* C, T* OUT, int64_t ldo)                     \
    { return do_lincomb_normal_masked<T>(h, b, cls, mask, a0, seed, stream, first, k, mean, C, OUT, ldo); }                         \
    lbfgs_b200_status lbfgs_b200_hist_quad_diag_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask,   \
                                                             T a0, const T* K, T* out)                                               \
    { return do_quad_diag_masked<T>(h, b, cls, mask, a0, K, out); }                                                                  \
    lbfgs_b200_status lbfgs_b200_box_final_classes_##SUF(lbfgs_b200_box* b, const T* x, const T* lb, const T* ub, T tol, int64_t* nfree) \
    { return do_final_classes<T>(b, x, lb, ub, tol, nfree); }

MOCK_BOX_HESSIAN(double, f64)
MOCK_BOX_HESSIAN(float, f32)
#undef MOCK_BOX_HESSIAN

}  // extern "C"
