// mock_abi_hessian_ops.cpp -- the host-memory TEST DOUBLE of the C ABI (mock_abi.cpp, included whole) plus host versions of the two
// k-vector passes behind the operator form of the final approximation (lbfgs_b200_hist_wt_dot_multi / lbfgs_b200_hist_lincomb_multi).
// TEST INFRASTRUCTURE ONLY: compiled in place of mock_abi.cpp by the tests of that operator form.
//   R[2c][k] = [Y S]'V                                       each dot summed left to right in double
//   OUT[:,j] = a0*V[:,j] + sum_a C[a][j]*y_a + C[c+a][j]*s_a   added in that order
#include "mock_abi.cpp"

namespace {

template <class T> lbfgs_b200_status check_multi(lbfgs_b200_hist* h, int k, int64_t ldv, const char* what)
{
    if (auto st = check_hist<T>(h)) return st;
    if (k < 1 || k > 16) return fail(h->ctx, LBFGS_B200_ERR_INVALID, (std::string(what) + ": k must be in 1..16").c_str());
    if (ldv < h->get<T>().n) return fail(h->ctx, LBFGS_B200_ERR_INVALID, (std::string(what) + ": leading dimension smaller than n").c_str());
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_wt_dot_multi(lbfgs_b200_hist* h, int k, const T* V, int64_t ldv, T* R)
{
    if (auto st = check_multi<T>(h, k, ldv, "hist_wt_dot_multi")) return st;
    if (!V || !R) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_wt_dot_multi: NULL argument");
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr;
    for (int a = 0; a < 2 * c; a++)
    {
        const T* col = static_cast<const T*>(column<T>(h, a >= c, a % c));
        for (int j = 0; j < k; j++)
        {
            double acc = 0.0;
            for (long i = 0; i < H.n; i++) acc += double(col[i]) * double(V[j * ldv + i]);
            R[a * k + j] = T(acc);
        }
    }
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_lincomb_multi(lbfgs_b200_hist* h, T a0, int k, const T* V, int64_t ldv, const T* C, T* OUT, int64_t ldo)
{
    if (auto st = check_multi<T>(h, k, ldv, "hist_lincomb_multi")) return st;
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr;
    if (!V || !OUT || (c > 0 && !C)) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_lincomb_multi: NULL argument");
    if (ldo < H.n) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_lincomb_multi: leading dimension smaller than n");
    for (int j = 0; j < k; j++)
        for (long i = 0; i < H.n; i++)
        {
            T r = a0 * V[j * ldv + i];
            for (int a = 0; a < c; a++) r += C[a * k + j] * static_cast<const T*>(column<T>(h, false, a))[i];
            for (int a = 0; a < c; a++) r += C[(c + a) * k + j] * static_cast<const T*>(column<T>(h, true, a))[i];
            OUT[j * ldo + i] = r;
        }
    return LBFGS_B200_OK;
}

}  // namespace

extern "C" {

#define MOCK_MULTI(T, SUF)                                                                                                       \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_multi_##SUF(lbfgs_b200_hist* h, int k, const T* V, int64_t ldv, T* R)               \
    { return do_wt_dot_multi<T>(h, k, V, ldv, R); }                                                                              \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_multi_##SUF(lbfgs_b200_hist* h, T a0, int k, const T* V, int64_t ldv, const T* C,  \
                                                          T* OUT, int64_t ldo)                                                   \
    { return do_lincomb_multi<T>(h, a0, k, V, ldv, C, OUT, ldo); }
MOCK_MULTI(double, f64)
MOCK_MULTI(float, f32)

}  // extern "C"
