// mock_abi_hessian_whiten.cpp -- the host-memory TEST DOUBLE of the C ABI with the sampler's passes (mock_abi_hessian_sample.cpp,
// included whole) plus host versions of the whitening passes (lbfgs_b200_hist_s_dot_multi / lbfgs_b200_hist_wt_dot_diff), so that the
// front's L', L^-1, L^-T and log density run on a CPU.  TEST INFRASTRUCTURE ONLY.
//   R[c][k] = S'V                                          each dot summed left to right in double, rounded to T
//   R[2c][k] = [Y S]'(X - mean), nrm[j] = |x_j - mean|^2    x - mean formed in T, each sum left to right in double, returned in double
// Like the rest of the test double it has no small-batch history, so it exports no lbfgs_b200_small_hist_* entry.
#include "mock_abi_hessian_sample.cpp"

namespace {

template <class T>
lbfgs_b200_status do_s_dot_multi(lbfgs_b200_hist* h, int k, const T* V, int64_t ldv, T* R)
{
    if (auto st = check_multi<T>(h, k, ldv, "hist_s_dot_multi")) return st;
    if (!V || !R) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_s_dot_multi: NULL argument");
    orc::History<T>& H = h->get<T>();
    for (int a = 0; a < H.ncorr; a++)
    {
        const T* col = static_cast<const T*>(column<T>(h, true, a));
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
lbfgs_b200_status do_wt_dot_diff(lbfgs_b200_hist* h, int k, const T* X, int64_t ldx, const T* mean, double* R, double* nrm)
{
    if (auto st = check_multi<T>(h, k, ldx, "hist_wt_dot_diff")) return st;
    if (!X || !mean || !R || !nrm) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_wt_dot_diff: NULL argument");
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr;
    std::vector<T> v(size_t(H.n));
    for (int j = 0; j < k; j++)
    {
        for (long i = 0; i < H.n; i++) v[size_t(i)] = T(X[j * ldx + i] - mean[i]);
        for (int a = 0; a < 2 * c; a++)
        {
            const T* col = static_cast<const T*>(column<T>(h, a >= c, a % c));
            double acc = 0.0;
            for (long i = 0; i < H.n; i++) acc += double(col[i]) * double(v[size_t(i)]);
            R[a * k + j] = acc;
        }
        double acc = 0.0;
        for (long i = 0; i < H.n; i++) acc += double(v[size_t(i)]) * double(v[size_t(i)]);
        nrm[j] = acc;
    }
    return LBFGS_B200_OK;
}

}  // namespace

extern "C" {

lbfgs_b200_status lbfgs_b200_hist_s_dot_multi_f64(lbfgs_b200_hist* h, int k, const double* V, int64_t ldv, double* R)
{ return do_s_dot_multi<double>(h, k, V, ldv, R); }
lbfgs_b200_status lbfgs_b200_hist_s_dot_multi_f32(lbfgs_b200_hist* h, int k, const float* V, int64_t ldv, float* R)
{ return do_s_dot_multi<float>(h, k, V, ldv, R); }
lbfgs_b200_status lbfgs_b200_hist_wt_dot_diff_f64(lbfgs_b200_hist* h, int k, const double* X, int64_t ldx, const double* mean, double* R,
                                                  double* nrm)
{ return do_wt_dot_diff<double>(h, k, X, ldx, mean, R, nrm); }
lbfgs_b200_status lbfgs_b200_hist_wt_dot_diff_f32(lbfgs_b200_hist* h, int k, const float* X, int64_t ldx, const float* mean, double* R,
                                                  double* nrm)
{ return do_wt_dot_diff<float>(h, k, X, ldx, mean, R, nrm); }

}  // extern "C"
