// mock_abi_hessian_diag.cpp -- the host-memory TEST DOUBLE of the C ABI with the k-vector passes (mock_abi_hessian_ops.cpp, included
// whole) plus a host version of the diagonal pass behind the diagonals of the final approximation (lbfgs_b200_hist_quad_diag).
// TEST INFRASTRUCTURE ONLY: compiled in place of mock_abi_hessian_ops.cpp by the tests of those diagonals.
//   out_i = a0 + r_i' K r_i,  r_i = (y_0[i] .. y_{c-1}[i], s_0[i] .. s_{c-1}[i]) taken to double, K's upper triangle only:
//     t_p = K_pp r_p,  t_p = fma(2 K_pq, r_q, t_p) for q = p+1 .. 2c-1;   acc = 0,  acc = fma(r_p, t_p, acc) for p = 0 .. 2c-1;
//     out_i = a0 + acc   (everything in double, as the device pass takes it)
#include <cmath>

#include "mock_abi_hessian_ops.cpp"

namespace {

template <class T>
lbfgs_b200_status do_quad_diag(lbfgs_b200_hist* h, T a0, const T* K, T* out)
{
    if (auto st = check_hist<T>(h)) return st;
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr, w = 2 * c;
    if (!out || (c > 0 && !K)) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_quad_diag: NULL argument");
    std::vector<const T*> col(static_cast<size_t>(w));
    for (int a = 0; a < c; a++)
    {
        col[size_t(a)] = static_cast<const T*>(column<T>(h, false, a));
        col[size_t(c + a)] = static_cast<const T*>(column<T>(h, true, a));
    }
    std::vector<double> r(static_cast<size_t>(w));
    for (long i = 0; i < H.n; i++)
    {
        for (int q = 0; q < w; q++) r[size_t(q)] = double(col[size_t(q)][i]);
        double acc = 0.0;
        for (int p = 0; p < w; p++)
        {
            double t = double(K[p * w + p]) * r[size_t(p)];
            for (int q = p + 1; q < w; q++) t = std::fma(2.0 * double(K[p * w + q]), r[size_t(q)], t);
            acc = std::fma(r[size_t(p)], t, acc);
        }
        out[i] = T(double(a0) + acc);
    }
    return LBFGS_B200_OK;
}

}  // namespace

extern "C" {

lbfgs_b200_status lbfgs_b200_hist_quad_diag_f64(lbfgs_b200_hist* h, double a0, const double* K, double* out) { return do_quad_diag<double>(h, a0, K, out); }
lbfgs_b200_status lbfgs_b200_hist_quad_diag_f32(lbfgs_b200_hist* h, float a0, const float* K, float* out) { return do_quad_diag<float>(h, a0, K, out); }

}  // extern "C"
