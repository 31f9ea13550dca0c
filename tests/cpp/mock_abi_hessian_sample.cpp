// mock_abi_hessian_sample.cpp -- the host-memory TEST DOUBLE of the C ABI with the diagonal pass (mock_abi_hessian_diag.cpp, included
// whole) plus host versions of the sampler's two passes (lbfgs_b200_hist_wt_dot_normal / lincomb_normal), so that the front's
// factor, sampler and log-determinant run on a CPU.  TEST INFRASTRUCTURE ONLY.
// The normals restate lbfgspp_b200/csrc/philox.cuh: Philox4x32-10 with the same key and counter, the same uniforms, and Box-Muller
// with std::cos / std::sin of 2 pi u1 in place of sincospi (equal to rounding, not bit for bit).  Dots in double, in row order.
#include <cmath>
#include <cstdint>

#include "mock_abi_hessian_diag.cpp"

namespace {

void mock_normal_pair(uint64_t seed, uint32_t stream, uint32_t j, uint64_t q, double& z0, double& z1)
{
    uint32_t c0 = uint32_t(q), c1 = uint32_t(q >> 32), c2 = j, c3 = stream, k0 = uint32_t(seed), k1 = uint32_t(seed >> 32);
    for (int r = 0; r < 10; r++)
    {
        const uint64_t p0 = uint64_t(0xD2511F53u) * c0, p1 = uint64_t(0xCD9E8D57u) * c2;
        const uint32_t n0 = uint32_t(p1 >> 32) ^ c1 ^ k0, n2 = uint32_t(p0 >> 32) ^ c3 ^ k1;
        c0 = n0; c1 = uint32_t(p1); c2 = n2; c3 = uint32_t(p0);
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    const uint64_t x0 = ((uint64_t(c1) << 32) | c0) >> 11, x1 = ((uint64_t(c3) << 32) | c2) >> 11;
    const double u0 = double(x0 + 1) * 0x1p-53, u1 = double(x1) * 0x1p-53;
    const double r = std::sqrt(-2.0 * std::log(u0)), a = 2.0 * 3.14159265358979323846 * u1;
    z0 = r * std::cos(a);
    z1 = r * std::sin(a);
}

template <class T> double mock_normal(uint64_t seed, uint32_t stream, uint32_t j, long i)
{
    double z0, z1;
    mock_normal_pair(seed, stream, j, uint64_t(i) / 2, z0, z1);
    return double(T(i % 2 ? z1 : z0));   // fp32 storage rounds the fp64 normal
}

template <class T>
lbfgs_b200_status do_wt_dot_normal(lbfgs_b200_hist* h, uint64_t seed, uint32_t stream, uint32_t first, int k, T* R)
{
    if (auto st = check_hist<T>(h)) return st;
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr;
    if (k < 1 || k > 16) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_wt_dot_normal: k must be in 1..16");
    if (uint64_t(first) + uint64_t(k) > (uint64_t(1) << 32)) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_wt_dot_normal: draws past 2^32");
    if (!R) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_wt_dot_normal: NULL argument");
    for (int r = 0; r < 2 * c; r++)
    {
        const T* col = static_cast<const T*>(column<T>(h, r >= c, r < c ? r : r - c));
        for (int j = 0; j < k; j++)
        {
            double acc = 0.0;
            for (long i = 0; i < H.n; i++) acc += double(col[i]) * mock_normal<T>(seed, stream, first + uint32_t(j), i);
            R[r * k + j] = T(acc);
        }
    }
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_lincomb_normal(lbfgs_b200_hist* h, T a0, uint64_t seed, uint32_t stream, uint32_t first, int k, const T* mean,
                                    const T* Cf, T* OUT, int64_t ldo)
{
    if (auto st = check_hist<T>(h)) return st;
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr;
    if (k < 1 || k > 16) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_lincomb_normal: k must be in 1..16");
    if (uint64_t(first) + uint64_t(k) > (uint64_t(1) << 32)) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_lincomb_normal: draws past 2^32");
    if (!OUT || (c > 0 && !Cf)) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_lincomb_normal: NULL argument");
    if (ldo < H.n) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_lincomb_normal: leading dimension is smaller than n");
    for (int j = 0; j < k; j++)
        for (long i = 0; i < H.n; i++)
        {
            T r = a0 * T(mock_normal<T>(seed, stream, first + uint32_t(j), i));
            if (mean) r = mean[i] + r;
            for (int a = 0; a < c; a++) r += Cf[(c + a) * k + j] * static_cast<const T*>(column<T>(h, true, a))[i];
            OUT[j * ldo + i] = r;
        }
    return LBFGS_B200_OK;
}

}  // namespace

extern "C" {

lbfgs_b200_status lbfgs_b200_hist_wt_dot_normal_f64(lbfgs_b200_hist* h, uint64_t seed, uint32_t stream, uint32_t first, int k, double* R)
{ return do_wt_dot_normal<double>(h, seed, stream, first, k, R); }
lbfgs_b200_status lbfgs_b200_hist_wt_dot_normal_f32(lbfgs_b200_hist* h, uint64_t seed, uint32_t stream, uint32_t first, int k, float* R)
{ return do_wt_dot_normal<float>(h, seed, stream, first, k, R); }
lbfgs_b200_status lbfgs_b200_hist_lincomb_normal_f64(lbfgs_b200_hist* h, double a0, uint64_t seed, uint32_t stream, uint32_t first, int k,
                                                     const double* mean, const double* Cf, double* OUT, int64_t ldo)
{ return do_lincomb_normal<double>(h, a0, seed, stream, first, k, mean, Cf, OUT, ldo); }
lbfgs_b200_status lbfgs_b200_hist_lincomb_normal_f32(lbfgs_b200_hist* h, float a0, uint64_t seed, uint32_t stream, uint32_t first, int k,
                                                     const float* mean, const float* Cf, float* OUT, int64_t ldo)
{ return do_lincomb_normal<float>(h, a0, seed, stream, first, k, mean, Cf, OUT, ldo); }

}  // extern "C"
