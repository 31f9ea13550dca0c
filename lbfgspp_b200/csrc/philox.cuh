// philox.cuh -- the counter-based normal generator of the samplers of the final approximation (lbfgs_b200_hist_*_normal_*,
// lbfgs_b200_small_hist_sample_*): Philox4x32-10 (Salmon et al., SC'11), written out here so that a host restatement
// (tests/test_hessian_sample_cpu.py) can reproduce it bit for bit.
//   key     = (seed low 32 bits, seed high 32 bits)
//   counter = (q low, q high, draw j, stream),  q = i / 2: one call serves coordinates 2q and 2q + 1
//   x0 = ((w1 << 32) | w0) >> 11,  x1 = ((w3 << 32) | w2) >> 11           (53 bits each, w = the four output words)
//   u0 = (x0 + 1) 2^-53 in (0, 1],  u1 = x1 2^-53 in [0, 1)                (exact in fp64)
//   z_2q = sqrt(-2 log u0) cospi(2 u1),  z_2q+1 = sqrt(-2 log u0) sinpi(2 u1)   (Box-Muller, fp64; fp32 storage rounds these)
// A draw depends on (seed, stream, j, i) only.
#pragma once

#include <cstdint>

namespace lb {

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t out[4])
{
#pragma unroll
    for (int r = 0; r < 10; r++)
    {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        c0 = n0; c1 = (uint32_t)p1; c2 = n2; c3 = (uint32_t)p0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// the normals of coordinates 2q and 2q + 1 of draw j of a stream
__device__ __forceinline__ void normal_pair(unsigned long long seed, uint32_t stream, uint32_t j, unsigned long long q, double& z0, double& z1)
{
    uint32_t w[4];
    philox4x32_10((uint32_t)q, (uint32_t)(q >> 32), j, stream, (uint32_t)seed, (uint32_t)(seed >> 32), w);
    const uint64_t x0 = ((((uint64_t)w[1]) << 32) | w[0]) >> 11, x1 = ((((uint64_t)w[3]) << 32) | w[2]) >> 11;
    const double u0 = (double)(x0 + 1) * 0x1p-53, u1 = (double)x1 * 0x1p-53;
    const double r = sqrt(-2.0 * log(u0));
    double s, c;
    sincospi(2.0 * u1, &s, &c);
    z0 = r * c;
    z1 = r * s;
}

// what the samplers draw for one coordinate (both precisions draw the same fp64 stream)
struct NormalSrc
{
    unsigned long long seed;
    uint32_t stream, first;   // draw first + j for vector j of a call
};

}  // namespace lb
