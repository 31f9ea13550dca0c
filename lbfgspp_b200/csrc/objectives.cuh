// objectives.cuh -- device versions of the benchmark objective functions (SURVEY.md 8a row A12).
//
// Each functor evaluates 4 consecutive coordinates at once ("pack") so that it can sit inside the fused
// line-search trial kernel between the wide loads of xp/d and the wide stores of x/g.
//   eval(i0, cnt, x[4], xl, xr, g[4]) -> this pack's contribution to f
//     i0   local index of x[0];  cnt valid lanes (ragged tail);  xl = x_{i0-1}, xr = x_{i0+4} (0 outside the GLOBAL vector)
// n-sharding: a functor whose coordinates couple to their neighbours (kHalo) also carries the global position of its block
// (gofs, n_glob) and a pointer to the halo record that the exchange kernel fills before every evaluation:
//     halo[kHaloLeftA] + step*halo[kHaloLeftB]   = the left neighbour's last  coordinate of the trial point
//     halo[kHaloRightA] + step*halo[kHaloRightB] = the right neighbour's first coordinate
// (halo == nullptr on a single GPU).
// The arithmetic follows the reference example functors expression by expression:
//   RosenbrockPaired   examples/example-rosenbrock.cpp:15-27
//   QuadShift          examples/example-quadratic.cpp:9-19
//   RosenbrockChained  examples/example-rosenbrock-box.cpp:18-33
//   QuadTridiag        f = 1/2 x'Ax - b'x, A = diag(d) + 1/2 tridiag(-1,2,-1)   (SURVEY.md 8d, config C3)
#pragma once
#include <stdint.h>

namespace lb {

// layout of the 12-double halo record: [0..3] own {a_first, b_first, a_last, b_last}, [4..7] the left neighbour's four,
// [8..11] the right neighbour's four (a = xp or x, b = search direction or 0)
constexpr int kHaloDoubles = 12;
constexpr int kHaloLeftA = 6, kHaloLeftB = 7, kHaloRightA = 8, kHaloRightB = 9;

template <class T> struct RosenbrockPaired
{
    static constexpr bool kHalo = false;
    static constexpr int kDataVectors = 0;   // per-coordinate data vectors read by every evaluation
    int64_t n;
    __device__ __forceinline__ T eval(int64_t, int cnt, const T (&x)[4], T, T, T (&g)[4]) const
    {
        T f = T(0);
#pragma unroll
        for (int k = 0; k < 4; k += 2)
        {
            if (k < cnt)
            {
                const T t1 = T(1) - x[k];
                const T t2 = T(10) * (x[k + 1] - x[k] * x[k]);
                g[k + 1] = T(20) * t2;
                g[k] = T(-2) * (x[k] * g[k + 1] + t1);
                f += t1 * t1 + t2 * t2;
            }
            else
                g[k] = g[k + 1] = T(0);
        }
        return f;
    }
};

template <class T> struct QuadShift
{
    static constexpr bool kHalo = false;
    static constexpr int kDataVectors = 0;
    int64_t n;
    int64_t index_offset;  // global index of local element 0 (n-sharding)
    __device__ __forceinline__ T eval(int64_t i0, int cnt, const T (&x)[4], T, T, T (&g)[4]) const
    {
        T f = T(0);
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            const T r = x[k] - T(i0 + index_offset + k);
            g[k] = (k < cnt) ? T(2) * r : T(0);
            f += (k < cnt) ? r * r : T(0);
        }
        return f;
    }
};

template <class T> struct RosenbrockChained
{
    static constexpr bool kHalo = true;
    static constexpr int kDataVectors = 0;
    __device__ __forceinline__ RosenbrockChained staged(const T*, const T*, int64_t) const { return *this; }
    int64_t n;             // local length
    int64_t gofs, n_glob;  // global index of local element 0, global length (gofs = 0, n_glob = n unsharded)
    const double* halo;
    __device__ __forceinline__ T eval(int64_t i0, int cnt, const T (&x)[4], T xl, T xr, T (&g)[4]) const
    {
        T f = T(0);
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            const int64_t i = gofs + i0 + k;
            const T xm = (k == 0) ? xl : x[k > 0 ? k - 1 : 0];
            const T xn = (k == 3) ? xr : x[k < 3 ? k + 1 : 3];
            T gi, fi;
            if (i == 0)
            {
                fi = (x[k] - T(1)) * (x[k] - T(1));
                gi = T(2) * (x[k] - T(1)) + T(16) * (x[k] * x[k] - xn) * x[k];
            }
            else
            {
                const T u = x[k] - xm * xm;
                fi = T(4) * u * u;
                gi = (i == n_glob - 1) ? T(8) * u : T(8) * u + T(16) * (x[k] * x[k] - xn) * x[k];
            }
            g[k] = (k < cnt) ? gi : T(0);
            f += (k < cnt) ? fi : T(0);
        }
        return f;
    }
};

template <class T> struct QuadTridiag
{
    static constexpr bool kHalo = true;
    static constexpr int kDataVectors = 2;
    int64_t n;
    const T* diag;  // d (this rank's block)
    const T* rhs;   // b
    int64_t gofs, n_glob;
    const double* halo;
    // the same objective reading its two data vectors from a staged tile: `d_tile[0]` / `b_tile[0]` hold element `e0`
    __device__ __forceinline__ QuadTridiag staged(const T* d_tile, const T* b_tile, int64_t e0) const
    {
        QuadTridiag o = *this;
        o.diag = d_tile - e0;
        o.rhs = b_tile - e0;
        return o;
    }
    __device__ __forceinline__ T eval(int64_t i0, int cnt, const T (&x)[4], T xl, T xr, T (&g)[4]) const
    {
        T f = T(0);
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            if (k < cnt)
            {
                const T xm = (k == 0) ? xl : x[k > 0 ? k - 1 : 0];
                const T xn = (k == 3) ? xr : x[k < 3 ? k + 1 : 3];
                const T dk = diag[i0 + k], bk = rhs[i0 + k];
                const T ax = (dk + T(1)) * x[k] - T(0.5) * (xm + xn);
                g[k] = ax - bk;
                f += x[k] * (T(0.5) * ax - bk);
            }
            else
                g[k] = T(0);
        }
        return f;
    }
};

}  // namespace lb
