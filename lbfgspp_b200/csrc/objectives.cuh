// objectives.cuh -- the built-in objective functions (SURVEY.md 8a row A12) as both solver loops use them: the functors, the record
// they are built from and the device steps that evaluate one pack.  Their id -> type dispatch and argument checks are the host side
// (with_objective, objective_geometry in internal.cuh).
//
// Each functor evaluates 4 consecutive coordinates at once ("pack") so that it can sit inside the fused line-search trial pass
// between the wide loads of xp/d and the wide stores of x/g.
//   eval(i0, cnt, x[4], xl, xr, g[4]) -> this pack's contribution to f; g = 0 in the lanes past cnt (RosenbrockPaired works on
//   pairs of lanes, so this holds for it because its n is even, which makes cnt even)
//     i0   local index of x[0];  cnt valid lanes (ragged tail);  xl = x_{i0-1}, xr = x_{i0+4} (0 outside the GLOBAL vector)
// Every functor is an ObjGeom: the host-driven loop (k_trial) and the device-resident solve (k_persist) build it from the same record.
// n-sharding: a functor whose coordinates couple to their neighbours (kHalo) reads the global position of its block (gofs, n_glob)
// and, at the two ends of the block, the halo record that the exchange fills before every evaluation (pack_neighbours):
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

#include "device_utils.cuh"
#include "../../include/LBFGSpp/OWLQNCore.h"

namespace lb {

// layout of the 12-double halo record: [0..3] own {a_first, b_first, a_last, b_last}, [4..7] the left neighbour's four,
// [8..11] the right neighbour's four (a = xp or x, b = search direction or 0)
constexpr int kHaloDoubles = 12;
constexpr int kHaloLeftA = 6, kHaloLeftB = 7, kHaloRightA = 8, kHaloRightB = 9;

// where this rank's block of the objective lies, and its data
template <class T> struct ObjGeom
{
    int64_t n;               // local length
    int64_t gofs, n_glob;    // global index of local element 0, global length
    const double* halo;      // the halo record (neighbour-coupled objectives under n-sharding), else nullptr
    const T *data0, *data1;  // per-coordinate data vectors of this block (kDataVectors of them)
};

template <class T> struct RosenbrockPaired : ObjGeom<T>
{
    static constexpr bool kHalo = false;
    static constexpr int kDataVectors = 0;   // per-coordinate data vectors read by every evaluation
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

template <class T> struct QuadShift : ObjGeom<T>
{
    static constexpr bool kHalo = false;
    static constexpr int kDataVectors = 0;
    __device__ __forceinline__ T eval(int64_t i0, int cnt, const T (&x)[4], T, T, T (&g)[4]) const
    {
        T f = T(0);
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            const T r = x[k] - T(i0 + this->gofs + k);
            g[k] = (k < cnt) ? T(2) * r : T(0);
            f += (k < cnt) ? r * r : T(0);
        }
        return f;
    }
};

template <class T> struct RosenbrockChained : ObjGeom<T>
{
    static constexpr bool kHalo = true;
    static constexpr int kDataVectors = 0;
    __device__ __forceinline__ RosenbrockChained staged(const T*, const T*, int64_t) const { return *this; }
    __device__ __forceinline__ T eval(int64_t i0, int cnt, const T (&x)[4], T xl, T xr, T (&g)[4]) const
    {
        T f = T(0);
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            const int64_t i = this->gofs + i0 + k;
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
                gi = (i == this->n_glob - 1) ? T(8) * u : T(8) * u + T(16) * (x[k] * x[k] - xn) * x[k];
            }
            g[k] = (k < cnt) ? gi : T(0);
            f += (k < cnt) ? fi : T(0);
        }
        return f;
    }
};

// data0 = d, data1 = b
template <class T> struct QuadTridiag : ObjGeom<T>
{
    static constexpr bool kHalo = true;
    static constexpr int kDataVectors = 2;
    // the same objective reading its two data vectors from a staged tile: `d_tile[0]` / `b_tile[0]` hold element `e0`
    __device__ __forceinline__ QuadTridiag staged(const T* d_tile, const T* b_tile, int64_t e0) const
    {
        QuadTridiag o = *this;
        o.data0 = d_tile - e0;
        o.data1 = b_tile - e0;
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
                const T dk = this->data0[i0 + k], bk = this->data1[i0 + k];
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

// ---- device: the steps every pass that evaluates an objective shares ----------------------------------------------------------
// xl = x_{i0-1}, xr = x_{i0+4} of the pack at local index i0 of a block of n: inside the block `at(j)` gives
// x_{i0+j}; at a rank boundary the halo record gives the neighbour's coordinate (TRIAL: a + step*b, else a); beyond the ends of the
// global vector 0.  The record is read with volatile loads: the resident solve's leader rewrites it between rounds.
template <bool TRIAL, class T, class OBJ, class At>
__device__ __forceinline__ void pack_neighbours(const OBJ& obj, int64_t i0, int64_t n, T step, At at, T& xl, T& xr)
{
    auto from_halo = [&](int a, int b) {
        T v = T(ldv(obj.halo + a));
        if (TRIAL) v = v + step * T(ldv(obj.halo + b));
        return v;
    };
    xl = xr = T(0);
    if (i0 > 0) xl = at(-1);
    else if (obj.halo && obj.gofs > 0) xl = from_halo(kHaloLeftA, kHaloLeftB);
    if (i0 + 4 < n) xr = at(4);
    else if (obj.halo && i0 + 4 == n && obj.gofs + n < obj.n_glob) xr = from_halo(kHaloRightA, kHaloRightB);
}

// one pack at x with direction d (L = 4, or the lanes of a 16-byte unit): g of the pack into g, and its {f, g.d, g.g, x.x} over the
// cnt valid lanes added to acc[0..3].  The lanes past cnt add nothing: g is 0 there (eval), the caller passes d = 0 there, and x.x
// is masked.
template <class T, class OBJ, int L>
__device__ __forceinline__ void eval_pack(const OBJ& obj, int64_t i0, int cnt, const T (&x)[4], T xl, T xr, const T (&d)[L], T (&g)[4], T* acc)
{
    static_assert(L <= 4, "a pack has 4 lanes");
    acc[0] += obj.eval(i0, cnt, x, xl, xr, g);
#pragma unroll
    for (int k = 0; k < L; k++)
    {
        acc[1] += g[k] * d[k];
        acc[2] += g[k] * g[k];
        acc[3] += (k < cnt) ? x[k] * x[k] : T(0);
    }
}

// OWL-QN (LBFGSpp/OWLQNCore.h): one pack of the projected trial x = pi(xp + step d; xi), whose start point xp, direction d and start
// gradient gp the caller loaded; x and g of the pack into x, g, and its {f, |x|_1, pgp.(x - xp), pg.pg, x.x} over the cnt valid
// lanes added to acc[0..4].  The neighbours of a coupled objective are the projected trial coordinates, which `at(j)` returns from
// the three input vectors with the same expression (owlqn_point).  One GPU only: no halo.
template <class T, class OBJ, class At>
__device__ __forceinline__ void eval_pack_owlqn(const OBJ& obj, int64_t i0, int64_t n, int cnt, const T (&xp)[4], const T (&d)[4],
                                                const T (&gp)[4], T step, T lam, At at, T (&x)[4], T (&g)[4], T* acc)
{
    T pgp[4];
#pragma unroll
    for (int k = 0; k < 4; k++)
    {
        pgp[k] = LBFGSpp::owlqn_pg(xp[k], gp[k], lam);
        x[k] = (k < cnt) ? LBFGSpp::owlqn_project(xp[k] + step * d[k], LBFGSpp::owlqn_orthant(xp[k], pgp[k])) : T(0);
    }
    T xl = T(0), xr = T(0);
    if constexpr (OBJ::kHalo) pack_neighbours<false>(obj, i0, n, step, at, xl, xr);
    acc[0] += obj.eval(i0, cnt, x, xl, xr, g);
#pragma unroll
    for (int k = 0; k < 4; k++)
    {
        if (k < cnt)
        {
            const T pg = LBFGSpp::owlqn_pg(x[k], g[k], lam);
            acc[1] += x[k] < T(0) ? -x[k] : x[k];
            acc[2] += pgp[k] * (x[k] - xp[k]);
            acc[3] += pg * pg;
            acc[4] += x[k] * x[k];
        }
    }
}

// eval_pack_owlqn under per-coordinate weights w[0..3] of the pack: lam_i = lam * w_i (owlqn_lam_i), the trial coordinates are
// owlqn_point_w, acc[1] takes sum w_i |x_i|, and `at(j)` returns the neighbour's owlqn_point_w under the neighbour's own weight
template <class T, class OBJ, class At>
__device__ __forceinline__ void eval_pack_owlqn_w(const OBJ& obj, int64_t i0, int64_t n, int cnt, const T (&xp)[4], const T (&d)[4],
                                                  const T (&gp)[4], const T (&w)[4], T step, T lam, At at, T (&x)[4], T (&g)[4], T* acc)
{
    T pgp[4], lw[4];
#pragma unroll
    for (int k = 0; k < 4; k++)
    {
        lw[k] = LBFGSpp::owlqn_lam_i(lam, w[k]);
        pgp[k] = LBFGSpp::owlqn_pg(xp[k], gp[k], lw[k]);
        x[k] = (k < cnt) ? (lw[k] > T(0) ? LBFGSpp::owlqn_project(xp[k] + step * d[k], LBFGSpp::owlqn_orthant(xp[k], pgp[k]))
                                         : xp[k] + step * d[k])
                         : T(0);
    }
    T xl = T(0), xr = T(0);
    if constexpr (OBJ::kHalo) pack_neighbours<false>(obj, i0, n, step, at, xl, xr);
    acc[0] += obj.eval(i0, cnt, x, xl, xr, g);
#pragma unroll
    for (int k = 0; k < 4; k++)
    {
        if (k < cnt)
        {
            const T pg = LBFGSpp::owlqn_pg(x[k], g[k], lw[k]);
            acc[1] += w[k] * (x[k] < T(0) ? -x[k] : x[k]);
            acc[2] += pgp[k] * (x[k] - xp[k]);
            acc[3] += pg * pg;
            acc[4] += x[k] * x[k];
        }
    }
}

}  // namespace lb
