// lbfgsb_kernels.cuh -- device kernels for the bound-constrained solver (LBFGSBSolver, BASELINE config 4).
//
// The reference walks std::vector<int> index sets (free / active / L / U / P) sequentially
// (reference Cauchy.h, SubspaceMin.h, BFGSMat.h:307-615).  On the GPU every index set is a bit in a per-coordinate
// class byte and every "gather rows of W, multiply, scatter" becomes a masked streaming pass over the S/Y columns:
//   W'(mask o v)       -> k_gram_dots on the masked vector            (apply_WtPv, compute_FtBAb; BFGSMat.h:382-433,486-522)
//   (W_P)'(W_P)        -> k_masked_gram                                (solve_PtBP; BFGSMat.h:529-565)
//   W_P * coef         -> k_hist_lincomb                               (apply_PtWMv, apply_PtBQv; BFGSMat.h:435-478,570-615)
// (k_hist_lincomb and k_hist_wt_dot_multi also serve blocks of up to 16 vectors: the operator form of the final approximation;
// k_hist_quad_diag forms its diagonal)
// The generalized Cauchy point (Cauchy.h:86-284) is sort + prefix sums: after sorting the breakpoints, the state of the
// reference's sequential sweep just after crossing sorted position k is a function of prefix sums over positions <= k
// (sum g^2, sum g*w, sum t*g*w with w = row of W), so all segments are examined in parallel and the first one whose
// one-dimensional minimiser falls inside it is selected with an integer atomicMin.  Same values as the sequential
// updates in exact arithmetic; rounding differs (the reference's own result already depends on std::sort's tie order).
#pragma once

#include "device_utils.cuh"
#include "two_loop_gram.cuh"
#include "philox.cuh"

namespace lb {

// CLS_FINAL: the free set at the solution (k_box_final_classes); Cauchy rebuilds the other bits on every iteration and leaves it be
enum : unsigned char { CLS_FIXED = 1, CLS_ACT = 2, CLS_FREE = 4, SUB_L = 8, SUB_U = 16, SUB_P = 32, CLS_FINAL = 64 };

// The masked forms of the history passes (the final approximation on the free variables): Masked<A> is the pass of argument form A
// restricted to the rows i with (fcls_i & fmask) != 0.  Each form keeps the order of A, so with every row in the mask it computes
// A's bits; unmasked<A> names A and says whether a form is masked.
template <class A> struct Masked : A
{
    const unsigned char* fcls;
    unsigned char fmask;
};
template <class A> struct unmasked
{
    using type = A;
    static constexpr bool masked = false;
};
template <class A> struct unmasked<Masked<A>>
{
    using type = A;
    static constexpr bool masked = true;
};

// ---------------------------------------------------------------- reductions with max slots
// like grid_reduce, but slots whose bit is set in `maxmask` take the maximum instead of the sum (exact, order-free)
template <int NV> __device__ __forceinline__ void grid_reduce_mixed(const double (&acc)[NV], const ReduceBuf& rb, unsigned maxmask)
{
    __shared__ double s_part[NV][kThreads / 32];
    __shared__ bool s_last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; k++)
    {
        double w = acc[k];
        const bool mx = (maxmask >> k) & 1u;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
        {
            const double other = __shfl_xor_sync(0xffffffffu, w, o);
            w = mx ? fmax(w, other) : w + other;
        }
        if (lane == 0) s_part[k][warp] = w;
    }
    __syncthreads();
    if (threadIdx.x < NV)
    {
        const bool mx = (maxmask >> threadIdx.x) & 1u;
        double t = s_part[threadIdx.x][0];
        for (int w = 1; w < kThreads / 32; w++) t = mx ? fmax(t, s_part[threadIdx.x][w]) : t + s_part[threadIdx.x][w];
        rb.partials[blockIdx.x * kMaxRed + threadIdx.x] = t;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(rb.ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (threadIdx.x < NV)
    {
        const bool mx = (maxmask >> threadIdx.x) & 1u;
        double t = __ldcg(&rb.partials[threadIdx.x]);
        for (unsigned b = 1; b < gridDim.x; b++)
        {
            const double v = __ldcg(&rb.partials[b * kMaxRed + threadIdx.x]);
            t = mx ? fmax(t, v) : t + v;
        }
        rb.result[threadIdx.x] = t;
    }
    if (threadIdx.x == 0) *rb.ticket = 0u;
    __threadfence();
    __syncthreads();
    deliver_to_host(rb, NV);
}

// ---------------------------------------------------------------- simple bound kernels (LBFGSB.h:55-86)
template <class T> __global__ void __launch_bounds__(kThreads) k_box_clamp(int64_t n, T* x, const T* __restrict__ lb, const T* __restrict__ ub)
{
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
        x[i] = fmin(fmax(x[i], lb[i]), ub[i]);   // x.cwiseMax(lb).cwiseMin(ub), LBFGSB.h:57
}

// out = { max_i |clamp(x - g) - x| }   (LBFGSB.h:62-65)
template <class T> __global__ void __launch_bounds__(kThreads) k_box_pgnorm(int64_t n, const T* __restrict__ x, const T* __restrict__ g,
                                                                           const T* __restrict__ lb, const T* __restrict__ ub, ReduceBuf rb)
{
    double m = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    {
        const T p = fmin(fmax(x[i] - g[i], lb[i]), ub[i]) - x[i];
        m = fmax(m, (double)fabs(p));
    }
    double acc[1] = {m};
    grid_reduce_mixed<1>(acc, rb, 1u);
}

// out = { g.d , -min_i feasible step }  (LBFGSB.h:176 and 68-86; the min is carried as a max of the negated value)
template <class T> __global__ void __launch_bounds__(kThreads) k_box_dirinfo(int64_t n, const T* __restrict__ x, const T* __restrict__ d,
                                                                            const T* __restrict__ g, const T* __restrict__ lb,
                                                                            const T* __restrict__ ub, ReduceBuf rb)
{
    T dot = T(0);
    double negmin = -INFINITY;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    {
        const T di = d[i];
        dot += g[i] * di;
        if (di > T(0)) negmin = fmax(negmin, -(double)((ub[i] - x[i]) / di));
        else if (di < T(0)) negmin = fmax(negmin, -(double)((lb[i] - x[i]) / di));
    }
    double acc[2] = {(double)dot, negmin};
    grid_reduce_mixed<2>(acc, rb, 2u);
}

// The free set at the solution: coordinate i is fixed when lb_i == ub_i or x_i lies within tol * max(1, |bound|) of a finite bound
// (the solver does not clamp at exit, so a point on a bound can miss it by an ulp); every other one is free and gets CLS_FINAL.
// out = { number of free coordinates }
template <class T> __global__ void __launch_bounds__(kThreads) k_box_final_classes(int64_t n, const T* __restrict__ x, const T* __restrict__ lb,
                                                                                  const T* __restrict__ ub, T tol, unsigned char* __restrict__ cls,
                                                                                  ReduceBuf rb)
{
    double nfree = 0;
    const T inf = (T)INFINITY;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    {
        const T xi = x[i], li = lb[i], ui = ub[i];
        const bool fixed = li == ui || (li > -inf && xi <= li + tol * fmax(T(1), fabs(li))) || (ui < inf && xi >= ui - tol * fmax(T(1), fabs(ui)));
        cls[i] = fixed ? (unsigned char)(cls[i] & ~CLS_FINAL) : (unsigned char)(cls[i] | CLS_FINAL);
        nfree += fixed ? 0.0 : 1.0;
    }
    double acc[1] = {nfree};
    grid_reduce_mixed<1>(acc, rb, 0u);
}

// ---------------------------------------------------------------- Cauchy point, phase 1 (Cauchy.h:111-129)
// brk_i, d_i = -g_i (0 for coordinates that cannot move); counts of the three kinds; d.d; smallest breakpoint
template <class T> __global__ void __launch_bounds__(kThreads) k_cauchy_breaks(int64_t n, const T* __restrict__ x, const T* __restrict__ g,
                                                                              const T* __restrict__ lb, const T* __restrict__ ub,
                                                                              T* __restrict__ brk, T* __restrict__ dvec,
                                                                              unsigned char* __restrict__ cls, ReduceBuf rb)
{
    double nfixed = 0, ninf = 0, nord = 0, dd = 0, negtmin = -INFINITY;
    const T inf = (T)INFINITY;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    {
        const T gi = g[i], xi = x[i], li = lb[i], ui = ub[i];
        T b;
        if (li == ui) b = T(0);
        else if (gi < T(0)) b = (xi - ui) / gi;
        else if (gi > T(0)) b = (xi - li) / gi;
        else b = inf;
        const bool zero = (b == T(0));
        const T di = zero ? T(0) : -gi;
        brk[i] = b;
        dvec[i] = di;
        dd += (double)(di * di);
        if (b == inf) { ninf += 1; cls[i] = CLS_FREE; }
        else if (!zero) { nord += 1; negtmin = fmax(negtmin, -(double)b); cls[i] = 0; }
        else { nfixed += 1; cls[i] = CLS_FIXED; }
    }
    double acc[5] = {nfixed, ninf, nord, dd, negtmin};
    grid_reduce_mixed<5>(acc, rb, 16u);
}

// ---------------------------------------------------------------- LSD radix sort of (key, index) pairs
// Replaces the reference's std::sort of the breakpoints (Cauchy.h:31-50).  Keys: bit patterns of the positive finite breakpoints
// (order-preserving as unsigned integers), padded with ~0 up to a whole number of tiles; payload: the coordinate index.  8 bits per
// pass, least significant digit first, every pass stable -- so equal keys end up ordered by index (deterministic; std::sort leaves
// ties unspecified).  Per pass: digit histogram of every 2048-pair tile -> exclusive scan over (digit, tile) -> stable scatter.
// The pair arrays (12 bytes per coordinate) stay in L2; fp64 keys take 8 passes, fp32 keys 4.
constexpr int kSortTile = 2048;   // pairs per CTA (256 threads: 8 warps x 8 rounds x 32 lanes)
constexpr int kRadix = 256;

__global__ void __launch_bounds__(kThreads) k_sort_fill(int64_t n, int64_t npad, const double* __restrict__ brk, const unsigned char* __restrict__ cls,
                                                       unsigned long long* keys, unsigned* idx)
{
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < npad; i += (int64_t)gridDim.x * kThreads)
    {
        unsigned long long k = ~0ull;
        if (i < n && cls[i] == 0) k = (unsigned long long)__double_as_longlong(brk[i]);
        keys[i] = k;
        idx[i] = (unsigned)i;
    }
}
__global__ void __launch_bounds__(kThreads) k_sort_fill_f32(int64_t n, int64_t npad, const float* __restrict__ brk, const unsigned char* __restrict__ cls,
                                                           unsigned long long* keys, unsigned* idx)
{
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < npad; i += (int64_t)gridDim.x * kThreads)
    {
        unsigned long long k = ~0ull;
        if (i < n && cls[i] == 0) k = (unsigned long long)__float_as_uint(brk[i]);
        keys[i] = k;
        idx[i] = (unsigned)i;
    }
}

// hist[d * ntiles + tile] = number of keys of the tile whose digit (bits [shift, shift+8)) is d
__global__ void __launch_bounds__(256) k_radix_hist(const unsigned long long* __restrict__ keys, int shift, unsigned* __restrict__ hist, unsigned ntiles)
{
    __shared__ unsigned s_hist[kRadix];
    s_hist[threadIdx.x] = 0u;
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * kSortTile;
    for (int t = threadIdx.x; t < kSortTile; t += 256) atomicAdd(&s_hist[(unsigned)(keys[base + t] >> shift) & 255u], 1u);
    __syncthreads();
    hist[(size_t)threadIdx.x * ntiles + blockIdx.x] = s_hist[threadIdx.x];
}

// exclusive scan of `total` counters in place (one CTA of 1024 threads; digit-major order = the order of the sorted output)
__global__ void __launch_bounds__(1024) k_radix_scan(unsigned* hist, unsigned total)
{
    __shared__ unsigned s_part[1024];
    const unsigned per = (total + 1023u) / 1024u;
    const unsigned lo = threadIdx.x * per, hi = (lo + per < total) ? lo + per : total;
    unsigned sum = 0u;
    for (unsigned i = lo; i < hi; i++) sum += hist[i];
    s_part[threadIdx.x] = sum;
    __syncthreads();
    for (unsigned off = 1; off < 1024u; off <<= 1)          // Hillis-Steele inclusive scan of the per-thread totals
    {
        const unsigned v = (threadIdx.x >= off) ? s_part[threadIdx.x - off] : 0u;
        __syncthreads();
        s_part[threadIdx.x] += v;
        __syncthreads();
    }
    unsigned run = (threadIdx.x == 0) ? 0u : s_part[threadIdx.x - 1];
    for (unsigned i = lo; i < hi; i++) { const unsigned c = hist[i]; hist[i] = run; run += c; }
}

// stable scatter of one tile: position = scanned[digit][tile] + (pairs of this tile with the same digit that come before)
__global__ void __launch_bounds__(256) k_radix_scatter(const unsigned long long* __restrict__ keys_in, const unsigned* __restrict__ idx_in,
                                                       unsigned long long* __restrict__ keys_out, unsigned* __restrict__ idx_out, int shift,
                                                       const unsigned* __restrict__ scanned, unsigned ntiles)
{
    __shared__ unsigned s_cnt[8][kRadix];     // per warp: pairs seen so far with each digit; later: exclusive offsets across warps
    __shared__ unsigned s_base[kRadix];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int t = threadIdx.x; t < 8 * kRadix; t += 256) (&s_cnt[0][0])[t] = 0u;
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * kSortTile + warp * 256;   // a warp owns 256 consecutive pairs, 32 per round
    unsigned long long key[8];
    unsigned rank[8];
#pragma unroll
    for (int r = 0; r < 8; r++)
    {
        key[r] = keys_in[base + r * 32 + lane];
        const unsigned d = (unsigned)(key[r] >> shift) & 255u;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int leader = __ffs(peers) - 1;
        unsigned old = 0u;
        if (lane == leader) { old = s_cnt[warp][d]; s_cnt[warp][d] = old + __popc(peers); }
        old = __shfl_sync(0xffffffffu, old, leader);
        rank[r] = old + __popc(peers & ((1u << lane) - 1u));
        __syncwarp();
    }
    __syncthreads();
    {
        const unsigned d = threadIdx.x;
        unsigned run = 0u;
#pragma unroll
        for (int w = 0; w < 8; w++) { const unsigned c = s_cnt[w][d]; s_cnt[w][d] = run; run += c; }
        s_base[d] = scanned[(size_t)d * ntiles + blockIdx.x];
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 8; r++)
    {
        const unsigned d = (unsigned)(key[r] >> shift) & 255u;
        const unsigned pos = s_base[d] + s_cnt[warp][d] + rank[r];
        keys_out[pos] = key[r];
        idx_out[pos] = idx_in[base + r * 32 + lane];
    }
}

// ---------------------------------------------------------------- Cauchy point, phase 2: the sweep as prefix sums
// Per sorted position k (coordinate i = ord[k], t = brk_i, g = g_i):  e_k = [ g^2 , g*w_i (2c) , t*g*w_i (2c) ],
// w_i = (y_0[i..c), theta*s_0[i..c)) by age.  Block sums -> block offsets -> per-position prefix -> segment test.
constexpr int kScanBlock = 128;
constexpr int kMaxW = 2 * kMaxM;   // 2c <= 128

template <class T> struct SweepArgs
{
    int64_t nord, ld;
    const unsigned long long* keys;   // sorted
    const unsigned* ord;              // sorted coordinate indices
    const T* g;
    const T* S;
    const T* Y;
    int c;
    T theta;
    unsigned char slots[kMaxM];
    // inputs for the segment test
    const T* Mmat;      // [2c][2c] row-major, device
    const T* p0;        // [2c]  W'd at t = 0
    T gt;               // sum of g_i^2 over moving coordinates ( = d.d )
    int nfree_inf;      // coordinates that never hit a bound
    // scratch / outputs
    T* block_sums;      // [nblocks][4c+1]
    long long* best;    // smallest qualifying sorted position (group end), initialised to LLONG_MAX
    T* out;             // finalize: [0]=t_cross, [1]=tfinal, [2]=fp, [3]=fpp, [4..4+2c) = vecc (W'(xcp-x0))
};

template <class T> __device__ __forceinline__ T key_to_t(unsigned long long k);
template <> __device__ __forceinline__ double key_to_t<double>(unsigned long long k) { return __longlong_as_double((long long)k); }
template <> __device__ __forceinline__ float key_to_t<float>(unsigned long long k) { return __uint_as_float((unsigned)k); }

// e_k into registers: nv = 4c+1 values
template <class T> __device__ __forceinline__ void sweep_element(const SweepArgs<T>& a, int64_t k, T* e /*[4c+1]*/)
{
    const int c = a.c, nv = 4 * c + 1;
    if (k >= a.nord) { for (int q = 0; q < nv; q++) e[q] = T(0); return; }
    const int64_t i = a.ord[k];
    const T gi = a.g[i];
    const T t = key_to_t<T>(a.keys[k]);
    e[0] = gi * gi;
    for (int j = 0; j < c; j++)
    {
        const T wy = a.Y[(int64_t)a.slots[j] * a.ld + i];
        const T ws = a.theta * a.S[(int64_t)a.slots[j] * a.ld + i];
        e[1 + j] = gi * wy;
        e[1 + c + j] = gi * ws;
        e[1 + 2 * c + j] = t * gi * wy;
        e[1 + 3 * c + j] = t * gi * ws;
    }
}

// pass 1: per-block totals (one thread per position, block = kScanBlock positions)
template <class T, int MAXV> __global__ void __launch_bounds__(kScanBlock) k_sweep_blocksum(SweepArgs<T> a)
{
    __shared__ T red[kScanBlock / 32][MAXV];
    const int nv = 4 * a.c + 1;
    T e[MAXV];
    sweep_element<T>(a, (int64_t)blockIdx.x * kScanBlock + threadIdx.x, e);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int q = 0; q < nv; q++)
    {
        T w = e[q];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
        if (lane == 0) red[warp][q] = w;
    }
    __syncthreads();
    for (int q = threadIdx.x; q < nv; q += kScanBlock)
    {
        T t = T(0);
        for (int w = 0; w < kScanBlock / 32; w++) t += red[w][q];
        a.block_sums[(int64_t)blockIdx.x * nv + q] = t;
    }
}

// pass 2: exclusive scan of the block totals, in place (one CTA; thread q owns value q, walks the blocks in order)
template <class T> __global__ void k_sweep_scan_blocks(T* block_sums, int64_t nblocks, int nv)
{
    // one warp per value: the lanes take 32 contiguous runs of blocks, sum them, the warp scans the 32 run totals with a fixed
    // shuffle ladder, every lane rewrites its run with the running prefix (a single thread walking 7800 blocks cost ~1 ms of L2
    // round trips per Cauchy point at n = 1e6)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int64_t per = (nblocks + 31) / 32;
    const int64_t lo = lane * per, hi = (lo + per < nblocks) ? lo + per : nblocks;
    for (int q = warp; q < nv; q += nwarps)
    {
        T sum = T(0);
#pragma unroll 4
        for (int64_t b = lo; b < hi; b++) sum += block_sums[b * nv + q];
        T incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1)
        {
            const T up = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += up;
        }
        T run = __shfl_up_sync(0xffffffffu, incl, 1);   // exclusive prefix of this lane's run
        if (lane == 0) run = T(0);
#pragma unroll 4
        for (int64_t b = lo; b < hi; b++)
        {
            const T v = block_sums[b * nv + q];
            block_sums[b * nv + q] = run;
            run += v;
        }
    }
}

// segment quantities at the START of the segment that follows sorted position k (all positions <= k crossed):
//   p = p0 + A ; c = t*p - C ; fp = -(gt - G)(1 - theta t) - p'M c ; fpp = theta (gt - G) - p'M p
template <class T> __device__ __forceinline__ void segment_eval(const SweepArgs<T>& a, const T* pre /*[4c+1] inclusive prefix*/, T t,
                                                                T& fp, T& fpp, T* pvec /*[2c]*/, T* cvec /*[2c]*/)
{
    const int w = 2 * a.c;
    const T rest = a.gt - pre[0];
    for (int q = 0; q < w; q++)
    {
        pvec[q] = a.p0[q] + pre[1 + q];
        cvec[q] = t * pvec[q] - pre[1 + w + q];
    }
    T pMc = T(0), pMp = T(0);
    for (int r = 0; r < w; r++)
    {
        T mc = T(0), mp = T(0);
        for (int q = 0; q < w; q++)
        {
            const T m = a.Mmat[r * w + q];
            mc += m * cvec[q];
            mp += m * pvec[q];
        }
        pMc += pvec[r] * mc;
        pMp += pvec[r] * mp;
    }
    fp = -rest * (T(1) - a.theta * t) - pMc;
    fpp = a.theta * rest - pMp;
}

// pass 3: in-block inclusive scan + segment test; FINALIZE = false: atomicMin of the first qualifying group end;
// FINALIZE = true (grid of one CTA = the block that holds *best): write the result for that position
template <class T, int MAXV, bool FINALIZE> __global__ void __launch_bounds__(kScanBlock) k_sweep_select(SweepArgs<T> a, long long target)
{
    extern __shared__ __align__(16) unsigned char sweep_smem[];
    const int nv = 4 * a.c + 1;
    T (*scan)[MAXV + 1] = reinterpret_cast<T (*)[MAXV + 1]>(sweep_smem);
    const int64_t blk = FINALIZE ? (target / kScanBlock) : blockIdx.x;
    const int64_t k = blk * kScanBlock + threadIdx.x;
    T e[MAXV];
    sweep_element<T>(a, k, e);
    for (int q = 0; q < nv; q++) scan[threadIdx.x][q] = e[q];
    __syncthreads();
    // Hillis-Steele inclusive scan over the kScanBlock rows, all nv values
    for (int off = 1; off < kScanBlock; off <<= 1)
    {
        T add[MAXV];
        const bool act = threadIdx.x >= off;
        if (act) for (int q = 0; q < nv; q++) add[q] = scan[threadIdx.x - off][q];
        __syncthreads();
        if (act) for (int q = 0; q < nv; q++) scan[threadIdx.x][q] += add[q];
        __syncthreads();
    }
    if (k >= a.nord) return;
    T pre[MAXV];
    for (int q = 0; q < nv; q++) pre[q] = scan[threadIdx.x][q] + a.block_sums[blk * nv + q];
    const T t = key_to_t<T>(a.keys[k]);
    const bool last = (k + 1 == a.nord);
    const T tnext = last ? (T)INFINITY : key_to_t<T>(a.keys[k + 1]);
    if (!last && tnext == t) return;          // not the end of its tie group
    if (FINALIZE && k != target) return;
    T fp, fpp, pvec[kMaxW], cvec[kMaxW];
    segment_eval<T>(a, pre, t, fp, fpp, pvec, cvec);
    if (!FINALIZE)
    {
        // Cauchy.h:183 `while (deltatmin >= deltat)`: the sweep stops in the first segment with deltatmin < deltat.
        // Crossing the very last group with no never-bounded coordinate left ends the sweep too (Cauchy.h:190-201).
        const T dtmin = -fp / fpp;
        const T dt = tnext - t;
        const bool all_crossed = last && a.nfree_inf == 0;
        if (!(dtmin >= dt) || all_crossed) atomicMin((unsigned long long*)a.best, (unsigned long long)k);
        return;
    }
    // finalize (Cauchy.h:258-283)
    const int w = 2 * a.c;
    const bool all_crossed = last && a.nfree_inf == 0;
    T dtmin = -fp / fpp;
    const T eps = (sizeof(T) == 8) ? (T)2.220446049250313e-16 : (T)1.1920929e-07f;
    if (fpp < eps) dtmin = -fp / eps;
    dtmin = fmax(dtmin, T(0));
    if (all_crossed) dtmin = T(0);
    a.out[0] = t;
    a.out[1] = t + dtmin;
    a.out[2] = fp;
    a.out[3] = fpp;
    a.out[4] = all_crossed ? T(1) : T(0);
    for (int q = 0; q < w; q++) a.out[5 + q] = cvec[q] + dtmin * pvec[q];   // W'(xcp - x0) at tfinal
}

// ---------------------------------------------------------------- Cauchy point, phase 3: build xcp and the class bytes
// crossed (brk <= t_cross): xcp = bound, class ACT ; otherwise xcp = x0 + tfinal*d, class FREE ; fixed stay (Cauchy.h:205-216,268-283)
template <class T> __global__ void __launch_bounds__(kThreads) k_cauchy_build(int64_t n, const T* __restrict__ x, const T* __restrict__ dvec,
                                                                             const T* __restrict__ brk, const T* __restrict__ lb,
                                                                             const T* __restrict__ ub, T t_cross, T tfinal,
                                                                             T* __restrict__ xcp, unsigned char* __restrict__ cls, ReduceBuf rb)
{
    double nact = 0, nfree = 0;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    {
        const unsigned char c0 = cls[i];
        T out = x[i];
        unsigned char c1 = c0;
        if (c0 != CLS_FIXED)
        {
            const bool crossed = (c0 != CLS_FREE) && (brk[i] <= t_cross);
            if (crossed) { out = (dvec[i] > T(0)) ? ub[i] : lb[i]; c1 = CLS_ACT; nact += 1; }
            else { out = x[i] + tfinal * dvec[i]; c1 = CLS_FREE; nfree += 1; }
        }
        xcp[i] = out;
        cls[i] = c1;
    }
    double acc[2] = {nact, nfree};
    grid_reduce_mixed<2>(acc, rb, 0u);
}

// ---------------------------------------------------------------- history primitives on blocks of k vectors
// Both passes read every history column once per call, whatever k (1 <= k <= kMaxK): one product with the compact form of B or H
// moves w*n*(4c + 3k) bytes instead of w*n*(4c + 3)*k for k single-vector passes.
constexpr int kMaxK = 16;

// OUT[:,j] = a0*V[:,j] + sum_a C[a][j]*y_a + C[c+a][j]*s_a   (C row-major [2c][k], y then s by age; V == nullptr: no a0 term)
// for rows with (cls_i & mask) != 0 (cls == nullptr: all rows); rows outside the mask are left untouched.  Per element the terms are
// added in the order a0*v, y by age, s by age; with k = 1 this is the L-BFGS-B combination (apply_PtWMv / apply_PtBQv / solve_PtBP).
template <class T> struct LincombArgs
{
    int64_t n, ld, ldv, ldo;
    const T* S;
    const T* Y;
    const T* V;        // may be nullptr
    T a0;
    const T* coef;     // device [2c][k]
    const unsigned char* cls;
    unsigned char mask;
    T* out;
    int c, k;
    unsigned char slots[kMaxM];
};

// The sampler's form (LincombNormalArgs): V is not read but generated, z_j = the normals of draw first + j (philox.cuh), and
// OUT[:,j] = mean + a0*z_j + sum_a C[c+a][j]*s_a (mean == nullptr: no mean term; the y rows of C are not read, they are zero).  A
// thread takes the coordinate pair (2q, 2q + 1) that one generator call serves; per element the terms are added in the order
// mean, a0*z, s by age.
template <class T> struct LincombNormalArgs : LincombArgs<T>
{
    const T* mean;
    NormalSrc src;
};

// Masked<LincombNormalArgs>: the draws of N(mean, H_F) on the free rows (mean_i elsewhere), so the y rows of C are read too: per element
// mean, a0*z, y by age, s by age; with zero y rows and every row in the mask, the bits of the unmasked form.
template <class T, int KMAX, class A> __device__ __forceinline__ void k_hist_lincomb_normal(const A& a)
{
    constexpr bool kMask = unmasked<A>::masked;
    __shared__ T s_coef[kMaxW * KMAX];
    __shared__ const T* s_s[kMask ? 2 * kMaxM : kMaxM];   // masked: the y columns at kMaxM + age
    const int k = KMAX == 1 ? 1 : a.k;
    for (int e = threadIdx.x; e < 2 * a.c * k; e += kThreads) s_coef[e] = a.coef[e];
    for (int j = threadIdx.x; j < a.c; j += kThreads) s_s[j] = a.S + (int64_t)a.slots[j] * a.ld;
    if constexpr (kMask)
        for (int j = threadIdx.x; j < a.c; j += kThreads) s_s[kMaxM + j] = a.Y + (int64_t)a.slots[j] * a.ld;
    __syncthreads();
    const int64_t npairs = (a.n + 1) / 2;
    for (int64_t q = (int64_t)blockIdx.x * kThreads + threadIdx.x; q < npairs; q += (int64_t)gridDim.x * kThreads)
    {
        const int64_t i0 = 2 * q;
        const bool two = i0 + 1 < a.n;
        const T m0 = a.mean ? a.mean[i0] : T(0), m1 = a.mean && two ? a.mean[i0 + 1] : T(0);
        T r0[KMAX], r1[KMAX];
#pragma unroll
        for (int j = 0; j < KMAX; j++)
            if (j < k)
            {
                double z0, z1;
                normal_pair(a.src.seed, a.src.stream, a.src.first + (uint32_t)j, (unsigned long long)q, z0, z1);
                r0[j] = a.mean ? m0 + a.a0 * (T)z0 : a.a0 * (T)z0;
                r1[j] = a.mean ? m1 + a.a0 * (T)z1 : a.a0 * (T)z1;
            }
        if constexpr (kMask)
            for (int p = 0; p < a.c; p++)
            {
                const T y0 = s_s[kMaxM + p][i0], y1 = two ? s_s[kMaxM + p][i0 + 1] : T(0);
#pragma unroll
                for (int j = 0; j < KMAX; j++)
                    if (j < k)
                    {
                        r0[j] += s_coef[p * k + j] * y0;
                        r1[j] += s_coef[p * k + j] * y1;
                    }
            }
        for (int p = 0; p < a.c; p++)
        {
            const T s0 = s_s[p][i0], s1 = two ? s_s[p][i0 + 1] : T(0);
#pragma unroll
            for (int j = 0; j < KMAX; j++)
                if (j < k)
                {
                    r0[j] += s_coef[(a.c + p) * k + j] * s0;
                    r1[j] += s_coef[(a.c + p) * k + j] * s1;
                }
        }
        bool in0 = true, in1 = true;
        if constexpr (kMask)
        {
            in0 = (a.fcls[i0] & a.fmask) != 0;
            in1 = two && (a.fcls[i0 + 1] & a.fmask) != 0;
        }
#pragma unroll
        for (int j = 0; j < KMAX; j++)
            if (j < k)
            {
                a.out[j * a.ldo + i0] = in0 ? r0[j] : m0;
                if (two) a.out[j * a.ldo + i0 + 1] = in1 ? r1[j] : m1;
            }
    }
}

// KMAX: 1 (the L-BFGS-B pass, and any k = 1 call) or kMaxK; the k running sums of an element stay in registers.  Masked<LincombArgs>:
// rows outside the mask are written as 0 instead of being skipped.
template <class T, int KMAX, class A = LincombArgs<T>> __global__ void __launch_bounds__(kThreads) k_hist_lincomb(A a)
{
    constexpr bool kMask = unmasked<A>::masked;
    if constexpr (!std::is_same<typename unmasked<A>::type, LincombArgs<T>>::value)
    {
        k_hist_lincomb_normal<T, KMAX>(a);
        return;
    }
    else
    {
    __shared__ T s_coef[kMaxW * KMAX];
    __shared__ const T* s_y[kMaxM];
    __shared__ const T* s_s[kMaxM];
    const int k = KMAX == 1 ? 1 : a.k;
    for (int e = threadIdx.x; e < 2 * a.c * k; e += kThreads) s_coef[e] = a.coef[e];
    for (int j = threadIdx.x; j < a.c; j += kThreads)
    {
        s_y[j] = a.Y + (int64_t)a.slots[j] * a.ld;
        s_s[j] = a.S + (int64_t)a.slots[j] * a.ld;
    }
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * kThreads)
    {
        if constexpr (kMask)
        {
            if (!(a.fcls[i] & a.fmask))
            {
#pragma unroll
                for (int j = 0; j < KMAX; j++)
                    if (j < k) a.out[j * a.ldo + i] = T(0);
                continue;
            }
        }
        else if (a.cls && !(a.cls[i] & a.mask)) continue;
        T r[KMAX];
#pragma unroll
        for (int j = 0; j < KMAX; j++)
            if (j < k) r[j] = a.V ? a.a0 * a.V[j * a.ldv + i] : T(0);
        for (int q = 0; q < a.c; q++)
        {
            const T yq = s_y[q][i];
#pragma unroll
            for (int j = 0; j < KMAX; j++)
                if (j < k) r[j] += s_coef[q * k + j] * yq;
        }
        for (int q = 0; q < a.c; q++)
        {
            const T sq = s_s[q][i];
#pragma unroll
            for (int j = 0; j < KMAX; j++)
                if (j < k) r[j] += s_coef[(a.c + q) * k + j] * sq;
        }
#pragma unroll
        for (int j = 0; j < KMAX; j++)
            if (j < k) a.out[j * a.ldo + i] = r[j];
    }
    }
}

// The diagonal of a0 I + W K W' (W = [Y S] by age, K symmetric 2c x 2c): out_i = a0 + r_i' K r_i, r_i = row i of W.  Kp holds the
// upper triangle packed row by row with the off-diagonal entries doubled, in double: row p is K_pp, 2K_p,p+1, ..., 2K_p,2c-1.  Per
// element, with every operation in fp64 (fp32 storage is taken up to double) and every multiply-add a fused fma:
//     t_p = Kp_pp r_p,  t_p = fma(Kp_pq, r_q, t_p) for q = p+1, ..., 2c-1;   acc = 0,  acc = fma(r_p, t_p, acc) for p = 0, ..., 2c-1;
//     out_i = a0 + acc
// so out_i depends on row i and K only (not on the grid, n or i).  2c^2 + 3c multiply-adds per element over (2c + 1) words.
// WMAX >= 2c: the row sits in registers (loops unrolled for WMAX <= 64; at 64 part of it stays on the stack) and each K value read
// from shared memory serves RPT rows; WMAX = kMaxW (c > 32) keeps the row in local memory.
template <class T> struct QuadDiagArgs
{
    int64_t n, ld;
    const T* S;
    const T* Y;
    const double* Kp;   // device, w(w+1)/2 values
    double a0;
    T* out;
    int c;
    unsigned char slots[kMaxM];
};

template <int WMAX> __host__ __device__ constexpr int quad_diag_rpt() { return WMAX <= 32 ? 64 / WMAX : 1; }

// Masked<QuadDiagArgs>: out_i = 0 on the rows outside the mask
template <class T, int WMAX, class A = QuadDiagArgs<T>> __global__ void __launch_bounds__(kThreads) k_hist_quad_diag(A a)
{
    constexpr int RPT = quad_diag_rpt<WMAX>();
    constexpr int UNROLL = WMAX <= 64 ? WMAX : 1;
    extern __shared__ double s_kp[];
    __shared__ const T* s_col[kMaxW];
    const int c = a.c, w = 2 * c;
    for (int e = threadIdx.x; e < w * (w + 1) / 2; e += kThreads) s_kp[e] = a.Kp[e];
    for (int q = threadIdx.x; q < w; q += kThreads) s_col[q] = (q < c ? a.Y + (int64_t)a.slots[q] * a.ld : a.S + (int64_t)a.slots[q - c] * a.ld);
    __syncthreads();
    const int64_t span = (int64_t)kThreads * RPT;
    for (int64_t i0 = (int64_t)blockIdx.x * span + threadIdx.x; i0 < a.n; i0 += (int64_t)gridDim.x * span)
    {
        double r[RPT][WMAX];
#pragma unroll
        for (int j = 0; j < RPT; j++)
        {
            const int64_t i = i0 + (int64_t)j * kThreads;
#pragma unroll UNROLL
            for (int q = 0; q < WMAX; q++)
                if (q < w) r[j][q] = i < a.n ? (double)s_col[q][i] : 0.0;
        }
        double acc[RPT];
#pragma unroll
        for (int j = 0; j < RPT; j++) acc[j] = 0.0;
        int off = 0;   // row p of the packed triangle starts at off
#pragma unroll UNROLL
        for (int p = 0; p < WMAX; p++)
        {
            if (p < w)
            {
                double t[RPT];
#pragma unroll
                for (int j = 0; j < RPT; j++) t[j] = s_kp[off] * r[j][p];
#pragma unroll UNROLL
                for (int q = p + 1; q < WMAX; q++)
                {
                    if (q < w)
                    {
                        const double kq = s_kp[off + q - p];
#pragma unroll
                        for (int j = 0; j < RPT; j++) t[j] = fma(kq, r[j][q], t[j]);
                    }
                }
#pragma unroll
                for (int j = 0; j < RPT; j++) acc[j] = fma(r[j][p], t[j], acc[j]);
                off += w - p;
            }
        }
#pragma unroll
        for (int j = 0; j < RPT; j++)
        {
            const int64_t i = i0 + (int64_t)j * kThreads;
            if constexpr (unmasked<A>::masked)
            {
                if (i < a.n) a.out[i] = (a.fcls[i] & a.fmask) ? (T)(a.a0 + acc[j]) : T(0);
            }
            else if (i < a.n) a.out[i] = (T)(a.a0 + acc[j]);
        }
    }
}

// R[2c][k] = [Y S]' V  (y then s by age), summed in fp64.  A CTA stages a strip of kWtRows rows of the 2c history columns and of the
// k vectors in shared memory (every element read once from HBM) and thread (g, j) accumulates the dots of vector j = tid % k with
// columns g, g + G, ... (G = kThreads / k groups).  Strips go to CTAs round robin and the grid depends on n only, so a dot's sum
// (over a CTA's strips in order, then over CTAs in order by the last CTA) does not depend on k: column j of a k = 16 call is
// bit-identical to the k = 1 call on that column alone.
constexpr int kWtRows = 128;
constexpr int kWtPitch = kWtRows + 1;   // row pitch of the staged strip: the k threads reading one row index hit k different banks
template <class T> struct WtDotMultiArgs
{
    int64_t n, ld, ldv;
    const T* S;
    const T* Y;
    const T* V;
    int c, k;
    double* partials;   // [grid][2c*k]
    unsigned* ticket;
    double* result;     // [2c*k]
    unsigned char slots[kMaxM];
};

// The sampler's form (WtDotNormalArgs): the k vectors are not read but generated, vector j = the normals of draw first + j
// (philox.cuh), staged into the same strip rows as loaded vectors, so every dot keeps the order above.
template <class T> struct WtDotNormalArgs : WtDotMultiArgs<T>
{
    NormalSrc src;
};

// The whitening forms.  WtDotSArgs: the s columns alone, R[c][k] = S'V by age, each dot summed exactly as the s row of that age in
// the form above.  WtDotDiffArgs: vector j is staged as x_j - mean (V holds the points x_j), formed in T as the two-operand pass
// lbfgs_b200_axpy_out(x, -1, mean) forms it, and one more column per vector, the vector row itself, gives |x_j - mean|^2 in the
// same order; the result holds R[2c][k] and then the k squared norms.
template <class T> struct WtDotSArgs : WtDotMultiArgs<T>
{
};
template <class T> struct WtDotDiffArgs : WtDotMultiArgs<T>
{
    const T* mean;
};

// Masked<WtDotMultiArgs / WtDotDiffArgs / WtDotNormalArgs>: the vector rows outside the mask (loaded, differences or generated) are
// staged as 0, the history rows as always, so every dot and norm is taken over the rows of the mask in the order above.
template <class T, class A = WtDotMultiArgs<T>> __global__ void __launch_bounds__(kThreads) k_hist_wt_dot_multi(A a)
{
    using B = typename unmasked<A>::type;
    constexpr bool kMask = unmasked<A>::masked;
    constexpr bool kGen = std::is_same<B, WtDotNormalArgs<T>>::value;
    constexpr bool kSOnly = std::is_same<B, WtDotSArgs<T>>::value;
    constexpr bool kDiff = std::is_same<B, WtDotDiffArgs<T>>::value;
    static_assert(!(kMask && kSOnly), "no masked S-only form");
    extern __shared__ __align__(16) unsigned char wt_smem[];
    T* rows = reinterpret_cast<T*>(wt_smem);   // [w + k][kWtPitch]: y by age, s by age (S only: s by age), then the k vectors
    __shared__ const T* s_col[kMaxW + kMaxK];
    __shared__ bool s_last;
    __shared__ bool s_in[kMask ? kWtRows : 1];   // masked: whether row r of the strip is in the mask
    const int w = kSOnly ? a.c : 2 * a.c, k = a.k, nrows = w + k, tid = threadIdx.x;
    const int ncol = kDiff ? w + 1 : w;   // dots per vector: the history columns, and for kDiff the vector with itself
    const int nload = kGen ? w : nrows;   // rows staged from memory
    for (int q = tid; q < nload; q += kThreads)
        if constexpr (kSOnly) s_col[q] = q < w ? a.S + (int64_t)a.slots[q] * a.ld : a.V + (int64_t)(q - w) * a.ldv;
        else s_col[q] = q < a.c ? a.Y + (int64_t)a.slots[q] * a.ld : q < w ? a.S + (int64_t)a.slots[q - a.c] * a.ld : a.V + (int64_t)(q - w) * a.ldv;
    const int groups = kThreads / k, j = tid % k, g = tid / k;
    const bool active = g < groups;
    constexpr int kMaxOwn = kMaxW / (kThreads / kMaxK) + (kDiff ? 1 : 0);   // columns per thread: ceil(ncol / G) with G >= 16
    double acc[kMaxOwn];
#pragma unroll
    for (int q = 0; q < kMaxOwn; q++) acc[q] = 0.0;
    __syncthreads();
    const int64_t nstrips = (a.n + kWtRows - 1) / kWtRows;
    for (int64_t strip = blockIdx.x; strip < nstrips; strip += gridDim.x)
    {
        const int64_t r0 = strip * kWtRows;
        if constexpr (kMask)
        {
            for (int r = tid; r < kWtRows; r += kThreads) s_in[r] = r0 + r < a.n && (a.fcls[r0 + r] & a.fmask) != 0;
            __syncthreads();
            for (int t = tid; t < nload * kWtRows; t += kThreads)   // every load issued as in the unmasked form, then selected
            {
                const int q = t / kWtRows, r = t % kWtRows;
                const int64_t i = r0 + r;
                T v;
                if constexpr (kDiff) v = i < a.n ? (q < w ? __ldcs(s_col[q] + i) : __ldcs(s_col[q] + i) - a.mean[i]) : T(0);
                else v = i < a.n ? __ldcs(s_col[q] + i) : T(0);
                rows[q * kWtPitch + r] = (q < w || s_in[r]) ? v : T(0);
            }
        }
        else
            for (int t = tid; t < nload * kWtRows; t += kThreads)
            {
                const int q = t / kWtRows, r = t % kWtRows;
                const int64_t i = r0 + r;
                if constexpr (kDiff) rows[q * kWtPitch + r] = i < a.n ? (q < w ? __ldcs(s_col[q] + i) : __ldcs(s_col[q] + i) - a.mean[i]) : T(0);
                else rows[q * kWtPitch + r] = i < a.n ? __ldcs(s_col[q] + i) : T(0);
            }
        if constexpr (kGen)
            for (int t = tid; t < k * (kWtRows / 2); t += kThreads)   // one generator call per coordinate pair (r0 is even)
            {
                const int jv = t / (kWtRows / 2), r = 2 * (t % (kWtRows / 2));
                const int64_t i = r0 + r;
                double z0, z1;
                normal_pair(a.src.seed, a.src.stream, a.src.first + (uint32_t)jv, (unsigned long long)(i / 2), z0, z1);
                if constexpr (kMask)
                {
                    rows[(w + jv) * kWtPitch + r] = s_in[r] ? (T)z0 : T(0);
                    rows[(w + jv) * kWtPitch + r + 1] = s_in[r + 1] ? (T)z1 : T(0);
                }
                else
                {
                    rows[(w + jv) * kWtPitch + r] = i < a.n ? (T)z0 : T(0);
                    rows[(w + jv) * kWtPitch + r + 1] = i + 1 < a.n ? (T)z1 : T(0);
                }
            }
        __syncthreads();
        if (active)
        {
            // one running sum per owned column over the strip's rows in order; the vector's element is read once per row
            const T* vr = rows + (w + j) * kWtPitch;
            double s[kMaxOwn];
#pragma unroll
            for (int q = 0; q < kMaxOwn; q++) s[q] = 0.0;
            for (int r = 0; r < kWtRows; r++)
            {
                const double v = (double)vr[r];
#pragma unroll
                for (int q = 0; q < kMaxOwn; q++)
                    if constexpr (kDiff)
                    {
                        const int col = g + q * groups;
                        if (col < ncol) s[q] += (double)rows[(col < w ? col : w + j) * kWtPitch + r] * v;
                    }
                    else if (g + q * groups < w) s[q] += (double)rows[(g + q * groups) * kWtPitch + r] * v;
            }
#pragma unroll
            for (int q = 0; q < kMaxOwn; q++) acc[q] += s[q];
        }
        __syncthreads();
    }
    if (active)
#pragma unroll
        for (int q = 0; q < kMaxOwn; q++)
        {
            const int col = g + q * groups;
            if (col < ncol) a.partials[(size_t)blockIdx.x * (ncol * k) + col * k + j] = acc[q];
        }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(a.ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    for (int e = tid; e < ncol * k; e += kThreads)
    {
        double t = 0.0;
        for (unsigned b = 0; b < gridDim.x; b++) t += __ldcg(&a.partials[(size_t)b * (ncol * k) + e]);
        a.result[e] = t;
    }
    if (tid == 0) *a.ticket = 0u;
}

// G[a][b] = sum over masked rows of r_i[a]*r_i[b],  r_i = (y_0[i]..y_{c-1}[i], s_0[i]..s_{c-1}[i]) by age.
// One CTA handles a strip of rows: rows are staged through shared memory (coalesced column reads) and every thread
// accumulates a fixed set of (a,b) entries over the strip; per-CTA partials are summed in CTA order by the last CTA.
constexpr int kMgRows = 128;      // rows per staged strip

template <class T> struct MaskedGramArgs
{
    int64_t n, ld;
    const T* S;
    const T* Y;
    const unsigned char* cls;
    unsigned char mask;
    int c;
    double* partials;   // [grid][(2c)^2]
    unsigned* ticket;
    double* result;     // [(2c)^2]
    const XComm* xc;
    unsigned long long epoch;
    unsigned char slots[kMaxM];
};

template <class T> __global__ void __launch_bounds__(kThreads) k_masked_gram(MaskedGramArgs<T> a)
{
    extern __shared__ __align__(16) unsigned char mg_smem[];
    T* rows = reinterpret_cast<T*>(mg_smem);          // [2c][kMgRows]
    __shared__ bool s_last;
    const int w = 2 * a.c, nent = w * w;
    // entries owned by this thread: e = tid, tid + 256, ...
    constexpr int kMaxOwn = (kMaxW * kMaxW + kThreads - 1) / kThreads;   // 64 for 2c = 128
    double acc[kMaxOwn];
#pragma unroll
    for (int q = 0; q < kMaxOwn; q++) acc[q] = 0.0;
    const int64_t nstrips = (a.n + kMgRows - 1) / kMgRows;
    for (int64_t strip = blockIdx.x; strip < nstrips; strip += gridDim.x)
    {
        const int64_t r0 = strip * kMgRows;
        for (int t = threadIdx.x; t < w * kMgRows; t += kThreads)
        {
            const int col = t / kMgRows, r = t % kMgRows;
            const int64_t i = r0 + r;
            T v = T(0);
            if (i < a.n && (a.cls == nullptr || (a.cls[i] & a.mask)))
                v = (col < a.c) ? a.Y[(int64_t)a.slots[col] * a.ld + i] : a.S[(int64_t)a.slots[col - a.c] * a.ld + i];
            rows[col * kMgRows + r] = v;
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < kMaxOwn; q++)
        {
            const int e = threadIdx.x + q * kThreads;
            if (e < nent)
            {
                const T* ra = rows + (e / w) * kMgRows;
                const T* rbp = rows + (e % w) * kMgRows;
                T s = T(0);
                for (int r = 0; r < kMgRows; r++) s += ra[r] * rbp[r];
                acc[q] += (double)s;
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < kMaxOwn; q++)
    {
        const int e = threadIdx.x + q * kThreads;
        if (e < nent) a.partials[(size_t)blockIdx.x * nent + e] = acc[q];
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(a.ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    for (int e = threadIdx.x; e < nent; e += kThreads)
    {
        double t = 0.0;
        for (unsigned b = 0; b < gridDim.x; b++) t += __ldcg(&a.partials[(size_t)b * nent + e]);
        a.result[e] = t;
    }
    if (threadIdx.x == 0) *a.ticket = 0u;
}

// ---------------------------------------------------------------- subspace minimisation, element-wise steps
// (SubspaceMin.h:122-302).  Per-coordinate state lives in n-vectors owned by the box workspace; index sets are bits of
// the class byte.  Every step is one pass over n with at most three counters reduced.
template <class T> struct SubVec
{
    int64_t n;
    const T *x0, *xcp, *g, *lb, *ub;
    unsigned char* cls;
    T *vecc, *vecy, *lambda, *mu, *tmp, *tmp2, *yfb, *drt;
    T theta;
};

enum { SUB_OP_INIT = 0, SUB_OP_ACT_DIR = 1, SUB_OP_ADD_G = 2, SUB_OP_NEG_C_FREE = 3, SUB_OP_CHECK_BOUNDS = 4,
       SUB_OP_CLASSIFY = 5, SUB_OP_LU_VEC = 6, SUB_OP_RHS_P = 7, SUB_OP_FREE_VEC = 8, SUB_OP_MULTIPLIERS = 9,
       SUB_OP_CONVERGED = 10, SUB_OP_WRITE_DRT = 11, SUB_OP_COUNT = 12 };

template <class T, int OP> __global__ void __launch_bounds__(kThreads) k_sub_step(SubVec<T> s, int flag, ReduceBuf rb)
{
    double c0 = 0, c1 = 0, c2 = 0;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < s.n; i += (int64_t)gridDim.x * kThreads)
    {
        const unsigned char c = s.cls[i];
        const bool is_free = (c & CLS_FREE) != 0;
        if (OP == SUB_OP_INIT)        // drt = xcp - x0 (SubspaceMin.h:133); multipliers start at 0 (:174)
        {
            s.drt[i] = s.xcp[i] - s.x0[i];
            s.lambda[i] = T(0);
            s.mu[i] = T(0);
            s.vecc[i] = T(0);
            s.vecy[i] = T(0);
        }
        if (OP == SUB_OP_ACT_DIR)     // tmp = A'd: (xcp - x0) on the newly active set, 0 elsewhere (BFGSMat.h:504-507)
            s.tmp[i] = (c & CLS_ACT) ? (s.xcp[i] - s.x0[i]) : T(0);
        if (OP == SUB_OP_ADD_G)       // vecc += g on the free set (SubspaceMin.h:157)
            if (is_free) s.vecc[i] += s.g[i];
        if (OP == SUB_OP_NEG_C_FREE)  // tmp = -vecc on the free set: right-hand side of the unconstrained solve (:164)
            s.tmp[i] = is_free ? -s.vecc[i] : T(0);
        if (OP == SUB_OP_CHECK_BOUNDS)  // in_bounds(vecy, vecl, vecu) over the free set (:60-70, :165)
            if (is_free)
            {
                const T l = s.lb[i] - s.x0[i], u = s.ub[i] - s.x0[i];
                if (s.vecy[i] < l || s.vecy[i] > u) c0 += 1;
            }
        if (OP == SUB_OP_CLASSIFY)    // partition of the free set into L / U / P (:194-219)
            if (is_free)
            {
                const T l = s.lb[i] - s.x0[i], u = s.ub[i] - s.x0[i];
                const T y = s.vecy[i];
                unsigned char nc = c & (unsigned char)~(SUB_L | SUB_U | SUB_P);
                if ((y < l) || (y == l && s.lambda[i] >= T(0))) { nc |= SUB_L; s.vecy[i] = l; s.mu[i] = T(0); c0 += 1; }
                else if ((y > u) || (y == u && s.mu[i] >= T(0))) { nc |= SUB_U; s.vecy[i] = u; s.lambda[i] = T(0); c1 += 1; }
                else { nc |= SUB_P; s.lambda[i] = T(0); s.mu[i] = T(0); c2 += 1; }
                s.cls[i] = nc;
            }
        if (OP == SUB_OP_LU_VEC)      // tmp = l on L, u on U, 0 elsewhere (:233-234; the reference skips zeros, same sum)
            s.tmp[i] = (c & SUB_L) ? (s.lb[i] - s.x0[i]) : ((c & SUB_U) ? (s.ub[i] - s.x0[i]) : T(0));
        if (OP == SUB_OP_RHS_P)       // tmp = -(vecc + P'B(L,U) terms) on P (:232-243); flag: tmp2 holds those terms
            s.tmp[i] = (c & SUB_P) ? -(s.vecc[i] + (flag ? s.tmp2[i] : T(0))) : T(0);
        if (OP == SUB_OP_FREE_VEC)    // tmp = vecy on the free set (F'y for W'F y, :250)
            s.tmp[i] = is_free ? s.vecy[i] : T(0);
        if (OP == SUB_OP_MULTIPLIERS) // :252-267 with tmp2 = -(W M W'F y) rows
        {
            if (c & SUB_L) s.lambda[i] = s.tmp2[i] + s.vecc[i] + s.theta * s.vecy[i];
            if (c & SUB_U) s.mu[i] = -(s.tmp2[i] + s.vecc[i] + s.theta * s.vecy[i]);
        }
        if (OP == SUB_OP_CONVERGED)   // L_converged, U_converged, P_converged (:72-108, :270)
        {
            if ((c & CLS_FREE) && (c & SUB_L) && s.lambda[i] < T(0)) c0 += 1;
            if ((c & CLS_FREE) && (c & SUB_U) && s.mu[i] < T(0)) c1 += 1;
            if ((c & CLS_FREE) && (c & SUB_P))
            {
                const T l = s.lb[i] - s.x0[i], u = s.ub[i] - s.x0[i];
                if (s.vecy[i] < l || s.vecy[i] > u) c2 += 1;
            }
        }
        if (OP == SUB_OP_WRITE_DRT)   // subvec_assign(drt, fv_set, .) (+ optional projection) and drt.g (:276-301)
        {
            // flag bit0: project onto [l,u]; bit1: source is the saved unconstrained solution yfb instead of vecy
            if (is_free)
            {
                T y = (flag & 2) ? s.yfb[i] : s.vecy[i];
                if (flag & 1)
                {
                    const T l = s.lb[i] - s.x0[i], u = s.ub[i] - s.x0[i];
                    y = fmin(fmax(y, l), u);
                }
                s.drt[i] = y;
            }
            c0 += (double)(s.drt[i] * s.g[i]);
        }
    }
    if (OP == SUB_OP_CHECK_BOUNDS || OP == SUB_OP_CLASSIFY || OP == SUB_OP_CONVERGED || OP == SUB_OP_WRITE_DRT)
    {
        double acc[3] = {c0, c1, c2};
        grid_reduce_mixed<3>(acc, rb, 0u);
    }
}

}  // namespace lb
