// device_utils.cuh -- wide global-memory accessors and the deterministic grid reduction used by every
// kernel of liblbfgs_b200.so (sm_90a only).
//
// Memory model of the path: all operands are long contiguous fp64/fp32 vectors streamed once per kernel,
// so the kernels are HBM-bound.  Rules applied here:
//   * one pack = 4 elements: two 128-bit accesses for fp64 (the widest global access on sm_90), one for fp32;
//   * history columns are read with L1::no_allocate + L2::evict_first (touched once per pass), the running
//     vector q/r with L2::evict_last so that it can survive in the 50 MB L2 between consecutive stages;
//   * grids are a multiple of the SM count; every thread keeps several independent packs in flight.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace lb {

constexpr int kThreads = 256;        // threads per CTA for all streaming kernels
constexpr int kMaxRed = 8;           // max simultaneous reductions per kernel launch
constexpr int kMaxBlocks = 132 * 8;  // H100 SXM: 132 SMs; upper bound on any reducing grid (partials buffer size)

// ----------------------------------------------------------------------------- packs of 4 elements
template <class T> struct Pack { T v[4]; };

enum class Hint { Stream, Keep, Plain };

// sm_90 has neither 256-bit global accesses nor the .L2::evict_* qualifiers of ld/st: a pack of 4 doubles is two 128-bit
// accesses to adjacent 16-byte halves, and the L2 eviction priority travels as a cache policy (createpolicy + .L2::cache_hint)
template <Hint H> __device__ __forceinline__ uint64_t l2_policy()
{
    uint64_t pol;
    if (H == Hint::Stream) asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    else asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
#define LB_LD2H(p, a, b, pol) asm("ld.global.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;" : "=d"(a), "=d"(b) : "l"(p), "l"(pol))
#define LB_ST2H(p, a, b, pol) asm volatile("st.global.L1::no_allocate.L2::cache_hint.v2.f64 [%0], {%1,%2}, %3;" :: "l"(p), "d"(a), "d"(b), "l"(pol) : "memory")
template <Hint H> __device__ __forceinline__ Pack<double> ld_pack(const double* p)
{
    Pack<double> r;
    if (H == Hint::Plain)
    {
        asm("ld.global.v2.f64 {%0,%1}, [%2];" : "=d"(r.v[0]), "=d"(r.v[1]) : "l"(p));
        asm("ld.global.v2.f64 {%0,%1}, [%2];" : "=d"(r.v[2]), "=d"(r.v[3]) : "l"(p + 2));
    }
    else
    {
        const uint64_t pol = l2_policy<H>();
        LB_LD2H(p, r.v[0], r.v[1], pol);
        LB_LD2H(p + 2, r.v[2], r.v[3], pol);
    }
    return r;
}
template <Hint H> __device__ __forceinline__ void st_pack(double* p, const Pack<double>& r)
{
    if (H == Hint::Plain)
    {
        asm volatile("st.global.v2.f64 [%0], {%1,%2};" :: "l"(p), "d"(r.v[0]), "d"(r.v[1]) : "memory");
        asm volatile("st.global.v2.f64 [%0], {%1,%2};" :: "l"(p + 2), "d"(r.v[2]), "d"(r.v[3]) : "memory");
    }
    else
    {
        const uint64_t pol = l2_policy<H>();
        LB_ST2H(p, r.v[0], r.v[1], pol);
        LB_ST2H(p + 2, r.v[2], r.v[3], pol);
    }
}
#undef LB_LD2H
#undef LB_ST2H
// fp32: 128-bit packs (no L2 eviction hint)
template <Hint H> __device__ __forceinline__ Pack<float> ld_pack(const float* p)
{
    Pack<float> r;
    if (H == Hint::Plain)
        asm("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(r.v[0]), "=f"(r.v[1]), "=f"(r.v[2]), "=f"(r.v[3]) : "l"(p));
    else
        asm("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(r.v[0]), "=f"(r.v[1]), "=f"(r.v[2]), "=f"(r.v[3]) : "l"(p));
    return r;
}
template <Hint H> __device__ __forceinline__ void st_pack(float* p, const Pack<float>& r)
{
    asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "f"(r.v[0]), "f"(r.v[1]), "f"(r.v[2]), "f"(r.v[3]) : "memory");
}

template <class T> __host__ __device__ __forceinline__ bool pack_aligned(const void* p)
{
    return (reinterpret_cast<uintptr_t>(p) & (sizeof(T) * 4 - 1)) == 0;
}

// Guarded pack access: full aligned packs take the wide path, the ragged tail (and misaligned callers)
// go element by element.  `cnt` = number of valid elements (1..4); missing lanes read as 0.
template <class T, Hint H, bool VEC> __device__ __forceinline__ Pack<T> load4(const T* base, int64_t i0, int cnt)
{
    if (VEC && cnt == 4) return ld_pack<H>(base + i0);
    Pack<T> r;
#pragma unroll
    for (int k = 0; k < 4; k++) r.v[k] = (k < cnt) ? base[i0 + k] : T(0);
    return r;
}
template <class T, Hint H, bool VEC> __device__ __forceinline__ void store4(T* base, int64_t i0, int cnt, const Pack<T>& r)
{
    if (VEC && cnt == 4) { st_pack<H>(base + i0, r); return; }
#pragma unroll
    for (int k = 0; k < 4; k++)
        if (k < cnt) base[i0 + k] = r.v[k];
}

// ----------------------------------------------------------------------------- deterministic reduction
// Every reducing kernel ends with grid_reduce<NV>():
//   thread partials -> warp shuffle tree -> smem across warps -> one slot per (block, value) in `partials`
//   -> integer ticket -> the LAST block to arrive sums the slots in a fixed order and writes `result[k]`.
// The only atomic is the integer ticket, so the floating-point result depends on (n, grid) alone and is
// reproducible run to run.  Accumulation across warps/blocks is in double also for fp32 inputs.
// ---- cross-GPU exchange fused into the tail of a reducing kernel ------------------------------------------------
// n-sharded mode: after the last CTA has the local sums it pushes them straight into every peer's inbox over NVLink
// (peer-mapped memory, cudaIpc), raises a per-source flag carrying the collective's epoch, waits for all sources'
// flags in its own inbox and adds the contributions in RANK ORDER -- every rank ends with the same bits and the kernel
// that follows can consume result[] without a separate all-reduce launch.  Inboxes form a ring of kXRing epochs.
constexpr int kXMaxRanks = 8;
constexpr int kXRing = 4;
constexpr int kXMaxVals = 4608;  // per exchange: >= kMaxM * (values per column pair of k_gram_dots), and >= B * (6 m + 4) for a batch of B
                                 // problems whose sums travel in ONE exchange per round (persist.cuh): 64 * (60 + 4) = 4096
constexpr int kMailVals = 384;   // host mailbox slots

struct XInbox
{
    double vals[kXRing][kXMaxRanks][kXMaxVals];
    unsigned long long flag[kXRing][kXMaxRanks];
    // the persistent solve's exchange: every double travels as two self-validating 8-byte words {32 data bits, 32-bit epoch tag}
    // (single-copy atomic stores): no fence, no flag, one NVLink crossing (see ll_push / ll_pull)
    unsigned long long ll[kXRing][kXMaxRanks][kXMaxVals][2];
};

__device__ __forceinline__ void ll_push(unsigned long long* dst2, double v, unsigned tag)
{
    const unsigned long long bits = (unsigned long long)__double_as_longlong(v);
    const unsigned long long w0 = (bits & 0xffffffffull) | ((unsigned long long)tag << 32);
    const unsigned long long w1 = (bits >> 32) | ((unsigned long long)tag << 32);
    asm volatile("st.volatile.global.v2.u64 [%0], {%1, %2};" :: "l"(dst2), "l"(w0), "l"(w1) : "memory");
}
// spins until both words carry `tag`; false when `give_up` says so (watchdog)
template <class GiveUp> __device__ __forceinline__ bool ll_pull(const unsigned long long* src2, unsigned tag, double& v, GiveUp give_up)
{
    for (;;)
    {
        unsigned long long w0, w1;
        asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(src2) : "memory");
        if ((unsigned)(w0 >> 32) == tag && (unsigned)(w1 >> 32) == tag)
        {
            v = __longlong_as_double((long long)((w0 & 0xffffffffull) | (w1 << 32)));
            return true;
        }
        if (give_up()) return false;
    }
}

struct XComm
{
    XInbox* inbox[kXMaxRanks];   // inbox[r] = rank r's inbox as mapped into THIS process (inbox[rank] is local)
    int rank, nranks;
};

struct ReduceBuf
{
    double* partials;    // [kMaxBlocks][kMaxRed]
    unsigned* ticket;    // zero between launches (the last block resets it)
    double* result;      // [kMaxRed] device result slots of this launch
    const XComm* xc;     // nullptr on a single GPU (or when NCCL does the all-reduce)
    unsigned long long epoch;  // sequence number of this launch's exchange (identical on all ranks)
    // host delivery: when mail_seq != 0 the last CTA also copies result[] into a mapped pinned-host mailbox and then
    // publishes mail_seq there; the host spins on the sequence word instead of paying memcpy + stream synchronise
    double* mail_vals;
    unsigned long long* mail_word;
    unsigned long long mail_seq;
    const int* mail_flag_src;  // optional device int forwarded into the mailbox (e.g. the curvature-gate flag)
    int* mail_flag_dst;
};

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v)
{
    asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p)
{
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ double ld_volatile_f64(const double* p)
{
    double v;
    asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}

// Called by ALL threads of the last CTA once result[0..nv) holds the local sums.  On return result[] holds the
// rank-ordered global sums (visible to the kernels that follow on this stream).
__device__ __forceinline__ void xrank_allreduce(double* result, int nv, const XComm* xc, unsigned long long epoch)
{
    const int tid = threadIdx.x, nt = blockDim.x;
    const int slot = (int)(epoch % kXRing), me = xc->rank, R = xc->nranks;
    __syncthreads();
    for (int i = tid; i < nv * R; i += nt)
    {
        const int dst = i / nv, k = i % nv;
        xc->inbox[dst]->vals[slot][me][k] = result[k];
    }
    __threadfence_system();
    __syncthreads();
    if (tid < R) st_release_sys(&xc->inbox[tid]->flag[slot][me], epoch);
    if (tid < R)
    {
        const unsigned long long* f = &xc->inbox[me]->flag[slot][tid];
        while (ld_acquire_sys(f) != epoch) {}
    }
    __syncthreads();
    for (int k = tid; k < nv; k += nt)
    {
        double t = 0.0;
        for (int r = 0; r < R; r++) t += ld_volatile_f64(&xc->inbox[me]->vals[slot][r][k]);
        result[k] = t;
    }
    __threadfence();
    __syncthreads();
}

__device__ __forceinline__ void deliver_to_host(const ReduceBuf& rb, int nv)
{
    if (rb.mail_seq == 0ull) return;
    for (int k = threadIdx.x; k < nv; k += blockDim.x) rb.mail_vals[k] = rb.result[k];
    if (threadIdx.x == 0 && rb.mail_flag_src) *rb.mail_flag_dst = *rb.mail_flag_src;
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) st_release_sys(rb.mail_word, rb.mail_seq);
}


__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Returns true in the threads of the last block once result[] is final (so a caller can append a tiny
// "finalizer" that consumes the reduced values in the same launch); false elsewhere.
template <int NV> __device__ __forceinline__ bool grid_reduce(const double (&acc)[NV], const ReduceBuf& rb)
{
    __shared__ double s_part[NV][kThreads / 32];
    __shared__ bool s_last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; k++)
    {
        const double w = warp_sum(acc[k]);
        if (lane == 0) s_part[k][warp] = w;
    }
    __syncthreads();
    if (threadIdx.x < NV)
    {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < kThreads / 32; w++) t += s_part[threadIdx.x][w];
        rb.partials[blockIdx.x * kMaxRed + threadIdx.x] = t;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0)
    {
        const unsigned t = atomicAdd(rb.ticket, 1u);
        s_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return false;
    __threadfence();
    // last block: fixed-order sum over blocks: thread t takes blocks t, t+256, ...; then the block tree
    double mine[NV];
#pragma unroll
    for (int k = 0; k < NV; k++) mine[k] = 0.0;
    for (unsigned b = threadIdx.x; b < gridDim.x; b += kThreads)
#pragma unroll
        for (int k = 0; k < NV; k++) mine[k] += __ldcg(&rb.partials[b * kMaxRed + k]);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < NV; k++)
    {
        const double w = warp_sum(mine[k]);
        if (lane == 0) s_part[k][warp] = w;
    }
    __syncthreads();
    if (threadIdx.x < NV)
    {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < kThreads / 32; w++) t += s_part[threadIdx.x][w];
        rb.result[threadIdx.x] = t;
    }
    if (threadIdx.x == 0) *rb.ticket = 0u;
    __threadfence();
    __syncthreads();
    if (rb.xc != nullptr) xrank_allreduce(rb.result, NV, rb.xc, rb.epoch);
    deliver_to_host(rb, NV);
    return true;
}

}  // namespace lb
