// internal.cuh -- what the translation units of liblbfgs_b200.so share: the context and history objects behind the opaque
// handles of include/lbfgs_b200.h, the error helpers and the status macros.  Not part of the ABI.
#pragma once
#include <cuda_runtime.h>
#include <nccl.h>

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <new>
#include <algorithm>
#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/lbfgs_b200.h"
#include "device_utils.cuh"
#include "objectives.cuh"


using lb::ReduceBuf; using lb::XInbox; using lb::XComm; using lb::kXMaxRanks; using lb::kMailVals;

// ---- context ----
struct lbfgs_b200_ctx
{
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int sm_count = 132;
    int ctas_per_sm_cap = 8;       // streaming grids: at most this many CTAs per SM (tuning knob LBFGS_B200_CTAS_PER_SM, 1..8)
    ReduceBuf rb{};                // device scratch for grid_reduce
    double* h_result = nullptr;    // pinned mirror of rb.result (+ extra slots)
    double* gram_partials = nullptr;  // [sm_count][kMaxM*kGramVals] block partials of k_gram_dots
    double* gram_raw = nullptr;    // [kMaxM*kGramVals] reduced dots
    int* d_flag = nullptr;         // device int flags (accepted, ...)
    int* h_flag = nullptr;         // pinned
    // mapped pinned mailbox: kernels publish host-bound scalars here (see deliver_to_host)
    struct Mail { volatile unsigned long long word; int flag; int pad; double vals[kMailVals]; };
    Mail* h_mail = nullptr;        // host view
    Mail* d_mail = nullptr;        // device view of the same memory
    unsigned long long mail_seq = 0;
    unsigned smem_optin = 0;       // which k_gram_dots instantiations already have their shared-memory opt-in on this device
    ncclComm_t comm = nullptr;
    int rank = 0, nranks = 1;
    // in-kernel exchange over peer memory (lbfgs_b200_comm_p2p_*): replaces the NCCL all-reduce when attached
    XInbox* x_inbox = nullptr;          // this rank's inbox (cudaMalloc, exported through cudaIpc)
    XComm* x_comm = nullptr;            // device copy of the peer table
    void* x_peer[kXMaxRanks] = {};      // cudaIpcOpenMemHandle results (to close)
    bool x_active = false;
    unsigned long long x_epoch = 0;
    int64_t index_offset = 0;      // global index of this rank's element 0
    int64_t n_global = 0;          // global vector length (0 = not declared; needed only by neighbour-coupled objectives)
    double* d_halo = nullptr;      // kHaloDoubles: boundary coordinates of this rank and of its two neighbours (objectives.cuh)
    uint64_t launches = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    // optional per-phase device timing (lbfgs_b200_profile_*): event pairs recorded around each call
    bool profiling = false;
    struct Span { cudaEvent_t a, b; };
    std::vector<Span> spans[3];   // recorded, not yet read
    std::vector<Span> free_spans;
    double prof_ms[3] = {0, 0, 0};
    uint64_t prof_calls[3] = {0, 0, 0};
    double prof_bytes[3] = {0, 0, 0};   // algorithmic bytes (DESIGN.md) of the calls made while profiling
    // device-memory pool (pool_alloc / pool_free below): the reference reallocates its work vectors and the history in every
    // minimize() (reference LBFGS.h:84-90, BFGSMat.h:61-67); on the GPU a cudaMalloc/cudaFree pair costs 0.1-1 ms and a device-wide
    // synchronisation, so blocks released by DeviceVector / hist / box objects are kept and handed out again (exact size match).
    // Everything the library does is ordered on ctx->stream, so a recycled block needs no synchronisation.
    struct Pool
    {
        std::mutex mu;
        std::multimap<size_t, void*> free_blocks;
        std::unordered_map<void*, size_t> sizes;    // every block the pool handed out (live or cached)
        size_t cached = 0, limit = size_t(64) << 30;
        uint64_t hits = 0, misses = 0;
    } pool;
    std::string err;
};

// pool_alloc: `bytes` rounded up to whole 256-byte lines (callers read ragged tails as full packs / bulk copies; the last line
// of a recycled block is cleared like the one of a fresh block usually is).  Returns cudaErrorMemoryAllocation only after the
// cached blocks have been given back to the driver and the allocation failed again.
inline cudaError_t pool_alloc(lbfgs_b200_ctx* ctx, void** out, size_t bytes)
{
    const size_t size = ((bytes ? bytes : 1) + 255) & ~size_t(255);
    std::lock_guard<std::mutex> lock(ctx->pool.mu);
    auto it = ctx->pool.free_blocks.find(size);
    if (it != ctx->pool.free_blocks.end())
    {
        *out = it->second;
        ctx->pool.free_blocks.erase(it);
        ctx->pool.cached -= size;
        ctx->pool.hits++;
        const size_t keep = bytes & ~size_t(255);
        return cudaMemsetAsync(static_cast<char*>(*out) + keep, 0, size - keep, ctx->stream);
    }
    ctx->pool.misses++;
    cudaError_t e = cudaMalloc(out, size);
    if (e == cudaErrorMemoryAllocation && !ctx->pool.free_blocks.empty())
    {
        cudaGetLastError();
        cudaStreamSynchronize(ctx->stream);
        for (auto& kv : ctx->pool.free_blocks) { cudaFree(kv.second); ctx->pool.sizes.erase(kv.second); }
        ctx->pool.free_blocks.clear();
        ctx->pool.cached = 0;
        e = cudaMalloc(out, size);
    }
    if (e == cudaSuccess) ctx->pool.sizes[*out] = size;
    else *out = nullptr;
    return e;
}
inline void pool_free(lbfgs_b200_ctx* ctx, void* p)
{
    if (!p) return;
    if (!ctx) { cudaFree(p); return; }
    std::lock_guard<std::mutex> lock(ctx->pool.mu);
    auto it = ctx->pool.sizes.find(p);
    if (it == ctx->pool.sizes.end()) { cudaFree(p); return; }      // not one of ours
    const size_t size = it->second;
    if (ctx->pool.cached + size > ctx->pool.limit) { ctx->pool.sizes.erase(it); cudaFree(p); return; }
    ctx->pool.free_blocks.emplace(size, p);
    ctx->pool.cached += size;
}
// give every cached block back to the driver (lbfgs_b200_trim, context destruction)
inline void pool_trim(lbfgs_b200_ctx* ctx)
{
    std::lock_guard<std::mutex> lock(ctx->pool.mu);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    for (auto& kv : ctx->pool.free_blocks) { cudaFree(kv.second); ctx->pool.sizes.erase(kv.second); }
    ctx->pool.free_blocks.clear();
    ctx->pool.cached = 0;
}

enum { PH_APPLY_HV = 0, PH_TRIAL = 1, PH_UPDATE = 2 };

// RAII span: records an event pair on the context's stream around a C-ABI call when profiling is on
struct ProfSpan
{
    lbfgs_b200_ctx* ctx;
    int phase;
    lbfgs_b200_ctx::Span sp{nullptr, nullptr};
    ProfSpan(lbfgs_b200_ctx* c, int ph, double alg_bytes = 0.0) : ctx(c), phase(ph)
    {
        if (!ctx || !ctx->profiling) return;
        ctx->prof_bytes[ph] += alg_bytes;
        if (!ctx->free_spans.empty()) { sp = ctx->free_spans.back(); ctx->free_spans.pop_back(); }
        else { cudaEventCreate(&sp.a); cudaEventCreate(&sp.b); }
        cudaEventRecord(sp.a, ctx->stream);
    }
    void stop()
    {
        if (!sp.a) return;
        cudaEventRecord(sp.b, ctx->stream);
        ctx->spans[phase].push_back(sp);
        sp.a = nullptr;
    }
    ~ProfSpan() { stop(); }
};

inline thread_local std::string g_create_err;

inline lbfgs_b200_status fail(lbfgs_b200_ctx* ctx, lbfgs_b200_status st, const char* fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf; else g_create_err = buf;
    return st;
}

#define CU(ctx, call)                                                                                      \
    do {                                                                                                   \
        cudaError_t e__ = (call);                                                                          \
        if (e__ != cudaSuccess)                                                                            \
            return fail(ctx, e__ == cudaErrorMemoryAllocation ? LBFGS_B200_ERR_ALLOC : LBFGS_B200_ERR_CUDA, \
                        "%s failed: %s", #call, cudaGetErrorString(e__));                                  \
    } while (0)

#define NC(ctx, call)                                                                                      \
    do {                                                                                                   \
        ncclResult_t r__ = (call);                                                                         \
        if (r__ != ncclSuccess)                                                                            \
            return fail(ctx, LBFGS_B200_ERR_COMM, "%s failed: %s", #call, ncclGetErrorString(r__));        \
    } while (0)

#define REQUIRE(ctx, cond, ...)                                                                            \
    do { if (!(cond)) return fail(ctx, LBFGS_B200_ERR_INVALID, __VA_ARGS__); } while (0)


// ---- the S/Y ring ----
struct lbfgs_b200_hist
{
    lbfgs_b200_ctx* ctx = nullptr;
    int64_t n = 0, ld = 0;
    int m = 0, M = 0, elem = 8;
    void *S = nullptr, *Y = nullptr, *ys = nullptr, *alpha = nullptr, *theta = nullptr;
    void* SY[2] = {nullptr, nullptr};  // Gram matrices [M][M] by physical slot, double-buffered (see k_gram_combine)
    void* YY[2] = {nullptr, nullptr};
    void* SS[2] = {nullptr, nullptr};
    int gram_cur = 0;  // which buffer is current
    int pending = -1;  // physical slot of the newest pair whose Gram row/column has not been folded in yet
    int head = 0;   // physical slot the next pair is written to
    int ncorr = 0;  // valid pairs (<= m)
    // physical slot of the pair with the given age (0 = newest)
    int slot(int age) const { return ((head - 1 - age) % M + M) % M; }
    template <class T> T* s_col(int phys) const { return static_cast<T*>(S) + (int64_t)phys * ld; }
    template <class T> T* y_col(int phys) const { return static_cast<T*>(Y) + (int64_t)phys * ld; }
};

