// two_loop_gram.cuh -- "vector-free" form of BFGSMat::apply_Hv (reference BFGSMat.h:276-302).
//
// The two-loop recursion only ever combines the vectors {v, s_j, y_j}; every inner product it takes
// (s_j'q in the backward sweep, y_j'r in the forward sweep) is a linear combination of the entries of
//   b_s[j] = s_j'v,  b_y[j] = y_j'v,  SY[i][j] = s_i'y_j,  YY[i][j] = y_i'y_j .
// So the recursion can be carried out on 2c coefficients by one thread (k_gram_solve) once those inner
// products are known, and the result is a single linear combination  res = cv*v + sum_j cy_j*y_j + cs_j*s_j.
// HBM traffic per call: one pass over S,Y,v for the dots + one pass over S,Y,v for the combination
//   = (4c+3) n words   vs  (8c+4) n words for the stage-by-stage recursion (and 2c collectives -> 1).
// SY / YY are kept incrementally: the pair appended last contributes one new row/column, whose 3c dots
// (S'y_new, Y'y_new, Y's_new) are taken in the SAME pass that computes b_s, b_y -- no extra traffic.
// The arithmetic differs from the literal recursion only by rounding (same operations on the same exact
// quantities, re-associated); tests/test_gpu_* bound the difference and oracle/lbfgs_oracle.hpp carries
// a CPU twin (History::apply_Hv_gram) used to study it.
//
// k_gram_dots: tall-skinny [S Y]'[v s_new y_new].  One warp (or `split` warps) per history column pair;
// the three right-hand vectors are staged tile by tile into shared memory with TMA bulk copies
// (cp.async.bulk + mbarrier, 3-stage ring) and shared by all warps of the CTA; the S/Y columns stream from
// HBM straight into registers with 128-bit evict-first loads.  Deterministic: fixed-slot block partials,
// fixed-order final sum, integer ticket only.
#pragma once

#include "device_utils.cuh"
#include "../../include/LBFGSpp/OWLQNCore.h"

namespace lb {

constexpr int kGramTE = 2048;      // tile length in elements (16 KB of fp64 per staged vector)
constexpr int kGramStages = 3;
constexpr int kGramMaxWarps = 24;  // 768 threads, one CTA per SM (85 registers per thread available)
constexpr int kGramMaxThreads = kGramMaxWarps * 32;
constexpr int kMaxM = 64;
constexpr int kGramVals = 6;       // per column pair: s.v, y.v, s.ynew, y.ynew, y.snew, s.snew

template <class T> struct GramDotsArgs
{
    int64_t n, ld;
    const T* v;        // may be nullptr (refresh only)
    const T* S;
    const T* Y;
    int c;             // number of valid pairs
    int new_slot;      // physical slot of the pair whose Gram row/column is still missing, or -1
    int split;         // warps cooperating on one column pair (1, 2, 4 or 8)
    int cols_per_round;  // column pairs processed concurrently by one CTA (warps = cols_per_round * split)
    int use_tma;       // v 16-byte aligned
    unsigned char slots[kMaxM];  // physical slot by age (0 = newest)
    // FORM variant ("update + dots" in one pass, LBFGS.h:159-165): the newest pair is not in the ring yet; it is formed tile by
    // tile as s = fx - fxp, y = v - fgp (v = the new gradient), written to columns `new_slot` of S and Y, and used from shared
    // memory for its own dots.  All five pointers 32-byte aligned.
    const T* fx;
    const T* fxp;
    const T* fgp;
    T* s_out;
    T* y_out;
};

// ---- mbarrier / TMA helpers (sm_90 PTX) -----------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_inval(uint64_t* bar)    // before the barrier's memory is initialised again
{
    asm volatile("mbarrier.inval.shared::cta.b64 [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)   // one arrival, release semantics (the default of mbarrier.arrive)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, unsigned parity)
{
    unsigned ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity)
{
    while (!mbar_try_wait(bar, parity)) {}
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, unsigned bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// Pack of 4 consecutive elements owned by this lane, read from a staged tile.  A lane's pack is 32 bytes, so the
// two 128-bit halves of neighbouring lanes would collide on the same banks; lanes whose (lane>>2) is odd fetch
// their upper half first, which makes both LDS.128 wavefronts conflict-free.
__device__ __forceinline__ Pack<double> lds_pack(const double* p, int lane)
{
    const int flip = (lane >> 2) & 1;
    const double2 a = *reinterpret_cast<const double2*>(p + 2 * flip);
    const double2 b = *reinterpret_cast<const double2*>(p + 2 * (1 - flip));
    Pack<double> r;
    r.v[0] = flip ? b.x : a.x;
    r.v[1] = flip ? b.y : a.y;
    r.v[2] = flip ? a.x : b.x;
    r.v[3] = flip ? a.y : b.y;
    return r;
}
__device__ __forceinline__ Pack<float> lds_pack(const float* p, int)
{
    const float4 a = *reinterpret_cast<const float4*>(p);
    Pack<float> r;
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
    return r;
}

// FORM ("update + dots"): forms the newest pair from (x, xp, g, gp) while it computes [S Y]'[g s_new y_new]  (see GramDotsArgs)
// PG (OWL-QN, FORM only): the right-hand vector is the pseudo-gradient pg(x, g; lam) (LBFGSpp/OWLQNCore.h), formed per element
// from the staged x and g tiles before they become s and y: [S Y]'[pg s_new y_new], the same HBM traffic as FORM
// W (PG only): per-coordinate weights, lam_i = lam * w[i] (owlqn_lam_i).  w is not staged (a fifth staged vector does not fit the
// shared memory of three fp64 stages): each element's weight is a plain streaming load by the thread that forms that element's pg.
template <class T, int ROUNDS, bool FORM, bool PG, bool W = false>
__device__ __forceinline__ void gram_dots_body(unsigned char* gram_smem, const GramDotsArgs<T>& a, T lam, double* partials, unsigned* ticket,
                                               double* result, const XComm* xc, unsigned long long epoch, const T* w = nullptr)
{
    static_assert(FORM || !PG, "the pseudo-gradient is formed from the staged x and g of the FORM variant");
    static_assert(PG || !W, "weights apply to the pseudo-gradient");
    constexpr int NT = FORM ? 4 : 3;                             // staged vectors per tile: v, s_new, y_new (+ xp while forming)
    T* tiles = reinterpret_cast<T*>(gram_smem);                  // [stage][NT][TE]
    __shared__ __align__(8) uint64_t full_bar[kGramStages];
    __shared__ double s_red[kGramMaxWarps][ROUNDS * kGramVals];
    __shared__ unsigned char s_slots[kMaxM];
    __shared__ bool s_last;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nthreads = blockDim.x;
    const bool with_v = a.v != nullptr, with_new = a.new_slot >= 0;
    const T* snew = (with_new && !FORM) ? a.S + (int64_t)a.new_slot * a.ld : nullptr;
    const T* ynew = (with_new && !FORM) ? a.Y + (int64_t)a.new_slot * a.ld : nullptr;
    const int64_t ntiles = (a.n + kGramTE - 1) / kGramTE;
    const int my_col = warp / a.split, my_part = warp % a.split;
    const int part_len = kGramTE / a.split;                        // elements of a tile handled by this warp

    if (tid < kMaxM) s_slots[tid] = a.slots[tid];
    if (tid == 0)
    {
        for (int s = 0; s < kGramStages; s++) mbar_init(&full_bar[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // stage a tile of the right-hand vectors: TMA for full aligned tiles, guarded element loads for the tail
    auto stage_tile = [&](int64_t tile, int stage) {
        T* dst = tiles + (size_t)stage * NT * kGramTE;
        const int64_t e0 = tile * kGramTE;
        const int64_t len = (a.n - e0 < kGramTE) ? (a.n - e0) : kGramTE;
        if (a.use_tma && len == kGramTE)
        {
            if (tid == 0)
            {
                const unsigned bytes = kGramTE * sizeof(T);
                if constexpr (FORM)
                {
                    mbar_expect_tx(&full_bar[stage], bytes * 4);
                    tma_load_1d(dst, a.v + e0, bytes, &full_bar[stage]);                   // g  (stays: v)
                    tma_load_1d(dst + kGramTE, a.fx + e0, bytes, &full_bar[stage]);        // x  -> s
                    tma_load_1d(dst + 2 * kGramTE, a.fgp + e0, bytes, &full_bar[stage]);   // gp -> y
                    tma_load_1d(dst + 3 * kGramTE, a.fxp + e0, bytes, &full_bar[stage]);   // xp
                }
                else
                {
                    mbar_expect_tx(&full_bar[stage], bytes * ((with_v ? 1 : 0) + (with_new ? 2 : 0)));
                    if (with_v) tma_load_1d(dst, a.v + e0, bytes, &full_bar[stage]);
                    if (with_new)
                    {
                        tma_load_1d(dst + kGramTE, snew + e0, bytes, &full_bar[stage]);
                        tma_load_1d(dst + 2 * kGramTE, ynew + e0, bytes, &full_bar[stage]);
                    }
                }
            }
        }
        else
        {
            for (int i = tid; i < kGramTE; i += nthreads)
            {
                const bool ok = i < len;
                if constexpr (FORM)
                {
                    const T gv = ok ? a.v[e0 + i] : T(0);
                    const T sv = ok ? a.fx[e0 + i] - a.fxp[e0 + i] : T(0);
                    const T yv = ok ? gv - a.fgp[e0 + i] : T(0);
                    if constexpr (W) dst[i] = ok ? LBFGSpp::owlqn_pg(a.fx[e0 + i], gv, LBFGSpp::owlqn_lam_i(lam, w[e0 + i])) : T(0);
                    else if constexpr (PG) dst[i] = ok ? LBFGSpp::owlqn_pg(a.fx[e0 + i], gv, lam) : T(0);
                    else dst[i] = gv;
                    dst[kGramTE + i] = sv;
                    dst[2 * kGramTE + i] = yv;
                    if (ok) { a.s_out[e0 + i] = sv; a.y_out[e0 + i] = yv; }
                }
                else
                {
                    dst[i] = (with_v && ok) ? a.v[e0 + i] : T(0);
                    dst[kGramTE + i] = (with_new && ok) ? snew[e0 + i] : T(0);
                    dst[2 * kGramTE + i] = (with_new && ok) ? ynew[e0 + i] : T(0);
                }
            }
        }
    };
    auto tile_is_tma = [&](int64_t tile) { return a.use_tma && (a.n - tile * kGramTE >= kGramTE); };

    T acc[ROUNDS][kGramVals];
#pragma unroll
    for (int r = 0; r < ROUNDS; r++)
#pragma unroll
        for (int k = 0; k < kGramVals; k++) acc[r][k] = T(0);

    // prologue: fill the ring
    int64_t next_tile = blockIdx.x;
    for (int s = 0; s < kGramStages; s++, next_tile += gridDim.x)
        if (next_tile < ntiles) stage_tile(next_tile, s);

    unsigned phase_bits = 0;  // one parity bit per stage
    auto wait_tile = [&](int64_t tile, int st) {
        if (tile_is_tma(tile))
        {
            mbar_wait(&full_bar[st], (phase_bits >> st) & 1u);
            phase_bits ^= (1u << st);
        }
    };
    // FORM: turn a landed TMA tile {g, x, gp, xp} into {g, s = x - xp, y = g - gp} in place and write s, y to the ring columns
    // (tiles staged element by element were formed by stage_tile already)
    auto form_tile = [&](int64_t tile, int st) {
        if (!tile_is_tma(tile)) return;
        T* t0 = tiles + (size_t)st * NT * kGramTE;
        const int64_t e0f = tile * kGramTE;
        for (int i = tid * 4; i < kGramTE; i += nthreads * 4)
        {
            Pack<T> ps, py, pp, pw;
            if constexpr (W) pw = ld_pack<Hint::Stream>(w + e0f + i);
#pragma unroll
            for (int k = 0; k < 4; k++)
            {
                ps.v[k] = t0[kGramTE + i + k] - t0[3 * kGramTE + i + k];
                py.v[k] = t0[i + k] - t0[2 * kGramTE + i + k];
                if constexpr (W) pp.v[k] = LBFGSpp::owlqn_pg(t0[kGramTE + i + k], t0[i + k], LBFGSpp::owlqn_lam_i(lam, pw.v[k]));
                else if constexpr (PG) pp.v[k] = LBFGSpp::owlqn_pg(t0[kGramTE + i + k], t0[i + k], lam);
            }
#pragma unroll
            for (int k = 0; k < 4; k++)
            {
                t0[kGramTE + i + k] = ps.v[k];
                t0[2 * kGramTE + i + k] = py.v[k];
                if constexpr (PG) t0[i + k] = pp.v[k];
            }
            st_pack<Hint::Plain>(a.s_out + e0f + i, ps);
            st_pack<Hint::Plain>(a.y_out + e0f + i, py);
        }
    };
    if constexpr (FORM)
    {
        // the pair of the first tile is formed up front; every later tile is formed by the warps as they finish the dots of
        // the tile before it, so that the column loads of slower warps keep HBM busy meanwhile
        if ((int64_t)blockIdx.x < ntiles) { wait_tile(blockIdx.x, 0); form_tile(blockIdx.x, 0); }
        __syncthreads();
    }
    int stage = 0;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
    {
        if constexpr (!FORM)
        {
            if (tile_is_tma(tile)) wait_tile(tile, stage);
            else __syncthreads();  // element-wise staged tile: make the stores visible
        }
        const T* vt = tiles + (size_t)stage * NT * kGramTE;
        const T* snt = vt + kGramTE;
        const T* ynt = vt + 2 * kGramTE;
        const int64_t e0 = tile * kGramTE;
        const int64_t len = (a.n - e0 < kGramTE) ? (a.n - e0) : kGramTE;
        const bool full_tile = (len == kGramTE);

#pragma unroll
        for (int r = 0; r < ROUNDS; r++)
        {
            const int j = r * a.cols_per_round + my_col;
            if (my_col < a.cols_per_round && j < a.c)
            {
                const int slot = s_slots[j];
                const bool is_new = with_new && slot == a.new_slot;   // this column is already staged in shared memory
                const T* scol = a.S + (int64_t)slot * a.ld + e0;
                const T* ycol = a.Y + (int64_t)slot * a.ld + e0;
                // this warp's part of the tile, 2 packs (8 elements) per lane per step
#pragma unroll 2
                for (int base = my_part * part_len + lane * 4; base < (my_part + 1) * part_len; base += 256)
                {
                    Pack<T> ps[2], py[2];
#pragma unroll
                    for (int u = 0; u < 2; u++)
                    {
                        const int off = base + u * 128;
                        if (is_new)
                        {
                            ps[u] = lds_pack(snt + off, lane);
                            py[u] = lds_pack(ynt + off, lane);
                        }
                        else if (full_tile)
                        {
                            ps[u] = ld_pack<Hint::Stream>(scol + off);
                            py[u] = ld_pack<Hint::Stream>(ycol + off);
                        }
                        else
                        {
#pragma unroll
                            for (int k = 0; k < 4; k++)
                            {
                                const bool ok = off + k < len;
                                ps[u].v[k] = ok ? scol[off + k] : T(0);
                                py[u].v[k] = ok ? ycol[off + k] : T(0);
                            }
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 2; u++)
                    {
                        const int off = base + u * 128;
                        if (with_v)
                        {
                            const Pack<T> pv = lds_pack(vt + off, lane);
#pragma unroll
                            for (int k = 0; k < 4; k++)
                            {
                                acc[r][0] += ps[u].v[k] * pv.v[k];
                                acc[r][1] += py[u].v[k] * pv.v[k];
                            }
                        }
                        if (with_new)
                        {
                            const Pack<T> pyn = lds_pack(ynt + off, lane), psn = lds_pack(snt + off, lane);
#pragma unroll
                            for (int k = 0; k < 4; k++)
                            {
                                acc[r][2] += ps[u].v[k] * pyn.v[k];
                                acc[r][3] += py[u].v[k] * pyn.v[k];
                                acc[r][4] += py[u].v[k] * psn.v[k];
                                acc[r][5] += ps[u].v[k] * psn.v[k];
                            }
                        }
                    }
                }
            }
        }
        if constexpr (FORM)
        {
            const int64_t upcoming = tile + gridDim.x;
            const int nstage = (stage + 1 == kGramStages) ? 0 : stage + 1;
            if (upcoming < ntiles) { wait_tile(upcoming, nstage); form_tile(upcoming, nstage); }
        }
        // the stage was read (and, when forming, rewritten) through the generic proxy: order that before the bulk copy that re-arms it
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();  // everyone is done with this stage's tile (and the next tile's pair is formed)
        if (next_tile < ntiles) stage_tile(next_tile, stage);
        next_tile += gridDim.x;
        stage = (stage + 1 == kGramStages) ? 0 : stage + 1;
    }

    // ---- block reduction: lanes -> warp, then the `split` warps of a column ------------------------------
#pragma unroll
    for (int r = 0; r < ROUNDS; r++)
#pragma unroll
        for (int k = 0; k < kGramVals; k++)
        {
            const double w = warp_sum((double)acc[r][k]);
            if (lane == 0) s_red[warp][r * kGramVals + k] = w;
        }
    __syncthreads();
    const int nvals = a.c * kGramVals;
    for (int idx = tid; idx < nvals; idx += nthreads)
    {
        const int j = idx / kGramVals, k = idx % kGramVals;
        const int r = j / a.cols_per_round, col = j % a.cols_per_round;
        double t = 0.0;
        for (int p = 0; p < a.split; p++) t += s_red[col * a.split + p][r * kGramVals + k];
        partials[(size_t)blockIdx.x * (kMaxM * kGramVals) + idx] = t;
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    for (int idx = tid; idx < nvals; idx += nthreads)
    {
        double t = 0.0;
        for (unsigned b = 0; b < gridDim.x; b++) t += __ldcg(&partials[(size_t)b * (kMaxM * kGramVals) + idx]);
        result[idx] = t;
    }
    if (tid == 0) *ticket = 0u;
    if (xc != nullptr)
    {
        __threadfence();
        xrank_allreduce(result, nvals, xc, epoch);
    }
}

template <class T, int ROUNDS, bool FORM>
__global__ void __launch_bounds__(kGramMaxThreads, 1) k_gram_dots(GramDotsArgs<T> a, double* partials, unsigned* ticket, double* result, const XComm* xc, unsigned long long epoch)
{
    extern __shared__ __align__(128) unsigned char gram_smem[];
    gram_dots_body<T, ROUNDS, FORM, false>(gram_smem, a, T(0), partials, ticket, result, xc, epoch);
}

// OWL-QN: the pair-forming dots with pg(x, g; lam) as the right-hand vector (the FORM variant's staging, see gram_dots_body)
template <class T, int ROUNDS>
__global__ void __launch_bounds__(kGramMaxThreads, 1) k_gram_dots_pg(GramDotsArgs<T> a, T lam, double* partials, unsigned* ticket, double* result,
                                                                     const XComm* xc, unsigned long long epoch)
{
    extern __shared__ __align__(128) unsigned char gram_smem[];
    gram_dots_body<T, ROUNDS, true, true>(gram_smem, a, lam, partials, ticket, result, xc, epoch);
}

// OWL-QN with per-coordinate weights: k_gram_dots_pg with lam_i = lam * w[i] (w on the alignment of x)
template <class T, int ROUNDS>
__global__ void __launch_bounds__(kGramMaxThreads, 1) k_gram_dots_pg_w(GramDotsArgs<T> a, T lam, const T* __restrict__ w, double* partials,
                                                                       unsigned* ticket, double* result)
{
    extern __shared__ __align__(128) unsigned char gram_smem[];
    gram_dots_body<T, ROUNDS, true, true, true>(gram_smem, a, lam, partials, ticket, result, nullptr, 0ull, w);
}

// ---- the O(c^2) recursion on coefficients ---------------------------------------------------------------------
// Runs in shared memory in the prologue of EVERY CTA of the combine kernel (identical arithmetic everywhere, ~2 us,
// no extra launch); CTA 0 also writes the folded Gram matrices and the alphas back for the next call.
template <class T> struct GramSolveArgs
{
    int c, M, new_slot, with_v;
    T a;                     // scale of v
    const double* raw;       // [c][5] reduced dots (after the all-reduce)
    const T* SY_in;          // [M][M] by physical slot: SY[i*M+j] = s_i'y_j
    const T* YY_in;          // [M][M]
    const T* SS_in;          // [M][M]  s_i's_j (not used by the recursion; kept for the L-BFGS-B middle matrix)
    T* SY_out;               // folded matrices (a second buffer: other CTAs may still be reading *_in)
    T* YY_out;
    T* SS_out;
    const T* ys;             // [M]
    T* alpha;                // [M]
    const T* theta;
    unsigned char slots[kMaxM];
};

// smem layout (T units): SY[c*c] | YY[c*c] | coef[2c+1] | alpha[c] | a*S'v[c] | a*Y'v[c] | ys[c] | theta ; everything indexed by AGE (0 = newest).
__host__ __device__ inline size_t gram_solve_smem_elems(int c) { return (size_t)2 * c * c + 6 * c + 2; }

// All global reads go through L2 (__ldcg): inside the persistent solve these scalars are rewritten by another CTA between rounds.
// GLOBAL = false: the operands (raw, Gram matrices, ys, theta) live in this CTA's shared memory (the small-batch solve) and are read
// with ordinary loads.
template <class T, bool GLOBAL = true>
__device__ void gram_solve_in_smem(const GramSolveArgs<T>& g, T* sm, bool writer)
{
    auto ld = [](const auto* p) { if constexpr (GLOBAL) return __ldcg(p); else return *p; };
    const int c = g.c, M = g.M, tid = threadIdx.x, nt = blockDim.x;
    T* sSY = sm;
    T* sYY = sm + c * c;
    T* coef = sm + 2 * c * c;
    T* al = coef + 2 * c + 1;
    // the pending pair is always the newest one: age 0
    for (int idx = tid; idx < c * c; idx += nt)
    {
        const int i = idx / c, j = idx % c;
        const int pi = g.slots[i], pj = g.slots[j];
        T sy = ld(g.SY_in + pi * M + pj), yy = ld(g.YY_in + pi * M + pj);
        if (g.new_slot >= 0)
        {
            if (j == 0) { sy = (T)ld(g.raw + i * kGramVals + 2); yy = (T)ld(g.raw + i * kGramVals + 3); }       // s_i'y_new, y_i'y_new
            else if (i == 0) { sy = (T)ld(g.raw + j * kGramVals + 4); yy = (T)ld(g.raw + j * kGramVals + 3); }  // s_new'y_j, y_new'y_j
        }
        sSY[idx] = sy;
        sYY[idx] = yy;
        if (writer && g.new_slot >= 0)
        {
            T ss = ld(g.SS_in + pi * M + pj);
            if (j == 0) ss = (T)ld(g.raw + i * kGramVals + 5);        // s_i's_new
            else if (i == 0) ss = (T)ld(g.raw + j * kGramVals + 5);   // s_new's_j
            g.SY_out[pi * M + pj] = sy;
            g.YY_out[pi * M + pj] = yy;
            g.SS_out[pi * M + pj] = ss;
        }
    }
    // right-hand sides, ys and theta by age next to the matrices: fetched by the LAST threads of the block, so that their L2 round trip
    // overlaps the matrices' (the first threads') instead of following it
    T* b0 = al + c;        // a * s_i'v
    T* b1 = b0 + c;        // a * y_i'v
    T* ysv = b1 + c;
    T* th = ysv + c;       // theta
    if (g.with_v)
    {
        for (int i = nt - 1 - tid; i < c; i += nt)
        {
            b0[i] = g.a * (T)ld(g.raw + i * kGramVals + 0);
            b1[i] = g.a * (T)ld(g.raw + i * kGramVals + 1);
            ysv[i] = ld(g.ys + g.slots[i]);
        }
        if (tid == nt - 1) th[0] = ld(g.theta);
    }
    __syncthreads();
    if (tid < 32 && g.with_v)
    {
        // One warp runs the two triangular sweeps COLUMN by column: lane t owns the entries t and t + 32 of the running right-hand
        // side; a step is { multiply the pivot entry by 1/ys, broadcast it (one shuffle), one multiply-subtract per lane } -- no
        // reduction tree, no division and no shared-memory round trip on the critical path (~50 cycles per step instead of ~400
        // for the row-oriented sweep with a shuffle tree and a division per step; measured 16 us -> ~1 us at c = 20).
        const int lane = tid;
        const T theta = th[0];
        const int tA = lane, tB = lane + 32;
        const bool hasA = tA < c, hasB = tB < c;
        const T rA = hasA ? T(1) / ysv[tA] : T(0), rB = hasB ? T(1) / ysv[tB] : T(0);
        // backward sweep (BFGSMat.h:285-290): alpha_i = s_i'q / ys_i with q = a*v - sum_{newer t} alpha_t y_t
        //   acc_t = a*s_t'v - sum_{i < t} alpha_i s_t'y_i, subtracted in the order i = 0, 1, ... (the order q is built in)
        T accA = hasA ? b0[tA] : T(0), accB = hasB ? b0[tB] : T(0);
        T alA = T(0), alB = T(0);
        for (int i = 0; i < c; i++)
        {
            const bool hi = i >= 32;
            const T mine = hi ? accB * rB : accA * rA;
            const T ai = __shfl_sync(0xffffffffu, mine, i & 31);
            if (lane == (i & 31)) { if (hi) alB = ai; else alA = ai; }
            if (hasA && tA > i) accA -= ai * sSY[tA * c + i];
            if (hasB && tB > i) accB -= ai * sSY[tB * c + i];
        }
        if (hasA) al[tA] = alA;
        if (hasB) al[tB] = alB;
        __syncwarp();
        // forward sweep (BFGSMat.h:293-301): r = q/theta + sum_{older t} (alpha_t - beta_t) s_t ; beta_i = y_i'r / ys_i
        //   w_i = (a*y_i'v - sum_t alpha_t y_i'y_t) / theta : independent of the sweep, every lane does its own (Y'Y is symmetric:
        //   lane i reads column i, consecutive addresses across lanes)
        T wA = T(0), wB = T(0);
        if (hasA) { T z = T(0); for (int t = 0; t < c; t++) z += al[t] * sYY[t * c + tA]; wA = (b1[tA] - z) / theta; }
        if (hasB) { T z = T(0); for (int t = 0; t < c; t++) z += al[t] * sYY[t * c + tB]; wB = (b1[tB] - z) / theta; }
        //   then w_t += cs_i * s_i'y_t for the older i = c-1 .. t+1, cs_i = alpha_i - w_i / ys_i
        T* cs = coef + 1 + c;
        T csA = T(0), csB = T(0);
        for (int i = c - 1; i >= 0; i--)
        {
            const bool hi = i >= 32;
            const T mine = hi ? alB - wB * rB : alA - wA * rA;
            const T ci = __shfl_sync(0xffffffffu, mine, i & 31);
            if (lane == (i & 31)) { if (hi) csB = ci; else csA = ci; }
            if (hasA && tA < i) wA += ci * sSY[i * c + tA];
            if (hasB && tB < i) wB += ci * sSY[i * c + tB];
        }
        if (hasA) { cs[tA] = csA; coef[1 + tA] = -(alA / theta); if (writer) g.alpha[g.slots[tA]] = alA; }
        if (hasB) { cs[tB] = csB; coef[1 + tB] = -(alB / theta); if (writer) g.alpha[g.slots[tB]] = alB; }
        if (lane == 0) coef[0] = g.a / theta;
    }
    __syncthreads();
}

// fold only (pairs appended back to back without an apply_Hv in between)
template <class T> __global__ void k_gram_fold(GramSolveArgs<T> g)
{
    extern __shared__ __align__(16) unsigned char fold_smem[];
    gram_solve_in_smem<T>(g, reinterpret_cast<T*>(fold_smem), true);
}

// ---- res = cv*v + sum_j cy_j*y_j + cs_j*s_j  (+ v.res), preceded by the coefficient recursion -----------------
template <class T> struct GramCombineArgs
{
    int64_t n, ld;
    const T* v;
    const T* S;
    const T* Y;
    T* res;
    int want_dot;
    GramSolveArgs<T> solve;
};

template <class T, bool VEC>
__global__ void __launch_bounds__(kThreads) k_gram_combine(GramCombineArgs<T> a, ReduceBuf rb)
{
    extern __shared__ __align__(16) unsigned char comb_smem[];
    T* sm = reinterpret_cast<T*>(comb_smem);
    const int c = a.solve.c;
    gram_solve_in_smem<T>(a.solve, sm, blockIdx.x == 0);
    const T* s_coef = sm + 2 * c * c;
    __shared__ const T* s_ycol[kMaxM];
    __shared__ const T* s_scol[kMaxM];
    for (int j = threadIdx.x; j < c; j += kThreads)
    {
        s_ycol[j] = a.Y + (int64_t)a.solve.slots[j] * a.ld;
        s_scol[j] = a.S + (int64_t)a.solve.slots[j] * a.ld;
    }
    __syncthreads();
    const T cv = s_coef[0];
    T dot = T(0);
    const int64_t packs = (a.n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (a.n - i0 >= 4) ? 4 : int(a.n - i0);
        const Pack<T> pv = load4<T, Hint::Stream, VEC>(a.v, i0, cnt);
        T r[4];
#pragma unroll
        for (int k = 0; k < 4; k++) r[k] = cv * pv.v[k];
        // y terms newest -> oldest, then s terms oldest -> newest (the order the recursion would add them)
#pragma unroll 4
        for (int j = 0; j < c; j++)
        {
            const Pack<T> py = load4<T, Hint::Stream, VEC>(s_ycol[j], i0, cnt);
            const T cy = s_coef[1 + j];
#pragma unroll
            for (int k = 0; k < 4; k++) r[k] += cy * py.v[k];
        }
#pragma unroll 4
        for (int j = c - 1; j >= 0; j--)
        {
            const Pack<T> ps = load4<T, Hint::Stream, VEC>(s_scol[j], i0, cnt);
            const T cs = s_coef[1 + c + j];
#pragma unroll
            for (int k = 0; k < 4; k++) r[k] += cs * ps.v[k];
        }
        Pack<T> out;
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            out.v[k] = r[k];
            dot += (k < cnt) ? pv.v[k] * r[k] : T(0);
        }
        store4<T, Hint::Plain, VEC>(a.res, i0, cnt, out);
    }
    if (a.want_dot)
    {
        double dacc[1] = {(double)dot};
        grid_reduce<1>(dacc, rb);
    }
}

// OWL-QN: k_gram_combine with v = pg(x, g; lam) formed per element from x and g = a.v, res = the orthant-constrained combination
// (owlqn_constrain against pg: d = -H pg projected, with a = -1) and the dot pg.res over the constrained res
template <class T, bool VEC>
__global__ void __launch_bounds__(kThreads) k_gram_combine_pg(GramCombineArgs<T> a, const T* x, T lam, ReduceBuf rb)
{
    extern __shared__ __align__(16) unsigned char comb_smem[];
    T* sm = reinterpret_cast<T*>(comb_smem);
    const int c = a.solve.c;
    gram_solve_in_smem<T>(a.solve, sm, blockIdx.x == 0);
    const T* s_coef = sm + 2 * c * c;
    __shared__ const T* s_ycol[kMaxM];
    __shared__ const T* s_scol[kMaxM];
    for (int j = threadIdx.x; j < c; j += kThreads)
    {
        s_ycol[j] = a.Y + (int64_t)a.solve.slots[j] * a.ld;
        s_scol[j] = a.S + (int64_t)a.solve.slots[j] * a.ld;
    }
    __syncthreads();
    const T cv = s_coef[0];
    T dot = T(0);
    const int64_t packs = (a.n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (a.n - i0 >= 4) ? 4 : int(a.n - i0);
        const Pack<T> px = load4<T, Hint::Stream, VEC>(x, i0, cnt);
        Pack<T> pv = load4<T, Hint::Stream, VEC>(a.v, i0, cnt);
#pragma unroll
        for (int k = 0; k < 4; k++) pv.v[k] = LBFGSpp::owlqn_pg(px.v[k], pv.v[k], lam);
        T r[4];
#pragma unroll
        for (int k = 0; k < 4; k++) r[k] = cv * pv.v[k];
        // y terms newest -> oldest, then s terms oldest -> newest (the order the recursion would add them)
#pragma unroll 4
        for (int j = 0; j < c; j++)
        {
            const Pack<T> py = load4<T, Hint::Stream, VEC>(s_ycol[j], i0, cnt);
            const T cy = s_coef[1 + j];
#pragma unroll
            for (int k = 0; k < 4; k++) r[k] += cy * py.v[k];
        }
#pragma unroll 4
        for (int j = c - 1; j >= 0; j--)
        {
            const Pack<T> ps = load4<T, Hint::Stream, VEC>(s_scol[j], i0, cnt);
            const T cs = s_coef[1 + c + j];
#pragma unroll
            for (int k = 0; k < 4; k++) r[k] += cs * ps.v[k];
        }
        Pack<T> out;
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            out.v[k] = LBFGSpp::owlqn_constrain(r[k], pv.v[k]);
            dot += (k < cnt) ? pv.v[k] * out.v[k] : T(0);
        }
        store4<T, Hint::Plain, VEC>(a.res, i0, cnt, out);
    }
    if (a.want_dot)
    {
        double dacc[1] = {(double)dot};
        grid_reduce<1>(dacc, rb);
    }
}

// OWL-QN with per-coordinate weights: k_gram_combine_pg with lam_i = lam * w[i] (owlqn_lam_i) in pg and in the constraint
// (owlqn_constrain_w), w read on the packs of x.  A kernel of its own: a shared body moved the registers of k_gram_combine_pg.
template <class T, bool VEC>
__global__ void __launch_bounds__(kThreads) k_gram_combine_pg_w(GramCombineArgs<T> a, const T* x, T lam, const T* w, ReduceBuf rb)
{
    extern __shared__ __align__(16) unsigned char comb_smem[];
    T* sm = reinterpret_cast<T*>(comb_smem);
    const int c = a.solve.c;
    gram_solve_in_smem<T>(a.solve, sm, blockIdx.x == 0);
    const T* s_coef = sm + 2 * c * c;
    __shared__ const T* s_ycol[kMaxM];
    __shared__ const T* s_scol[kMaxM];
    for (int j = threadIdx.x; j < c; j += kThreads)
    {
        s_ycol[j] = a.Y + (int64_t)a.solve.slots[j] * a.ld;
        s_scol[j] = a.S + (int64_t)a.solve.slots[j] * a.ld;
    }
    __syncthreads();
    const T cv = s_coef[0];
    T dot = T(0);
    const int64_t packs = (a.n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (a.n - i0 >= 4) ? 4 : int(a.n - i0);
        const Pack<T> px = load4<T, Hint::Stream, VEC>(x, i0, cnt);
        Pack<T> pv = load4<T, Hint::Stream, VEC>(a.v, i0, cnt);
        const Pack<T> pw = load4<T, Hint::Stream, VEC>(w, i0, cnt);
        T lw[4];
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            lw[k] = LBFGSpp::owlqn_lam_i(lam, pw.v[k]);
            pv.v[k] = LBFGSpp::owlqn_pg(px.v[k], pv.v[k], lw[k]);
        }
        T r[4];
#pragma unroll
        for (int k = 0; k < 4; k++) r[k] = cv * pv.v[k];
        // y terms newest -> oldest, then s terms oldest -> newest (the order the recursion would add them)
#pragma unroll 4
        for (int j = 0; j < c; j++)
        {
            const Pack<T> py = load4<T, Hint::Stream, VEC>(s_ycol[j], i0, cnt);
            const T cy = s_coef[1 + j];
#pragma unroll
            for (int k = 0; k < 4; k++) r[k] += cy * py.v[k];
        }
#pragma unroll 4
        for (int j = c - 1; j >= 0; j--)
        {
            const Pack<T> ps = load4<T, Hint::Stream, VEC>(s_scol[j], i0, cnt);
            const T cs = s_coef[1 + c + j];
#pragma unroll
            for (int k = 0; k < 4; k++) r[k] += cs * ps.v[k];
        }
        Pack<T> out;
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            out.v[k] = LBFGSpp::owlqn_constrain_w(r[k], pv.v[k], lw[k]);
            dot += (k < cnt) ? pv.v[k] * out.v[k] : T(0);
        }
        store4<T, Hint::Plain, VEC>(a.res, i0, cnt, out);
    }
    if (a.want_dot)
    {
        double dacc[1] = {(double)dot};
        grid_reduce<1>(dacc, rb);
    }
}

}  // namespace lb
