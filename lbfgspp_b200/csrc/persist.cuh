// persist.cuh -- the device-resident L-BFGS solve: LBFGSSolver::minimize() (reference LBFGS.h:78-173) for built-in objectives as
// ONE persistent cooperative kernel launch, for one problem or for a batch of B independent problems (BASELINE config 5).
// Included by persist_f64.cu / persist_f32.cu.  The objective comes from objectives.cuh: built from the same geometry record as the
// host-driven loop's, checked by the same rules before the launch, and every pass evaluates it with the same pack steps.
//
// The kernel is a "phase machine".  One CTA per SM (768 threads), all co-resident (cooperative launch).  Work proceeds in ROUNDS;
// in a round every problem that is still running executes the ONE streaming pass its state asks for:
//     FIRST          g = grad f(x0), d = -g (stored: HALO only)  ; {f, g.g, x.x}                            LBFGS.h:91-108
//     TRIAL          x = xp + step*d, g = grad f(x)              ; {f, g.d, g.g, x.x}                       LineSearch*.h trial, LBFGS.h:130,137
//     DOTS_FORM      s = x - xp, y = g - gp -> free ring slot    ; [S Y]'[g s y] (6 dots per column pair)   LBFGS.h:159-162, BFGSMat.h:85-92 + apply_Hv pass 1
//     DOTS_PLAIN     (pair rejected by the curvature gate)       ; [S Y]'g over the old history
//                    (both in p_dots: forming warps prepare each staged element once -- g, and the new pair -- the column warps read it)
//     COMBINE        coefficient recursion (every CTA, shared memory) ; d = cv*g + sum cy_j y_j + cs_j s_j ; {g.d}   BFGSMat.h:283-301 in Gram form
//     COMBINE_TRIAL  COMBINE + the first trial of the next line search in the same pass: the reference restarts every search
//                    at step = 1 (LBFGS.h:168), so x1 = x + d, g1 = grad f(x1) ; {g.d, f1, g1.d, g1.g1, x1.x1}
//     RESTORE        x = xp, g = gp (a search that never improved on its start point; LineSearchMoreThuente.h:602-614)
//     MATERIALIZE    x = xp + step*d (or x = xp, or x as stored), g = grad f(x): writes the point a finished problem stopped at
// Trials on the ray.  For objectives without neighbour coupling g = grad f(x) is a per-element function of x, and every trial point
// is x = xp + step*d, so a trial stores nothing: its point is IMPLIED by {step, at_start} (PT_START: the start point xp).
// The pass after the search -- DOTS_FORM, which reads the point anyway -- rebuilds the accepted point from xp, d with the trial's own
// arithmetic, bit for bit, writes x, and forms the pair from it.  Nor is g itself stored between passes: the passes that need the
// gradient of a stored point (gp = grad f(xp) in DOTS_FORM, g = grad f(x) in DOTS_PLAIN and COMBINE) evaluate it from that point
// with the same arithmetic, bit for bit the g a pass would have stored; that spares DOTS_FORM the read of gp and the write of g and
// COMBINE the read of g.  Only MATERIALIZE writes g: a problem that stops takes one MATERIALIZE round for the point it stopped at --
// on the ray, its search's start point, or the point in x (it converged at x0, or arming the next search failed).  The direction of
// the first search, d = -grad f(x0), is not stored either: FIRST writes x0 to its point row only, and while PRound::d_implied is
// set (k == 1: until the first combination pass writes d) TRIAL, MATERIALIZE on the ray and the first DOTS_FORM evaluate d = T(-1) *
// grad f(xp) from xp, bit for bit the d FIRST would have stored, instead of reading it.  The kept best trial of a search is its
// step, so there is no x_lo/g_lo and no RESTORE pass.
// History of iterates.  For the same objectives a pair is a function of its two endpoints (s = x - xp, y = grad f(x) - grad f(xp)),
// and consecutive accepted pairs share one: the ring holds iterates (PState::pts), x and xp are rows of it, and the dots and
// combination passes stage the c + 1 endpoints of c chained pairs instead of 2c columns and rebuild each pair where they read it,
// with the arithmetic that formed it (point_plan).  The flat x, g hold only the caller's start point and the result.
// Neighbour-coupled objectives (kHalo) store every trial's x, g and keep the best one by pointer swap with x_lo/g_lo, as the
// reference's search does (LineSearchMoreThuente.h:534,553), restore the start point with RESTORE, and keep an S|Y ring.
// Every CTA owns the same contiguous chunk (granularity: the block length of the tiled history) of EVERY vector in EVERY pass, so a CTA only ever reads vector
// elements it wrote itself (halo coordinates excepted, those are read through L2) and streams long contiguous runs.  Between rounds there is one
// grid-wide synchronisation: CTAs deposit their partial sums in fixed slots, CTA 0 adds them in a fixed order (deterministic: no
// floating-point atomics, result independent of which other problems are in flight), exchanges them with the other ranks when
// n is sharded (ONE exchange per round carrying the sums of all running problems = "one all-reduce of a B-vector per dot"), runs
// each problem's scalar logic -- the line search (a RunTimeCore and a SearchRecord of include/LBFGSpp/LineSearchCore.h), the stopping
// rules (LBFGS.h:137-154) and the curvature gate (:161) of include/LBFGSpp/LoopRules.h: the same code the host loop runs -- plus the
// ring bookkeeping (BFGSMat.h:81-97) and the buffer rotation (pointer swaps) -- and publishes one 128-byte descriptor per problem that tells every CTA what the next round does.  The host is
// not involved between launch and completion: 1 launch per minimize(), 2 + (T - 1) rounds per iteration with T line-search trials.
//
// Data movement: ALL operands of the dots and combination passes -- the right-hand vectors and the history rows, which live in
// a tiled layout (PHist) so that the rows of a tile are one or two contiguous runs -- are staged into shared memory by TMA bulk
// copies (cp.async.bulk + mbarrier) in a two-stage ring of ~90 KB stages: the bytes in flight per SM are set by the ring, not by
// registers.  The trial pass streams through registers (128-bit loads / stores).  Vectors owned by the solver are padded to whole
// 256-byte lines, so every tile -- the ragged end of a vector included -- is a legal bulk copy; lanes past n are masked in the
// arithmetic.  The coefficient recursion of a combination pass runs from a scratch area of its own while the pass's first tiles
// are in flight.  DESIGN.md section 10 has what was measured about the limits of this arrangement.
#pragma once

#include "problem_machine.cuh"

namespace lb {

constexpr int kPThreads = kGramMaxThreads;   // 768: one CTA per SM
constexpr int kPWarps = kPThreads / 32;
constexpr int kPStageBytes = kGramStages * 4 * kGramTE * 8;   // dynamic shared memory of the kernel: 196608 bytes
constexpr int kPMaxStages = 4;
constexpr int kPCache = 4;                   // problems whose leader-side state is kept in shared memory

constexpr int kPOps = 10;   // accounting slots (ops + the "mixed" bucket 0; 9 unused, kept for the solver_profile ABI)
constexpr int kPGramScratch = 1024;   // doubles

// what every CTA needs to know about a problem's next round: one 128-byte line, written by the leader, read through L2
template <class T> struct alignas(128) PRound
{
    T *x, *xp, *g, *gp, *drt;
    T step;                     // TRIAL: the trial's step; DOTS_FORM / MATERIALIZE of an implied point: the step of that point
    int op, c_round, head, pending, gram_cur;
    int at_start;               // DOTS_FORM / MATERIALIZE of an implied point: which point (PT_RAY, PT_START, PT_X)
    int px, pxp;                // objectives without neighbour coupling: the point rows of x and xp in the ring
    int d_implied;              // ... and the first search (k == 1): d = -grad f(xp) is not stored, the passes that read d evaluate it
};
static_assert(sizeof(PRound<double>) == 128 && sizeof(PRound<float>) == 128, "a round descriptor is one 128-byte line");

struct alignas(128) PCtl
{
    unsigned arrive;            // grid barrier: arrivals so far (monotonic); a cache line of its own
    unsigned pad0[31];
    unsigned release;           // grid barrier: last episode released by the leader; bit 31 = nothing left to do
    unsigned pad1[31];
    int abort;                  // watchdog tripped (a wait exceeded its budget): everybody leaves
    int nactive;                // problems still running
    unsigned long long epoch;   // cross-rank exchange sequence number (continues the context's)
    unsigned long long rounds;
    // accounting by CTA 0 (clock64 cycles of its SM): wall time of the rounds by the op they ran (bucket 0: rounds in which
    // problems ran different ops), the part of it spent between CTA 0's own arrival and the release (waiting for the slowest
    // CTA + the leader's work), and the algorithmic n-words of the passes (what the design has to move, see words_of)
    long long cyc_op[kPOps];
    long long cyc_sync;
    long long cyc_wait_all;     // of cyc_sync: from CTA 0's own arrival until the last CTA has arrived
    long long cyc_exchange;     // of cyc_sync: the cross-rank exchange (push, wait for every peer's flag, rank-ordered sums)
    unsigned long long n_op[kPOps];
    double words_op[kPOps];
};
constexpr unsigned kPStopBit = 0x80000000u;

template <class T> struct PArgs
{
    PState<T>* probs;
    PRound<T>* rounds;
    int B;
    PCtl* ctl;
    double* partials;           // [B][pstride][G]
    int pstride;
    int64_t n;
    int grain;                  // chunk boundaries are multiples of this many elements (= the history's block length)
    const XComm* xc;
    int64_t index_offset, n_global;
    long long wait_cycles;      // watchdog budget of a grid-barrier wait (clock64 ticks); cross-rank waits get 4x, the release wait 6x
    bool evict_first_stores;    // the streaming passes (FIRST, MATERIALIZE) store with L2 evict-first: +3 % on the trial pass when it stored x, g at n = 1e7 (set by the host when the vectors cannot stay
                                // in L2 anyway).  Measured and dropped: unrolling the pass 4x (no change), prefetching its inputs into L2 (-5 %), a
                                // grid-stride instead of a chunked sweep (+1 %)
};

// ---- shared memory of the kernel ----------------------------------------------------------------------------------------------
struct PShared
{
    uint64_t full_bar[kPMaxStages];
    double red[kPWarps][3 * kGramVals];     // block reduction scratch (dots: ROUNDS*6 values per warp)
    double coef[2 * kMaxM + 2];             // combination coefficients {cv, cy[c], cs[c]} (stored as T)
    const void* vecs[2 * kMaxM + 2];        // combination pass: the staged vectors {g, (x), y_0.., s_0..} in coefficient order
    unsigned char slots[kMaxM];             // by age: packed row of the column in the staged history block
    unsigned char slotid[kMaxM];            // by age: physical ring slot
    double margin[2][2 * kMaxM + 2];        // neighbour-coupled combination pass: products of the element on either side of a tile
    double carry[2];                        // ... and x1 of the last element of the previous tile (two slots, alternating)
    unsigned char ops[4096];                // this round's op of every problem
    // objectives without neighbour coupling: the point rows a dots / combination pass stages (point_plan)
    unsigned char prow[2 * kMaxM + 2];      // by point row of the ring: its row among the staged points
    unsigned char pstart[kMaxM], pend[kMaxM];   // by column: staged row of the start / end point of its pair
    unsigned char run_at[2 * kMaxM + 2], run_len[2 * kMaxM + 2], run_row[2 * kMaxM + 2];   // one bulk copy per run of ring rows
    int nruns, npts, xrow;                  // copies, staged point rows, staged row of the pass's own point (x, or xp in DOTS_FORM)
};

// Ownership.  CTA i owns the contiguous chunk [c0, c1) of every vector (boundaries on multiples of the history's block length, the
// chunks differ by at most one block) in EVERY pass: a CTA only ever reads what it wrote itself, and every CTA streams long contiguous
// runs of each vector (measured faster than dealing 2048-element blocks round-robin: 14.3 vs 15.1 ms per config-2 solve).
struct Own
{
    int64_t n;
    int G, cta;
    int64_t c0, c1;
    __device__ __forceinline__ Own(int64_t n_, int G_, int cta_, int grain) : n(n_), G(G_), cta(cta_)
    {
        const int64_t units = (n + grain - 1) / grain;
        const int64_t K = units < G ? units : G;
        if (cta >= K) { c0 = c1 = 0; return; }
        c0 = ((units * cta) / K) * grain;
        c1 = ((units * (cta + 1)) / K) * grain;
        if (c1 > n) c1 = n;
    }
    // tiles of TE elements: number owned, first element and length of the t-th (the last one may be shorter)
    __device__ __forceinline__ int64_t ntiles(int TE) const { return (c1 - c0 + TE - 1) / TE; }
    __device__ __forceinline__ int64_t start(int64_t t, int TE) const { return c0 + t * TE; }
    __device__ __forceinline__ int len(int64_t t, int TE) const
    {
        const int64_t rest = c1 - start(t, TE);
        return rest <= 0 ? 0 : (rest < TE ? (int)rest : TE);
    }
};

// block-wide sums of NV per-thread values -> dst[k * G] (this CTA's slot of value k).  All threads call.
template <int NV> __device__ __forceinline__ void block_sums(const double (&acc)[NV], PShared& sh, double* dst, int G)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();   // sh.red may still be read from the previous use
#pragma unroll
    for (int k = 0; k < NV; k++)
    {
        const double w = warp_sum(acc[k]);
        if (lane == 0) sh.red[warp][k] = w;
    }
    __syncthreads();
    if (threadIdx.x < NV)
    {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < kPWarps; w++) t += sh.red[w][threadIdx.x];
        dst[(size_t)threadIdx.x * G] = t;
    }
}

// ---- FIRST / TRIAL -------------------------------------------------------------------------------------------------------------
// MODE 0: FIRST (evaluate at the flat x, write x into point row `pout` of the ring: neither g nor d = -g is stored) ; MODE 1: TRIAL
// (evaluate at x = xp + step*d, xp = point row `pin`, store nothing: the point is rebuilt by the pass that needs it) ; MODE 2:
// MATERIALIZE of a ray point (x = xp + step*d, write the flat x and g; no sums) ; MODE 3: MATERIALIZE of a stored point (evaluate at
// point row `pin`, write the flat x and g; no sums).  d_implied (MODES 1, 2 in the first search): d is not read but evaluated as
// T(-1) * grad f(xp) with FIRST's expressions, bit for bit the d FIRST would have stored; a run-time flag, not a template parameter:
// two more inlined copies of the pass made the dots and combination passes of the kernel 1-2 % slower per round (C5 -1.1 %), measured,
// and unrolling the flag's loop 4x instead of 2x gained nothing (0.0577 against 0.0581 ms per trial round).  Operands stream through
// registers with 128-bit loads/stores (a shared-memory staged variant measured slower for this 1:1 read/write pass); a pack never crosses a block of
// the ring (BT >= 32).  Objectives without neighbour coupling only: the coupled ones take p_trial_halo.
template <class T, class OBJ, int MODE>
__device__ __forceinline__ void p_trial(const OBJ& obj, const Own& own, const PHist<T>& h, int pin, const T* __restrict__ d, T step,
                                        T* __restrict__ x, T* __restrict__ g, int pout, PShared& sh, double* dst, int G, bool evict_first,
                                        bool d_implied = false)
{
    static_assert(!OBJ::kHalo, "neighbour-coupled objectives take p_trial_halo");
    T acc[4] = {T(0), T(0), T(0), T(0)};
    const int64_t n = own.n;
    const int64_t p1 = (own.c1 + 3) >> 2;
    auto store = [&](T* base, int64_t i0, int cnt, const Pack<T>& v) {
        if (evict_first) store4<T, Hint::Stream, true>(base, i0, cnt, v);
        else store4<T, Hint::Plain, true>(base, i0, cnt, v);
    };
    auto body = [&](int64_t q) {
        const int64_t i0 = q << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        T xv[4], dv[4] = {T(0), T(0), T(0), T(0)}, gv[4];
        const T* xin = (MODE == 0) ? x + i0 : h.pt_at(pin, i0);
        const Pack<T> px = load4<T, Hint::Stream, true>(xin, 0, cnt);
        if constexpr (MODE == 1 || MODE == 2)
        {
            if (d_implied)
            {
                T gp[4];
                obj.eval(i0, cnt, px.v, T(0), T(0), gp);   // grad f(xp): FIRST's evaluation of the same point
#pragma unroll
                for (int k = 0; k < 4; k++) dv[k] = (k < cnt) ? T(-1) * gp[k] : T(0);
            }
            else
            {
                const Pack<T> pd = load4<T, Hint::Stream, true>(d, i0, cnt);
#pragma unroll
                for (int k = 0; k < 4; k++) dv[k] = pd.v[k];
            }
#pragma unroll
            for (int k = 0; k < 4; k++) xv[k] = px.v[k] + step * dv[k];
        }
        else
        {
#pragma unroll
            for (int k = 0; k < 4; k++) xv[k] = px.v[k];
        }
        eval_pack(obj, i0, cnt, xv, T(0), T(0), dv, gv, acc);
        Pack<T> pxo;
#pragma unroll
        for (int k = 0; k < 4; k++) pxo.v[k] = xv[k];
        if constexpr (MODE == 0) store(h.pt_at(pout, i0), 0, cnt, pxo);
        if constexpr (MODE >= 2)
        {
            Pack<T> pg;
#pragma unroll
            for (int k = 0; k < 4; k++) pg.v[k] = gv[k];
            store(x, i0, cnt, pxo);
            store(g, i0, cnt, pg);
        }
    };
#pragma unroll 2
    for (int64_t q = (own.c0 >> 2) + threadIdx.x; q < p1; q += kPThreads) body(q);
    if constexpr (MODE < 2)
    {
        const double dacc[4] = {(double)acc[0], (double)acc[1], (double)acc[2], (double)acc[3]};
        block_sums<4>(dacc, sh, dst, G);
    }
}

// Neighbour-coupled objectives (chained Rosenbrock, tridiagonal quadratic): the same pass with its inputs staged tile by tile through
// shared memory by bulk copies, every tile with one 16-byte granule of margin on either side, so that x_{i-1} and x_{i+1} of a pack
// come from the tile instead of from single-word L2 loads per pack (3x faster on config 3).  Only the two ends of the GLOBAL vector
// take their neighbours from the halo record (n-sharding) or as 0.
constexpr int kTrialTE = 2016;    // 63 x 32 elements: with the margins, six fp64 (xp, d) stages fit the ring

template <class T, class OBJ, int MODE>
__device__ __forceinline__ void p_trial_halo(const OBJ& obj, const Own& own, const T* __restrict__ xp, const T* __restrict__ d, T step,
                                             T* __restrict__ x, T* __restrict__ g, T* __restrict__ dout, T* tiles, PShared& sh, unsigned& phase_bits,
                                             double* dst, int G)
{
    constexpr int NIN = (MODE == 1) ? 2 : 1;                         // xp, d  /  x
    constexpr int DV = OBJ::kDataVectors;                            // the objective's data vectors are staged with them
    constexpr int NVEC = NIN + DV;
    constexpr int PAD = 16 / (int)sizeof(T);                         // margin in elements = one 16-byte granule
    constexpr int TS = kTrialTE + 2 * PAD;                           // staged elements per vector per tile
    constexpr int STAGES_MAX = kPStageBytes / (NVEC * TS * (int)sizeof(T));
    constexpr int STAGES = STAGES_MAX > kPMaxStages ? kPMaxStages : STAGES_MAX;
    const int tid = threadIdx.x, lane = tid & 31;
    uint64_t* full_bar = sh.full_bar;
    const T* in0 = (MODE == 1) ? xp : x;
    const int64_t n = own.n;
    const int64_t ntl = own.ntiles(kTrialTE);
    const int64_t n_pad = (n + 31) & ~int64_t(31);                   // the vectors are allocated in whole 256-byte lines

    auto stage_tile = [&](int64_t t, int stage) {
        if (tid != 0) return;
        T* dstt = tiles + (size_t)stage * NVEC * TS;
        const int64_t e0 = own.start(t, kTrialTE);
        const int64_t lo = e0 >= PAD ? e0 - PAD : 0;                 // first element copied
        int64_t hi = e0 + ((own.len(t, kTrialTE) + 31) & ~31) + PAD; // one past the last element copied
        if (hi > n_pad) hi = n_pad;
        const unsigned bytes = (unsigned)(hi - lo) * (unsigned)sizeof(T);
        const int shift = (int)(lo - (e0 - PAD));                    // 0, or PAD at the very start of the vector
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_expect_tx(&full_bar[stage], bytes * NVEC);
        tma_load_1d(dstt + shift, in0 + lo, bytes, &full_bar[stage]);
        if (MODE == 1) tma_load_1d(dstt + TS + shift, d + lo, bytes, &full_bar[stage]);
        if constexpr (DV == 2)
        {
            tma_load_1d(dstt + (size_t)NIN * TS + shift, obj.data0 + lo, bytes, &full_bar[stage]);
            tma_load_1d(dstt + (size_t)(NIN + 1) * TS + shift, obj.data1 + lo, bytes, &full_bar[stage]);
        }
    };

    T acc[4] = {T(0), T(0), T(0), T(0)};
    __syncthreads();   // the tile area is free
    int64_t next_tile = 0;
    for (int s = 0; s < STAGES; s++, next_tile++)
        if (next_tile < ntl) stage_tile(next_tile, s);
    int stage = 0;
    for (int64_t t = 0; t < ntl; t++)
    {
        mbar_wait(&full_bar[stage], (phase_bits >> stage) & 1u);
        phase_bits ^= (1u << stage);
        const T* ta = tiles + (size_t)stage * NVEC * TS + PAD;       // element 0 of the tile
        const T* tb = ta + TS;
        const int64_t e0 = own.start(t, kTrialTE);
        const int len = own.len(t, kTrialTE);
        for (int off = tid * 4; off < len; off += kPThreads * 4)
        {
            const int64_t i0 = e0 + off;
            const int cnt = (len - off >= 4) ? 4 : (len - off);
            T xv[4], dv[4] = {T(0), T(0), T(0), T(0)};
            T xl, xr;
            const Pack<T> pa = lds_pack(ta + off, lane);
            if (MODE == 1)
            {
                const Pack<T> pb = lds_pack(tb + off, lane);
#pragma unroll
                for (int k = 0; k < 4; k++) { dv[k] = (k < cnt) ? pb.v[k] : T(0); xv[k] = (k < cnt) ? pa.v[k] + step * pb.v[k] : T(0); }
                pack_neighbours<true>(obj, i0, n, step, [&](int j) { return ta[off + j] + step * tb[off + j]; }, xl, xr);
            }
            else
            {
#pragma unroll
                for (int k = 0; k < 4; k++) xv[k] = (k < cnt) ? pa.v[k] : T(0);
                pack_neighbours<false>(obj, i0, n, step, [&](int j) { return ta[off + j]; }, xl, xr);
            }
            Pack<T> pg, po;
            eval_pack(obj.staged(ta + (size_t)NIN * TS, ta + (size_t)(NIN + 1) * TS, e0), i0, cnt, xv, xl, xr, dv, pg.v, acc);
#pragma unroll
            for (int k = 0; k < 4; k++) po.v[k] = (MODE == 1) ? xv[k] : T(-1) * pg.v[k];
            if (MODE == 1) store4<T, Hint::Plain, true>(x, i0, cnt, po);
            else store4<T, Hint::Plain, true>(dout, i0, cnt, po);
            store4<T, Hint::Plain, true>(g, i0, cnt, pg);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        if (next_tile < ntl) stage_tile(next_tile, stage);
        next_tile++;
        stage = (stage + 1 == STAGES) ? 0 : stage + 1;
    }
    const double dacc[4] = {(double)acc[0], (double)acc[1], (double)acc[2], (double)acc[3]};
    block_sums<4>(dacc, sh, dst, G);
}

// ---- RESTORE (neighbour-coupled objectives) -----------------------------------------------------------------------------------
template <class T>
__device__ __forceinline__ void p_restore(const Own& own, const T* __restrict__ xp, const T* __restrict__ gp, T* __restrict__ x, T* __restrict__ g)
{
    const int64_t n = own.n;
    const int64_t p1 = (own.c1 + 3) >> 2;
    for (int64_t q = (own.c0 >> 2) + threadIdx.x; q < p1; q += kPThreads)
    {
        const int64_t i0 = q << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        store4<T, Hint::Plain, true>(x, i0, cnt, load4<T, Hint::Stream, true>(xp, i0, cnt));
        store4<T, Hint::Plain, true>(g, i0, cnt, load4<T, Hint::Stream, true>(gp, i0, cnt));
    }
}

// the `cnt` slots of the ring that end just below `end` (cyclically), as <= 2 ascending runs of slots; packed row of a slot
struct SlotRuns
{
    int a0, a1, b0, b1;   // run A = [a0, a1), run B = [b0, b1) (empty when b0 == b1); rows: A first, then B
    __device__ __forceinline__ SlotRuns(int end, int cnt, int M)
    {
        if (cnt <= end) { a0 = end - cnt; a1 = end; b0 = b1 = 0; }
        else { a0 = 0; a1 = end; b0 = M - (cnt - end); b1 = M; }
    }
    __device__ __forceinline__ int row_of(int slot) const { return (slot >= a0 && slot < a1) ? slot - a0 : (a1 - a0) + (slot - b0); }
};

// 16-byte units (2 doubles / 4 floats): the granularity of the staged passes
template <class T> struct alignas(16) Unit { T v[16 / sizeof(T)]; };
template <class T> __device__ __forceinline__ Unit<T> lds_unit(const T* p)
{
    Unit<T> u;
    *reinterpret_cast<float4*>(u.v) = *reinterpret_cast<const float4*>(p);
    return u;
}
template <class T> __device__ __forceinline__ void st_unit(T* base, int64_t i0, int cnt, const Unit<T>& u)
{
    constexpr int EPT = 16 / (int)sizeof(T);
    if (cnt >= EPT) { *reinterpret_cast<float4*>(base + i0) = *reinterpret_cast<const float4*>(u.v); return; }
#pragma unroll
    for (int k = 0; k < EPT; k++)
        if (k < cnt) base[i0 + k] = u.v[k];
}
template <class T> __device__ __forceinline__ void mask_unit(Unit<T>& u, int cnt)
{
#pragma unroll
    for (int k = 0; k < 16 / (int)sizeof(T); k++) u.v[k] = (k < cnt) ? u.v[k] : T(0);
}
// g = grad f(x) of the unit at elements i0.. of an objective without neighbour coupling (lanes past cnt: x = 0): the arithmetic of
// every pass that evaluates the objective, so bit for bit the g a pass would have stored for that point
template <class T, class OBJ> __device__ __forceinline__ Unit<T> grad_unit(const OBJ& obj, int64_t i0, int cnt, const Unit<T>& ux)
{
    constexpr int EPT = 16 / (int)sizeof(T);
    const int c4 = cnt < EPT ? cnt : EPT;
    T xv[4] = {T(0), T(0), T(0), T(0)}, gv[4];
#pragma unroll
    for (int k = 0; k < EPT; k++) xv[k] = (k < c4) ? ux.v[k] : T(0);
    obj.eval(i0, c4, xv, T(0), T(0), gv);
    Unit<T> ug;
#pragma unroll
    for (int k = 0; k < EPT; k++) ug.v[k] = gv[k];
    return ug;
}

// copies of one tile: `nrhs` right-hand rows, of which the first `nload` are loaded (sh.vecs[0..nload), round_up(len, 32) elements
// each) and the others are left for the pass to fill, + the history runs of block `blk`; one lane per copy.  Returns nothing; the
// stage's barrier has been told the byte count.
template <class T>
__device__ __forceinline__ void stage_tiled(T* dstt, int TE, int nrhs, int nload, int64_t e0, int len, const PHist<T>& h, const SlotRuns& runs,
                                            PShared& sh, uint64_t* bar)
{
    const int tid = threadIdx.x;
    if (tid >= 32) return;
    const unsigned rbytes = (unsigned)((len + 31) & ~31) * (unsigned)sizeof(T);
    const unsigned abytes = (unsigned)(runs.a1 - runs.a0) * 2u * (unsigned)TE * (unsigned)sizeof(T);
    const unsigned bbytes = (unsigned)(runs.b1 - runs.b0) * 2u * (unsigned)TE * (unsigned)sizeof(T);
    if (tid == 0)
    {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy accesses of this stage before the copies that overwrite it
        mbar_expect_tx(bar, rbytes * (unsigned)nload + abytes + bbytes);
    }
    __syncwarp();
    const T* blk = h.H + (e0 >> h.bt_log) * h.bstride;
    if (tid < nload) tma_load_1d(dstt + (size_t)tid * TE, static_cast<const T*>(sh.vecs[tid]) + e0, rbytes, bar);
    else if (tid == nrhs && abytes) tma_load_1d(dstt + (size_t)nrhs * TE, blk + (size_t)runs.a0 * 2 * TE, abytes, bar);
    else if (tid == nrhs + 1 && bbytes) tma_load_1d(dstt + (size_t)(nrhs + 2 * (runs.a1 - runs.a0)) * TE, blk + (size_t)runs.b0 * 2 * TE, bbytes, bar);
}

// Objectives without neighbour coupling: the point rows a pass stages -- the start and end points of the pairs of ages
// 0 .. ncols-1 (columns col0 .. col0+ncols-1) and the pass's own point `own_pt` -- in ring order, one bulk copy per run of consecutive
// rows: a chained history (every pair starting where the older one ends) is one run, or two where it wraps.  A pair rejected by the
// curvature gate breaks the chain and leaves more, shorter runs.  All threads call; the previous pass no longer reads sh.
template <class T>
__device__ void point_plan(const PState<T>* st, int head, int ncols, int col0, int own_pt, PShared& sh)
{
    const int tid = threadIdx.x;
    const int M = st->hist.M, P = 2 * M;
    for (int p = tid; p < P; p += kPThreads) sh.prow[p] = 0;
    __syncthreads();
    if (tid < ncols)
    {
        const int slot = slot_by_age(head, M, tid);
        const unsigned char a = __ldcg(st->pts + 2 * slot), b = __ldcg(st->pts + 2 * slot + 1);
        sh.pstart[col0 + tid] = a;
        sh.pend[col0 + tid] = b;
        sh.prow[a] = 1;
        sh.prow[b] = 1;
    }
    if (tid == 0) sh.prow[own_pt] = 1;
    __syncthreads();
    if (tid == 0)
    {
        int rows = 0, runs = 0;
        bool prev = false;
        for (int p = 0; p < P; p++)
        {
            const bool used = sh.prow[p] != 0;
            if (used)
            {
                if (!prev) { sh.run_at[runs] = (unsigned char)p; sh.run_len[runs] = 0; sh.run_row[runs] = (unsigned char)rows; runs++; }
                sh.run_len[runs - 1]++;
                sh.prow[p] = (unsigned char)rows++;
            }
            prev = used;
        }
        sh.nruns = runs;
        sh.npts = rows;
        sh.xrow = sh.prow[own_pt];
    }
    __syncthreads();
    if (tid < ncols)
    {
        sh.pstart[col0 + tid] = sh.prow[sh.pstart[col0 + tid]];
        sh.pend[col0 + tid] = sh.prow[sh.pend[col0 + tid]];
    }
    __syncthreads();
}

// copies of one tile, objectives without neighbour coupling: `nload` right-hand rows (sh.vecs), room for nrhs - nload rows the pass
// fills, then the sh.npts point rows of point_plan; lanes of warp 0.  The stage's barrier has been told the byte count.
template <class T>
__device__ __forceinline__ void stage_points(T* dstt, int TE, int nrhs, int nload, int64_t e0, int len, const PHist<T>& h, const PShared& sh,
                                             uint64_t* bar)
{
    const int tid = threadIdx.x;
    if (tid >= 32) return;
    const unsigned rbytes = (unsigned)((len + 31) & ~31) * (unsigned)sizeof(T);
    if (tid == 0)
    {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy accesses of this stage before the copies that overwrite it
        mbar_expect_tx(bar, rbytes * (unsigned)nload + (unsigned)sh.npts * (unsigned)TE * (unsigned)sizeof(T));
    }
    __syncwarp();
    const T* blk = h.H + (e0 >> h.bt_log) * h.bstride;
    T* prows = dstt + (size_t)nrhs * TE;
    if (tid < nload) tma_load_1d(dstt + (size_t)tid * TE, static_cast<const T*>(sh.vecs[tid]) + e0, rbytes, bar);
    for (int r = tid; r < sh.nruns; r += 32)
        tma_load_1d(prows + (size_t)sh.run_row[r] * TE, blk + ((size_t)sh.run_at[r] << h.bt_log), (unsigned)sh.run_len[r] * (unsigned)TE * (unsigned)sizeof(T), bar);
}

// ---- DOTS -----------------------------------------------------------------------------------------------------------------------
// [S Y]'[g s_new y_new] (FORM) or [S Y]'g over the old history (PLAIN), over this CTA's chunk, one block (tile) at a time, everything
// staged by bulk copies.  Column j (by age) belongs to warp group j, whose `split` warps share the tile's units.  Before the column
// groups read a staged tile, forming warps take each of its units once and leave what the columns read in its first right-hand rows:
// g in row 0 and, in FORM, the new pair s, y in rows 1 and 2:
//     FORM,  implied point (no neighbour coupling)   staged d (+ two rows no copy fills) and the points: gp = grad f(xp), x = xp +
//                                                    step*d and g = grad f(x) with the trial's own arithmetic (or x = xp, g = gp when
//                                                    the search ended on its start point), s = x - xp, y = g - gp; x is written to its
//                                                    point row (g is not stored: the next pass evaluates it from x; nor is the pair:
//                                                    its readers rebuild it from its endpoints).  Iteration 1 (d_implied): d is not
//                                                    staged but taken as T(-1) * gp, FIRST's d
//     FORM,  stored point (neighbour-coupled)        staged g, x, gp, xp: s = x - xp, y = g - gp, written to ring slot `new_slot`
//                                                    (row 0 stays g)
//     PLAIN, no neighbour coupling                   the points: g = grad f(x)
//     PLAIN, neighbour-coupled                       staged g: nothing to form
// In FORM the new pair is column 0; in PLAIN every column, age 0 included, is an old pair.  Objectives without neighbour coupling
// stage the pairs' endpoints (point_plan) and a column warp rebuilds s = x_end - x_start, y = grad f(x_end) - grad f(x_start) of
// each unit with the arithmetic that formed it, bit for bit the pair the forming pass had; neighbour-coupled objectives stage the
// ring's S|Y slots (the column of age j: sh.slots[j]).  The forming warps are the ones
// dots_geometry leaves without a column (c = 10: 4 of 24) or, when every warp has a column (c = 3, 6, 12, ...), the warps of column 0,
// which form a tile before taking their own dots of it.  Neither the unit-to-lane mapping of the columns nor any accumulator depends on
// who forms, so the sums are bit-identical to forming the pair in every column warp.
// No CTA-wide barrier per tile (a per-tile __syncthreads() left the column warps idle ~30 % of a tile at c = 10, DESIGN.md section 3):
// every stage has three mbarriers -- full (the bulk copies; parity in phase_bits), formed (arrivals of the forming warps, which arrive
// also when they have nothing to form) and empty (arrivals of the column warps), the latter two initialised by the pass -- and warp 0,
// after its own dots of a tile, waits for the stage's empty barrier and re-arms it.  So a column group starts a tile as soon as it is
// formed.
template <class T> struct PDots
{
    int64_t n;
    PHist<T> h;
    int c;               // columns taking part (FORM: including the new pair)
    int end, cnt_old;    // the old columns: the cnt_old slots below `end`
    int new_slot, split, cols_per_round;
    T step;              // FORM of an implied point: its step (PT_RAY), or the start point (PT_START)
    int at_start;
    int px;              // FORM of an implied point: the point row it is written to
    bool d_implied;      // FORM of an implied point: d = -grad f(xp) is not stored (iteration 1); the d row is not loaded
};

template <class T, class OBJ, int ROUNDS, bool FORM>
__device__ __forceinline__ void p_dots(const PDots<T>& a, const OBJ& obj, const Own& own, T* tiles, PShared& sh, unsigned& phase_bits, double* dst,
                                       int G)
{
    constexpr int EPT = 16 / (int)sizeof(T);
    constexpr bool HALO = OBJ::kHalo;
    constexpr int NRHS = !FORM ? 1 : (HALO ? 4 : 3);             // right-hand rows: g / (formed) ; FORM: g, x, gp, xp / d, (formed) x 2
    const int nload = HALO ? NRHS : (FORM && !a.d_implied ? 1 : 0);   // ... of which the bulk copies fill the first nload
    __shared__ uint64_t formed_bar[kPMaxStages], empty_bar[kPMaxStages];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int TE = a.h.BT();
    const int units = TE / EPT;
    const int my_col = warp / a.split, my_part = warp % a.split;
    const int upp = units / a.split;                             // units of a tile per warp of a column group
    const SlotRuns runs(a.end, a.cnt_old, a.h.M);
    const int nrows = NRHS + (HALO ? 2 * a.cnt_old : sh.npts);
    int stages = (int)((size_t)kPStageBytes / ((size_t)nrows * TE * sizeof(T)));
    stages = stages > kPMaxStages ? kPMaxStages : stages;
    const int64_t ntl = own.ntiles(TE);
    uint64_t* full_bar = sh.full_bar;
    const int col_warps = (a.c < a.cols_per_round ? a.c : a.cols_per_round) * a.split;   // warps with a column
    const bool spare = col_warps < kPWarps;
    const int nform = spare ? kPWarps - col_warps : a.split;
    const int fw = spare ? warp - col_warps : warp;              // index among the forming warps
    const bool former = fw >= 0 && fw < nform;

    T acc[ROUNDS][kGramVals];
#pragma unroll
    for (int r = 0; r < ROUNDS; r++)
#pragma unroll
        for (int k = 0; k < kGramVals; k++) acc[r][k] = T(0);

    if (tid == 0)
        for (int s = 0; s < stages; s++) { mbar_init(&formed_bar[s], nform); mbar_init(&empty_bar[s], col_warps); }
    __syncthreads();   // sh.vecs / sh.slots and the barriers are in place, the staging ring is free
    int64_t next_tile = 0;
    auto stage_one = [&](T* dstt, int64_t t, uint64_t* bar) {
        if constexpr (HALO) stage_tiled<T>(dstt, TE, NRHS, NRHS, own.start(t, TE), own.len(t, TE), a.h, runs, sh, bar);
        else stage_points<T>(dstt, TE, NRHS, nload, own.start(t, TE), own.len(t, TE), a.h, sh, bar);
    };
    for (int s = 0; s < stages; s++, next_tile++)
        if (next_tile < ntl) stage_one(tiles + (size_t)s * nrows * TE, next_tile, &full_bar[s]);
    const unsigned full_phase = phase_bits;
    int stage = 0;
    unsigned lap = 0;                                            // parity of the current use of `stage` in this pass
    for (int64_t t = 0; t < ntl; t++)
    {
        T* base = tiles + (size_t)stage * nrows * TE;
        const T* hist = base + (size_t)NRHS * TE;
        const int64_t e0 = own.start(t, TE);
        const int len = own.len(t, TE);
        if (former)
        {
            mbar_wait(&full_bar[stage], ((full_phase >> stage) & 1u) ^ lap);
            if constexpr (FORM || !HALO)
            {
                for (int u = fw * 32 + lane; u < units; u += nform * 32)
                {
                    const int off = u * EPT;
                    const int cnt = len - off;
                    if (cnt <= 0) break;
                    if constexpr (!FORM)
                    {
                        const Unit<T> ug = grad_unit(obj, e0 + off, cnt, lds_unit<T>(hist + (size_t)sh.xrow * TE + off));
                        *reinterpret_cast<float4*>(base + off) = *reinterpret_cast<const float4*>(ug.v);
                    }
                    else
                    {
                        Unit<T> ux, ug, uxp, ugp, usn, uyn;
                        if constexpr (HALO)
                        {
                            ug = lds_unit<T>(base + off);
                            ux = lds_unit<T>(base + TE + off);
                            ugp = lds_unit<T>(base + 2 * TE + off);
                            uxp = lds_unit<T>(base + 3 * TE + off);
                        }
                        else
                        {
                            uxp = lds_unit<T>(hist + (size_t)sh.xrow * TE + off);
                            ugp = grad_unit(obj, e0 + off, cnt, uxp);
                            if (a.at_start) { ux = uxp; ug = ugp; }
                            else
                            {
                                Unit<T> ud;
                                if (a.d_implied)   // FIRST's d = T(-1) * grad f(x0)
                                {
#pragma unroll
                                    for (int k = 0; k < EPT; k++) ud.v[k] = T(-1) * ugp.v[k];
                                }
                                else ud = lds_unit<T>(base + off);
                                // the trial's arithmetic (p_trial, and p_combine's first trial with step 1 on the stored d)
#pragma unroll
                                for (int k = 0; k < EPT; k++) ux.v[k] = (k < cnt) ? uxp.v[k] + a.step * ud.v[k] : T(0);
                                ug = grad_unit(obj, e0 + off, cnt, ux);
                            }
                        }
#pragma unroll
                        for (int k = 0; k < EPT; k++) { usn.v[k] = ux.v[k] - uxp.v[k]; uyn.v[k] = ug.v[k] - ugp.v[k]; }
                        if (cnt < EPT) { mask_unit(usn, cnt); mask_unit(uyn, cnt); }
                        if constexpr (HALO)
                        {
                            T* s_new = a.h.s_at(a.new_slot, e0);
                            st_unit<T>(s_new, off, cnt, usn);
                            st_unit<T>(s_new + TE, off, cnt, uyn);
                        }
                        else
                        {
                            st_unit<T>(a.h.pt_at(a.px, e0), off, cnt, ux);
                            *reinterpret_cast<float4*>(base + off) = *reinterpret_cast<const float4*>(ug.v);
                        }
                        *reinterpret_cast<float4*>(base + TE + off) = *reinterpret_cast<const float4*>(usn.v);
                        *reinterpret_cast<float4*>(base + 2 * TE + off) = *reinterpret_cast<const float4*>(uyn.v);
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // these writes before the bulk copies that re-arm the stage
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&formed_bar[stage]);
        }
        if (warp < col_warps)
        {
            mbar_wait(&formed_bar[stage], lap);
#pragma unroll
            for (int r = 0; r < ROUNDS; r++)
            {
                const int j = r * a.cols_per_round + my_col;
                if (my_col < a.cols_per_round && j < a.c)
                {
                    const bool is_new = FORM && j == 0;
                    // HALO: sh.slots[j] = packed row of the column of age j ; otherwise the staged rows of its pair's endpoints
                    const T* srow = HALO ? hist + (size_t)2 * (is_new ? 0 : sh.slots[j]) * TE : hist + (size_t)(is_new ? 0 : sh.pstart[j]) * TE;
                    const T* yrow = HALO ? srow + TE : hist + (size_t)(is_new ? 0 : sh.pend[j]) * TE;
                    for (int u = my_part * upp + lane; u < (my_part + 1) * upp; u += 32)
                    {
                        const int off = u * EPT;
                        const int cnt = len - off;
                        if (cnt <= 0) break;
                        Unit<T> ug = lds_unit<T>(base + off), us, uy, usn{}, uyn{};
                        if constexpr (FORM) { usn = lds_unit<T>(base + TE + off); uyn = lds_unit<T>(base + 2 * TE + off); }
                        if (is_new) { us = usn; uy = uyn; }
                        else if constexpr (HALO) { us = lds_unit<T>(srow + off); uy = lds_unit<T>(yrow + off); }
                        else
                        {
                            const Unit<T> ua = lds_unit<T>(srow + off), ub = lds_unit<T>(yrow + off);   // x_start, x_end
                            const Unit<T> ga = grad_unit(obj, e0 + off, cnt, ua), gb = grad_unit(obj, e0 + off, cnt, ub);
#pragma unroll
                            for (int k = 0; k < EPT; k++) { us.v[k] = ub.v[k] - ua.v[k]; uy.v[k] = gb.v[k] - ga.v[k]; }
                        }
                        if (cnt < EPT) { mask_unit(ug, cnt); mask_unit(us, cnt); mask_unit(uy, cnt); }
#pragma unroll
                        for (int k = 0; k < EPT; k++)
                        {
                            acc[r][0] += us.v[k] * ug.v[k];
                            acc[r][1] += uy.v[k] * ug.v[k];
                        }
                        if constexpr (FORM)
                        {
#pragma unroll
                            for (int k = 0; k < EPT; k++)
                            {
                                acc[r][2] += us.v[k] * uyn.v[k];
                                acc[r][3] += uy.v[k] * uyn.v[k];
                                acc[r][4] += uy.v[k] * usn.v[k];
                                acc[r][5] += us.v[k] * usn.v[k];
                            }
                        }
                    }
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // these reads before the bulk copies that re-arm the stage
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
        }
        if (warp == 0 && next_tile < ntl)
        {
            mbar_wait(&empty_bar[stage], lap);
            stage_one(base, next_tile, &full_bar[stage]);
        }
        next_tile++;
        if (++stage == stages) { stage = 0; lap ^= 1u; }
    }
    // the full barriers: one completed phase per tile a stage carried (every thread keeps the same parities, waiting or not)
    for (int s = 0; s < stages; s++)
        if (s < ntl) phase_bits ^= (unsigned)(((ntl - 1 - s) / stages + 1) & 1) << s;

    // block reduction: lanes -> warp, then the `split` warps of a column; value (j, k) -> dst[(j*6 + k) * G] (the forming warps
    // without a column contribute zeros that nobody reads)
#pragma unroll
    for (int r = 0; r < ROUNDS; r++)
#pragma unroll
        for (int k = 0; k < kGramVals; k++)
        {
            const double w = warp_sum((double)acc[r][k]);
            if (lane == 0) sh.red[warp][r * kGramVals + k] = w;
        }
    __syncthreads();   // (also: every arrival on and wait for the formed / empty barriers is done)
    if (tid == 0)
        for (int s = 0; s < stages; s++) { mbar_inval(&formed_bar[s]); mbar_inval(&empty_bar[s]); }
    const int nvals = a.c * kGramVals;
    for (int idx = tid; idx < nvals; idx += kPThreads)
    {
        const int j = idx / kGramVals, k = idx % kGramVals;
        const int r = j / a.cols_per_round, col = j % a.cols_per_round;
        double t = 0.0;
        for (int p = 0; p < a.split; p++) t += sh.red[col * a.split + p][r * kGramVals + k];
        dst[(size_t)idx * G] = t;
    }
}

// how the warps of the dots pass share the columns: `split` warps per column pair, cols_per_round column pairs at a time
__device__ __forceinline__ void dots_geometry(int c, int units, int& split, int& cols_per_round)
{
    split = 8;
    while (split > 1 && (c * split > kGramMaxWarps || units / split < 32)) split >>= 1;
    cols_per_round = c < kGramMaxWarps / split ? c : kGramMaxWarps / split;
}

// ---- COMBINE (+ first trial) ---------------------------------------------------------------------------------------------------
// d = cv*v + sum_j cy_j*y_j + cs_j*s_j ; FUSE: x1 = xc + d, g1 = grad f(x1) and the four trial sums (neighbour-coupled objectives:
// x1, g1 written to (x1_out, g1_out)).
// Staged rows of a tile: v, (xc,) then the history block's live slots; sh.slots[j] = packed row of the pair of age j (objectives
// without neighbour coupling stage points instead and take p_combine_points).  A thread owns
// one 16-byte unit of the tile and adds the terms in the order the recursion would (y newest -> oldest, then s oldest -> newest), with
// the operand loads of 8 columns in flight before their multiply-adds retire (the pass is bound by shared-memory latency otherwise).
// HALO (neighbour-coupled objectives, one GPU): x1 goes back into the staged x row, two spare warps form d and x1 of the element on
// either side of the tile from global memory with the very arithmetic of the tile that owns it, and after a barrier the objective
// takes x1_{i-1}, x1_{i+1} from shared memory.
// `between` (all threads) runs after the bulk copies of the first tiles have been issued and before anything reads the coefficients:
// the coefficient recursion overlaps the latency of those copies when it has a scratch area of its own.
template <class T, class OBJ, bool FUSE, bool HALO, class Between>
__device__ __forceinline__ void p_combine(const OBJ& obj, const Own& own, const PHist<T>& h, int c, int end, T* tiles, T* __restrict__ res,
                                          T* __restrict__ x1_out, T* __restrict__ g1_out, PShared& sh, unsigned& phase_bits, double* dst, int G,
                                          Between between)
{
    constexpr int EPT = 16 / (int)sizeof(T);
    static_assert(OBJ::kHalo, "objectives without neighbour coupling take p_combine_points");
    constexpr int DV = HALO ? OBJ::kDataVectors : 0;              // HALO: the objective's data vectors ride in the stage as well
    constexpr int NRHS = (FUSE ? 2 : 1) + DV;                     // v (, xc) (, data0, data1)
    constexpr int PAD = EPT;                                      // HALO: room for x1 of the neighbouring element on either side of the x row
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int TE = h.BT();
    const SlotRuns runs(end, c, h.M);
    const int nrows = NRHS + 2 * c;
    const size_t stage_elems = (size_t)nrows * TE + (HALO ? 2 * PAD : 0);
    int stages = (int)((size_t)kPStageBytes / (stage_elems * sizeof(T)));
    stages = stages > kPMaxStages ? kPMaxStages : stages;
    const int64_t n = own.n;
    const int64_t ntl = own.ntiles(TE);
    const T* s_coef = reinterpret_cast<const T*>(sh.coef);
    uint64_t* full_bar = sh.full_bar;
    // HALO: the x row is staged one granule into the stage (row 1 starts at TE + PAD), everything after it shifts by 2*PAD
    auto stage_one = [&](int64_t t, int s) {
        T* dstt = tiles + (size_t)s * stage_elems;
        if (!HALO) { stage_tiled<T>(dstt, TE, NRHS, NRHS, own.start(t, TE), own.len(t, TE), h, runs, sh, &full_bar[s]); return; }
        if (tid >= 32) return;
        const int64_t e0 = own.start(t, TE);
        const int len = own.len(t, TE);
        const unsigned rbytes = (unsigned)((len + 31) & ~31) * (unsigned)sizeof(T);
        const unsigned abytes = (unsigned)(runs.a1 - runs.a0) * 2u * (unsigned)TE * (unsigned)sizeof(T);
        const unsigned bbytes = (unsigned)(runs.b1 - runs.b0) * 2u * (unsigned)TE * (unsigned)sizeof(T);
        if (tid == 0)
        {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(&full_bar[s], rbytes * (unsigned)NRHS + abytes + bbytes);
        }
        __syncwarp();
        const T* blk = h.H + (e0 >> h.bt_log) * h.bstride;
        T* hist = dstt + (size_t)NRHS * TE + 2 * PAD;
        if (tid == 0) tma_load_1d(dstt, static_cast<const T*>(sh.vecs[0]) + e0, rbytes, &full_bar[s]);
        else if (tid == 1) tma_load_1d(dstt + TE + PAD, static_cast<const T*>(sh.vecs[1]) + e0, rbytes, &full_bar[s]);
        else if (tid == 2 && abytes) tma_load_1d(hist, blk + (size_t)runs.a0 * 2 * TE, abytes, &full_bar[s]);
        else if (tid == 3 && bbytes) tma_load_1d(hist + (size_t)2 * (runs.a1 - runs.a0) * TE, blk + (size_t)runs.b0 * 2 * TE, bbytes, &full_bar[s]);
        else if (tid >= 4 && tid < 4 + DV) tma_load_1d(dstt + (size_t)(tid - 2) * TE + 2 * PAD, static_cast<const T*>(sh.vecs[tid - 2]) + e0, rbytes, &full_bar[s]);
    };

    T acc[5] = {T(0), T(0), T(0), T(0), T(0)};
    T pre[5] = {T(0), T(0), T(0), T(0), T(0)};   // HALO, right-margin warp: operands of the element after the current tile
    // FUSE: the trial of one unit at x1 = xv (lanes past EPT: 0, or x1 of the right neighbour) -> acc[1..4]; x1 and g1 stored
    auto first_trial = [&](const OBJ& o, int64_t i0, int cnt, const T (&xv)[4], T xl, T xr, const T (&r)[EPT]) {
        T dv[EPT], gv[4];
#pragma unroll
        for (int k = 0; k < EPT; k++) dv[k] = (k < cnt) ? r[k] : T(0);   // (past cnt, d comes from whatever the vectors' padding holds)
        eval_pack(o, i0, cnt, xv, xl, xr, dv, gv, acc + 1);
        Unit<T> ug, uo;
#pragma unroll
        for (int k = 0; k < EPT; k++) { ug.v[k] = gv[k]; uo.v[k] = xv[k]; }
        st_unit<T>(x1_out, i0, cnt, uo);
        st_unit<T>(g1_out, i0, cnt, ug);
    };
    __syncthreads();   // sh.vecs / sh.slots are in place and the staging ring is free
    int64_t next_tile = 0;
    for (int s = 0; s < stages; s++, next_tile++)
        if (next_tile < ntl) stage_one(next_tile, s);
    between();         // (ends with a barrier: sh.coef is in place)
    const T cv = s_coef[0];
    int stage = 0;
    for (int64_t t = 0; t < ntl; t++)
    {
        mbar_wait(&full_bar[stage], (phase_bits >> stage) & 1u);
        phase_bits ^= (1u << stage);
        T* base = tiles + (size_t)stage * stage_elems;                          // row 0: v
        T* xrow = base + TE + (HALO ? PAD : 0);                                  // row 1: xc (FUSE)
        const T* hist = base + (size_t)NRHS * TE + (HALO ? 2 * PAD : 0);
        const int len = own.len(t, TE);
        const int64_t e0 = own.start(t, TE);
        // d of one unit: the arithmetic every owner of an element uses
        auto direction = [&](int off, T (&r)[EPT], Unit<T>& uv) {
            uv = lds_unit<T>(base + off);
#pragma unroll
            for (int k = 0; k < EPT; k++) r[k] = cv * uv.v[k];
#pragma unroll 8
            for (int j = 0; j < c; j++)                    // y terms newest -> oldest
            {
                const Unit<T> uy = lds_unit<T>(hist + ((size_t)2 * sh.slots[j] + 1) * TE + off);
                const T cy = s_coef[1 + j];
#pragma unroll
                for (int k = 0; k < EPT; k++) r[k] += cy * uy.v[k];
            }
#pragma unroll 8
            for (int j = c - 1; j >= 0; j--)               // s terms oldest -> newest
            {
                const Unit<T> us = lds_unit<T>(hist + (size_t)2 * sh.slots[j] * TE + off);
                const T cs = s_coef[1 + c + j];
#pragma unroll
                for (int k = 0; k < EPT; k++) r[k] += cs * us.v[k];
            }
        };
        if constexpr (!HALO)
        {
            for (int off = tid * EPT; off < len; off += kPThreads * EPT)
            {
                const int cnt = (len - off >= EPT) ? EPT : (len - off);
                T r[EPT];
                Unit<T> uv;
                direction(off, r, uv);
                Unit<T> out;
#pragma unroll
                for (int k = 0; k < EPT; k++)
                {
                    out.v[k] = r[k];
                    acc[0] += (k < cnt) ? uv.v[k] * r[k] : T(0);
                }
                const int64_t i0 = e0 + off;
                st_unit<T>(res, i0, cnt, out);
                if constexpr (FUSE)
                {
                    const Unit<T> ux = lds_unit<T>(xrow + off);
                    T xv[4] = {T(0), T(0), T(0), T(0)};
#pragma unroll
                    for (int k = 0; k < EPT; k++) xv[k] = (k < cnt) ? ux.v[k] + T(1) * r[k] : T(0);
                    first_trial(obj, i0, cnt, xv, T(0), T(0), r);
                }
            }
        }
        else
        {
            // ---- phase 1: d and x1 of the tile's units (one per thread: a tile has at most 512 units) ----
            const int off = tid * EPT;
            const bool mine = off < len;
            const int64_t i0 = e0 + off;
            const int cnt = mine ? ((len - off >= EPT) ? EPT : (len - off)) : 0;
            T r[EPT];
#pragma unroll
            for (int k = 0; k < EPT; k++) r[k] = T(0);
            if (mine)
            {
                Unit<T> uv;
                direction(off, r, uv);
                Unit<T> out;
#pragma unroll
                for (int k = 0; k < EPT; k++)
                {
                    out.v[k] = r[k];
                    acc[0] += (k < cnt) ? uv.v[k] * r[k] : T(0);
                }
                st_unit<T>(res, i0, cnt, out);
                const Unit<T> ux = lds_unit<T>(xrow + off);
                Unit<T> u1;
#pragma unroll
                for (int k = 0; k < EPT; k++) u1.v[k] = (k < cnt) ? ux.v[k] + T(1) * r[k] : T(0);
                *reinterpret_cast<float4*>(xrow + off) = *reinterpret_cast<const float4*>(u1.v);
            }
            // the element on either side of the tile.  Left: the previous tile of this chunk left its last x1 in sh.carry (only a chunk's
            // first tile asks global memory).  Right: warp kPWarps-1 holds the operands of the element after the tile (fetched through
            // L2 one tile ahead: other CTAs wrote them in earlier rounds), multiplies them by their coefficients in parallel and lane 0
            // adds the products in the owner's order -- the owner's arithmetic, bit for bit.
            if (warp == kPWarps - 2 && lane == 0 && t > 0) xrow[-1] = *reinterpret_cast<const T*>(&sh.carry[(t - 1) & 1]);
            if (warp >= kPWarps - 2 && (warp == kPWarps - 1 || t == 0))
            {
                const bool left = warp == kPWarps - 2;
                const int64_t im = left ? e0 - 1 : e0 + len;
                T* scratch = reinterpret_cast<T*>(sh.margin[left ? 0 : 1]);
                auto fetch = [&](int64_t i, T (&dstv)[5]) {
#pragma unroll
                    for (int w = 0; w < 5; w++)
                    {
                        const int q = lane + 32 * w;
                        T val = T(0);
                        if (i >= 0 && i < n && q < 2 * c + 2)
                        {
                            if (q == 0) val = __ldcg(static_cast<const T*>(sh.vecs[0]) + i);
                            else if (q == 1) val = __ldcg(static_cast<const T*>(sh.vecs[1]) + i);
                            else if (q < 2 + c) val = __ldcg(h.y_at(sh.slotid[q - 2], i));          // y of age q-2
                            else val = __ldcg(h.s_at(sh.slotid[q - 2 - c], i));                      // s of age q-2-c
                        }
                        dstv[w] = val;
                    }
                };
                if (left || t == 0) fetch(im, pre);        // (the right-margin warp fetched this tile's element during the previous tile)
                if (im >= 0 && im < n)
                {
#pragma unroll
                    for (int w = 0; w < 5; w++)
                    {
                        const int q = lane + 32 * w;
                        if (q < 2 * c + 2)
                            scratch[q] = (q == 0) ? cv * pre[w] : (q == 1) ? pre[w] : (q < 2 + c) ? s_coef[1 + (q - 2)] * pre[w] : s_coef[1 + c + (q - 2 - c)] * pre[w];
                    }
                    __syncwarp();
                    if (lane == 0)
                    {
                        T rm = scratch[0];
                        for (int j = 0; j < c; j++) rm += scratch[2 + j];
                        for (int j = c - 1; j >= 0; j--) rm += scratch[2 + c + j];
                        xrow[left ? -1 : len] = scratch[1] + T(1) * rm;
                    }
                }
                if (!left && t + 1 < ntl) fetch(own.start(t + 1, TE) + own.len(t + 1, TE), pre);   // next tile's right neighbour, in flight meanwhile
            }
            if (mine && off + EPT >= len) *reinterpret_cast<T*>(&sh.carry[t & 1]) = xrow[len - 1];   // (this thread wrote it above; two slots: the next tile reads the other one)
            __syncthreads();
            // ---- phase 2: the objective at x1 with its neighbours from shared memory ----
            if (mine)
            {
                T xv[4] = {T(0), T(0), T(0), T(0)};
                const Unit<T> u1 = lds_unit<T>(xrow + off);
#pragma unroll
                for (int k = 0; k < EPT; k++) xv[k] = u1.v[k];
                const T xl = (i0 > 0) ? xrow[off - 1] : T(0);
                const T right = (i0 + EPT < n) ? xrow[off + EPT] : T(0);
                T xr = T(0);
                if (EPT < 4) xv[EPT < 4 ? EPT : 3] = right; else xr = right;
                first_trial(obj.staged(base + 2 * (size_t)TE + 2 * PAD, base + 3 * (size_t)TE + 2 * PAD, e0), i0, cnt, xv, xl, xr, r);
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        if (next_tile < ntl) stage_one(next_tile, stage);
        next_tile++;
        stage = (stage + 1 == stages) ? 0 : stage + 1;
    }
    if (FUSE)
    {
        const double dacc[5] = {(double)acc[0], (double)acc[1], (double)acc[2], (double)acc[3], (double)acc[4]};
        block_sums<5>(dacc, sh, dst, G);
    }
    else
    {
        const double dacc[1] = {(double)acc[0]};
        block_sums<1>(dacc, sh, dst, G);
    }
}

// ---- COMBINE (+ first trial), objectives without neighbour coupling --------------------------------------------------------------
// The same d and trial sums as p_combine.  The ring holds points, and a tile stages only the point rows of point_plan -- xc and the
// endpoints of the c pairs (c + 1 rows for a chained history, xc being the newest end).  v = grad f(xc) and the pairs are not stored:
// they are rebuilt with the arithmetic that formed them, y_j = grad f(x_end) - grad f(x_start), s_j = x_end - x_start, bit for bit the
// stored vectors.  The c + 1 gradient evaluations per unit are most of the pass's arithmetic, so the CTA's warps take a tile in two roles:
//     gradient warps   v = grad f(xc) and d = cv*v + sum_j cy_j*y_j (newest -> oldest, keeping the gradient of a pair's start, which
//                      is the next pair's end in a chained history) + sum_j cs_j*s_j (oldest -> newest), into a hand-off slot after
//                      the staging ring.  They work in `ng` groups, group k taking tiles k, k + ng, ... with a slot of its own.
//                      With 512 units per tile (fp64, m <= 4) the 8 spare warps are too few: ng = 0, and the owners form their units
//     owner warps      thread u owns unit u of every tile -- the thread that owned it when one thread did a unit's whole arithmetic,
//                      so each per-thread sum adds the same terms in the same order: stores d, adds v.d and, FUSE, the first trial
//                      at x1 = xc + 1*d
// (Also handing the s terms to the owners measured slower: 0.328 against 0.320 ms per round on config 2, DESIGN.md section 10.)
// Which thread computes a value does not change its bits, so d and the sums are those of one thread doing a unit's whole arithmetic.
// No CTA-wide barrier per tile: a stage has a full barrier (the bulk copies; parity in phase_bits) and an empty one (the owner warps,
// which read a tile after its gradient warps); a hand-off slot has a formed barrier (its gradient warps) and a free one (the owner
// warps).  Warp 0 re-arms a stage once its empty barrier completes.
template <class T, class OBJ, bool FUSE, class Between>
__device__ __forceinline__ void p_combine_points(const OBJ& obj, const Own& own, const PHist<T>& h, int c, T* tiles, T* __restrict__ res,
                                                 PShared& sh, unsigned& phase_bits, double* dst, int G, Between between)
{
    static_assert(!OBJ::kHalo, "neighbour-coupled objectives take p_combine");
    constexpr int EPT = 16 / (int)sizeof(T);
    constexpr int kMaxGroups = kPMaxStages - 1;                  // a group works ahead of the owners on a loaded stage: at most stages - 1 tiles
    __shared__ uint64_t empty_bar[kPMaxStages], formed_bar[kMaxGroups], free_bar[kMaxGroups];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int TE = h.BT();
    const int units = TE / EPT;                                  // 32 .. 512
    const int ow = (units + 31) / 32;                            // owner warps: 0 .. ow-1, one unit per thread
    const int spare = kPWarps - ow;
    const int gs = ow < spare ? ow : spare;                      // warps per gradient group
    int ng = spare < ow ? 0 : spare / gs;                        // 0: the owners form their own units (512 units: 8 spare warps are too few)
    ng = ng > kMaxGroups ? kMaxGroups : ng;
    const size_t stage_elems = (size_t)sh.npts * TE;
    int stages = (int)(((size_t)kPStageBytes / sizeof(T) - (size_t)ng * 2 * TE) / stage_elems);   // (>= 2: see bt_log in persist_host.cuh)
    stages = stages > kPMaxStages ? kPMaxStages : stages;
    ng = ng > stages - 1 ? stages - 1 : ng;
    T* const hand = tiles + (size_t)stages * stage_elems;       // slot k: v, d (TE elements each)
    const int64_t ntl = own.ntiles(TE);
    const T* s_coef = reinterpret_cast<const T*>(sh.coef);
    uint64_t* full_bar = sh.full_bar;
    const bool owner = warp < ow;
    const int grp = owner ? -1 : (warp - ow) / gs, gw = owner ? 0 : (warp - ow) % gs;

    T acc[5] = {T(0), T(0), T(0), T(0), T(0)};
    if (tid == 0)
    {
        for (int s = 0; s < stages; s++) mbar_init(&empty_bar[s], ow);
        for (int k = 0; k < ng; k++) { mbar_init(&formed_bar[k], gs); mbar_init(&free_bar[k], ow); }
    }
    __syncthreads();   // sh.vecs / point_plan are in place, the barriers initialised and the staging ring is free
    for (int s = 0; s < stages; s++)
        if (s < ntl) stage_points<T>(tiles + (size_t)s * stage_elems, TE, 0, 0, own.start(s, TE), own.len(s, TE), h, sh, &full_bar[s]);
    between();         // (ends with a barrier when it runs the recursion: sh.coef is in place)
    const unsigned full_phase = phase_bits;
    // v = grad f(xc) and d of one unit (lanes past cnt: x = 0), in the order of the recursion
    auto form = [&](const T* base, int64_t i0, int off, int cnt, Unit<T>& uv, Unit<T>& ud) {
        const T cv = s_coef[0];
        uv = grad_unit(obj, i0, cnt, lds_unit<T>(base + (size_t)sh.xrow * TE + off));
#pragma unroll
        for (int k = 0; k < EPT; k++) ud.v[k] = cv * uv.v[k];
        Unit<T> gk = uv;                                       // grad f of staged point row `kept`
        int kept = sh.xrow;
        for (int j = 0; j < c; j++)                            // y terms newest -> oldest
        {
            const int re = sh.pend[j], rs = sh.pstart[j];
            const Unit<T> ge = (re == kept) ? gk : grad_unit(obj, i0, cnt, lds_unit<T>(base + (size_t)re * TE + off));
            gk = grad_unit(obj, i0, cnt, lds_unit<T>(base + (size_t)rs * TE + off));
            kept = rs;
            const T cy = s_coef[1 + j];
#pragma unroll
            for (int k = 0; k < EPT; k++) ud.v[k] += cy * (ge.v[k] - gk.v[k]);
        }
#pragma unroll 4
        for (int j = c - 1; j >= 0; j--)                       // s terms oldest -> newest
        {
            const Unit<T> ue = lds_unit<T>(base + (size_t)sh.pend[j] * TE + off), us = lds_unit<T>(base + (size_t)sh.pstart[j] * TE + off);
            const T cs = s_coef[1 + c + j];
#pragma unroll
            for (int k = 0; k < EPT; k++) ud.v[k] += cs * (ue.v[k] - us.v[k]);
        }
    };
    if (owner)
    {
        for (int64_t t = 0; t < ntl; t++)
        {
            const int stage = (int)(t % stages), slot = ng ? (int)(t % ng) : 0;
            const unsigned lap = (unsigned)(t / stages) & 1u;
            const T* base = tiles + (size_t)stage * stage_elems;
            const T* xrow = base + (size_t)sh.xrow * TE;
            const T* hv = hand + (size_t)slot * 2 * TE;
            const int len = own.len(t, TE);
            const int64_t e0 = own.start(t, TE);
            mbar_wait(&full_bar[stage], ((full_phase >> stage) & 1u) ^ lap);
            if (ng) mbar_wait(&formed_bar[slot], (unsigned)(t / ng) & 1u);
            for (int off = tid * EPT; off < len; off += ow * 32 * EPT)
            {
                const int cnt = (len - off >= EPT) ? EPT : (len - off);
                Unit<T> uv, ud;
                if (ng) { uv = lds_unit<T>(hv + off); ud = lds_unit<T>(hv + TE + off); }
                else form(base, e0 + off, off, len - off, uv, ud);
#pragma unroll
                for (int k = 0; k < EPT; k++) acc[0] += (k < cnt) ? uv.v[k] * ud.v[k] : T(0);
                const int64_t i0 = e0 + off;
                st_unit<T>(res, i0, cnt, ud);
                if constexpr (FUSE)
                {
                    // the trial at x1 = xc + 1*d -> acc[1..4] (nothing stored: the pair-forming pass rebuilds the point if the search
                    // accepts it)
                    const Unit<T> ux = lds_unit<T>(xrow + off);
                    T xv[4] = {T(0), T(0), T(0), T(0)}, dv[EPT], gv[4];
#pragma unroll
                    for (int k = 0; k < EPT; k++)
                    {
                        xv[k] = (k < cnt) ? ux.v[k] + T(1) * ud.v[k] : T(0);
                        dv[k] = (k < cnt) ? ud.v[k] : T(0);
                    }
                    eval_pack(obj, i0, cnt, xv, T(0), T(0), dv, gv, acc + 1);
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // these reads before the bulk copies that re-arm the stage
            __syncwarp();
            if (lane == 0) { if (ng) mbar_arrive(&free_bar[slot]); mbar_arrive(&empty_bar[stage]); }
            if (warp == 0 && t + stages < ntl)
            {
                mbar_wait(&empty_bar[stage], lap);
                stage_points<T>(tiles + (size_t)stage * stage_elems, TE, 0, 0, own.start(t + stages, TE), own.len(t + stages, TE), h, sh,
                                &full_bar[stage]);
            }
        }
    }
    else if (grp < ng)
    {
        T* const hv = hand + (size_t)grp * 2 * TE;
        for (int64_t t = grp; t < ntl; t += ng)
        {
            const int stage = (int)(t % stages);
            const T* base = tiles + (size_t)stage * stage_elems;
            const int len = own.len(t, TE);
            const int64_t e0 = own.start(t, TE);
            // A parity wait is only right when the barrier's previous phase has completed.  The stage's previous occupant in this pass is
            // tile t - stages, which another group may have formed, so first wait until the owners are done with this slot's previous
            // tile t - ng: they have then waited on the full barrier of every tile up to t - ng >= t - stages + 1 (ng < stages).  For
            // t < ng this is the stage's first tile of the pass, and every earlier phase completed in an earlier pass.
            if (t >= ng) mbar_wait(&free_bar[grp], (unsigned)(t / ng - 1) & 1u);
            mbar_wait(&full_bar[stage], ((full_phase >> stage) & 1u) ^ ((unsigned)(t / stages) & 1u));
            for (int off = (gw * 32 + lane) * EPT; off < len; off += gs * 32 * EPT)
            {
                Unit<T> uv, ud;
                form(base, e0 + off, off, len - off, uv, ud);
                *reinterpret_cast<float4*>(hv + off) = *reinterpret_cast<const float4*>(uv.v);
                *reinterpret_cast<float4*>(hv + TE + off) = *reinterpret_cast<const float4*>(ud.v);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // these accesses before later bulk copies into this memory
            __syncwarp();
            if (lane == 0) mbar_arrive(&formed_bar[grp]);
        }
    }
    // the full barriers: one completed phase per tile a stage carried (every thread keeps the same parities, waiting or not)
    for (int s = 0; s < stages; s++)
        if (s < ntl) phase_bits ^= (unsigned)(((ntl - 1 - s) / stages + 1) & 1) << s;
    if (FUSE)
    {
        const double dacc[5] = {(double)acc[0], (double)acc[1], (double)acc[2], (double)acc[3], (double)acc[4]};
        block_sums<5>(dacc, sh, dst, G);
    }
    else
    {
        const double dacc[1] = {(double)acc[0]};
        block_sums<1>(dacc, sh, dst, G);
    }
    // (block_sums began with a barrier: every arrival on and wait for the pass's barriers is done)
    if (tid == 0)
    {
        for (int s = 0; s < stages; s++) mbar_inval(&empty_bar[s]);
        for (int k = 0; k < ng; k++) { mbar_inval(&formed_bar[k]); mbar_inval(&free_bar[k]); }
    }
}

// ---- waits with a watchdog ----------------------------------------------------------------------------------------------------
constexpr long long kPWaitCycles = 6000000000ll;   // default watchdog budget, ~3 s at 2 GHz: far beyond any legitimate wait (LBFGS_B200_WATCHDOG_SCALE multiplies it, e.g. under compute-sanitizer)

__device__ __forceinline__ unsigned ld_acquire_gpu_u32(const unsigned* p)
{
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu_u32(unsigned* p, unsigned v)
{
    asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

// n-words a pass has to move (reads + writes of whole vectors): the roofline numerator of the persistent kernel.  stored: the
// trials store their points, every pass reads the stored g and the ring holds the c pairs as 2c columns (neighbour-coupled
// objectives).  Otherwise g is evaluated from x wherever it is needed, only FIRST and MATERIALIZE write it, and the ring holds
// points: c chained pairs are c + 1 of them (a chain broken by the curvature gate stages up to c more, not counted here).  pt: the
// point a MATERIALIZE writes (PT_*); d_implied: the first search's d = -grad f(xp) is evaluated, not read
__device__ __forceinline__ double words_of(int op, int c, int data_vectors, bool stored, int pt, bool d_implied)
{
    const double dw = d_implied ? 0.0 : 1.0;
    switch (op)
    {
    case POP_FIRST: return (stored ? 3.0 : 2.0) + data_vectors;   // R x ; W g, d  /  R x ; W x to its point row
    case POP_TRIAL: return (stored ? 4.0 : 1.0 + dw) + data_vectors;   // R xp, d (; W x, g)
    case POP_RESTORE: return 4.0;                           // R xp, gp ; W x, g
    case POP_MATERIALIZE: return stored ? 4.0 : (pt == PT_RAY ? 3.0 + dw : 3.0);   // R xp, d / xp / x ; W x, g
    case POP_DOTS_FORM: return stored ? 2.0 * c + 4.0 : c + 1.0 + dw;   // R x, xp, g, gp, 2(c-1) columns ; W s, y  /  R d, c points ; W x
    case POP_DOTS_PLAIN: return stored ? 2.0 * c + 1.0 : c + 2.0;  // R g, 2c columns  /  R x, c + 1 points
    case POP_COMBINE: return stored ? 2.0 * c + 2.0 : c + 2.0;     // R g, 2c columns / c + 1 points ; W d
    case POP_COMBINE_TRIAL: return (stored ? 2.0 * c + 5.0 : c + 2.0) + data_vectors;   // R g, x, 2c columns / c + 1 points ; W d (, x1, g1)
    default: return 0.0;
    }
}

// Fixed-order sums of the CTAs' partials of every running problem into raw[], (optional) cross-rank exchange, scalar logic,
// publication of the next round's descriptors.  Called by all threads of CTA 0 once every CTA has arrived.  Returns (in every
// thread) the number of problems still running.
template <class T, bool HALO>
__device__ int leader_round(const PArgs<T>& a, int G, PShared& sh, PState<T>* cache)
{
    const int tid = threadIdx.x;
    // the leader's working copies: the first kPCache problems live in shared memory for the duration of the kernel
    auto state_of = [&](int b) -> PState<T>* { return b < kPCache ? cache + b : a.probs + b; };
    // 1. local sums: 16 threads per value (CTAs s, s+16, ... then a fixed shuffle tree), 48 values per sweep
    for (int b = 0; b < a.B; b++)
    {
        PState<T>* st = state_of(b);
        const int op = st->op;           // the pass this problem just ran (advance_problem below moves it on)
        if (op == POP_IDLE) continue;
        const int nv = nvals_of(st);
        const double* part = a.partials + (size_t)b * a.pstride * G;
        for (int v0 = 0; v0 < nv; v0 += kPThreads / 16)
        {
            const int v = v0 + tid / 16, sub = tid & 15;
            double t = 0.0;
            if (v < nv)
                for (int cta = sub; cta < G; cta += 16) t += __ldcg(part + (size_t)v * G + cta);
            t += __shfl_xor_sync(0xffffffffu, t, 8);
            t += __shfl_xor_sync(0xffffffffu, t, 4);
            t += __shfl_xor_sync(0xffffffffu, t, 2);
            t += __shfl_xor_sync(0xffffffffu, t, 1);
            if (v < nv && sub == 0) st->raw[v] = t;
        }
    }
    __syncthreads();
    // 2. n sharded over ranks: ONE exchange for all running problems (sums in rank order: identical bits on every rank)
    if (a.xc != nullptr)
    {
        const long long t_x0 = clock64();
        const XComm* xc = a.xc;
        const int me = xc->rank, R = xc->nranks;
        const unsigned long long epoch = a.ctl->epoch + 1ull;
        const int slot = (int)(epoch % kXRing);
        const unsigned tag = (unsigned)epoch;
        auto give_up = [&]() {
            if (clock64() - t_x0 > 4 * a.wait_cycles || ldv(&a.ctl->abort)) { a.ctl->abort = 1; return true; }
            return false;
        };
        // payload layout: problem after problem, nv sums then (HALO) 4 gathered boundary values.  Every value goes to every rank
        // (this one included) as two tagged 8-byte words: the receiver needs no flag and the sender no fence.
        int ofs = 0;
        for (int b = 0; b < a.B; b++)
        {
            PState<T>* st = state_of(b);
            const int op = st->op;
            if (op == POP_IDLE) continue;
            const int nv = nvals_of(st);
            for (int r = tid; r < R * nv; r += kPThreads)
                ll_push(xc->inbox[r / nv]->ll[slot][me][ofs + r % nv], st->raw[r % nv], tag);
            ofs += nv;
            if (HALO)
            {
                // boundary coordinates for the neighbours' next evaluations: the next search starts from the current x along drt
                if (tid < 4 * R)
                {
                    const int k = tid & 3;
                    const T* src = (k & 1) ? st->drt : st->x;
                    const double val = (double)__ldcg(src + ((k & 2) ? a.n - 1 : 0));
                    ll_push(xc->inbox[tid >> 2]->ll[slot][me][ofs + k], val, tag);
                }
                ofs += 4;
            }
        }
        __syncthreads();   // (raw[] is about to be overwritten with the global sums)
        ofs = 0;
        for (int b = 0; b < a.B; b++)
        {
            PState<T>* st = state_of(b);
            const int op = st->op;
            if (op == POP_IDLE) continue;
            const int nv = nvals_of(st);
            for (int k = tid; k < nv; k += kPThreads)
            {
                double t = 0.0;
                for (int r = 0; r < R; r++)           // rank order: identical bits on every rank
                {
                    double v = 0.0;
                    ll_pull(xc->inbox[me]->ll[slot][r][ofs + k], tag, v, give_up);
                    t += v;
                }
                st->raw[k] = t;
            }
            ofs += nv;
            if (HALO)
            {
                if ((op == POP_FIRST || op == POP_COMBINE || op == POP_COMBINE_TRIAL) && tid < 8)
                {
                    const int side = tid >> 2, k = tid & 3;       // side 0: left neighbour, 1: right neighbour
                    const int nb = side == 0 ? me - 1 : me + 1;
                    double v = 0.0;
                    if (nb >= 0 && nb < R) ll_pull(xc->inbox[me]->ll[slot][nb][ofs + k], tag, v, give_up);
                    st->halo[4 + 4 * side + k] = v;
                }
                ofs += 4;
            }
        }
        __syncthreads();
        if (tid == 0) { a.ctl->epoch = epoch; a.ctl->cyc_exchange += clock64() - t_x0; }
    }
    // 3. scalar logic, one thread per problem; the outcome goes into the problem's round descriptor
    int still = 0;
    for (int b0 = 0; b0 < a.B; b0 += kPThreads)
    {
        const int b = b0 + tid;
        int running = 0;
        if (b < a.B && state_of(b)->op != POP_IDLE)
        {
            PState<T>* st = state_of(b);
            advance_problem<T, HALO, !HALO, !HALO>(st, st->raw);
            PRound<T>* rd = a.rounds + b;
            rd->x = st->x; rd->xp = st->xp; rd->g = st->g; rd->gp = st->gp; rd->drt = st->drt;
            rd->step = st->step; rd->at_start = st->at_start;
            if (!HALO) { rd->px = st->px; rd->pxp = st->pxp; rd->d_implied = st->k == 1; }
            rd->c_round = st->c_round; rd->head = st->head; rd->pending = st->pending; rd->gram_cur = st->gram_cur;
            rd->op = st->op;
            running = st->op != POP_IDLE;
        }
        still += __syncthreads_count(running);
    }
    if (tid == 0) { a.ctl->nactive = still; a.ctl->rounds++; }
    return still;
}

// exchange-only prelude for neighbour-coupled objectives under n-sharding: the first evaluation needs the neighbours' boundary
// coordinates of x0 (later rounds piggyback the boundaries of (x, drt) on the sums, see leader_round).  All threads of CTA 0.
template <class T> __device__ void leader_halo_prelude(const PArgs<T>& a)
{
    const int tid = threadIdx.x;
    const XComm* xc = a.xc;
    const int me = xc->rank, R = xc->nranks;
    const unsigned long long epoch = a.ctl->epoch + 1ull;
    const int slot = (int)(epoch % kXRing);
    const unsigned tag = (unsigned)epoch;
    const long long t_x0 = clock64();
    auto give_up = [&]() {
        if (clock64() - t_x0 > 4 * a.wait_cycles || ldv(&a.ctl->abort)) { a.ctl->abort = 1; return true; }
        return false;
    };
    for (int b = 0; b < a.B; b++)
    {
        PState<T>* st = a.probs + b;
        if (tid < 4 * R)
        {
            const int k = tid & 3;
            const double val = (k & 1) ? 0.0 : (double)__ldcg(st->x + ((k & 2) ? a.n - 1 : 0));
            ll_push(xc->inbox[tid >> 2]->ll[slot][me][4 * b + k], val, tag);
        }
    }
    for (int b = 0; b < a.B; b++)
    {
        PState<T>* st = a.probs + b;
        if (tid < 8)
        {
            const int side = tid >> 2, k = tid & 3;
            const int nb = side == 0 ? me - 1 : me + 1;
            double v = 0.0;
            if (nb >= 0 && nb < R) ll_pull(xc->inbox[me]->ll[slot][nb][4 * b + k], tag, v, give_up);
            st->halo[4 + 4 * side + k] = v;
        }
    }
    __syncthreads();
    if (tid == 0) a.ctl->epoch = epoch;
}

// ---- the kernel ----------------------------------------------------------------------------------------------------------------
template <class T, class OBJ, int ROUNDS>
__global__ void __launch_bounds__(kPThreads, 1) k_persist(PArgs<T> a)
{
    extern __shared__ __align__(128) unsigned char p_smem[];
    T* tiles = reinterpret_cast<T*>(p_smem);      // the staging ring of the dots / combination passes
    __shared__ PShared sh;
    const int tid = threadIdx.x, G = gridDim.x, cta = blockIdx.x;
    const Own own(a.n, G, cta, a.grain);
    if (tid == 0)
    {
        for (int s = 0; s < kPMaxStages; s++) mbar_init(&sh.full_bar[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    unsigned phase_bits = 0;
    unsigned episode = 0;    // grid-barrier episodes so far
    constexpr bool HALO = OBJ::kHalo;
    constexpr int kDataVectors = OBJ::kDataVectors;
    long long t_last = clock64(), t_arrive = 0;   // CTA 0, thread 0: accounting (PCtl::cyc_*)
    int acct_bucket = 0;
    double acct_words = 0.0;
    __shared__ unsigned s_release;
    __shared__ __align__(16) double s_gram[kPGramScratch];   // the coefficient recursion's own scratch (c <= 21: it then runs while the first tiles of the pass are in flight)
    __shared__ PState<T> s_state[kPCache];     // CTA 0: working copies of the first problems' states (scalar logic at shared-memory latency)
    const int ncache = a.B < kPCache ? a.B : kPCache;
    if (cta == 0)
    {
        const unsigned* src = reinterpret_cast<const unsigned*>(a.probs);
        unsigned* dstw = reinterpret_cast<unsigned*>(s_state);
        for (int w = tid; w < (int)(sizeof(PState<T>) / 4) * ncache; w += kPThreads) dstw[w] = src[w];
        __syncthreads();
    }

    // Grid-wide barrier.  Arrival: the CTA's partial sums are written, bar.sync, thread 0 fences and counts in.  Between the last
    // arrival and the release CTA 0 runs `leader_work` (all its threads; returns true when nothing is left to do).  Returns that
    // verdict in every thread of every CTA (it travels in bit 31 of the release word).
    auto grid_barrier = [&](auto leader_work) -> bool {
        episode++;
        asm volatile("fence.proxy.async;" ::: "memory");   // this round's generic-proxy stores before later bulk (async-proxy) reads
        if (HALO) __threadfence();                           // boundary coordinates are read by the neighbouring CTA next round
        __syncthreads();
        if (tid == 0) { __threadfence(); atomicAdd(&a.ctl->arrive, 1u); }
        if (cta == 0)
        {
            if (tid == 0)
            {
                const long long t_start = clock64();
                t_arrive = t_start;
                while (ld_acquire_gpu_u32(&a.ctl->arrive) != episode * (unsigned)G)
                    if (clock64() - t_start > a.wait_cycles || ldv(&a.ctl->abort)) { a.ctl->abort = 1; break; }
                a.ctl->cyc_wait_all += clock64() - t_start;
            }
            __syncthreads();
            const bool stop = leader_work();
            __syncthreads();
            if (tid == 0)
            {
                const long long now = clock64();
                a.ctl->cyc_op[acct_bucket] += now - t_last;
                a.ctl->cyc_sync += now - t_arrive;
                a.ctl->n_op[acct_bucket] += 1ull;
                a.ctl->words_op[acct_bucket] += acct_words;
                t_last = now;
                st_release_gpu_u32(&a.ctl->release, episode | (stop ? kPStopBit : 0u));
            }
        }
        if (tid == 0)
        {
            const long long t_start = clock64();
            unsigned v;
            while (((v = ld_acquire_gpu_u32(&a.ctl->release)) & ~kPStopBit) < episode)
                if (clock64() - t_start > 6 * a.wait_cycles || ldv(&a.ctl->abort)) { a.ctl->abort = 1; v = kPStopBit; break; }
            s_release = v;
        }
        __syncthreads();
        return (s_release & kPStopBit) != 0u;
    };

    if (HALO && a.xc != nullptr)
        if (grid_barrier([&]() { leader_halo_prelude<T>(a); return ldv(&a.ctl->abort) != 0; })) return;

    for (;;)
    {
        // this round's op of every problem (the descriptors were published before the release that let us through)
        if (a.B > 1)
        {
            for (int b = tid; b < a.B; b += kPThreads) sh.ops[b] = (unsigned char)ldv(&a.rounds[b].op);
            __syncthreads();
        }
        acct_bucket = -1;
        acct_words = 0.0;
        for (int b = 0; b < a.B; b++)
        {
            const PRound<T>* rd = a.rounds + b;
            if (a.B > 1 && sh.ops[b] == POP_IDLE) continue;
            // a single problem: the op travels with the rest of the descriptor, and all its fields are requested before the first one is
            // looked at (one trip to L2 per round instead of two)
            const int op = (a.B > 1) ? (int)sh.ops[b] : ldv(&rd->op);
            const PState<T>* st = a.probs + b;     // fields that are fixed for the duration of the kernel only
            T* const vx = ldv(&rd->x); T* const vxp = ldv(&rd->xp); T* const vg = ldv(&rd->g); T* const vgp = ldv(&rd->gp); T* const vd = ldv(&rd->drt);
            const T step = ldv(&rd->step);
            const int c_round = ldv(&rd->c_round), head = ldv(&rd->head), pending = ldv(&rd->pending), gram_cur = ldv(&rd->gram_cur);
            const int at_start = ldv(&rd->at_start);
            const int px = HALO ? 0 : ldv(&rd->px), pxp = HALO ? 0 : ldv(&rd->pxp);
            const bool d_implied = HALO ? false : ldv(&rd->d_implied) != 0;
            if (op == POP_IDLE) continue;
            acct_bucket = (acct_bucket == -1 || acct_bucket == op) ? op : 0;
            acct_words += words_of(op, c_round, kDataVectors, HALO, at_start, d_implied);
            double* dst = a.partials + (size_t)b * a.pstride * G + cta;
            const OBJ obj{ObjGeom<T>{a.n, a.index_offset, a.n_global, (HALO && a.xc != nullptr) ? st->halo : nullptr, st->data0, st->data1}};
            switch (op)
            {
            case POP_FIRST:
                if constexpr (HALO) p_trial_halo<T, OBJ, 0>(obj, own, nullptr, nullptr, T(0), vx, vg, vd, tiles, sh, phase_bits, dst, G);
                else p_trial<T, OBJ, 0>(obj, own, st->hist, 0, nullptr, T(0), vx, nullptr, px, sh, dst, G, a.evict_first_stores);
                break;
            case POP_TRIAL:
                if constexpr (HALO) p_trial_halo<T, OBJ, 1>(obj, own, vxp, vd, step, vx, vg, nullptr, tiles, sh, phase_bits, dst, G);
                else p_trial<T, OBJ, 1>(obj, own, st->hist, pxp, vd, step, nullptr, nullptr, 0, sh, dst, G, a.evict_first_stores, d_implied);
                break;
            case POP_RESTORE:
                p_restore<T>(own, vxp, vgp, vx, vg);
                break;
            case POP_MATERIALIZE:
                if constexpr (!HALO)
                {
                    if (at_start == PT_RAY) p_trial<T, OBJ, 2>(obj, own, st->hist, pxp, vd, step, vx, vg, 0, sh, dst, G, a.evict_first_stores, d_implied);
                    else   // PT_START: x = xp ; PT_X: x = x (its point row) ; g = grad f(x)
                        p_trial<T, OBJ, 3>(obj, own, st->hist, at_start == PT_START ? pxp : px, nullptr, T(0), vx, vg, 0, sh, dst, G, a.evict_first_stores);
                }
                break;
            case POP_DOTS_FORM:
            case POP_DOTS_PLAIN:
            {
                const bool form = op == POP_DOTS_FORM;
                PDots<T> d;
                d.n = a.n; d.h = st->hist; d.c = c_round;
                d.end = head;                                   // the old columns: the slots below the free slot `head`
                d.cnt_old = form ? c_round - 1 : c_round;
                d.new_slot = form ? head : -1;
                d.step = step; d.at_start = at_start; d.px = px; d.d_implied = d_implied;
                dots_geometry(d.c, d.h.BT() / (16 / (int)sizeof(T)), d.split, d.cols_per_round);
                __syncthreads();   // sh.slots / sh.vecs may still be read by the previous problem's pass
                if constexpr (!HALO)
                {
                    // the point is rebuilt from d and xp / g from x; the old pairs (FORM: columns 1..) from their endpoints
                    if (tid == 0) sh.vecs[0] = vd;
                    point_plan<T>(st, head, d.cnt_old, form ? 1 : 0, form ? pxp : px, sh);
                }
                else
                {
                    const SlotRuns runs(d.end, d.cnt_old, d.h.M);
                    // age j (FORM: j >= 1) -> packed row of its slot in the staged block
                    if (tid < d.c && !(form && tid == 0))
                        sh.slots[tid] = (unsigned char)runs.row_of(slot_by_age(head, d.h.M, form ? tid - 1 : tid));
                    if (tid == 0) { sh.vecs[0] = vg; sh.vecs[1] = vx; sh.vecs[2] = vgp; sh.vecs[3] = vxp; }
                }
                if (form) p_dots<T, OBJ, ROUNDS, true>(d, obj, own, tiles, sh, phase_bits, dst, G);
                else p_dots<T, OBJ, ROUNDS, false>(d, obj, own, tiles, sh, phase_bits, dst, G);
                break;
            }
            case POP_COMBINE:
            case POP_COMBINE_TRIAL:
            {
                GramSolveArgs<T> g;
                g.c = c_round;
                g.M = st->hist.M; g.new_slot = pending; g.with_v = 1; g.a = T(-1);
                g.raw = st->raw;
                const int in = gram_cur, out = (g.new_slot >= 0) ? 1 - in : in;
                g.SY_in = st->SY[in]; g.YY_in = st->YY[in]; g.SS_in = st->SS[in];
                g.SY_out = st->SY[out]; g.YY_out = st->YY[out]; g.SS_out = st->SS[out];
                g.ys = st->ys; g.alpha = st->alpha; g.theta = st->theta;
                for (int age = 0; age < g.c; age++) g.slots[age] = (unsigned char)slot_by_age(head, g.M, age);
                __syncthreads();   // the tile area / tables may still be in use by the previous problem's pass
                // per age: packed row of the column in a staged block, and its ring slot
                const bool fuse = op == POP_COMBINE_TRIAL;
                if constexpr (!HALO) point_plan<T>(st, head, g.c, 0, px, sh);   // g is evaluated from x, the pairs from their endpoints
                else
                {
                    const SlotRuns runs(head, g.c, g.M);
                    for (int j = tid; j < g.c; j += kPThreads)
                    {
                        sh.slots[j] = (unsigned char)runs.row_of(g.slots[j]);
                        sh.slotid[j] = g.slots[j];
                    }
                    if (tid == 0) { sh.vecs[0] = vg; sh.vecs[1] = vx; sh.vecs[2] = st->data0; sh.vecs[3] = st->data1; }
                }
                // the coefficient recursion (every CTA; CTA 0 also writes the folded Gram matrices back) and its 2c+1 results into sh.coef
                const bool own_scratch = gram_solve_smem_elems(g.c) * sizeof(T) <= sizeof(s_gram);
                auto solve_into = [&](T* scratch) {
                    gram_solve_in_smem<T>(g, scratch, cta == 0);
                    const T* s_coef = scratch + 2 * g.c * g.c;
                    T* keep = reinterpret_cast<T*>(sh.coef);
                    for (int q = tid; q < 2 * g.c + 1; q += kPThreads) keep[q] = s_coef[q];
                    __syncthreads();
                };
                if (!own_scratch) solve_into(tiles);   // a long history: the staging ring is the scratch, the copies start afterwards
                auto between = [&]() { if (own_scratch) solve_into(reinterpret_cast<T*>(s_gram)); };
                if constexpr (!HALO)
                {
                    if (fuse) p_combine_points<T, OBJ, true>(obj, own, st->hist, g.c, tiles, vd, sh, phase_bits, dst, G, between);
                    else p_combine_points<T, OBJ, false>(obj, own, st->hist, g.c, tiles, vd, sh, phase_bits, dst, G, between);
                }
                else if (fuse) p_combine<T, OBJ, true, true>(obj, own, st->hist, g.c, head, tiles, vd, vxp, vgp, sh, phase_bits, dst, G, between);
                else p_combine<T, OBJ, false, false>(obj, own, st->hist, g.c, head, tiles, vd, nullptr, nullptr, sh, phase_bits, dst, G, between);
                break;
            }
            default: break;
            }
        }
        if (acct_bucket < 0) acct_bucket = 0;
        if (grid_barrier([&]() { return leader_round<T, HALO>(a, G, sh, s_state) == 0 || ldv(&a.ctl->abort) != 0; })) break;
    }
    if (cta == 0)
    {
        __syncthreads();
        const unsigned* src = reinterpret_cast<const unsigned*>(s_state);
        unsigned* dstw = reinterpret_cast<unsigned*>(a.probs);
        for (int w = tid; w < (int)(sizeof(PState<T>) / 4) * ncache; w += kPThreads) dstw[w] = src[w];
    }
}

}  // namespace lb
