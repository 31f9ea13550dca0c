// small_batch.cuh -- many small L-BFGS problems in one launch: LBFGSSolver::minimize() (reference LBFGS.h:78-173) for B independent
// problems of a built-in objective, one thread block (CTA) per problem, the whole solve in that CTA's shared memory.
// Included by small_batch.cu.
//
// The device-resident solve (persist.cuh) spreads one pass of a problem over every SM and separates rounds by grid-wide barriers;
// below a few thousand coordinates it has nothing to spread, and a batch of such problems runs one after another on one SM.  Here a
// CTA runs one problem's whole minimize() with nobody to wait for: an ordinary launch of B CTAs (they run in waves), no grid
// barrier, no atomics, no watchdog.  HBM is read once (x0 and the problem's data vectors) and written once (x and, optionally, g).
//
// The scalar side is the resident solve's own: PState, the POP_* ops and advance_problem of problem_machine.cuh.  The CTA loops
//     run the pass for st->op over the vectors in shared memory -> reduce its nvals_of(st) values into raw[] -> thread 0 calls
//     advance_problem -> __syncthreads
// until the op is POP_IDLE.  The passes are the resident ones restated for one CTA over on-chip vectors: FIRST, TRIAL and
// MATERIALIZE with the resident solve's implied-point rule (a trial of an objective without neighbour coupling stores nothing; the
// pair-forming pass rebuilds the accepted point with the trial's arithmetic), DOTS_FORM / DOTS_PLAIN in k_gram_dots' layout
// (kGramVals values per column pair), COMBINE(_TRIAL) with the coefficient recursion of gram_solve_in_smem, RESTORE for the
// neighbour-coupled objectives, whose trials store their points and keep the best one in x_lo / g_lo.  The first trial of every
// search always rides on the combination pass.
//
// Determinism.  A CTA has small_threads(n) threads: one warp up to n = 128, four warps above.  A thread owns the packs of 4
// coordinates q = tid, tid + nt, ... and accumulates them in index order (in T, as the resident passes do); the block sum is a fixed
// shuffle tree per warp and the warp totals added in warp order, in double for both precisions.  So a problem's result depends on n
// (and the precision) only -- not on B, nor on where the problem sits in the batch.  It is not bit-identical to LBFGSSolver's resident
// solve or to LBFGSBatchSolver, whose sums are associated across CTAs; the decisions follow the same code, the sums differ by rounding.
//
// Shared memory of one CTA (byte offsets: small_layout; the budget in include/lbfgs_b200.h):
//     [ PState + slot table: kSStateBytes ][ raw: p doubles ][ red: kSMaxWarps x p doubles ][ ys M | alpha M | theta (4) | SY,YY,SS x2:
//     6 M^2 ][ recursion scratch: gram_solve_smem_elems(m) ][ vectors, ld = round_up(n, 4) elements each: x xp g gp d, S/Y of slot 0..M-1,
//     (x_lo g_lo), (data0 data1) ]          with M = m + 1 ring slots and p = round_up(max(6m, 8), 8)
#pragma once

#include "../../include/LBFGSpp/CompactForm.h"
#include "problem_machine.cuh"
#include "philox.cuh"

namespace lb {

constexpr int kSMaxThreads = 128;
constexpr int kSMaxWarps = kSMaxThreads / 32;
constexpr size_t kSStateBytes = 2048;          // the problem's PState and its slot table
constexpr size_t kSSmemLimit = 232448;         // largest dynamic shared memory of one CTA on sm_90 (227 KB)
static_assert(sizeof(PState<double>) + kMaxM <= kSStateBytes && sizeof(PState<float>) + kMaxM <= kSStateBytes, "state region");

// threads per CTA: a fixed function of n, so that a problem's sums never depend on anything else
__host__ __device__ inline int small_threads(int64_t n) { return n <= 128 ? 32 : kSMaxThreads; }

struct SmallLayout
{
    size_t raw, red, small, gram, vecs, total;   // byte offsets (the state is at 0)
    int64_t ld;                                   // elements per vector
    int pstride, nvec;
};
inline size_t small_align16(size_t b) { return (b + 15) & ~size_t(15); }
inline SmallLayout small_layout(int64_t n, int m, int elem, bool stored, int data_vectors)
{
    SmallLayout L;
    const size_t M = (size_t)m + 1;
    L.ld = (n + 3) & ~int64_t(3);
    L.pstride = ((m * kGramVals > 8 ? m * kGramVals : 8) + 7) & ~7;
    L.nvec = 5 + 2 * (int)M + (stored ? 2 : 0) + data_vectors;
    L.raw = kSStateBytes;
    L.red = L.raw + sizeof(double) * (size_t)L.pstride;
    L.small = L.red + sizeof(double) * (size_t)kSMaxWarps * L.pstride;
    L.gram = L.small + small_align16((size_t)elem * (2 * M + 4 + 6 * M * M));
    L.vecs = L.gram + small_align16((size_t)elem * gram_solve_smem_elems(m));
    L.total = L.vecs + (size_t)elem * (size_t)L.nvec * (size_t)L.ld;
    return L;
}

// The final history of one problem as kept for the products (lbfgs_b200_small_hist): c = its pair count <= m, every block by age
// (0 = newest pair), T elements from the problem's record start: s_a at a*n, y_a at (m + a)*n, ys_a, the c x c Gram blocks S'Y, Y'Y,
// S'S (row-major, leading dimension c), theta.  rec = 2m*n + m + 3m^2 + 2 elements per problem.
struct SmallHistLayout
{
    int64_t n;
    int m;
    __host__ __device__ int64_t s(int age) const { return age * n; }
    __host__ __device__ int64_t y(int age) const { return (m + age) * n; }
    __host__ __device__ int64_t ys() const { return 2 * m * n; }
    __host__ __device__ int64_t SY() const { return ys() + m; }
    __host__ __device__ int64_t YY() const { return SY() + (int64_t)m * m; }
    __host__ __device__ int64_t SS() const { return YY() + (int64_t)m * m; }
    __host__ __device__ int64_t theta() const { return SS() + (int64_t)m * m; }
    __host__ __device__ int64_t rec() const { return theta() + 2; }
};

template <class T> struct SmallArgs
{
    const PState<T>* proto;     // options and initial ring / op (init_problem_state), the same for every problem (device memory)
    int M;                      // ring slots: m + 1
    SmallLayout L;
    int64_t n;
    const T *data0, *data1;     // problem b's data at data + b*ldd (ldd = 0: shared)
    int64_t ldd;
    T* X;                       // problem b: X + b*ldx (start point in, solution out)
    int64_t ldx;
    T* G;                       // optional: final gradients, same layout as X
    lbfgs_b200_outcome* outs;   // [B]
    T* hist;                    // optional: the final history of problem b at hist + b*SmallHistLayout::rec (see there)
    int* hist_c;                // [B] with hist: its pair count
};

// block sums of NV per-thread values -> raw[0..NV): a fixed shuffle tree per warp, warp totals in warp order.  All threads call.
template <int NV> __device__ __forceinline__ void small_sums(const double (&v)[NV], double* red, int ps, double* raw)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; k++)
    {
        const double w = warp_sum(v[k]);
        if (lane == 0) red[warp * ps + k] = w;
    }
    __syncthreads();
    if (threadIdx.x < NV)
    {
        double t = 0.0;
        for (int w = 0; w < nw; w++) t += red[w * ps + threadIdx.x];
        raw[threadIdx.x] = t;
    }
}

// the export after the solve, out of line so that it leaves the solve loop's register allocation alone
template <class T>
__device__ __noinline__ void small_export_history(const PState<T>* st, const T* ring, int64_t ld, T* rec, int* c_out, int64_t n)
{
    const int tid = threadIdx.x, nt = blockDim.x, M = st->M;
    const SmallHistLayout HL{n, M - 1};
    const int c = st->ncorr, head = st->head, cur = st->gram_cur;
    for (int age = 0; age < c; age++)
    {
        const T* sj = ring + 2 * (int64_t)slot_by_age(head, M, age) * ld;
        const T* yj = sj + ld;
        for (int64_t i = tid; i < n; i += nt) { rec[HL.s(age) + i] = sj[i]; rec[HL.y(age) + i] = yj[i]; }
    }
    for (int idx = tid; idx < c * c; idx += nt)
    {
        const int pi = slot_by_age(head, M, idx / c), pj = slot_by_age(head, M, idx % c);
        rec[HL.SY() + idx] = st->SY[cur][pi * M + pj];
        rec[HL.YY() + idx] = st->YY[cur][pi * M + pj];
        rec[HL.SS() + idx] = st->SS[cur][pi * M + pj];
    }
    for (int age = tid; age < c; age += nt) rec[HL.ys() + age] = st->ys[slot_by_age(head, M, age)];
    if (tid == 0)
    {
        rec[HL.theta()] = *st->theta;
        *c_out = c;
    }
}

template <class T, class OBJ>
__global__ void __launch_bounds__(kSMaxThreads) k_small_batch(const SmallArgs<T> a)
{
    extern __shared__ __align__(16) unsigned char s_smem[];
    constexpr bool STORED = OBJ::kHalo;          // neighbour-coupled objectives: trials store their points
    constexpr int DV = OBJ::kDataVectors;
    const int tid = threadIdx.x, nt = blockDim.x;
    const int64_t b = blockIdx.x, n = a.n, ld = a.L.ld;
    const int64_t npacks = (n + 3) >> 2;
    const int M = a.M, ps = a.L.pstride;
    PState<T>* st = reinterpret_cast<PState<T>*>(s_smem);
    unsigned char* s_slot = s_smem + sizeof(PState<T>);   // by age: physical ring slot (combination pass)
    double* raw = reinterpret_cast<double*>(s_smem + a.L.raw);
    double* red = reinterpret_cast<double*>(s_smem + a.L.red);
    T* small = reinterpret_cast<T*>(s_smem + a.L.small);
    T* gram = reinterpret_cast<T*>(s_smem + a.L.gram);
    T* vec = reinterpret_cast<T*>(s_smem + a.L.vecs);
    T* const ring = vec + 5 * ld;                            // S of slot k at ring + 2k*ld, Y of slot k right after it
    T* const sdata = ring + (2 * M + (STORED ? 2 : 0)) * ld;
    auto s_col = [&](int slot) { return ring + 2 * (int64_t)slot * ld; };

    // ---- the problem's state, history and vectors ----
    {
        const unsigned* src = reinterpret_cast<const unsigned*>(a.proto);
        unsigned* dst = reinterpret_cast<unsigned*>(st);
        for (int w = tid; w < (int)(sizeof(PState<T>) / 4); w += nt) dst[w] = src[w];
    }
    const size_t small_elems = (size_t)2 * M + 4 + 6 * (size_t)M * M;
    for (size_t i = tid; i < small_elems; i += nt) small[i] = T(0);   // BFGSMat::reset (BFGSMat.h:61-78): no pairs, Gram cleared
    for (int64_t i = tid; i < (int64_t)a.L.nvec * ld; i += nt) vec[i] = T(0);   // (lanes past n stay 0 in every vector)
    __syncthreads();
    if (tid == 0)
    {
        const size_t mm = (size_t)M * M;
        st->x = vec; st->xp = vec + ld; st->g = vec + 2 * ld; st->gp = vec + 3 * ld; st->drt = vec + 4 * ld;
        st->x_lo = STORED ? ring + 2 * M * ld : nullptr;
        st->g_lo = STORED ? ring + (2 * M + 1) * ld : nullptr;
        st->hist.H = ring; st->hist.M = M; st->hist.bt_log = 0; st->hist.bstride = 0;   // (the ring is addressed through s_col)
        st->ys = small; st->alpha = small + M; st->theta = small + 2 * M;
        for (int k = 0; k < 2; k++) { st->SY[k] = small + 2 * M + 4 + (3 * k + 0) * mm; st->YY[k] = small + 2 * M + 4 + (3 * k + 1) * mm; st->SS[k] = small + 2 * M + 4 + (3 * k + 2) * mm; }
        st->data0 = DV ? sdata : nullptr;
        st->data1 = DV ? sdata + ld : nullptr;
        st->raw = raw; st->halo = nullptr; st->trace = nullptr; st->trace_cap = 0;
        *st->theta = T(1);
    }
    {
        const T* x0 = a.X + b * a.ldx;
        for (int64_t i = tid; i < n; i += nt) vec[i] = x0[i];
        if constexpr (DV == 2)
        {
            const T* d0 = a.data0 + b * a.ldd;
            const T* d1 = a.data1 + b * a.ldd;
            for (int64_t i = tid; i < n; i += nt) { sdata[i] = d0[i]; sdata[ld + i] = d1[i]; }
        }
    }
    // neighbours straight from shared memory: no index offset, the whole vector, no halo
    const OBJ obj{ObjGeom<T>{n, 0, n, nullptr, DV ? sdata : nullptr, DV ? sdata + ld : nullptr}};

    for (;;)
    {
        __syncthreads();   // the state thread 0 left, and every vector of the last pass
        const int op = st->op;
        if (op == POP_IDLE) break;
        T* const x = st->x; T* const xp = st->xp; T* const g = st->g; T* const gp = st->gp; T* const d = st->drt;
        const T step = st->step;
        const int at_start = st->at_start, c = st->c_round, head = st->head;
        switch (op)
        {
        // FIRST: g = grad f(x), d = -g ; {f, g.d (= 0), g.g, x.x}.  TRIAL: x = xp + step*d, g = grad f(x) ; {f, g.d, g.g, x.x}, stored
        // only by the neighbour-coupled objectives.  MATERIALIZE: x = xp + step*d, g = grad f(x), stored; no sums.
        case POP_FIRST:
        case POP_TRIAL:
        case POP_MATERIALIZE:
        {
            if (op == POP_MATERIALIZE && at_start)
            {
                for (int64_t i = tid; i < n; i += nt) { x[i] = xp[i]; g[i] = gp[i]; }
                break;
            }
            const bool first = op == POP_FIRST;
            const bool store = first || STORED || op == POP_MATERIALIZE;
            T acc[4] = {T(0), T(0), T(0), T(0)};
            for (int64_t q = tid; q < npacks; q += nt)
            {
                const int64_t i0 = q << 2;
                const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
                T xv[4], dv[4], gv[4], xl = T(0), xr = T(0);
#pragma unroll
                for (int k = 0; k < 4; k++)
                {
                    dv[k] = (!first && k < cnt) ? d[i0 + k] : T(0);
                    xv[k] = (k < cnt) ? (first ? x[i0 + k] : xp[i0 + k] + step * d[i0 + k]) : T(0);
                }
                if constexpr (OBJ::kHalo)
                {
                    if (first) pack_neighbours<false>(obj, i0, n, step, [&](int j) { return x[i0 + j]; }, xl, xr);
                    else pack_neighbours<true>(obj, i0, n, step, [&](int j) { return xp[i0 + j] + step * d[i0 + j]; }, xl, xr);
                }
                eval_pack(obj, i0, cnt, xv, xl, xr, dv, gv, acc);
                if (store)
                {
#pragma unroll
                    for (int k = 0; k < 4; k++)
                        if (k < cnt)
                        {
                            g[i0 + k] = gv[k];
                            if (first) d[i0 + k] = T(-1) * gv[k];
                            else x[i0 + k] = xv[k];
                        }
                }
            }
            if (op == POP_MATERIALIZE) break;
            const double dacc[4] = {(double)acc[0], (double)acc[1], (double)acc[2], (double)acc[3]};
            small_sums<4>(dacc, red, ps, raw);
            break;
        }
        case POP_RESTORE:
            for (int64_t i = tid; i < n; i += nt) { x[i] = xp[i]; g[i] = gp[i]; }
            break;
        // [S Y]'[g s_new y_new], kGramVals values per column pair, by age.  FORM: the new pair s = x - xp, y = g - gp goes into ring slot
        // `head` and takes part as column 0; an implied point is rebuilt first (the trial's arithmetic) and written to (x, g).
        // PLAIN: s.g and y.g of the old columns only.  A thread only touches its own packs, so no barrier is needed in between.
        case POP_DOTS_FORM:
        case POP_DOTS_PLAIN:
        {
            const bool form = op == POP_DOTS_FORM;
            T* const sn = s_col(head);
            T* const yn = sn + ld;
            if (form)
                for (int64_t q = tid; q < npacks; q += nt)
                {
                    const int64_t i0 = q << 2;
                    const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
                    if (!STORED)
                    {
                        T xv[4], gv[4];
                        if (at_start)
                        {
#pragma unroll
                            for (int k = 0; k < 4; k++) { xv[k] = (k < cnt) ? xp[i0 + k] : T(0); gv[k] = (k < cnt) ? gp[i0 + k] : T(0); }
                        }
                        else
                        {
#pragma unroll
                            for (int k = 0; k < 4; k++) xv[k] = (k < cnt) ? xp[i0 + k] + step * d[i0 + k] : T(0);
                            obj.eval(i0, cnt, xv, T(0), T(0), gv);
                        }
#pragma unroll
                        for (int k = 0; k < 4; k++)
                            if (k < cnt) { x[i0 + k] = xv[k]; g[i0 + k] = gv[k]; }
                    }
#pragma unroll
                    for (int k = 0; k < 4; k++)
                        if (k < cnt) { sn[i0 + k] = x[i0 + k] - xp[i0 + k]; yn[i0 + k] = g[i0 + k] - gp[i0 + k]; }
                }
            for (int j = 0; j < c; j++)
            {
                const int slot = form ? (j == 0 ? head : slot_by_age(head, M, j - 1)) : slot_by_age(head, M, j);
                const T* sj = s_col(slot);
                const T* yj = sj + ld;
                T acc[kGramVals] = {T(0), T(0), T(0), T(0), T(0), T(0)};
                for (int64_t q = tid; q < npacks; q += nt)
                {
                    const int64_t i0 = q << 2;
                    const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
#pragma unroll
                    for (int k = 0; k < 4; k++)
                        if (k < cnt)
                        {
                            const int64_t i = i0 + k;
                            const T s = sj[i], y = yj[i], v = g[i];
                            acc[0] += s * v;
                            acc[1] += y * v;
                            if (form)
                            {
                                const T ynew = yn[i], snew = sn[i];
                                acc[2] += s * ynew;
                                acc[3] += y * ynew;
                                acc[4] += y * snew;
                                acc[5] += s * snew;
                            }
                        }
                }
                const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
                for (int k = 0; k < kGramVals; k++)
                {
                    const double w = warp_sum((double)acc[k]);
                    if (lane == 0) red[warp * ps + j * kGramVals + k] = w;
                }
            }
            __syncthreads();
            for (int idx = tid; idx < c * kGramVals; idx += nt)
            {
                double t = 0.0;
                for (int w = 0; w < (nt >> 5); w++) t += red[w * ps + idx];
                raw[idx] = t;
            }
            break;
        }
        // d = -H g by the coefficient recursion (gram_solve_in_smem, which also folds the new pair into the Gram matrices) and one
        // combination d = cv*g + sum_j cy_j y_j + cs_j s_j (y newest -> oldest, then s oldest -> newest) ; {g.d}.  COMBINE_TRIAL: the
        // first trial of the next search, x1 = x + d, in the same pass ; {g.d, f1, g1.d, g1.g1, x1.x1}; the neighbour-coupled objectives
        // write x1, g1 to (xp, gp), which the rotation of begin_search turns into (x, g).
        case POP_COMBINE:
        case POP_COMBINE_TRIAL:
        {
            const bool fuse = op == POP_COMBINE_TRIAL;
            GramSolveArgs<T> ga;
            ga.c = c; ga.M = M; ga.new_slot = st->pending; ga.with_v = 1; ga.a = T(-1);
            ga.raw = raw;
            const int in = st->gram_cur, out = (ga.new_slot >= 0) ? 1 - in : in;
            ga.SY_in = st->SY[in]; ga.YY_in = st->YY[in]; ga.SS_in = st->SS[in];
            ga.SY_out = st->SY[out]; ga.YY_out = st->YY[out]; ga.SS_out = st->SS[out];
            ga.ys = st->ys; ga.alpha = st->alpha; ga.theta = st->theta;
            for (int age = 0; age < c; age++) ga.slots[age] = (unsigned char)slot_by_age(head, M, age);
            for (int age = tid; age < c; age += nt) s_slot[age] = ga.slots[age];
            gram_solve_in_smem<T, false>(ga, gram, true);   // (ends with a barrier: the coefficients and s_slot are in place)
            const T* coef = gram + 2 * c * c;
            const T cv = coef[0];
            T acc[5] = {T(0), T(0), T(0), T(0), T(0)};
            for (int64_t q = tid; q < npacks; q += nt)
            {
                const int64_t i0 = q << 2;
                const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
                T r[4], xv[4] = {T(0), T(0), T(0), T(0)};
#pragma unroll
                for (int k = 0; k < 4; k++) r[k] = (k < cnt) ? cv * g[i0 + k] : T(0);
                for (int j = 0; j < c; j++)
                {
                    const T* yj = s_col(s_slot[j]) + ld;
                    const T cy = coef[1 + j];
#pragma unroll
                    for (int k = 0; k < 4; k++) r[k] += (k < cnt) ? cy * yj[i0 + k] : T(0);
                }
                for (int j = c - 1; j >= 0; j--)
                {
                    const T* sj = s_col(s_slot[j]);
                    const T cs = coef[1 + c + j];
#pragma unroll
                    for (int k = 0; k < 4; k++) r[k] += (k < cnt) ? cs * sj[i0 + k] : T(0);
                }
#pragma unroll
                for (int k = 0; k < 4; k++)
                    if (k < cnt)
                    {
                        d[i0 + k] = r[k];
                        acc[0] += g[i0 + k] * r[k];
                        xv[k] = x[i0 + k] + T(1) * r[k];
                    }
                if (fuse && !STORED)
                {
                    T gv[4];
                    eval_pack(obj, i0, cnt, xv, T(0), T(0), r, gv, acc + 1);
                }
                else if (fuse)
                {
#pragma unroll
                    for (int k = 0; k < 4; k++)
                        if (k < cnt) xp[i0 + k] = xv[k];
                }
            }
            if (fuse && STORED)
            {
                __syncthreads();   // x1 of every coordinate is in xp: the objective takes its neighbours from there
                for (int64_t q = tid; q < npacks; q += nt)
                {
                    const int64_t i0 = q << 2;
                    const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
                    T xv[4], dv[4], gv[4], xl, xr;
#pragma unroll
                    for (int k = 0; k < 4; k++) { xv[k] = (k < cnt) ? xp[i0 + k] : T(0); dv[k] = (k < cnt) ? d[i0 + k] : T(0); }
                    pack_neighbours<false>(obj, i0, n, T(0), [&](int j) { return xp[i0 + j]; }, xl, xr);
                    eval_pack(obj, i0, cnt, xv, xl, xr, dv, gv, acc + 1);
#pragma unroll
                    for (int k = 0; k < 4; k++)
                        if (k < cnt) gp[i0 + k] = gv[k];
                }
            }
            if (fuse)
            {
                const double dacc[5] = {(double)acc[0], (double)acc[1], (double)acc[2], (double)acc[3], (double)acc[4]};
                small_sums<5>(dacc, red, ps, raw);
            }
            else
            {
                const double dacc[1] = {(double)acc[0]};
                small_sums<1>(dacc, red, ps, raw);
            }
            break;
        }
        default: break;
        }
        __syncthreads();   // raw[] and the pass's vectors are complete
        if (tid == 0) advance_problem<T, STORED>(st, raw);
    }

    // ---- the final history (optional): what BFGSMat holds when minimize() returns.  A solve stops only in after_search (before the
    // pair-forming dots of that iteration, so the last step's pair never enters: reference LBFGS.h:137-162), in digest_trial (a
    // line-search error) or in begin_search (a search that refuses to start); all three run when no pair is pending.  The
    // combination pass of the iteration that accepted the newest pair folded its Gram rows and columns into SY/YY/SS[1 - gram_cur]
    // and advance_problem flipped gram_cur and cleared `pending` in the same step, and a rejected pair (DOTS_PLAIN) touches neither
    // the ring nor the Gram blocks.  So at every exit -- max_iterations, past/delta, a line-search error, convergence at x0 with
    // ncorr = 0 -- SY/YY/SS[gram_cur] hold exactly the dots of the ncorr pairs that head, ys and theta describe.
    if (a.hist) small_export_history(st, s_col(0), ld, a.hist + b * SmallHistLayout{n, M - 1}.rec(), a.hist_c + b, n);

    // ---- results: the point (and gradient) the problem stopped at, and its outcome ----
    {
        T* const xo = a.X + b * a.ldx;
        const T* xs = st->x;
        const T* gs = st->g;
        for (int64_t i = tid; i < n; i += nt) xo[i] = xs[i];
        if (a.G)
        {
            T* const go = a.G + b * a.ldx;
            for (int64_t i = tid; i < n; i += nt) go[i] = gs[i];
        }
        if (tid == 0)
        {
            lbfgs_b200_outcome o;
            o.status = st->status; o.niter = st->niter; o.nfev = st->nfev;
            o.fx = (double)st->rec.fx; o.gnorm = (double)st->gnorm; o.rounds = st->rounds;
            a.outs[b] = o;
        }
    }
}


// ---- products with the kept approximations: OUT_p = B_b V_p or H_b V_p for problems b = b0 + p --------------------------------
// One CTA per (problem, group of up to kSGroup vectors), small_threads(n) threads: the dots [Y S]'V (per thread in fp64 over the
// coordinates i = tid, tid + nt, ..., then small_sums), the coefficients of CompactForm.h (B: Minv factorised by thread 0, the 2c
// columns of M = Minv^-1 solved by 2c threads; H: R and Y'Y set up once; one thread per vector for its coefficients), and
// OUT = a0 V + sum_a cy_a y_a + sum_a cs_a s_a (terms in that order).  Every sum's order depends on n only, so a problem's products
// do not depend on b0, count or its position, and column j of a call equals a one-vector call on that column.
constexpr int kSGroup = 16;

template <class T> struct SmallTimesArgs
{
    const T* hist;              // records of SmallHistLayout
    const int* hist_c;
    SmallHistLayout HL;
    int64_t b0;
    int k, inverse;
    const T* V;                 // problem p's vector j at V + p*ldvp + j*ldv
    int64_t ldv, ldvp;
    T* OUT;                     // at OUT + p*ldop + j*ldo
    int64_t ldo, ldop;
};

// dynamic shared memory of k_small_hist_times (bytes): block sums, [Y S]'V and the coefficients (2m x kSGroup each), and the
// algebra: B needs Minv's factor and M (2m x 2m each), H needs R, Y'Y (m x m each) and two scratch rows per vector
inline size_t small_times_smem(int m, int elem)
{
    const size_t w = 2 * (size_t)m;
    const size_t alg_b = 2 * w * w, alg_h = 2 * (size_t)m * m + 2 * (size_t)m * kSGroup;
    return sizeof(double) * (size_t)kSMaxWarps * kSGroup + (size_t)elem * (2 * w * kSGroup + (alg_b > alg_h ? alg_b : alg_h));
}

// The 2c x 2c algebra of a kept problem, on the chip, for the products and the diagonal.  Every thread of the CTA calls it; it ends
// with a barrier.  B: Minv factorised in place by thread 0 in alg[0, w^2) (w = 2c), then M = Minv^-1 in alg[w^2, 2w^2), column j
// solved by thread j.  H: R and Y'Y in chronological order in alg[0, c^2) and alg[c^2, 2c^2), set up by thread 0.
template <class T>
__device__ __forceinline__ void small_compact_setup(const T* rec, const SmallHistLayout& HL, int c, T theta, bool inverse, T* alg, int* order,
                                                    unsigned char* tag)
{
    const int tid = threadIdx.x, nt = blockDim.x;
    const T* SY = rec + HL.SY();
    if (!inverse)
    {
        const int w = 2 * c;
        T* F = alg;            // Minv, factorised in place
        T* Mm = alg + w * w;   // M = Minv^-1
        if (tid == 0)
        {
            LBFGSpp::compact_minv(c, SY, rec + HL.SS(), c, theta, F);
            LBFGSpp::bk_factor(F, w, order, tag);
        }
        __syncthreads();
        for (int j = tid; j < w; j += nt)   // column j of M: Minv^-1 e_j
        {
            T z[2 * kMaxM];
            for (int i = 0; i < w; i++) Mm[i * w + j] = i == j ? T(1) : T(0);
            LBFGSpp::bk_solve(F, w, order, tag, Mm + j, w, z);
        }
    }
    else if (tid == 0)
        LBFGSpp::compact_h_setup(c, SY, rec + HL.YY(), c, alg, alg + c * c);
    __syncthreads();
}

template <class T>
__global__ void __launch_bounds__(kSMaxThreads) k_small_hist_times(const SmallTimesArgs<T> a)
{
    extern __shared__ __align__(16) unsigned char s_smem[];
    __shared__ int s_order[2 * kMaxM];
    __shared__ unsigned char s_tag[2 * kMaxM];
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
    const int64_t p = blockIdx.x, b = a.b0 + p, n = a.HL.n;
    const int m = a.HL.m, j0 = blockIdx.y * kSGroup, kk = min(kSGroup, a.k - j0);
    const T* rec = a.hist + b * a.HL.rec();
    const T* V = a.V + p * a.ldvp + j0 * a.ldv;
    T* OUT = a.OUT + p * a.ldop + j0 * a.ldo;
    const int c = a.hist_c[b];
    const T theta = rec[a.HL.theta()];
    const T a0 = a.inverse ? T(1) / theta : theta;
    double* red = reinterpret_cast<double*>(s_smem);
    T* wv = reinterpret_cast<T*>(red + kSMaxWarps * kSGroup);        // [2c][kSGroup]
    T* C = wv + 2 * m * kSGroup;                                     // [2c][kSGroup]
    T* alg = C + 2 * m * kSGroup;
    if (c > 0)
    {
        // [Y S]'V, one history row at a time
        for (int r = 0; r < 2 * c; r++)
        {
            const T* h = rec + (r < c ? a.HL.y(r) : a.HL.s(r - c));
            double acc[kSGroup];
#pragma unroll
            for (int j = 0; j < kSGroup; j++) acc[j] = 0.0;
            for (int64_t i = tid; i < n; i += nt)
            {
                const double hv = (double)h[i];
#pragma unroll
                for (int j = 0; j < kSGroup; j++)
                    if (j < kk) acc[j] += hv * (double)V[j * a.ldv + i];
            }
            // block sums as small_sums takes them: a fixed shuffle tree per warp, warp totals in warp order
#pragma unroll
            for (int j = 0; j < kSGroup; j++)
            {
                const double w = warp_sum(acc[j]);
                if (lane == 0) red[warp * kSGroup + j] = w;
            }
            __syncthreads();
            if (tid < kk)
            {
                double t = 0.0;
                for (int w = 0; w < (nt >> 5); w++) t += red[w * kSGroup + tid];
                wv[r * kSGroup + tid] = (T)t;
            }
            __syncthreads();
        }
        small_compact_setup(rec, a.HL, c, theta, a.inverse != 0, alg, s_order, s_tag);
        if (tid < kk)
        {
            if (!a.inverse) LBFGSpp::compact_b_coef(c, alg + 4 * c * c, theta, wv + tid, kSGroup, C + tid, kSGroup);
            else
            {
                T* scr = alg + 2 * c * c;   // per vector: w, us (c each), column tid
                LBFGSpp::compact_h_coef(c, alg, alg + c * c, theta, wv + tid, kSGroup, scr + tid, scr + c * kSGroup + tid, kSGroup, C + tid, kSGroup);
            }
        }
        __syncthreads();
    }
    // OUT = a0 V + sum_a cy_a y_a + sum_a cs_a s_a
    for (int64_t i = tid; i < n; i += nt)
    {
        T r[kSGroup];
#pragma unroll
        for (int j = 0; j < kSGroup; j++) r[j] = j < kk ? a0 * V[j * a.ldv + i] : T(0);
        for (int row = 0; row < 2 * c; row++)
        {
            const T hv = rec[(row < c ? a.HL.y(row) : a.HL.s(row - c)) + i];
#pragma unroll
            for (int j = 0; j < kSGroup; j++) r[j] += C[row * kSGroup + j] * hv;
        }
#pragma unroll
        for (int j = 0; j < kSGroup; j++)
            if (j < kk) OUT[j * a.ldo + i] = r[j];
    }
}


// ---- the diagonals of the kept approximations: OUT + p*ldo = diag(B_b) or diag(H_b) for problems b = b0 + p ----------------------
// One CTA per problem, small_threads(n) threads.  The CTA forms K of B = theta I + W K_B W' or H = I/theta + W K_H W' (W = [Y S] by
// age; CompactForm.h: compact_kb / compact_kh column by column, then compact_k_symmetrise) after small_compact_setup, and makes one
// pass over its rows: out_i = a0 + r_i' K r_i in the order of k_hist_quad_diag (lbfgsb_kernels.cuh), all in fp64:
//     t_p = K_pp r_p,  t_p = fma(2 K_pq, r_q, t_p) for q = p+1, ..., 2c-1;   acc = fma(r_p, t_p, acc) for p = 0, ..., 2c-1;  a0 + acc
// Nothing depends on b0, count or the problem's position.
template <class T> struct SmallDiagArgs
{
    const T* hist;              // records of SmallHistLayout
    const int* hist_c;
    SmallHistLayout HL;
    int64_t b0;
    int inverse;
    T* OUT;                     // problem p's diagonal at OUT + p*ldo
    int64_t ldo;
};

// elements of the algebra region: B needs Minv's factor (K takes its place once M is formed) and M; H needs R, Y'Y, the scratch of
// kSGroup columns and K.  With the unit vector of compact_kb / compact_kh (4m - 1) this never exceeds small_times_smem.
__host__ __device__ inline size_t small_diag_alg(int m)
{
    const size_t w = 2 * (size_t)m;
    const size_t alg_b = 2 * w * w, alg_h = 2 * (size_t)m * m + 2 * (size_t)m * kSGroup + w * w;
    return alg_b > alg_h ? alg_b : alg_h;
}
inline size_t small_diag_smem(int m, int elem) { return (size_t)elem * (small_diag_alg(m) + 4 * (size_t)m); }

template <class T>
__global__ void __launch_bounds__(kSMaxThreads) k_small_hist_diag(const SmallDiagArgs<T> a)
{
    extern __shared__ __align__(16) unsigned char s_smem[];
    __shared__ int s_order[2 * kMaxM];
    __shared__ unsigned char s_tag[2 * kMaxM];
    const int tid = threadIdx.x, nt = blockDim.x;
    const int64_t p = blockIdx.x, b = a.b0 + p, n = a.HL.n;
    const T* rec = a.hist + b * a.HL.rec();
    T* out = a.OUT + p * a.ldo;
    const int c = a.hist_c[b], w = 2 * c;
    const T theta = rec[a.HL.theta()];
    const double a0 = (double)(a.inverse ? T(1) / theta : theta);
    T* alg = reinterpret_cast<T*>(s_smem);
    T* unit = alg + small_diag_alg(a.HL.m);
    T* K = a.inverse ? alg + 2 * c * c + 2 * c * kSGroup : alg;
    if (c > 0)
    {
        for (int e = tid; e < 2 * w - 1; e += nt) unit[e] = e == w - 1 ? T(1) : T(0);
        small_compact_setup(rec, a.HL, c, theta, a.inverse != 0, alg, s_order, s_tag);
        if (!a.inverse) LBFGSpp::compact_kb(c, alg + w * w, theta, unit, tid, nt, K);
        else if (tid < kSGroup) LBFGSpp::compact_kh(c, alg, alg + c * c, theta, unit, tid, kSGroup, alg + 2 * c * c + tid, kSGroup, K);
        __syncthreads();
        LBFGSpp::compact_k_symmetrise(w, K, tid, nt);
        __syncthreads();
    }
    for (int64_t i = tid; i < n; i += nt)
    {
        double r[2 * kMaxM];
        for (int q = 0; q < w; q++) r[q] = (double)rec[(q < c ? a.HL.y(q) : a.HL.s(q - c)) + i];
        double acc = 0.0;
        for (int pp = 0; pp < w; pp++)
        {
            const T* kr = K + pp * w;
            double t = (double)kr[pp] * r[pp];
            for (int q = pp + 1; q < w; q++) t = fma(2.0 * (double)kr[q], r[q], t);
            acc = fma(r[pp], t, acc);
        }
        out[i] = (T)(a0 + acc);
    }
}


// ---- the square-root factor of the kept H_b: OUT = L_b V (factor_times) or MEAN + L_b Z (sample) -----------------------------------
// One CTA per (problem, group of <= kSGroup vectors or draws), small_threads(n) threads, the shape of k_small_hist_times: [Y S]'V in
// fp64 through the same block sums, the algebra of CompactForm.h on the chip (compact_factor_setup by thread 0, then
// compact_factor_coef, one thread per vector) and the combination L v = v/sqrt(theta) + sum_a alpha_a s_a (terms a0 v, then s by age;
// the sampler adds the mean first).  GEN: the vectors are draws first + j0 + j of stream b (philox.cuh), generated once into OUT
// (one generator call per coordinate pair) and read back from there, each element by the thread that overwrites it.  Nothing depends
// on b0, count or the problem's position.  A problem whose pairs fail compact_factor_setup's check gets NaN.
template <class T> struct SmallFactorArgs
{
    const T* hist;              // records of SmallHistLayout
    const int* hist_c;
    SmallHistLayout HL;
    int64_t b0;
    int k;
    const T* V;                 // loaded: problem p's vector j at V + p*ldvp + j*ldv;  GEN: the mean of problem p at V + p*ldvp (or NULL)
    int64_t ldv, ldvp;
    T* OUT;                     // at OUT + p*ldop + j*ldo
    int64_t ldo, ldop;
    unsigned long long seed;
    uint32_t first;
};

// dynamic shared memory of k_small_hist_factor (bytes): block sums, [Y S]'V and the coefficients (2m x kSGroup each, as
// small_times_smem), then beta (2m x m) and Tm (m x m) in double: never more than small_times_smem
inline size_t small_factor_smem(int m, int elem)
{
    return sizeof(double) * (size_t)kSMaxWarps * kSGroup + (size_t)elem * 4 * (size_t)m * kSGroup + sizeof(double) * 3 * (size_t)m * m;
}

// OP (LBFGS_B200_FACTOR_*): L as above; L' and L^-T take the dots of the c s rows only and combine over all 2c columns (a0 V, y by
// age, s by age), L^-1 takes all 2c dots and combines over the s columns; a0 = 1/sqrt(theta) for L and L', sqrt(theta) for the
// inverses.  The recursion of each op (compact_factor_t_coef / _inv_coef / _invt_coef, after compact_factor_upper for the inverses)
// runs in fp64 in a per-thread array.
template <class T, bool GEN, int OP = LBFGS_B200_FACTOR_L>
__global__ void __launch_bounds__(kSMaxThreads) k_small_hist_factor(const SmallFactorArgs<T> a)
{
    constexpr bool kSDots = OP == LBFGS_B200_FACTOR_LT || OP == LBFGS_B200_FACTOR_LINVT;   // S'V only, combination over W
    constexpr bool kInv = OP == LBFGS_B200_FACTOR_LINV || OP == LBFGS_B200_FACTOR_LINVT;
    extern __shared__ __align__(16) unsigned char s_smem[];
    __shared__ int s_ok;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
    const int64_t p = blockIdx.x, b = a.b0 + p, n = a.HL.n;
    const int m = a.HL.m, j0 = blockIdx.y * kSGroup, kk = min(kSGroup, a.k - j0);
    const T* rec = a.hist + b * a.HL.rec();
    T* OUT = a.OUT + p * a.ldop + j0 * a.ldo;
    const T* V = GEN ? OUT : a.V + p * a.ldvp + j0 * a.ldv;
    const int64_t ldv = GEN ? a.ldo : a.ldv;
    const T* mean = GEN && a.V ? a.V + p * a.ldvp : nullptr;
    const int c = a.hist_c[b];
    const T theta = rec[a.HL.theta()];
    const double rsq = 1.0 / sqrt((double)theta);
    const T a0 = kInv ? (T)sqrt((double)theta) : (T)rsq;
    double* red = reinterpret_cast<double*>(s_smem);
    T* wv = reinterpret_cast<T*>(red + kSMaxWarps * kSGroup);        // [2c][kSGroup]
    T* C = wv + 2 * m * kSGroup;                                     // [2c][kSGroup]
    double* beta = reinterpret_cast<double*>(C + 2 * m * kSGroup);   // [2c][c]
    double* Tm = beta + 2 * m * m;                                   // [c][c]
    if (GEN)
    {
        for (int64_t q = tid; 2 * q < n; q += nt)
#pragma unroll
            for (int j = 0; j < kSGroup; j++)
                if (j < kk)
                {
                    double z0, z1;
                    normal_pair(a.seed, (uint32_t)b, a.first + (uint32_t)(j0 + j), (unsigned long long)q, z0, z1);
                    OUT[j * a.ldo + 2 * q] = (T)z0;
                    if (2 * q + 1 < n) OUT[j * a.ldo + 2 * q + 1] = (T)z1;
                }
        __syncthreads();
    }
    bool ok = true;
    if (c > 0)
    {
        // [Y S]'V, one history row at a time (the sums of k_small_hist_times)
        for (int r = kSDots ? c : 0; r < 2 * c; r++)
        {
            const T* h = rec + (r < c ? a.HL.y(r) : a.HL.s(r - c));
            double acc[kSGroup];
#pragma unroll
            for (int j = 0; j < kSGroup; j++) acc[j] = 0.0;
            for (int64_t i = tid; i < n; i += nt)
            {
                const double hv = (double)h[i];
#pragma unroll
                for (int j = 0; j < kSGroup; j++)
                    if (j < kk) acc[j] += hv * (double)V[j * ldv + i];
            }
#pragma unroll
            for (int j = 0; j < kSGroup; j++)
            {
                const double w = warp_sum(acc[j]);
                if (lane == 0) red[warp * kSGroup + j] = w;
            }
            __syncthreads();
            if (tid < kk)
            {
                double t = 0.0;
                for (int w = 0; w < (nt >> 5); w++) t += red[w * kSGroup + tid];
                wv[r * kSGroup + tid] = (T)t;
            }
            __syncthreads();
        }
        if (tid == 0)
        {
            double ls;
            s_ok = LBFGSpp::compact_factor_setup(c, rec + a.HL.SY(), rec + a.HL.SS(), rec + a.HL.YY(), c, theta, beta, Tm, &ls) == 0;
            if constexpr (kInv)
                if (s_ok) LBFGSpp::compact_factor_upper(c, rec + a.HL.SY(), c, Tm);
        }
        __syncthreads();
        ok = s_ok != 0;
        if (ok && tid < kk)
        {
            if constexpr (OP == LBFGS_B200_FACTOR_L) LBFGSpp::compact_factor_coef(c, beta, Tm, rsq, wv + tid, kSGroup, C + tid, kSGroup);
            else
            {
                double z[kMaxM];
                const double sq = sqrt((double)theta);
                if constexpr (OP == LBFGS_B200_FACTOR_LT)
                    LBFGSpp::compact_factor_t_coef(c, beta, Tm, rsq, wv + c * kSGroup + tid, kSGroup, z, C + tid, kSGroup);
                else if constexpr (OP == LBFGS_B200_FACTOR_LINV)
                    LBFGSpp::compact_factor_inv_coef(c, beta, Tm, sq, wv + tid, kSGroup, z, C + tid, kSGroup);
                else LBFGSpp::compact_factor_invt_coef(c, beta, Tm, sq, wv + c * kSGroup + tid, kSGroup, z, C + tid, kSGroup);
            }
        }
        __syncthreads();
    }
    // OUT = [mean +] a0 V [+ sum_a cy_a y_a] + sum_a cs_a s_a
    const T nan = (T)__longlong_as_double(0x7ff8000000000000ll);
    for (int64_t i = tid; i < n; i += nt)
    {
        T r[kSGroup];
        const T mi = mean ? mean[i] : T(0);
#pragma unroll
        for (int j = 0; j < kSGroup; j++) r[j] = j < kk ? (mean ? mi + a0 * V[j * ldv + i] : a0 * V[j * ldv + i]) : T(0);
        if constexpr (kSDots)
            for (int q = 0; q < c; q++)
            {
                const T yv = rec[a.HL.y(q) + i];
#pragma unroll
                for (int j = 0; j < kSGroup; j++) r[j] += C[q * kSGroup + j] * yv;
            }
        for (int q = 0; q < c; q++)
        {
            const T sv = rec[a.HL.s(q) + i];
#pragma unroll
            for (int j = 0; j < kSGroup; j++) r[j] += C[(c + q) * kSGroup + j] * sv;
        }
#pragma unroll
        for (int j = 0; j < kSGroup; j++)
            if (j < kk) OUT[j * a.ldo + i] = ok ? r[j] : nan;
    }
}

// log det H_b = -n log theta + sum_t log(rho_t sigma_t) (compact_factor_setup) for problems b0 + p: one CTA of one warp per problem,
// thread 0 does the O(c^3) recursion in dynamic shared memory (3c^2 doubles).  NaN when the check fails.
template <class T> __global__ void k_small_hist_logdet(const T* hist, const int* hist_c, SmallHistLayout HL, int64_t b0, double* out)
{
    extern __shared__ __align__(16) unsigned char s_smem[];
    if (threadIdx.x != 0) return;
    const int64_t p = blockIdx.x, b = b0 + p;
    const T* rec = hist + b * HL.rec();
    const int c = hist_c[b];
    const T theta = rec[HL.theta()];
    double* beta = reinterpret_cast<double*>(s_smem);
    double ls = 0.0;
    const int st = LBFGSpp::compact_factor_setup(c, rec + HL.SY(), rec + HL.SS(), rec + HL.YY(), c, theta, beta, beta + 2 * c * c, &ls);
    out[p] = st ? __longlong_as_double(0x7ff8000000000000ll) : -(double)HL.n * log((double)theta) + ls;
}

// log N(x_pj; mean_p, H_b) for problems b = b0 + p and points j: one CTA per (problem, group of <= kSGroup points), small_threads(n)
// threads.  v_j = x_j - mean is formed in T; W'v_j and |v_j|^2 are summed in fp64 through the block sums of k_small_hist_factor (a
// row of W at a time, then the points with themselves), thread 0 runs compact_factor_setup and compact_factor_upper, and thread j
// the recursion of compact_factor_quad.  Every sum's order depends on n only, so a problem's values do not depend on b0, count, its
// position or k.  NaN when the check fails.
template <class T> struct SmallDensityArgs
{
    const T* hist;
    const int* hist_c;
    SmallHistLayout HL;
    int64_t b0;
    int k;
    const T* X;                 // problem p's point j at X + p*ldxp + j*ldx
    int64_t ldx, ldxp;
    const T* MEAN;              // problem p's mean at MEAN + p*ldm
    int64_t ldm;
    double* out;                // [count][k]
};

// dynamic shared memory of k_small_hist_log_density (bytes): block sums, W'v and |v|^2 ((2m + 1) x kSGroup), beta and Tm, all in
// double.  At most small_times_smem for m >= 2 and under 1 KB for m = 1, so any history small_hist_create accepts fits.
inline size_t small_density_smem(int m)
{
    return sizeof(double) * ((size_t)kSMaxWarps * kSGroup + (2 * (size_t)m + 1) * kSGroup + 3 * (size_t)m * m);
}

template <class T>
__global__ void __launch_bounds__(kSMaxThreads) k_small_hist_log_density(const SmallDensityArgs<T> a)
{
    extern __shared__ __align__(16) unsigned char s_smem[];
    __shared__ int s_ok;
    __shared__ double s_ls;
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
    const int64_t p = blockIdx.x, b = a.b0 + p, n = a.HL.n;
    const int m = a.HL.m, j0 = blockIdx.y * kSGroup, kk = min(kSGroup, a.k - j0);
    const T* rec = a.hist + b * a.HL.rec();
    const T* X = a.X + p * a.ldxp + j0 * a.ldx;
    const T* mean = a.MEAN + p * a.ldm;
    const int c = a.hist_c[b];
    const T theta = rec[a.HL.theta()];
    double* red = reinterpret_cast<double*>(s_smem);
    double* wv = red + kSMaxWarps * kSGroup;   // [2c + 1][kSGroup]: W'v, then |v|^2
    double* beta = wv + (2 * m + 1) * kSGroup;
    double* Tm = beta + 2 * m * m;
    for (int r = 0; r <= 2 * c; r++)
    {
        const T* h = r < c ? rec + a.HL.y(r) : r < 2 * c ? rec + a.HL.s(r - c) : nullptr;
        double acc[kSGroup];
#pragma unroll
        for (int j = 0; j < kSGroup; j++) acc[j] = 0.0;
        for (int64_t i = tid; i < n; i += nt)
        {
            const T mi = mean[i];
#pragma unroll
            for (int j = 0; j < kSGroup; j++)
                if (j < kk)
                {
                    const double v = (double)(X[j * a.ldx + i] - mi);
                    acc[j] += (h ? (double)h[i] : v) * v;
                }
        }
#pragma unroll
        for (int j = 0; j < kSGroup; j++)
        {
            const double w = warp_sum(acc[j]);
            if (lane == 0) red[warp * kSGroup + j] = w;
        }
        __syncthreads();
        if (tid < kk)
        {
            double t = 0.0;
            for (int w = 0; w < (nt >> 5); w++) t += red[w * kSGroup + tid];
            wv[r * kSGroup + tid] = t;
        }
        __syncthreads();
    }
    if (tid == 0)
    {
        double ls = 0.0;
        s_ok = LBFGSpp::compact_factor_setup(c, rec + a.HL.SY(), rec + a.HL.SS(), rec + a.HL.YY(), c, theta, beta, Tm, &ls) == 0;
        if (s_ok) LBFGSpp::compact_factor_upper(c, rec + a.HL.SY(), c, Tm);
        s_ls = ls;
    }
    __syncthreads();
    if (tid < kk)
    {
        double z[kMaxM];
        double r = __longlong_as_double(0x7ff8000000000000ll);
        if (s_ok)
        {
            const double q = LBFGSpp::compact_factor_quad(c, beta, Tm, rec + a.HL.SS(), c, theta, wv + tid, kSGroup, wv[2 * c * kSGroup + tid], z);
            r = LBFGSpp::compact_log_density(q, -(double)n * log((double)theta) + s_ls, (double)n);
        }
        a.out[p * a.k + j0 + tid] = r;
    }
}

}  // namespace lb
