// problem_machine.cuh -- the scalar side of one L-BFGS problem solved on the device: its state (PState), the ops of the pass it asks
// for next (POP_*), and the rules that digest the reduced values of that pass and choose the next one (advance_problem and its
// helpers).  They hold every scalar rule of LBFGSSolver::minimize() (reference LBFGS.h:78-173) through the line-search cores of
// include/LBFGSpp/LineSearchCore.h and the stopping rules of include/LBFGSpp/LoopRules.h.  Two kernels drive it: the device-resident
// solve (persist.cuh: one problem spread over every SM, the leader CTA advancing every problem between rounds) and the small-batch
// solve (small_batch.cuh: one CTA per problem, the whole solve in shared memory).  Whoever drives it runs the pass for st->op,
// reduces its nvals_of(st) values into double raw[] and calls advance_problem, until st->op is POP_IDLE.
#pragma once

#include "../../include/LBFGSpp/LoopRules.h"
#include "two_loop_gram.cuh"

namespace lb {

constexpr int kMaxPast = 64;

enum { POP_IDLE = 0, POP_FIRST = 1, POP_TRIAL = 2, POP_DOTS_FORM = 3, POP_DOTS_PLAIN = 4, POP_COMBINE = 5, POP_COMBINE_TRIAL = 6, POP_RESTORE = 7,
       POP_MATERIALIZE = 8 };

// which point an implied (x, g) stands for (PState::at_start): the ray point xp + step*d, the search's start point, or (only when
// the gradient itself is implied, G_IMPLIED below) the point already in x, whose g is grad f(x) but not stored
enum { PT_RAY = 0, PT_START = 1, PT_X = 2 };

// ---- the S/Y history of the solve: tiled layout ---------------------------------------------------------------------------------
// H[block][slot][S|Y][BT]: all ring slots of one block of BT coordinates lie next to each other (BT = the largest power of two for
// which two stages of 2m+4 rows fit the kernel's shared memory: 512 for fp64 m = 10).  A pass over a tile then needs the right-hand
// vectors plus ONE or TWO bulk copies of 8..90 KB for all history columns (the live slots form a cyclic range of the ring), instead
// of one 4 KB copy per column: measured, the per-copy cost of 22 separate copies was ~15 % of the combination pass, and 42 copies of
// 2 KB at m = 20 made it 2.8x slower per byte.  The new pair of an iteration is written as one 2*BT run per block.
template <class T> struct PHist
{
    T* H;
    int bt_log, M;
    int64_t bstride;      // elements per block: M * 2 * BT
    __device__ __forceinline__ int BT() const { return 1 << bt_log; }
    __device__ __forceinline__ T* s_at(int slot, int64_t i) const { return H + (i >> bt_log) * bstride + ((int64_t)slot << (bt_log + 1)) + (i & (BT() - 1)); }
    __device__ __forceinline__ T* y_at(int slot, int64_t i) const { return s_at(slot, i) + BT(); }
    // the ring as 2M point rows (objectives without neighbour coupling, see PState::pts): row `p` of element i
    __device__ __forceinline__ T* pt_at(int p, int64_t i) const { return H + (i >> bt_log) * bstride + ((int64_t)p << bt_log) + (i & (BT() - 1)); }
};

// ---- per-problem state (device memory; the leader CTA's working copy) ----------------------------------------------------------
template <class T> struct PState
{
    // vectors (rotate by pointer swap); x_lo, g_lo: neighbour-coupled objectives only (nullptr otherwise)
    T *x, *xp, *g, *gp, *drt, *x_lo, *g_lo;
    // history storage (fixed for the duration of the kernel: other CTAs read these fields with ordinary loads)
    PHist<T> hist;              // the S/Y ring, tiled (see PHist)
    T *ys, *alpha, *theta;
    T *SY[2], *YY[2], *SS[2];
    const T *data0, *data1;
    double* raw;               // [pstride] reduced values of the last round
    double* halo;              // kHaloDoubles (neighbour-coupled objectives under n-sharding)
    // ring geometry
    int head, ncorr, M, m, gram_cur, pending;
    // what the next round does
    int op, c_round;
    // options (LBFGSParam)
    T epsilon, epsilon_rel, delta, max_step;
    int past, max_iterations, fuse_first_trial;
    LBFGSpp::LineSearchOptions<T> ls_opt;
    // line-search state
    LBFGSpp::RunTimeCore<T> ls;
    LBFGSpp::SearchRecord<T> rec;   // fx, dg, gg, xx of the current point
    // iteration scalars.  step: the trial to evaluate, or (objectives without neighbour coupling) the step of the point (x, g)
    // stand for while they are implied; step_kept: the step of the search's kept trial; at_start: which point they stand for (PT_*)
    T gnorm, step, step_kept;
    int at_start;
    int k;
    long long nfev;
    int status;     // 0 ok, otherwise a LineSearchError code
    int finished;
    int niter;      // return value of minimize()
    T fx_hist[kMaxPast];
    // POINTS (the resident solve, objectives without neighbour coupling): the ring's 2M rows per block hold iterates instead of M
    // pairs S|Y.  x and xp are rows of it (the flat x, g stay the caller's start point and result); a pair is rebuilt from its two
    // endpoints wherever it is read: s = x_end - x_start, y = grad f(x_end) - grad f(x_start).
    int px, pxp;                // point rows of x and xp
    unsigned char* pts;         // [2M] device memory: start and end point row of the pair in each pair slot (read by every CTA)
    double* trace;              // optional: f of every evaluation
    long long trace_cap;
    long long rounds;           // rounds this problem took part in
};

template <class P> __device__ __forceinline__ void dswap(P& a, P& b) { P t = a; a = b; b = t; }
__host__ __device__ __forceinline__ int slot_by_age(int head, int M, int age) { return ((head - 1 - age) % M + M) % M; }

// ---- the leader's work between two rounds ------------------------------------------------------------------------------------
template <class T> __device__ __forceinline__ void record_eval(PState<T>* st, T fx)
{
    if (st->trace && st->nfev < st->trace_cap) st->trace[st->nfev] = (double)fx;
    st->nfev++;
}
// the problem stops; `implied`: (x, g) do not hold its point yet, one MATERIALIZE round writes them (step, at_start) first
template <class T> __device__ __forceinline__ void finish(PState<T>* st, int niter, int status = 0, bool implied = false)
{
    st->finished = 1;
    st->niter = niter;
    if (status) st->status = status;
    st->op = implied ? POP_MATERIALIZE : POP_IDLE;
}

// POINTS: the point row the pair-forming pass writes x to -- the first row after xp's, cyclically, that neither xp nor an endpoint
// of a live pair holds.  A chained history then stays one cyclic run of rows.  2M rows always leave one free: m live pairs have at
// most 2m endpoints.
template <class T> __device__ int free_point(const PState<T>* st)
{
    const int P = 2 * st->M;
    unsigned long long used[3] = {0ull, 0ull, 0ull};   // 2M <= 2 (kMaxM + 1) rows
    auto mark = [&](int p) { used[p >> 6] |= 1ull << (p & 63); };
    mark(st->pxp);
    for (int age = 0; age < st->ncorr; age++)
    {
        const int s = slot_by_age(st->head, st->M, age);
        mark(ldv(st->pts + 2 * s));
        mark(ldv(st->pts + 2 * s + 1));
    }
    for (int k = 1; k < P; k++)
    {
        const int p = (st->pxp + k) % P;
        if (!((used[p >> 6] >> (p & 63)) & 1ull)) return p;
    }
    return st->pxp;   // (not reached)
}

// after a search has produced its point -- in (x, g) when STORED, else implied by (step, at_start): the stopping rules
// (LBFGS.h:137-154), then on to the pair-forming dots
template <class T, bool STORED, bool POINTS = false> __device__ __forceinline__ void after_search(PState<T>* st)
{
    using namespace LBFGSpp;
    const int k = st->k;
    st->gnorm = std::sqrt(st->rec.gg);
    if (gradient_converged(st->gnorm, st->rec.xx, st->epsilon, st->epsilon_rel) || stalled(st->fx_hist, st->past, k, st->rec.fx, st->delta) ||
        iteration_cap(k, st->max_iterations))
    {
        finish(st, k, 0, !STORED);
        return;
    }
    st->op = POP_DOTS_FORM;
    st->c_round = st->ncorr < st->m ? st->ncorr + 1 : st->m;
    if (POINTS) st->px = free_point(st);
}

// the trial at st->step has been evaluated: {fx, dg, gg, xx}.  Sets the next op.  STORED: the trial is in (x, g), a kept trial
// moves to (x_lo, g_lo) by pointer swap; otherwise a trial is its step, and the kept one is st->step_kept.
template <class T, bool STORED, bool POINTS = false> __device__ __forceinline__ void digest_trial(PState<T>* st, T fx, T dg, T gg, T xx)
{
    record_eval(st, fx);
    bool keep = false;
    const int action = st->ls.advance(fx, dg, keep);
    const int next = st->rec.digest(action, keep, fx, dg, gg, xx, st->ls.best_fx(), st->ls.best_dg());
    if (next >= LBFGSpp::LSE_STEP_NOT_POSITIVE) { finish(st, st->k, next, !STORED); return; }   // (x, g): this trial
    if (keep)
    {
        if (STORED) { dswap(st->x, st->x_lo); dswap(st->g, st->g_lo); }
        else st->step_kept = st->step;
    }
    switch (next)
    {
    case LBFGSpp::SEARCH_EVALUATE: st->op = POP_TRIAL; st->step = st->ls.step(); return;
    case LBFGSpp::SEARCH_TAKE_KEPT:
        if (STORED) { dswap(st->x, st->x_lo); dswap(st->g, st->g_lo); }
        else st->step = st->step_kept;
        break;
    case LBFGSpp::SEARCH_TAKE_START:
        if (STORED) { st->op = POP_RESTORE; return; }   // copy xp/gp back, then carry on
        st->at_start = PT_START;
        break;
    }
    after_search<T, STORED, POINTS>(st);
}

// top of an iteration (LBFGS.h:121-127): the search is armed, the current point becomes the previous one.  G_IMPLIED: only x of
// the current point is stored (the pair-forming pass of an objective without neighbour coupling does not write g)
// POINTS: x and xp are point rows; the flat x, g are left alone (they only ever hold the start point and the result)
template <class T, bool G_IMPLIED = false, bool POINTS = false> __device__ __forceinline__ bool begin_search(PState<T>* st, T step)
{
    // the search validates its inputs before anything moves (the reference throws before touching x): on failure x stays the
    // current point (FIRST or the pair-forming pass wrote it; G_IMPLIED: one MATERIALIZE round writes its g)
    const int rc = st->ls.init(st->ls_opt, st->rec.fx, st->rec.dg, step, st->max_step);
    if (rc != 0)
    {
        if (G_IMPLIED) st->at_start = PT_X;
        finish(st, st->k, rc, G_IMPLIED);
        return false;
    }
    if (POINTS) dswap(st->pxp, st->px);
    else
    {
        dswap(st->xp, st->x);
        dswap(st->gp, st->g);
    }
    st->rec.begin();
    st->at_start = 0;
    st->op = POP_TRIAL;
    st->step = st->ls.step();
    return true;
}

// G_IMPLIED (the resident solve, objectives without neighbour coupling): g is stored by MATERIALIZE only; every other pass that needs
// grad f of a stored point evaluates it from x, bit for bit the g that would have been stored, and the first search's direction
// -grad f(x0) (k == 1: until the first combination pass writes d) is evaluated from x0 as well.  So every stop, at FIRST too, takes
// one MATERIALIZE round.  POINTS (the same solve): the ring holds iterates (see PState::pts)
template <class T, bool STORED, bool G_IMPLIED = false, bool POINTS = false> __device__ void advance_problem(PState<T>* st, const double* vals)
{
    st->rounds++;
    switch (st->op)
    {
    case POP_FIRST:
    {
        const T fx = (T)vals[0], gg = (T)vals[2], xx = (T)vals[3];
        st->nfev = 0;
        record_eval(st, fx);
        st->rec.fx = fx; st->rec.gg = gg; st->rec.xx = xx;
        st->k = 1;
        if (st->past > 0) st->fx_hist[0] = fx;
        st->gnorm = std::sqrt(gg);
        if (LBFGSpp::gradient_converged(st->gnorm, xx, st->epsilon, st->epsilon_rel))
        {
            if (G_IMPLIED) st->at_start = PT_X;   // FIRST wrote x0 to point row px only
            finish(st, 1, 0, G_IMPLIED);
            return;
        }
        st->rec.dg = -gg;                   // grad . (-grad)
        begin_search<T, G_IMPLIED, POINTS>(st, T(1) / st->gnorm); // LBFGS.h:108
        return;
    }
    case POP_TRIAL:
        digest_trial<T, STORED, POINTS>(st, (T)vals[0], (T)vals[1], (T)vals[2], (T)vals[3]);
        return;
    case POP_RESTORE:           // (x, g) now hold the search's start point; its sums were restored before
        after_search<T, STORED, POINTS>(st);
        return;
    case POP_MATERIALIZE:       // (x, g) now hold the point the problem stopped at
        st->op = POP_IDLE;
        return;
    case POP_DOTS_FORM:
    {
        // curvature gate on the pair's own dots (age-0 column: [2] = s'y, [3] = y'y), LBFGS.h:161; commit = BFGSMat.h:89-97
        const T sy = (T)vals[2], yy = (T)vals[3];
        if (LBFGSpp::curvature_ok(sy, yy, LBFGSpp::lsdetail::eps_of<T>()))
        {
            st->ys[st->head] = sy;
            if (POINTS) { st->pts[2 * st->head] = (unsigned char)st->pxp; st->pts[2 * st->head + 1] = (unsigned char)st->px; }
            *st->theta = yy / sy;
            st->pending = st->head;
            st->head = (st->head + 1) % st->M;
            st->ncorr = st->c_round;
            st->op = st->fuse_first_trial ? POP_COMBINE_TRIAL : POP_COMBINE;
        }
        else if (st->ncorr > 0) { st->op = POP_DOTS_PLAIN; st->c_round = st->ncorr; }
        else { st->op = st->fuse_first_trial ? POP_COMBINE_TRIAL : POP_COMBINE; st->c_round = 0; }
        return;
    }
    case POP_DOTS_PLAIN:
        st->op = st->fuse_first_trial ? POP_COMBINE_TRIAL : POP_COMBINE;
        return;
    case POP_COMBINE:
    case POP_COMBINE_TRIAL:
    {
        const bool fused = st->op == POP_COMBINE_TRIAL;
        if (st->pending >= 0) { st->gram_cur = 1 - st->gram_cur; st->pending = -1; }
        st->rec.dg = (T)vals[0];            // LBFGS.h:123 for the next pass
        st->k += 1;
        if (!begin_search<T, G_IMPLIED, POINTS>(st, T(1))) return;   // LBFGS.h:168
        // the pass already evaluated xp + 1*d (STORED: into the buffers that the rotation just made (x, g))
        if (fused && st->ls.step() == T(1)) digest_trial<T, STORED, POINTS>(st, (T)vals[1], (T)vals[2], (T)vals[3], (T)vals[4]);
        return;
    }
    default: return;
    }
}

template <class T> __device__ __forceinline__ int nvals_of(const PState<T>* st)
{
    switch (st->op)
    {
    case POP_FIRST: case POP_TRIAL: return 4;
    case POP_DOTS_FORM: case POP_DOTS_PLAIN: return st->c_round * kGramVals;
    case POP_COMBINE: return 1;
    case POP_COMBINE_TRIAL: return 5;
    default: return 0;
    }
}

// The options of a solve (lbfgs_b200_param) and the initial ring / op of a problem: the part of a PState that both solve kernels
// fill the same way.  Vectors, history storage and the data pointers are the caller's.
template <class T> inline void init_problem_state(PState<T>& p, const lbfgs_b200_param& prm, int ls_kind, bool fuse_first_trial)
{
    p.head = 0; p.ncorr = 0; p.M = prm.m + 1; p.m = prm.m; p.gram_cur = 0; p.pending = -1;
    p.op = POP_FIRST; p.c_round = 0;
    p.px = 0; p.pxp = 0;
    p.epsilon = (T)prm.epsilon; p.epsilon_rel = (T)prm.epsilon_rel; p.delta = (T)prm.delta; p.max_step = (T)prm.max_step;
    p.past = prm.past; p.max_iterations = prm.max_iterations;
    p.fuse_first_trial = fuse_first_trial;
    p.ls.kind = ls_kind;
    p.ls_opt = LBFGSpp::line_search_options<T>(prm, ls_kind);
}

}  // namespace lb
