// lbfgs_b200.cu -- kernels + C ABI of liblbfgs_b200.so (declared in include/lbfgs_b200.h).
//
// Build (see lbfgspp_b200/build.py):
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -shared -Xcompiler -fPIC ... -lnccl
//
// Kernel inventory (all HBM-bound streaming kernels; algorithmic words moved per element in brackets):
//   k_trial<OBJ>      x = xp + step*d ; g = grad f(x) ; {f, g.d, g.g, x.x}      [R 2 + W 2 (+data)]
//   k_dot3 / k_dot    reductions for user functors                              [R 3 / R 2]
//   k_axpy_out, k_scale_out                                                      [R 2 W 1 / R 1 W 1]
//   k_update          s = x-xp, y = g-gp -> ring slot ; {s.y, y.y}               [R 4 + W 2]
//   k_hv_stage<KIND>  one fused AXPY+dot stage of the two-loop recursion         [R 3 + W 1]
//   (k_gram_dots, k_gram_fold, k_gram_combine live in two_loop_gram.cuh; the device-resident solve in persist.cuh; the built-in
//   objectives and the steps k_trial shares with the resident solve in objectives.cuh, their id dispatch and checks in internal.cuh)
#include "internal.cuh"
#include "two_loop_gram.cuh"
#include "../../include/LBFGSpp/LoopRules.h"

using namespace lb;

// grid for a streaming kernel over n elements: a multiple of the SM count, capped so that every CTA has
// at least a few packs; 4 CTAs of 256 threads per SM are resident (register budget <= 64/thread).
constexpr int kCtasPerSmCap = 8;   // streaming grids: at most this many CTAs per SM
static int grid_for(const lbfgs_b200_ctx* ctx, int64_t n, int packs_per_thread = 4)
{
    const int64_t packs = (n + 3) / 4;
    const int64_t want = (packs + (int64_t)kThreads * packs_per_thread - 1) / ((int64_t)kThreads * packs_per_thread);
    const int64_t cap = (int64_t)ctx->sm_count * kCtasPerSmCap;
    int64_t g = want < 1 ? 1 : want;
    if (g > cap) g = cap;
    if (g > ctx->sm_count) g = (g / ctx->sm_count) * ctx->sm_count;  // whole waves
    if (g > kMaxBlocks) g = kMaxBlocks;
    return (int)g;
}

static lbfgs_b200_status post_launch(lbfgs_b200_ctx* ctx, const char* what)
{
    ctx->launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, LBFGS_B200_ERR_CUDA, "launch of %s failed: %s", what, cudaGetErrorString(e));
    return LBFGS_B200_OK;
}

// ReduceBuf for the next reducing launch: in p2p mode it carries the peer table and a fresh epoch
// to_host: the kernel's last CTA also publishes result[] in the mapped mailbox (not possible when a separate NCCL
// all-reduce still has to run after the kernel)
static bool mail_ok(const lbfgs_b200_ctx* ctx) { return ctx->nranks == 1 || ctx->x_active; }
static ReduceBuf next_rb(lbfgs_b200_ctx* ctx, bool to_host = false)
{
    ReduceBuf rb = ctx->rb;
    if (ctx->x_active) { rb.xc = ctx->x_comm; rb.epoch = ++ctx->x_epoch; }
    if (to_host && mail_ok(ctx))
    {
        rb.mail_vals = ctx->d_mail->vals;
        rb.mail_word = const_cast<unsigned long long*>(&ctx->d_mail->word);
        rb.mail_seq = ++ctx->mail_seq;
    }
    return rb;
}

// wait until the kernel that carries the current mail_seq has published; h_result mirrors the values afterwards
static lbfgs_b200_status wait_mail(lbfgs_b200_ctx* ctx, int count)
{
    const unsigned long long want = ctx->mail_seq;
    unsigned spins = 0;
    while (ctx->h_mail->word != want)
    {
        if ((++spins & 0x3fff) == 0)
        {
            cudaError_t e = cudaStreamQuery(ctx->stream);
            if (e != cudaSuccess && e != cudaErrorNotReady)
                return fail(ctx, LBFGS_B200_ERR_CUDA, "stream failed while waiting for a result: %s", cudaGetErrorString(e));
            if (e == cudaSuccess && ctx->h_mail->word != want)
                return fail(ctx, LBFGS_B200_ERR_CUDA, "kernel finished without publishing its result (sequence %llu)", want);
        }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    for (int k = 0; k < count; k++) ctx->h_result[k] = ctx->h_mail->vals[k];
    return LBFGS_B200_OK;
}

// copy result slots to the host and wait
static lbfgs_b200_status fetch_result(lbfgs_b200_ctx* ctx, int count)
{
    CU(ctx, cudaMemcpyAsync(ctx->h_result, ctx->rb.result, sizeof(double) * count, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return LBFGS_B200_OK;
}

// host receives `count` result slots: mailbox when the kernel delivered there, else memcpy + synchronise
static lbfgs_b200_status receive(lbfgs_b200_ctx* ctx, int count)
{
    if (mail_ok(ctx)) return wait_mail(ctx, count);
    return fetch_result(ctx, count);
}

// sum the first `count` result slots over all ranks (no-op on one GPU, and in p2p mode where the kernel did it)
static lbfgs_b200_status allreduce_result(lbfgs_b200_ctx* ctx, int count)
{
    if (ctx->nranks > 1 && !ctx->x_active)
        NC(ctx, ncclAllReduce(ctx->rb.result, ctx->rb.result, count, ncclDouble, ncclSum, ctx->comm, ctx->stream));
    return LBFGS_B200_OK;
}

// =====================================================================================================
// level-1 kernels
// =====================================================================================================
template <class T, bool VEC>
__global__ void __launch_bounds__(kThreads) k_axpy_out(int64_t n, const T* __restrict__ a, T s, const T* __restrict__ b, T* out)
{
    const int64_t packs = (n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        const Pack<T> pa = load4<T, Hint::Stream, VEC>(a, i0, cnt), pb = load4<T, Hint::Stream, VEC>(b, i0, cnt);
        Pack<T> r;
#pragma unroll
        for (int k = 0; k < 4; k++) r.v[k] = pa.v[k] + s * pb.v[k];
        store4<T, Hint::Plain, VEC>(out, i0, cnt, r);
    }
}

template <class T, bool VEC>
__global__ void __launch_bounds__(kThreads) k_scale_out(int64_t n, T s, const T* __restrict__ a, T* out)
{
    const int64_t packs = (n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        Pack<T> r = load4<T, Hint::Stream, VEC>(a, i0, cnt);
#pragma unroll
        for (int k = 0; k < 4; k++) r.v[k] = s * r.v[k];
        store4<T, Hint::Plain, VEC>(out, i0, cnt, r);
    }
}

// NV = 1: a.b ; NV = 3: {a.b, a.a, c.c}
template <class T, int NV, bool VEC>
__global__ void __launch_bounds__(kThreads) k_dots(int64_t n, const T* __restrict__ a, const T* __restrict__ b,
                                                   const T* __restrict__ c, ReduceBuf rb)
{
    T acc[NV];
#pragma unroll
    for (int k = 0; k < NV; k++) acc[k] = T(0);
    const int64_t packs = (n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
#pragma unroll 2
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        const Pack<T> pa = load4<T, Hint::Stream, VEC>(a, i0, cnt), pb = load4<T, Hint::Stream, VEC>(b, i0, cnt);
#pragma unroll
        for (int k = 0; k < 4; k++) acc[0] += pa.v[k] * pb.v[k];
        if constexpr (NV == 3)
        {
            const Pack<T> pc = load4<T, Hint::Stream, VEC>(c, i0, cnt);
#pragma unroll
            for (int k = 0; k < 4; k++)
            {
                acc[1] += pa.v[k] * pa.v[k];
                acc[2] += pc.v[k] * pc.v[k];
            }
        }
    }
    double dacc[NV];
#pragma unroll
    for (int k = 0; k < NV; k++) dacc[k] = (double)acc[k];
    grid_reduce<NV>(dacc, rb);
}

// =====================================================================================================
// halo exchange for neighbour-coupled objectives under n-sharding (SURVEY.md 8e: one element per side per evaluation)
//   a = xp (or x), b = d (or nullptr): every rank publishes {a[0], b[0], a[n-1], b[n-1]} and receives its neighbours' four.
// =====================================================================================================
template <class T>
__global__ void k_halo_pack(int64_t n, const T* __restrict__ a, const T* __restrict__ b, double* __restrict__ halo)
{
    if (threadIdx.x == 0)
    {
        halo[0] = (double)a[0];
        halo[1] = b ? (double)b[0] : 0.0;
        halo[2] = (double)a[n - 1];
        halo[3] = b ? (double)b[n - 1] : 0.0;
    }
}

// peer-memory variant: one warp; lane 0 talks to the left neighbour, lane 1 to the right one.  Uses the inbox slot of this
// launch's epoch exactly like xrank_allreduce (every rank issues the same sequence of exchanges, so epochs agree).
template <class T>
__global__ void k_halo_exchange(int64_t n, const T* __restrict__ a, const T* __restrict__ b, double* __restrict__ halo,
                                const XComm* __restrict__ xc, unsigned long long epoch)
{
    const int lane = threadIdx.x;
    if (lane > 1) return;
    const int me = xc->rank, R = xc->nranks, slot = (int)(epoch % kXRing);
    const int nb = (lane == 0) ? me - 1 : me + 1;
    double* mine = halo + 4 + 4 * lane;   // [4..7] from the left, [8..11] from the right
    if (nb < 0 || nb >= R)
    {
        for (int k = 0; k < 4; k++) mine[k] = 0.0;
        return;
    }
    const double v[4] = {(double)a[0], b ? (double)b[0] : 0.0, (double)a[n - 1], b ? (double)b[n - 1] : 0.0};
    for (int k = 0; k < 4; k++) xc->inbox[nb]->vals[slot][me][k] = v[k];
    __threadfence_system();
    st_release_sys(&xc->inbox[nb]->flag[slot][me], epoch);
    const unsigned long long* f = &xc->inbox[me]->flag[slot][nb];
    while (ld_acquire_sys(f) != epoch) {}
    for (int k = 0; k < 4; k++) mine[k] = ld_volatile_f64(&xc->inbox[me]->vals[slot][nb][k]);
}

// =====================================================================================================
// fused line-search trial  (x = xp + step*d ; g = grad f(x) ; {f, g.d, g.g, x.x})
//   TRIAL = false: plain objective evaluation at x (no xp/d, no x store), reduces {f, -, g.g, x.x}
// =====================================================================================================
template <class T, class OBJ, bool TRIAL, bool VEC>
__global__ void __launch_bounds__(kThreads) k_trial(OBJ obj, int64_t n, const T* __restrict__ xp, const T* __restrict__ d,
                                                    T step, T* __restrict__ x, T* __restrict__ g, ReduceBuf rb)
{
    T acc[4] = {T(0), T(0), T(0), T(0)};
    const int64_t packs = (n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
#pragma unroll 2
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        T xv[4], dv[4] = {T(0), T(0), T(0), T(0)}, gv[4];
        T xl = T(0), xr = T(0);
        if (TRIAL)
        {
            const Pack<T> px = load4<T, Hint::Stream, VEC>(xp, i0, cnt), pd = load4<T, Hint::Stream, VEC>(d, i0, cnt);
#pragma unroll
            for (int k = 0; k < 4; k++) { dv[k] = pd.v[k]; xv[k] = px.v[k] + step * pd.v[k]; }
            if constexpr (OBJ::kHalo) pack_neighbours<true>(obj, i0, n, step, [&](int j) { return xp[i0 + j] + step * d[i0 + j]; }, xl, xr);
        }
        else
        {
            const Pack<T> px = load4<T, Hint::Stream, VEC>(x, i0, cnt);
#pragma unroll
            for (int k = 0; k < 4; k++) xv[k] = px.v[k];
            if constexpr (OBJ::kHalo) pack_neighbours<false>(obj, i0, n, step, [&](int j) { return x[i0 + j]; }, xl, xr);
        }
        eval_pack(obj, i0, cnt, xv, xl, xr, dv, gv, acc);
        Pack<T> pg, pxo;
#pragma unroll
        for (int k = 0; k < 4; k++) { pg.v[k] = gv[k]; pxo.v[k] = xv[k]; }
        if (TRIAL) store4<T, Hint::Plain, VEC>(x, i0, cnt, pxo);
        store4<T, Hint::Plain, VEC>(g, i0, cnt, pg);
    }
    double dacc[4] = {(double)acc[0], (double)acc[1], (double)acc[2], (double)acc[3]};
    grid_reduce<4>(dacc, rb);
}

// =====================================================================================================
// OWL-QN (F = f + lam |x|_1; the expressions of LBFGSpp/OWLQNCore.h).  The pseudo-gradient is never stored: each pass forms it from
// the x and g it reads.
// Per-coordinate weights (F = f + lam sum_i w_i |x_i|): each pass has a weighted form (the _w kernels) that reads w on the same packs,
// one more word per coordinate, forms lam_i = lam * w_i (owlqn_lam_i), reports sum w_i |x_i| in place of |x|_1, and leaves the
// coordinates with lam_i == 0 unprojected and unconstrained (owlqn_point_w, owlqn_constrain_w).  Both forms keep the launch geometry,
// element ownership and summation order, so w = 1 reproduces the unweighted bits.  The projection, the sums and the pseudo-gradient
// passes are one body each, compiled without weights (W = false: lam on every coordinate, w never read) and with them.
// =====================================================================================================
// fused projected trial for a built-in objective: x = pi(xp + step d; xi(xp, pgp)); g = grad f(x);
// {f, |x|_1, pgp.(x - xp), pg.pg, x.x}                                                              [R 3 + W 2 (+data)]
template <class T, class OBJ, bool VEC>
__global__ void __launch_bounds__(kThreads) k_owlqn_trial(OBJ obj, int64_t n, const T* __restrict__ xp, const T* __restrict__ d,
                                                          const T* __restrict__ gp, T step, T lam, T* __restrict__ x, T* __restrict__ g,
                                                          ReduceBuf rb)
{
    T acc[5] = {T(0), T(0), T(0), T(0), T(0)};
    const int64_t packs = (n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
#pragma unroll 2
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        const Pack<T> pxp = load4<T, Hint::Stream, VEC>(xp, i0, cnt), pd = load4<T, Hint::Stream, VEC>(d, i0, cnt),
                      pgp = load4<T, Hint::Stream, VEC>(gp, i0, cnt);
        T xv[4], gv[4];
        eval_pack_owlqn(obj, i0, n, cnt, pxp.v, pd.v, pgp.v, step, lam,
                        [&](int j) { return LBFGSpp::owlqn_point(xp[i0 + j], d[i0 + j], gp[i0 + j], step, lam); }, xv, gv, acc);
        Pack<T> pg, pxo;
#pragma unroll
        for (int k = 0; k < 4; k++) { pg.v[k] = gv[k]; pxo.v[k] = xv[k]; }
        store4<T, Hint::Plain, VEC>(x, i0, cnt, pxo);
        store4<T, Hint::Plain, VEC>(g, i0, cnt, pg);
    }
    double dacc[5] = {(double)acc[0], (double)acc[1], (double)acc[2], (double)acc[3], (double)acc[4]};
    grid_reduce<5>(dacc, rb);
}

// The weighted trial is a kernel of its own beside the unweighted one: one body behind the weight flag took the vectorised fp32
// tridiagonal trial from 5 to 4 CTAs per SM and the vectorised fp64 chained-Rosenbrock weighted trial from 3 to 2 (DESIGN.md, §8h).
//
// weighted fused projected trial                                                                   [R 4 + W 2 (+data)]
template <class T, class OBJ, bool VEC>
__global__ void __launch_bounds__(kThreads) k_owlqn_trial_w(OBJ obj, int64_t n, const T* __restrict__ xp, const T* __restrict__ d,
                                                            const T* __restrict__ gp, T step, T lam, const T* __restrict__ w,
                                                            T* __restrict__ x, T* __restrict__ g, ReduceBuf rb)
{
    T acc[5] = {T(0), T(0), T(0), T(0), T(0)};
    const int64_t packs = (n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
#pragma unroll 2
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        const Pack<T> pxp = load4<T, Hint::Stream, VEC>(xp, i0, cnt), pd = load4<T, Hint::Stream, VEC>(d, i0, cnt),
                      pgp = load4<T, Hint::Stream, VEC>(gp, i0, cnt), pw = load4<T, Hint::Stream, VEC>(w, i0, cnt);
        T xv[4], gv[4];
        // the neighbours of a coupled objective are projected under their own weights
        const auto at = [&](int j) {
            return LBFGSpp::owlqn_point_w(xp[i0 + j], d[i0 + j], gp[i0 + j], step, LBFGSpp::owlqn_lam_i(lam, w[i0 + j]));
        };
        eval_pack_owlqn_w(obj, i0, n, cnt, pxp.v, pd.v, pgp.v, pw.v, step, lam, at, xv, gv, acc);
        Pack<T> pg, pxo;
#pragma unroll
        for (int k = 0; k < 4; k++) { pg.v[k] = gv[k]; pxo.v[k] = xv[k]; }
        store4<T, Hint::Plain, VEC>(x, i0, cnt, pxo);
        store4<T, Hint::Plain, VEC>(g, i0, cnt, pg);
    }
    double dacc[5] = {(double)acc[0], (double)acc[1], (double)acc[2], (double)acc[3], (double)acc[4]};
    grid_reduce<5>(dacc, rb);
}

// the projection alone, for any objective: x = pi(xp + step d; xi(xp, pgp)); {|x|_1, pgp.(x - xp)}    [R 3 (+W 1) + W 1]
template <class T, bool VEC, bool W>
__device__ __forceinline__ void owlqn_project_body(int64_t n, const T* xp, const T* d, const T* gp, T step, T lam, const T* w, T* x,
                                                   const ReduceBuf& rb)
{
    T acc[2] = {T(0), T(0)};
    const int64_t packs = (n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
#pragma unroll 2
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        const Pack<T> pxp = load4<T, Hint::Stream, VEC>(xp, i0, cnt), pd = load4<T, Hint::Stream, VEC>(d, i0, cnt),
                      pgp = load4<T, Hint::Stream, VEC>(gp, i0, cnt);
        Pack<T> pw;
        if constexpr (W) pw = load4<T, Hint::Stream, VEC>(w, i0, cnt);
        Pack<T> px;
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            const T lk = W ? LBFGSpp::owlqn_lam_i(lam, pw.v[k]) : lam;
            const T pgk = LBFGSpp::owlqn_pg(pxp.v[k], pgp.v[k], lk);
            px.v[k] = (k < cnt) ? (!W || lk > T(0) ? LBFGSpp::owlqn_project(pxp.v[k] + step * pd.v[k], LBFGSpp::owlqn_orthant(pxp.v[k], pgk))
                                                   : pxp.v[k] + step * pd.v[k])
                                : T(0);
            const T ax = px.v[k] < T(0) ? -px.v[k] : px.v[k];
            acc[0] += W ? pw.v[k] * ax : ax;
            acc[1] += pgk * (px.v[k] - pxp.v[k]);
        }
        store4<T, Hint::Plain, VEC>(x, i0, cnt, px);
    }
    double dacc[2] = {(double)acc[0], (double)acc[1]};
    grid_reduce<2>(dacc, rb);
}
template <class T, bool VEC>
__global__ void __launch_bounds__(kThreads) k_owlqn_project(int64_t n, const T* __restrict__ xp, const T* __restrict__ d,
                                                            const T* __restrict__ gp, T step, T lam, T* __restrict__ x, ReduceBuf rb)
{
    owlqn_project_body<T, VEC, false>(n, xp, d, gp, step, lam, nullptr, x, rb);
}
template <class T, bool VEC>
__global__ void __launch_bounds__(kThreads) k_owlqn_project_w(int64_t n, const T* __restrict__ xp, const T* __restrict__ d,
                                                              const T* __restrict__ gp, T step, T lam, const T* __restrict__ w,
                                                              T* __restrict__ x, ReduceBuf rb)
{
    owlqn_project_body<T, VEC, true>(n, xp, d, gp, step, lam, w, x, rb);
}

// the sums at a point: {|x|_1, pg.pg, x.x}, with W also the number of weights owlqn_weight_ok refuses; START also writes the first
// search's direction d = -pg                                                                             [R 2 (+W 1) (+W 1)]
template <class T, bool START, bool VEC, bool W>
__device__ __forceinline__ void owlqn_sums_body(int64_t n, const T* x, const T* g, T lam, const T* w,
                                                T* d, const ReduceBuf& rb)
{
    constexpr int NS = W ? 4 : 3;
    T acc[NS] = {T(0), T(0), T(0)};
    const int64_t packs = (n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
#pragma unroll 2
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        const Pack<T> px = load4<T, Hint::Stream, VEC>(x, i0, cnt), pg = load4<T, Hint::Stream, VEC>(g, i0, cnt);
        Pack<T> pw;
        if constexpr (W) pw = load4<T, Hint::Stream, VEC>(w, i0, cnt);
        Pack<T> pd;
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            const T pgk = LBFGSpp::owlqn_pg(px.v[k], pg.v[k], W ? LBFGSpp::owlqn_lam_i(lam, pw.v[k]) : lam);
            pd.v[k] = -pgk;
            const T ax = px.v[k] < T(0) ? -px.v[k] : px.v[k];
            acc[0] += W ? pw.v[k] * ax : ax;
            acc[1] += pgk * pgk;
            acc[2] += px.v[k] * px.v[k];
            if constexpr (W) acc[3] += LBFGSpp::owlqn_weight_ok(lam, pw.v[k]) ? T(0) : T(1);   // the lanes past cnt read w = 0
        }
        if (START) store4<T, Hint::Plain, VEC>(d, i0, cnt, pd);
    }
    double dacc[NS];
#pragma unroll
    for (int k = 0; k < NS; k++) dacc[k] = (double)acc[k];
    grid_reduce<NS>(dacc, rb);
}
template <class T, bool START, bool VEC>
__global__ void __launch_bounds__(kThreads) k_owlqn_sums(int64_t n, const T* __restrict__ x, const T* __restrict__ g, T lam,
                                                         T* __restrict__ d, ReduceBuf rb)
{
    owlqn_sums_body<T, START, VEC, false>(n, x, g, lam, nullptr, d, rb);
}
template <class T, bool START, bool VEC>
__global__ void __launch_bounds__(kThreads) k_owlqn_sums_w(int64_t n, const T* __restrict__ x, const T* __restrict__ g, T lam,
                                                           const T* __restrict__ w, T* __restrict__ d, ReduceBuf rb)
{
    owlqn_sums_body<T, START, VEC, true>(n, x, g, lam, w, d, rb);
}

// pg(x, g) into out (the spare ring column), for the dots round that follows a pair the curvature gate refused     [R 2 (+W 1) + W 1]
template <class T, bool W>
__device__ __forceinline__ void owlqn_pg_body(int64_t n, const T* x, const T* g, T lam, const T* w,
                                              T* out)
{
    const int64_t stride = (int64_t)gridDim.x * kThreads;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride)
        out[i] = LBFGSpp::owlqn_pg(x[i], g[i], W ? LBFGSpp::owlqn_lam_i(lam, w[i]) : lam);
}
template <class T>
__global__ void __launch_bounds__(kThreads) k_owlqn_pg(int64_t n, const T* __restrict__ x, const T* __restrict__ g, T lam, T* __restrict__ out)
{
    owlqn_pg_body<T, false>(n, x, g, lam, nullptr, out);
}
template <class T>
__global__ void __launch_bounds__(kThreads) k_owlqn_pg_w(int64_t n, const T* __restrict__ x, const T* __restrict__ g, T lam,
                                                         const T* __restrict__ w, T* __restrict__ out)
{
    owlqn_pg_body<T, true>(n, x, g, lam, w, out);
}

// =====================================================================================================
// the S/Y ring
// =====================================================================================================
// Device-resident scalars of BFGSMat (BFGSMat.h:35-48): theta, ys[], alpha[] indexed by PHYSICAL slot.
// The ring has M = m+1 physical columns so that the pair of an iteration can be written speculatively into
// the free slot `head` before the curvature gate (LBFGS.h:161) is known; a rejected pair simply leaves
// `head` where it was and the m older pairs untouched (the reference would not have called add_correction).

// s = x - xp ; y = g - gp -> slot ; {s.y, y.y}
template <class T, bool VEC>
__global__ void __launch_bounds__(kThreads) k_update(int64_t n, const T* __restrict__ x, const T* __restrict__ xp,
                                                     const T* __restrict__ g, const T* __restrict__ gp,
                                                     T* __restrict__ s_out, T* __restrict__ y_out, ReduceBuf rb)
{
    T acc[2] = {T(0), T(0)};
    const int64_t packs = (n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
#pragma unroll 2
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        const Pack<T> a = load4<T, Hint::Stream, VEC>(x, i0, cnt), b = load4<T, Hint::Stream, VEC>(xp, i0, cnt);
        const Pack<T> c = load4<T, Hint::Stream, VEC>(g, i0, cnt), e = load4<T, Hint::Stream, VEC>(gp, i0, cnt);
        Pack<T> s, y;
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            s.v[k] = a.v[k] - b.v[k];
            y.v[k] = c.v[k] - e.v[k];
            acc[0] += s.v[k] * y.v[k];
            acc[1] += y.v[k] * y.v[k];
        }
        store4<T, Hint::Plain, VEC>(s_out, i0, cnt, s);
        store4<T, Hint::Plain, VEC>(y_out, i0, cnt, y);
    }
    double dacc[2] = {(double)acc[0], (double)acc[1]};
    grid_reduce<2>(dacc, rb);
}

// {s.y, y.y} of an explicitly given pair while copying it into the slot (BFGSMat::add_correction)
template <class T, bool VEC>
__global__ void __launch_bounds__(kThreads) k_add_pair(int64_t n, const T* __restrict__ s, const T* __restrict__ y,
                                                       T* __restrict__ s_out, T* __restrict__ y_out, ReduceBuf rb)
{
    T acc[2] = {T(0), T(0)};
    const int64_t packs = (n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (n - i0 >= 4) ? 4 : int(n - i0);
        const Pack<T> a = load4<T, Hint::Stream, VEC>(s, i0, cnt), c = load4<T, Hint::Stream, VEC>(y, i0, cnt);
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            acc[0] += a.v[k] * c.v[k];
            acc[1] += c.v[k] * c.v[k];
        }
        store4<T, Hint::Plain, VEC>(s_out, i0, cnt, a);
        store4<T, Hint::Plain, VEC>(y_out, i0, cnt, c);
    }
    double dacc[2] = {(double)acc[0], (double)acc[1]};
    grid_reduce<2>(dacc, rb);
}

// gate + ys/theta bookkeeping from the reduced {s.y, y.y}: one thread (runs after the all-reduce)
template <class T>
__global__ void k_commit_pair(const double* result, T eps, int gate, T* ys_slot, T* theta, int* accepted,
                              double* mail_vals, int* mail_flag, unsigned long long* mail_word, unsigned long long mail_seq)
{
    const T sy = (T)result[0], yy = (T)result[1];
    const bool ok = gate ? LBFGSpp::curvature_ok(sy, yy, eps) : true;
    if (ok)
    {
        *ys_slot = sy;
        *theta = yy / sy;
    }
    *accepted = ok ? 1 : 0;
    if (mail_seq != 0ull)
    {
        mail_vals[0] = result[0];
        mail_vals[1] = result[1];
        *mail_flag = ok ? 1 : 0;
        __threadfence_system();
        st_release_sys(mail_word, mail_seq);
    }
}

// ----------------------------------------------------------------------------- literal two-loop stages
// One launch per history column.  Stage kinds (q lives in `res`, updated in place):
//   FIRST : q = a*v                                       ; dot(B, q)
//   BACK  : alpha_j = dot_prev/ys_j ; q -= alpha_j*A      ; dot(B, q)          A = y_j, B = s_{j-1 older}
//   MID   : alpha_j = dot_prev/ys_j ; q = (q - alpha_j*A)/theta ; dot(B, q)    A = y_oldest, B = y_oldest
//   FWD   : beta = dot_prev/ys_j ; q += (alpha_j - beta)*A ; dot(B, q)         A = s_j, B = y_{j+1 newer} (or v)
// The coefficient is recomputed from the previous stage's reduced dot by every thread (identical arithmetic),
// so the only dependency between stages is stream order -- no host round trip (BFGSMat.h:283-301).
enum { HV_FIRST = 0, HV_BACK = 1, HV_MID = 2, HV_FWD = 3, HV_ONLY = 4 };

template <class T> struct StageArgs
{
    int64_t n;
    const T* v;       // FIRST/ONLY: input vector
    T a;              // FIRST/ONLY: scale
    T* q;             // running vector (res)
    const T* A;       // axpy column
    const T* B;       // dot column (nullptr: no dot)
    const double* dot_prev;  // reduced dot of the previous stage
    const T* ys_j;    // &ys[j]
    T* alpha_j;       // &alpha[j]
    const T* theta;
};

template <class T, int KIND, bool VEC>
__global__ void __launch_bounds__(kThreads) k_hv_stage(StageArgs<T> s, ReduceBuf rb)
{
    T coef = T(0), theta = T(1);
    if (KIND == HV_BACK || KIND == HV_MID)
    {
        coef = (T)(*s.dot_prev) / *s.ys_j;  // alpha_j = s_j'q / ys_j   (BFGSMat.h:288, a division)
        if (blockIdx.x == 0 && threadIdx.x == 0) *s.alpha_j = coef;
    }
    if (KIND == HV_FWD)
    {
        const T beta = (T)(*s.dot_prev) / *s.ys_j;  // BFGSMat.h:298
        coef = *s.alpha_j - beta;
    }
    if (KIND == HV_MID || KIND == HV_ONLY) theta = *s.theta;

    T acc = T(0);
    const int64_t packs = (s.n + 3) >> 2, stride = (int64_t)gridDim.x * kThreads;
#pragma unroll 2
    for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < packs; p += stride)
    {
        const int64_t i0 = p << 2;
        const int cnt = (s.n - i0 >= 4) ? 4 : int(s.n - i0);
        Pack<T> q;
        if (KIND == HV_FIRST || KIND == HV_ONLY)
        {
            const Pack<T> pv = load4<T, Hint::Stream, VEC>(s.v, i0, cnt);
#pragma unroll
            for (int k = 0; k < 4; k++) q.v[k] = (KIND == HV_ONLY) ? (s.a * pv.v[k]) / theta : s.a * pv.v[k];
        }
        else
        {
            q = load4<T, Hint::Keep, VEC>(s.q, i0, cnt);
            const Pack<T> pa = load4<T, Hint::Stream, VEC>(s.A, i0, cnt);
#pragma unroll
            for (int k = 0; k < 4; k++)
            {
                if (KIND == HV_BACK) q.v[k] = q.v[k] - coef * pa.v[k];
                if (KIND == HV_MID) q.v[k] = (q.v[k] - coef * pa.v[k]) / theta;
                if (KIND == HV_FWD) q.v[k] = q.v[k] + coef * pa.v[k];
            }
        }
        if (s.B != nullptr)
        {
            const Pack<T> pb = load4<T, Hint::Stream, VEC>(s.B, i0, cnt);
#pragma unroll
            for (int k = 0; k < 4; k++) acc += pb.v[k] * q.v[k];
        }
        store4<T, Hint::Keep, VEC>(s.q, i0, cnt, q);
    }
    if (s.B != nullptr)
    {
        double dacc[1] = {(double)acc};
        grid_reduce<1>(dacc, rb);
    }
}

// =====================================================================================================
// C ABI: context, memory, communicator
// =====================================================================================================
extern "C" {

const char* lbfgs_b200_version(void) { return "lbfgs_b200 0.1 (sm_90a)"; }

lbfgs_b200_status lbfgs_b200_ctx_create(lbfgs_b200_ctx** out, int device, void* stream)
{
    if (!out) return fail(nullptr, LBFGS_B200_ERR_INVALID, "ctx_create: out is NULL");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, LBFGS_B200_ERR_CUDA, "no CUDA device available (%s); liblbfgs_b200 has no CPU fallback",
                    e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    if (device < 0 || device >= ndev) return fail(nullptr, LBFGS_B200_ERR_INVALID, "device %d out of range [0,%d)", device, ndev);
    lbfgs_b200_ctx* ctx = new (std::nothrow) lbfgs_b200_ctx();
    if (!ctx) return fail(nullptr, LBFGS_B200_ERR_ALLOC, "out of host memory");
    ctx->device = device;
#define CUC(call)                                                                                          \
    do {                                                                                                   \
        cudaError_t e__ = (call);                                                                          \
        if (e__ != cudaSuccess) {                                                                          \
            fail(nullptr, LBFGS_B200_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(e__));           \
            lbfgs_b200_ctx_destroy(ctx);                                                                   \
            return LBFGS_B200_ERR_CUDA;                                                                    \
        }                                                                                                  \
    } while (0)
    CUC(cudaSetDevice(device));
    cudaDeviceProp prop;
    CUC(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
    {
        fail(nullptr, LBFGS_B200_ERR_CUDA, "device %d is sm_%d%d; this library contains sm_90a code only", device, prop.major, prop.minor);
        lbfgs_b200_ctx_destroy(ctx);
        return LBFGS_B200_ERR_CUDA;
    }
    ctx->sm_count = prop.multiProcessorCount;
    if (stream) ctx->stream = static_cast<cudaStream_t>(stream);
    else { CUC(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)); ctx->own_stream = true; }
    CUC(cudaMalloc(&ctx->rb.partials, sizeof(double) * kMaxBlocks * kMaxRed));
    CUC(cudaMalloc(&ctx->rb.ticket, sizeof(unsigned)));
    CUC(cudaMalloc(&ctx->rb.result, sizeof(double) * 256));
    CUC(cudaMalloc(&ctx->d_flag, sizeof(int) * 16));
    CUC(cudaMalloc(&ctx->gram_partials, sizeof(double) * (size_t)ctx->sm_count * kMaxM * kGramVals));
    CUC(cudaMalloc(&ctx->gram_raw, sizeof(double) * kMaxM * kGramVals));
    CUC(cudaMalloc(&ctx->d_halo, sizeof(double) * kHaloDoubles));
    CUC(cudaMemsetAsync(ctx->d_halo, 0, sizeof(double) * kHaloDoubles, ctx->stream));
    CUC(cudaMemsetAsync(ctx->rb.ticket, 0, sizeof(unsigned), ctx->stream));
    CUC(cudaMemsetAsync(ctx->rb.result, 0, sizeof(double) * 256, ctx->stream));
    CUC(cudaMallocHost(&ctx->h_result, sizeof(double) * 256));
    CUC(cudaMallocHost(&ctx->h_flag, sizeof(int) * 16));
    CUC(cudaHostAlloc(&ctx->h_mail, sizeof(lbfgs_b200_ctx::Mail), cudaHostAllocMapped));
    memset((void*)ctx->h_mail, 0, sizeof(lbfgs_b200_ctx::Mail));
    CUC(cudaHostGetDevicePointer(&ctx->d_mail, ctx->h_mail, 0));
    CUC(cudaEventCreate(&ctx->ev0));
    CUC(cudaEventCreate(&ctx->ev1));
    CUC(cudaStreamSynchronize(ctx->stream));
#undef CUC
    *out = ctx;
    return LBFGS_B200_OK;
}

void lbfgs_b200_ctx_destroy(lbfgs_b200_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    pool_trim(ctx);
    if (ctx->comm) ncclCommDestroy(ctx->comm);
    for (int r = 0; r < kXMaxRanks; r++) if (ctx->x_peer[r]) cudaIpcCloseMemHandle(ctx->x_peer[r]);
    cudaFree(ctx->x_comm);
    cudaFree(ctx->x_inbox);
    cudaFree(ctx->rb.partials);
    cudaFree(ctx->rb.ticket);
    cudaFree(ctx->rb.result);
    cudaFree(ctx->d_flag);
    cudaFree(ctx->gram_partials);
    cudaFree(ctx->gram_raw);
    cudaFree(ctx->d_halo);
    if (ctx->h_result) cudaFreeHost(ctx->h_result);
    if (ctx->h_flag) cudaFreeHost(ctx->h_flag);
    if (ctx->h_mail) cudaFreeHost((void*)ctx->h_mail);
    for (int ph = 0; ph < 3; ph++) for (auto& sp : ctx->spans[ph]) { cudaEventDestroy(sp.a); cudaEventDestroy(sp.b); }
    for (auto& sp : ctx->free_spans) { cudaEventDestroy(sp.a); cudaEventDestroy(sp.b); }
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* lbfgs_b200_last_error(const lbfgs_b200_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }
void* lbfgs_b200_stream(const lbfgs_b200_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int lbfgs_b200_sm_count(const lbfgs_b200_ctx* ctx) { return ctx ? ctx->sm_count : 0; }
uint64_t lbfgs_b200_launch_count(const lbfgs_b200_ctx* ctx) { return ctx ? ctx->launches : 0; }

lbfgs_b200_status lbfgs_b200_malloc(lbfgs_b200_ctx* ctx, void** dptr, size_t bytes)
{
    REQUIRE(ctx, ctx && dptr, "malloc: NULL argument");
    CU(ctx, cudaSetDevice(ctx->device));
    // round up to a whole number of 256-byte lines so that ragged tails can be read as full packs by callers
    // (pool_alloc does the rounding); blocks come from / go back to the context's pool, see internal.cuh
    CU(ctx, pool_alloc(ctx, dptr, bytes));
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_free(lbfgs_b200_ctx* ctx, void* dptr)
{
    if (!dptr) return LBFGS_B200_OK;
    if (ctx) pool_free(ctx, dptr);
    else CU(ctx, cudaFree(dptr));
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_trim(lbfgs_b200_ctx* ctx)
{
    REQUIRE(ctx, ctx, "trim: NULL context");
    CU(ctx, cudaSetDevice(ctx->device));
    pool_trim(ctx);
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_malloc_host(lbfgs_b200_ctx* ctx, void** hptr, size_t bytes)
{
    REQUIRE(ctx, ctx && hptr, "malloc_host: NULL argument");
    CU(ctx, cudaMallocHost(hptr, bytes ? bytes : 1));
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_free_host(lbfgs_b200_ctx* ctx, void* hptr)
{
    if (!hptr) return LBFGS_B200_OK;
    CU(ctx, cudaFreeHost(hptr));
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_memcpy_h2d(lbfgs_b200_ctx* ctx, void* dst, const void* src, size_t bytes)
{
    CU(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_memcpy_d2h(lbfgs_b200_ctx* ctx, void* dst, const void* src, size_t bytes)
{
    CU(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_memcpy_d2d(lbfgs_b200_ctx* ctx, void* dst, const void* src, size_t bytes)
{
    CU(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_memset_zero(lbfgs_b200_ctx* ctx, void* dst, size_t bytes)
{
    CU(ctx, cudaMemsetAsync(dst, 0, bytes, ctx->stream));
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_sync(lbfgs_b200_ctx* ctx)
{
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return LBFGS_B200_OK;
}

lbfgs_b200_status lbfgs_b200_timer_start(lbfgs_b200_ctx* ctx)
{
    CU(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_timer_stop(lbfgs_b200_ctx* ctx, float* ms)
{
    CU(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    CU(ctx, cudaEventSynchronize(ctx->ev1));
    CU(ctx, cudaEventElapsedTime(ms, ctx->ev0, ctx->ev1));
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_profile_enable(lbfgs_b200_ctx* ctx, int on)
{
    REQUIRE(ctx, ctx != nullptr, "profile_enable: NULL context");
    ctx->profiling = on != 0;
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_profile_read(lbfgs_b200_ctx* ctx, int phase, double* total_ms, uint64_t* calls, int reset)
{
    REQUIRE(ctx, ctx && phase >= 0 && phase < 3, "profile_read: bad arguments");
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    for (auto& sp : ctx->spans[phase])
    {
        float ms = 0.f;
        CU(ctx, cudaEventElapsedTime(&ms, sp.a, sp.b));
        ctx->prof_ms[phase] += ms;
        ctx->prof_calls[phase]++;
        ctx->free_spans.push_back(sp);
    }
    ctx->spans[phase].clear();
    if (total_ms) *total_ms = ctx->prof_ms[phase];
    if (calls) *calls = ctx->prof_calls[phase];
    if (reset) { ctx->prof_ms[phase] = 0; ctx->prof_calls[phase] = 0; }
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_profile_bytes(lbfgs_b200_ctx* ctx, int phase, double* alg_bytes, int reset)
{
    REQUIRE(ctx, ctx && phase >= 0 && phase < 3 && alg_bytes, "profile_bytes: bad arguments");
    *alg_bytes = ctx->prof_bytes[phase];
    if (reset) ctx->prof_bytes[phase] = 0;
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_set_index_offset(lbfgs_b200_ctx* ctx, int64_t offset)
{
    REQUIRE(ctx, ctx != nullptr, "set_index_offset: NULL context");
    ctx->index_offset = offset;
    return LBFGS_B200_OK;
}

lbfgs_b200_status lbfgs_b200_set_global_extent(lbfgs_b200_ctx* ctx, int64_t offset, int64_t n_global)
{
    REQUIRE(ctx, ctx != nullptr && offset >= 0 && n_global >= offset, "set_global_extent: need 0 <= offset <= n_global");
    ctx->index_offset = offset;
    ctx->n_global = n_global;
    return LBFGS_B200_OK;
}

lbfgs_b200_status lbfgs_b200_comm_unique_id(void* unique_id_128)
{
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    ncclResult_t r = ncclGetUniqueId(&id);
    if (r != ncclSuccess) return fail(nullptr, LBFGS_B200_ERR_COMM, "ncclGetUniqueId failed: %s", ncclGetErrorString(r));
    memcpy(unique_id_128, &id, sizeof(id));
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_comm_init(lbfgs_b200_ctx* ctx, const void* unique_id_128, int rank, int nranks)
{
    REQUIRE(ctx, ctx && unique_id_128 && nranks >= 1 && rank >= 0 && rank < nranks, "comm_init: bad arguments");
    ncclUniqueId id;
    memcpy(&id, unique_id_128, sizeof(id));
    CU(ctx, cudaSetDevice(ctx->device));
    NC(ctx, ncclCommInitRank(&ctx->comm, nranks, id, rank));
    ctx->rank = rank;
    ctx->nranks = nranks;
    return LBFGS_B200_OK;
}
int lbfgs_b200_comm_size(const lbfgs_b200_ctx* ctx) { return ctx ? ctx->nranks : 0; }

lbfgs_b200_status lbfgs_b200_comm_p2p_export(lbfgs_b200_ctx* ctx, void* ipc_handle_64)
{
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    REQUIRE(ctx, ctx && ipc_handle_64, "comm_p2p_export: NULL argument");
    CU(ctx, cudaSetDevice(ctx->device));
    if (!ctx->x_inbox)
    {
        CU(ctx, cudaMalloc(&ctx->x_inbox, sizeof(XInbox)));
        CU(ctx, cudaMemset(ctx->x_inbox, 0, sizeof(XInbox)));
        CU(ctx, cudaDeviceSynchronize());
    }
    cudaIpcMemHandle_t hnd;
    CU(ctx, cudaIpcGetMemHandle(&hnd, ctx->x_inbox));
    memcpy(ipc_handle_64, &hnd, sizeof(hnd));
    return LBFGS_B200_OK;
}

lbfgs_b200_status lbfgs_b200_comm_p2p_attach(lbfgs_b200_ctx* ctx, const void* all_handles, int rank, int nranks)
{
    REQUIRE(ctx, ctx && all_handles && ctx->x_inbox, "comm_p2p_attach: export first");
    REQUIRE(ctx, nranks >= 1 && nranks <= kXMaxRanks && rank >= 0 && rank < nranks, "comm_p2p_attach: 1 <= nranks <= %d", kXMaxRanks);
    CU(ctx, cudaSetDevice(ctx->device));
    XComm host{};
    host.rank = rank;
    host.nranks = nranks;
    for (int r = 0; r < nranks; r++)
    {
        if (r == rank) { host.inbox[r] = ctx->x_inbox; continue; }
        cudaIpcMemHandle_t hnd;
        memcpy(&hnd, static_cast<const char*>(all_handles) + 64 * r, sizeof(hnd));
        void* p = nullptr;
        CU(ctx, cudaIpcOpenMemHandle(&p, hnd, cudaIpcMemLazyEnablePeerAccess));
        ctx->x_peer[r] = p;
        host.inbox[r] = static_cast<XInbox*>(p);
    }
    if (!ctx->x_comm) CU(ctx, cudaMalloc(&ctx->x_comm, sizeof(XComm)));
    CU(ctx, cudaMemcpy(ctx->x_comm, &host, sizeof(XComm), cudaMemcpyHostToDevice));
    ctx->rank = rank;
    ctx->nranks = nranks;
    ctx->x_epoch = 0;
    ctx->x_active = nranks > 1;
    return LBFGS_B200_OK;
}

}  // extern "C"

// =====================================================================================================
// typed implementations behind the f64 / f32 entry points
// =====================================================================================================
template <class T> static bool all_aligned(std::initializer_list<const void*> ps)
{
    for (const void* p : ps)
        if (p && !pack_aligned<T>(p)) return false;
    return true;
}

template <class T>
static lbfgs_b200_status do_dot(lbfgs_b200_ctx* ctx, int64_t n, const T* a, const T* b, T* out_host)
{
    REQUIRE(ctx, ctx && a && b && out_host && n >= 0, "dot: bad arguments");
    const int grid = grid_for(ctx, n);
    const ReduceBuf rb = next_rb(ctx, true);
    if (all_aligned<T>({a, b})) k_dots<T, 1, true><<<grid, kThreads, 0, ctx->stream>>>(n, a, b, nullptr, rb);
    else k_dots<T, 1, false><<<grid, kThreads, 0, ctx->stream>>>(n, a, b, nullptr, rb);
    if (auto st = post_launch(ctx, "k_dots<1>")) return st;
    if (auto st = allreduce_result(ctx, 1)) return st;
    if (auto st = receive(ctx, 1)) return st;
    *out_host = (T)ctx->h_result[0];
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_dot3(lbfgs_b200_ctx* ctx, int64_t n, const T* g, const T* d, const T* x, T* out3)
{
    REQUIRE(ctx, ctx && g && d && x && out3 && n >= 0, "dot3: bad arguments");
    const int grid = grid_for(ctx, n);
    const ReduceBuf rb = next_rb(ctx, true);
    if (all_aligned<T>({g, d, x})) k_dots<T, 3, true><<<grid, kThreads, 0, ctx->stream>>>(n, g, d, x, rb);
    else k_dots<T, 3, false><<<grid, kThreads, 0, ctx->stream>>>(n, g, d, x, rb);
    if (auto st = post_launch(ctx, "k_dots<3>")) return st;
    if (auto st = allreduce_result(ctx, 3)) return st;
    if (auto st = receive(ctx, 3)) return st;
    for (int k = 0; k < 3; k++) out3[k] = (T)ctx->h_result[k];
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_axpy_out(lbfgs_b200_ctx* ctx, int64_t n, const T* a, T s, const T* b, T* out)
{
    REQUIRE(ctx, ctx && a && b && out && n >= 0, "axpy_out: bad arguments");
    const int grid = grid_for(ctx, n);
    if (all_aligned<T>({a, b, out})) k_axpy_out<T, true><<<grid, kThreads, 0, ctx->stream>>>(n, a, s, b, out);
    else k_axpy_out<T, false><<<grid, kThreads, 0, ctx->stream>>>(n, a, s, b, out);
    return post_launch(ctx, "k_axpy_out");
}

template <class T>
static lbfgs_b200_status do_scale_out(lbfgs_b200_ctx* ctx, int64_t n, T s, const T* a, T* out)
{
    REQUIRE(ctx, ctx && a && out && n >= 0, "scale_out: bad arguments");
    const int grid = grid_for(ctx, n);
    if (all_aligned<T>({a, out})) k_scale_out<T, true><<<grid, kThreads, 0, ctx->stream>>>(n, s, a, out);
    else k_scale_out<T, false><<<grid, kThreads, 0, ctx->stream>>>(n, s, a, out);
    return post_launch(ctx, "k_scale_out");
}

// Boundary coordinates of the evaluation point to and from the neighbouring ranks (objectives.cuh: halo record).  Stream-ordered;
// in peer-memory mode it consumes one exchange epoch, with NCCL it is a grouped send/recv pair per neighbour.
template <class T>
static lbfgs_b200_status exchange_halo(lbfgs_b200_ctx* ctx, int64_t n, const T* a, const T* b)
{
    if (ctx->x_active)
    {
        k_halo_exchange<T><<<1, 32, 0, ctx->stream>>>(n, a, b, ctx->d_halo, ctx->x_comm, ++ctx->x_epoch);
        return post_launch(ctx, "k_halo_exchange");
    }
    REQUIRE(ctx, ctx->comm != nullptr, "halo exchange: no communicator attached");
    k_halo_pack<T><<<1, 32, 0, ctx->stream>>>(n, a, b, ctx->d_halo);
    if (auto st = post_launch(ctx, "k_halo_pack")) return st;
    CU(ctx, cudaMemsetAsync(ctx->d_halo + 4, 0, sizeof(double) * 8, ctx->stream));
    NC(ctx, ncclGroupStart());
    if (ctx->rank > 0)
    {
        NC(ctx, ncclSend(ctx->d_halo, 4, ncclDouble, ctx->rank - 1, ctx->comm, ctx->stream));
        NC(ctx, ncclRecv(ctx->d_halo + 4, 4, ncclDouble, ctx->rank - 1, ctx->comm, ctx->stream));
    }
    if (ctx->rank < ctx->nranks - 1)
    {
        NC(ctx, ncclSend(ctx->d_halo, 4, ncclDouble, ctx->rank + 1, ctx->comm, ctx->stream));
        NC(ctx, ncclRecv(ctx->d_halo + 8, 4, ncclDouble, ctx->rank + 1, ctx->comm, ctx->stream));
    }
    NC(ctx, ncclGroupEnd());
    return LBFGS_B200_OK;
}

template <class T, class OBJ, bool TRIAL>
static lbfgs_b200_status launch_trial(lbfgs_b200_ctx* ctx, const OBJ& obj, int64_t n, const T* xp, const T* d, T step,
                                      T* x, T* g, bool vec)
{
    const int grid = grid_for(ctx, n, 2);
    const ReduceBuf rb = next_rb(ctx, true);
    if (vec) k_trial<T, OBJ, TRIAL, true><<<grid, kThreads, 0, ctx->stream>>>(obj, n, xp, d, step, x, g, rb);
    else k_trial<T, OBJ, TRIAL, false><<<grid, kThreads, 0, ctx->stream>>>(obj, n, xp, d, step, x, g, rb);
    return post_launch(ctx, "k_trial");
}

template <class T, bool TRIAL>
static lbfgs_b200_status do_trial(lbfgs_b200_ctx* ctx, int objective, const T* data0, const T* data1, int64_t n,
                                  const T* xp, const T* d, T step, T* x, T* g, T* out_host)
{
    REQUIRE(ctx, ctx && x && g && out_host && n >= 1, "trial/objective: bad arguments");
    if (TRIAL) REQUIRE(ctx, xp && d, "trial: xp/d are NULL");
    return with_objective<T>(ctx, objective, [&](auto tag) -> lbfgs_b200_status {
        using OBJ = decltype(tag);
        ObjGeom<T> geo;
        if (auto st = objective_geometry<OBJ>(ctx, n, data0, data1, geo)) return st;
        if (OBJ::kHalo && ctx->nranks > 1)
        {
            if (auto st = exchange_halo<T>(ctx, n, TRIAL ? xp : x, TRIAL ? d : nullptr)) return st;
            geo.halo = ctx->d_halo;
        }
        ProfSpan span(ctx, PH_TRIAL, double(sizeof(T)) * double(n) * ((TRIAL ? 4.0 : 2.0) + OBJ::kDataVectors));
        if (auto st = launch_trial<T, OBJ, TRIAL>(ctx, OBJ{geo}, n, xp, d, step, x, g, all_aligned<T>({xp, d, x, g}))) return st;
        if (auto st = allreduce_result(ctx, 4)) return st;
        span.stop();
        if (auto st = receive(ctx, 4)) return st;
        for (int k = 0; k < 4; k++) out_host[k] = (T)ctx->h_result[k];
        if (!TRIAL) out_host[1] = T(0);
        return LBFGS_B200_OK;
    });
}

// ----------------------------------------------------------------------------- history
template <class T> static lbfgs_b200_status hist_check(lbfgs_b200_hist* h)
{
    if (!h || !h->ctx) return LBFGS_B200_ERR_INVALID;
    if (h->elem != (int)sizeof(T)) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "history holds %d-byte elements, called with %zu-byte type", h->elem, sizeof(T));
    return LBFGS_B200_OK;
}

template <class T> static lbfgs_b200_status gram_refresh(lbfgs_b200_hist* h);

// src: device doubles {s'y, y'y} of the pair sitting in slot h->head; nullptr = the reduction slots of the kernel just launched
// (still to be all-reduced), otherwise already global sums.
template <class T>
static lbfgs_b200_status commit_pair(lbfgs_b200_hist* h, T eps, int gate, int* accepted_host, T* sy_yy_host, const double* src = nullptr)
{
    lbfgs_b200_ctx* ctx = h->ctx;
    if (!src)
    {
        if (auto st = allreduce_result(ctx, 2)) return st;
        src = ctx->rb.result;
    }
    T* ys = static_cast<T*>(h->ys) + h->head;
    int ok = 0;
    if (mail_ok(ctx))
    {
        const unsigned long long seq = ++ctx->mail_seq;
        k_commit_pair<T><<<1, 1, 0, ctx->stream>>>(src, eps, gate, ys, static_cast<T*>(h->theta), ctx->d_flag,
                                                   ctx->d_mail->vals, &ctx->d_mail->flag,
                                                   const_cast<unsigned long long*>(&ctx->d_mail->word), seq);
        if (auto st = post_launch(ctx, "k_commit_pair")) return st;
        if (auto st = wait_mail(ctx, 2)) return st;
        ok = ctx->h_mail->flag;
    }
    else
    {
        k_commit_pair<T><<<1, 1, 0, ctx->stream>>>(src, eps, gate, ys, static_cast<T*>(h->theta), ctx->d_flag,
                                                   nullptr, nullptr, nullptr, 0ull);
        if (auto st = post_launch(ctx, "k_commit_pair")) return st;
        CU(ctx, cudaMemcpyAsync(ctx->h_flag, ctx->d_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CU(ctx, cudaMemcpyAsync(ctx->h_result, src, sizeof(double) * 2, cudaMemcpyDeviceToHost, ctx->stream));
        CU(ctx, cudaStreamSynchronize(ctx->stream));
        ok = ctx->h_flag[0];
    }
    if (ok)
    {
        // two pairs appended back to back: fold the earlier one while it is still the newest (age 0)
        if (h->pending >= 0)
            if (auto st = gram_refresh<T>(h)) return st;
        const int written = h->head;
        h->head = (h->head + 1) % h->M;
        if (h->ncorr < h->m) h->ncorr++;
        h->pending = written;
    }
    if (accepted_host) *accepted_host = ok;
    if (sy_yy_host) { sy_yy_host[0] = (T)ctx->h_result[0]; sy_yy_host[1] = (T)ctx->h_result[1]; }
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_hist_update(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, T eps,
                                        int* accepted_host, T* sy_yy_host)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, x && xp && g && gp, "hist_update: NULL vector");
    T* s_out = h->s_col<T>(h->head);
    T* y_out = h->y_col<T>(h->head);
    ProfSpan span(ctx, PH_UPDATE, double(sizeof(T)) * double(h->n) * 6.0);
    const int grid = grid_for(ctx, h->n, 2);
    const ReduceBuf rb = next_rb(ctx);
    if (all_aligned<T>({x, xp, g, gp}))
        k_update<T, true><<<grid, kThreads, 0, ctx->stream>>>(h->n, x, xp, g, gp, s_out, y_out, rb);
    else
        k_update<T, false><<<grid, kThreads, 0, ctx->stream>>>(h->n, x, xp, g, gp, s_out, y_out, rb);
    if (auto st = post_launch(ctx, "k_update")) return st;
    span.stop();
    return commit_pair<T>(h, eps, 1, accepted_host, sy_yy_host);
}

template <class T> static lbfgs_b200_status do_hist_add(lbfgs_b200_hist* h, const T* s, const T* y)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, s && y, "hist_add: NULL vector");
    const int grid = grid_for(ctx, h->n, 2);
    const ReduceBuf rb = next_rb(ctx);
    if (all_aligned<T>({s, y}))
        k_add_pair<T, true><<<grid, kThreads, 0, ctx->stream>>>(h->n, s, y, h->s_col<T>(h->head), h->y_col<T>(h->head), rb);
    else
        k_add_pair<T, false><<<grid, kThreads, 0, ctx->stream>>>(h->n, s, y, h->s_col<T>(h->head), h->y_col<T>(h->head), rb);
    if (auto st = post_launch(ctx, "k_add_pair")) return st;
    return commit_pair<T>(h, T(0), 0, nullptr, nullptr);
}

template <class T, int KIND>
static lbfgs_b200_status launch_stage(lbfgs_b200_ctx* ctx, const StageArgs<T>& s, bool vec)
{
    const int grid = grid_for(ctx, s.n, 2);
    const ReduceBuf rb = (s.B != nullptr) ? next_rb(ctx) : ctx->rb;
    if (vec) k_hv_stage<T, KIND, true><<<grid, kThreads, 0, ctx->stream>>>(s, rb);
    else k_hv_stage<T, KIND, false><<<grid, kThreads, 0, ctx->stream>>>(s, rb);
    if (auto st = post_launch(ctx, "k_hv_stage")) return st;
    if (s.B != nullptr) return allreduce_result(ctx, 1);
    return LBFGS_B200_OK;
}

// literal two-loop recursion, one stage kernel per column visit (2c+1 launches, no host sync in between)
template <class T>
static lbfgs_b200_status hv_two_loop(lbfgs_b200_hist* h, const T* v, T a, T* res, bool want_vdot)
{
    lbfgs_b200_ctx* ctx = h->ctx;
    const int c = h->ncorr;
    const bool vec = all_aligned<T>({v, res});
    T* ys = static_cast<T*>(h->ys);
    T* al = static_cast<T*>(h->alpha);
    StageArgs<T> s{};
    s.n = h->n; s.v = v; s.a = a; s.q = res; s.dot_prev = ctx->rb.result; s.theta = static_cast<T*>(h->theta);
    if (c == 0)
    {
        s.B = want_vdot ? v : nullptr;
        return launch_stage<T, HV_ONLY>(ctx, s, vec);
    }
    // FIRST: q = a*v ; dot(s_newest, q)
    s.B = h->s_col<T>(h->slot(0));
    if (auto st = launch_stage<T, HV_FIRST>(ctx, s, vec)) return st;
    // backward sweep, newest -> oldest (BFGSMat.h:285-290)
    for (int age = 0; age < c; age++)
    {
        const int j = h->slot(age);
        s.A = h->y_col<T>(j);
        s.ys_j = ys + j;
        s.alpha_j = al + j;
        if (age + 1 < c)
        {
            s.B = h->s_col<T>(h->slot(age + 1));
            if (auto st = launch_stage<T, HV_BACK>(ctx, s, vec)) return st;
        }
        else
        {
            s.B = h->y_col<T>(j);  // the forward sweep starts at the oldest pair (BFGSMat.h:293-298)
            if (auto st = launch_stage<T, HV_MID>(ctx, s, vec)) return st;
        }
    }
    // forward sweep, oldest -> newest (BFGSMat.h:296-301)
    for (int age = c - 1; age >= 0; age--)
    {
        const int j = h->slot(age);
        s.A = h->s_col<T>(j);
        s.ys_j = ys + j;
        s.alpha_j = al + j;
        s.B = (age > 0) ? h->y_col<T>(h->slot(age - 1)) : (want_vdot ? v : nullptr);
        if (auto st = launch_stage<T, HV_FWD>(ctx, s, vec)) return st;
    }
    return LBFGS_B200_OK;
}

// ----------------------------------------------------------------------------- Gram-form apply_Hv
template <class T> static void fill_slots(const lbfgs_b200_hist* h, unsigned char* slots)
{
    for (int age = 0; age < h->ncorr; age++) slots[age] = (unsigned char)h->slot(age);
}

// [S Y]'[v s_new y_new] (+ all-reduce).  v == nullptr: only the new pair's Gram row/column ("refresh").
// Speculative "update + dots" (form != nullptr): the pair (s, y) = (x - xp, v - gp) is formed on the fly into the spare slot
// h->head and takes part as the newest column, exactly as if it had been appended already; the caller commits or discards it.
template <class T> struct PairForm { const T* x; const T* xp; const T* gp; };

// k_gram_dots for `rounds` rounds of column pairs.  The opt-in for > 48 KB of dynamic shared memory is per device and
// instantiation: the context remembers which instantiations have it.
template <class T, bool FORM>
static lbfgs_b200_status launch_gram_dots(lbfgs_b200_ctx* ctx, const GramDotsArgs<T>& a, int rounds, int grid, int threads, size_t smem,
                                          const XComm* xc, unsigned long long epoch)
{
    const int r = rounds <= 1 ? 1 : rounds == 2 ? 2 : 3;
    const auto kernel = r == 1 ? k_gram_dots<T, 1, FORM> : r == 2 ? k_gram_dots<T, 2, FORM> : k_gram_dots<T, 3, FORM>;
    const unsigned bit = 1u << ((FORM ? 8 : 0) + (sizeof(T) == 8 ? 0 : 4) + r);
    if (!(ctx->smem_optin & bit))
    {
        CU(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ctx->smem_optin |= bit;
    }
    kernel<<<grid, threads, smem, ctx->stream>>>(a, ctx->gram_partials, ctx->rb.ticket, ctx->gram_raw, xc, epoch);
    return post_launch(ctx, FORM ? "k_gram_dots<FORM>" : "k_gram_dots");
}

template <class T>
static lbfgs_b200_status gram_dots(lbfgs_b200_hist* h, const T* v, const PairForm<T>* form = nullptr)
{
    lbfgs_b200_ctx* ctx = h->ctx;
    const int c = form ? (h->ncorr < h->m ? h->ncorr + 1 : h->m) : h->ncorr;
    GramDotsArgs<T> a{};
    a.n = h->n; a.ld = h->ld; a.v = v;
    a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y);
    a.c = c; a.new_slot = form ? h->head : h->pending;
    if (form)
    {
        a.fx = form->x; a.fxp = form->xp; a.fgp = form->gp;
        a.s_out = h->s_col<T>(h->head); a.y_out = h->y_col<T>(h->head);
    }
    // warps = (column pairs in flight) x (warps per column pair); as many of the 24 warp slots as divide evenly
    int split = 8;
    while (split > 1 && c * split > kGramMaxWarps) split >>= 1;
    a.split = split;
    a.cols_per_round = c < kGramMaxWarps / split ? c : kGramMaxWarps / split;
    a.use_tma = (v == nullptr || (reinterpret_cast<uintptr_t>(v) & 15) == 0) ? 1 : 0;
    if (form)
    {
        a.slots[0] = (unsigned char)h->head;                      // ages as they will be once the pair is committed
        for (int age = 1; age < c; age++) a.slots[age] = (unsigned char)h->slot(age - 1);
    }
    else
        fill_slots<T>(h, a.slots);
    const int rounds = (c + a.cols_per_round - 1) / a.cols_per_round;
    const int threads = a.cols_per_round * split * 32;
    const int64_t ntiles = (h->n + kGramTE - 1) / kGramTE;
    const int grid = (int)(ntiles < ctx->sm_count ? ntiles : ctx->sm_count);
    const size_t smem = (size_t)kGramStages * (form ? 4 : 3) * kGramTE * sizeof(T);
    const XComm* xc = ctx->x_active ? ctx->x_comm : nullptr;
    const unsigned long long epoch = ctx->x_active ? ++ctx->x_epoch : 0ull;
    if (auto st = form ? launch_gram_dots<T, true>(ctx, a, rounds, grid, threads, smem, xc, epoch)
                       : launch_gram_dots<T, false>(ctx, a, rounds, grid, threads, smem, xc, epoch)) return st;
    if (ctx->nranks > 1 && !ctx->x_active)
        NC(ctx, ncclAllReduce(ctx->gram_raw, ctx->gram_raw, c * kGramVals, ncclDouble, ncclSum, ctx->comm, ctx->stream));
    return LBFGS_B200_OK;
}

template <class T> static GramSolveArgs<T> make_solve_args(lbfgs_b200_hist* h, T a_scale, bool with_v)
{
    lbfgs_b200_ctx* ctx = h->ctx;
    GramSolveArgs<T> g{};
    g.c = h->ncorr; g.M = h->M; g.new_slot = h->pending; g.with_v = with_v ? 1 : 0; g.a = a_scale;
    g.raw = ctx->gram_raw;
    const int in = h->gram_cur, out = (h->pending >= 0) ? 1 - h->gram_cur : h->gram_cur;
    g.SY_in = static_cast<const T*>(h->SY[in]); g.YY_in = static_cast<const T*>(h->YY[in]);
    g.SS_in = static_cast<const T*>(h->SS[in]);
    g.SY_out = static_cast<T*>(h->SY[out]); g.YY_out = static_cast<T*>(h->YY[out]);
    g.SS_out = static_cast<T*>(h->SS[out]);
    g.ys = static_cast<const T*>(h->ys); g.alpha = static_cast<T*>(h->alpha);
    g.theta = static_cast<const T*>(h->theta);
    fill_slots<T>(h, g.slots);
    return g;
}
// after a kernel that folded the pending pair: the freshly written buffer becomes current
static void gram_folded(lbfgs_b200_hist* h)
{
    if (h->pending >= 0) h->gram_cur = 1 - h->gram_cur;
    h->pending = -1;
}

// fold a pending pair into SY/YY without an apply_Hv (only needed when pairs are appended back to back)
template <class T> static lbfgs_b200_status gram_refresh(lbfgs_b200_hist* h)
{
    if (h->pending < 0 || h->ncorr == 0) { h->pending = -1; return LBFGS_B200_OK; }
    lbfgs_b200_ctx* ctx = h->ctx;
    if (auto st = gram_dots<T>(h, nullptr)) return st;
    const GramSolveArgs<T> g = make_solve_args<T>(h, T(0), false);
    const size_t smem = gram_solve_smem_elems(h->ncorr) * sizeof(T);
    if (smem > 48 * 1024)
        CU(ctx, cudaFuncSetAttribute(k_gram_fold<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_gram_fold<T><<<1, 256, smem, ctx->stream>>>(g);
    if (auto st = post_launch(ctx, "k_gram_fold")) return st;
    gram_folded(h);
    return LBFGS_B200_OK;
}

template <class T> static lbfgs_b200_status hv_gram_combine(lbfgs_b200_hist* h, const T* v, T a, T* res, bool want_vdot);

template <class T>
static lbfgs_b200_status hv_gram(lbfgs_b200_hist* h, const T* v, T a, T* res, bool want_vdot)
{
    if (auto st = gram_dots<T>(h, v)) return st;
    return hv_gram_combine<T>(h, v, a, res, want_vdot);
}

// second half of the Gram-form apply_Hv: ctx->gram_raw holds the (all-reduced) dots of the current history against v
template <class T>
static lbfgs_b200_status hv_gram_combine(lbfgs_b200_hist* h, const T* v, T a, T* res, bool want_vdot)
{
    lbfgs_b200_ctx* ctx = h->ctx;
    GramCombineArgs<T> k{};
    k.n = h->n; k.ld = h->ld; k.v = v;
    k.S = static_cast<const T*>(h->S); k.Y = static_cast<const T*>(h->Y);
    k.res = res; k.want_dot = want_vdot ? 1 : 0;
    k.solve = make_solve_args<T>(h, a, true);
    const int grid = grid_for(ctx, h->n, 1);
    const size_t smem = gram_solve_smem_elems(h->ncorr) * sizeof(T);
    const bool vec = all_aligned<T>({v, res});
    if (smem > 40 * 1024)
    {
        if (vec) CU(ctx, cudaFuncSetAttribute(k_gram_combine<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        else CU(ctx, cudaFuncSetAttribute(k_gram_combine<T, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    const ReduceBuf rb = want_vdot ? next_rb(ctx, true) : ctx->rb;
    if (vec) k_gram_combine<T, true><<<grid, kThreads, smem, ctx->stream>>>(k, rb);
    else k_gram_combine<T, false><<<grid, kThreads, smem, ctx->stream>>>(k, rb);
    if (auto st = post_launch(ctx, "k_gram_combine")) return st;
    gram_folded(h);
    if (want_vdot) return allreduce_result(ctx, 1);
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_hist_apply_Hv(lbfgs_b200_hist* h, const T* v, T a, T* res, int algo, T* vdot_host)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, v && res && v != res, "apply_Hv: v/res NULL or aliased");
    REQUIRE(ctx, algo >= LBFGS_B200_HV_AUTO && algo <= LBFGS_B200_HV_GRAM, "apply_Hv: unknown algorithm %d", algo);
    const bool gram = (algo != LBFGS_B200_HV_TWO_LOOP) && h->ncorr > 0;
    ProfSpan span(ctx, PH_APPLY_HV, double(sizeof(T)) * double(h->n) * (4.0 * h->ncorr + 2.0));
    lbfgs_b200_status st = gram ? hv_gram<T>(h, v, a, res, vdot_host != nullptr)
                                : hv_two_loop<T>(h, v, a, res, vdot_host != nullptr);
    span.stop();
    if (st) return st;
    if (vdot_host)
    {
        if (auto s2 = (gram ? receive(ctx, 1) : fetch_result(ctx, 1))) return s2;
        *vdot_host = (T)ctx->h_result[0];
    }
    return LBFGS_B200_OK;
}

// LBFGS.h:159-165 as one call: { s = x - xp; y = g - gp; if (s'y > eps*y'y) add_correction(s, y); res = a*H*g } (+ g.res).
// With the Gram form the pair is formed inside the dots pass (k_gram_dots<FORM>): no separate update kernel, x/xp/g/gp are read
// once, s and y are written once.  The pair is committed only after the gate has seen s'y, y'y (its own dots); a rejected
// pair leaves the history untouched and the old history answers, as in the reference.
template <class T>
static lbfgs_b200_status do_hist_update_apply_Hv(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, T eps,
                                                 T a, T* res, int algo, int* accepted_host, T* vdot_host)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, x && xp && g && gp && res, "update_apply_Hv: NULL vector");
    REQUIRE(ctx, res != g && res != x && res != xp && res != gp, "update_apply_Hv: res aliases an input");
    REQUIRE(ctx, algo >= LBFGS_B200_HV_AUTO && algo <= LBFGS_B200_HV_GRAM, "update_apply_Hv: unknown algorithm %d", algo);
    if (algo == LBFGS_B200_HV_TWO_LOOP || !all_aligned<T>({x, xp, g, gp}))
    {
        if (auto st = do_hist_update<T>(h, x, xp, g, gp, eps, accepted_host, nullptr)) return st;
        return do_hist_apply_Hv<T>(h, g, a, res, algo, vdot_host);
    }
    if (h->pending >= 0)
        if (auto st = gram_refresh<T>(h)) return st;
    const int c_new = h->ncorr < h->m ? h->ncorr + 1 : h->m;
    ProfSpan span(ctx, PH_APPLY_HV, double(sizeof(T)) * double(h->n) * (4.0 * c_new + 2.0 + 6.0));
    const PairForm<T> form{x, xp, gp};
    if (auto st = gram_dots<T>(h, g, &form)) return st;
    int ok = 0;
    if (auto st = commit_pair<T>(h, eps, 1, &ok, nullptr, ctx->gram_raw + 2)) return st;  // age-0 column: [2] = s'y, [3] = y'y
    if (accepted_host) *accepted_host = ok;
    const bool want = vdot_host != nullptr;
    bool gram = true;
    lbfgs_b200_status st;
    if (ok) st = hv_gram_combine<T>(h, g, a, res, want);
    else if (h->ncorr > 0) st = hv_gram<T>(h, g, a, res, want);
    else { gram = false; st = hv_two_loop<T>(h, g, a, res, want); }
    span.stop();
    if (st) return st;
    if (vdot_host)
    {
        if (auto s2 = (gram ? receive(ctx, 1) : fetch_result(ctx, 1))) return s2;
        *vdot_host = (T)ctx->h_result[0];
    }
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_hist_scalars(lbfgs_b200_hist* h, T* theta_host, T* ys_host, T* alpha_host)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    T tmp[2 * 65 + 1];
    REQUIRE(ctx, h->M <= 65, "hist_scalars: m too large for the inspection buffer");
    CU(ctx, cudaMemcpyAsync(tmp, h->ys, sizeof(T) * h->M, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaMemcpyAsync(tmp + 65, h->alpha, sizeof(T) * h->M, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaMemcpyAsync(tmp + 130, h->theta, sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    if (theta_host) *theta_host = tmp[130];
    for (int age = 0; age < h->ncorr; age++)
    {
        if (ys_host) ys_host[age] = tmp[h->slot(age)];
        if (alpha_host) alpha_host[age] = tmp[65 + h->slot(age)];
    }
    return LBFGS_B200_OK;
}

// ----------------------------------------------------------------------------- OWL-QN
// Every entry refuses a lambda that is not positive and finite, and a context with more than one rank (no n-sharding).  The weighted
// entries (`weighted`, named `what`) first refuse a NULL w; past this check w != nullptr selects the weighted kernels.  Only the
// sums entry reads every weight for validity (its count of refused weights costs no extra pass); the others trust w.
template <class T> static lbfgs_b200_status owlqn_check(lbfgs_b200_ctx* ctx, T lam, bool weighted, const T* w, const char* what)
{
    REQUIRE(ctx, !weighted || w, "%s: NULL weights", what);
    REQUIRE(ctx, lam > T(0) && lam <= std::numeric_limits<T>::max(), "owlqn: lambda must be positive and finite (got %g)", double(lam));
    REQUIRE(ctx, ctx->nranks == 1, "owlqn: one rank only, the vectors cannot be sharded (the context has %d)", ctx->nranks);
    return LBFGS_B200_OK;
}

// `count` result slots of the reducing kernel just launched, to the host
template <class T> static lbfgs_b200_status owlqn_receive(lbfgs_b200_ctx* ctx, int count, T* out_host)
{
    if (auto st = receive(ctx, count)) return st;
    for (int k = 0; k < count; k++) out_host[k] = (T)ctx->h_result[k];
    return LBFGS_B200_OK;
}

// launch(W, VEC) with the weight and vector-width choices as std::bool_constant: one place turns them into template arguments
template <class F> static void owlqn_variant(bool weighted, bool vec, F&& launch)
{
    if (weighted)
    {
        if (vec) launch(std::true_type{}, std::true_type{});
        else launch(std::true_type{}, std::false_type{});
    }
    else if (vec) launch(std::false_type{}, std::true_type{});
    else launch(std::false_type{}, std::false_type{});
}

template <class T, class OBJ, bool W, bool VEC>
static void launch_owlqn_trial(lbfgs_b200_ctx* ctx, int grid, const ObjGeom<T>& geo, int64_t n, const T* xp, const T* d, const T* gp,
                               T step, T lam, const T* w, T* x, T* g, const ReduceBuf& rb)
{
    if constexpr (W) k_owlqn_trial_w<T, OBJ, VEC><<<grid, kThreads, 0, ctx->stream>>>(OBJ{geo}, n, xp, d, gp, step, lam, w, x, g, rb);
    else k_owlqn_trial<T, OBJ, VEC><<<grid, kThreads, 0, ctx->stream>>>(OBJ{geo}, n, xp, d, gp, step, lam, x, g, rb);
}

template <class T>
static lbfgs_b200_status do_owlqn_trial(lbfgs_b200_ctx* ctx, int objective, const T* data0, const T* data1, int64_t n, const T* xp,
                                        const T* d, const T* gp, T step, T lam, const T* w, bool weighted, T* x, T* g, T* out5)
{
    REQUIRE(ctx, ctx && xp && d && gp && x && g && out5 && n >= 1, "owlqn_trial: bad arguments");
    if (auto st = owlqn_check<T>(ctx, lam, weighted, w, "owlqn_weighted_trial")) return st;
    return with_objective<T>(ctx, objective, [&](auto tag) -> lbfgs_b200_status {
        using OBJ = decltype(tag);
        ObjGeom<T> geo;
        if (auto st = objective_geometry<OBJ>(ctx, n, data0, data1, geo)) return st;
        ProfSpan span(ctx, PH_TRIAL, double(sizeof(T)) * double(n) * ((w ? 6.0 : 5.0) + OBJ::kDataVectors));
        const int grid = grid_for(ctx, n, 2);
        const ReduceBuf rb = next_rb(ctx, true);
        owlqn_variant(w != nullptr, all_aligned<T>({xp, d, gp, x, g, w}), [&](auto W, auto VEC) {
            launch_owlqn_trial<T, OBJ, W, VEC>(ctx, grid, geo, n, xp, d, gp, step, lam, w, x, g, rb);
        });
        if (auto st = post_launch(ctx, w ? "k_owlqn_trial_w" : "k_owlqn_trial")) return st;
        span.stop();
        return owlqn_receive<T>(ctx, 5, out5);
    });
}

template <class T, bool W, bool VEC>
static void launch_owlqn_project(lbfgs_b200_ctx* ctx, int grid, int64_t n, const T* xp, const T* d, const T* gp, T step, T lam, const T* w,
                                 T* x, const ReduceBuf& rb)
{
    if constexpr (W) k_owlqn_project_w<T, VEC><<<grid, kThreads, 0, ctx->stream>>>(n, xp, d, gp, step, lam, w, x, rb);
    else k_owlqn_project<T, VEC><<<grid, kThreads, 0, ctx->stream>>>(n, xp, d, gp, step, lam, x, rb);
}

template <class T>
static lbfgs_b200_status do_owlqn_project(lbfgs_b200_ctx* ctx, int64_t n, const T* xp, const T* d, const T* gp, T step, T lam, const T* w,
                                          bool weighted, T* x, T* out2)
{
    REQUIRE(ctx, ctx && xp && d && gp && x && out2 && n >= 1, "owlqn_project: bad arguments");
    if (auto st = owlqn_check<T>(ctx, lam, weighted, w, "owlqn_weighted_project")) return st;
    const int grid = grid_for(ctx, n);
    const ReduceBuf rb = next_rb(ctx, true);
    owlqn_variant(w != nullptr, all_aligned<T>({xp, d, gp, x, w}), [&](auto W, auto VEC) {
        launch_owlqn_project<T, W, VEC>(ctx, grid, n, xp, d, gp, step, lam, w, x, rb);
    });
    if (auto st = post_launch(ctx, w ? "k_owlqn_project_w" : "k_owlqn_project")) return st;
    return owlqn_receive<T>(ctx, 2, out2);
}

template <class T, bool W, bool VEC, bool START>
static void launch_owlqn_sums(lbfgs_b200_ctx* ctx, int grid, int64_t n, const T* x, const T* g, T lam, const T* w, T* d, const ReduceBuf& rb)
{
    if constexpr (W) k_owlqn_sums_w<T, START, VEC><<<grid, kThreads, 0, ctx->stream>>>(n, x, g, lam, w, d, rb);
    else k_owlqn_sums<T, START, VEC><<<grid, kThreads, 0, ctx->stream>>>(n, x, g, lam, d, rb);
}

// weighted: the kernel also counts the weights owlqn_weight_ok refuses; any such weight makes the entry return
// LBFGS_B200_ERR_INVALID with that count (out3 is written all the same)
template <class T>
static lbfgs_b200_status do_owlqn_sums(lbfgs_b200_ctx* ctx, int64_t n, const T* x, const T* g, T lam, const T* w, bool weighted, T* d, T* out3)
{
    REQUIRE(ctx, ctx && x && g && out3 && n >= 1, "owlqn_sums: bad arguments");
    REQUIRE(ctx, d != x && d != g, "owlqn_sums: d aliases x or g");
    if (auto st = owlqn_check<T>(ctx, lam, weighted, w, "owlqn_weighted_sums")) return st;
    const int grid = grid_for(ctx, n);
    const ReduceBuf rb = next_rb(ctx, true);
    owlqn_variant(w != nullptr, all_aligned<T>({x, g, d, w}), [&](auto W, auto VEC) {
        if (d) launch_owlqn_sums<T, W, VEC, true>(ctx, grid, n, x, g, lam, w, d, rb);
        else launch_owlqn_sums<T, W, VEC, false>(ctx, grid, n, x, g, lam, w, nullptr, rb);
    });
    if (auto st = post_launch(ctx, w ? "k_owlqn_sums_w" : "k_owlqn_sums")) return st;
    if (!w) return owlqn_receive<T>(ctx, 3, out3);
    if (auto st = receive(ctx, 4)) return st;
    for (int k = 0; k < 3; k++) out3[k] = (T)ctx->h_result[k];
    const double bad = ctx->h_result[3];
    REQUIRE(ctx, bad == 0.0, "owlqn_weighted_sums: %.0f weights are negative, not finite, or make lambda * w overflow", bad);
    return LBFGS_B200_OK;
}

// d = the orthant-constrained -H pg and pg.d, after the new pair's update: the Gram form of do_hist_update_apply_Hv with
// pg(x, g; lam) as the right-hand vector.  The pair (s, y) = (x - xp, g - gp) is formed in the dots pass (k_gram_dots_pg); if the
// curvature gate refuses it, the dots of the kept history are taken again against pg written into the spare ring column.
// Weighted: k_gram_dots_pg_w / k_gram_combine_pg_w / k_owlqn_pg_w, the same passes with one more word per coordinate each.
template <class T, bool W>
static lbfgs_b200_status launch_gram_dots_pg(lbfgs_b200_ctx* ctx, const GramDotsArgs<T>& a, T lam, const T* w, int rounds, int grid, int threads,
                                             size_t smem)
{
    const int r = rounds <= 1 ? 1 : rounds == 2 ? 2 : 3;
    const unsigned bit = 1u << ((W ? 24 : 16) + (sizeof(T) == 8 ? 0 : 4) + r);
    const auto kernel = [r] {
        if constexpr (W) return r == 1 ? k_gram_dots_pg_w<T, 1> : r == 2 ? k_gram_dots_pg_w<T, 2> : k_gram_dots_pg_w<T, 3>;
        else return r == 1 ? k_gram_dots_pg<T, 1> : r == 2 ? k_gram_dots_pg<T, 2> : k_gram_dots_pg<T, 3>;
    }();
    if (!(ctx->smem_optin & bit))
    {
        CU(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ctx->smem_optin |= bit;
    }
    if constexpr (W) kernel<<<grid, threads, smem, ctx->stream>>>(a, lam, w, ctx->gram_partials, ctx->rb.ticket, ctx->gram_raw);
    else kernel<<<grid, threads, smem, ctx->stream>>>(a, lam, ctx->gram_partials, ctx->rb.ticket, ctx->gram_raw, nullptr, 0ull);
    return post_launch(ctx, W ? "k_gram_dots_pg_w" : "k_gram_dots_pg");
}

template <class T, bool W, bool VEC>
static lbfgs_b200_status launch_gram_combine_pg(lbfgs_b200_ctx* ctx, const GramCombineArgs<T>& k, const T* x, T lam, const T* w, int grid,
                                                size_t smem)
{
    const auto kernel = [] {
        if constexpr (W) return k_gram_combine_pg_w<T, VEC>;
        else return k_gram_combine_pg<T, VEC>;
    }();
    if (smem > 40 * 1024) CU(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const ReduceBuf rb = next_rb(ctx, true);
    if constexpr (W) kernel<<<grid, kThreads, smem, ctx->stream>>>(k, x, lam, w, rb);
    else kernel<<<grid, kThreads, smem, ctx->stream>>>(k, x, lam, rb);
    return post_launch(ctx, W ? "k_gram_combine_pg_w" : "k_gram_combine_pg");
}

// pg(x, g) into out, for the dots round that follows a refused pair
template <class T, bool W>
static lbfgs_b200_status launch_owlqn_pg(lbfgs_b200_ctx* ctx, int64_t n, const T* x, const T* g, T lam, const T* w, T* out)
{
    if constexpr (W) k_owlqn_pg_w<T><<<grid_for(ctx, n), kThreads, 0, ctx->stream>>>(n, x, g, lam, w, out);
    else k_owlqn_pg<T><<<grid_for(ctx, n), kThreads, 0, ctx->stream>>>(n, x, g, lam, out);
    return post_launch(ctx, W ? "k_owlqn_pg_w" : "k_owlqn_pg");
}

template <class T>
static lbfgs_b200_status do_owlqn_update_dir(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, T eps, T lam, const T* w,
                                             bool weighted, T* d, int* accepted_host, T* dg_host)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, x && xp && g && gp && d && dg_host, "owlqn_update_dir: NULL argument");
    REQUIRE(ctx, d != g && d != x && d != xp && d != gp, "owlqn_update_dir: d aliases an input");
    REQUIRE(ctx, all_aligned<T>({x, xp, g, gp}), "owlqn_update_dir: x, xp, g and gp must start on %zu-byte boundaries", 4 * sizeof(T));
    REQUIRE(ctx, all_aligned<T>({w}), "owlqn_weighted_update_dir: w must start on a %zu-byte boundary, like x", 4 * sizeof(T));
    if (auto st = owlqn_check<T>(ctx, lam, weighted, w, "owlqn_weighted_update_dir")) return st;
    if (h->pending >= 0)
        if (auto st = gram_refresh<T>(h)) return st;
    const int c_new = h->ncorr < h->m ? h->ncorr + 1 : h->m;
    ProfSpan span(ctx, PH_APPLY_HV, double(sizeof(T)) * double(h->n) * (4.0 * c_new + 3.0 + (w ? 9.0 : 7.0)));
    // the FORM dots of gram_dots(), with pg in place of g
    GramDotsArgs<T> a{};
    a.n = h->n; a.ld = h->ld; a.v = g;
    a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y);
    a.c = c_new; a.new_slot = h->head;
    a.fx = x; a.fxp = xp; a.fgp = gp;
    a.s_out = h->s_col<T>(h->head); a.y_out = h->y_col<T>(h->head);
    int split = 8;
    while (split > 1 && c_new * split > kGramMaxWarps) split >>= 1;
    a.split = split;
    a.cols_per_round = c_new < kGramMaxWarps / split ? c_new : kGramMaxWarps / split;
    a.use_tma = 1;
    a.slots[0] = (unsigned char)h->head;
    for (int age = 1; age < c_new; age++) a.slots[age] = (unsigned char)h->slot(age - 1);
    const int rounds = (c_new + a.cols_per_round - 1) / a.cols_per_round;
    const int64_t ntiles = (h->n + kGramTE - 1) / kGramTE;
    const int grid = (int)(ntiles < ctx->sm_count ? ntiles : ctx->sm_count);
    const size_t dots_smem = (size_t)kGramStages * 4 * kGramTE * sizeof(T);
    if (auto st = w ? launch_gram_dots_pg<T, true>(ctx, a, lam, w, rounds, grid, a.cols_per_round * split * 32, dots_smem)
                    : launch_gram_dots_pg<T, false>(ctx, a, lam, w, rounds, grid, a.cols_per_round * split * 32, dots_smem))
        return st;
    int ok = 0;
    if (auto st = commit_pair<T>(h, eps, 1, &ok, nullptr, ctx->gram_raw + 2)) return st;   // age-0 column: [2] = s'y, [3] = y'y
    if (!ok && h->ncorr > 0)
    {
        T* pg = h->s_col<T>(h->head);   // the refused pair's column is free again
        if (auto st = w ? launch_owlqn_pg<T, true>(ctx, h->n, x, g, lam, w, pg) : launch_owlqn_pg<T, false>(ctx, h->n, x, g, lam, w, pg))
            return st;
        if (auto st = gram_dots<T>(h, pg)) return st;
    }
    // the combination: with no pair kept, H = I / theta and the recursion runs on no columns
    GramCombineArgs<T> k{};
    k.n = h->n; k.ld = h->ld; k.v = g;
    k.S = static_cast<const T*>(h->S); k.Y = static_cast<const T*>(h->Y);
    k.res = d; k.want_dot = 1;
    k.solve = make_solve_args<T>(h, T(-1), true);
    const int cgrid = grid_for(ctx, h->n, 1);
    const size_t smem = gram_solve_smem_elems(h->ncorr) * sizeof(T);
    lbfgs_b200_status st = LBFGS_B200_OK;
    owlqn_variant(w != nullptr, all_aligned<T>({d}), [&](auto W, auto VEC) {
        st = launch_gram_combine_pg<T, W, VEC>(ctx, k, x, lam, w, cgrid, smem);
    });
    if (st) return st;
    gram_folded(h);
    span.stop();
    if (accepted_host) *accepted_host = ok;
    return owlqn_receive<T>(ctx, 1, dg_host);
}

// =====================================================================================================
// C ABI: typed entry points
// =====================================================================================================
extern "C" {

#define DEFINE_L1(T, SUF)                                                                                      \
    lbfgs_b200_status lbfgs_b200_dot_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* a, const T* b, T* o)         \
    { return do_dot<T>(c, n, a, b, o); }                                                                       \
    lbfgs_b200_status lbfgs_b200_dot3_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* g, const T* d, const T* x,  \
                                            T* o) { return do_dot3<T>(c, n, g, d, x, o); }                     \
    lbfgs_b200_status lbfgs_b200_axpy_out_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* a, T s, const T* b,     \
                                                T* o) { return do_axpy_out<T>(c, n, a, s, b, o); }             \
    lbfgs_b200_status lbfgs_b200_scale_out_##SUF(lbfgs_b200_ctx* c, int64_t n, T s, const T* a, T* o)          \
    { return do_scale_out<T>(c, n, s, a, o); }                                                                 \
    lbfgs_b200_status lbfgs_b200_objective_##SUF(lbfgs_b200_ctx* c, int obj, const T* d0, const T* d1,         \
                                                 int64_t n, const T* x, T* g, T* fx)                           \
    { return do_trial<T, false>(c, obj, d0, d1, n, nullptr, nullptr, T(0), const_cast<T*>(x), g, fx); }        \
    lbfgs_b200_status lbfgs_b200_trial_##SUF(lbfgs_b200_ctx* c, int obj, const T* d0, const T* d1, int64_t n,  \
                                             const T* xp, const T* d, T step, T* x, T* g, T* out4)             \
    { return do_trial<T, true>(c, obj, d0, d1, n, xp, d, step, x, g, out4); }

DEFINE_L1(double, f64)
DEFINE_L1(float, f32)

lbfgs_b200_status lbfgs_b200_hist_create(lbfgs_b200_ctx* ctx, lbfgs_b200_hist** out, int64_t n, int m, int elem_bytes)
{
    REQUIRE(ctx, ctx && out, "hist_create: NULL argument");
    *out = nullptr;
    REQUIRE(ctx, n >= 1 && m >= 1 && m <= 64, "hist_create: need n >= 1 and 1 <= m <= 64 (got n=%lld m=%d)", (long long)n, m);
    REQUIRE(ctx, elem_bytes == 8 || elem_bytes == 4, "hist_create: elem_bytes must be 8 or 4");
    lbfgs_b200_hist* h = new (std::nothrow) lbfgs_b200_hist();
    if (!h) return fail(ctx, LBFGS_B200_ERR_ALLOC, "out of host memory");
    h->ctx = ctx; h->n = n; h->m = m; h->M = m + 1; h->elem = elem_bytes;
    h->ld = (n + 31) & ~int64_t(31);  // columns start on 256-byte (fp64) / 128-byte (fp32) boundaries
    const size_t colbytes = (size_t)h->ld * elem_bytes * h->M;
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e == cudaSuccess) e = pool_alloc(ctx, &h->S, colbytes);
    if (e == cudaSuccess) e = pool_alloc(ctx, &h->Y, colbytes);
    if (e == cudaSuccess) e = pool_alloc(ctx, &h->ys, (size_t)elem_bytes * h->M);
    if (e == cudaSuccess) e = pool_alloc(ctx, &h->alpha, (size_t)elem_bytes * h->M);
    if (e == cudaSuccess) e = pool_alloc(ctx, &h->theta, 8);
    for (int b = 0; b < 2; b++)
    {
        if (e == cudaSuccess) e = pool_alloc(ctx, &h->SY[b], (size_t)elem_bytes * h->M * h->M);
        if (e == cudaSuccess) e = pool_alloc(ctx, &h->YY[b], (size_t)elem_bytes * h->M * h->M);
        if (e == cudaSuccess) e = pool_alloc(ctx, &h->SS[b], (size_t)elem_bytes * h->M * h->M);
    }
    if (e != cudaSuccess)
    {
        lbfgs_b200_hist_destroy(h);
        return fail(ctx, e == cudaErrorMemoryAllocation ? LBFGS_B200_ERR_ALLOC : LBFGS_B200_ERR_CUDA,
                    "hist_create(n=%lld, m=%d): %s", (long long)n, m, cudaGetErrorString(e));
    }
    *out = h;
    return lbfgs_b200_hist_reset(h);
}

void lbfgs_b200_hist_destroy(lbfgs_b200_hist* h)
{
    if (!h) return;
    // (no synchronisation: the blocks go back to the context's pool and everything that used them is ordered on its stream)
    for (void* p : {h->S, h->Y, h->ys, h->alpha, h->theta, h->SY[0], h->YY[0], h->SS[0], h->SY[1], h->YY[1], h->SS[1], h->multi, h->quad}) pool_free(h->ctx, p);
    delete h;
}

lbfgs_b200_status lbfgs_b200_hist_reset(lbfgs_b200_hist* h)
{
    if (!h || !h->ctx) return LBFGS_B200_ERR_INVALID;
    lbfgs_b200_ctx* ctx = h->ctx;
    h->head = 0;
    h->ncorr = 0;
    h->pending = -1;
    h->gram_cur = 0;
    for (int b = 0; b < 2; b++)
    {
        CU(ctx, cudaMemsetAsync(h->SY[b], 0, (size_t)h->elem * h->M * h->M, ctx->stream));
        CU(ctx, cudaMemsetAsync(h->YY[b], 0, (size_t)h->elem * h->M * h->M, ctx->stream));
        CU(ctx, cudaMemsetAsync(h->SS[b], 0, (size_t)h->elem * h->M * h->M, ctx->stream));
    }
    CU(ctx, cudaMemsetAsync(h->ys, 0, (size_t)h->elem * h->M, ctx->stream));
    CU(ctx, cudaMemsetAsync(h->alpha, 0, (size_t)h->elem * h->M, ctx->stream));
    if (h->elem == 8) { const double one = 1.0; CU(ctx, cudaMemcpyAsync(h->theta, &one, 8, cudaMemcpyHostToDevice, ctx->stream)); }
    else { const float one = 1.0f; CU(ctx, cudaMemcpyAsync(h->theta, &one, 4, cudaMemcpyHostToDevice, ctx->stream)); }
    CU(ctx, cudaStreamSynchronize(ctx->stream));  // `one` lives on this stack frame
    return LBFGS_B200_OK;
}

int lbfgs_b200_hist_ncorr(const lbfgs_b200_hist* h) { return h ? h->ncorr : 0; }
int lbfgs_b200_hist_m(const lbfgs_b200_hist* h) { return h ? h->m : 0; }
const void* lbfgs_b200_hist_s_col(const lbfgs_b200_hist* h, int age)
{
    if (!h || age < 0 || age >= h->ncorr) return nullptr;
    return static_cast<const char*>(h->S) + (size_t)h->slot(age) * h->ld * h->elem;
}
const void* lbfgs_b200_hist_y_col(const lbfgs_b200_hist* h, int age)
{
    if (!h || age < 0 || age >= h->ncorr) return nullptr;
    return static_cast<const char*>(h->Y) + (size_t)h->slot(age) * h->ld * h->elem;
}

#define DEFINE_HIST(T, SUF)                                                                                    \
    lbfgs_b200_status lbfgs_b200_hist_update_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g,    \
                                                   const T* gp, T eps, int* acc, T* sy_yy)                     \
    { return do_hist_update<T>(h, x, xp, g, gp, eps, acc, sy_yy); }                                            \
    lbfgs_b200_status lbfgs_b200_hist_add_##SUF(lbfgs_b200_hist* h, const T* s, const T* y)                    \
    { return do_hist_add<T>(h, s, y); }                                                                        \
    lbfgs_b200_status lbfgs_b200_hist_apply_Hv_##SUF(lbfgs_b200_hist* h, const T* v, T a, T* res, int algo,    \
                                                     T* vdot) { return do_hist_apply_Hv<T>(h, v, a, res, algo, vdot); } \
    lbfgs_b200_status lbfgs_b200_hist_update_apply_Hv_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, \
                                                            const T* gp, T eps, T a, T* res, int algo, int* acc, T* vdot) \
    { return do_hist_update_apply_Hv<T>(h, x, xp, g, gp, eps, a, res, algo, acc, vdot); }                      \
    lbfgs_b200_status lbfgs_b200_hist_scalars_##SUF(lbfgs_b200_hist* h, T* th, T* ys, T* al)                   \
    { return do_hist_scalars<T>(h, th, ys, al); }

DEFINE_HIST(double, f64)
DEFINE_HIST(float, f32)

#define DEFINE_OWLQN(T, SUF)                                                                                   \
    lbfgs_b200_status lbfgs_b200_owlqn_trial_##SUF(lbfgs_b200_ctx* c, int obj, const T* d0, const T* d1, int64_t n, \
                                                   const T* xp, const T* d, const T* gp, T step, T lam, T* x, T* g, \
                                                   T* out5)                                                     \
    { return do_owlqn_trial<T>(c, obj, d0, d1, n, xp, d, gp, step, lam, nullptr, false, x, g, out5); }         \
    lbfgs_b200_status lbfgs_b200_owlqn_project_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* xp, const T* d, const T* gp, \
                                                     T step, T lam, T* x, T* out2)                              \
    { return do_owlqn_project<T>(c, n, xp, d, gp, step, lam, nullptr, false, x, out2); }                       \
    lbfgs_b200_status lbfgs_b200_owlqn_sums_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* x, const T* g, T lam, T* d, \
                                                  T* out3) { return do_owlqn_sums<T>(c, n, x, g, lam, nullptr, false, d, out3); } \
    lbfgs_b200_status lbfgs_b200_owlqn_update_dir_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g,  \
                                                        const T* gp, T eps, T lam, T* d, int* acc, T* dg)       \
    { return do_owlqn_update_dir<T>(h, x, xp, g, gp, eps, lam, nullptr, false, d, acc, dg); }                  \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_trial_##SUF(lbfgs_b200_ctx* c, int obj, const T* d0, const T* d1, int64_t n, \
                                                            const T* xp, const T* d, const T* gp, T step, T lam, const T* w, \
                                                            T* x, T* g, T* out5)                                \
    { return do_owlqn_trial<T>(c, obj, d0, d1, n, xp, d, gp, step, lam, w, true, x, g, out5); }                \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_project_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* xp, const T* d, \
                                                              const T* gp, T step, T lam, const T* w, T* x, T* out2) \
    { return do_owlqn_project<T>(c, n, xp, d, gp, step, lam, w, true, x, out2); }                              \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_sums_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* x, const T* g, T lam, \
                                                           const T* w, T* d, T* out3)                           \
    { return do_owlqn_sums<T>(c, n, x, g, lam, w, true, d, out3); }                                            \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_update_dir_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, \
                                                                 const T* gp, T eps, T lam, const T* w, T* d, int* acc, \
                                                                 T* dg)                                         \
    { return do_owlqn_update_dir<T>(h, x, xp, g, gp, eps, lam, w, true, d, acc, dg); }

DEFINE_OWLQN(double, f64)
DEFINE_OWLQN(float, f32)

}  // extern "C"
#include "lbfgsb_impl.cuh"
