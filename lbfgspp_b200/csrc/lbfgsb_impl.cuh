// lbfgsb_impl.cuh -- C ABI of the bound-constrained primitives (included at the end of lbfgs_b200.cu).
// Host glue only; kernels are in lbfgsb_kernels.cuh.  L-BFGS-B runs replicated per GPU (SURVEY.md 8e: the global sort
// and the index sets do not shard cleanly), so these entry points refuse a context with a communicator attached.
#pragma once

#include <climits>

#include "lbfgsb_kernels.cuh"

struct lbfgs_b200_box
{
    lbfgs_b200_hist* h = nullptr;
    int64_t n = 0, npad = 0;
    void *brk = nullptr, *dvec = nullptr, *xcp = nullptr, *vecc = nullptr, *vecy = nullptr, *lambda = nullptr, *mu = nullptr,
         *tmp = nullptr, *tmp2 = nullptr, *yfb = nullptr;
    unsigned char* cls = nullptr;
    unsigned long long* keys = nullptr;
    unsigned* ord = nullptr;
    unsigned long long* keys2 = nullptr;   // radix sort: the other side of the ping-pong
    unsigned* ord2 = nullptr;
    unsigned* radix_hist = nullptr;        // [256][npad / kSortTile]
    void* block_sums = nullptr;   // [(npad/kScanBlock)][4m+1]
    long long* best = nullptr;
    void* small = nullptr;        // device scratch for small host-supplied arrays: Mmat [2m*2m] | p0 [2m] | coef [2m] | out [5+2m]
    double* mg_partials = nullptr;  // masked-Gram block partials [sm_count][(2m)^2]
    double* mg_result = nullptr;    // [(2m)^2]
};

template <class T> static lbfgs_b200_status box_check(lbfgs_b200_box* b)
{
    if (!b || !b->h || !b->h->ctx) return LBFGS_B200_ERR_INVALID;
    if (b->h->elem != (int)sizeof(T)) return fail(b->h->ctx, LBFGS_B200_ERR_INVALID, "box workspace element size mismatch");
    if (b->h->ctx->nranks > 1) return fail(b->h->ctx, LBFGS_B200_ERR_INVALID, "the bound-constrained path is not n-sharded (replicas only)");
    return LBFGS_B200_OK;
}

// ------------------------------------------------------------------------------------------------ history primitives
// raw[2c] = { y_age . v , s_age . v }  (BFGSMat::apply_Wtv / apply_WtPv on a pre-masked vector, BFGSMat.h:315-320,382-433)
template <class T> static lbfgs_b200_status do_hist_wt_dot(lbfgs_b200_hist* h, const T* v, T* raw_host)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, v && raw_host, "hist_wt_dot: NULL argument");
    const int c = h->ncorr;
    if (c == 0) return LBFGS_B200_OK;
    if (h->pending >= 0) if (auto st = gram_refresh<T>(h)) return st;
    if (auto st = gram_dots<T>(h, v)) return st;
    CU(ctx, cudaMemcpyAsync(ctx->h_result, ctx->gram_raw, sizeof(double) * c * kGramVals, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    for (int j = 0; j < c; j++)
    {
        raw_host[j] = (T)ctx->h_result[j * kGramVals + 1];       // y_j . v
        raw_host[c + j] = (T)ctx->h_result[j * kGramVals + 0];   // s_j . v
    }
    return LBFGS_B200_OK;
}

// c x c matrices by age (row-major): SY[i][j] = s_i.y_j, SS[i][j] = s_i.s_j, YY[i][j] = y_i.y_j ; ys by age ; theta
template <class T> static lbfgs_b200_status do_hist_gram(lbfgs_b200_hist* h, T* SY, T* SS, T* YY, T* ys, T* theta)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    const int c = h->ncorr, M = h->M;
    if (h->pending >= 0) if (auto st = gram_refresh<T>(h)) return st;
    std::vector<T> buf((size_t)M * M * 3 + M + 1);
    const int cur = h->gram_cur;
    CU(ctx, cudaMemcpyAsync(buf.data(), h->SY[cur], sizeof(T) * M * M, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaMemcpyAsync(buf.data() + M * M, h->SS[cur], sizeof(T) * M * M, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaMemcpyAsync(buf.data() + 2 * M * M, h->YY[cur], sizeof(T) * M * M, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaMemcpyAsync(buf.data() + 3 * M * M, h->ys, sizeof(T) * M, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaMemcpyAsync(buf.data() + 3 * M * M + M, h->theta, sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < c; i++)
    {
        const int pi = h->slot(i);
        for (int j = 0; j < c; j++)
        {
            const int pj = h->slot(j);
            if (SY) SY[i * c + j] = buf[pi * M + pj];
            if (SS) SS[i * c + j] = buf[M * M + pi * M + pj];
            if (YY) YY[i * c + j] = buf[2 * M * M + pi * M + pj];
        }
        if (ys) ys[i] = buf[3 * M * M + pi];
    }
    if (theta) *theta = buf[3 * M * M + M];
    return LBFGS_B200_OK;
}

// OUT[:,j] = a0*V[:,j] + sum_a C[a][j]*y_a + C[c+a][j]*s_a on the rows of (cls, mask); coef_dev: device [2c][k] (see k_hist_lincomb)
template <class T>
static lbfgs_b200_status launch_lincomb(lbfgs_b200_hist* h, T a0, int k, const T* V, int64_t ldv, const T* coef_dev, const unsigned char* cls,
                                        int mask, T* out, int64_t ldo)
{
    lbfgs_b200_ctx* ctx = h->ctx;
    LincombArgs<T> a{};
    a.n = h->n; a.ld = h->ld; a.ldv = ldv; a.ldo = ldo; a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y);
    a.V = V; a.a0 = a0; a.coef = coef_dev; a.cls = cls; a.mask = (unsigned char)mask; a.out = out; a.c = h->ncorr; a.k = k;
    fill_slots<T>(h, a.slots);
    if (k == 1) k_hist_lincomb<T, 1><<<grid_for(ctx, h->n * 4, 4), kThreads, 0, ctx->stream>>>(a);
    else k_hist_lincomb<T, kMaxK><<<grid_for(ctx, h->n * 4, 4), kThreads, 0, ctx->stream>>>(a);
    return post_launch(ctx, "k_hist_lincomb");
}

template <class T>
static lbfgs_b200_status do_hist_lincomb(lbfgs_b200_hist* h, lbfgs_b200_box* b, T a0, const T* v0, const T* coef_host,
                                         const unsigned char* cls, int mask, T* out)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, out && b && b->small, "hist_lincomb: NULL argument");
    const int c = h->ncorr;
    T* coef_dev = static_cast<T*>(b->small) + (size_t)4 * h->m * h->m + 2 * h->m;
    if (c > 0)
    {
        REQUIRE(ctx, coef_host != nullptr, "hist_lincomb: coefficients missing");
        CU(ctx, cudaMemcpyAsync(coef_dev, coef_host, sizeof(T) * 2 * c, cudaMemcpyHostToDevice, ctx->stream));
        CU(ctx, cudaStreamSynchronize(ctx->stream));   // coef_host may be a stack array of the caller
    }
    return launch_lincomb<T>(h, a0, 1, v0, h->n, coef_dev, cls, mask, out, h->n);
}

// ------------------------------------------------------------------------------------------------ k-vector passes (compact B / H products)
// Grid of k_hist_wt_dot_multi: a function of n and the device only, so that a dot's summation order does not depend on k.
static int wt_multi_grid(const lbfgs_b200_hist* h)
{
    const int64_t nstrips = (h->n + kWtRows - 1) / kWtRows;
    return (int)(nstrips < 4 * h->ctx->sm_count ? nstrips : 4 * h->ctx->sm_count);
}

// The history's scratch for the k-vector passes, made on first use: partials [grid][(2m+1)*kMaxK] | result [(2m+1)*kMaxK] |
// coefficients [(2m+1)*kMaxK] (doubles; the coefficients are stored as T).  The extra row holds the squared norms of hist_wt_dot_diff.
static lbfgs_b200_status multi_scratch(lbfgs_b200_hist* h, double** partials, double** result, void** coef)
{
    lbfgs_b200_ctx* ctx = h->ctx;
    const size_t vals = (size_t)(2 * h->m + 1) * kMaxK;
    if (!h->multi)
    {
        const cudaError_t e = pool_alloc(ctx, &h->multi, sizeof(double) * vals * (wt_multi_grid(h) + 2));
        if (e != cudaSuccess)
            return fail(ctx, e == cudaErrorMemoryAllocation ? LBFGS_B200_ERR_ALLOC : LBFGS_B200_ERR_CUDA, "history scratch: %s", cudaGetErrorString(e));
    }
    double* base = static_cast<double*>(h->multi);
    *partials = base;
    *result = base + vals * wt_multi_grid(h);
    *coef = base + vals * (wt_multi_grid(h) + 1);
    return LBFGS_B200_OK;
}

template <class T> static lbfgs_b200_status multi_check(lbfgs_b200_hist* h, int k, int64_t ldv, const char* what)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, k >= 1 && k <= kMaxK, "%s: k must be in 1..%d (got %d)", what, kMaxK, k);
    REQUIRE(ctx, ldv >= h->n, "%s: leading dimension %lld is smaller than n = %lld", what, (long long)ldv, (long long)h->n);
    REQUIRE(ctx, ctx->nranks == 1, "%s: replicas only, not for a context with %d ranks", what, ctx->nranks);
    return LBFGS_B200_OK;
}

// R_host[2c][k] = [Y S]' V  (rows: y by age, then s by age)
template <class T> static lbfgs_b200_status do_hist_wt_dot_multi(lbfgs_b200_hist* h, int k, const T* V, int64_t ldv, T* R_host)
{
    if (auto st = multi_check<T>(h, k, ldv, "hist_wt_dot_multi")) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, V && R_host, "hist_wt_dot_multi: NULL argument");
    const int c = h->ncorr, w = 2 * c;
    if (c == 0) return LBFGS_B200_OK;
    double *partials, *result;
    void* coef;
    if (auto st = multi_scratch(h, &partials, &result, &coef)) return st;
    WtDotMultiArgs<T> a{};
    a.n = h->n; a.ld = h->ld; a.ldv = ldv; a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y); a.V = V;
    a.c = c; a.k = k; a.partials = partials; a.ticket = ctx->rb.ticket; a.result = result;
    fill_slots<T>(h, a.slots);
    const size_t smem = (size_t)(w + k) * kWtPitch * sizeof(T);
    if (smem > 48 * 1024) CU(ctx, cudaFuncSetAttribute(k_hist_wt_dot_multi<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_hist_wt_dot_multi<T><<<wt_multi_grid(h), kThreads, smem, ctx->stream>>>(a);
    if (auto st = post_launch(ctx, "k_hist_wt_dot_multi")) return st;
    std::vector<double> tmp((size_t)w * k);
    CU(ctx, cudaMemcpyAsync(tmp.data(), result, sizeof(double) * w * k, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    for (int e = 0; e < w * k; e++) R_host[e] = (T)tmp[(size_t)e];
    return LBFGS_B200_OK;
}

// The whitening forms of the dots pass (k_hist_wt_dot_multi with WtDotSArgs / WtDotDiffArgs): the launch of the loaded form with w
// staged history columns and ncol dots per vector, the ncol * k results copied to tmp
template <class T, class A>
static lbfgs_b200_status run_wt_dots(lbfgs_b200_hist* h, A& a, int w, int ncol, std::vector<double>& tmp, const char* what)
{
    lbfgs_b200_ctx* ctx = h->ctx;
    double *partials, *result;
    void* coef;
    if (auto st = multi_scratch(h, &partials, &result, &coef)) return st;
    a.n = h->n; a.ld = h->ld; a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y);
    a.c = h->ncorr; a.partials = partials; a.ticket = ctx->rb.ticket; a.result = result;
    fill_slots<T>(h, a.slots);
    auto kernel = k_hist_wt_dot_multi<T, A>;
    const size_t smem = (size_t)(w + a.k) * kWtPitch * sizeof(T);
    if (smem > 48 * 1024) CU(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<wt_multi_grid(h), kThreads, smem, ctx->stream>>>(a);
    if (auto st = post_launch(ctx, what)) return st;
    tmp.resize((size_t)ncol * a.k);
    CU(ctx, cudaMemcpyAsync(tmp.data(), result, sizeof(double) * tmp.size(), cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return LBFGS_B200_OK;
}

// R_host[c][k] = S'V (rows: s by age), each dot bit-identical to the s row of that age from hist_wt_dot_multi on the same V
template <class T> static lbfgs_b200_status do_hist_s_dot_multi(lbfgs_b200_hist* h, int k, const T* V, int64_t ldv, T* R_host)
{
    if (auto st = multi_check<T>(h, k, ldv, "hist_s_dot_multi")) return st;
    REQUIRE(h->ctx, V && R_host, "hist_s_dot_multi: NULL argument");
    const int c = h->ncorr;
    if (c == 0) return LBFGS_B200_OK;
    WtDotSArgs<T> a{};
    a.V = V; a.ldv = ldv; a.k = k;
    std::vector<double> tmp;
    if (auto st = run_wt_dots<T>(h, a, c, c, tmp, "k_hist_s_dot_multi")) return st;
    for (int e = 0; e < c * k; e++) R_host[e] = (T)tmp[(size_t)e];
    return LBFGS_B200_OK;
}

// R_host[2c][k] = [Y S]'(X - mean) and nrm_host[j] = |x_j - mean|^2, both as summed in fp64, the differences formed in the pass
template <class T>
static lbfgs_b200_status do_hist_wt_dot_diff(lbfgs_b200_hist* h, int k, const T* X, int64_t ldx, const T* mean, double* R_host,
                                             double* nrm_host)
{
    if (auto st = multi_check<T>(h, k, ldx, "hist_wt_dot_diff")) return st;
    REQUIRE(h->ctx, X && mean && R_host && nrm_host, "hist_wt_dot_diff: NULL argument");
    const int w = 2 * h->ncorr;
    WtDotDiffArgs<T> a{};
    a.V = X; a.ldv = ldx; a.k = k; a.mean = mean;
    std::vector<double> tmp;
    if (auto st = run_wt_dots<T>(h, a, w, w + 1, tmp, "k_hist_wt_dot_diff")) return st;
    for (int e = 0; e < w * k; e++) R_host[e] = tmp[(size_t)e];
    for (int j = 0; j < k; j++) nrm_host[j] = tmp[(size_t)(w * k + j)];
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_hist_lincomb_multi(lbfgs_b200_hist* h, T a0, int k, const T* V, int64_t ldv, const T* C_host, T* OUT, int64_t ldo)
{
    if (auto st = multi_check<T>(h, k, ldv, "hist_lincomb_multi")) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, V && OUT, "hist_lincomb_multi: NULL argument");
    REQUIRE(ctx, ldo >= h->n, "hist_lincomb_multi: leading dimension %lld is smaller than n = %lld", (long long)ldo, (long long)h->n);
    const int c = h->ncorr;
    double *partials, *result;
    void* coef;
    if (auto st = multi_scratch(h, &partials, &result, &coef)) return st;
    if (c > 0)
    {
        REQUIRE(ctx, C_host != nullptr, "hist_lincomb_multi: NULL argument");
        CU(ctx, cudaMemcpyAsync(coef, C_host, sizeof(T) * 2 * c * k, cudaMemcpyHostToDevice, ctx->stream));
        CU(ctx, cudaStreamSynchronize(ctx->stream));   // C_host may be a stack array of the caller
    }
    return launch_lincomb<T>(h, a0, k, V, ldv, static_cast<const T*>(coef), nullptr, 0, OUT, ldo);
}

// The sampler's two passes: the k-vector passes above with the vectors generated in the kernels (philox.cuh), draws first .. first+k-1
template <class T> static lbfgs_b200_status normal_check(lbfgs_b200_hist* h, int k, uint32_t first, const char* what)
{
    if (auto st = multi_check<T>(h, k, h ? h->n : 0, what)) return st;
    REQUIRE(h->ctx, (uint64_t)first + (uint64_t)k <= 0x100000000ull, "%s: draws %u + %d run past 2^32", what, first, k);
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_hist_wt_dot_normal(lbfgs_b200_hist* h, uint64_t seed, uint32_t stream, uint32_t first, int k, T* R_host)
{
    if (auto st = normal_check<T>(h, k, first, "hist_wt_dot_normal")) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, R_host, "hist_wt_dot_normal: NULL argument");
    const int c = h->ncorr, w = 2 * c;
    if (c == 0) return LBFGS_B200_OK;
    double *partials, *result;
    void* coef;
    if (auto st = multi_scratch(h, &partials, &result, &coef)) return st;
    WtDotNormalArgs<T> a{};
    a.n = h->n; a.ld = h->ld; a.ldv = 0; a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y); a.V = nullptr;
    a.c = c; a.k = k; a.partials = partials; a.ticket = ctx->rb.ticket; a.result = result;
    a.src = NormalSrc{(unsigned long long)seed, stream, first};
    fill_slots<T>(h, a.slots);
    auto kernel = k_hist_wt_dot_multi<T, WtDotNormalArgs<T>>;
    const size_t smem = (size_t)(w + k) * kWtPitch * sizeof(T);
    if (smem > 48 * 1024) CU(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<wt_multi_grid(h), kThreads, smem, ctx->stream>>>(a);
    if (auto st = post_launch(ctx, "k_hist_wt_dot_normal")) return st;
    std::vector<double> tmp((size_t)w * k);
    CU(ctx, cudaMemcpyAsync(tmp.data(), result, sizeof(double) * w * k, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    for (int e = 0; e < w * k; e++) R_host[e] = (T)tmp[(size_t)e];
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_hist_lincomb_normal(lbfgs_b200_hist* h, T a0, uint64_t seed, uint32_t stream, uint32_t first, int k, const T* mean,
                                                const T* C_host, T* OUT, int64_t ldo)
{
    if (auto st = normal_check<T>(h, k, first, "hist_lincomb_normal")) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, OUT, "hist_lincomb_normal: NULL argument");
    REQUIRE(ctx, ldo >= h->n, "hist_lincomb_normal: leading dimension %lld is smaller than n = %lld", (long long)ldo, (long long)h->n);
    const int c = h->ncorr;
    double *partials, *result;
    void* coef;
    if (auto st = multi_scratch(h, &partials, &result, &coef)) return st;
    if (c > 0)
    {
        REQUIRE(ctx, C_host != nullptr, "hist_lincomb_normal: NULL argument");
        CU(ctx, cudaMemcpyAsync(coef, C_host, sizeof(T) * 2 * c * k, cudaMemcpyHostToDevice, ctx->stream));
        CU(ctx, cudaStreamSynchronize(ctx->stream));   // C_host may be a stack array of the caller
    }
    LincombNormalArgs<T> a{};
    a.n = h->n; a.ld = h->ld; a.ldv = 0; a.ldo = ldo; a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y);
    a.V = nullptr; a.a0 = a0; a.coef = static_cast<const T*>(coef); a.cls = nullptr; a.mask = 0; a.out = OUT; a.c = c; a.k = k;
    a.mean = mean; a.src = NormalSrc{(unsigned long long)seed, stream, first};
    fill_slots<T>(h, a.slots);
    const int64_t npairs = (h->n + 1) / 2;
    if (k == 1) k_hist_lincomb<T, 1, LincombNormalArgs<T>><<<grid_for(ctx, npairs * 4, 4), kThreads, 0, ctx->stream>>>(a);
    else k_hist_lincomb<T, kMaxK, LincombNormalArgs<T>><<<grid_for(ctx, npairs * 4, 4), kThreads, 0, ctx->stream>>>(a);
    return post_launch(ctx, "k_hist_lincomb_normal");
}

// out_i = a0 + r_i' K r_i (see k_hist_quad_diag): K's upper triangle is packed, off-diagonal entries doubled, on the host (exact
// in binary floating point), and the kernel's width is chosen from c alone, so a row's arithmetic depends on c, K and the row only
template <class T, class A = QuadDiagArgs<T>>
static lbfgs_b200_status do_hist_quad_diag(lbfgs_b200_hist* h, T a0, const T* K_host, T* out, const unsigned char* fcls = nullptr, int fmask = 0)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, ctx->nranks == 1, "hist_quad_diag: replicas only, not for a context with %d ranks", ctx->nranks);
    const int c = h->ncorr, w = 2 * c;
    REQUIRE(ctx, out && (c == 0 || K_host), "hist_quad_diag: NULL argument");
    const int nk = w * (w + 1) / 2;
    std::vector<double> kp((size_t)(nk > 0 ? nk : 1));
    for (int p = 0, e = 0; p < w; p++)
        for (int q = p; q < w; q++, e++) kp[(size_t)e] = (q == p ? 1.0 : 2.0) * (double)K_host[p * w + q];
    if (!h->quad)
    {
        const cudaError_t e = pool_alloc(ctx, &h->quad, sizeof(double) * (size_t)h->m * (2 * h->m + 1));
        if (e != cudaSuccess)
            return fail(ctx, e == cudaErrorMemoryAllocation ? LBFGS_B200_ERR_ALLOC : LBFGS_B200_ERR_CUDA, "history scratch: %s", cudaGetErrorString(e));
    }
    if (nk > 0)
    {
        CU(ctx, cudaMemcpyAsync(h->quad, kp.data(), sizeof(double) * (size_t)nk, cudaMemcpyHostToDevice, ctx->stream));
        CU(ctx, cudaStreamSynchronize(ctx->stream));   // kp is freed on return
    }
    A a{};
    a.n = h->n; a.ld = h->ld; a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y);
    a.Kp = static_cast<const double*>(h->quad); a.a0 = (double)a0; a.out = out; a.c = c;
    if constexpr (unmasked<A>::masked) { a.fcls = fcls; a.fmask = (unsigned char)fmask; }
    else (void)fcls, (void)fmask;
    fill_slots<T>(h, a.slots);
    const size_t smem = sizeof(double) * (size_t)nk;
    auto launch = [&](auto kernel, int rpt) -> lbfgs_b200_status {
        if (smem > 48 * 1024) CU(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const int64_t span = (int64_t)kThreads * rpt, want = (h->n + span - 1) / span, cap = (int64_t)ctx->sm_count * 8;
        kernel<<<(int)(want < 1 ? 1 : want < cap ? want : cap), kThreads, smem, ctx->stream>>>(a);
        return post_launch(ctx, "k_hist_quad_diag");
    };
    if (w <= 16) return launch(k_hist_quad_diag<T, 16, A>, quad_diag_rpt<16>());
    if (w <= 32) return launch(k_hist_quad_diag<T, 32, A>, quad_diag_rpt<32>());
    if (w <= 64) return launch(k_hist_quad_diag<T, 64, A>, quad_diag_rpt<64>());
    if constexpr (unmasked<A>::masked) return fail(ctx, LBFGS_B200_ERR_INVALID, "hist_quad_diag_masked: the box path keeps m <= 20");
    else return launch(k_hist_quad_diag<T, kMaxW>, quad_diag_rpt<kMaxW>());
}

// G[(2c)x(2c)] over rows with (cls & mask) != 0, ordering [Y by age, S by age]   (WP'WP of BFGSMat.h:529-565)
template <class T>
static lbfgs_b200_status do_hist_masked_gram(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, T* G_host)
{
    if (auto st = hist_check<T>(h)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    const int c = h->ncorr, w = 2 * c;
    if (c == 0) return LBFGS_B200_OK;
    REQUIRE(ctx, b && G_host, "hist_masked_gram: NULL argument");
    MaskedGramArgs<T> a{};
    a.n = h->n; a.ld = h->ld; a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y);
    a.cls = cls; a.mask = (unsigned char)mask; a.c = c;
    a.partials = b->mg_partials; a.ticket = ctx->rb.ticket; a.result = b->mg_result;
    fill_slots<T>(h, a.slots);
    const int64_t nstrips = (h->n + kMgRows - 1) / kMgRows;
    const int grid = (int)(nstrips < 2 * ctx->sm_count ? nstrips : 2 * ctx->sm_count);
    const size_t smem = (size_t)w * kMgRows * sizeof(T);
    if (smem > 48 * 1024) CU(ctx, cudaFuncSetAttribute(k_masked_gram<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_masked_gram<T><<<grid, kThreads, smem, ctx->stream>>>(a);
    if (auto st = post_launch(ctx, "k_masked_gram")) return st;
    std::vector<double> tmp((size_t)w * w);
    CU(ctx, cudaMemcpyAsync(tmp.data(), b->mg_result, sizeof(double) * w * w, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    for (int e = 0; e < w * w; e++) G_host[e] = (T)tmp[e];
    return LBFGS_B200_OK;
}

// ------------------------------------------------------------------------------------------------ the masked k-vector passes
// The passes above restricted to the rows with (cls & mask) != 0 (k_hist_wt_dot_multi / k_hist_lincomb / k_hist_quad_diag with
// Masked<A>): the final approximation on the free variables of a bound-constrained solve.  Each follows its twin's rules (replicas
// only, 1 <= k <= 16) and needs the history's box workspace and class bytes.
static lbfgs_b200_status mask_check(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, const char* what)
{
    REQUIRE(h->ctx, b && b->h == h && cls, "%s: NULL argument or a box of another history", what);
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_hist_wt_dot_multi_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, int k,
                                                     const T* V, int64_t ldv, T* R_host)
{
    if (auto st = multi_check<T>(h, k, ldv, "hist_wt_dot_multi_masked")) return st;
    if (auto st = mask_check(h, b, cls, "hist_wt_dot_multi_masked")) return st;
    REQUIRE(h->ctx, V && R_host, "hist_wt_dot_multi_masked: NULL argument");
    const int w = 2 * h->ncorr;
    if (w == 0) return LBFGS_B200_OK;
    Masked<WtDotMultiArgs<T>> a{};
    a.V = V; a.ldv = ldv; a.k = k; a.fcls = cls; a.fmask = (unsigned char)mask;
    std::vector<double> tmp;
    if (auto st = run_wt_dots<T>(h, a, w, w, tmp, "k_hist_wt_dot_multi_masked")) return st;
    for (int e = 0; e < w * k; e++) R_host[e] = (T)tmp[(size_t)e];
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_hist_wt_dot_diff_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, int k, const T* X,
                                                    int64_t ldx, const T* mean, double* R_host, double* nrm_host)
{
    if (auto st = multi_check<T>(h, k, ldx, "hist_wt_dot_diff_masked")) return st;
    if (auto st = mask_check(h, b, cls, "hist_wt_dot_diff_masked")) return st;
    REQUIRE(h->ctx, X && mean && R_host && nrm_host, "hist_wt_dot_diff_masked: NULL argument");
    const int w = 2 * h->ncorr;
    Masked<WtDotDiffArgs<T>> a{};
    a.V = X; a.ldv = ldx; a.k = k; a.mean = mean; a.fcls = cls; a.fmask = (unsigned char)mask;
    std::vector<double> tmp;
    if (auto st = run_wt_dots<T>(h, a, w, w + 1, tmp, "k_hist_wt_dot_diff_masked")) return st;
    for (int e = 0; e < w * k; e++) R_host[e] = tmp[(size_t)e];
    for (int j = 0; j < k; j++) nrm_host[j] = tmp[(size_t)(w * k + j)];
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_hist_wt_dot_normal_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, uint64_t seed,
                                                      uint32_t stream, uint32_t first, int k, T* R_host)
{
    if (auto st = normal_check<T>(h, k, first, "hist_wt_dot_normal_masked")) return st;
    if (auto st = mask_check(h, b, cls, "hist_wt_dot_normal_masked")) return st;
    REQUIRE(h->ctx, R_host, "hist_wt_dot_normal_masked: NULL argument");
    const int w = 2 * h->ncorr;
    if (w == 0) return LBFGS_B200_OK;
    Masked<WtDotNormalArgs<T>> a{};
    a.V = nullptr; a.ldv = 0; a.k = k; a.src = NormalSrc{(unsigned long long)seed, stream, first}; a.fcls = cls; a.fmask = (unsigned char)mask;
    std::vector<double> tmp;
    if (auto st = run_wt_dots<T>(h, a, w, w, tmp, "k_hist_wt_dot_normal_masked")) return st;
    for (int e = 0; e < w * k; e++) R_host[e] = (T)tmp[(size_t)e];
    return LBFGS_B200_OK;
}

// the coefficients [2c][k] to the scratch of the k-vector passes (C_host may be a stack array of the caller)
template <class T> static lbfgs_b200_status upload_coef(lbfgs_b200_hist* h, int k, const T* C_host, void** coef, const char* what)
{
    double *partials, *result;
    if (auto st = multi_scratch(h, &partials, &result, coef)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    if (h->ncorr > 0)
    {
        REQUIRE(ctx, C_host != nullptr, "%s: NULL argument", what);
        CU(ctx, cudaMemcpyAsync(*coef, C_host, sizeof(T) * 2 * h->ncorr * k, cudaMemcpyHostToDevice, ctx->stream));
        CU(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_hist_lincomb_multi_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, T a0, int k,
                                                      const T* V, int64_t ldv, const T* C_host, T* OUT, int64_t ldo)
{
    if (auto st = multi_check<T>(h, k, ldv, "hist_lincomb_multi_masked")) return st;
    if (auto st = mask_check(h, b, cls, "hist_lincomb_multi_masked")) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, V && OUT, "hist_lincomb_multi_masked: NULL argument");
    REQUIRE(ctx, ldo >= h->n, "hist_lincomb_multi_masked: leading dimension %lld is smaller than n = %lld", (long long)ldo, (long long)h->n);
    void* coef;
    if (auto st = upload_coef<T>(h, k, C_host, &coef, "hist_lincomb_multi_masked")) return st;
    Masked<LincombArgs<T>> a{};
    a.n = h->n; a.ld = h->ld; a.ldv = ldv; a.ldo = ldo; a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y);
    a.V = V; a.a0 = a0; a.coef = static_cast<const T*>(coef); a.cls = nullptr; a.mask = 0; a.out = OUT; a.c = h->ncorr; a.k = k;
    a.fcls = cls; a.fmask = (unsigned char)mask;
    fill_slots<T>(h, a.slots);
    if (k == 1) k_hist_lincomb<T, 1, Masked<LincombArgs<T>>><<<grid_for(ctx, h->n * 4, 4), kThreads, 0, ctx->stream>>>(a);
    else k_hist_lincomb<T, kMaxK, Masked<LincombArgs<T>>><<<grid_for(ctx, h->n * 4, 4), kThreads, 0, ctx->stream>>>(a);
    return post_launch(ctx, "k_hist_lincomb_masked");
}

template <class T>
static lbfgs_b200_status do_hist_lincomb_normal_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, T a0,
                                                       uint64_t seed, uint32_t stream, uint32_t first, int k, const T* mean, const T* C_host,
                                                       T* OUT, int64_t ldo)
{
    if (auto st = normal_check<T>(h, k, first, "hist_lincomb_normal_masked")) return st;
    if (auto st = mask_check(h, b, cls, "hist_lincomb_normal_masked")) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, OUT, "hist_lincomb_normal_masked: NULL argument");
    REQUIRE(ctx, ldo >= h->n, "hist_lincomb_normal_masked: leading dimension %lld is smaller than n = %lld", (long long)ldo, (long long)h->n);
    void* coef;
    if (auto st = upload_coef<T>(h, k, C_host, &coef, "hist_lincomb_normal_masked")) return st;
    Masked<LincombNormalArgs<T>> a{};
    a.n = h->n; a.ld = h->ld; a.ldv = 0; a.ldo = ldo; a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y);
    a.V = nullptr; a.a0 = a0; a.coef = static_cast<const T*>(coef); a.cls = nullptr; a.mask = 0; a.out = OUT; a.c = h->ncorr; a.k = k;
    a.mean = mean; a.src = NormalSrc{(unsigned long long)seed, stream, first}; a.fcls = cls; a.fmask = (unsigned char)mask;
    fill_slots<T>(h, a.slots);
    const int64_t npairs = (h->n + 1) / 2;
    if (k == 1) k_hist_lincomb<T, 1, Masked<LincombNormalArgs<T>>><<<grid_for(ctx, npairs * 4, 4), kThreads, 0, ctx->stream>>>(a);
    else k_hist_lincomb<T, kMaxK, Masked<LincombNormalArgs<T>>><<<grid_for(ctx, npairs * 4, 4), kThreads, 0, ctx->stream>>>(a);
    return post_launch(ctx, "k_hist_lincomb_normal_masked");
}

template <class T>
static lbfgs_b200_status do_hist_quad_diag_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, T a0, const T* K_host,
                                                  T* out)
{
    if (auto st = hist_check<T>(h)) return st;
    if (auto st = mask_check(h, b, cls, "hist_quad_diag_masked")) return st;
    return do_hist_quad_diag<T, Masked<QuadDiagArgs<T>>>(h, a0, K_host, out, cls, mask);
}

// CLS_FINAL on the free coordinates of x (k_box_final_classes); *nfree_host = their number
template <class T>
static lbfgs_b200_status do_box_final_classes(lbfgs_b200_box* b, const T* x, const T* lb, const T* ub, T tol, int64_t* nfree_host)
{
    if (auto st = box_check<T>(b)) return st;
    lbfgs_b200_ctx* ctx = b->h->ctx;
    REQUIRE(ctx, x && lb && ub && nfree_host, "box_final_classes: NULL argument");
    REQUIRE(ctx, tol >= T(0), "box_final_classes: tol must be >= 0");
    const ReduceBuf rb = next_rb(ctx, true);
    k_box_final_classes<T><<<grid_for(ctx, b->n * 4, 4), kThreads, 0, ctx->stream>>>(b->n, x, lb, ub, tol, b->cls, rb);
    if (auto st = post_launch(ctx, "k_box_final_classes")) return st;
    if (auto st = receive(ctx, 1)) return st;
    *nfree_host = (int64_t)ctx->h_result[0];
    return LBFGS_B200_OK;
}

// ------------------------------------------------------------------------------------------------ box workspace
static void box_free(lbfgs_b200_box* b)
{
    if (!b) return;
    for (void* p : {b->brk, b->dvec, b->xcp, b->vecc, b->vecy, b->lambda, b->mu, b->tmp, b->tmp2, b->yfb, (void*)b->cls,
                    (void*)b->keys, (void*)b->ord, (void*)b->keys2, (void*)b->ord2, (void*)b->radix_hist, b->block_sums, (void*)b->best, b->small, (void*)b->mg_partials, (void*)b->mg_result})
        pool_free(b->h ? b->h->ctx : nullptr, p);
    delete b;
}

template <class T> static lbfgs_b200_status sweep_launch(lbfgs_b200_box* b, const SweepArgs<T>& a, int which, long long target, int64_t nblocks)
{
    lbfgs_b200_ctx* ctx = b->h->ctx;
    const int nv = 4 * a.c + 1;
    const size_t smem = (size_t)kScanBlock * (size_t)((nv <= 25 ? 25 : nv <= 41 ? 41 : 81) + 1) * sizeof(T);
#define SWEEP_CASE(MAXV)                                                                                                   \
    do {                                                                                                                   \
        if (which == 0) k_sweep_blocksum<T, MAXV><<<(unsigned)nblocks, kScanBlock, 0, ctx->stream>>>(a);                   \
        else if (which == 1) {                                                                                             \
            if (smem > 48 * 1024) CU(ctx, cudaFuncSetAttribute(k_sweep_select<T, MAXV, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            k_sweep_select<T, MAXV, false><<<(unsigned)nblocks, kScanBlock, smem, ctx->stream>>>(a, 0);                    \
        } else {                                                                                                           \
            if (smem > 48 * 1024) CU(ctx, cudaFuncSetAttribute(k_sweep_select<T, MAXV, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            k_sweep_select<T, MAXV, true><<<1, kScanBlock, smem, ctx->stream>>>(a, target);                                \
        }                                                                                                                  \
    } while (0)
    if (nv <= 25) SWEEP_CASE(25);
    else if (nv <= 41) SWEEP_CASE(41);
    else SWEEP_CASE(81);
#undef SWEEP_CASE
    return post_launch(ctx, "k_sweep");
}

// sort the finite positive breakpoints by (breakpoint, index): LSD radix sort, 8 bits per pass (lbfgsb_kernels.cuh)
template <class T> static lbfgs_b200_status box_sort(lbfgs_b200_box* b)
{
    lbfgs_b200_ctx* ctx = b->h->ctx;
    const int64_t npad = b->npad;
    const int g = grid_for(ctx, npad * 4, 4);
    if (sizeof(T) == 8) k_sort_fill<<<g, kThreads, 0, ctx->stream>>>(b->n, npad, static_cast<const double*>(b->brk), b->cls, b->keys, b->ord);
    else k_sort_fill_f32<<<g, kThreads, 0, ctx->stream>>>(b->n, npad, static_cast<const float*>(b->brk), b->cls, b->keys, b->ord);
    if (auto st = post_launch(ctx, "k_sort_fill")) return st;
    const unsigned tiles = (unsigned)(npad / kSortTile);
    unsigned long long* kin = b->keys; unsigned long long* kout = b->keys2;
    unsigned* iin = b->ord; unsigned* iout = b->ord2;
    const int passes = (sizeof(T) == 8) ? 8 : 4;          // an even number of passes: the result is back in keys / ord
    for (int p = 0; p < passes; p++)
    {
        k_radix_hist<<<tiles, 256, 0, ctx->stream>>>(kin, 8 * p, b->radix_hist, tiles);
        if (auto st = post_launch(ctx, "k_radix_hist")) return st;
        k_radix_scan<<<1, 1024, 0, ctx->stream>>>(b->radix_hist, (unsigned)kRadix * tiles);
        if (auto st = post_launch(ctx, "k_radix_scan")) return st;
        k_radix_scatter<<<tiles, 256, 0, ctx->stream>>>(kin, iin, kout, iout, 8 * p, b->radix_hist, tiles);
        if (auto st = post_launch(ctx, "k_radix_scatter")) return st;
        std::swap(kin, kout);
        std::swap(iin, iout);
    }
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_box_cauchy_breaks(lbfgs_b200_box* b, const T* x, const T* g, const T* lb, const T* ub, T* out5_host)
{
    if (auto st = box_check<T>(b)) return st;
    lbfgs_b200_ctx* ctx = b->h->ctx;
    REQUIRE(ctx, x && g && lb && ub && out5_host, "box_cauchy_breaks: NULL argument");
    const ReduceBuf rb = next_rb(ctx, true);
    k_cauchy_breaks<T><<<grid_for(ctx, b->n * 4, 4), kThreads, 0, ctx->stream>>>(b->n, x, g, lb, ub, static_cast<T*>(b->brk),
                                                                                static_cast<T*>(b->dvec), b->cls, rb);
    if (auto st = post_launch(ctx, "k_cauchy_breaks")) return st;
    if (auto st = receive(ctx, 5)) return st;
    for (int k = 0; k < 4; k++) out5_host[k] = (T)ctx->h_result[k];
    out5_host[4] = (T)(-ctx->h_result[4]);   // smallest breakpoint (+inf when there is none)
    return LBFGS_B200_OK;
}

// The sweep over the sorted breakpoints (Cauchy.h:132-256) for the case where the minimiser is not in the first segment.
// Mmat_host: [2c][2c] row-major (M of B = theta*I - W M W'), p0_host: W'd [2c] (theta applied), gt = d.d, nord / nfree_inf
// from box_cauchy_breaks.  out_host: [0]=t_cross, [1]=tfinal, [2]=fp, [3]=fpp, [4]=all crossed (0/1), [5..5+2c)=W'(xcp-x0).
template <class T>
static lbfgs_b200_status do_box_cauchy_sweep(lbfgs_b200_box* b, const T* g, const T* Mmat_host, const T* p0_host, T theta, T gt,
                                             int64_t nord, int64_t nfree_inf, T* out_host)
{
    if (auto st = box_check<T>(b)) return st;
    lbfgs_b200_hist* h = b->h;
    lbfgs_b200_ctx* ctx = h->ctx;
    const int c = h->ncorr, w = 2 * c, m = h->m;
    REQUIRE(ctx, g && out_host && nord >= 1, "box_cauchy_sweep: bad arguments");
    REQUIRE(ctx, m <= 20, "the bound-constrained path supports m <= 20 (got %d)", m);
    if (h->pending >= 0) if (auto st = gram_refresh<T>(h)) return st;
    if (auto st = box_sort<T>(b)) return st;
    T* small = static_cast<T*>(b->small);
    T* d_M = small;
    T* d_p0 = small + (size_t)4 * m * m;
    T* d_out = small + (size_t)4 * m * m + 4 * m;
    if (c > 0)
    {
        CU(ctx, cudaMemcpyAsync(d_M, Mmat_host, sizeof(T) * w * w, cudaMemcpyHostToDevice, ctx->stream));
        CU(ctx, cudaMemcpyAsync(d_p0, p0_host, sizeof(T) * w, cudaMemcpyHostToDevice, ctx->stream));
    }
    const long long init = LLONG_MAX;
    CU(ctx, cudaMemcpyAsync(b->best, &init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    SweepArgs<T> a{};
    a.nord = nord; a.ld = h->ld; a.keys = b->keys; a.ord = b->ord; a.g = g;
    a.S = static_cast<const T*>(h->S); a.Y = static_cast<const T*>(h->Y); a.c = c; a.theta = theta;
    fill_slots<T>(h, a.slots);
    a.Mmat = d_M; a.p0 = d_p0; a.gt = gt; a.nfree_inf = (int)(nfree_inf > 0 ? 1 : 0);
    a.block_sums = static_cast<T*>(b->block_sums); a.best = b->best; a.out = d_out;
    const int64_t nblocks = (nord + kScanBlock - 1) / kScanBlock;
    if (auto st = sweep_launch<T>(b, a, 0, 0, nblocks)) return st;
    k_sweep_scan_blocks<T><<<1, 1024, 0, ctx->stream>>>(static_cast<T*>(b->block_sums), nblocks, 4 * c + 1);
    if (auto st = post_launch(ctx, "k_sweep_scan_blocks")) return st;
    if (auto st = sweep_launch<T>(b, a, 1, 0, nblocks)) return st;
    long long best = 0;
    CU(ctx, cudaMemcpyAsync(&best, b->best, sizeof(best), cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    REQUIRE(ctx, best >= 0 && best < nord, "cauchy sweep found no segment (internal error)");
    if (auto st = sweep_launch<T>(b, a, 2, best, nblocks)) return st;
    std::vector<T> tmp(5 + w);
    CU(ctx, cudaMemcpyAsync(tmp.data(), d_out, sizeof(T) * (5 + w), cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < 5 + w; k++) out_host[k] = tmp[k];
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_box_cauchy_build(lbfgs_b200_box* b, const T* x, const T* lb, const T* ub, T t_cross, T tfinal, T* counts2_host)
{
    if (auto st = box_check<T>(b)) return st;
    lbfgs_b200_ctx* ctx = b->h->ctx;
    const ReduceBuf rb = next_rb(ctx, true);
    k_cauchy_build<T><<<grid_for(ctx, b->n * 4, 4), kThreads, 0, ctx->stream>>>(b->n, x, static_cast<const T*>(b->dvec),
                                                                               static_cast<const T*>(b->brk), lb, ub, t_cross, tfinal,
                                                                               static_cast<T*>(b->xcp), b->cls, rb);
    if (auto st = post_launch(ctx, "k_cauchy_build")) return st;
    if (auto st = receive(ctx, 2)) return st;
    counts2_host[0] = (T)ctx->h_result[0];
    counts2_host[1] = (T)ctx->h_result[1];
    return LBFGS_B200_OK;
}

template <class T>
static lbfgs_b200_status do_box_sub_step(lbfgs_b200_box* b, int op, int flag, const T* x0, const T* g, const T* lb, const T* ub, T* drt,
                                         T theta, T* out3_host)
{
    if (auto st = box_check<T>(b)) return st;
    lbfgs_b200_ctx* ctx = b->h->ctx;
    REQUIRE(ctx, op >= 0 && op < SUB_OP_COUNT, "box_sub_step: unknown op %d", op);
    SubVec<T> s{};
    s.n = b->n; s.x0 = x0; s.xcp = static_cast<const T*>(b->xcp); s.g = g; s.lb = lb; s.ub = ub; s.cls = b->cls;
    s.vecc = static_cast<T*>(b->vecc); s.vecy = static_cast<T*>(b->vecy); s.lambda = static_cast<T*>(b->lambda);
    s.mu = static_cast<T*>(b->mu); s.tmp = static_cast<T*>(b->tmp); s.tmp2 = static_cast<T*>(b->tmp2);
    s.yfb = static_cast<T*>(b->yfb); s.drt = drt; s.theta = theta;
    const bool reduces = (op == SUB_OP_CHECK_BOUNDS || op == SUB_OP_CLASSIFY || op == SUB_OP_CONVERGED || op == SUB_OP_WRITE_DRT);
    const ReduceBuf rb = reduces ? next_rb(ctx, true) : ctx->rb;
    const int grid = grid_for(ctx, b->n * 4, 4);
#define SUB_CASE(OP) case OP: k_sub_step<T, OP><<<grid, kThreads, 0, ctx->stream>>>(s, flag, rb); break;
    switch (op)
    {
        SUB_CASE(SUB_OP_INIT) SUB_CASE(SUB_OP_ACT_DIR) SUB_CASE(SUB_OP_ADD_G) SUB_CASE(SUB_OP_NEG_C_FREE)
        SUB_CASE(SUB_OP_CHECK_BOUNDS) SUB_CASE(SUB_OP_CLASSIFY) SUB_CASE(SUB_OP_LU_VEC) SUB_CASE(SUB_OP_RHS_P)
        SUB_CASE(SUB_OP_FREE_VEC) SUB_CASE(SUB_OP_MULTIPLIERS) SUB_CASE(SUB_OP_CONVERGED) SUB_CASE(SUB_OP_WRITE_DRT)
    }
#undef SUB_CASE
    if (auto st = post_launch(ctx, "k_sub_step")) return st;
    if (reduces)
    {
        if (auto st = receive(ctx, 3)) return st;
        if (out3_host) for (int k = 0; k < 3; k++) out3_host[k] = (T)ctx->h_result[k];
    }
    return LBFGS_B200_OK;
}

extern "C" {

lbfgs_b200_status lbfgs_b200_box_create(lbfgs_b200_hist* h, lbfgs_b200_box** out)
{
    if (!h || !h->ctx || !out) return LBFGS_B200_ERR_INVALID;
    lbfgs_b200_ctx* ctx = h->ctx;
    *out = nullptr;
    REQUIRE(ctx, h->m <= 20, "the bound-constrained path supports m <= 20 (got %d)", h->m);
    lbfgs_b200_box* b = new (std::nothrow) lbfgs_b200_box();
    if (!b) return fail(ctx, LBFGS_B200_ERR_ALLOC, "out of host memory");
    b->h = h; b->n = h->n;
    const int64_t npad = ((h->n + kSortTile - 1) / kSortTile) * kSortTile;   // whole tiles of the radix sort
    b->npad = npad;
    const size_t vb = (size_t)h->ld * h->elem;
    const int m = h->m, w = 2 * m;
    cudaError_t e = cudaSetDevice(ctx->device);
    for (void** p : {&b->brk, &b->dvec, &b->xcp, &b->vecc, &b->vecy, &b->lambda, &b->mu, &b->tmp, &b->tmp2, &b->yfb})
        if (e == cudaSuccess) e = pool_alloc(ctx, p, vb);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&b->cls, (size_t)h->ld);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&b->keys, sizeof(unsigned long long) * npad);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&b->ord, sizeof(unsigned) * npad);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&b->keys2, sizeof(unsigned long long) * npad);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&b->ord2, sizeof(unsigned) * npad);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&b->radix_hist, sizeof(unsigned) * (size_t)kRadix * (npad / kSortTile));
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&b->block_sums, (size_t)h->elem * (npad / kScanBlock + 1) * (4 * m + 1));
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&b->best, sizeof(long long));
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&b->small, (size_t)h->elem * (4 * m * m + 4 * m + 5 + w + 16));
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&b->mg_partials, sizeof(double) * 2 * ctx->sm_count * w * w);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&b->mg_result, sizeof(double) * w * w);
    if (e != cudaSuccess)
    {
        box_free(b);
        return fail(ctx, e == cudaErrorMemoryAllocation ? LBFGS_B200_ERR_ALLOC : LBFGS_B200_ERR_CUDA, "box_create: %s", cudaGetErrorString(e));
    }
    *out = b;
    return LBFGS_B200_OK;
}

void lbfgs_b200_box_destroy(lbfgs_b200_box* b)
{
    box_free(b);
}

const void* lbfgs_b200_box_xcp(const lbfgs_b200_box* b) { return b ? b->xcp : nullptr; }
const unsigned char* lbfgs_b200_box_classes(const lbfgs_b200_box* b) { return b ? b->cls : nullptr; }
void* lbfgs_b200_box_vector(lbfgs_b200_box* b, int which)
{
    if (!b) return nullptr;
    void* v[] = {b->vecc, b->vecy, b->lambda, b->mu, b->tmp, b->tmp2, b->yfb, b->dvec, b->brk, b->xcp};
    return (which >= 0 && which < 10) ? v[which] : nullptr;
}

#define DEFINE_BOX(T, SUF)                                                                                                  \
    lbfgs_b200_status lbfgs_b200_box_clamp_##SUF(lbfgs_b200_ctx* ctx, int64_t n, T* x, const T* lb, const T* ub)            \
    {                                                                                                                       \
        REQUIRE(ctx, ctx && x && lb && ub && n >= 0, "box_clamp: bad arguments");                                           \
        k_box_clamp<T><<<grid_for(ctx, n * 4, 4), kThreads, 0, ctx->stream>>>(n, x, lb, ub);                               \
        return post_launch(ctx, "k_box_clamp");                                                                             \
    }                                                                                                                       \
    lbfgs_b200_status lbfgs_b200_box_proj_grad_norm_##SUF(lbfgs_b200_ctx* ctx, int64_t n, const T* x, const T* g,           \
                                                          const T* lb, const T* ub, T* out_host)                            \
    {                                                                                                                       \
        REQUIRE(ctx, ctx && x && g && lb && ub && out_host, "box_proj_grad_norm: bad arguments");                           \
        REQUIRE(ctx, ctx->nranks == 1, "the bound-constrained path is not n-sharded");                                      \
        const ReduceBuf rb = next_rb(ctx, true);                                                                            \
        k_box_pgnorm<T><<<grid_for(ctx, n * 4, 4), kThreads, 0, ctx->stream>>>(n, x, g, lb, ub, rb);                       \
        if (auto st = post_launch(ctx, "k_box_pgnorm")) return st;                                                          \
        if (auto st = receive(ctx, 1)) return st;                                                                           \
        *out_host = (T)ctx->h_result[0];                                                                                    \
        return LBFGS_B200_OK;                                                                                               \
    }                                                                                                                       \
    lbfgs_b200_status lbfgs_b200_box_dir_info_##SUF(lbfgs_b200_ctx* ctx, int64_t n, const T* x, const T* d, const T* g,     \
                                                    const T* lb, const T* ub, T* out2_host)                                 \
    {                                                                                                                       \
        REQUIRE(ctx, ctx && x && d && g && lb && ub && out2_host, "box_dir_info: bad arguments");                           \
        REQUIRE(ctx, ctx->nranks == 1, "the bound-constrained path is not n-sharded");                                      \
        const ReduceBuf rb = next_rb(ctx, true);                                                                            \
        k_box_dirinfo<T><<<grid_for(ctx, n * 4, 4), kThreads, 0, ctx->stream>>>(n, x, d, g, lb, ub, rb);                   \
        if (auto st = post_launch(ctx, "k_box_dirinfo")) return st;                                                         \
        if (auto st = receive(ctx, 2)) return st;                                                                           \
        out2_host[0] = (T)ctx->h_result[0];                                                                                 \
        out2_host[1] = (T)(-ctx->h_result[1]);                                                                              \
        return LBFGS_B200_OK;                                                                                               \
    }                                                                                                                       \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_##SUF(lbfgs_b200_hist* h, const T* v, T* raw_host)                             \
    { return do_hist_wt_dot<T>(h, v, raw_host); }                                                                           \
    lbfgs_b200_status lbfgs_b200_hist_gram_##SUF(lbfgs_b200_hist* h, T* SY, T* SS, T* YY, T* ys, T* theta)                  \
    { return do_hist_gram<T>(h, SY, SS, YY, ys, theta); }                                                                   \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, T a0, const T* v0,               \
                                                    const T* coef_host, const unsigned char* cls, int mask, T* out)         \
    { return do_hist_lincomb<T>(h, b, a0, v0, coef_host, cls, mask, out); }                                                 \
    lbfgs_b200_status lbfgs_b200_hist_masked_gram_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls,    \
                                                        int mask, T* G_host)                                                \
    { return do_hist_masked_gram<T>(h, b, cls, mask, G_host); }                                                             \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_multi_##SUF(lbfgs_b200_hist* h, int k, const T* V, int64_t ldv, T* R_host)     \
    { return do_hist_wt_dot_multi<T>(h, k, V, ldv, R_host); }                                                               \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_multi_##SUF(lbfgs_b200_hist* h, T a0, int k, const T* V, int64_t ldv,         \
                                                          const T* C_host, T* OUT, int64_t ldo)                             \
    { return do_hist_lincomb_multi<T>(h, a0, k, V, ldv, C_host, OUT, ldo); }                                                \
    lbfgs_b200_status lbfgs_b200_hist_quad_diag_##SUF(lbfgs_b200_hist* h, T a0, const T* K_host, T* out)                    \
    { return do_hist_quad_diag<T>(h, a0, K_host, out); }                                                                    \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_normal_##SUF(lbfgs_b200_hist* h, uint64_t seed, uint32_t stream, uint32_t first,  \
                                                          int k, T* R_host)                                                 \
    { return do_hist_wt_dot_normal<T>(h, seed, stream, first, k, R_host); }                                                  \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_normal_##SUF(lbfgs_b200_hist* h, T a0, uint64_t seed, uint32_t stream,          \
                                                           uint32_t first, int k, const T* mean, const T* C_host, T* OUT,    \
                                                           int64_t ldo)                                                      \
    { return do_hist_lincomb_normal<T>(h, a0, seed, stream, first, k, mean, C_host, OUT, ldo); }                            \
    lbfgs_b200_status lbfgs_b200_hist_s_dot_multi_##SUF(lbfgs_b200_hist* h, int k, const T* V, int64_t ldv, T* R_host)       \
    { return do_hist_s_dot_multi<T>(h, k, V, ldv, R_host); }                                                                 \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_diff_##SUF(lbfgs_b200_hist* h, int k, const T* X, int64_t ldx, const T* mean,   \
                                                        double* R_host, double* nrm_host)                                    \
    { return do_hist_wt_dot_diff<T>(h, k, X, ldx, mean, R_host, nrm_host); }                                                 \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_multi_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, \
                                                                int mask, int k, const T* V, int64_t ldv, T* R_host)          \
    { return do_hist_wt_dot_multi_masked<T>(h, b, cls, mask, k, V, ldv, R_host); }                                           \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_diff_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls,  \
                                                               int mask, int k, const T* X, int64_t ldx, const T* mean,        \
                                                               double* R_host, double* nrm_host)                               \
    { return do_hist_wt_dot_diff_masked<T>(h, b, cls, mask, k, X, ldx, mean, R_host, nrm_host); }                            \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_normal_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, \
                                                                 int mask, uint64_t seed, uint32_t stream, uint32_t first,     \
                                                                 int k, T* R_host)                                             \
    { return do_hist_wt_dot_normal_masked<T>(h, b, cls, mask, seed, stream, first, k, R_host); }                             \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_multi_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, \
                                                                 int mask, T a0, int k, const T* V, int64_t ldv,               \
                                                                 const T* C_host, T* OUT, int64_t ldo)                         \
    { return do_hist_lincomb_multi_masked<T>(h, b, cls, mask, a0, k, V, ldv, C_host, OUT, ldo); }                            \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_normal_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b,                      \
                                                                  const unsigned char* cls, int mask, T a0, uint64_t seed,     \
                                                                  uint32_t stream, uint32_t first, int k, const T* mean,      \
                                                                  const T* C_host, T* OUT, int64_t ldo)                        \
    { return do_hist_lincomb_normal_masked<T>(h, b, cls, mask, a0, seed, stream, first, k, mean, C_host, OUT, ldo); }         \
    lbfgs_b200_status lbfgs_b200_hist_quad_diag_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls,   \
                                                             int mask, T a0, const T* K_host, T* out)                          \
    { return do_hist_quad_diag_masked<T>(h, b, cls, mask, a0, K_host, out); }                                                \
    lbfgs_b200_status lbfgs_b200_box_final_classes_##SUF(lbfgs_b200_box* b, const T* x, const T* lb, const T* ub, T tol,      \
                                                         int64_t* nfree_host)                                                  \
    { return do_box_final_classes<T>(b, x, lb, ub, tol, nfree_host); }                                                       \
    lbfgs_b200_status lbfgs_b200_box_cauchy_breaks_##SUF(lbfgs_b200_box* b, const T* x, const T* g, const T* lb,            \
                                                         const T* ub, T* out5_host)                                         \
    { return do_box_cauchy_breaks<T>(b, x, g, lb, ub, out5_host); }                                                         \
    lbfgs_b200_status lbfgs_b200_box_cauchy_sweep_##SUF(lbfgs_b200_box* b, const T* g, const T* Mmat_host,                  \
                                                        const T* p0_host, T theta, T gt, int64_t nord, int64_t nfree_inf,   \
                                                        T* out_host)                                                        \
    { return do_box_cauchy_sweep<T>(b, g, Mmat_host, p0_host, theta, gt, nord, nfree_inf, out_host); }                      \
    lbfgs_b200_status lbfgs_b200_box_cauchy_build_##SUF(lbfgs_b200_box* b, const T* x, const T* lb, const T* ub,            \
                                                        T t_cross, T tfinal, T* counts2_host)                               \
    { return do_box_cauchy_build<T>(b, x, lb, ub, t_cross, tfinal, counts2_host); }                                         \
    lbfgs_b200_status lbfgs_b200_box_sub_step_##SUF(lbfgs_b200_box* b, int op, int flag, const T* x0, const T* g,           \
                                                    const T* lb, const T* ub, T* drt, T theta, T* out3_host)                \
    { return do_box_sub_step<T>(b, op, flag, x0, g, lb, ub, drt, theta, out3_host); }

DEFINE_BOX(double, f64)
DEFINE_BOX(float, f32)

}  // extern "C"
