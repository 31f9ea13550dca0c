// small_batch.cu -- the small-batch solve (small_batch.cuh): fp64 / fp32 instantiations, the shared-memory budget and the C ABI.
#include "internal.cuh"
#include "two_loop_gram.cuh"
#include "small_batch.cuh"

// the kept final histories of a small-batch solve (SmallHistLayout per problem) and their pair counts
struct lbfgs_b200_small_hist
{
    lbfgs_b200_ctx* ctx = nullptr;
    int64_t n = 0, B = 0;
    int m = 0, elem = 8;
    void* data = nullptr;
    int* counts = nullptr;
    bool filled = false;   // a solve has written every problem's record
};

namespace {

// what a built-in objective adds to the vectors of a problem: x_lo/g_lo when its trials are stored, and its data vectors
bool small_objective_shape(int objective, bool& stored, int& data_vectors)
{
    if (objective < LBFGS_B200_OBJ_ROSENBROCK_PAIRED || objective > LBFGS_B200_OBJ_QUAD_TRIDIAG) return false;
    with_objective<double>(nullptr, objective, [&](auto tag) {
        using OBJ = decltype(tag);
        stored = OBJ::kHalo;
        data_vectors = OBJ::kDataVectors;
        return LBFGS_B200_OK;
    });
    return true;
}

template <class T>
lbfgs_b200_status small_minimize(lbfgs_b200_ctx* ctx, int objective, const T* data0, const T* data1, int64_t ldd, int64_t n, int64_t B,
                                 const lbfgs_b200_param* prm, int ls_kind, T* X, int64_t ldx, T* G, lbfgs_b200_outcome* outs_host,
                                 lbfgs_b200_small_hist* keep = nullptr)
{
    using namespace lb;
    if (!ctx) return LBFGS_B200_ERR_INVALID;
    REQUIRE(ctx, prm && X && outs_host, "small_minimize: NULL argument");
    REQUIRE(ctx, ctx->nranks == 1, "small_minimize: one CTA holds a whole problem, so n cannot be sharded (the context has %d ranks)", ctx->nranks);
    REQUIRE(ctx, prm->m >= 1 && prm->m <= kMaxM, "small_minimize: need 1 <= m <= %d (got %d)", kMaxM, prm->m);
    REQUIRE(ctx, ls_kind >= 0 && ls_kind <= 3, "unknown line search %d", ls_kind);
    REQUIRE(ctx, prm->past <= kMaxPast, "past > %d is not supported by the small-batch solve", kMaxPast);
    REQUIRE(ctx, B >= 1 && B <= 0x7fffffff, "small_minimize: need 1 <= B <= 2^31 - 1 problems (got %lld)", (long long)B);
    REQUIRE(ctx, n >= 1, "small_minimize: need n >= 1 (got %lld)", (long long)n);
    REQUIRE(ctx, ldx >= n, "small_minimize: the batch stride of X (%lld) is shorter than n (%lld)", (long long)ldx, (long long)n);
    REQUIRE(ctx, ldd == 0 || ldd >= n, "small_minimize: the batch stride of the data (%lld) must be 0 (shared) or at least n (%lld)",
            (long long)ldd, (long long)n);
    void* kernel = nullptr;
    bool stored = false;
    int data_vectors = 0;
    lb::ObjGeom<T> geo;
    if (auto st = with_objective<T>(ctx, objective, [&](auto tag) {
            using OBJ = decltype(tag);
            kernel = (void*)k_small_batch<T, OBJ>;
            stored = OBJ::kHalo;
            data_vectors = OBJ::kDataVectors;
            return objective_geometry<OBJ>(ctx, n, data0, data1, geo);
        }))
        return st;
    if (keep)
        REQUIRE(ctx, keep->ctx == ctx && keep->n == n && keep->m == prm->m && keep->elem == (int)sizeof(T) && keep->B == B,
                "small_minimize_keep: the history was made (on this context?) for n = %lld, m = %d, %s, B = %lld; the solve has n = %lld, m = %d, %s, B = %lld",
                (long long)keep->n, keep->m, keep->elem == 8 ? "fp64" : "fp32", (long long)keep->B, (long long)n, prm->m,
                sizeof(T) == 8 ? "fp64" : "fp32", (long long)B);
    const int64_t max_n = lbfgs_b200_small_max_n(prm->m, (int)sizeof(T), objective);
    REQUIRE(ctx, n <= max_n, "small_minimize: n = %lld exceeds %lld, the largest n whose solve fits one CTA's shared memory for m = %d and this "
            "objective in %s; solve larger problems with LBFGSBatchSolver", (long long)n, (long long)max_n, prm->m, sizeof(T) == 8 ? "fp64" : "fp32");

    // the options and the initial ring / op, the same for every problem (the resident solve fills its states with the same helper)
    std::vector<unsigned char> img(sizeof(PState<T>), 0);
    PState<T>& proto = *reinterpret_cast<PState<T>*>(img.data());
    init_problem_state<T>(proto, *prm, ls_kind, true);
    void* buf = nullptr;
    const size_t outs_bytes = sizeof(lbfgs_b200_outcome) * (size_t)B;
    const size_t proto_ofs = (outs_bytes + 255) & ~size_t(255);
    CU(ctx, pool_alloc(ctx, &buf, proto_ofs + sizeof(PState<T>)));
    SmallArgs<T> a{};
    a.proto = reinterpret_cast<const PState<T>*>(static_cast<char*>(buf) + proto_ofs);
    a.M = prm->m + 1;
    a.L = small_layout(n, prm->m, (int)sizeof(T), stored, data_vectors);
    a.n = n;
    a.data0 = data0; a.data1 = data1; a.ldd = ldd;
    a.X = X; a.ldx = ldx; a.G = G;
    a.outs = static_cast<lbfgs_b200_outcome*>(buf);
    if (keep)
    {
        keep->filled = false;
        a.hist = static_cast<T*>(keep->data);
        a.hist_c = keep->counts;
    }
    auto run = [&]() -> cudaError_t {
        cudaError_t e = cudaMemcpyAsync((void*)a.proto, &proto, sizeof(PState<T>), cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)a.L.total);
        void* kargs[] = {&a};
        if (e == cudaSuccess) e = cudaLaunchKernel(kernel, dim3((unsigned)B), dim3((unsigned)small_threads(n)), kargs, a.L.total, ctx->stream);
        if (e == cudaSuccess) ctx->launches++;
        if (e == cudaSuccess) e = cudaMemcpyAsync(outs_host, a.outs, outs_bytes, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        return e;
    };
    const cudaError_t e = run();
    pool_free(ctx, buf);
    CU(ctx, e);
    if (keep) keep->filled = true;
    return LBFGS_B200_OK;
}

template <class T> lbfgs_b200_status small_hist_check(lbfgs_b200_small_hist* h, const char* what)
{
    if (!h) return LBFGS_B200_ERR_INVALID;
    REQUIRE(h->ctx, h->elem == (int)sizeof(T), "%s: the history holds %s values", what, h->elem == 8 ? "fp64" : "fp32");
    REQUIRE(h->ctx, h->filled, "%s: no solve has filled the history", what);
    return LBFGS_B200_OK;
}

template <class T> lbfgs_b200_status small_hist_info(lbfgs_b200_small_hist* h, int* c_host, T* theta_host)
{
    if (auto st = small_hist_check<T>(h, "small_hist_info")) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    const lb::SmallHistLayout HL{h->n, h->m};
    if (c_host) CU(ctx, cudaMemcpyAsync(c_host, h->counts, sizeof(int) * (size_t)h->B, cudaMemcpyDeviceToHost, ctx->stream));
    if (theta_host)
        CU(ctx, cudaMemcpy2DAsync(theta_host, sizeof(T), static_cast<const T*>(h->data) + HL.theta(), sizeof(T) * (size_t)HL.rec(), sizeof(T),
                                  (size_t)h->B, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status small_hist_times(lbfgs_b200_small_hist* h, int inverse, int64_t b0, int64_t count, int k, const T* V, int64_t ldv, int64_t ldvp,
                                   T* OUT, int64_t ldo, int64_t ldop)
{
    using namespace lb;
    if (auto st = small_hist_check<T>(h, "small_hist_times")) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    const int64_t n = h->n;
    REQUIRE(ctx, V && OUT, "small_hist_times: NULL argument");
    REQUIRE(ctx, k >= 1 && (k + kSGroup - 1) / kSGroup <= 65535, "small_hist_times: k must be in 1..%d (got %d)", 65535 * kSGroup, k);
    REQUIRE(ctx, b0 >= 0 && count >= 1 && count <= h->B - b0, "small_hist_times: problems [%lld, %lld) are not within the %lld of the history",
            (long long)b0, (long long)(b0 + count), (long long)h->B);
    REQUIRE(ctx, ldv >= n && ldo >= n, "small_hist_times: leading dimensions ldv = %lld, ldo = %lld must be at least n = %lld", (long long)ldv,
            (long long)ldo, (long long)n);
    REQUIRE(ctx, ldvp >= 0 && ldop >= 0, "small_hist_times: negative problem stride");
    REQUIRE(ctx, (const void*)V != (const void*)OUT || (ldo == ldv && ldop == ldvp && (ldvp > 0 || count == 1)),
            "small_hist_times: OUT may be V only with the same layout (ldo == ldv, ldop == ldvp) and vectors of its own per problem");
    SmallTimesArgs<T> a{};
    a.hist = static_cast<const T*>(h->data); a.hist_c = h->counts; a.HL = SmallHistLayout{n, h->m};
    a.b0 = b0; a.k = k; a.inverse = inverse ? 1 : 0;
    a.V = V; a.ldv = ldv; a.ldvp = ldvp; a.OUT = OUT; a.ldo = ldo; a.ldop = ldop;
    const size_t smem = small_times_smem(h->m, (int)sizeof(T));
    CU(ctx, cudaFuncSetAttribute(k_small_hist_times<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_small_hist_times<T><<<dim3((unsigned)count, (unsigned)((k + kSGroup - 1) / kSGroup)), small_threads(n), smem, ctx->stream>>>(a);
    CU(ctx, cudaGetLastError());
    ctx->launches++;
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status small_hist_diag(lbfgs_b200_small_hist* h, int inverse, int64_t b0, int64_t count, T* OUT, int64_t ldo)
{
    using namespace lb;
    if (auto st = small_hist_check<T>(h, "small_hist_diag")) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    const int64_t n = h->n;
    REQUIRE(ctx, OUT, "small_hist_diag: NULL argument");
    REQUIRE(ctx, b0 >= 0 && count >= 1 && count <= h->B - b0, "small_hist_diag: problems [%lld, %lld) are not within the %lld of the history",
            (long long)b0, (long long)(b0 + count), (long long)h->B);
    REQUIRE(ctx, ldo >= n, "small_hist_diag: leading dimension ldo = %lld must be at least n = %lld", (long long)ldo, (long long)n);
    REQUIRE(ctx, ctx->nranks == 1, "small_hist_diag: one CTA holds a whole problem, so n cannot be sharded (the context has %d ranks)", ctx->nranks);
    SmallDiagArgs<T> a{};
    a.hist = static_cast<const T*>(h->data); a.hist_c = h->counts; a.HL = SmallHistLayout{n, h->m};
    a.b0 = b0; a.inverse = inverse ? 1 : 0; a.OUT = OUT; a.ldo = ldo;
    const size_t smem = small_diag_smem(h->m, (int)sizeof(T));
    CU(ctx, cudaFuncSetAttribute(k_small_hist_diag<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_small_hist_diag<T><<<(unsigned)count, small_threads(n), smem, ctx->stream>>>(a);
    CU(ctx, cudaGetLastError());
    ctx->launches++;
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status small_hist_factor(lbfgs_b200_small_hist* h, bool gen, uint64_t seed, uint32_t first, int64_t b0, int64_t count, int k,
                                    const T* V, int64_t ldv, int64_t ldvp, T* OUT, int64_t ldo, int64_t ldop, int op = LBFGS_B200_FACTOR_L,
                                    const char* what = nullptr)
{
    using namespace lb;
    if (!what) what = gen ? "small_hist_sample" : "small_hist_factor_times";
    if (auto st = small_hist_check<T>(h, what)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, op >= LBFGS_B200_FACTOR_L && op <= LBFGS_B200_FACTOR_LINVT, "%s: op %d is not one of LBFGS_B200_FACTOR_*", what, op);
    const int64_t n = h->n;
    REQUIRE(ctx, OUT && (gen || V), "%s: NULL argument", what);
    REQUIRE(ctx, k >= 1 && (k + kSGroup - 1) / kSGroup <= 65535, "%s: k must be in 1..%d (got %d)", what, 65535 * kSGroup, k);
    REQUIRE(ctx, !gen || (uint64_t)first + (uint64_t)k <= 0x100000000ull, "%s: draws %u + %d run past 2^32", what, first, k);
    REQUIRE(ctx, b0 >= 0 && count >= 1 && count <= h->B - b0, "%s: problems [%lld, %lld) are not within the %lld of the history", what,
            (long long)b0, (long long)(b0 + count), (long long)h->B);
    REQUIRE(ctx, (gen || ldv >= n) && ldo >= n, "%s: leading dimensions ldv = %lld, ldo = %lld must be at least n = %lld", what,
            (long long)ldv, (long long)ldo, (long long)n);
    REQUIRE(ctx, ldvp >= 0 && ldop >= 0, "%s: negative problem stride", what);
    REQUIRE(ctx, gen || (const void*)V != (const void*)OUT || (ldo == ldv && ldop == ldvp && (ldvp > 0 || count == 1)),
            "%s: OUT may be V only with the same layout (ldo == ldv, ldop == ldvp) and vectors of its own per problem", what);
    // the sampler writes its draws into OUT and reads them back: problems' output ranges must not overlap, nor may MEAN lie in OUT
    REQUIRE(ctx, !gen || count == 1 || ldop >= (int64_t)k * ldo, "%s: problems' draws overlap (ldop = %lld < k * ldo = %lld)", what,
            (long long)ldop, (long long)k * ldo);
    if (gen && V)
    {
        const T* out_end = OUT + (count - 1) * ldop + (int64_t)(k - 1) * ldo + n;
        const T* mean_end = V + (count - 1) * ldvp + n;
        REQUIRE(ctx, mean_end <= OUT || out_end <= V, "%s: MEAN overlaps OUT", what);
    }
    REQUIRE(ctx, ctx->nranks == 1, "%s: one CTA holds a whole problem, so n cannot be sharded (the context has %d ranks)", what, ctx->nranks);
    SmallFactorArgs<T> a{};
    a.hist = static_cast<const T*>(h->data); a.hist_c = h->counts; a.HL = SmallHistLayout{n, h->m};
    a.b0 = b0; a.k = k; a.V = V; a.ldv = ldv; a.ldvp = ldvp; a.OUT = OUT; a.ldo = ldo; a.ldop = ldop; a.seed = seed; a.first = first;
    const size_t smem = small_factor_smem(h->m, (int)sizeof(T));
    auto kernel = gen ? k_small_hist_factor<T, true>
                : op == LBFGS_B200_FACTOR_LT    ? k_small_hist_factor<T, false, LBFGS_B200_FACTOR_LT>
                : op == LBFGS_B200_FACTOR_LINV  ? k_small_hist_factor<T, false, LBFGS_B200_FACTOR_LINV>
                : op == LBFGS_B200_FACTOR_LINVT ? k_small_hist_factor<T, false, LBFGS_B200_FACTOR_LINVT>
                                                : k_small_hist_factor<T, false>;
    CU(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<dim3((unsigned)count, (unsigned)((k + kSGroup - 1) / kSGroup)), small_threads(n), smem, ctx->stream>>>(a);
    CU(ctx, cudaGetLastError());
    ctx->launches++;
    return LBFGS_B200_OK;
}

template <class T> lbfgs_b200_status small_hist_logdet(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, double* out_host)
{
    using namespace lb;
    if (auto st = small_hist_check<T>(h, "small_hist_logdet")) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    REQUIRE(ctx, out_host, "small_hist_logdet: NULL argument");
    REQUIRE(ctx, b0 >= 0 && count >= 1 && count <= h->B - b0, "small_hist_logdet: problems [%lld, %lld) are not within the %lld of the history",
            (long long)b0, (long long)(b0 + count), (long long)h->B);
    REQUIRE(ctx, ctx->nranks == 1, "small_hist_logdet: a context with %d ranks", ctx->nranks);
    double* d = nullptr;
    cudaError_t e = pool_alloc(ctx, reinterpret_cast<void**>(&d), sizeof(double) * (size_t)count);
    if (e != cudaSuccess)
        return fail(ctx, e == cudaErrorMemoryAllocation ? LBFGS_B200_ERR_ALLOC : LBFGS_B200_ERR_CUDA, "small_hist_logdet: %s", cudaGetErrorString(e));
    const size_t smem = sizeof(double) * 3 * (size_t)h->m * h->m;
    e = cudaFuncSetAttribute(k_small_hist_logdet<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess)
    {
        k_small_hist_logdet<T><<<(unsigned)count, 32, smem, ctx->stream>>>(static_cast<const T*>(h->data), h->counts, SmallHistLayout{h->n, h->m}, b0, d);
        e = cudaGetLastError();
        ctx->launches++;
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_host, d, sizeof(double) * (size_t)count, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    pool_free(ctx, d);
    CU(ctx, e);
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status small_hist_log_density(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, int k, const T* X, int64_t ldx, int64_t ldxp,
                                         const T* MEAN, int64_t ldm, double* out_host)
{
    using namespace lb;
    const char* what = "small_hist_log_density";
    if (auto st = small_hist_check<T>(h, what)) return st;
    lbfgs_b200_ctx* ctx = h->ctx;
    const int64_t n = h->n;
    REQUIRE(ctx, X && MEAN && out_host, "%s: NULL argument", what);
    REQUIRE(ctx, k >= 1 && (k + kSGroup - 1) / kSGroup <= 65535, "%s: k must be in 1..%d (got %d)", what, 65535 * kSGroup, k);
    REQUIRE(ctx, b0 >= 0 && count >= 1 && count <= h->B - b0, "%s: problems [%lld, %lld) are not within the %lld of the history", what,
            (long long)b0, (long long)(b0 + count), (long long)h->B);
    REQUIRE(ctx, ldx >= n, "%s: leading dimension ldx = %lld must be at least n = %lld", what, (long long)ldx, (long long)n);
    REQUIRE(ctx, ldxp >= 0 && ldm >= 0, "%s: negative problem stride", what);
    REQUIRE(ctx, ctx->nranks == 1, "%s: one CTA holds a whole problem, so n cannot be sharded (the context has %d ranks)", what, ctx->nranks);
    double* d = nullptr;
    const size_t nout = (size_t)count * (size_t)k;
    cudaError_t e = pool_alloc(ctx, reinterpret_cast<void**>(&d), sizeof(double) * nout);
    if (e != cudaSuccess)
        return fail(ctx, e == cudaErrorMemoryAllocation ? LBFGS_B200_ERR_ALLOC : LBFGS_B200_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
    SmallDensityArgs<T> a{};
    a.hist = static_cast<const T*>(h->data); a.hist_c = h->counts; a.HL = SmallHistLayout{n, h->m};
    a.b0 = b0; a.k = k; a.X = X; a.ldx = ldx; a.ldxp = ldxp; a.MEAN = MEAN; a.ldm = ldm; a.out = d;
    const size_t smem = small_density_smem(h->m);
    e = cudaFuncSetAttribute(k_small_hist_log_density<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess)
    {
        k_small_hist_log_density<T><<<dim3((unsigned)count, (unsigned)((k + kSGroup - 1) / kSGroup)), small_threads(n), smem, ctx->stream>>>(a);
        e = cudaGetLastError();
        ctx->launches++;
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out_host, d, sizeof(double) * nout, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    pool_free(ctx, d);
    CU(ctx, e);
    return LBFGS_B200_OK;
}

}  // namespace

extern "C" {

int64_t lbfgs_b200_small_max_n(int m, int elem_bytes, int objective)
{
    bool stored = false;
    int data_vectors = 0;
    if (m < 1 || m > lb::kMaxM || (elem_bytes != 8 && elem_bytes != 4) || !small_objective_shape(objective, stored, data_vectors)) return 0;
    const lb::SmallLayout L = lb::small_layout(0, m, elem_bytes, stored, data_vectors);
    if (L.vecs >= lb::kSSmemLimit) return 0;
    const int64_t per_coord = (int64_t)elem_bytes * L.nvec;               // every vector holds round_up(n, 4) elements
    return (((int64_t)(lb::kSSmemLimit - L.vecs) / per_coord) / 4) * 4;
}

lbfgs_b200_status lbfgs_b200_small_hist_create(lbfgs_b200_ctx* ctx, int64_t n, int m, int elem_bytes, int64_t B, lbfgs_b200_small_hist** out)
{
    if (!ctx) return LBFGS_B200_ERR_INVALID;
    REQUIRE(ctx, out, "small_hist_create: NULL argument");
    *out = nullptr;
    REQUIRE(ctx, n >= 1 && m >= 1 && m <= lb::kMaxM && (elem_bytes == 8 || elem_bytes == 4) && B >= 1 && B <= 0x7fffffff,
            "small_hist_create: need n >= 1, 1 <= m <= %d, elem_bytes 8 or 4 and 1 <= B <= 2^31 - 1", lb::kMaxM);
    REQUIRE(ctx, lb::small_times_smem(m, elem_bytes) <= lb::kSSmemLimit, "small_hist_create: m = %d is too large for the products", m);
    auto* h = new lbfgs_b200_small_hist();
    h->ctx = ctx; h->n = n; h->m = m; h->elem = elem_bytes; h->B = B;
    const lb::SmallHistLayout HL{n, m};
    cudaError_t e = pool_alloc(ctx, &h->data, (size_t)elem_bytes * (size_t)HL.rec() * (size_t)B);
    if (e == cudaSuccess) e = pool_alloc(ctx, reinterpret_cast<void**>(&h->counts), sizeof(int) * (size_t)B);
    if (e != cudaSuccess)
    {
        lbfgs_b200_small_hist_destroy(h);
        cudaGetLastError();
        return fail(ctx, e == cudaErrorMemoryAllocation ? LBFGS_B200_ERR_ALLOC : LBFGS_B200_ERR_CUDA, "small_hist_create: %s", cudaGetErrorString(e));
    }
    *out = h;
    return LBFGS_B200_OK;
}

void lbfgs_b200_small_hist_destroy(lbfgs_b200_small_hist* h)
{
    if (!h) return;
    pool_free(h->ctx, h->data);
    pool_free(h->ctx, h->counts);
    delete h;
}

static const void* small_hist_col(const lbfgs_b200_small_hist* h, int64_t b, int age, bool y)
{
    if (!h || b < 0 || b >= h->B || age < 0 || age >= h->m) return nullptr;
    const lb::SmallHistLayout HL{h->n, h->m};
    return static_cast<const char*>(h->data) + (size_t)h->elem * (size_t)(b * HL.rec() + (y ? HL.y(age) : HL.s(age)));
}
const void* lbfgs_b200_small_hist_s_col(const lbfgs_b200_small_hist* h, int64_t b, int age) { return small_hist_col(h, b, age, false); }
const void* lbfgs_b200_small_hist_y_col(const lbfgs_b200_small_hist* h, int64_t b, int age) { return small_hist_col(h, b, age, true); }

#define LBFGS_B200_SMALL_KEEP(T, SUF)                                                                                              \
    lbfgs_b200_status lbfgs_b200_small_minimize_keep_##SUF(lbfgs_b200_ctx* ctx, int objective, const T* data0, const T* data1,     \
                                                           int64_t ldd, int64_t n, int64_t B, const lbfgs_b200_param* prm,          \
                                                           int line_search, T* X, int64_t ldx, T* G, lbfgs_b200_outcome* outs_host, \
                                                           lbfgs_b200_small_hist* hist)                                           \
    {                                                                                                                              \
        if (ctx) REQUIRE(ctx, hist, "small_minimize_keep: NULL history");                                                           \
        return small_minimize<T>(ctx, objective, data0, data1, ldd, n, B, prm, line_search, X, ldx, G, outs_host, hist);          \
    }                                                                                                                              \
    lbfgs_b200_status lbfgs_b200_small_hist_info_##SUF(lbfgs_b200_small_hist* h, int* c_host, T* theta_host)                       \
    { return small_hist_info<T>(h, c_host, theta_host); }                                                                         \
    lbfgs_b200_status lbfgs_b200_small_hist_times_##SUF(lbfgs_b200_small_hist* h, int inverse, int64_t b0, int64_t count, int k,   \
                                                        const T* V, int64_t ldv, int64_t ldvp, T* OUT, int64_t ldo, int64_t ldop)  \
    { return small_hist_times<T>(h, inverse, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop); }                                      \
    lbfgs_b200_status lbfgs_b200_small_hist_diag_##SUF(lbfgs_b200_small_hist* h, int inverse, int64_t b0, int64_t count, T* OUT,    \
                                                       int64_t ldo)                                                                \
    { return small_hist_diag<T>(h, inverse, b0, count, OUT, ldo); }                                                            \
    lbfgs_b200_status lbfgs_b200_small_hist_factor_times_##SUF(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, int k,         \
                                                               const T* V, int64_t ldv, int64_t ldvp, T* OUT, int64_t ldo,       \
                                                               int64_t ldop)                                                     \
    { return small_hist_factor<T>(h, false, 0, 0, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop); }                                  \
    lbfgs_b200_status lbfgs_b200_small_hist_sample_##SUF(lbfgs_b200_small_hist* h, uint64_t seed, uint32_t first, int64_t b0,       \
                                                         int64_t count, int k, const T* MEAN, int64_t ldm, T* OUT, int64_t ldo,  \
                                                         int64_t ldop)                                                           \
    { return small_hist_factor<T>(h, true, seed, first, b0, count, k, MEAN, 0, ldm, OUT, ldo, ldop); }                            \
    lbfgs_b200_status lbfgs_b200_small_hist_logdet_##SUF(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, double* out_host)    \
    { return small_hist_logdet<T>(h, b0, count, out_host); }                                                                \
    lbfgs_b200_status lbfgs_b200_small_hist_factor_apply_##SUF(lbfgs_b200_small_hist* h, int op, int64_t b0, int64_t count, int k, \
                                                               const T* V, int64_t ldv, int64_t ldvp, T* OUT, int64_t ldo,       \
                                                               int64_t ldop)                                                     \
    { return small_hist_factor<T>(h, false, 0, 0, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop, op, "small_hist_factor_apply"); }  \
    lbfgs_b200_status lbfgs_b200_small_hist_log_density_##SUF(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, int k,          \
                                                               const T* X, int64_t ldx, int64_t ldxp, const T* MEAN, int64_t ldm, \
                                                               double* out_host)                                                 \
    { return small_hist_log_density<T>(h, b0, count, k, X, ldx, ldxp, MEAN, ldm, out_host); }

LBFGS_B200_SMALL_KEEP(double, f64)
LBFGS_B200_SMALL_KEEP(float, f32)

lbfgs_b200_status lbfgs_b200_small_minimize_f64(lbfgs_b200_ctx* ctx, int objective, const double* data0, const double* data1, int64_t ldd,
                                                int64_t n, int64_t B, const lbfgs_b200_param* prm, int line_search, double* X, int64_t ldx,
                                                double* G, lbfgs_b200_outcome* outs_host)
{
    return small_minimize<double>(ctx, objective, data0, data1, ldd, n, B, prm, line_search, X, ldx, G, outs_host);
}

lbfgs_b200_status lbfgs_b200_small_minimize_f32(lbfgs_b200_ctx* ctx, int objective, const float* data0, const float* data1, int64_t ldd,
                                                int64_t n, int64_t B, const lbfgs_b200_param* prm, int line_search, float* X, int64_t ldx,
                                                float* G, lbfgs_b200_outcome* outs_host)
{
    return small_minimize<float>(ctx, objective, data0, data1, ldd, n, B, prm, line_search, X, ldx, G, outs_host);
}

}  // extern "C"
