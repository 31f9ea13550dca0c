// small_batch.cu -- the small-batch solve (small_batch.cuh): fp64 / fp32 instantiations, the shared-memory budget and the C ABI.
#include "internal.cuh"
#include "two_loop_gram.cuh"
#include "small_batch.cuh"

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
                                 const lbfgs_b200_param* prm, int ls_kind, T* X, int64_t ldx, T* G, lbfgs_b200_outcome* outs_host)
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
