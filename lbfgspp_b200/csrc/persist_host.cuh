// persist_host.cuh -- host side of the device-resident solve (persist.cuh): solver handle, state upload, ONE cooperative launch per
// minimize() (single problem or batch), C ABI.  Included at the end of lbfgs_b200.cu.
#pragma once

struct lbfgs_b200_solver
{
    lbfgs_b200_ctx* ctx = nullptr;
    int64_t n = 0;
    int m = 0, elem = 8, B = 1;
    // the rings, tiled: H[problem][block][slot][S|Y][BT] (lb::PHist) -- or, for objectives without neighbour coupling,
    // H[problem][block][point][BT] with 2M points; small per-problem arrays in one slab each
    void* d_hist = nullptr;
    int bt_log = 9, M = 0;
    size_t hist_elems = 0;                // elements of one problem's tiled ring
    void* d_small = nullptr;              // [B][ ys M | alpha M | theta 1 (padded to 4) | SY,YY,SS x2: 6 M^2 ]
    size_t small_elems = 0;
    unsigned char* d_pts = nullptr;       // [B][2M]: start and end point of the pair in each slot (lb::PState::pts)
    std::vector<int> ring_head, ring_ncorr, ring_gram_cur;   // ring state after the last solve (for the export below)
    // how the last solve's rings hold their pairs: as points (then the export rebuilds S, Y with the objective's gradient) or as S|Y
    bool ring_points = false;
    int ring_objective = -1;
    int64_t ring_gofs = 0, ring_nglob = 0;
    std::vector<unsigned char> ring_pts;  // host copy of d_pts after the last solve
    std::vector<lbfgs_b200_hist*> exported;                   // column-major copies made on request (lbfgs_b200_solver_history_of)
    std::vector<char> export_fresh;
    void* vec_slab = nullptr;             // [B][5][vec_elems] : x, xp, g, gp, drt
    void* lo_slab = nullptr;              // [B][2][vec_elems] : x_lo, g_lo (made on the first solve of a neighbour-coupled objective)
    size_t vec_elems = 0;                 // n rounded up to a whole number of 256-byte lines
    void* d_state = nullptr;              // PState<T>[B]
    void* d_rounds = nullptr;             // PRound<T>[B]
    lb::PCtl* d_ctl = nullptr;
    double* d_partials = nullptr;         // [B][pstride][sm_count]
    double* d_raw = nullptr;              // [B][pstride]
    double* d_halo = nullptr;             // [B][kHaloDoubles]
    int pstride = 0;
    double* d_trace = nullptr;
    long long trace_cap = 0;
    std::vector<void*> final_g, final_x;  // device pointers of each problem's final gradient / point (inside vec_slab)
    std::vector<unsigned char> h_state;   // host copy of the states
    std::vector<unsigned char> h_rounds;  // host image of the initial round descriptors
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    float last_kernel_ms = 0.f;           // device time of the last solve's kernel (CUDA events around the launch)
    lb::PCtl last_ctl{};                  // its accounting
};

template <class T, class OBJ> static void* persist_kernel_for(int rounds)
{
    using lb::k_persist;
    return rounds <= 1 ? (void*)k_persist<T, OBJ, 1> : rounds == 2 ? (void*)k_persist<T, OBJ, 2> : (void*)k_persist<T, OBJ, 3>;
}

// x_inout: B vectors of n elements, `ldx` elements apart (device).  data0/data1: nullptr, or per-problem vectors `ldd` apart (ldd = 0:
// every problem shares the same data).  outs: B outcomes.  trace_host: only with B == 1.
template <class T>
static lbfgs_b200_status solver_minimize(lbfgs_b200_solver* s, int objective, const T* data0, const T* data1, int64_t ldd, const lbfgs_b200_param* prm,
                                         int ls_kind, T* x_inout, int64_t ldx, double* trace_host, long long trace_cap, lbfgs_b200_outcome* outs)
{
    using namespace lb;
    lbfgs_b200_ctx* ctx = s->ctx;
    const int B = s->B;
    REQUIRE(ctx, s->elem == (int)sizeof(T), "solver element size mismatch");
    REQUIRE(ctx, prm && outs && x_inout, "solver_minimize: NULL argument");
    REQUIRE(ctx, prm->m == s->m, "solver was created for m = %d, called with m = %d", s->m, prm->m);
    REQUIRE(ctx, ls_kind >= 0 && ls_kind <= 3, "unknown line search %d", ls_kind);
    REQUIRE(ctx, prm->past <= kMaxPast, "past > %d is not supported by the device-resident solve", kMaxPast);
    REQUIRE(ctx, ctx->nranks == 1 || ctx->x_active, "the device-resident solve needs the in-kernel exchange (comm_p2p) when sharded");
    REQUIRE(ctx, B == 1 || ldx >= s->n, "solver_minimize: the batch stride of x is shorter than n");
    // the passes read a problem's data with bulk copies that start on 16-byte boundaries of data + b*ldd
    REQUIRE(ctx, ldd == 0 || ldd >= s->n, "solver_minimize: the batch stride of the data (%lld) must be 0 (shared) or at least n (%lld)",
            (long long)ldd, (long long)s->n);
    REQUIRE(ctx, ldd * (int64_t)sizeof(T) % 16 == 0, "solver_minimize: the batch stride of the data (%lld elements) must be a multiple of 16 bytes",
            (long long)ldd);
    REQUIRE(ctx, (uintptr_t)data0 % 16 == 0 && (uintptr_t)data1 % 16 == 0, "solver_minimize: the data vectors must start on a 16-byte boundary");
    REQUIRE(ctx, trace_host == nullptr || B == 1, "solver_minimize: traces are recorded for single problems only");
    if (ctx->x_active) REQUIRE(ctx, (size_t)B * (s->pstride + 4) <= (size_t)kXMaxVals, "batch of %d problems with m = %d exceeds the exchange buffer", B, s->m);
    const int rounds = (s->m + kGramMaxWarps - 1) / kGramMaxWarps;   // column pairs per round of the dots pass: at most one per warp
    ObjGeom<T> geo;
    void* kernel = nullptr;
    // the first trial of every search rides on the combination pass; a neighbour-coupled objective needs its neighbours' x + d,
    // which only exist on this rank when n is not sharded
    bool fuse_first_trial = true;
    bool stored_trials = false;   // the trials store their points and the search keeps its best one in (x_lo, g_lo)
    if (auto st = with_objective<T>(ctx, objective, [&](auto tag) {
            using OBJ = decltype(tag);
            kernel = persist_kernel_for<T, OBJ>(rounds);
            fuse_first_trial = !(OBJ::kHalo && ctx->nranks > 1);
            stored_trials = OBJ::kHalo;
            return objective_geometry<OBJ>(ctx, s->n, data0, data1, geo);
        }))
        return st;
    if (stored_trials && !s->lo_slab) CU(ctx, pool_alloc(ctx, &s->lo_slab, (size_t)B * 2 * s->vec_elems * sizeof(T)));

    if (trace_host && trace_cap > s->trace_cap)
    {
        pool_free(ctx, s->d_trace);
        s->d_trace = nullptr;
        CU(ctx, pool_alloc(ctx, (void**)&s->d_trace, sizeof(double) * (size_t)trace_cap));
        s->trace_cap = trace_cap;
    }

    // ---- states ----
    s->h_state.assign(sizeof(PState<T>) * (size_t)B, 0);
    PState<T>* hs = reinterpret_cast<PState<T>*>(s->h_state.data());
    const size_t vb = sizeof(T) * (size_t)s->n;
    for (int b = 0; b < B; b++)
    {
        PState<T>& p = hs[b];
        T* base = static_cast<T*>(s->vec_slab) + (size_t)b * 5 * s->vec_elems;
        p.x = base; p.xp = base + s->vec_elems; p.g = base + 2 * s->vec_elems; p.gp = base + 3 * s->vec_elems;
        p.drt = base + 4 * s->vec_elems;
        T* lo = stored_trials ? static_cast<T*>(s->lo_slab) + (size_t)b * 2 * s->vec_elems : nullptr;
        p.x_lo = lo; p.g_lo = lo ? lo + s->vec_elems : nullptr;
        p.hist.H = static_cast<T*>(s->d_hist) + (size_t)b * s->hist_elems;
        p.hist.bt_log = s->bt_log; p.hist.M = s->M; p.hist.bstride = (int64_t)s->M * 2 * ((int64_t)1 << s->bt_log);
        T* small = static_cast<T*>(s->d_small) + (size_t)b * s->small_elems;
        const size_t mm = (size_t)s->M * s->M;
        p.ys = small; p.alpha = small + s->M; p.theta = small + 2 * s->M;
        for (int k = 0; k < 2; k++) { p.SY[k] = small + 2 * s->M + 4 + (3 * k + 0) * mm; p.YY[k] = small + 2 * s->M + 4 + (3 * k + 1) * mm; p.SS[k] = small + 2 * s->M + 4 + (3 * k + 2) * mm; }
        p.data0 = data0 ? data0 + (size_t)b * ldd : nullptr;
        p.data1 = data1 ? data1 + (size_t)b * ldd : nullptr;
        p.raw = s->d_raw + (size_t)b * s->pstride;
        p.pts = s->d_pts + (size_t)b * 2 * s->M;
        p.halo = s->d_halo + (size_t)b * kHaloDoubles;
        init_problem_state<T>(p, *prm, ls_kind, fuse_first_trial);   // (prm->m == s->m: p.M == s->M)
        p.trace = trace_host ? s->d_trace : nullptr;
        p.trace_cap = trace_host ? trace_cap : 0;
        CU(ctx, cudaMemcpyAsync(p.x, x_inout + (size_t)b * ldx, vb, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    s->h_rounds.assign(sizeof(PRound<T>) * (size_t)B, 0);
    PRound<T>* hr = reinterpret_cast<PRound<T>*>(s->h_rounds.data());
    for (int b = 0; b < B; b++)
    {
        const PState<T>& p = hs[b];
        hr[b].x = p.x; hr[b].xp = p.xp; hr[b].g = p.g; hr[b].gp = p.gp; hr[b].drt = p.drt;
        hr[b].step = T(0); hr[b].op = p.op; hr[b].c_round = 0; hr[b].head = 0; hr[b].pending = -1; hr[b].gram_cur = p.gram_cur;
        hr[b].px = p.px; hr[b].pxp = p.pxp;
    }
    // BFGSMat::reset (BFGSMat.h:61-78): no pairs, theta = 1, Gram matrices cleared
    CU(ctx, cudaMemsetAsync(s->d_small, 0, sizeof(T) * s->small_elems * (size_t)B, ctx->stream));
    {
        static const T one = T(1);
        for (int b = 0; b < B; b++) CU(ctx, cudaMemcpyAsync(hs[b].theta, &one, sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    }
    CU(ctx, cudaMemcpyAsync(s->d_state, hs, sizeof(PState<T>) * (size_t)B, cudaMemcpyHostToDevice, ctx->stream));
    CU(ctx, cudaMemcpyAsync(s->d_rounds, hr, sizeof(PRound<T>) * (size_t)B, cudaMemcpyHostToDevice, ctx->stream));
    PCtl hc{};
    hc.nactive = B;
    hc.epoch = ctx->x_epoch;
    CU(ctx, cudaMemcpyAsync(s->d_ctl, &hc, sizeof(hc), cudaMemcpyHostToDevice, ctx->stream));
    CU(ctx, cudaMemsetAsync(s->d_halo, 0, sizeof(double) * kHaloDoubles * (size_t)B, ctx->stream));

    // ---- one cooperative launch: one CTA per SM (fewer when the vector has fewer tiles than SMs) ----
    const int64_t units = (s->n + ((int64_t)1 << s->bt_log) - 1) >> s->bt_log;
    const int grid = (int)(units < ctx->sm_count ? (units < 1 ? 1 : units) : ctx->sm_count);
    const size_t smem = (size_t)kPStageBytes;
    CU(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    CU(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kPThreads, smem));
    REQUIRE(ctx, per_sm >= 1, "the persistent solve kernel does not fit on an SM of this device");
    PArgs<T> a{};
    a.probs = static_cast<PState<T>*>(s->d_state); a.rounds = static_cast<PRound<T>*>(s->d_rounds); a.B = B; a.ctl = s->d_ctl; a.partials = s->d_partials; a.pstride = s->pstride;
    a.n = s->n; a.grain = 1 << s->bt_log; a.xc = ctx->x_active ? ctx->x_comm : nullptr;
    a.index_offset = geo.gofs; a.n_global = geo.n_glob;
    a.wait_cycles = kPWaitCycles;
    if (const char* e = getenv("LBFGS_B200_WATCHDOG_SCALE")) { const long long k = atoll(e); if (k >= 1 && k <= 100000) a.wait_cycles *= k; }
    a.evict_first_stores = (size_t)s->n * sizeof(T) * 4 > ((size_t)36 << 20);     // x, xp, g, d of one problem exceed ~3/4 of the 50 MB L2
    void* kargs[] = {&a};
    CU(ctx, cudaEventRecord(s->ev0, ctx->stream));
    CU(ctx, cudaLaunchCooperativeKernel(kernel, dim3((unsigned)grid), dim3(kPThreads), kargs, smem, ctx->stream));
    CU(ctx, cudaEventRecord(s->ev1, ctx->stream));
    ctx->launches++;
    CU(ctx, cudaMemcpyAsync(hs, s->d_state, sizeof(PState<T>) * (size_t)B, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaMemcpyAsync(&hc, s->d_ctl, sizeof(hc), cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->x_epoch = hc.epoch;
    s->last_ctl = hc;
    CU(ctx, cudaEventElapsedTime(&s->last_kernel_ms, s->ev0, s->ev1));
    if (hc.abort) return fail(ctx, LBFGS_B200_ERR_CUDA, "the persistent solve gave up waiting at a grid / cross-rank barrier after %llu rounds (watchdog)", hc.rounds);

    // the states tell where the results live after all the pointer rotations
    for (int b = 0; b < B; b++)
    {
        const PState<T>& p = hs[b];
        CU(ctx, cudaMemcpyAsync(x_inout + (size_t)b * ldx, p.x, vb, cudaMemcpyDeviceToDevice, ctx->stream));
        s->final_g[b] = p.g;
        s->final_x[b] = p.x;
        s->ring_head[b] = p.head; s->ring_ncorr[b] = p.ncorr; s->ring_gram_cur[b] = p.gram_cur;
        s->export_fresh[b] = 0;
        outs[b].status = p.status;
        outs[b].niter = p.niter;
        outs[b].nfev = p.nfev;
        outs[b].fx = (double)p.rec.fx;
        outs[b].gnorm = (double)p.gnorm;
        outs[b].rounds = p.rounds;
    }
    s->ring_points = !stored_trials;
    s->ring_objective = objective;
    s->ring_gofs = geo.gofs; s->ring_nglob = geo.n_glob;
    if (s->ring_points) CU(ctx, cudaMemcpyAsync(s->ring_pts.data(), s->d_pts, s->ring_pts.size(), cudaMemcpyDeviceToHost, ctx->stream));
    if (trace_host)
    {
        const long long cnt = hs[0].nfev < trace_cap ? hs[0].nfev : trace_cap;
        CU(ctx, cudaMemcpyAsync(trace_host, s->d_trace, sizeof(double) * (size_t)cnt, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CU(ctx, cudaStreamSynchronize(ctx->stream));
    return LBFGS_B200_OK;
}

// The ring of problem b as an ordinary (column-major) lbfgs_b200_hist, for final_approx_hessian() and inspection: made on request,
// refreshed after every solve.  nullptr on failure (the context holds the message).
template <class T> __global__ void k_untile_history(lb::PHist<T> h, int64_t n, int64_t ld, T* __restrict__ S, T* __restrict__ Y)
{
    const int slot = blockIdx.y;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    {
        S[(int64_t)slot * ld + i] = *h.s_at(slot, i);
        Y[(int64_t)slot * ld + i] = *h.y_at(slot, i);
    }
}
// ... of a ring of points: pair slot `slot` from its endpoints (ends[2 slot], ends[2 slot + 1]; -1: no live pair, zeros), with the
// arithmetic of the passes that read it, 16-byte unit by 16-byte unit: bit for bit the s and y the solve used
struct PairEnds { short v[2 * (lb::kMaxM + 1)]; };
template <class T, class OBJ> __global__ void k_untile_points(lb::PHist<T> h, OBJ obj, PairEnds ends, int64_t n, int64_t ld, T* __restrict__ S, T* __restrict__ Y)
{
    constexpr int EPT = 16 / (int)sizeof(T);
    const int slot = blockIdx.y;
    const int ps = ends.v[2 * slot], pe = ends.v[2 * slot + 1];
    for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * EPT; i0 < n; i0 += (int64_t)gridDim.x * blockDim.x * EPT)
    {
        const int cnt = n - i0 >= EPT ? EPT : (int)(n - i0);
        lb::Unit<T> us, uy;
        if (ps >= 0)
        {
            const lb::Unit<T> ua = lb::lds_unit<T>(h.pt_at(ps, i0)), ub = lb::lds_unit<T>(h.pt_at(pe, i0));
            const lb::Unit<T> ga = lb::grad_unit(obj, i0, cnt, ua), gb = lb::grad_unit(obj, i0, cnt, ub);
#pragma unroll
            for (int k = 0; k < EPT; k++) { us.v[k] = ub.v[k] - ua.v[k]; uy.v[k] = gb.v[k] - ga.v[k]; }
        }
        else
            for (int k = 0; k < EPT; k++) us.v[k] = uy.v[k] = T(0);
        for (int k = 0; k < cnt; k++)
        {
            S[(int64_t)slot * ld + i0 + k] = us.v[k];
            Y[(int64_t)slot * ld + i0 + k] = uy.v[k];
        }
    }
}
#if defined(LBFGS_B200_PERSIST_F64)
template <class T> static lbfgs_b200_hist* export_history(lbfgs_b200_solver* s, int b)
{
    lbfgs_b200_ctx* ctx = s->ctx;
    lbfgs_b200_hist*& h = s->exported[(size_t)b];
    if (h && s->export_fresh[(size_t)b]) return h;
    if (!h && lbfgs_b200_hist_create(ctx, &h, s->n, s->m, s->elem) != LBFGS_B200_OK) return nullptr;
    lb::PHist<T> ph;
    ph.H = static_cast<T*>(s->d_hist) + (size_t)b * s->hist_elems;
    ph.bt_log = s->bt_log; ph.M = s->M; ph.bstride = (int64_t)s->M * 2 * ((int64_t)1 << s->bt_log);
    const dim3 grid((unsigned)std::min<int64_t>((s->n + 255) / 256, 4 * ctx->sm_count), (unsigned)s->M);
    if (s->ring_points)
    {
        // the live pairs: ages 0 .. ncorr-1 below head
        PairEnds ends;
        for (int k = 0; k < 2 * s->M; k++) ends.v[k] = -1;
        const unsigned char* pts = s->ring_pts.data() + (size_t)b * 2 * s->M;
        for (int age = 0; age < s->ring_ncorr[(size_t)b]; age++)
        {
            const int slot = lb::slot_by_age(s->ring_head[(size_t)b], s->M, age);
            ends.v[2 * slot] = pts[2 * slot];
            ends.v[2 * slot + 1] = pts[2 * slot + 1];
        }
        const lb::ObjGeom<T> geo{s->n, s->ring_gofs, s->ring_nglob, nullptr, nullptr, nullptr};
        if (with_objective<T>(ctx, s->ring_objective, [&](auto tag) {
                using OBJ = decltype(tag);
                if constexpr (!OBJ::kHalo)
                    k_untile_points<T, OBJ><<<grid, 256, 0, ctx->stream>>>(ph, OBJ{geo}, ends, s->n, h->ld, static_cast<T*>(h->S), static_cast<T*>(h->Y));
                return LBFGS_B200_OK;
            }) != LBFGS_B200_OK)
            return nullptr;
    }
    else k_untile_history<T><<<grid, 256, 0, ctx->stream>>>(ph, s->n, h->ld, static_cast<T*>(h->S), static_cast<T*>(h->Y));
    const T* small = static_cast<const T*>(s->d_small) + (size_t)b * s->small_elems;
    const size_t mm = (size_t)s->M * s->M;
    cudaMemcpyAsync(h->ys, small, sizeof(T) * s->M, cudaMemcpyDeviceToDevice, ctx->stream);
    cudaMemcpyAsync(h->alpha, small + s->M, sizeof(T) * s->M, cudaMemcpyDeviceToDevice, ctx->stream);
    cudaMemcpyAsync(h->theta, small + 2 * s->M, sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream);
    for (int k = 0; k < 2; k++)
    {
        cudaMemcpyAsync(h->SY[k], small + 2 * s->M + 4 + (3 * k + 0) * mm, sizeof(T) * mm, cudaMemcpyDeviceToDevice, ctx->stream);
        cudaMemcpyAsync(h->YY[k], small + 2 * s->M + 4 + (3 * k + 1) * mm, sizeof(T) * mm, cudaMemcpyDeviceToDevice, ctx->stream);
        cudaMemcpyAsync(h->SS[k], small + 2 * s->M + 4 + (3 * k + 2) * mm, sizeof(T) * mm, cudaMemcpyDeviceToDevice, ctx->stream);
    }
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess || cudaGetLastError() != cudaSuccess) { fail(ctx, LBFGS_B200_ERR_CUDA, "exporting the solver's history failed"); return nullptr; }
    h->head = s->ring_head[(size_t)b]; h->ncorr = s->ring_ncorr[(size_t)b]; h->gram_cur = s->ring_gram_cur[(size_t)b]; h->pending = -1;
    s->export_fresh[(size_t)b] = 1;
    return h;
}
#endif

extern "C" {

#ifdef LBFGS_B200_PERSIST_F64
lbfgs_b200_status lbfgs_b200_solver_create_batch(lbfgs_b200_ctx* ctx, int64_t n, int m, int elem_bytes, int batch, lbfgs_b200_solver** out)
{
    REQUIRE(ctx, ctx && out, "solver_create: NULL argument");
    *out = nullptr;
    REQUIRE(ctx, batch >= 1 && batch <= 4096, "solver_create: 1 <= batch <= 4096 (got %d)", batch);
    REQUIRE(ctx, n >= 1 && m >= 1 && m <= 64, "solver_create: need n >= 1 and 1 <= m <= 64 (got n=%lld m=%d)", (long long)n, m);
    REQUIRE(ctx, elem_bytes == 8 || elem_bytes == 4, "solver_create: elem_bytes must be 8 or 4");
    lbfgs_b200_solver* s = new (std::nothrow) lbfgs_b200_solver();
    if (!s) return fail(ctx, LBFGS_B200_ERR_ALLOC, "out of host memory");
    s->ctx = ctx; s->n = n; s->m = m; s->elem = elem_bytes; s->B = batch;
    s->final_g.assign((size_t)batch, nullptr);
    s->final_x.assign((size_t)batch, nullptr);
    s->M = m + 1;
    // block length of the tiled history: the largest power of two for which two stages of 2m+4 rows fit the kernel's staging ring
    {
        int bt = 1024;
        while (bt > 32 && (size_t)2 * (2 * m + 4) * bt * elem_bytes > (size_t)lb::kPStageBytes) bt >>= 1;
        s->bt_log = 0;
        while ((1 << s->bt_log) < bt) s->bt_log++;
    }
    const int64_t nblocks = (n + ((int64_t)1 << s->bt_log) - 1) >> s->bt_log;
    s->hist_elems = (size_t)nblocks * s->M * 2 * ((size_t)1 << s->bt_log);
    s->small_elems = (size_t)2 * s->M + 4 + 6 * (size_t)s->M * s->M;
    s->ring_head.assign((size_t)batch, 0); s->ring_ncorr.assign((size_t)batch, 0); s->ring_gram_cur.assign((size_t)batch, 0);
    s->ring_pts.assign((size_t)batch * 2 * s->M, 0);
    s->exported.assign((size_t)batch, nullptr); s->export_fresh.assign((size_t)batch, 0);
    cudaError_t e = cudaSuccess;
    s->vec_elems = (((size_t)n * elem_bytes + 255) & ~size_t(255)) / elem_bytes;
    s->pstride = ((m * lb::kGramVals > 8 ? m * lb::kGramVals : 8) + 7) & ~7;
    const size_t state_bytes = (elem_bytes == 8 ? sizeof(lb::PState<double>) : sizeof(lb::PState<float>)) * (size_t)batch;
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&s->vec_slab, (size_t)batch * 5 * s->vec_elems * elem_bytes);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&s->d_hist, (size_t)batch * s->hist_elems * elem_bytes);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&s->d_small, (size_t)batch * s->small_elems * elem_bytes);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&s->d_pts, (size_t)batch * 2 * s->M);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&s->d_state, state_bytes);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&s->d_rounds, (elem_bytes == 8 ? sizeof(lb::PRound<double>) : sizeof(lb::PRound<float>)) * (size_t)batch);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&s->d_ctl, sizeof(lb::PCtl));
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&s->d_partials, sizeof(double) * (size_t)batch * s->pstride * ctx->sm_count);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&s->d_raw, sizeof(double) * (size_t)batch * s->pstride);
    if (e == cudaSuccess) e = pool_alloc(ctx, (void**)&s->d_halo, sizeof(double) * (size_t)batch * lb::kHaloDoubles);
    if (e == cudaSuccess) e = cudaEventCreate(&s->ev0);
    if (e == cudaSuccess) e = cudaEventCreate(&s->ev1);
    if (e != cudaSuccess)
    {
        lbfgs_b200_solver_destroy(s);
        return fail(ctx, e == cudaErrorMemoryAllocation ? LBFGS_B200_ERR_ALLOC : LBFGS_B200_ERR_CUDA, "solver_create: %s", cudaGetErrorString(e));
    }
    *out = s;
    return LBFGS_B200_OK;
}

lbfgs_b200_status lbfgs_b200_solver_create(lbfgs_b200_ctx* ctx, int64_t n, int m, int elem_bytes, lbfgs_b200_solver** out)
{
    return lbfgs_b200_solver_create_batch(ctx, n, m, elem_bytes, 1, out);
}

void lbfgs_b200_solver_destroy(lbfgs_b200_solver* s)
{
    if (!s) return;
    if (s->ctx && s->ctx->stream) cudaStreamSynchronize(s->ctx->stream);   // the events below must not be in use
    for (void* p : {(void*)s->vec_slab, (void*)s->lo_slab, (void*)s->d_state, (void*)s->d_rounds, (void*)s->d_ctl, (void*)s->d_partials, (void*)s->d_raw, (void*)s->d_halo,
                    (void*)s->d_trace, (void*)s->d_hist, (void*)s->d_small, (void*)s->d_pts})
        pool_free(s->ctx, p);
    if (s->ev0) cudaEventDestroy(s->ev0);
    if (s->ev1) cudaEventDestroy(s->ev1);
    for (lbfgs_b200_hist* h : s->exported) lbfgs_b200_hist_destroy(h);
    delete s;
}

int lbfgs_b200_solver_batch(const lbfgs_b200_solver* s) { return s ? s->B : 0; }
lbfgs_b200_status lbfgs_b200_solver_profile(const lbfgs_b200_solver* s, double* kernel_ms, double* ms_by_op10, unsigned long long* rounds_by_op10,
                                            double* alg_bytes_by_op10, double* sync_ms)
{
    if (!s) return LBFGS_B200_ERR_INVALID;
    const lb::PCtl& c = s->last_ctl;
    long long total = 0;
    for (int k = 0; k < lb::kPOps; k++) total += c.cyc_op[k];
    const double scale = total > 0 ? (double)s->last_kernel_ms / (double)total : 0.0;   // CTA 0's cycles -> share of the event-timed kernel
    if (kernel_ms) *kernel_ms = s->last_kernel_ms;
    for (int k = 0; k < lb::kPOps; k++)
    {
        if (ms_by_op10) ms_by_op10[k] = scale * (double)c.cyc_op[k];
        if (rounds_by_op10) rounds_by_op10[k] = c.n_op[k];
        if (alg_bytes_by_op10) alg_bytes_by_op10[k] = c.words_op[k] * (double)s->n * (double)s->elem;
    }
    if (sync_ms) { sync_ms[0] = scale * (double)c.cyc_sync; sync_ms[1] = scale * (double)c.cyc_wait_all; sync_ms[2] = scale * (double)c.cyc_exchange; }
    return LBFGS_B200_OK;
}
const void* lbfgs_b200_solver_final_grad(const lbfgs_b200_solver* s) { return s ? s->final_g[0] : nullptr; }
const void* lbfgs_b200_solver_final_grad_of(const lbfgs_b200_solver* s, int b) { return (s && b >= 0 && b < s->B) ? s->final_g[(size_t)b] : nullptr; }
lbfgs_b200_hist* lbfgs_b200_solver_history_of(lbfgs_b200_solver* s, int b)
{
    if (!s || b < 0 || b >= s->B) return nullptr;
    if (s->elem == 8) return export_history<double>(s, b);
    return export_history<float>(s, b);
}
lbfgs_b200_hist* lbfgs_b200_solver_history(lbfgs_b200_solver* s) { return lbfgs_b200_solver_history_of(s, 0); }

lbfgs_b200_status lbfgs_b200_solver_minimize_f64(lbfgs_b200_solver* s, int objective, const double* data0, const double* data1,
                                                 const lbfgs_b200_param* prm, int line_search, double* x_inout, double* trace_host,
                                                 long long trace_cap, lbfgs_b200_outcome* out)
{
    if (!s || !s->ctx) return LBFGS_B200_ERR_INVALID;
    if (s->B != 1) return fail(s->ctx, LBFGS_B200_ERR_INVALID, "solver_minimize: the solver holds a batch of %d problems, use solver_minimize_batch", s->B);
    return solver_minimize<double>(s, objective, data0, data1, 0, prm, line_search, x_inout, s->n, trace_host, trace_cap, out);
}
lbfgs_b200_status lbfgs_b200_solver_minimize_batch_f64(lbfgs_b200_solver* s, int objective, const double* data0, const double* data1, int64_t ldd,
                                                       const lbfgs_b200_param* prm, int line_search, double* x_inout, int64_t ldx,
                                                       lbfgs_b200_outcome* outs)
{
    if (!s || !s->ctx) return LBFGS_B200_ERR_INVALID;
    return solver_minimize<double>(s, objective, data0, data1, ldd, prm, line_search, x_inout, ldx, nullptr, 0, outs);
}
#endif  // LBFGS_B200_PERSIST_F64

#ifdef LBFGS_B200_PERSIST_F32
lbfgs_b200_status lbfgs_b200_solver_minimize_f32(lbfgs_b200_solver* s, int objective, const float* data0, const float* data1,
                                                 const lbfgs_b200_param* prm, int line_search, float* x_inout, double* trace_host,
                                                 long long trace_cap, lbfgs_b200_outcome* out)
{
    if (!s || !s->ctx) return LBFGS_B200_ERR_INVALID;
    if (s->B != 1) return fail(s->ctx, LBFGS_B200_ERR_INVALID, "solver_minimize: the solver holds a batch of %d problems, use solver_minimize_batch", s->B);
    return solver_minimize<float>(s, objective, data0, data1, 0, prm, line_search, x_inout, s->n, trace_host, trace_cap, out);
}
lbfgs_b200_status lbfgs_b200_solver_minimize_batch_f32(lbfgs_b200_solver* s, int objective, const float* data0, const float* data1, int64_t ldd,
                                                       const lbfgs_b200_param* prm, int line_search, float* x_inout, int64_t ldx,
                                                       lbfgs_b200_outcome* outs)
{
    if (!s || !s->ctx) return LBFGS_B200_ERR_INVALID;
    return solver_minimize<float>(s, objective, data0, data1, ldd, prm, line_search, x_inout, ldx, nullptr, 0, outs);
}

#endif  // LBFGS_B200_PERSIST_F32

}  // extern "C"
