/* lbfgs_b200.h -- C ABI of liblbfgs_b200.so: the L-BFGS hot path of LBFGSpp on NVIDIA H100 (sm_90a).
 *
 * The reference (yixuan/LBFGSpp @ ebef584) has no FFI: its boundary is a C++ template API whose
 * floating-point work happens inside Eigen expressions.  This header is the contract between the
 * header-only C++ front in include/LBFGS.h (same class names / template parameters as the reference)
 * and the hand-written CUDA kernels.  Every entry point names the reference expression it replaces
 * (paths relative to the reference root).  Conventions:
 *   - plain C types only; device pointers are `void*`/typed pointers into memory obtained from
 *     lbfgs_b200_malloc (256-byte aligned) -- never host memory unless the name says `_host`;
 *   - every call returns a lbfgs_b200_status; no exception crosses the boundary; the text of the last
 *     failure is available from lbfgs_b200_last_error();
 *   - calls are stream-ordered on the context's stream; a call that returns scalars to the host
 *     (`*_host` out-parameters) synchronises the stream before returning, all others are asynchronous;
 *   - reductions are deterministic (fixed grid, fixed-order block partials, no floating-point atomics);
 *     with a communicator attached (n sharded over ranks) every reduction is summed over all ranks;
 *   - a context (and everything created from it) must be used by one host thread at a time;
 *   - there is NO CPU fallback: without a CUDA device every call fails with LBFGS_B200_ERR_CUDA.
 * `T` in {f64, f32} via the suffix.
 */
#ifndef LBFGS_B200_H
#define LBFGS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    LBFGS_B200_OK = 0,
    LBFGS_B200_ERR_INVALID = 1, /* bad argument (maps to std::invalid_argument in the C++ front) */
    LBFGS_B200_ERR_CUDA = 2,    /* CUDA runtime / driver failure, or no device (std::runtime_error) */
    LBFGS_B200_ERR_COMM = 3,    /* NCCL failure (std::runtime_error)                               */
    LBFGS_B200_ERR_ALLOC = 4    /* out of device memory (std::bad_alloc)                           */
} lbfgs_b200_status;

typedef struct lbfgs_b200_ctx lbfgs_b200_ctx;   /* device + stream + reduction scratch + communicator */
typedef struct lbfgs_b200_hist lbfgs_b200_hist; /* the S/Y ring of BFGSMat, resident in HBM           */

/* built-in device objective functions (the reference's example functors, SURVEY.md 8a row A12) */
enum {
    LBFGS_B200_OBJ_ROSENBROCK_PAIRED = 0,  /* examples/example-rosenbrock.cpp:15-27      */
    LBFGS_B200_OBJ_QUAD_SHIFT = 1,         /* examples/example-quadratic.cpp:9-19        */
    LBFGS_B200_OBJ_ROSENBROCK_CHAINED = 2, /* examples/example-rosenbrock-box.cpp:18-33  */
    LBFGS_B200_OBJ_QUAD_TRIDIAG = 3        /* f = 1/2 x'Ax - b'x, A = diag(d) + 1/2 tridiag(-1,2,-1); data0=d, data1=b */
};

/* apply_Hv algorithms */
enum {
    LBFGS_B200_HV_AUTO = 0,      /* currently GRAM                                                             */
    LBFGS_B200_HV_TWO_LOOP = 1,  /* literal two-loop recursion, one fused AXPY+dot stage kernel per history column:
                                    (8c+4) n words of traffic, 2c+1 launches, 2c collectives when sharded      */
    LBFGS_B200_HV_GRAM = 2       /* the same recursion carried out on 2c coefficients: two passes over S,Y,
                                    (4c+3) n words, 3 launches, 1 collective; differs from TWO_LOOP by rounding */
};

/* ---------------------------------------------------------------- context, memory, communicator */
const char* lbfgs_b200_version(void);
/* stream: a cudaStream_t to run on, or NULL to let the context create its own non-blocking stream. */
lbfgs_b200_status lbfgs_b200_ctx_create(lbfgs_b200_ctx** out, int device, void* stream);
void lbfgs_b200_ctx_destroy(lbfgs_b200_ctx* ctx);
const char* lbfgs_b200_last_error(const lbfgs_b200_ctx* ctx); /* ctx may be NULL: creation errors */
void* lbfgs_b200_stream(const lbfgs_b200_ctx* ctx);
int lbfgs_b200_sm_count(const lbfgs_b200_ctx* ctx);
uint64_t lbfgs_b200_launch_count(const lbfgs_b200_ctx* ctx); /* kernels launched so far by this context */

lbfgs_b200_status lbfgs_b200_malloc(lbfgs_b200_ctx* ctx, void** dptr, size_t bytes); /* replaces Eigen resize(): LBFGS.h:40-50 */
lbfgs_b200_status lbfgs_b200_free(lbfgs_b200_ctx* ctx, void* dptr);
/* Device blocks released by lbfgs_b200_free / *_destroy stay with the context and are handed out again (exact size match): the
 * reference reallocates its work vectors and history in every minimize() (LBFGS.h:84-90, BFGSMat.h:61-67), which on the GPU would
 * cost a cudaMalloc/cudaFree pair and a device-wide synchronisation each.  lbfgs_b200_trim returns the cached blocks to the driver
 * (lbfgs_b200_ctx_destroy does so as well). */
lbfgs_b200_status lbfgs_b200_trim(lbfgs_b200_ctx* ctx);
lbfgs_b200_status lbfgs_b200_malloc_host(lbfgs_b200_ctx* ctx, void** hptr, size_t bytes); /* pinned */
lbfgs_b200_status lbfgs_b200_free_host(lbfgs_b200_ctx* ctx, void* hptr);
lbfgs_b200_status lbfgs_b200_memcpy_h2d(lbfgs_b200_ctx* ctx, void* dst, const void* src_host, size_t bytes);
lbfgs_b200_status lbfgs_b200_memcpy_d2h(lbfgs_b200_ctx* ctx, void* dst_host, const void* src, size_t bytes); /* synchronises */
lbfgs_b200_status lbfgs_b200_memcpy_d2d(lbfgs_b200_ctx* ctx, void* dst, const void* src, size_t bytes);      /* `m_xp = x`, LBFGS.h:121-122 */
lbfgs_b200_status lbfgs_b200_memset_zero(lbfgs_b200_ctx* ctx, void* dst, size_t bytes);
lbfgs_b200_status lbfgs_b200_sync(lbfgs_b200_ctx* ctx);
/* CUDA-event stopwatch on the context's stream (device time of everything enqueued in between) */
lbfgs_b200_status lbfgs_b200_timer_start(lbfgs_b200_ctx* ctx);
lbfgs_b200_status lbfgs_b200_timer_stop(lbfgs_b200_ctx* ctx, float* elapsed_ms_host); /* synchronises */
/* Optional device-time accounting per phase (0 = apply_Hv, 1 = line-search trial, 2 = history update): when
 * enabled every such call is bracketed by a CUDA event pair on the context's stream; profile_read synchronises,
 * returns the accumulated milliseconds / call count and optionally clears them. */
lbfgs_b200_status lbfgs_b200_profile_enable(lbfgs_b200_ctx* ctx, int on);
lbfgs_b200_status lbfgs_b200_profile_read(lbfgs_b200_ctx* ctx, int phase, double* total_ms_host, uint64_t* calls_host, int reset);
/* algorithmic bytes of the profiled calls: apply_Hv w*n*(4c+2), trial w*n*4 (+2 for data vectors), update w*n*6 */
lbfgs_b200_status lbfgs_b200_profile_bytes(lbfgs_b200_ctx* ctx, int phase, double* alg_bytes_host, int reset);
/* n-sharding: global index of this rank's element 0 (used by objectives that depend on the coordinate index) */
lbfgs_b200_status lbfgs_b200_set_index_offset(lbfgs_b200_ctx* ctx, int64_t offset);
/* n-sharding: offset as above plus the global vector length.  Required before a neighbour-coupled built-in objective
 * (chained Rosenbrock, tridiagonal quadratic) is evaluated on a sharded vector: those exchange one boundary coordinate per
 * side with the neighbouring ranks before every evaluation (every block but the last must hold a multiple of 4 coordinates). */
lbfgs_b200_status lbfgs_b200_set_global_extent(lbfgs_b200_ctx* ctx, int64_t offset, int64_t n_global);

/* n-sharding over GPUs (SURVEY.md 8e): rank r owns a contiguous block of every vector; all scalars replicated.
 * unique_id is NCCL's 128-byte ncclUniqueId, created on one rank and shipped to the others by the caller. */
lbfgs_b200_status lbfgs_b200_comm_unique_id(void* unique_id_128);
lbfgs_b200_status lbfgs_b200_comm_init(lbfgs_b200_ctx* ctx, const void* unique_id_128, int rank, int nranks);
int lbfgs_b200_comm_size(const lbfgs_b200_ctx* ctx);
/* In-kernel all-reduce over NVLink peer memory (one process per GPU, same node), replacing the per-reduction NCCL call:
 * every rank exports its inbox (64-byte cudaIpcMemHandle), the application gathers the nranks handles in rank order and
 * every rank attaches them.  From then on the last CTA of every reducing kernel pushes its partial sums into all peers'
 * inboxes, waits for theirs and adds them in rank order: deterministic, identical bits on all ranks, no extra launch.
 * All ranks must issue the same sequence of library calls (they do: the host logic is replicated). */
lbfgs_b200_status lbfgs_b200_comm_p2p_export(lbfgs_b200_ctx* ctx, void* ipc_handle_64);
lbfgs_b200_status lbfgs_b200_comm_p2p_attach(lbfgs_b200_ctx* ctx, const void* all_handles_nranks_x_64, int rank, int nranks);

/* ---------------------------------------------------------------- level-1 kernels (f64 / f32) */
#define LBFGS_B200_DECLARE_L1(T, SUF)                                                                          \
    /* a.dot(b)                                   LBFGS.h:123,161; every LineSearch*.h `grad.dot(drt)` */      \
    lbfgs_b200_status lbfgs_b200_dot_##SUF(lbfgs_b200_ctx*, int64_t n, const T* a, const T* b, T* out_host);   \
    /* out3 = { g.d, g.g, x.x } in one pass       LineSearchMoreThuente.h:414 + LBFGS.h:130,137 */             \
    lbfgs_b200_status lbfgs_b200_dot3_##SUF(lbfgs_b200_ctx*, int64_t n, const T* g, const T* d, const T* x,    \
                                            T* out3_host);                                                    \
    /* out = a + s*b  (out may alias a or b)      `x = xp + step*drt`, LineSearchMoreThuente.h:412 */          \
    lbfgs_b200_status lbfgs_b200_axpy_out_##SUF(lbfgs_b200_ctx*, int64_t n, const T* a, T s, const T* b,       \
                                                T* out);                                                      \
    /* out = s*a                                  `m_drt = -m_grad`, LBFGS.h:106 */                            \
    lbfgs_b200_status lbfgs_b200_scale_out_##SUF(lbfgs_b200_ctx*, int64_t n, T s, const T* a, T* out);         \
    /* built-in objective: g = grad f(x), out4 = { f(x), 0, g.g, x.x }   (user functor, LBFGS.h:69-71,91-92) */ \
    lbfgs_b200_status lbfgs_b200_objective_##SUF(lbfgs_b200_ctx*, int objective, const T* data0,               \
                                                 const T* data1, int64_t n, const T* x, T* g, T* out4_host);   \
    /* One line-search trial for a built-in objective in ONE kernel:                                           \
     *   x = xp + step*d;  g = grad f(x);  out4 = { f(x), g.d, g.g, x.x }                                      \
     * replaces LineSearchMoreThuente.h:412-414 (and the same three lines of the other three line searches)    \
     * plus the norms of LBFGS.h:130,137. */                                                                   \
    lbfgs_b200_status lbfgs_b200_trial_##SUF(lbfgs_b200_ctx*, int objective, const T* data0, const T* data1,   \
                                             int64_t n, const T* xp, const T* d, T step, T* x, T* g,          \
                                             T* out4_host);

LBFGS_B200_DECLARE_L1(double, f64)
LBFGS_B200_DECLARE_L1(float, f32)

/* ---------------------------------------------------------------- the S/Y ring (BFGSMat, L-BFGS part) */
/* elem_bytes: 8 (fp64) or 4 (fp32).  Replaces BFGSMat::reset's allocations, BFGSMat.h:61-78. */
lbfgs_b200_status lbfgs_b200_hist_create(lbfgs_b200_ctx* ctx, lbfgs_b200_hist** out, int64_t n, int m,
                                         int elem_bytes);
void lbfgs_b200_hist_destroy(lbfgs_b200_hist* h);
/* theta = 1, ncorr = 0 (no reallocation).  BFGSMat.h:61-78. */
lbfgs_b200_status lbfgs_b200_hist_reset(lbfgs_b200_hist* h);
int lbfgs_b200_hist_ncorr(const lbfgs_b200_hist* h);
int lbfgs_b200_hist_m(const lbfgs_b200_hist* h);
/* device pointers of logical column `age` (0 = newest) for inspection / tests; NULL if age >= ncorr */
const void* lbfgs_b200_hist_s_col(const lbfgs_b200_hist* h, int age);
const void* lbfgs_b200_hist_y_col(const lbfgs_b200_hist* h, int age);

#define LBFGS_B200_DECLARE_HIST(T, SUF)                                                                        \
    /* s = x - xp, y = g - gp written straight into the next ring slot, gate s'y > eps*y'y, ys, theta:         \
     * LBFGS.h:159-162 + BFGSMat::add_correction BFGSMat.h:81-97, one kernel.  sy_yy_host (2 values) optional. */ \
    lbfgs_b200_status lbfgs_b200_hist_update_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g,    \
                                                   const T* gp, T eps, int* accepted_host, T* sy_yy_host);    \
    /* add_correction(s, y) for explicit vectors (BFGSMat.h:81-97); no gate. */                                \
    lbfgs_b200_status lbfgs_b200_hist_add_##SUF(lbfgs_b200_hist* h, const T* s, const T* y);                   \
    /* res = a * H * v by the two-loop recursion, BFGSMat::apply_Hv BFGSMat.h:276-302.                         \
     * gdotres_host (optional) receives v.res, i.e. `dg = m_grad.dot(m_drt)` of LBFGS.h:123 when v = grad.     \
     * res must not alias v. */                                                                                \
    lbfgs_b200_status lbfgs_b200_hist_apply_Hv_##SUF(lbfgs_b200_hist* h, const T* v, T a, T* res, int algo,    \
                                                     T* vdotres_host);                                        \
    /* LBFGS.h:159-165 in one call: hist_update(x, xp, g, gp) followed by apply_Hv(v = g, a, res) (+ g.res).   \
     * With the Gram form the pair is formed inside the dots pass, so x, xp, g, gp are read once and no         \
     * separate update kernel runs; otherwise equivalent to the two calls.  res must not alias an input. */    \
    lbfgs_b200_status lbfgs_b200_hist_update_apply_Hv_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp,       \
                                                            const T* g, const T* gp, T eps, T a, T* res,       \
                                                            int algo, int* accepted_host, T* gdotres_host);    \
    /* host copies of theta and of ys/alpha by age (newest first), for tests */                                \
    lbfgs_b200_status lbfgs_b200_hist_scalars_##SUF(lbfgs_b200_hist* h, T* theta_host, T* ys_host,             \
                                                    T* alpha_host);

LBFGS_B200_DECLARE_HIST(double, f64)
LBFGS_B200_DECLARE_HIST(float, f32)

/* ---------------------------------------------------------------- L1-regularised path (OWLQNSolver, include/OWLQN.h)
 * OWL-QN (Andrew & Gao, "Scalable training of L1-regularized log-linear models", ICML 2007) for F(x) = f(x) + lam |x|_1.  The
 * pseudo-gradient pg(x, g; lam) (g = grad f(x)) is never stored: every pass forms it from x and g with the expressions of
 * include/LBFGSpp/OWLQNCore.h (owlqn_pg, owlqn_orthant, owlqn_project, owlqn_constrain).  Every entry refuses (LBFGS_B200_ERR_INVALID)
 * a lam that is not positive and finite and a context with more than one rank (no n-sharding); the history entry also refuses a
 * history of the other precision. */
#define LBFGS_B200_DECLARE_OWLQN(T, SUF)                                                                       \
    /* The paper's projected line-search trial (section 3.2, "projected line search") for a built-in objective, ONE kernel:     \
     *   x = pi(xp + step*d; xi), xi_i = sign(xp_i) or, at xp_i = 0, sign(-pgp_i), pgp = pg(xp, gp);  g = grad f(x);           \
     *   out5 = { f(x), |x|_1, pgp.(x - xp), pg.pg, x.x }.  Neighbour-coupled objectives see the projected neighbours.          \
     * 5 words per coordinate (+ data vectors). */                                                             \
    lbfgs_b200_status lbfgs_b200_owlqn_trial_##SUF(lbfgs_b200_ctx*, int objective, const T* data0, const T* data1,   \
                                                   int64_t n, const T* xp, const T* d, const T* gp, T step, T lam,    \
                                                   T* x, T* g, T* out5_host);                                        \
    /* The same projection for any objective (the user functor then evaluates f and g at x):                     \
     * x = pi(xp + step*d; xi);  out2 = { |x|_1, pgp.(x - xp) }.  4 words per coordinate. */                     \
    lbfgs_b200_status lbfgs_b200_owlqn_project_##SUF(lbfgs_b200_ctx*, int64_t n, const T* xp, const T* d,         \
                                                     const T* gp, T step, T lam, T* x, T* out2_host);              \
    /* The sums at a point (x, g): out3 = { |x|_1, pg.pg, x.x }.  With d != NULL also the first search's direction   \
     * d = -pg (the paper's steepest-descent start; LBFGS.h:106-108 with pg in place of g).  d may not alias x or g. */ \
    lbfgs_b200_status lbfgs_b200_owlqn_sums_##SUF(lbfgs_b200_ctx*, int64_t n, const T* x, const T* g, T lam, T* d, \
                                                  T* out3_host);                                                    \
    /* The paper's direction (section 3.2, "choosing a direction") after the pair update: the curvature-gated pair  \
     * s = x - xp, y = g - gp (smooth gradients) formed into the ring inside the Gram dots pass, whose right-hand vector is \
     * pg(x, g) formed from the staged x and g tiles; then d = -H pg in the Gram form with d_i = 0 wherever d_i pg_i >= 0, and \
     * dg_host = pg.d over the constrained d.  x, xp, g, gp on 4-element boundaries (lbfgs_b200_malloc); d may not alias them. \
     * accepted_host (optional) = the gate's verdict. */                                                        \
    lbfgs_b200_status lbfgs_b200_owlqn_update_dir_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g,  \
                                                        const T* gp, T eps, T lam, T* d, int* accepted_host,       \
                                                        T* dg_host);                                                \
    /* Per-coordinate weights, F(x) = f(x) + lam sum_i w_i |x_i|: each entry above with w (n entries, device memory) after   \
     * lam.  Coordinate i carries lam_i = lam * w_i rounded once in T; where lam_i > 0 the expressions above apply with lam_i, \
     * where lam_i == 0 (w_i = 0, or a w_i so small that lam * w_i underflows) the coordinate is smooth: pg_i = g_i, the trial \
     * coordinate is xp_i + step d_i unprojected, d_i is not constrained.  The sums report sum_i w_i |x_i| in place of       \
     * |x|_1.  Each refuses a NULL w, and update_dir a w off the 4-element boundary it asks of x.  The sums entry checks     \
     * every weight in its pass: any w_i negative or not finite, or with lam * w_i not finite, makes it return               \
     * LBFGS_B200_ERR_INVALID with their count in the error message; the other entries trust w.  One more word per         \
     * coordinate in each pass. */                                                                              \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_trial_##SUF(lbfgs_b200_ctx*, int objective, const T* data0,       \
                                                            const T* data1, int64_t n, const T* xp, const T* d,   \
                                                            const T* gp, T step, T lam, const T* w, T* x, T* g,   \
                                                            T* out5_host);                                          \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_project_##SUF(lbfgs_b200_ctx*, int64_t n, const T* xp, const T* d, \
                                                              const T* gp, T step, T lam, const T* w, T* x,       \
                                                              T* out2_host);                                        \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_sums_##SUF(lbfgs_b200_ctx*, int64_t n, const T* x, const T* g, T lam, \
                                                           const T* w, T* d, T* out3_host);                        \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_update_dir_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp,     \
                                                                 const T* g, const T* gp, T eps, T lam, const T* w, \
                                                                 T* d, int* accepted_host, T* dg_host);

LBFGS_B200_DECLARE_OWLQN(double, f64)
LBFGS_B200_DECLARE_OWLQN(float, f32)

/* ---------------------------------------------------------------- bound-constrained path (LBFGSBSolver, config 4)
 * Index sets of the reference (std::vector<int> free / active / L / U / P sets of Cauchy.h and SubspaceMin.h) are bits of
 * a per-coordinate class byte; W = [Y, theta*S] is never gathered: every W-product is a masked pass over the S/Y columns.
 * The 2m x 2m algebra (Minv, BKLDLT, the BOXCQP bookkeeping) stays on the host in the C++ front, as in the reference.
 * Replicas only: these entry points refuse a context with more than one rank.  m <= 20. */
typedef struct lbfgs_b200_box lbfgs_b200_box;   /* n-sized temporaries of Cauchy / SubspaceMin + sort buffers */
enum { LBFGS_B200_CLS_FIXED = 1, LBFGS_B200_CLS_ACT = 2, LBFGS_B200_CLS_FREE = 4,
       LBFGS_B200_SUB_L = 8, LBFGS_B200_SUB_U = 16, LBFGS_B200_SUB_P = 32 };
/* element-wise steps of SubspaceMin::subspace_minimize (SubspaceMin.h:122-302), see lbfgsb_kernels.cuh */
enum { LBFGS_B200_SUB_INIT = 0, LBFGS_B200_SUB_ACT_DIR = 1, LBFGS_B200_SUB_ADD_G = 2, LBFGS_B200_SUB_NEG_C_FREE = 3,
       LBFGS_B200_SUB_CHECK_BOUNDS = 4, LBFGS_B200_SUB_CLASSIFY = 5, LBFGS_B200_SUB_LU_VEC = 6, LBFGS_B200_SUB_RHS_P = 7,
       LBFGS_B200_SUB_FREE_VEC = 8, LBFGS_B200_SUB_MULTIPLIERS = 9, LBFGS_B200_SUB_CONVERGED = 10,
       LBFGS_B200_SUB_WRITE_DRT = 11 };
/* class bit of the free set at a solution (lbfgs_b200_box_final_classes); bits 1 to 32 belong to Cauchy and the subspace step */
enum { LBFGS_B200_CLS_FINAL = 64 };
/* work vectors of the box workspace, for lbfgs_b200_box_vector() */
enum { LBFGS_B200_BOXV_VECC = 0, LBFGS_B200_BOXV_VECY = 1, LBFGS_B200_BOXV_LAMBDA = 2, LBFGS_B200_BOXV_MU = 3,
       LBFGS_B200_BOXV_TMP = 4, LBFGS_B200_BOXV_TMP2 = 5, LBFGS_B200_BOXV_YFB = 6, LBFGS_B200_BOXV_DVEC = 7,
       LBFGS_B200_BOXV_BRK = 8, LBFGS_B200_BOXV_XCP = 9 };

lbfgs_b200_status lbfgs_b200_box_create(lbfgs_b200_hist* h, lbfgs_b200_box** out);
void lbfgs_b200_box_destroy(lbfgs_b200_box* b);
const void* lbfgs_b200_box_xcp(const lbfgs_b200_box* b);                 /* generalized Cauchy point (device, n)   */
const unsigned char* lbfgs_b200_box_classes(const lbfgs_b200_box* b);    /* class bytes (device, n)                */
void* lbfgs_b200_box_vector(lbfgs_b200_box* b, int which);               /* LBFGS_B200_BOXV_* (device, n)          */

#define LBFGS_B200_DECLARE_BOX(T, SUF)                                                                         \
    /* x = x.cwiseMax(lb).cwiseMin(ub)                                   force_bounds, LBFGSB.h:55-58 */        \
    lbfgs_b200_status lbfgs_b200_box_clamp_##SUF(lbfgs_b200_ctx*, int64_t n, T* x, const T* lb, const T* ub);  \
    /* max_i |clamp(x - g) - x|                                          proj_grad_norm, LBFGSB.h:62-65 */      \
    lbfgs_b200_status lbfgs_b200_box_proj_grad_norm_##SUF(lbfgs_b200_ctx*, int64_t n, const T* x, const T* g,  \
                                                          const T* lb, const T* ub, T* out_host);              \
    /* out2 = { g.d , largest feasible step along d }                    LBFGSB.h:176 + max_step_size :68-86 */ \
    lbfgs_b200_status lbfgs_b200_box_dir_info_##SUF(lbfgs_b200_ctx*, int64_t n, const T* x, const T* d,        \
                                                    const T* g, const T* lb, const T* ub, T* out2_host);       \
    /* raw[2c] = { y_age.v (c), s_age.v (c) }        apply_Wtv / apply_WtPv without theta, BFGSMat.h:315-320,382-433 */ \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_##SUF(lbfgs_b200_hist*, const T* v, T* raw_host);                 \
    /* c x c Gram blocks by age (row-major, any may be NULL): s_i.y_j, s_i.s_j, y_i.y_j; ys[c]; theta  (the material   \
     * of m_permMinv, BFGSMat.h:99-146) */                                                                     \
    lbfgs_b200_status lbfgs_b200_hist_gram_##SUF(lbfgs_b200_hist*, T* SY_host, T* SS_host, T* YY_host,         \
                                                 T* ys_host, T* theta_host);                                   \
    /* out_i = a0*v0_i + sum_j cy_j*y_j[i] + cs_j*s_j[i] on rows with (cls_i & mask) != 0 (cls NULL: all rows);        \
     * coef_host = { cy by age (c), cs by age (c) }.    apply_PtWMv / apply_PtBQv / solve_PtBP tail, BFGSMat.h:435-615 */ \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_##SUF(lbfgs_b200_hist*, lbfgs_b200_box*, T a0, const T* v0,      \
                                                    const T* coef_host, const unsigned char* cls, int mask,    \
                                                    T* out);                                                   \
    /* G[(2c)x(2c)] = sum over rows with (cls & mask) of r r', r = (y_0[i]..,s_0[i]..) by age.  WP'WP, BFGSMat.h:529-565 */ \
    lbfgs_b200_status lbfgs_b200_hist_masked_gram_##SUF(lbfgs_b200_hist*, lbfgs_b200_box*,                     \
                                                        const unsigned char* cls, int mask, T* G_host);        \
    /* Products of the final quasi-Newton approximation with blocks of vectors (LBFGSSolver::final_approx_hessian_times /     \
     * final_approx_inverse_hessian_times, the operator form of final_approx_hessian(), LBFGS.h:192-197 / BFGSMat.h:150-271): \
     * V and OUT hold k column vectors (1 <= k <= 16) with leading dimensions ldv, ldo >= n; every history column and every     \
     * column of V is read once per call.  No box workspace, any m; replicas only (a context with more than one rank is refused).     \
     * R_host[2c][k] = [Y S]'V, rows y by age then s by age, summed in fp64 in an order that does not depend on k.           */ \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_multi_##SUF(lbfgs_b200_hist* h, int k, const T* V, int64_t ldv,   \
                                                         T* R_host);                                           \
    /* OUT[:,j] = a0*V[:,j] + sum_a C[a][j]*y_a + C[c+a][j]*s_a, C_host row-major [2c][k] (y by age, then s by age); per       \
     * element the terms are added in that order (with k = 1 the arithmetic of hist_lincomb).  OUT may be V when ldo == ldv. */ \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_multi_##SUF(lbfgs_b200_hist* h, T a0, int k, const T* V,         \
                                                          int64_t ldv, const T* C_host, T* OUT, int64_t ldo);  \
    /* The diagonal of the final approximation (LBFGSSolver::final_approx_hessian_diagonal / _inverse_hessian_diagonal): with  \
     * B or H = a0 I + W K W', W = [Y S] (include/LBFGSpp/CompactForm.h, compact_kb / compact_kh), out_i = a0 + r_i' K r_i for   \
     * i < n, r_i = (y_0[i] .. y_{c-1}[i], s_0[i] .. s_{c-1}[i]).  K_host [2c][2c] row-major, symmetric: only its upper triangle \
     * is read (NULL allowed when c = 0).  One pass over the 2c history columns, no reductions; per element the sum is taken   \
     * in fp64 in a fixed order (lbfgsb_kernels.cuh, k_hist_quad_diag), so out_i depends on row i and K only.  Any m; replicas \
     * only (a context with more than one rank is refused).  Entries of out past n are not written.                          */ \
    lbfgs_b200_status lbfgs_b200_hist_quad_diag_##SUF(lbfgs_b200_hist* h, T a0, const T* K_host, T* out);      \
    /* The sampler of N(mean, H) (BFGSMat::sample): the two k-vector passes above with V = Z generated in the kernels, never   \
     * stored, z_j = the standard normals of draw first + j of stream `stream` (Philox4x32-10, counter layout in              \
     * csrc/philox.cuh; a draw depends on (seed, stream, j, i) only).  wt_dot_normal: R_host[2c][k] = [Y S]' Z in the order of  \
     * hist_wt_dot_multi (column j of a call equals a k = 1 call with first + j).  lincomb_normal: OUT_j = mean + a0 z_j +      \
     * sum_a C[c+a][j] s_a (C_host [2c][k] as hist_lincomb_multi takes it; its y rows are not read; mean may be NULL: zero).   \
     * 1 <= k <= 16, first + k <= 2^32; replicas only.                                                                       */ \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_normal_##SUF(lbfgs_b200_hist* h, uint64_t seed, uint32_t stream, uint32_t first, \
                                                          int k, T* R_host);                                               \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_normal_##SUF(lbfgs_b200_hist* h, T a0, uint64_t seed, uint32_t stream,         \
                                                           uint32_t first, int k, const T* mean, const T* C_host, T* OUT,   \
                                                           int64_t ldo);                                                    \
    /* Whitening and log densities under N(mean, H) (BFGSMat::inverse_hessian_factor_transpose_times / _solve /              \
     * _transpose_solve / log_density; each replaces hist_wt_dot_multi on a full W'V).  s_dot_multi: R_host[c][k] = S'V, rows s  \
     * by age, row a bit-identical to the s row of age a from hist_wt_dot_multi on the same V; only the c s columns are read.    \
     * wt_dot_diff: R_host[2c][k] = [Y S]'(X - mean) and nrm_host[j] = |x_j - mean|^2, both as summed in fp64 (no rounding to T), \
     * the differences formed in the pass as x - mean in T (R rounded to T is bit-identical to hist_wt_dot_multi on X - mean    \
     * from lbfgs_b200_axpy_out(x, -1, mean)).                                                                                  \
     * 1 <= k <= 16, ldv, ldx >= n, any m; replicas only.                                                                       */ \
    lbfgs_b200_status lbfgs_b200_hist_s_dot_multi_##SUF(lbfgs_b200_hist* h, int k, const T* V, int64_t ldv, T* R_host);      \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_diff_##SUF(lbfgs_b200_hist* h, int k, const T* X, int64_t ldx, const T* mean,    \
                                                        double* R_host, double* nrm_host);                                   \
    /* The final approximation on the free variables of a bound-constrained solve (LBFGSBSolver::final_approx_free_*): the     \
     * passes above restricted to the rows i with (cls_i & mask) != 0, cls the class bytes of box b (of history h).  Each keeps  \
     * its twin's order, so with every row in the mask it computes its twin's bits, and follows its twin's rules (1 <= k <= 16,  \
     * leading dimensions, replicas only).  wt_dot_multi / wt_dot_diff / wt_dot_normal: the vector rows outside the mask count   \
     * as 0 (the norms of wt_dot_diff too).  lincomb_multi: OUT rows outside the mask are written as 0.  lincomb_normal: reads   \
     * every row of C_host (y and s), OUT rows outside the mask are mean_i (0 when mean is NULL).  quad_diag: out_i = 0 outside  \
     * the mask.                                                                                                                */ \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_multi_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, \
                                                                int mask, int k, const T* V, int64_t ldv, T* R_host);          \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_diff_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls,  \
                                                               int mask, int k, const T* X, int64_t ldx, const T* mean,        \
                                                               double* R_host, double* nrm_host);                              \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_normal_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, \
                                                                 int mask, uint64_t seed, uint32_t stream, uint32_t first,     \
                                                                 int k, T* R_host);                                            \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_multi_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, \
                                                                 int mask, T a0, int k, const T* V, int64_t ldv,               \
                                                                 const T* C_host, T* OUT, int64_t ldo);                        \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_normal_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b,                      \
                                                                  const unsigned char* cls, int mask, T a0, uint64_t seed,     \
                                                                  uint32_t stream, uint32_t first, int k, const T* mean,      \
                                                                  const T* C_host, T* OUT, int64_t ldo);                       \
    lbfgs_b200_status lbfgs_b200_hist_quad_diag_masked_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls,   \
                                                             int mask, T a0, const T* K_host, T* out);                         \
    /* The free set at a solution x: LBFGS_B200_CLS_FINAL set in the class bytes of the free coordinates and cleared elsewhere   \
     * (the other bits are kept).  Coordinate i is fixed when lb_i == ub_i, x_i <= lb_i + tol max(1, |lb_i|) or                 \
     * x_i >= ub_i - tol max(1, |ub_i|) (infinite bounds never fix); *nfree_host = the number of free ones.  Cauchy rebuilds   \
     * the class bytes, so the set lasts until the next iteration of a solve.                                                  */ \
    lbfgs_b200_status lbfgs_b200_box_final_classes_##SUF(lbfgs_b200_box* b, const T* x, const T* lb, const T* ub, T tol,      \
                                                         int64_t* nfree_host);                                                 \
    /* Cauchy.h:111-129: breakpoints, d = -g on movable coordinates, class bytes.                                      \
     * out5 = { #fixed, #never-bounded, #with a finite breakpoint, d.d, smallest breakpoint } */                       \
    lbfgs_b200_status lbfgs_b200_box_cauchy_breaks_##SUF(lbfgs_b200_box*, const T* x, const T* g, const T* lb, \
                                                         const T* ub, T* out5_host);                           \
    /* Cauchy.h:132-256: sort the breakpoints, prefix sums, first segment holding its one-dimensional minimiser.       \
     * Mmat_host [2c][2c] (B = theta I - W M W'), p0_host = W'd [2c].                                                  \
     * out = { t_cross, tfinal, f', f'', all-crossed flag, W'(xcp - x0) [2c] } */                                      \
    lbfgs_b200_status lbfgs_b200_box_cauchy_sweep_##SUF(lbfgs_b200_box*, const T* g, const T* Mmat_host,       \
                                                        const T* p0_host, T theta, T gt, int64_t nord,         \
                                                        int64_t nfree_inf, T* out_host);                       \
    /* Cauchy.h:205-216,268-283: xcp and the ACT / FREE classes from (t_cross, tfinal); counts2 = { #act, #free } */   \
    lbfgs_b200_status lbfgs_b200_box_cauchy_build_##SUF(lbfgs_b200_box*, const T* x, const T* lb, const T* ub, \
                                                        T t_cross, T tfinal, T* counts2_host);                 \
    /* one element-wise step (LBFGS_B200_SUB_*) of SubspaceMin.h:122-302; reducing steps return 3 counters */          \
    lbfgs_b200_status lbfgs_b200_box_sub_step_##SUF(lbfgs_b200_box*, int op, int flag, const T* x0,            \
                                                    const T* g, const T* lb, const T* ub, T* drt, T theta,     \
                                                    T* out3_host);

LBFGS_B200_DECLARE_BOX(double, f64)
LBFGS_B200_DECLARE_BOX(float, f32)

/* ---------------------------------------------------------------- device-resident solve (built-in objectives)
 * LBFGSSolver<Scalar, LineSearch>::minimize() (reference LBFGS.h:78-173) as ONE persistent cooperative kernel launch, for one problem
 * or for a batch of B independent problems of the same shape (BASELINE config 5).  One CTA per SM stays resident for the whole
 * solve; the work proceeds in rounds of one streaming pass per running problem (first evaluation / line-search trial /
 * pair-forming dots [S Y]'[g s y] / combination d = -H g fused with the first trial of the next search) separated by one grid-wide
 * synchronisation in which CTA 0 sums the CTAs' partial sums in a fixed order, exchanges them with the other ranks when n is
 * sharded (ONE exchange per round for all running problems: a B-vector all-reduce per dot) and runs every problem's scalar logic:
 * the line-search state machines (include/LBFGSpp/LineSearchCore.h, the code the host front uses), the convergence tests of
 * LBFGS.h:137-154, the curvature gate of :161, the ring bookkeeping of BFGSMat.h:81-97 and the buffer rotation.  The host is not
 * involved between launch and completion.  Reductions are deterministic and a problem's result does not depend on what else is
 * in the batch: every problem of a batch is bit-identical to the same problem solved alone.
 * When n is sharded the in-kernel NVLink exchange must be attached (lbfgs_b200_comm_p2p_*); neighbour-coupled objectives then
 * also need lbfgs_b200_set_global_extent (their boundary coordinates travel with the sums). */
typedef struct lbfgs_b200_solver lbfgs_b200_solver;
typedef struct {             /* LBFGSParam (reference Param.h:67-219); doubles for both precisions */
    int m;
    double epsilon, epsilon_rel;
    int past;
    double delta;
    int max_iterations;
    int linesearch;
    int max_linesearch;
    double min_step, max_step, ftol, wolfe;
} lbfgs_b200_param;
typedef struct {
    int status;              /* 0, or a LBFGSpp::LineSearchError code (>= 16) = the exception the reference would throw */
    int niter;               /* return value of minimize()                                                          */
    long long nfev;          /* objective evaluations                                                               */
    double fx, gnorm;
    long long rounds;        /* streaming passes (= grid-wide synchronisations) this problem took part in           */
} lbfgs_b200_outcome;
enum { LBFGS_B200_LS_BACKTRACKING = 0, LBFGS_B200_LS_BRACKETING = 1, LBFGS_B200_LS_NOCEDAL_WRIGHT = 2, LBFGS_B200_LS_MORE_THUENTE = 3 };

lbfgs_b200_status lbfgs_b200_solver_create(lbfgs_b200_ctx* ctx, int64_t n, int m, int elem_bytes, lbfgs_b200_solver** out);
/* batch problems of n coordinates each (n = this rank's block when sharded), all with history size m */
lbfgs_b200_status lbfgs_b200_solver_create_batch(lbfgs_b200_ctx* ctx, int64_t n, int m, int elem_bytes, int batch, lbfgs_b200_solver** out);
void lbfgs_b200_solver_destroy(lbfgs_b200_solver* s);
int lbfgs_b200_solver_batch(const lbfgs_b200_solver* s);
/* Accounting of the last solve.  kernel_ms: device time of the one kernel (CUDA events around its launch).  The arrays have 10 slots
 * indexed by the pass a round ran: 0 = rounds in which the problems of a batch ran different passes, 1 FIRST, 2 TRIAL, 3 DOTS_FORM,
 * 4 DOTS_PLAIN, 5 COMBINE, 6 COMBINE_TRIAL, 7 RESTORE, 8 MATERIALIZE (9 unused).  ms_by_op10: the kernel's time split by round (CTA 0's cycle counter scaled
 * to kernel_ms; includes each round's synchronisation); alg_bytes_by_op10: algorithmic bytes of those passes (whole vectors read and
 * written: FIRST 2n, TRIAL 2n (first search 1n), DOTS_FORM (c+2)n (iteration 1 (c+1)n), DOTS_PLAIN (c+2)n, COMBINE (c+2)n,
 * COMBINE_TRIAL (c+2)n, MATERIALIZE 4n (first search 3n) or 3n words (the point on the ray; the search's start point or the point
 * already in x: the gradient is evaluated from x, not stored, before MATERIALIZE, the first search's direction -grad f(x0) is evaluated
 * from x0, not stored, and the history ring holds the c+1 iterates of c chained pairs, not the pairs); for the neighbour-coupled
 * objectives, whose trials store their points, whose passes read the stored gradient and whose ring holds S|Y: FIRST 3n, TRIAL 4n,
 * DOTS_FORM (2c+4)n, DOTS_PLAIN (2c+1)n, COMBINE (2c+2)n, COMBINE_TRIAL (2c+5)n, MATERIALIZE 4n, RESTORE 4n; + the objective's
 * data vectors per evaluation); sync_ms[3]: { the part of kernel_ms between CTA 0's arrival at a grid barrier and its release, the part of that spent waiting for
 * the last CTA to arrive, the part spent in the cross-rank exchange }. */
lbfgs_b200_status lbfgs_b200_solver_profile(const lbfgs_b200_solver* s, double* kernel_ms, double* ms_by_op10, unsigned long long* rounds_by_op10,
                                            double* alg_bytes_by_op10, double* sync_ms);
const void* lbfgs_b200_solver_final_grad(const lbfgs_b200_solver* s);   /* device pointer (problem 0), valid until the next minimize */
const void* lbfgs_b200_solver_final_grad_of(const lbfgs_b200_solver* s, int problem);
lbfgs_b200_hist* lbfgs_b200_solver_history(lbfgs_b200_solver* s);       /* the S/Y ring of problem 0 as left by the last solve   */
lbfgs_b200_hist* lbfgs_b200_solver_history_of(lbfgs_b200_solver* s, int problem);
/* x_inout: device vector (start point in, solution out).  trace_host (optional): f of every evaluation.
 * data0/data1 (as the objective needs, here and in the batch entry points below): device vectors that start on a 16-byte boundary.
 * The solve reads each problem's data with bulk copies of whole 32-element groups, up to round_up(n, 32) elements from its start
 * (the values past n are not used); a vector of n elements from lbfgs_b200_malloc has that room.  LBFGS_B200_ERR_INVALID, before
 * anything is launched, for a misaligned data vector. */
lbfgs_b200_status lbfgs_b200_solver_minimize_f64(lbfgs_b200_solver* s, int objective, const double* data0, const double* data1,
                                                 const lbfgs_b200_param* prm, int line_search, double* x_inout,
                                                 double* trace_host, long long trace_cap, lbfgs_b200_outcome* out);
lbfgs_b200_status lbfgs_b200_solver_minimize_f32(lbfgs_b200_solver* s, int objective, const float* data0, const float* data1,
                                                 const lbfgs_b200_param* prm, int line_search, float* x_inout,
                                                 double* trace_host, long long trace_cap, lbfgs_b200_outcome* out);
/* Batch: problem b starts from x_inout + b*ldx (device) and leaves its solution there; data0/data1 (optional) per problem at
 * data + b*ldd (ldd = 0: shared by all problems); outs[batch].  ldd must be 0 or at least n, and ldd*elem_bytes a multiple of 16, so
 * that every problem's data starts on a 16-byte boundary; the buffers must hold (batch-1)*ldd + round_up(n, 32) elements.
 * LBFGS_B200_ERR_INVALID, before anything is launched, otherwise. */
lbfgs_b200_status lbfgs_b200_solver_minimize_batch_f64(lbfgs_b200_solver* s, int objective, const double* data0, const double* data1,
                                                       int64_t ldd, const lbfgs_b200_param* prm, int line_search, double* x_inout,
                                                       int64_t ldx, lbfgs_b200_outcome* outs);
lbfgs_b200_status lbfgs_b200_solver_minimize_batch_f32(lbfgs_b200_solver* s, int objective, const float* data0, const float* data1,
                                                       int64_t ldd, const lbfgs_b200_param* prm, int line_search, float* x_inout,
                                                       int64_t ldx, lbfgs_b200_outcome* outs);

/* ---------------------------------------------------------------- small-batch solve (built-in objectives)
 * Many independent small problems in ONE ordinary launch: one thread block per problem runs that problem's whole minimize()
 * (reference LBFGS.h:78-173) in its own shared memory, with the device-resident solve's per-problem state machine (same line
 * searches, stopping rules, curvature gate and outcomes).  No grid-wide synchronisation: B is limited only by device memory for
 * X (and G).  Every problem's sums are taken in an order that depends on n only (32 threads per block up to n = 128, 128 above), so
 * a problem's result is bit-identical whatever B is and wherever it sits in the batch; it equals LBFGSSolver's result to rounding
 * (the sums are associated differently), not bit for bit.  One rank only.
 * Shared memory of one block, with M = m + 1, p = round_up(max(6m, 8), 8), e = elem_bytes and N = round_up(n, 4):
 *     e*N*(5 + 2M + 2*[chained Rosenbrock, tridiagonal quadratic: stored trials] + 2*[tridiagonal quadratic: data])
 *   + 2048 (problem state) + 8*5p (sums) + a16(e*(2M + 4 + 6M^2)) (ys, alpha, theta, Gram matrices) + a16(e*(2m^2 + 6m + 2)) (recursion)
 * where a16 rounds up to a multiple of 16; it must not exceed 232448 bytes (227 KB, the per-block limit of sm_90).  For fp64 paired
 * Rosenbrock that is 152 bytes per coordinate at m = 6 (n <= 1480) and 216 at m = 10 (n <= 1016); at large m the Gram matrices
 * alone exceed the limit. */
/* largest n that fits one block's shared memory for (m, precision, objective): a multiple of 4, 0 if none.  Pure host function. */
int64_t lbfgs_b200_small_max_n(int m, int elem_bytes, int objective);
/* B independent problems of n coordinates, one block each.  X: B device vectors ldx >= n elements apart (start points in,
 * solutions out); G (nullable): the final gradients, same layout; data0/data1 (as the objective needs): problem b's at data + b*ldd
 * (ldd = 0: shared by all problems); outs_host[B]: status / niter / nfev / fx / gnorm / rounds exactly as
 * lbfgs_b200_solver_minimize_batch reports them.  LBFGS_B200_ERR_INVALID for n > lbfgs_b200_small_max_n, B < 1, ldx < n,
 * past > 64 or a context with more than one rank.  Synchronises. */
lbfgs_b200_status lbfgs_b200_small_minimize_f64(lbfgs_b200_ctx* ctx, int objective, const double* data0, const double* data1, int64_t ldd,
                                                int64_t n, int64_t B, const lbfgs_b200_param* prm, int line_search,
                                                double* X, int64_t ldx, double* G, lbfgs_b200_outcome* outs_host);
lbfgs_b200_status lbfgs_b200_small_minimize_f32(lbfgs_b200_ctx* ctx, int objective, const float* data0, const float* data1, int64_t ldd,
                                                int64_t n, int64_t B, const lbfgs_b200_param* prm, int line_search,
                                                float* X, int64_t ldx, float* G, lbfgs_b200_outcome* outs_host);

/* The final quasi-Newton approximations of a small-batch solve, kept on the device (the small-batch counterpart of
 * final_approx_hessian() / final_approx_inverse_hessian(), reference LBFGS.h:192-197, BFGSMat.h:150-271).  A history made for
 * (n, m, precision, B) receives, from lbfgs_b200_small_minimize_keep_*, every problem's pairs, ys, theta and Gram blocks as BFGSMat
 * holds them when minimize() returns (the last step's pair is not among them).  Device memory: B*(2m*n + m + 3m^2 + 2) elements
 * plus B ints; fp64, B = 65536, n = 256, m = 10: about 2.8 GB.  LBFGS_B200_ERR_ALLOC when that cannot be had. */
typedef struct lbfgs_b200_small_hist lbfgs_b200_small_hist;
lbfgs_b200_status lbfgs_b200_small_hist_create(lbfgs_b200_ctx* ctx, int64_t n, int m, int elem_bytes, int64_t B, lbfgs_b200_small_hist** out);
void lbfgs_b200_small_hist_destroy(lbfgs_b200_small_hist* h);
/* device pointers to s / y of problem b at `age` (0 = newest; meaningful for age < its pair count), for tests; NULL out of range */
const void* lbfgs_b200_small_hist_s_col(const lbfgs_b200_small_hist* h, int64_t b, int age);
const void* lbfgs_b200_small_hist_y_col(const lbfgs_b200_small_hist* h, int64_t b, int age);

/* op of lbfgs_b200_small_hist_factor_apply_*: with H = L L' (include/LBFGSpp/CompactForm.h), L, L', L^-1 or L^-T */
enum { LBFGS_B200_FACTOR_L = 0, LBFGS_B200_FACTOR_LT = 1, LBFGS_B200_FACTOR_LINV = 2, LBFGS_B200_FACTOR_LINVT = 3 };

#define LBFGS_B200_DECLARE_SMALL_HIST(T, SUF)                                                                                     \
    /* lbfgs_b200_small_minimize_* that also fills `hist`, whose n, m, precision and B must match the solve's             \
     * (LBFGS_B200_ERR_INVALID before anything is launched otherwise).  Everything else is the same launch.            */ \
    lbfgs_b200_status lbfgs_b200_small_minimize_keep_##SUF(lbfgs_b200_ctx* ctx, int objective, const T* data0, const T* data1,   \
                                                           int64_t ldd, int64_t n, int64_t B, const lbfgs_b200_param* prm,        \
                                                           int line_search, T* X, int64_t ldx, T* G, lbfgs_b200_outcome* outs_host, \
                                                           lbfgs_b200_small_hist* hist);                                        \
    /* per problem: its pair count c (c_host[B]) and theta (theta_host[B]); either may be NULL.  Synchronises.            */ \
    lbfgs_b200_status lbfgs_b200_small_hist_info_##SUF(lbfgs_b200_small_hist* h, int* c_host, T* theta_host);                    \
    /* OUT_p = B_b V_p (inverse = 0) or H_b V_p (inverse != 0) for the problems b = b0 + p, p < count, in one launch: k >= 1   \
     * vectors each, vector j of problem p at V + p*ldvp + j*ldv (ldvp = 0: one V for every problem), its product at          \
     * OUT + p*ldop + j*ldo; ldv, ldo >= n.  The arithmetic of LBFGSSolver::final_approx_*_times: [Y S]'V summed in fp64, the   \
     * coefficients of the compact form (include/LBFGSpp/CompactForm.h), OUT = a0 V + sum cy_a y_a + sum cs_a s_a in that order. \
     * A problem's products depend on n only, not on b0, count or k.  OUT may be V only with the same layout (ldo == ldv,       \
     * ldop == ldvp) and, for count > 1, vectors of its own per problem.  LBFGS_B200_ERR_INVALID for k < 1, ldv or ldo < n, a     \
     * problem range outside [0, B), NULL pointers or a history no solve has filled.  Asynchronous.                          */ \
    lbfgs_b200_status lbfgs_b200_small_hist_times_##SUF(lbfgs_b200_small_hist* h, int inverse, int64_t b0, int64_t count, int k, \
                                                        const T* V, int64_t ldv, int64_t ldvp, T* OUT, int64_t ldo, int64_t ldop);   \
    /* OUT + p*ldo = diag(B_b) (inverse = 0) or diag(H_b) (inverse != 0) for the problems b = b0 + p, p < count, in one launch  \
     * (one block per problem): the block forms its problem's K of CompactForm.h on the chip and makes one pass over its 2c    \
     * history columns, out_i = a0 + r_i' K r_i in the order of lbfgs_b200_hist_quad_diag.  A problem's diagonal depends on its   \
     * history only, not on b0, count or its position; with c = 0 it is theta (B) or 1/theta (H).  LBFGS_B200_ERR_INVALID for  \
     * ldo < n, a problem range outside [0, B), a NULL OUT, a history no solve has filled or a context with more than one      \
     * rank.  Asynchronous.                                                                                                   */ \
    lbfgs_b200_status lbfgs_b200_small_hist_diag_##SUF(lbfgs_b200_small_hist* h, int inverse, int64_t b0, int64_t count, T* OUT,   \
                                                       int64_t ldo);                                                              \
    /* The square-root factor H_b = L_b L_b' of include/LBFGSpp/CompactForm.h (compact_factor_setup / compact_factor_coef), formed \
     * on the chip per problem.  factor_times: OUT = L_b V in the layout of small_hist_times.  sample: OUT + p*ldop + j*ldo =    \
     * MEAN + p*ldm + L_b z_j, z_j = draw first + j of stream b (the absolute problem index; philox.cuh), so a problem's draws do \
     * not depend on b0 or count; MEAN may be NULL (zero).  The sampler uses OUT as scratch: with count > 1 it needs ldop >= k*ldo, and MEAN may not overlap OUT.  A problem whose pairs fail the check of compact_factor_setup gets NaN \
     * outputs.  logdet: out_host[p] = log det H_b (NaN on that failure), synchronous.  Errors as small_hist_times.            */ \
    lbfgs_b200_status lbfgs_b200_small_hist_factor_times_##SUF(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, int k,         \
                                                               const T* V, int64_t ldv, int64_t ldvp, T* OUT, int64_t ldo,       \
                                                               int64_t ldop);                                                    \
    lbfgs_b200_status lbfgs_b200_small_hist_sample_##SUF(lbfgs_b200_small_hist* h, uint64_t seed, uint32_t first, int64_t b0,       \
                                                         int64_t count, int k, const T* MEAN, int64_t ldm, T* OUT, int64_t ldo,  \
                                                         int64_t ldop);                                                          \
    lbfgs_b200_status lbfgs_b200_small_hist_logdet_##SUF(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, double* out_host);  \
    /* Whitening under N(x_b, H_b) (CompactForm.h, compact_factor_t_coef / _inv_coef / _invt_coef): OUT = op(L_b) V with op one  \
     * of LBFGS_B200_FACTOR_*, in the layouts and with the aliasing rules of factor_times (op L is factor_times).  Asynchronous.   \
     * log_density: out_host[p*k + j] = log N(x_pj; MEAN + p*ldm, H_b), point j of problem p at X + p*ldxp + j*ldx, from          \
     * W'(x - mean) and |x - mean|^2 alone (compact_factor_quad); MEAN is required.  Synchronous.  A problem whose pairs fail    \
     * the check of compact_factor_setup gets NaN outputs.  Errors as small_hist_times, and an op out of range.                */ \
    lbfgs_b200_status lbfgs_b200_small_hist_factor_apply_##SUF(lbfgs_b200_small_hist* h, int op, int64_t b0, int64_t count, int k, \
                                                               const T* V, int64_t ldv, int64_t ldvp, T* OUT, int64_t ldo,       \
                                                               int64_t ldop);                                                    \
    lbfgs_b200_status lbfgs_b200_small_hist_log_density_##SUF(lbfgs_b200_small_hist* h, int64_t b0, int64_t count, int k,          \
                                                               const T* X, int64_t ldx, int64_t ldxp, const T* MEAN, int64_t ldm, \
                                                               double* out_host);

LBFGS_B200_DECLARE_SMALL_HIST(double, f64)
LBFGS_B200_DECLARE_SMALL_HIST(float, f32)

#ifdef __cplusplus
}
#endif
#endif /* LBFGS_B200_H */
