/* oracle_api.h -- TEST INFRASTRUCTURE ONLY.
 *
 * One C ABI implemented twice:
 *   - oracle/_ref/libref_lbfgspp.so : the UNMODIFIED reference headers (LBFGSpp's include/)
 *     compiled over oracle/minieigen (built only when REF names a checkout), prefix "ref_";
 *   - oracle/liboracle.so           : the plain-C++ restatement (oracle/lbfgs_oracle.hpp),
 *     prefix "orc_".
 * Both are checkers.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load them; the product (lbfgspp_b200/, include/) never does.
 */
#ifndef LBFGS_ORACLE_API_H
#define LBFGS_ORACLE_API_H

/* Both checker libraries are built with -fvisibility=hidden -Wl,-Bsymbolic: only this C API is exported, and their internal
 * C++ symbols (namespace LBFGSpp of the reference, namespace orc) can never interpose with, or be interposed by, the product's
 * libraries when a test process loads several of them. */
#define ORC_API __attribute__((visibility("default")))

#ifdef __cplusplus
extern "C" {
#endif

/* objective functions (restated from the reference examples, see oracle/objectives.hpp) */
enum {
    ORC_OBJ_ROSENBROCK_PAIRED = 0,  /* examples/example-rosenbrock.cpp:15-27                     */
    ORC_OBJ_QUAD_SHIFT = 1,         /* examples/example-quadratic.cpp:9-19  f = |x - (0,1,2..)|^2 */
    ORC_OBJ_ROSENBROCK_CHAINED = 2, /* examples/example-rosenbrock-box.cpp:18-33                 */
    ORC_OBJ_QUAD_TRIDIAG = 3        /* SURVEY 8d C3: f = 1/2 x'Ax - b'x, A = diag(d)+1/2 tridiag(-1,2,-1);
                                       data0 = d (n), data1 = b (n)                              */
};

/* line-search policies = the reference's four LineSearch* templates */
enum { ORC_LS_BACKTRACKING = 0, ORC_LS_BRACKETING = 1, ORC_LS_NOCEDAL_WRIGHT = 2, ORC_LS_MORE_THUENTE = 3 };

/* dot-product summation order used by the restatement (the _ref build is always sequential) */
enum { ORC_SUM_SEQUENTIAL = 0, ORC_SUM_LANES8 = 1, ORC_SUM_LANES8_OMP = 2 };

/* union of LBFGSParam and LBFGSBParam fields (reference Param.h:67-219, 224-377) */
typedef struct {
    int m;
    double epsilon, epsilon_rel;
    int past;
    double delta;
    int max_iterations;
    int linesearch; /* LBFGSParam only  */
    int max_submin; /* LBFGSBParam only */
    int max_linesearch;
    double min_step, max_step, ftol, wolfe;
} orc_param;

enum { ORC_OK = 0, ORC_INVALID_ARGUMENT = 1, ORC_LOGIC_ERROR = 2, ORC_RUNTIME_ERROR = 3, ORC_OTHER_ERROR = 4 };

typedef struct {
    int status;      /* which std:: exception type escaped minimize(), ORC_OK if none */
    char msg[200];   /* its what()                                                    */
    int niter;       /* return value of minimize()                                    */
    long nfev;       /* functor calls                                                 */
    double fx;       /* fx out-parameter                                              */
    double gnorm;    /* final_grad_norm()                                             */
    long trace_len;  /* number of fx values written to fx_trace (<= trace_cap)        */
    double seconds;  /* wall time of minimize() alone                                 */
} orc_result;

#define ORC_DECLARE(P)                                                                                         \
    ORC_API void P##default_param(orc_param* p, int lbfgsb);                                                           \
    /* LBFGSSolver<double, LS>::minimize; x in/out (n), grad_out (n) = final_grad() or NULL */                 \
    ORC_API int P##lbfgs_f64(int objective, const double* data0, const double* data1, long n, int ls,                  \
                     const orc_param* prm, int sum_mode, double* x, double* grad_out, double* fx_trace,        \
                     long trace_cap, orc_result* out);                                                         \
    ORC_API int P##lbfgs_f32(int objective, const float* data0, const float* data1, long n, int ls,                    \
                     const orc_param* prm, int sum_mode, float* x, float* grad_out, double* fx_trace,          \
                     long trace_cap, orc_result* out);                                                         \
    /* LBFGSBSolver<double>::minimize (MoreThuente) */                                                         \
    ORC_API int P##lbfgsb_f64(int objective, const double* data0, const double* data1, long n, const orc_param* prm,   \
                      int sum_mode, double* x, const double* lb, const double* ub, double* grad_out,           \
                      double* fx_trace, long trace_cap, orc_result* out);                                      \
    /* BFGSMat<double>: reset(n,m); add_correction(S[:,k], Y[:,k]) for k < npairs (column-major, ld = n);     \
       then res = a*H*v.  ys_out/theta_out optional (m values / 1 value). */                                   \
    ORC_API int P##bfgs_apply_Hv_f64(long n, int m, int npairs, const double* S, const double* Y, const double* v,     \
                             double a, int sum_mode, double* res, double* ys_out, double* theta_out);          \
    /* evaluate an objective once: returns fx, writes grad */                                                  \
    ORC_API double P##objective_f64(int objective, const double* data0, const double* data1, long n, const double* x,  \
                            double* grad);

ORC_DECLARE(orc_)
ORC_DECLARE(ref_)

/* restatement only: ONE line search from (xp, fx0 = f(xp), grad0 = f'(xp)) along drt with initial `step`, by the restated
 * ls_* function `ls`.  Outputs: accepted step, fx, dg, x (n), grad (n); returns ORC_* status; nfev / msg in `out`. */
ORC_API int orc_line_search_f64(int objective, const double* data0, const double* data1, long n, int ls, const orc_param* prm,
                        const double* xp, const double* drt, double step_max, double* step_inout, double* fx_out, double* dg_out,
                        double* x_out, double* grad_out, double* fx_trace, long trace_cap, orc_result* out);
/* restatement only: repeated apply_Hv timing for the CPU baseline (returns seconds per call) */
ORC_API double orc_bfgs_apply_Hv_bench_f64(long n, int m, int reps, int sum_mode, int threads);
/* restatement only: Gram-form (vector-free) two-loop used to study the fast GPU variant on CPU */
ORC_API int orc_lbfgs_gram_f64(int objective, const double* data0, const double* data1, long n, int ls,
                       const orc_param* prm, int sum_mode, double* x, double* grad_out, double* fx_trace,
                       long trace_cap, orc_result* out);

#ifdef __cplusplus
}
#endif
#endif
