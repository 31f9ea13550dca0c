// mock_abi_owlqn.cpp -- the host-memory TEST DOUBLE of the C ABI (mock_abi_box_hessian.cpp, included whole) plus host versions of the
// OWL-QN entries, unweighted (lbfgs_b200_owlqn_*) and with per-coordinate weights (lbfgs_b200_owlqn_weighted_*), so that
// include/OWLQN.h and the driver's lbfgsb200_drv_owlqn_* run on a CPU.  TEST INFRASTRUCTURE ONLY.  The element-wise steps use the
// product's expressions (include/LBFGSpp/OWLQNCore.h), as the kernels do; every sum is taken left to right in T, and the direction is
// the test double's literal two-loop recursion (orc::History::apply_Hv), so a run matches the checker (owlqn_oracle.hpp,
// ORC_SUM_SEQUENTIAL) bit for bit unless the front's logic differs from it.
//   trial        lam_i = lam * w_i; x = owlqn_point_w; f, g at x; {f, sum w_i |x_i|, pgp.(x - xp), pg.pg, x.x}
//   project      x = owlqn_point_w; {sum w_i |x_i|, pgp.(x - xp)}
//   sums         {sum w_i |x_i|, pg.pg, x.x} (+ d = -pg); weighted: LBFGS_B200_ERR_INVALID when owlqn_weight_ok refuses a weight
//   update_dir   the gated pair update, d = -H pg, owlqn_constrain_w, pg.d
// The unweighted entries run the same code with w = nullptr, read as unit weights: lam * 1 == lam > 0 and 1 * |x_i| == |x_i|, so
// every coordinate is projected and constrained as by owlqn_point and owlqn_constrain, to the bit.
// The refusals are the product's: a NULL w at a weighted entry, lam not positive and finite, a history of the other precision, bad
// weights at the sums.  The test double has no communicator, so it never sees a context with more than one rank.
#include "mock_abi_box_hessian.cpp"
#include "../../include/LBFGSpp/OWLQNCore.h"

namespace {

// w_i, or 1 without weights
template <class T> T weight(const T* w, int64_t i) { return w ? w[i] : T(1); }

// refuses a NULL w at a weighted entry (what != nullptr names it), then a lam that is not positive and finite
template <class T> lbfgs_b200_status owlqn_check(lbfgs_b200_ctx* ctx, T lam, const T* w, const char* what)
{
    if (what && !w) return fail(ctx, LBFGS_B200_ERR_INVALID, (std::string(what) + ": NULL weights").c_str());
    if (!(lam > T(0)) || !(lam <= std::numeric_limits<T>::max()))
        return fail(ctx, LBFGS_B200_ERR_INVALID, "owlqn: lambda must be positive and finite");
    return LBFGS_B200_OK;
}

// x = owlqn_point_w into x; out2 = {sum w_i |x_i|, pgp.(x - xp)}
template <class T> void project_into(int64_t n, const T* xp, const T* d, const T* gp, T step, T lam, const T* w, T* x, T* out2)
{
    T l1 = T(0), dirder = T(0);
    for (int64_t i = 0; i < n; i++)
    {
        const T lk = LBFGSpp::owlqn_lam_i(lam, weight(w, i));
        const T pgp = LBFGSpp::owlqn_pg(xp[i], gp[i], lk);
        x[i] = LBFGSpp::owlqn_point_w(xp[i], d[i], gp[i], step, lk);
        l1 += weight(w, i) * std::fabs(x[i]);
        dirder += pgp * (x[i] - xp[i]);
    }
    out2[0] = l1;
    out2[1] = dirder;
}

// returns the number of weights owlqn_weight_ok refuses (0 without weights)
template <class T> long sums_into(int64_t n, const T* x, const T* g, T lam, const T* w, T* d, T* out3)
{
    T l1 = T(0), pgpg = T(0), xx = T(0);
    long bad = 0;
    for (int64_t i = 0; i < n; i++)
    {
        const T pg = LBFGSpp::owlqn_pg(x[i], g[i], LBFGSpp::owlqn_lam_i(lam, weight(w, i)));
        if (d) d[i] = -pg;
        bad += LBFGSpp::owlqn_weight_ok(lam, weight(w, i)) ? 0 : 1;
        l1 += weight(w, i) * std::fabs(x[i]);
        pgpg += pg * pg;
        xx += x[i] * x[i];
    }
    out3[0] = l1;
    out3[1] = pgpg;
    out3[2] = xx;
    return bad;
}

template <class T>
lbfgs_b200_status do_owlqn_trial(lbfgs_b200_ctx* ctx, int obj, const T* d0, const T* d1, int64_t n, const T* xp, const T* d, const T* gp,
                                 T step, T lam, const T* w, const char* weighted, T* x, T* g, T* out5)
{
    if (!ctx || !xp || !d || !gp || !x || !g || !out5 || n < 1) return fail(ctx, LBFGS_B200_ERR_INVALID, "owlqn_trial: bad arguments");
    if (auto st = owlqn_check<T>(ctx, lam, w, weighted)) return st;
    T p[2], s[3], o4[4];
    project_into<T>(n, xp, d, gp, step, lam, w, x, p);
    if (auto st = do_objective<T>(ctx, obj, d0, d1, n, x, g, o4)) return st;
    sums_into<T>(n, x, g, lam, w, nullptr, s);
    out5[0] = o4[0]; out5[1] = p[0]; out5[2] = p[1]; out5[3] = s[1]; out5[4] = s[2];
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_owlqn_project(lbfgs_b200_ctx* ctx, int64_t n, const T* xp, const T* d, const T* gp, T step, T lam, const T* w,
                                   const char* weighted, T* x, T* out2)
{
    if (!ctx || !xp || !d || !gp || !x || !out2 || n < 1) return fail(ctx, LBFGS_B200_ERR_INVALID, "owlqn_project: bad arguments");
    if (auto st = owlqn_check<T>(ctx, lam, w, weighted)) return st;
    project_into<T>(n, xp, d, gp, step, lam, w, x, out2);
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_owlqn_sums(lbfgs_b200_ctx* ctx, int64_t n, const T* x, const T* g, T lam, const T* w, const char* weighted, T* d, T* out3)
{
    if (!ctx || !x || !g || !out3 || n < 1) return fail(ctx, LBFGS_B200_ERR_INVALID, "owlqn_sums: bad arguments");
    if (auto st = owlqn_check<T>(ctx, lam, w, weighted)) return st;
    if (const long bad = sums_into<T>(n, x, g, lam, w, d, out3))
        return fail(ctx, LBFGS_B200_ERR_INVALID, ("owlqn_weighted_sums: " + std::to_string(bad) +
                                                  " weights are negative, not finite, or make lambda * w overflow").c_str());
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_owlqn_update_dir(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, T eps, T lam, const T* w,
                                      const char* weighted, T* d, int* acc, T* dg)
{
    if (auto st = check_hist<T>(h)) return st;
    if (!x || !xp || !g || !gp || !d || !dg) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "owlqn_update_dir: NULL argument");
    if (auto st = owlqn_check<T>(h->ctx, lam, w, weighted)) return st;
    if (auto st = do_update<T>(h, x, xp, g, gp, eps, acc, nullptr)) return st;
    orc::History<T>& H = h->get<T>();
    std::vector<T> pg(H.n), lw(H.n);
    for (long i = 0; i < H.n; i++)
    {
        lw[i] = LBFGSpp::owlqn_lam_i(lam, weight(w, i));
        pg[i] = LBFGSpp::owlqn_pg(x[i], g[i], lw[i]);
    }
    H.apply_Hv(pg.data(), T(-1), d);
    T sum = T(0);
    for (long i = 0; i < H.n; i++)
    {
        d[i] = LBFGSpp::owlqn_constrain_w(d[i], pg[i], lw[i]);
        sum += pg[i] * d[i];
    }
    *dg = sum;
    return LBFGS_B200_OK;
}

}  // namespace

extern "C" {

#define MOCK_OWLQN(T, SUF)                                                                                                            \
    lbfgs_b200_status lbfgs_b200_owlqn_trial_##SUF(lbfgs_b200_ctx* c, int obj, const T* d0, const T* d1, int64_t n, const T* xp,        \
                                                   const T* d, const T* gp, T step, T lam, T* x, T* g, T* o5)                         \
    { return do_owlqn_trial<T>(c, obj, d0, d1, n, xp, d, gp, step, lam, nullptr, nullptr, x, g, o5); }                                \
    lbfgs_b200_status lbfgs_b200_owlqn_project_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* xp, const T* d, const T* gp, T step,        \
                                                     T lam, T* x, T* o2)                                                              \
    { return do_owlqn_project<T>(c, n, xp, d, gp, step, lam, nullptr, nullptr, x, o2); }                                              \
    lbfgs_b200_status lbfgs_b200_owlqn_sums_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* x, const T* g, T lam, T* d, T* o3)            \
    { return do_owlqn_sums<T>(c, n, x, g, lam, nullptr, nullptr, d, o3); }                                                            \
    lbfgs_b200_status lbfgs_b200_owlqn_update_dir_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, T eps,   \
                                                        T lam, T* d, int* acc, T* dg)                                                 \
    { return do_owlqn_update_dir<T>(h, x, xp, g, gp, eps, lam, nullptr, nullptr, d, acc, dg); }                                       \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_trial_##SUF(lbfgs_b200_ctx* c, int obj, const T* d0, const T* d1, int64_t n,          \
                                                            const T* xp, const T* d, const T* gp, T step, T lam, const T* w, T* x,   \
                                                            T* g, T* o5)                                                               \
    { return do_owlqn_trial<T>(c, obj, d0, d1, n, xp, d, gp, step, lam, w, "owlqn_weighted_trial", x, g, o5); }                       \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_project_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* xp, const T* d, const T* gp,      \
                                                              T step, T lam, const T* w, T* x, T* o2)                                  \
    { return do_owlqn_project<T>(c, n, xp, d, gp, step, lam, w, "owlqn_weighted_project", x, o2); }                                   \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_sums_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* x, const T* g, T lam, const T* w,    \
                                                           T* d, T* o3)                                                                \
    { return do_owlqn_sums<T>(c, n, x, g, lam, w, "owlqn_weighted_sums", d, o3); }                                                    \
    lbfgs_b200_status lbfgs_b200_owlqn_weighted_update_dir_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, \
                                                                 T eps, T lam, const T* w, T* d, int* acc, T* dg)                     \
    { return do_owlqn_update_dir<T>(h, x, xp, g, gp, eps, lam, w, "owlqn_weighted_update_dir", d, acc, dg); }

MOCK_OWLQN(double, f64)
MOCK_OWLQN(float, f32)

}  // extern "C"
