// mock_abi_owlqn.cpp -- the host-memory TEST DOUBLE of the C ABI (mock_abi_box_hessian.cpp, included whole) plus host versions of the
// OWL-QN entries (lbfgs_b200_owlqn_*), so that include/OWLQN.h and the driver's lbfgsb200_drv_owlqn_* run on a CPU.  TEST
// INFRASTRUCTURE ONLY.  The element-wise steps use the product's expressions (include/LBFGSpp/OWLQNCore.h), as the kernels do; every
// sum is taken left to right in T, and the direction is the test double's literal two-loop recursion (orc::History::apply_Hv), so a
// run matches the checker (owlqn_oracle.hpp, ORC_SUM_SEQUENTIAL) bit for bit unless the front's logic differs from it.
//   trial        x = pi(xp + step d; xi); f, g at x; {f, |x|_1, pgp.(x - xp), pg.pg, x.x}
//   project      x = pi(xp + step d; xi); {|x|_1, pgp.(x - xp)}
//   sums         {|x|_1, pg.pg, x.x} (+ d = -pg)
//   update_dir   the gated pair update, d = -H pg, d_i = 0 where d_i pg_i >= 0, pg.d
// The refusals are the product's: lam not positive and finite, a history of the other precision.  The test double has no communicator,
// so it never sees a context with more than one rank.
#include "mock_abi_box_hessian.cpp"
#include "../../include/LBFGSpp/OWLQNCore.h"

namespace {

template <class T> lbfgs_b200_status owlqn_lam(lbfgs_b200_ctx* ctx, T lam)
{
    if (!(lam > T(0)) || !(lam <= std::numeric_limits<T>::max()))
        return fail(ctx, LBFGS_B200_ERR_INVALID, "owlqn: lambda must be positive and finite");
    return LBFGS_B200_OK;
}

// x = pi(xp + step d; xi) into x; out2 = {|x|_1, pgp.(x - xp)}
template <class T> void project_into(int64_t n, const T* xp, const T* d, const T* gp, T step, T lam, T* x, T* out2)
{
    T l1 = T(0), dirder = T(0);
    for (int64_t i = 0; i < n; i++)
    {
        const T pgp = LBFGSpp::owlqn_pg(xp[i], gp[i], lam);
        x[i] = LBFGSpp::owlqn_project(xp[i] + step * d[i], LBFGSpp::owlqn_orthant(xp[i], pgp));
        l1 += std::fabs(x[i]);
        dirder += pgp * (x[i] - xp[i]);
    }
    out2[0] = l1;
    out2[1] = dirder;
}

template <class T> void sums_into(int64_t n, const T* x, const T* g, T lam, T* d, T* out3)
{
    T l1 = T(0), pgpg = T(0), xx = T(0);
    for (int64_t i = 0; i < n; i++)
    {
        const T pg = LBFGSpp::owlqn_pg(x[i], g[i], lam);
        if (d) d[i] = -pg;
        l1 += std::fabs(x[i]);
        pgpg += pg * pg;
        xx += x[i] * x[i];
    }
    out3[0] = l1;
    out3[1] = pgpg;
    out3[2] = xx;
}

template <class T>
lbfgs_b200_status do_owlqn_trial(lbfgs_b200_ctx* ctx, int obj, const T* d0, const T* d1, int64_t n, const T* xp, const T* d, const T* gp,
                                 T step, T lam, T* x, T* g, T* out5)
{
    if (!ctx || !xp || !d || !gp || !x || !g || !out5 || n < 1) return fail(ctx, LBFGS_B200_ERR_INVALID, "owlqn_trial: bad arguments");
    if (auto st = owlqn_lam<T>(ctx, lam)) return st;
    T p[2], s[3], o4[4];
    project_into<T>(n, xp, d, gp, step, lam, x, p);
    if (auto st = do_objective<T>(ctx, obj, d0, d1, n, x, g, o4)) return st;
    sums_into<T>(n, x, g, lam, nullptr, s);
    out5[0] = o4[0]; out5[1] = p[0]; out5[2] = p[1]; out5[3] = s[1]; out5[4] = s[2];
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_owlqn_update_dir(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, T eps, T lam, T* d, int* acc, T* dg)
{
    if (auto st = check_hist<T>(h)) return st;
    if (!x || !xp || !g || !gp || !d || !dg) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "owlqn_update_dir: NULL argument");
    if (auto st = owlqn_lam<T>(h->ctx, lam)) return st;
    if (auto st = do_update<T>(h, x, xp, g, gp, eps, acc, nullptr)) return st;
    orc::History<T>& H = h->get<T>();
    std::vector<T> pg(H.n);
    for (long i = 0; i < H.n; i++) pg[i] = LBFGSpp::owlqn_pg(x[i], g[i], lam);
    H.apply_Hv(pg.data(), T(-1), d);
    T sum = T(0);
    for (long i = 0; i < H.n; i++)
    {
        d[i] = LBFGSpp::owlqn_constrain(d[i], pg[i]);
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
    { return do_owlqn_trial<T>(c, obj, d0, d1, n, xp, d, gp, step, lam, x, g, o5); }                                                  \
    lbfgs_b200_status lbfgs_b200_owlqn_project_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* xp, const T* d, const T* gp, T step,        \
                                                     T lam, T* x, T* o2)                                                              \
    {                                                                                                                                 \
        if (!c || !xp || !d || !gp || !x || !o2 || n < 1) return fail(c, LBFGS_B200_ERR_INVALID, "owlqn_project: bad arguments");       \
        if (auto st = owlqn_lam<T>(c, lam)) return st;                                                                                \
        project_into<T>(n, xp, d, gp, step, lam, x, o2);                                                                              \
        return LBFGS_B200_OK;                                                                                                         \
    }                                                                                                                                 \
    lbfgs_b200_status lbfgs_b200_owlqn_sums_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* x, const T* g, T lam, T* d, T* o3)            \
    {                                                                                                                                 \
        if (!c || !x || !g || !o3 || n < 1) return fail(c, LBFGS_B200_ERR_INVALID, "owlqn_sums: bad arguments");                      \
        if (auto st = owlqn_lam<T>(c, lam)) return st;                                                                                \
        sums_into<T>(n, x, g, lam, d, o3);                                                                                            \
        return LBFGS_B200_OK;                                                                                                         \
    }                                                                                                                                 \
    lbfgs_b200_status lbfgs_b200_owlqn_update_dir_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, T eps,   \
                                                        T lam, T* d, int* acc, T* dg)                                                 \
    { return do_owlqn_update_dir<T>(h, x, xp, g, gp, eps, lam, d, acc, dg); }

MOCK_OWLQN(double, f64)
MOCK_OWLQN(float, f32)

}  // extern "C"
