// mock_abi.cpp -- TEST DOUBLE of the C ABI (include/lbfgs_b200.h) on host memory.  TEST INFRASTRUCTURE ONLY.
//
// Purpose: run the product's header-only front (include/LBFGS.h, LBFGSpp/*.h: the solver loop, the line-search drivers and
// state machines, DeviceVector, the objective adapters, the host-functor compatibility mode) on a machine without a GPU, so
// that tests/test_front_cpu.py can hold that host logic to the CPU checker bit for bit.  Every "device" pointer is a host
// pointer; every sum is taken strictly left to right with the CPU checker's own routines (oracle/lbfgs_oracle.hpp), so any
// difference from the checker is a difference in the front's logic, not in rounding.
//
// This is NOT a backend of the product: it lives under tests/, is linked only into tests/cpp/front_harness.so, ignores the
// apply_Hv algorithm selector (always the literal recursion) and has no device-resident solve and no communicator (those return
// an error).  The bound-constrained entry points restate the semantics of lbfgspp_b200/csrc/lbfgsb_kernels.cuh with plain loops
// (the breakpoint sweep walks the sorted positions one by one and evaluates the same closed forms at every tie-group end).  The product library refuses to run without a CUDA device (tests/test_abi_cpu.py).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <limits>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/lbfgs_b200.h"
#include "../../oracle/lbfgs_oracle.hpp"
#include "../../oracle/objectives.hpp"

struct lbfgs_b200_ctx
{
    std::string err;
    uint64_t calls = 0;
    int64_t index_offset = 0;
};

struct lbfgs_b200_hist
{
    lbfgs_b200_ctx* ctx;
    int elem;
    std::unique_ptr<orc::History<double> > h64;
    std::unique_ptr<orc::History<float> > h32;
    std::vector<double> s64, y64;
    std::vector<float> s32, y32;
    template <class T> orc::History<T>& get();
    template <class T> std::vector<T>& sbuf();
    template <class T> std::vector<T>& ybuf();
};
template <> orc::History<double>& lbfgs_b200_hist::get<double>() { return *h64; }
template <> orc::History<float>& lbfgs_b200_hist::get<float>() { return *h32; }
template <> std::vector<double>& lbfgs_b200_hist::sbuf<double>() { return s64; }
template <> std::vector<float>& lbfgs_b200_hist::sbuf<float>() { return s32; }
template <> std::vector<double>& lbfgs_b200_hist::ybuf<double>() { return y64; }
template <> std::vector<float>& lbfgs_b200_hist::ybuf<float>() { return y32; }

// workspace of the bound-constrained path: the n-vectors of lbfgsb_impl.cuh (LBFGS_B200_BOXV_* order) and the class bytes
struct lbfgs_b200_box
{
    lbfgs_b200_hist* h;
    int64_t n;
    std::vector<unsigned char> cls;
    std::vector<double> v64[10];
    std::vector<float> v32[10];
    template <class T> T* vec(int which);
};
template <> double* lbfgs_b200_box::vec<double>(int which) { return v64[which].data(); }
template <> float* lbfgs_b200_box::vec<float>(int which) { return v32[which].data(); }
struct lbfgs_b200_solver { int unused; };

namespace {

std::string g_last_error;

lbfgs_b200_status fail(lbfgs_b200_ctx* ctx, lbfgs_b200_status st, const char* what)
{
    (ctx ? ctx->err : g_last_error) = what;
    return st;
}
lbfgs_b200_status unsupported(lbfgs_b200_ctx* ctx, const char* what)
{
    return fail(ctx, LBFGS_B200_ERR_INVALID, (std::string("test double: ") + what + " is not provided").c_str());
}

const orc::Blas1<double> kSeq64(ORC_SUM_SEQUENTIAL, 1);
const orc::Blas1<float> kSeq32(ORC_SUM_SEQUENTIAL, 1);
template <class T> const orc::Blas1<T>& seq();
template <> const orc::Blas1<double>& seq<double>() { return kSeq64; }
template <> const orc::Blas1<float>& seq<float>() { return kSeq32; }

template <class T>
lbfgs_b200_status do_objective(lbfgs_b200_ctx* ctx, int objective, const T* d0, const T* d1, int64_t n, const T* x, T* g, T* out4)
{
    if (!ctx || !x || !g || !out4 || n < 1) return fail(ctx, LBFGS_B200_ERR_INVALID, "objective: bad arguments");
    if (objective == LBFGS_B200_OBJ_ROSENBROCK_PAIRED && n % 2) return fail(ctx, LBFGS_B200_ERR_INVALID, "paired Rosenbrock needs an even n");
    ctx->calls++;
    out4[0] = orc::evaluate<T>(objective, d0, d1, long(n), x, g);
    out4[1] = T(0);
    out4[2] = seq<T>().dot(g, g, long(n));
    out4[3] = seq<T>().dot(x, x, long(n));
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_trial(lbfgs_b200_ctx* ctx, int objective, const T* d0, const T* d1, int64_t n, const T* xp, const T* d, T step, T* x,
                           T* g, T* out4)
{
    if (!ctx || !xp || !d || !x || !g || !out4 || n < 1) return fail(ctx, LBFGS_B200_ERR_INVALID, "trial: bad arguments");
    for (int64_t i = 0; i < n; i++) x[i] = xp[i] + step * d[i];
    if (auto st = do_objective<T>(ctx, objective, d0, d1, n, x, g, out4)) return st;
    out4[1] = seq<T>().dot(g, d, long(n));
    return LBFGS_B200_OK;
}

template <class T> lbfgs_b200_status check_hist(lbfgs_b200_hist* h)
{
    if (!h) return LBFGS_B200_ERR_INVALID;
    if (h->elem != int(sizeof(T))) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "history element size mismatch");
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_update(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, T eps, int* accepted, T* sy_yy)
{
    if (auto st = check_hist<T>(h)) return st;
    orc::History<T>& H = h->get<T>();
    std::vector<T>& s = h->sbuf<T>();
    std::vector<T>& y = h->ybuf<T>();
    seq<T>().diff(s.data(), x, xp, H.n);
    seq<T>().diff(y.data(), g, gp, H.n);
    const T sy = seq<T>().dot(s.data(), y.data(), H.n), yy = seq<T>().sqnorm(y.data(), H.n);
    const bool ok = sy > eps * yy;   // LBFGS.h:161
    if (ok) H.add(s.data(), y.data());
    if (accepted) *accepted = ok ? 1 : 0;
    if (sy_yy) { sy_yy[0] = sy; sy_yy[1] = yy; }
    h->ctx->calls++;
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_apply_Hv(lbfgs_b200_hist* h, const T* v, T a, T* res, T* vdot)
{
    if (auto st = check_hist<T>(h)) return st;
    if (!v || !res || v == res) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "apply_Hv: v/res NULL or aliased");
    orc::History<T>& H = h->get<T>();
    H.apply_Hv(v, a, res);
    if (vdot) *vdot = seq<T>().dot(v, res, H.n);
    h->ctx->calls++;
    return LBFGS_B200_OK;
}

template <class T> const void* column(const lbfgs_b200_hist* h, bool s, int age)
{
    orc::History<T>& H = const_cast<lbfgs_b200_hist*>(h)->get<T>();
    if (age < 0 || age >= H.ncorr) return nullptr;
    const int slot = ((H.ptr - 1 - age) % H.m + H.m) % H.m;
    return s ? H.s_col(slot) : H.y_col(slot);
}

// the c x c Gram blocks by age and W'v: shared by the dense B / H accessors (final_approx_hessian) and L-BFGS-B
template <class T>
lbfgs_b200_status do_gram(lbfgs_b200_hist* h, T* SY, T* SS, T* YY, T* ys, T* theta)
{
    if (auto st = check_hist<T>(h)) return st;
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr;
    for (int i = 0; i < c; i++)
    {
        const T* si = static_cast<const T*>(column<T>(h, true, i));
        const T* yi = static_cast<const T*>(column<T>(h, false, i));
        for (int j = 0; j < c; j++)
        {
            const T* sj = static_cast<const T*>(column<T>(h, true, j));
            const T* yj = static_cast<const T*>(column<T>(h, false, j));
            if (SY) SY[i * c + j] = seq<T>().dot(si, yj, H.n);
            if (SS) SS[i * c + j] = seq<T>().dot(si, sj, H.n);
            if (YY) YY[i * c + j] = seq<T>().dot(yi, yj, H.n);
        }
        if (ys) ys[i] = H.ys[((H.ptr - 1 - i) % H.m + H.m) % H.m];
    }
    if (theta) *theta = H.theta;
    return LBFGS_B200_OK;
}
template <class T>
lbfgs_b200_status do_wt_dot(lbfgs_b200_hist* h, const T* v, T* raw)
{
    if (auto st = check_hist<T>(h)) return st;
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr;
    for (int i = 0; i < c; i++)
    {
        raw[i] = seq<T>().dot(static_cast<const T*>(column<T>(h, false, i)), v, H.n);
        raw[c + i] = seq<T>().dot(static_cast<const T*>(column<T>(h, true, i)), v, H.n);
    }
    return LBFGS_B200_OK;
}

// ---- bound-constrained primitives: the semantics of lbfgspp_b200/csrc/lbfgsb_kernels.cuh, one coordinate after the other ----------
enum : unsigned char { CLS_FIXED = 1, CLS_ACT = 2, CLS_FREE = 4, SUB_L = 8, SUB_U = 16, SUB_P = 32 };
enum { V_VECC = 0, V_VECY = 1, V_LAMBDA = 2, V_MU = 3, V_TMP = 4, V_TMP2 = 5, V_YFB = 6, V_DVEC = 7, V_BRK = 8, V_XCP = 9 };

template <class T> lbfgs_b200_status check_box(lbfgs_b200_box* b)
{
    if (!b || !b->h) return LBFGS_B200_ERR_INVALID;
    return check_hist<T>(b->h);
}

template <class T>
lbfgs_b200_status do_lincomb(lbfgs_b200_hist* h, T a0, const T* v0, const T* coef, const unsigned char* cls, int mask, T* out)
{
    if (auto st = check_hist<T>(h)) return st;
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr;
    if (!out || (c > 0 && !coef)) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "hist_lincomb: NULL argument");
    for (long i = 0; i < H.n; i++)
    {
        if (cls && !(cls[i] & mask)) continue;
        T r = v0 ? a0 * v0[i] : T(0);
        for (int j = 0; j < c; j++) r += coef[j] * static_cast<const T*>(column<T>(h, false, j))[i];
        for (int j = 0; j < c; j++) r += coef[c + j] * static_cast<const T*>(column<T>(h, true, j))[i];
        out[i] = r;
    }
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_masked_gram(lbfgs_b200_hist* h, const unsigned char* cls, int mask, T* G)
{
    if (auto st = check_hist<T>(h)) return st;
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr, w = 2 * c;
    std::vector<const T*> col(static_cast<size_t>(w));
    for (int j = 0; j < c; j++) { col[j] = static_cast<const T*>(column<T>(h, false, j)); col[c + j] = static_cast<const T*>(column<T>(h, true, j)); }
    for (int a = 0; a < w; a++)
        for (int b = 0; b < w; b++)
        {
            T acc = T(0);
            for (long i = 0; i < H.n; i++)
                if (!cls || (cls[i] & mask)) acc += col[a][i] * col[b][i];
            G[a * w + b] = acc;
        }
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_cauchy_breaks(lbfgs_b200_box* b, const T* x, const T* g, const T* lb, const T* ub, T* out5)
{
    if (auto st = check_box<T>(b)) return st;
    T* brk = b->vec<T>(V_BRK);
    T* dvec = b->vec<T>(V_DVEC);
    const T inf = std::numeric_limits<T>::infinity();
    double nfixed = 0, ninf = 0, nord = 0, dd = 0;   // d.d accumulated in double, as k_cauchy_breaks does
    T tmin = inf;
    for (int64_t i = 0; i < b->n; i++)
    {
        T t;
        if (lb[i] == ub[i]) t = T(0);
        else if (g[i] < T(0)) t = (x[i] - ub[i]) / g[i];
        else if (g[i] > T(0)) t = (x[i] - lb[i]) / g[i];
        else t = inf;
        const bool zero = (t == T(0));
        const T di = zero ? T(0) : -g[i];
        brk[i] = t;
        dvec[i] = di;
        dd += double(di * di);
        if (t == inf) { ninf += 1; b->cls[i] = CLS_FREE; }
        else if (!zero) { nord += 1; tmin = std::min(tmin, t); b->cls[i] = 0; }
        else { nfixed += 1; b->cls[i] = CLS_FIXED; }
    }
    out5[0] = T(nfixed); out5[1] = T(ninf); out5[2] = T(nord); out5[3] = T(dd); out5[4] = tmin;
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_cauchy_sweep(lbfgs_b200_box* b, const T* g, const T* Mmat, const T* p0, T theta, T gt, int64_t nord, int64_t nfree_inf,
                                  T* out)
{
    if (auto st = check_box<T>(b)) return st;
    lbfgs_b200_hist* h = b->h;
    orc::History<T>& H = h->get<T>();
    const int c = H.ncorr, w = 2 * c;
    const T* brk = b->vec<T>(V_BRK);
    std::vector<int64_t> ord;
    for (int64_t i = 0; i < b->n; i++)
        if (b->cls[i] == 0) ord.push_back(i);
    if (int64_t(ord.size()) != nord || nord < 1) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "cauchy_sweep: nord does not match the classes");
    std::sort(ord.begin(), ord.end(), [brk](int64_t a, int64_t bb) { return brk[a] < brk[bb] || (brk[a] == brk[bb] && a < bb); });
    std::vector<const T*> ycol(static_cast<size_t>(c)), scol(static_cast<size_t>(c));
    for (int j = 0; j < c; j++) { ycol[j] = static_cast<const T*>(column<T>(h, false, j)); scol[j] = static_cast<const T*>(column<T>(h, true, j)); }
    // running prefix sums: G = sum g^2 ; A[2c] = sum g*w ; C[2c] = sum t*g*w  with w = (y_j[i], theta*s_j[i]) by age
    T G = T(0);
    std::vector<T> A(static_cast<size_t>(w), T(0)), Cc(static_cast<size_t>(w), T(0)), pvec(static_cast<size_t>(w)), cvec(static_cast<size_t>(w));
    const T inf = std::numeric_limits<T>::infinity();
    for (int64_t k = 0; k < nord; k++)
    {
        const int64_t i = ord[k];
        const T gi = g[i], t = brk[i];
        G += gi * gi;
        for (int j = 0; j < c; j++)
        {
            const T wy = ycol[j][i], ws = theta * scol[j][i];
            A[j] += gi * wy;
            A[c + j] += gi * ws;
            Cc[j] += t * gi * wy;
            Cc[c + j] += t * gi * ws;
        }
        const bool last = (k + 1 == nord);
        const T tnext = last ? inf : brk[ord[k + 1]];
        if (!last && tnext == t) continue;   // not the end of its tie group
        // quantities at the start of the segment that follows position k
        const T rest = gt - G;
        for (int q = 0; q < w; q++) { pvec[q] = p0[q] + A[q]; cvec[q] = t * pvec[q] - Cc[q]; }
        T pMc = T(0), pMp = T(0);
        for (int r = 0; r < w; r++)
        {
            T mc = T(0), mp = T(0);
            for (int q = 0; q < w; q++) { mc += Mmat[r * w + q] * cvec[q]; mp += Mmat[r * w + q] * pvec[q]; }
            pMc += pvec[r] * mc;
            pMp += pvec[r] * mp;
        }
        const T fp = -rest * (T(1) - theta * t) - pMc;
        const T fpp = theta * rest - pMp;
        T dtmin = -fp / fpp;
        const T dt = tnext - t;
        const bool all_crossed = last && nfree_inf == 0;
        if ((dtmin >= dt) && !all_crossed) continue;   // Cauchy.h:183: keep sweeping
        const T eps = std::numeric_limits<T>::epsilon();
        if (fpp < eps) dtmin = -fp / eps;
        dtmin = std::max(dtmin, T(0));
        if (all_crossed) dtmin = T(0);
        out[0] = t; out[1] = t + dtmin; out[2] = fp; out[3] = fpp; out[4] = all_crossed ? T(1) : T(0);
        for (int q = 0; q < w; q++) out[5 + q] = cvec[q] + dtmin * pvec[q];
        return LBFGS_B200_OK;
    }
    return fail(h->ctx, LBFGS_B200_ERR_INVALID, "cauchy sweep found no segment (internal error)");
}

template <class T>
lbfgs_b200_status do_cauchy_build(lbfgs_b200_box* b, const T* x, const T* lb, const T* ub, T t_cross, T tfinal, T* counts2)
{
    if (auto st = check_box<T>(b)) return st;
    const T* brk = b->vec<T>(V_BRK);
    const T* dvec = b->vec<T>(V_DVEC);
    T* xcp = b->vec<T>(V_XCP);
    double nact = 0, nfree = 0;
    for (int64_t i = 0; i < b->n; i++)
    {
        const unsigned char c0 = b->cls[i];
        T out = x[i];
        unsigned char c1 = c0;
        if (c0 != CLS_FIXED)
        {
            const bool crossed = (c0 != CLS_FREE) && (brk[i] <= t_cross);
            if (crossed) { out = (dvec[i] > T(0)) ? ub[i] : lb[i]; c1 = CLS_ACT; nact += 1; }
            else { out = x[i] + tfinal * dvec[i]; c1 = CLS_FREE; nfree += 1; }
        }
        xcp[i] = out;
        b->cls[i] = c1;
    }
    counts2[0] = T(nact); counts2[1] = T(nfree);
    return LBFGS_B200_OK;
}

template <class T>
lbfgs_b200_status do_sub_step(lbfgs_b200_box* b, int op, int flag, const T* x0, const T* g, const T* lb, const T* ub, T* drt, T theta, T* out3)
{
    if (auto st = check_box<T>(b)) return st;
    T *vecc = b->vec<T>(V_VECC), *vecy = b->vec<T>(V_VECY), *lambda = b->vec<T>(V_LAMBDA), *mu = b->vec<T>(V_MU), *tmp = b->vec<T>(V_TMP),
      *tmp2 = b->vec<T>(V_TMP2), *yfb = b->vec<T>(V_YFB), *xcp = b->vec<T>(V_XCP);
    double c0 = 0, c1 = 0, c2 = 0;
    T dotacc = T(0);
    for (int64_t i = 0; i < b->n; i++)
    {
        const unsigned char c = b->cls[i];
        const bool is_free = (c & CLS_FREE) != 0;
        switch (op)
        {
        case LBFGS_B200_SUB_INIT: drt[i] = xcp[i] - x0[i]; lambda[i] = mu[i] = vecc[i] = vecy[i] = T(0); break;
        case LBFGS_B200_SUB_ACT_DIR: tmp[i] = (c & CLS_ACT) ? (xcp[i] - x0[i]) : T(0); break;
        case LBFGS_B200_SUB_ADD_G: if (is_free) vecc[i] += g[i]; break;
        case LBFGS_B200_SUB_NEG_C_FREE: tmp[i] = is_free ? -vecc[i] : T(0); break;
        case LBFGS_B200_SUB_CHECK_BOUNDS:
            if (is_free && (vecy[i] < lb[i] - x0[i] || vecy[i] > ub[i] - x0[i])) c0 += 1;
            break;
        case LBFGS_B200_SUB_CLASSIFY:
            if (is_free)
            {
                const T l = lb[i] - x0[i], u = ub[i] - x0[i], y = vecy[i];
                unsigned char nc = c & static_cast<unsigned char>(~(SUB_L | SUB_U | SUB_P));
                if ((y < l) || (y == l && lambda[i] >= T(0))) { nc |= SUB_L; vecy[i] = l; mu[i] = T(0); c0 += 1; }
                else if ((y > u) || (y == u && mu[i] >= T(0))) { nc |= SUB_U; vecy[i] = u; lambda[i] = T(0); c1 += 1; }
                else { nc |= SUB_P; lambda[i] = T(0); mu[i] = T(0); c2 += 1; }
                b->cls[i] = nc;
            }
            break;
        case LBFGS_B200_SUB_LU_VEC: tmp[i] = (c & SUB_L) ? (lb[i] - x0[i]) : ((c & SUB_U) ? (ub[i] - x0[i]) : T(0)); break;
        case LBFGS_B200_SUB_RHS_P: tmp[i] = (c & SUB_P) ? -(vecc[i] + (flag ? tmp2[i] : T(0))) : T(0); break;
        case LBFGS_B200_SUB_FREE_VEC: tmp[i] = is_free ? vecy[i] : T(0); break;
        case LBFGS_B200_SUB_MULTIPLIERS:
            if (c & SUB_L) lambda[i] = tmp2[i] + vecc[i] + theta * vecy[i];
            if (c & SUB_U) mu[i] = -(tmp2[i] + vecc[i] + theta * vecy[i]);
            break;
        case LBFGS_B200_SUB_CONVERGED:
            if (is_free && (c & SUB_L) && lambda[i] < T(0)) c0 += 1;
            if (is_free && (c & SUB_U) && mu[i] < T(0)) c1 += 1;
            if (is_free && (c & SUB_P) && (vecy[i] < lb[i] - x0[i] || vecy[i] > ub[i] - x0[i])) c2 += 1;
            break;
        case LBFGS_B200_SUB_WRITE_DRT:
            if (is_free)
            {
                T y = (flag & 2) ? yfb[i] : vecy[i];
                if (flag & 1) y = std::min(std::max(y, lb[i] - x0[i]), ub[i] - x0[i]);
                drt[i] = y;
            }
            dotacc += drt[i] * g[i];
            break;
        default: return fail(b->h->ctx, LBFGS_B200_ERR_INVALID, "box_sub_step: unknown op");
        }
    }
    if (op == LBFGS_B200_SUB_WRITE_DRT) c0 = double(dotacc);
    if (out3) { out3[0] = T(c0); out3[1] = T(c1); out3[2] = T(c2); }
    return LBFGS_B200_OK;
}

}  // namespace

extern "C" {

const char* lbfgs_b200_version(void) { return "lbfgs_b200 test double (host memory, sequential sums)"; }
lbfgs_b200_status lbfgs_b200_ctx_create(lbfgs_b200_ctx** out, int, void*)
{
    if (!out) return fail(nullptr, LBFGS_B200_ERR_INVALID, "ctx_create: NULL out");
    *out = new lbfgs_b200_ctx();
    return LBFGS_B200_OK;
}
void lbfgs_b200_ctx_destroy(lbfgs_b200_ctx* ctx) { delete ctx; }
const char* lbfgs_b200_last_error(const lbfgs_b200_ctx* ctx) { return ctx ? ctx->err.c_str() : g_last_error.c_str(); }
void* lbfgs_b200_stream(const lbfgs_b200_ctx*) { return nullptr; }
int lbfgs_b200_sm_count(const lbfgs_b200_ctx*) { return 1; }
uint64_t lbfgs_b200_launch_count(const lbfgs_b200_ctx* ctx) { return ctx ? ctx->calls : 0; }

lbfgs_b200_status lbfgs_b200_malloc(lbfgs_b200_ctx* ctx, void** p, size_t bytes)
{
    if (!ctx || !p) return fail(ctx, LBFGS_B200_ERR_INVALID, "malloc: NULL argument");
    *p = std::aligned_alloc(256, (bytes + 255) / 256 * 256 + 256);
    return *p ? LBFGS_B200_OK : fail(ctx, LBFGS_B200_ERR_ALLOC, "out of memory");
}
lbfgs_b200_status lbfgs_b200_free(lbfgs_b200_ctx*, void* p) { std::free(p); return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_trim(lbfgs_b200_ctx*) { return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_malloc_host(lbfgs_b200_ctx* ctx, void** p, size_t bytes) { return lbfgs_b200_malloc(ctx, p, bytes); }
lbfgs_b200_status lbfgs_b200_free_host(lbfgs_b200_ctx*, void* p) { std::free(p); return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_memcpy_h2d(lbfgs_b200_ctx*, void* d, const void* s, size_t b) { std::memcpy(d, s, b); return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_memcpy_d2h(lbfgs_b200_ctx*, void* d, const void* s, size_t b) { std::memcpy(d, s, b); return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_memcpy_d2d(lbfgs_b200_ctx*, void* d, const void* s, size_t b) { std::memmove(d, s, b); return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_memset_zero(lbfgs_b200_ctx*, void* d, size_t b) { std::memset(d, 0, b); return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_sync(lbfgs_b200_ctx*) { return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_timer_start(lbfgs_b200_ctx*) { return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_timer_stop(lbfgs_b200_ctx*, float* ms) { if (ms) *ms = 0.f; return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_profile_enable(lbfgs_b200_ctx*, int) { return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_profile_read(lbfgs_b200_ctx*, int, double* ms, uint64_t* calls, int)
{
    if (ms) *ms = 0;
    if (calls) *calls = 0;
    return LBFGS_B200_OK;
}
lbfgs_b200_status lbfgs_b200_profile_bytes(lbfgs_b200_ctx*, int, double* b, int) { if (b) *b = 0; return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_set_index_offset(lbfgs_b200_ctx* ctx, int64_t off) { ctx->index_offset = off; return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_set_global_extent(lbfgs_b200_ctx* ctx, int64_t off, int64_t) { ctx->index_offset = off; return LBFGS_B200_OK; }
lbfgs_b200_status lbfgs_b200_comm_unique_id(void*) { return unsupported(nullptr, "a communicator"); }
lbfgs_b200_status lbfgs_b200_comm_init(lbfgs_b200_ctx* c, const void*, int, int) { return unsupported(c, "a communicator"); }
int lbfgs_b200_comm_size(const lbfgs_b200_ctx*) { return 1; }
lbfgs_b200_status lbfgs_b200_comm_p2p_export(lbfgs_b200_ctx* c, void*) { return unsupported(c, "a communicator"); }
lbfgs_b200_status lbfgs_b200_comm_p2p_attach(lbfgs_b200_ctx* c, const void*, int, int) { return unsupported(c, "a communicator"); }

#define MOCK_L1(T, SUF)                                                                                                          \
    lbfgs_b200_status lbfgs_b200_dot_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* a, const T* b, T* o)                           \
    { c->calls++; *o = seq<T>().dot(a, b, long(n)); return LBFGS_B200_OK; }                                                      \
    lbfgs_b200_status lbfgs_b200_dot3_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* g, const T* d, const T* x, T* o)              \
    { c->calls++; o[0] = seq<T>().dot(g, d, long(n)); o[1] = seq<T>().dot(g, g, long(n)); o[2] = seq<T>().dot(x, x, long(n)); return LBFGS_B200_OK; } \
    lbfgs_b200_status lbfgs_b200_axpy_out_##SUF(lbfgs_b200_ctx* c, int64_t n, const T* a, T s, const T* b, T* o)                 \
    { c->calls++; for (int64_t i = 0; i < n; i++) o[i] = a[i] + s * b[i]; return LBFGS_B200_OK; }                                \
    lbfgs_b200_status lbfgs_b200_scale_out_##SUF(lbfgs_b200_ctx* c, int64_t n, T s, const T* a, T* o)                            \
    { c->calls++; for (int64_t i = 0; i < n; i++) o[i] = s * a[i]; return LBFGS_B200_OK; }                                       \
    lbfgs_b200_status lbfgs_b200_objective_##SUF(lbfgs_b200_ctx* c, int obj, const T* d0, const T* d1, int64_t n, const T* x, T* g, T* o4) \
    { return do_objective<T>(c, obj, d0, d1, n, x, g, o4); }                                                                     \
    lbfgs_b200_status lbfgs_b200_trial_##SUF(lbfgs_b200_ctx* c, int obj, const T* d0, const T* d1, int64_t n, const T* xp,       \
                                             const T* d, T step, T* x, T* g, T* o4)                                              \
    { return do_trial<T>(c, obj, d0, d1, n, xp, d, step, x, g, o4); }
MOCK_L1(double, f64)
MOCK_L1(float, f32)

lbfgs_b200_status lbfgs_b200_hist_create(lbfgs_b200_ctx* ctx, lbfgs_b200_hist** out, int64_t n, int m, int elem)
{
    if (!ctx || !out || n < 1 || m < 1 || (elem != 4 && elem != 8)) return fail(ctx, LBFGS_B200_ERR_INVALID, "hist_create: bad arguments");
    lbfgs_b200_hist* h = new lbfgs_b200_hist();
    h->ctx = ctx;
    h->elem = elem;
    if (elem == 8) { h->h64.reset(new orc::History<double>(kSeq64)); h->h64->reset(long(n), m); h->s64.resize(n); h->y64.resize(n); }
    else { h->h32.reset(new orc::History<float>(kSeq32)); h->h32->reset(long(n), m); h->s32.resize(n); h->y32.resize(n); }
    *out = h;
    return LBFGS_B200_OK;
}
void lbfgs_b200_hist_destroy(lbfgs_b200_hist* h) { delete h; }
lbfgs_b200_status lbfgs_b200_hist_reset(lbfgs_b200_hist* h)
{
    if (!h) return LBFGS_B200_ERR_INVALID;
    if (h->elem == 8) h->h64->reset(h->h64->n, h->h64->m);
    else h->h32->reset(h->h32->n, h->h32->m);
    return LBFGS_B200_OK;
}
int lbfgs_b200_hist_ncorr(const lbfgs_b200_hist* h) { return h->elem == 8 ? h->h64->ncorr : h->h32->ncorr; }
int lbfgs_b200_hist_m(const lbfgs_b200_hist* h) { return h->elem == 8 ? h->h64->m : h->h32->m; }
const void* lbfgs_b200_hist_s_col(const lbfgs_b200_hist* h, int age) { return h->elem == 8 ? column<double>(h, true, age) : column<float>(h, true, age); }
const void* lbfgs_b200_hist_y_col(const lbfgs_b200_hist* h, int age) { return h->elem == 8 ? column<double>(h, false, age) : column<float>(h, false, age); }

#define MOCK_HIST(T, SUF)                                                                                                        \
    lbfgs_b200_status lbfgs_b200_hist_update_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g, const T* gp, T eps,  \
                                                   int* acc, T* sy_yy) { return do_update<T>(h, x, xp, g, gp, eps, acc, sy_yy); } \
    lbfgs_b200_status lbfgs_b200_hist_add_##SUF(lbfgs_b200_hist* h, const T* s, const T* y)                                      \
    { if (auto st = check_hist<T>(h)) return st; h->get<T>().add(s, y); return LBFGS_B200_OK; }                                  \
    lbfgs_b200_status lbfgs_b200_hist_apply_Hv_##SUF(lbfgs_b200_hist* h, const T* v, T a, T* res, int, T* vdot)                  \
    { return do_apply_Hv<T>(h, v, a, res, vdot); }                                                                               \
    lbfgs_b200_status lbfgs_b200_hist_update_apply_Hv_##SUF(lbfgs_b200_hist* h, const T* x, const T* xp, const T* g,             \
                                                            const T* gp, T eps, T a, T* res, int, int* acc, T* vdot)             \
    { if (auto st = do_update<T>(h, x, xp, g, gp, eps, acc, nullptr)) return st; return do_apply_Hv<T>(h, g, a, res, vdot); }    \
    lbfgs_b200_status lbfgs_b200_hist_scalars_##SUF(lbfgs_b200_hist* h, T* th, T* ys, T* al)                                     \
    {                                                                                                                            \
        if (auto st = check_hist<T>(h)) return st;                                                                               \
        orc::History<T>& H = h->get<T>();                                                                                        \
        if (th) *th = H.theta;                                                                                                   \
        for (int age = 0; age < H.ncorr; age++)                                                                                  \
        {                                                                                                                        \
            const int slot = ((H.ptr - 1 - age) % H.m + H.m) % H.m;                                                              \
            if (ys) ys[age] = H.ys[slot];                                                                                        \
            if (al) al[age] = H.alpha[slot];                                                                                     \
        }                                                                                                                        \
        return LBFGS_B200_OK;                                                                                                    \
    }
MOCK_HIST(double, f64)
MOCK_HIST(float, f32)

// ---- bound-constrained path ---------------------------------------------------------------------------------------------------
lbfgs_b200_status lbfgs_b200_box_create(lbfgs_b200_hist* h, lbfgs_b200_box** out)
{
    if (!h || !out) return LBFGS_B200_ERR_INVALID;
    if (lbfgs_b200_hist_m(h) > 20) return fail(h->ctx, LBFGS_B200_ERR_INVALID, "the bound-constrained path supports m <= 20");
    lbfgs_b200_box* b = new lbfgs_b200_box();
    b->h = h;
    b->n = h->elem == 8 ? h->h64->n : h->h32->n;
    b->cls.assign(size_t(b->n), 0);
    for (int k = 0; k < 10; k++)
    {
        if (h->elem == 8) b->v64[k].assign(size_t(b->n), 0.0);
        else b->v32[k].assign(size_t(b->n), 0.f);
    }
    *out = b;
    return LBFGS_B200_OK;
}
void lbfgs_b200_box_destroy(lbfgs_b200_box* b) { delete b; }
const void* lbfgs_b200_box_xcp(const lbfgs_b200_box* b) { return lbfgs_b200_box_vector(const_cast<lbfgs_b200_box*>(b), V_XCP); }
const unsigned char* lbfgs_b200_box_classes(const lbfgs_b200_box* b) { return b ? b->cls.data() : nullptr; }
void* lbfgs_b200_box_vector(lbfgs_b200_box* b, int which)
{
    if (!b || which < 0 || which >= 10) return nullptr;
    return b->h->elem == 8 ? static_cast<void*>(b->v64[which].data()) : static_cast<void*>(b->v32[which].data());
}
#define MOCK_BOX(T, SUF)                                                                                                         \
    lbfgs_b200_status lbfgs_b200_box_clamp_##SUF(lbfgs_b200_ctx*, int64_t n, T* x, const T* lb, const T* ub)                     \
    { for (int64_t i = 0; i < n; i++) x[i] = std::min(std::max(x[i], lb[i]), ub[i]); return LBFGS_B200_OK; }                     \
    lbfgs_b200_status lbfgs_b200_box_proj_grad_norm_##SUF(lbfgs_b200_ctx*, int64_t n, const T* x, const T* g, const T* lb,       \
                                                          const T* ub, T* o)                                                     \
    {                                                                                                                            \
        T m = T(0);                                                                                                              \
        for (int64_t i = 0; i < n; i++) m = std::max(m, std::abs(std::min(std::max(x[i] - g[i], lb[i]), ub[i]) - x[i]));         \
        *o = m;                                                                                                                  \
        return LBFGS_B200_OK;                                                                                                    \
    }                                                                                                                            \
    lbfgs_b200_status lbfgs_b200_box_dir_info_##SUF(lbfgs_b200_ctx*, int64_t n, const T* x, const T* d, const T* g, const T* lb, \
                                                    const T* ub, T* o2)                                                          \
    {                                                                                                                            \
        T dot = T(0), step = std::numeric_limits<T>::infinity();                                                                 \
        for (int64_t i = 0; i < n; i++)                                                                                          \
        {                                                                                                                        \
            dot += g[i] * d[i];                                                                                                  \
            if (d[i] > T(0)) step = std::min(step, (ub[i] - x[i]) / d[i]);                                                       \
            else if (d[i] < T(0)) step = std::min(step, (lb[i] - x[i]) / d[i]);                                                  \
        }                                                                                                                        \
        o2[0] = dot; o2[1] = step;                                                                                               \
        return LBFGS_B200_OK;                                                                                                    \
    }                                                                                                                            \
    lbfgs_b200_status lbfgs_b200_hist_wt_dot_##SUF(lbfgs_b200_hist* h, const T* v, T* raw) { return do_wt_dot<T>(h, v, raw); }  \
    lbfgs_b200_status lbfgs_b200_hist_gram_##SUF(lbfgs_b200_hist* h, T* sy, T* ss, T* yy, T* ys, T* th) { return do_gram<T>(h, sy, ss, yy, ys, th); } \
    lbfgs_b200_status lbfgs_b200_hist_lincomb_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box*, T a0, const T* v0, const T* coef,       \
                                                    const unsigned char* cls, int mask, T* out)                                  \
    { return do_lincomb<T>(h, a0, v0, coef, cls, mask, out); }                                                                   \
    lbfgs_b200_status lbfgs_b200_hist_masked_gram_##SUF(lbfgs_b200_hist* h, lbfgs_b200_box*, const unsigned char* cls, int mask, T* G) \
    { return do_masked_gram<T>(h, cls, mask, G); }                                                                               \
    lbfgs_b200_status lbfgs_b200_box_cauchy_breaks_##SUF(lbfgs_b200_box* b, const T* x, const T* g, const T* lb, const T* ub, T* o5) \
    { return do_cauchy_breaks<T>(b, x, g, lb, ub, o5); }                                                                         \
    lbfgs_b200_status lbfgs_b200_box_cauchy_sweep_##SUF(lbfgs_b200_box* b, const T* g, const T* M, const T* p0, T theta, T gt,    \
                                                        int64_t nord, int64_t ninf, T* out)                                      \
    { return do_cauchy_sweep<T>(b, g, M, p0, theta, gt, nord, ninf, out); }                                                      \
    lbfgs_b200_status lbfgs_b200_box_cauchy_build_##SUF(lbfgs_b200_box* b, const T* x, const T* lb, const T* ub, T tc, T tf, T* c2) \
    { return do_cauchy_build<T>(b, x, lb, ub, tc, tf, c2); }                                                                     \
    lbfgs_b200_status lbfgs_b200_box_sub_step_##SUF(lbfgs_b200_box* b, int op, int flag, const T* x0, const T* g, const T* lb,   \
                                                    const T* ub, T* drt, T theta, T* o3)                                         \
    { return do_sub_step<T>(b, op, flag, x0, g, lb, ub, drt, theta, o3); }
MOCK_BOX(double, f64)
MOCK_BOX(float, f32)

// ---- device-resident solve: not provided by the test double ------------------------------------------------------------------------
lbfgs_b200_status lbfgs_b200_solver_create(lbfgs_b200_ctx* c, int64_t, int, int, lbfgs_b200_solver**) { return unsupported(c, "the device-resident solve"); }
lbfgs_b200_status lbfgs_b200_solver_create_batch(lbfgs_b200_ctx* c, int64_t, int, int, int, lbfgs_b200_solver**) { return unsupported(c, "the device-resident solve"); }
void lbfgs_b200_solver_destroy(lbfgs_b200_solver*) {}
int lbfgs_b200_solver_batch(const lbfgs_b200_solver*) { return 0; }
const void* lbfgs_b200_solver_final_grad_of(const lbfgs_b200_solver*, int) { return nullptr; }
lbfgs_b200_hist* lbfgs_b200_solver_history_of(lbfgs_b200_solver*, int) { return nullptr; }
lbfgs_b200_status lbfgs_b200_solver_profile(const lbfgs_b200_solver*, double*, double*, unsigned long long*, double*, double*) { return LBFGS_B200_ERR_INVALID; }
lbfgs_b200_status lbfgs_b200_solver_minimize_batch_f64(lbfgs_b200_solver*, int, const double*, const double*, int64_t, const lbfgs_b200_param*, int, double*,
                                                       int64_t, lbfgs_b200_outcome*) { return unsupported(nullptr, "the device-resident solve"); }
lbfgs_b200_status lbfgs_b200_solver_minimize_batch_f32(lbfgs_b200_solver*, int, const float*, const float*, int64_t, const lbfgs_b200_param*, int, float*,
                                                       int64_t, lbfgs_b200_outcome*) { return unsupported(nullptr, "the device-resident solve"); }
const void* lbfgs_b200_solver_final_grad(const lbfgs_b200_solver*) { return nullptr; }
lbfgs_b200_hist* lbfgs_b200_solver_history(lbfgs_b200_solver*) { return nullptr; }
lbfgs_b200_status lbfgs_b200_solver_minimize_f64(lbfgs_b200_solver*, int, const double*, const double*, const lbfgs_b200_param*, int, double*,
                                                 double*, long long, lbfgs_b200_outcome*) { return unsupported(nullptr, "the device-resident solve"); }
lbfgs_b200_status lbfgs_b200_solver_minimize_f32(lbfgs_b200_solver*, int, const float*, const float*, const lbfgs_b200_param*, int, float*,
                                                 double*, long long, lbfgs_b200_outcome*) { return unsupported(nullptr, "the device-resident solve"); }

}  // extern "C"
