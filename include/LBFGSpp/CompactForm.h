// LBFGSpp/CompactForm.h -- the 2c x 2c algebra of the compact L-BFGS representation over raw arrays, written once for the host
// (BFGSMat.h, BKLDLT.h) and the device (the small-batch products of csrc/small_batch.cuh).  Compiled by g++ and nvcc alike; with
// -ffp-contract=off / -fmad=false both compute the same bits from the same inputs.
//
// Conventions: history columns by AGE (0 = newest pair); the c x c Gram blocks by age, row-major with leading dimension ldg:
// SY(a, b) = s_a'y_b, SS(a, b) = s_a's_b, YY(a, b) = y_a'y_b.  Per vector, wv[r * ldw] holds the dots [Y S]'v (rows y by age, then
// s by age) and the coefficients are written to C[r * ldc] in the same row order.
//   B v = theta v - W M W'v,  W = [Y, theta S],  M = Minv^-1,  Minv = [ -D   L' ; L   theta S'S ]
//       (D = diag(s_a'y_a), L(a, b) = s_a'y_b when pair a is newer than pair b)          C = -M W'v in W's convention, a0 = theta
//   H v = v/theta + S u_s + Y u_y/theta,  R = triu(S'Y) in chronological order t = c - 1 - age:
//       u_y = -R^-1 S'v,  u_s = R^-T ((D + Y'Y/theta) R^-1 S'v - Y'v/theta)                                    a0 = 1/theta
// With c = 0: B = theta I, H = I / theta.
// The same two matrices as B = theta I + W K_B W' and H = I/theta + W K_H W' over the raw W = [Y S]: compact_kb / compact_kh, whose
// diagonals a0 + r_i' K r_i (r_i: row i of W) need no products.
#ifndef LBFGSPP_B200_COMPACT_FORM_H
#define LBFGSPP_B200_COMPACT_FORM_H

#include <cmath>

#include "LineSearchCore.h"

namespace LBFGSpp {

// ---- Bunch-Kaufman LDL' of a symmetric indefinite n x n matrix (the pivot rule is documented in BKLDLT.h) ----------------------
enum { BK_SINGLE = 0, BK_PAIR_HEAD = 1, BK_PAIR_TAIL = 2 };

// w: the full symmetric matrix, row-major, factorised in place (strictly lower part: L; diagonal and the sub-diagonal inside a
// pair: D).  order[i]: original index now at position i; tag[i]: BK_*.  Returns 0 (SUCCESSFUL) or 2 (NUMERICAL_ISSUE).
template <typename T>
LBFGS_HD inline int bk_factor(T* w, int n, int* order, unsigned char* tag)
{
    using std::abs;
    auto W = [&](int i, int j) -> T& { return w[i * n + j]; };
    // symmetric interchange of positions p < q: whole rows, and the columns of the not-yet-eliminated block starting at `from`
    auto interchange = [&](int p, int q, int from) {
        if (p == q) return;
        for (int j = 0; j < n; j++) { const T t = W(p, j); W(p, j) = W(q, j); W(q, j) = t; }
        for (int i = from; i < n; i++) { const T t = W(i, p); W(i, p) = W(i, q); W(i, q) = t; }
        const int t = order[p]; order[p] = order[q]; order[q] = t;
    };
    for (int i = 0; i < n; i++) { order[i] = i; tag[i] = BK_SINGLE; }
    const T alpha = T((1.0 + std::sqrt(17.0)) / 8.0);
    int k = 0;
    while (k < n)
    {
        // largest off-diagonal magnitude of column k in the active block
        int r = k;
        T colmax = T(0);
        for (int i = k + 1; i < n; i++)
            if (abs(W(i, k)) > colmax) { colmax = abs(W(i, k)); r = i; }
        const T akk = abs(W(k, k));
        bool pair = false;
        if (colmax > T(0) && akk < alpha * colmax)
        {
            T rowmax = T(0);  // largest off-diagonal magnitude of row/column r in the active block
            for (int j = k; j < n; j++)
                if (j != r && abs(W(r, j)) > rowmax) rowmax = abs(W(r, j));
            if (akk * rowmax >= alpha * colmax * colmax) { /* a(k,k) is acceptable after all */ }
            else if (abs(W(r, r)) >= alpha * rowmax) interchange(k, r, k);
            else { interchange(k + 1, r, k); pair = true; }
        }
        if (!pair)
        {
            const T d = W(k, k);
            if (d == T(0)) return 2;
            for (int i = k + 1; i < n; i++)
            {
                const T li = W(i, k) / d;
                for (int j = k + 1; j <= i; j++) W(i, j) -= li * W(k, j);  // row k still holds column k unscaled
                W(i, k) = li;
            }
            for (int i = k + 1; i < n; i++)
                for (int j = i + 1; j < n; j++) W(i, j) = W(j, i);
            k += 1;
        }
        else
        {
            const T a = W(k, k), b = W(k + 1, k), c = W(k + 1, k + 1);
            const T det = a * c - b * b;
            if (det == T(0)) return 2;
            tag[k] = BK_PAIR_HEAD;
            tag[k + 1] = BK_PAIR_TAIL;
            for (int i = k + 2; i < n; i++)
            {
                const T u = W(i, k), v = W(i, k + 1);
                const T l1 = (u * c - v * b) / det, l2 = (v * a - u * b) / det;
                for (int j = k + 2; j <= i; j++) W(i, j) -= l1 * W(k, j) + l2 * W(k + 1, j);
                W(i, k) = l1;
                W(i, k + 1) = l2;
            }
            // mirror the updated block: the pivot search and the next elimination read rows as well as columns
            for (int i = k + 2; i < n; i++)
                for (int j = i + 1; j < n; j++) W(i, j) = W(j, i);
            k += 2;
        }
    }
    return 0;
}

// b <- A^-1 b for the factorisation above; b[i * bstride], z: n elements of scratch
template <typename T>
LBFGS_HD inline void bk_solve(const T* w, int n, const int* order, const unsigned char* tag, T* b, int bstride, T* z)
{
    auto W = [&](int i, int j) { return w[i * n + j]; };
    for (int i = 0; i < n; i++) z[i] = b[order[i] * bstride];
    // L z' = z : columns of a pair carry no entry on the pair's own rows
    for (int k = 0; k < n; k++)
    {
        const int first = (tag[k] == BK_PAIR_HEAD) ? k + 2 : k + 1;
        for (int i = first; i < n; i++) z[i] -= W(i, k) * z[k];
    }
    for (int k = 0; k < n; k++)
    {
        if (tag[k] == BK_SINGLE)
            z[k] /= W(k, k);
        else if (tag[k] == BK_PAIR_HEAD)
        {
            const T a = W(k, k), bb = W(k + 1, k), c = W(k + 1, k + 1), det = a * c - bb * bb;
            const T u = z[k], v = z[k + 1];
            z[k] = (u * c - v * bb) / det;
            z[k + 1] = (v * a - u * bb) / det;
        }
    }
    for (int k = n - 1; k >= 0; k--)
    {
        const int first = (tag[k] == BK_PAIR_HEAD) ? k + 2 : k + 1;
        T acc = T(0);
        for (int i = first; i < n; i++) acc += W(i, k) * z[i];
        z[k] -= acc;
    }
    for (int i = 0; i < n; i++) b[order[i] * bstride] = z[i];
}

// ---- the compact form ---------------------------------------------------------------------------------------------------------
// Minv [2c x 2c], row-major (every entry written)
template <typename T>
LBFGS_HD inline void compact_minv(int c, const T* SY, const T* SS, int ldg, T theta, T* Minv)
{
    const int w = 2 * c;
    for (int i = 0; i < w * w; i++) Minv[i] = T(0);
    for (int a = 0; a < c; a++)
    {
        Minv[a * w + a] = -SY[a * ldg + a];
        for (int b = 0; b < c; b++)
        {
            if (a < b)  // age a < age b: pair a is the newer one
            {
                Minv[(c + a) * w + b] = SY[a * ldg + b];
                Minv[b * w + c + a] = SY[a * ldg + b];
            }
            Minv[(c + a) * w + c + b] = theta * SS[a * ldg + b];
        }
    }
}

// B: C = -M u with u = [Y'v ; theta S'v] (M: the 2c x 2c inverse of Minv, row-major)
template <typename T>
LBFGS_HD inline void compact_b_coef(int c, const T* M, T theta, const T* wv, int ldw, T* C, int ldc)
{
    const int w = 2 * c;
    for (int i = 0; i < w; i++)
    {
        T acc = T(0);
        for (int j = 0; j < w; j++) acc += M[i * w + j] * (j < c ? wv[j * ldw] : theta * wv[j * ldw]);
        C[i * ldc] = i < c ? -acc : -theta * acc;
    }
}

// H: R(t, u) = s_t'y_u (t <= u, else 0) and Y'Y, both c x c in chronological order t = c - 1 - age
template <typename T>
LBFGS_HD inline void compact_h_setup(int c, const T* SY, const T* YY, int ldg, T* R, T* YYc)
{
    for (int t = 0; t < c; t++)
        for (int u = 0; u < c; u++)
        {
            R[t * c + u] = t <= u ? SY[(c - 1 - t) * ldg + (c - 1 - u)] : T(0);
            YYc[t * c + u] = YY[(c - 1 - t) * ldg + (c - 1 - u)];
        }
}

// H: the coefficients of one vector.  w, us: c elements of scratch each (stride ldt)
template <typename T>
LBFGS_HD inline void compact_h_coef(int c, const T* R, const T* YYc, T theta, const T* wv, int ldw, T* w, T* us, int ldt, T* C, int ldc)
{
    auto p = [&](int t) { return wv[(c + c - 1 - t) * ldw]; };   // s_t'v
    auto q = [&](int t) { return wv[(c - 1 - t) * ldw]; };       // y_t'v
    for (int t = c - 1; t >= 0; t--)   // w = R^-1 S'v
    {
        T acc = p(t);
        for (int s = t + 1; s < c; s++) acc -= R[t * c + s] * w[s * ldt];
        w[t * ldt] = acc / R[t * c + t];
    }
    for (int t = 0; t < c; t++)        // u_s = R^-T ((D + Y'Y/theta) w - Y'v/theta)
    {
        T z = R[t * c + t] * w[t * ldt];
        T yyw = T(0);
        for (int s = 0; s < c; s++) yyw += YYc[t * c + s] * w[s * ldt];
        z += (yyw - q(t)) / theta;
        for (int s = 0; s < t; s++) z -= R[s * c + t] * us[s * ldt];
        us[t * ldt] = z / R[t * c + t];
    }
    for (int t = 0; t < c; t++)
    {
        C[(c - 1 - t) * ldc] = -w[t * ldt] / theta;
        C[(c + c - 1 - t) * ldc] = us[t * ldt];
    }
}

// ---- the middle matrices over the raw columns: B = theta I + W K_B W',  H = I/theta + W K_H W',  W = [Y S] by age ----------------
// K_B = -diag(I, theta I) M diag(I, theta I); K_H = [ 0  -R^-1/theta ; -R^-T/theta  R^-T (D + Y'Y/theta) R^-1 ] (the blocks in
// chronological order).  Column r of K is the coefficient vector compact_b_coef / compact_h_coef make for e_r, so the two functions
// below write columns r0, r0 + dr, ... of K [2c x 2c] (row-major, rows y by age then s by age) and several threads can share a K;
// compact_k_symmetrise then makes it exactly symmetric.  unit: 4c - 1 elements, zero but unit[2c - 1] = 1, so that unit + 2c - 1 - r
// is e_r with stride 1.
template <typename T>
LBFGS_HD inline void compact_kb(int c, const T* M, T theta, const T* unit, int r0, int dr, T* K)
{
    const int w = 2 * c;
    for (int r = r0; r < w; r += dr) compact_b_coef(c, M, theta, unit + (w - 1 - r), 1, K + r, w);
}

// scr: compact_h_coef's w and us for one column, 2c elements at stride ldt
template <typename T>
LBFGS_HD inline void compact_kh(int c, const T* R, const T* YYc, T theta, const T* unit, int r0, int dr, T* scr, int ldt, T* K)
{
    const int w = 2 * c;
    for (int r = r0; r < w; r += dr) compact_h_coef(c, R, YYc, theta, unit + (w - 1 - r), 1, scr, scr + c * ldt, ldt, K + r, w);
}

// K = (K + K')/2 on rows i0, i0 + di, ...: row i owns the pairs (i, j > i), so rows may be done by different threads at once
template <typename T>
LBFGS_HD inline void compact_k_symmetrise(int w, T* K, int i0, int di)
{
    for (int i = i0; i < w; i += di)
        for (int j = i + 1; j < w; j++)
        {
            const T v = (K[i * w + j] + K[j * w + i]) * T(0.5);
            K[i * w + j] = v;
            K[j * w + i] = v;
        }
}

// ---- a square-root factor of H: H = L L' (Brodlie-Gourlay-Greenstadt) ----------------------------------------------------------
// Pairs in chronological order t = c - 1 - age, rho_t = 1/(y_t's_t), B_t the BFGS matrix after pairs 0..t-1 from theta I,
// p_t = B_t s_t, sigma_t = s_t'p_t.  H_{t+1} = (I + s_t b_t') H_t (I + b_t s_t') with b_t = -rho_t y_t + sqrt(rho_t / sigma_t) p_t, so
//     L = (I + s_{c-1} b_{c-1}') ... (I + s_0 b_0') / sqrt(theta),     log det H = -n log theta + sum_t log(rho_t sigma_t)
// and 1 + b_t's_t = sqrt(rho_t sigma_t) > 0.  p_t lies in span(W), W = [Y S]:
//     p_t = theta s_t + sum_{j<t} ( -p_j (p_j's_t) / sigma_j + rho_j y_j (y_j's_t) )
// needs only Gram entries, so b_t = W beta_t with beta_t in R^2c.  L z = z/sqrt(theta) + sum_t alpha_t s_t with the unit lower
// triangular recursion alpha_t = beta_t'(W'z)/sqrt(theta) + sum_{j<t} T(t, j) alpha_j, T(t, j) = beta_t'W's_j.
//
// compact_factor_setup: beta [2c][c] (row r in W's order: y by age, then s by age; column t chronological) and Tm [c][c]: T(t, j) in
// its strictly lower part (Tm[t * c + j], j < t); its diagonal holds sigma_t and its upper part p_t's_u (u > t), the intermediates.
// Everything is evaluated in fp64 whatever T is.  *logsum = sum_t log(rho_t sigma_t).  Returns 0, or 2 (NUMERICAL_ISSUE) when some
// rho_t or sigma_t is not positive and finite (beta and Tm are then incomplete).  O(c^3).
template <typename T>
LBFGS_HD inline int compact_factor_setup(int c, const T* SY, const T* SS, const T* YY, int ldg, T theta, double* beta, double* Tm,
                                         double* logsum)
{
    (void)YY;   // y'y never enters: b_t is tested against s columns only
    const double th = double(theta), big = 1.7976931348623157e308;
    auto sy = [&](int t, int u) { return double(SY[(c - 1 - t) * ldg + (c - 1 - u)]); };   // s_t'y_u, chronological
    *logsum = 0.0;
    for (int t = 0; t < c; t++)
    {
        // pi_t (the coefficients of p_t) in column t of beta
        for (int r = 0; r < 2 * c; r++) beta[r * c + t] = 0.0;
        beta[(2 * c - 1 - t) * c + t] = th;
        for (int j = 0; j < t; j++)
        {
            const double f = -Tm[j * c + t] / Tm[j * c + j];
            for (int r = 0; r < 2 * c; r++) beta[r * c + t] += f * beta[r * c + j];
            beta[(c - 1 - j) * c + t] += sy(t, j) / sy(j, j);
        }
        // row t of Tm: s_u'p_t for every u
        for (int u = 0; u < c; u++)
        {
            const int au = c - 1 - u;
            double acc = 0.0;
            for (int a = 0; a < c; a++) acc += beta[a * c + t] * double(SY[au * ldg + a]) + beta[(c + a) * c + t] * double(SS[au * ldg + a]);
            Tm[t * c + u] = acc;
        }
        const double rho = 1.0 / sy(t, t), sigma = Tm[t * c + t];
        if (!(rho > 0.0 && rho <= big && sigma > 0.0 && sigma <= big)) return 2;
        *logsum += std::log(rho * sigma);
    }
    // beta_t = -rho_t e_{y_t} + kappa_t pi_t,  T(t, j) = -rho_t y_t's_j + kappa_t p_t's_j,  kappa_t = sqrt(rho_t / sigma_t)
    for (int t = 0; t < c; t++)
    {
        const double rho = 1.0 / sy(t, t), kappa = std::sqrt(rho / Tm[t * c + t]);
        for (int r = 0; r < 2 * c; r++) beta[r * c + t] *= kappa;
        beta[(c - 1 - t) * c + t] -= rho;
        for (int j = 0; j < t; j++) Tm[t * c + j] = kappa * Tm[t * c + j] - rho * sy(j, t);
    }
    return 0;
}

// L z for one vector from its dots wv[r * ldw] = (W'z)_r: C[r * ldc] in compact_b_coef's row order, the y rows zero and the s row of
// age c - 1 - t holding alpha_t, so that L z = a0 z + sum_r C_r W_r with a0 = rsq = 1/sqrt(theta).  Sums in fp64; alpha_j is read back
// from C (as T).
template <typename T>
LBFGS_HD inline void compact_factor_coef(int c, const double* beta, const double* Tm, double rsq, const T* wv, int ldw, T* C, int ldc)
{
    for (int a = 0; a < c; a++) C[a * ldc] = T(0);
    for (int t = 0; t < c; t++)
    {
        double acc = 0.0;
        for (int r = 0; r < 2 * c; r++) acc += beta[r * c + t] * double(wv[r * ldw]);
        acc *= rsq;
        for (int j = 0; j < t; j++) acc += Tm[t * c + j] * double(C[(2 * c - 1 - j) * ldc]);
        C[(2 * c - 1 - t) * ldc] = T(acc);
    }
}

// ---- the transpose and the inverses of the factor, and the quadratic form of B = H^-1 ------------------------------------------
// (I + s b')^-1 = I - s b'/(1 + b's) with 1 + b_t's_t = d_t = sqrt(rho_t sigma_t) > 0, so with U(t, j) = b_t's_j (j > t):
//     L' v     = (v + W sum_t beta_t gamma_t) / sqrt(theta),   gamma_t = s_t'v + sum_{j>t} T(j, t) gamma_j          (t = c-1 .. 0)
//     L^-1 v   = sqrt(theta) (v + sum_t alpha_t s_t),           alpha_t = -(beta_t'W'v + sum_{j>t} U(t, j) alpha_j) / d_t   (t = c-1 .. 0)
//     L^-T v   = sqrt(theta) (v - W sum_t beta_t delta_t),      delta_t = (s_t'v - sum_{j<t} U(j, t) delta_j) / d_t  (t = 0 .. c-1)
//     v'B v    = |L^-1 v|^2 = theta (v'v + 2 alpha'S'v + alpha'S'S alpha)
// L' and L^-T need only S'v.  The coefficient functions take the dots of one vector (sv[a * ldw] = s_a'v by age; wv as above for
// L^-1), run the recursion in fp64 in z[0, c) (scratch of the caller) and write C[r * ldc] in compact_factor_coef's row order; the
// product is then a0 v + sum_r C_r W_r with a0 = 1/sqrt(theta) for L' and sqrt(theta) for both inverses.

// compact_factor_upper: after a successful compact_factor_setup, Tm's strict upper part becomes U(t, j) (j > t) and its diagonal d_t.
// The strict lower part (T) is left as it is.  Only the inverses call it, so the factor itself keeps its arithmetic.
template <typename T>
LBFGS_HD inline void compact_factor_upper(int c, const T* SY, int ldg, double* Tm)
{
    auto sy = [&](int t, int u) { return double(SY[(c - 1 - t) * ldg + (c - 1 - u)]); };   // s_t'y_u, chronological
    for (int t = 0; t < c; t++)
    {
        const double rho = 1.0 / sy(t, t), sigma = Tm[t * c + t], kappa = std::sqrt(rho / sigma);
        for (int j = t + 1; j < c; j++) Tm[t * c + j] = kappa * Tm[t * c + j] - rho * sy(j, t);   // b_t's_j = kappa p_t's_j - rho y_t's_j
        Tm[t * c + t] = std::sqrt(rho * sigma);
    }
}

// L' v: every row of C
template <typename T>
LBFGS_HD inline void compact_factor_t_coef(int c, const double* beta, const double* Tm, double rsq, const T* sv, int ldw, double* z, T* C, int ldc)
{
    for (int t = c - 1; t >= 0; t--)
    {
        double acc = double(sv[(c - 1 - t) * ldw]);
        for (int j = t + 1; j < c; j++) acc += Tm[j * c + t] * z[j];
        z[t] = acc;
    }
    for (int r = 0; r < 2 * c; r++)
    {
        double acc = 0.0;
        for (int t = 0; t < c; t++) acc += beta[r * c + t] * z[t];
        C[r * ldc] = T(rsq * acc);
    }
}

// alpha of L^-1 v into z (Tm after compact_factor_upper)
template <typename T>
LBFGS_HD inline void compact_factor_inv_alpha(int c, const double* beta, const double* Tm, const T* wv, int ldw, double* z)
{
    for (int t = c - 1; t >= 0; t--)
    {
        double acc = 0.0;
        for (int r = 0; r < 2 * c; r++) acc += beta[r * c + t] * double(wv[r * ldw]);
        for (int j = t + 1; j < c; j++) acc += Tm[t * c + j] * z[j];
        z[t] = -acc / Tm[t * c + t];
    }
}

// L^-1 v: the y rows zero, the s row of age c - 1 - t holding sqrt(theta) alpha_t
template <typename T>
LBFGS_HD inline void compact_factor_inv_coef(int c, const double* beta, const double* Tm, double sq, const T* wv, int ldw, double* z, T* C, int ldc)
{
    compact_factor_inv_alpha(c, beta, Tm, wv, ldw, z);
    for (int t = 0; t < c; t++)
    {
        C[(c - 1 - t) * ldc] = T(0);
        C[(2 * c - 1 - t) * ldc] = T(sq * z[t]);
    }
}

// L^-T v: every row of C
template <typename T>
LBFGS_HD inline void compact_factor_invt_coef(int c, const double* beta, const double* Tm, double sq, const T* sv, int ldw, double* z, T* C, int ldc)
{
    for (int t = 0; t < c; t++)
    {
        double acc = double(sv[(c - 1 - t) * ldw]);
        for (int j = 0; j < t; j++) acc -= Tm[j * c + t] * z[j];
        z[t] = acc / Tm[t * c + t];
    }
    for (int r = 0; r < 2 * c; r++)
    {
        double acc = 0.0;
        for (int t = 0; t < c; t++) acc += beta[r * c + t] * z[t];
        C[r * ldc] = T(-sq * acc);
    }
}

// q = v'B v = |L^-1 v|^2 from the dots wv = W'v and vv = v'v alone (no pass over v); the log density of N(mu, H) at x = mu + v is
// -q/2 - log det H / 2 - (n/2) log 2 pi.  With c = 0: theta v'v.
template <typename T, typename TW>
LBFGS_HD inline double compact_factor_quad(int c, const double* beta, const double* Tm, const T* SS, int ldg, T theta, const TW* wv, int ldw,
                                           double vv, double* z)
{
    compact_factor_inv_alpha(c, beta, Tm, wv, ldw, z);
    double q = vv;
    for (int t = 0; t < c; t++)
    {
        const int at = c - 1 - t;
        double acc = 2.0 * double(wv[(c + at) * ldw]);
        for (int u = 0; u < c; u++) acc += double(SS[at * ldg + (c - 1 - u)]) * z[u];
        q += z[t] * acc;
    }
    return double(theta) * q;
}

// log N(x; mu, H) from q = (x - mu)'B(x - mu) and log det H
LBFGS_HD inline double compact_log_density(double q, double logdet, double n)
{
    return -0.5 * q - 0.5 * logdet - 0.5 * n * 1.8378770664093453;   // log(2 pi)
}

// ---- the approximation restricted to a set F of coordinates: B_F = Z'BZ and H_F = (Z'BZ)^-1, Z selecting F -----------------------
// With G = W_F'W_F the Gram matrix of the rows of F (raw W = [Y S] by age, 2c x 2c), Woodbury on B_F = theta I - W_F M W_F' (W in
// [Y, theta S]) gives H_F = I/theta + W_F mid^-1 W_F' / theta^2 with
//     mid = Minv - W_F'W_F / theta   (in W's [Y, theta S] convention; solve_PtBP's inv(P'BP))
// and over the raw columns, with D = diag(I, theta I):
//     B_F = theta I + W_F K_B W_F',  K_B = -D M D (compact_kb);     H_F = I/theta + W_F K_HF W_F',  K_HF = D mid^-1 D / theta^2.
// diag B_F is diag B on F (a principal submatrix), diag H_F_i = 1/theta + r_i' K_HF r_i.  H_F is also the covariance of N(x*, H)
// conditioned on the coordinates outside F.

// mid [2c x 2c] row-major from Minv, the S'S block by age (leading dimension ldg) and the masked Gram G [2c x 2c]
template <typename T>
LBFGS_HD inline void compact_free_mid(int c, const T* Minv, const T* SS, int ldg, const T* G, T theta, T* mid)
{
    const int w = 2 * c;
    for (int a = 0; a < c; a++)
        for (int b = 0; b < c; b++)
        {
            mid[a * w + b] = Minv[a * w + b] - G[a * w + b] / theta;
            mid[(c + a) * w + b] = Minv[(c + a) * w + b] - G[(c + a) * w + b];
            mid[b * w + c + a] = mid[(c + a) * w + b];
            mid[(c + a) * w + c + b] = theta * (SS[a * ldg + b] - G[(c + a) * w + c + b]);
        }
}

// Host only: K_HF [2c x 2c] = D mid^-1 D / theta^2, symmetrised.  mid is factorised in place; order, tag, z: 2c elements of scratch each.
// Returns bk_factor's status (0, or 2 when mid is singular: K is then not written).
inline int compact_free_kh(int c, double* mid, double theta, int* order, unsigned char* tag, double* z, double* K)
{
    const int w = 2 * c;
    if (const int st = bk_factor(mid, w, order, tag)) return st;
    for (int r = 0; r < w; r++)
    {
        for (int i = 0; i < w; i++) K[i * w + r] = i == r ? 1.0 : 0.0;
        bk_solve(mid, w, order, tag, K + r, w, z);
        const double dr = r < c ? 1.0 : theta;
        for (int i = 0; i < w; i++) K[i * w + r] *= dr * (i < c ? 1.0 : theta) / (theta * theta);
    }
    compact_k_symmetrise(w, K, 0, 1);
    return 0;
}

// Host only: A = V diag(lam) V' for a symmetric n x n A (row-major, destroyed) by cyclic Jacobi rotations; V row-major, eigenvector j in column j.
inline void sym_eig_jacobi(int n, double* A, double* V, double* lam)
{
    for (int i = 0; i < n * n; i++) V[i] = 0.0;
    for (int i = 0; i < n; i++) V[i * n + i] = 1.0;
    for (int sweep = 0; sweep < 100; sweep++)
    {
        double off = 0.0, tot = 0.0;
        for (int i = 0; i < n; i++)
            for (int j = 0; j < n; j++) (i == j ? tot : off) += A[i * n + j] * A[i * n + j];
        if (!(off > 1e-30 * (tot + off))) break;
        for (int p = 0; p < n - 1; p++)
            for (int q = p + 1; q < n; q++)
            {
                const double apq = A[p * n + q];
                if (apq == 0.0) continue;
                const double tau = (A[q * n + q] - A[p * n + p]) / (2.0 * apq);
                const double t = (tau >= 0.0 ? 1.0 : -1.0) / (std::fabs(tau) + std::sqrt(1.0 + tau * tau));
                const double cs = 1.0 / std::sqrt(1.0 + t * t), sn = t * cs;
                for (int k = 0; k < n; k++)   // A <- J'A J with J the rotation in the (p, q) plane
                {
                    const double akp = A[k * n + p], akq = A[k * n + q];
                    A[k * n + p] = cs * akp - sn * akq;
                    A[k * n + q] = sn * akp + cs * akq;
                }
                for (int k = 0; k < n; k++)
                {
                    const double apk = A[p * n + k], aqk = A[q * n + k];
                    A[p * n + k] = cs * apk - sn * aqk;
                    A[q * n + k] = sn * apk + cs * aqk;
                }
                for (int k = 0; k < n; k++)
                {
                    const double vkp = V[k * n + p], vkq = V[k * n + q];
                    V[k * n + p] = cs * vkp - sn * vkq;
                    V[k * n + q] = sn * vkp + cs * vkq;
                }
            }
    }
    for (int i = 0; i < n; i++) lam[i] = A[i * n + i];
}

// Host only: a symmetric square root of H_F: L_F = (I + W_F E W_F') / sqrt(theta) with L_F L_F = H_F, and log det H_F = -n_F log theta + *logsum.
// G = W_F'W_F is equilibrated first, Gs = D G D with D = diag(G)^-1/2 (0 for a column that is zero on F): the y and s columns differ in
// size by the curvature (|y| ~ theta |s|), and a cut on the raw G would drop the directions of the smaller set once theta is far
// from 1.  Gs = V Lambda V' (eigenvalues <= 2c 2^-52 lambda_max dropped: W_F may be rank-deficient, e.g. n_F < 2c), Q = D^-1 V
// Lambda^1/2, A = theta Q' K_HF Q = U Sigma U', R = D V Lambda^-1/2 U, E = R (sqrt(1 + Sigma) - 1) R', *logsum = sum log(1 + sigma).
// G, K: w x w (w = 2c), E written w x w; scratch: 5 w^2 + 3 w doubles.  Returns 0, or 2 when some 1 + sigma_i is not positive and
// finite (E is then not written).
inline int compact_free_sqrt(int w, const double* G, const double* K, double theta, double* E, double* logsum, double* scratch)
{
    double *A = scratch, *V = A + w * w, *U = V + w * w, *Q = U + w * w, *R = Q + w * w, *lam = R + w * w, *sig = lam + w, *dg = sig + w;
    for (int i = 0; i < w; i++) dg[i] = G[i * w + i] > 0.0 ? std::sqrt(G[i * w + i]) : 0.0;   // D^-1
    for (int i = 0; i < w; i++)
        for (int j = 0; j < w; j++) A[i * w + j] = dg[i] > 0.0 && dg[j] > 0.0 ? G[i * w + j] / (dg[i] * dg[j]) : 0.0;
    sym_eig_jacobi(w, A, V, lam);
    double lmax = 0.0;
    for (int i = 0; i < w; i++) lmax = lam[i] > lmax ? lam[i] : lmax;
    auto kept = [&](int i) { return lmax > 0.0 && lam[i] > double(w) * 2.220446049250313e-16 * lmax; };
    int r = 0;   // Q = D^-1 V_r Lambda_r^1/2 and R without U: D V_r Lambda_r^-1/2 (w x r, columns packed; rows of zero columns are 0)
    for (int i = 0; i < w; i++)
        if (kept(i))
        {
            const double sl = std::sqrt(lam[i]);
            for (int k = 0; k < w; k++)
            {
                Q[k * w + r] = dg[k] * V[k * w + i] * sl;
                R[k * w + r] = dg[k] > 0.0 ? V[k * w + i] / (dg[k] * sl) : 0.0;
            }
            r++;
        }
    for (int a = 0; a < r; a++)   // A = theta Q' K Q  (r x r, leading dimension r)
        for (int b = 0; b < r; b++)
        {
            double acc = 0.0;
            for (int p = 0; p < w; p++)
            {
                double kq = 0.0;
                for (int q = 0; q < w; q++) kq += K[p * w + q] * Q[q * w + b];
                acc += Q[p * w + a] * kq;
            }
            A[a * r + b] = theta * acc;
        }
    for (int a = 0; a < r; a++)
        for (int b = a + 1; b < r; b++) A[a * r + b] = A[b * r + a] = 0.5 * (A[a * r + b] + A[b * r + a]);
    sym_eig_jacobi(r, A, U, sig);
    *logsum = 0.0;
    for (int i = 0; i < r; i++)
    {
        const double d = 1.0 + sig[i];
        if (!(d > 0.0 && d <= 1.7976931348623157e308)) return 2;
        *logsum += std::log1p(sig[i]);
    }
    for (int k = 0; k < w; k++)   // R <- R U
    {
        double row[128];
        for (int j = 0; j < r; j++)
        {
            double acc = 0.0;
            for (int i = 0; i < r; i++) acc += R[k * w + i] * U[i * r + j];
            row[j] = acc;
        }
        for (int j = 0; j < r; j++) R[k * w + j] = row[j];
    }
    for (int p = 0; p < w; p++)
        for (int q = 0; q < w; q++)
        {
            double acc = 0.0;
            for (int j = 0; j < r; j++) acc += R[p * w + j] * (std::sqrt(1.0 + sig[j]) - 1.0) * R[q * w + j];
            E[p * w + q] = acc;
        }
    return 0;
}

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_COMPACT_FORM_H
