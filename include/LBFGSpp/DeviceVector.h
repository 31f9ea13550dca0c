// LBFGSpp/DeviceVector.h -- the `Vector` type of the GPU front: an n-vector that lives in HBM.
//
// The reference's Vector is Eigen::Matrix<Scalar, Dynamic, 1> (reference LBFGS.h:25); here it is a handle to
// device memory obtained through the C ABI (include/lbfgs_b200.h).  The members the reference's solver and
// line searches rely on keep their names and meaning: size(), resize(), swap() (O(1) pointer swap, needed
// by `x_lo.swap(x)` at LineSearchMoreThuente.h:534), data(), norm(), squaredNorm(), dot().
// Host <-> device transfers are explicit (copy_from_host / copy_to_host / to_std_vector).
#ifndef LBFGSPP_B200_DEVICE_VECTOR_H
#define LBFGSPP_B200_DEVICE_VECTOR_H

#include <cmath>
#include <cstddef>
#include <memory>
#include <mutex>
#include <new>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "../lbfgs_b200.h"

namespace LBFGSpp {

// ----------------------------------------------------------------------------------------------------
// Device: owner of one lbfgs_b200_ctx (a GPU + a stream + reduction scratch [+ an NCCL communicator]).
// Status codes coming back over the C ABI are turned into the exception types the reference documents.
// ----------------------------------------------------------------------------------------------------
class Device
{
    lbfgs_b200_ctx* m_ctx;
    Device(const Device&);
    Device& operator=(const Device&);

public:
    explicit Device(int ordinal = 0, void* cuda_stream = nullptr) : m_ctx(nullptr)
    {
        const lbfgs_b200_status st = lbfgs_b200_ctx_create(&m_ctx, ordinal, cuda_stream);
        if (st != LBFGS_B200_OK) raise(st, lbfgs_b200_last_error(nullptr));
    }
    ~Device() { lbfgs_b200_ctx_destroy(m_ctx); }

    lbfgs_b200_ctx* ctx() const { return m_ctx; }

    static void raise(lbfgs_b200_status st, const char* what)
    {
        const std::string msg = std::string("lbfgs_b200: ") + (what ? what : "unknown error");
        switch (st)
        {
        case LBFGS_B200_ERR_INVALID: throw std::invalid_argument(msg);
        case LBFGS_B200_ERR_ALLOC: throw std::bad_alloc();
        default: throw std::runtime_error(msg);
        }
    }
    void check(lbfgs_b200_status st) const
    {
        if (st != LBFGS_B200_OK) raise(st, lbfgs_b200_last_error(m_ctx));
    }
    void synchronize() const { check(lbfgs_b200_sync(m_ctx)); }

    // Process-wide default device used by vectors constructed without an explicit Device
    // (so that `Vector x(n)` keeps working like in the reference).  Select with set_default().
    static std::shared_ptr<Device>& default_slot()
    {
        static std::shared_ptr<Device> dev;
        return dev;
    }
    static std::mutex& default_mutex()
    {
        static std::mutex m;
        return m;
    }
    static Device& get_default()
    {
        std::lock_guard<std::mutex> lock(default_mutex());   // solver objects may be constructed from several host threads
        std::shared_ptr<Device>& slot = default_slot();
        if (!slot) slot = std::make_shared<Device>(0);
        return *slot;
    }
    static void set_default(const std::shared_ptr<Device>& dev)
    {
        std::lock_guard<std::mutex> lock(default_mutex());
        default_slot() = dev;
    }
};

namespace detail {

template <class Scalar> struct Abi;
template <> struct Abi<double>
{
    static lbfgs_b200_status dot(lbfgs_b200_ctx* c, int64_t n, const double* a, const double* b, double* o) { return lbfgs_b200_dot_f64(c, n, a, b, o); }
    static lbfgs_b200_status dot3(lbfgs_b200_ctx* c, int64_t n, const double* g, const double* d, const double* x, double* o) { return lbfgs_b200_dot3_f64(c, n, g, d, x, o); }
    static lbfgs_b200_status axpy_out(lbfgs_b200_ctx* c, int64_t n, const double* a, double s, const double* b, double* o) { return lbfgs_b200_axpy_out_f64(c, n, a, s, b, o); }
    static lbfgs_b200_status scale_out(lbfgs_b200_ctx* c, int64_t n, double s, const double* a, double* o) { return lbfgs_b200_scale_out_f64(c, n, s, a, o); }
    static lbfgs_b200_status objective(lbfgs_b200_ctx* c, int obj, const double* d0, const double* d1, int64_t n, const double* x, double* g, double* fx) { return lbfgs_b200_objective_f64(c, obj, d0, d1, n, x, g, fx); }
    static lbfgs_b200_status trial(lbfgs_b200_ctx* c, int obj, const double* d0, const double* d1, int64_t n, const double* xp, const double* d, double step, double* x, double* g, double* o4) { return lbfgs_b200_trial_f64(c, obj, d0, d1, n, xp, d, step, x, g, o4); }
    static lbfgs_b200_status hist_update(lbfgs_b200_hist* h, const double* x, const double* xp, const double* g, const double* gp, double eps, int* acc, double* sy_yy) { return lbfgs_b200_hist_update_f64(h, x, xp, g, gp, eps, acc, sy_yy); }
    static lbfgs_b200_status hist_add(lbfgs_b200_hist* h, const double* s, const double* y) { return lbfgs_b200_hist_add_f64(h, s, y); }
    static lbfgs_b200_status hist_apply_Hv(lbfgs_b200_hist* h, const double* v, double a, double* res, int algo, double* vdot) { return lbfgs_b200_hist_apply_Hv_f64(h, v, a, res, algo, vdot); }
    static lbfgs_b200_status hist_update_apply_Hv(lbfgs_b200_hist* h, const double* x, const double* xp, const double* g, const double* gp, double eps, double a, double* res, int algo, int* acc, double* vdot) { return lbfgs_b200_hist_update_apply_Hv_f64(h, x, xp, g, gp, eps, a, res, algo, acc, vdot); }
};
template <> struct Abi<float>
{
    static lbfgs_b200_status dot(lbfgs_b200_ctx* c, int64_t n, const float* a, const float* b, float* o) { return lbfgs_b200_dot_f32(c, n, a, b, o); }
    static lbfgs_b200_status dot3(lbfgs_b200_ctx* c, int64_t n, const float* g, const float* d, const float* x, float* o) { return lbfgs_b200_dot3_f32(c, n, g, d, x, o); }
    static lbfgs_b200_status axpy_out(lbfgs_b200_ctx* c, int64_t n, const float* a, float s, const float* b, float* o) { return lbfgs_b200_axpy_out_f32(c, n, a, s, b, o); }
    static lbfgs_b200_status scale_out(lbfgs_b200_ctx* c, int64_t n, float s, const float* a, float* o) { return lbfgs_b200_scale_out_f32(c, n, s, a, o); }
    static lbfgs_b200_status objective(lbfgs_b200_ctx* c, int obj, const float* d0, const float* d1, int64_t n, const float* x, float* g, float* fx) { return lbfgs_b200_objective_f32(c, obj, d0, d1, n, x, g, fx); }
    static lbfgs_b200_status trial(lbfgs_b200_ctx* c, int obj, const float* d0, const float* d1, int64_t n, const float* xp, const float* d, float step, float* x, float* g, float* o4) { return lbfgs_b200_trial_f32(c, obj, d0, d1, n, xp, d, step, x, g, o4); }
    static lbfgs_b200_status hist_update(lbfgs_b200_hist* h, const float* x, const float* xp, const float* g, const float* gp, float eps, int* acc, float* sy_yy) { return lbfgs_b200_hist_update_f32(h, x, xp, g, gp, eps, acc, sy_yy); }
    static lbfgs_b200_status hist_add(lbfgs_b200_hist* h, const float* s, const float* y) { return lbfgs_b200_hist_add_f32(h, s, y); }
    static lbfgs_b200_status hist_apply_Hv(lbfgs_b200_hist* h, const float* v, float a, float* res, int algo, float* vdot) { return lbfgs_b200_hist_apply_Hv_f32(h, v, a, res, algo, vdot); }
    static lbfgs_b200_status hist_update_apply_Hv(lbfgs_b200_hist* h, const float* x, const float* xp, const float* g, const float* gp, float eps, float a, float* res, int algo, int* acc, float* vdot) { return lbfgs_b200_hist_update_apply_Hv_f32(h, x, xp, g, gp, eps, a, res, algo, acc, vdot); }
};

// bound-constrained primitives
template <class Scalar> struct BoxAbi;
#define LBFGSPP_B200_BOXABI(T, SUF)                                                                                             \
    template <> struct BoxAbi<T>                                                                                                \
    {                                                                                                                           \
        static lbfgs_b200_status clamp(lbfgs_b200_ctx* c, int64_t n, T* x, const T* lb, const T* ub) { return lbfgs_b200_box_clamp_##SUF(c, n, x, lb, ub); } \
        static lbfgs_b200_status proj_grad_norm(lbfgs_b200_ctx* c, int64_t n, const T* x, const T* g, const T* lb, const T* ub, T* o) { return lbfgs_b200_box_proj_grad_norm_##SUF(c, n, x, g, lb, ub, o); } \
        static lbfgs_b200_status dir_info(lbfgs_b200_ctx* c, int64_t n, const T* x, const T* d, const T* g, const T* lb, const T* ub, T* o) { return lbfgs_b200_box_dir_info_##SUF(c, n, x, d, g, lb, ub, o); } \
        static lbfgs_b200_status hist_wt_dot(lbfgs_b200_hist* h, const T* v, T* raw) { return lbfgs_b200_hist_wt_dot_##SUF(h, v, raw); } \
        static lbfgs_b200_status hist_gram(lbfgs_b200_hist* h, T* sy, T* ss, T* yy, T* ys, T* th) { return lbfgs_b200_hist_gram_##SUF(h, sy, ss, yy, ys, th); } \
        static lbfgs_b200_status hist_lincomb(lbfgs_b200_hist* h, lbfgs_b200_box* b, T a0, const T* v0, const T* coef, const unsigned char* cls, int mask, T* out) { return lbfgs_b200_hist_lincomb_##SUF(h, b, a0, v0, coef, cls, mask, out); } \
        static lbfgs_b200_status hist_masked_gram(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, T* G) { return lbfgs_b200_hist_masked_gram_##SUF(h, b, cls, mask, G); } \
        static lbfgs_b200_status hist_wt_dot_multi(lbfgs_b200_hist* h, int k, const T* V, int64_t ldv, T* R) { return lbfgs_b200_hist_wt_dot_multi_##SUF(h, k, V, ldv, R); } \
        static lbfgs_b200_status hist_lincomb_multi(lbfgs_b200_hist* h, T a0, int k, const T* V, int64_t ldv, const T* C, T* OUT, int64_t ldo) { return lbfgs_b200_hist_lincomb_multi_##SUF(h, a0, k, V, ldv, C, OUT, ldo); } \
        static lbfgs_b200_status hist_quad_diag(lbfgs_b200_hist* h, T a0, const T* K, T* out) { return lbfgs_b200_hist_quad_diag_##SUF(h, a0, K, out); } \
        static lbfgs_b200_status hist_wt_dot_normal(lbfgs_b200_hist* h, uint64_t seed, uint32_t stream, uint32_t first, int k, T* R) { return lbfgs_b200_hist_wt_dot_normal_##SUF(h, seed, stream, first, k, R); } \
        static lbfgs_b200_status hist_s_dot_multi(lbfgs_b200_hist* h, int k, const T* V, int64_t ldv, T* R) { return lbfgs_b200_hist_s_dot_multi_##SUF(h, k, V, ldv, R); } \
        static lbfgs_b200_status hist_wt_dot_diff(lbfgs_b200_hist* h, int k, const T* X, int64_t ldx, const T* mean, double* R, double* nrm) { return lbfgs_b200_hist_wt_dot_diff_##SUF(h, k, X, ldx, mean, R, nrm); } \
        static lbfgs_b200_status hist_lincomb_normal(lbfgs_b200_hist* h, T a0, uint64_t seed, uint32_t stream, uint32_t first, int k, const T* mean, const T* C, T* OUT, int64_t ldo) { return lbfgs_b200_hist_lincomb_normal_##SUF(h, a0, seed, stream, first, k, mean, C, OUT, ldo); } \
        static lbfgs_b200_status hist_wt_dot_multi_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, int k, const T* V, int64_t ldv, T* R) { return lbfgs_b200_hist_wt_dot_multi_masked_##SUF(h, b, cls, mask, k, V, ldv, R); } \
        static lbfgs_b200_status hist_wt_dot_diff_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, int k, const T* X, int64_t ldx, const T* mean, double* R, double* nrm) { return lbfgs_b200_hist_wt_dot_diff_masked_##SUF(h, b, cls, mask, k, X, ldx, mean, R, nrm); } \
        static lbfgs_b200_status hist_wt_dot_normal_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, uint64_t seed, uint32_t stream, uint32_t first, int k, T* R) { return lbfgs_b200_hist_wt_dot_normal_masked_##SUF(h, b, cls, mask, seed, stream, first, k, R); } \
        static lbfgs_b200_status hist_lincomb_multi_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, T a0, int k, const T* V, int64_t ldv, const T* C, T* OUT, int64_t ldo) { return lbfgs_b200_hist_lincomb_multi_masked_##SUF(h, b, cls, mask, a0, k, V, ldv, C, OUT, ldo); } \
        static lbfgs_b200_status hist_lincomb_normal_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, T a0, uint64_t seed, uint32_t stream, uint32_t first, int k, const T* mean, const T* C, T* OUT, int64_t ldo) { return lbfgs_b200_hist_lincomb_normal_masked_##SUF(h, b, cls, mask, a0, seed, stream, first, k, mean, C, OUT, ldo); } \
        static lbfgs_b200_status hist_quad_diag_masked(lbfgs_b200_hist* h, lbfgs_b200_box* b, const unsigned char* cls, int mask, T a0, const T* K, T* out) { return lbfgs_b200_hist_quad_diag_masked_##SUF(h, b, cls, mask, a0, K, out); } \
        static lbfgs_b200_status final_classes(lbfgs_b200_box* b, const T* x, const T* lb, const T* ub, T tol, int64_t* nfree) { return lbfgs_b200_box_final_classes_##SUF(b, x, lb, ub, tol, nfree); } \
        static lbfgs_b200_status cauchy_breaks(lbfgs_b200_box* b, const T* x, const T* g, const T* lb, const T* ub, T* o5) { return lbfgs_b200_box_cauchy_breaks_##SUF(b, x, g, lb, ub, o5); } \
        static lbfgs_b200_status cauchy_sweep(lbfgs_b200_box* b, const T* g, const T* M, const T* p0, T theta, T gt, int64_t nord, int64_t ninf, T* out) { return lbfgs_b200_box_cauchy_sweep_##SUF(b, g, M, p0, theta, gt, nord, ninf, out); } \
        static lbfgs_b200_status cauchy_build(lbfgs_b200_box* b, const T* x, const T* lb, const T* ub, T tc, T tf, T* cnt) { return lbfgs_b200_box_cauchy_build_##SUF(b, x, lb, ub, tc, tf, cnt); } \
        static lbfgs_b200_status sub_step(lbfgs_b200_box* b, int op, int flag, const T* x0, const T* g, const T* lb, const T* ub, T* drt, T theta, T* o3) { return lbfgs_b200_box_sub_step_##SUF(b, op, flag, x0, g, lb, ub, drt, theta, o3); } \
    };
LBFGSPP_B200_BOXABI(double, f64)
LBFGSPP_B200_BOXABI(float, f32)
#undef LBFGSPP_B200_BOXABI

}  // namespace detail

// ----------------------------------------------------------------------------------------------------
// DeviceVector
// ----------------------------------------------------------------------------------------------------
template <typename Scalar>
class DeviceVector
{
    static_assert(std::is_same<Scalar, double>::value || std::is_same<Scalar, float>::value,
                  "DeviceVector supports float and double");
    Device* m_dev;
    Scalar* m_ptr;
    std::ptrdiff_t m_size;
    std::ptrdiff_t m_capacity;

    Device& bound()
    {
        if (!m_dev) m_dev = &Device::get_default();
        return *m_dev;
    }
    void release()
    {
        if (m_ptr && m_dev) lbfgs_b200_free(m_dev->ctx(), m_ptr);
        m_ptr = nullptr;
        m_size = m_capacity = 0;
    }

public:
    typedef Scalar value_type;
    typedef std::ptrdiff_t Index;

    // A default-constructed vector is not bound to a device yet: it binds to the process-wide default device on first use
    // (or to another vector's device on assignment), so that solver objects can be created without touching a GPU.
    DeviceVector() : m_dev(nullptr), m_ptr(nullptr), m_size(0), m_capacity(0) {}
    explicit DeviceVector(Index n) : m_dev(&Device::get_default()), m_ptr(nullptr), m_size(0), m_capacity(0) { resize(n); }
    DeviceVector(Device& dev, Index n) : m_dev(&dev), m_ptr(nullptr), m_size(0), m_capacity(0) { resize(n); }
    explicit DeviceVector(Device& dev) : m_dev(&dev), m_ptr(nullptr), m_size(0), m_capacity(0) {}
    DeviceVector(const DeviceVector& o) : m_dev(o.m_dev), m_ptr(nullptr), m_size(0), m_capacity(0) { *this = o; }
    DeviceVector(DeviceVector&& o) noexcept : m_dev(o.m_dev), m_ptr(o.m_ptr), m_size(o.m_size), m_capacity(o.m_capacity)
    {
        o.m_ptr = nullptr;
        o.m_size = o.m_capacity = 0;
    }
    ~DeviceVector() { release(); }

    // deep copy on the device (the reference's `m_xp.noalias() = x`)
    DeviceVector& operator=(const DeviceVector& o)
    {
        if (this == &o) return *this;
        if (m_dev != o.m_dev) { release(); m_dev = o.m_dev; }
        resize(o.m_size);
        if (m_size > 0) m_dev->check(lbfgs_b200_memcpy_d2d(m_dev->ctx(), m_ptr, o.m_ptr, sizeof(Scalar) * size_t(m_size)));
        return *this;
    }
    DeviceVector& operator=(DeviceVector&& o) noexcept
    {
        if (this != &o) { swap(o); }
        return *this;
    }

    Device& device() const { return m_dev ? *m_dev : Device::get_default(); }
    bool is_bound_to(const Device& dev) const { return m_dev == &dev; }
    Index size() const { return m_size; }
    Scalar* data() { return m_ptr; }
    const Scalar* data() const { return m_ptr; }

    // Like Eigen's resize(): contents are unspecified afterwards.  Storage is reused when it is large enough.
    void resize(Index n)
    {
        if (n < 0) throw std::invalid_argument("DeviceVector::resize: negative size");
        if (n > m_capacity)
        {
            release();
            void* p = nullptr;
            bound().check(lbfgs_b200_malloc(m_dev->ctx(), &p, sizeof(Scalar) * size_t(n)));
            m_ptr = static_cast<Scalar*>(p);
            m_capacity = n;
        }
        m_size = n;
    }

    void swap(DeviceVector& o) noexcept
    {
        std::swap(m_dev, o.m_dev);
        std::swap(m_ptr, o.m_ptr);
        std::swap(m_size, o.m_size);
        std::swap(m_capacity, o.m_capacity);
    }

    void setZero()
    {
        if (m_size > 0) m_dev->check(lbfgs_b200_memset_zero(m_dev->ctx(), m_ptr, sizeof(Scalar) * size_t(m_size)));
    }

    // ---- host transfers ---------------------------------------------------------------------------
    void copy_from_host(const Scalar* src, Index n)
    {
        resize(n);
        if (n > 0)
        {
            m_dev->check(lbfgs_b200_memcpy_h2d(m_dev->ctx(), m_ptr, src, sizeof(Scalar) * size_t(n)));
            m_dev->synchronize();  // `src` may be pageable and reused by the caller right away
        }
    }
    void copy_to_host(Scalar* dst) const
    {
        if (m_size > 0) m_dev->check(lbfgs_b200_memcpy_d2h(m_dev->ctx(), dst, m_ptr, sizeof(Scalar) * size_t(m_size)));
    }
    std::vector<Scalar> to_std_vector() const
    {
        std::vector<Scalar> out(static_cast<size_t>(m_size));
        copy_to_host(out.data());
        return out;
    }
    static DeviceVector from_host(const std::vector<Scalar>& v)
    {
        DeviceVector out;
        out.copy_from_host(v.data(), Index(v.size()));
        return out;
    }
    static DeviceVector Zero(Index n)
    {
        DeviceVector out(n);
        out.setZero();
        return out;
    }
    static DeviceVector Constant(Index n, Scalar value)
    {
        std::vector<Scalar> h(static_cast<size_t>(n), value);
        return from_host(h);
    }

    // ---- reductions (each one kernel + one host synchronisation) -----------------------------------
    Scalar dot(const DeviceVector& o) const
    {
        if (o.m_size != m_size) throw std::invalid_argument("DeviceVector::dot: size mismatch");
        Scalar r = Scalar(0);
        if (m_size > 0) m_dev->check(detail::Abi<Scalar>::dot(m_dev->ctx(), m_size, m_ptr, o.m_ptr, &r));
        return r;
    }
    Scalar squaredNorm() const { return dot(*this); }
    Scalar norm() const { return std::sqrt(squaredNorm()); }
};

}  // namespace LBFGSpp

#endif  // LBFGSPP_B200_DEVICE_VECTOR_H
