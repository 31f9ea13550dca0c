// owlqn_oracle_weighted_capi.cpp -- C entry points of the weighted OWL-QN checker (owlqn_oracle_weighted.hpp) for the tests, in the
// result layout of the driver's lbfgsb200_drv_owlqn_* (status, msg, niter, nfev, fx, gnorm).  TEST INFRASTRUCTURE ONLY.
#include <cstring>
#include <stdexcept>

#include "owlqn_oracle_weighted.hpp"

extern "C" {

typedef struct
{
    int status;   // 0 ok, 1 invalid_argument, 2 logic_error, 3 runtime_error, 4 other
    char msg[200];
    int niter;
    long nfev;
    double fx;
    double gnorm;
} owlqn_oracle_result;

}  // extern "C"

namespace {

template <class T>
int run(int objective, const T* d0, const T* d1, long n, const orc_param* p, double lam, const T* w, int sum_mode, T* x, T* grad,
        owlqn_oracle_result* out)
{
    std::memset(out, 0, sizeof(*out));
    std::vector<T> g(n);
    long nfev = 0;
    auto fail = [&](int code, const char* what) {
        out->status = code;
        std::strncpy(out->msg, what, sizeof(out->msg) - 1);
    };
    try
    {
        const orc_owlqn::Outcome o =
            orc_owlqn::minimize_weighted<T>(objective, d0, d1, n, *p, T(lam), w, orc::Blas1<T>(sum_mode, 1), x, g.data(), nfev);
        out->niter = o.niter;
        out->fx = o.fx;
        out->gnorm = o.gnorm;
        if (grad) std::memcpy(grad, g.data(), sizeof(T) * n);
    }
    catch (const std::invalid_argument& e) { fail(1, e.what()); }
    catch (const std::logic_error& e) { fail(2, e.what()); }
    catch (const std::runtime_error& e) { fail(3, e.what()); }
    out->nfev = nfev;
    return out->status;
}

}  // namespace

extern "C" {

// w: n weights; sum_mode: ORC_SUM_SEQUENTIAL or ORC_SUM_LANES8 (oracle/oracle_api.h).  x: start point in, solution out.
int owlqn_oracle_weighted_f64(int objective, const double* d0, const double* d1, long n, const orc_param* p, double lam, const double* w,
                              int sum_mode, double* x, double* grad, owlqn_oracle_result* out)
{
    return run<double>(objective, d0, d1, n, p, lam, w, sum_mode, x, grad, out);
}
int owlqn_oracle_weighted_f32(int objective, const float* d0, const float* d1, long n, const orc_param* p, double lam, const float* w,
                              int sum_mode, float* x, float* grad, owlqn_oracle_result* out)
{
    return run<float>(objective, d0, d1, n, p, lam, w, sum_mode, x, grad, out);
}

}  // extern "C"
