"""lbfgspp_b200 -- H100-native L-BFGS hot path behind LBFGSpp's solver interface.

Layers (top to bottom):
  LBFGSParam / LBFGSSolver (this module)   Python mirror of the reference's classes for tests and bench.py;
                                           calls the C++ front through liblbfgs_b200_driver.so
  include/LBFGS.h, include/LBFGSpp/*.h     header-only C++ front = the drop-in (same class names as the reference)
  include/lbfgs_b200.h                     C ABI
  csrc/*.cu                                hand-written sm_90a kernels (liblbfgs_b200.so)

There is no CPU fallback: importing works anywhere, but creating a Context / solving raises unless the CUDA
library is built (lbfgspp_b200.build.build_all()) and an H100 is present.
"""
import ctypes as C
import os

import numpy as np

from . import build as _build

PKG = os.path.dirname(os.path.abspath(__file__))

OBJ_ROSENBROCK_PAIRED, OBJ_QUAD_SHIFT, OBJ_ROSENBROCK_CHAINED, OBJ_QUAD_TRIDIAG = 0, 1, 2, 3
HV_AUTO, HV_TWO_LOOP, HV_GRAM = 0, 1, 2
LINE_SEARCHES = {"Backtracking": 0, "Bracketing": 1, "NocedalWright": 2, "MoreThuente": 3}
LBFGS_LINESEARCH_BACKTRACKING_ARMIJO = 1
LBFGS_LINESEARCH_BACKTRACKING = 2
LBFGS_LINESEARCH_BACKTRACKING_WOLFE = 2
LBFGS_LINESEARCH_BACKTRACKING_STRONG_WOLFE = 3


class NativeLibraryMissing(RuntimeError):
    pass


class LbfgsB200Error(RuntimeError):
    def __init__(self, status, message):
        super().__init__("lbfgs_b200 status %d: %s" % (status, message))
        self.status = status


_libs = {}


def _load(name):
    if name not in _libs:
        path = os.path.join(PKG, name)
        if not os.path.exists(path):
            raise NativeLibraryMissing(
                "%s is not built; run `python -m lbfgspp_b200.build` (there is no CPU fallback)" % path)
        _libs[name] = C.CDLL(path)   # RTLD_LOCAL: nothing here may interpose with other loaded libraries
    return _libs[name]


def abi():
    """The raw C ABI (include/lbfgs_b200.h) as a ctypes library with argument types declared."""
    return _declare(_load("liblbfgs_b200.so"))


def _declare(lib):
    """Declare the argument and result types of every lbfgs_b200_* entry point on `lib` (any library exporting the ABI)."""
    if getattr(lib, "_typed", False):
        return lib
    vp, i64, ci, sz = C.c_void_p, C.c_int64, C.c_int, C.c_size_t
    lib.lbfgs_b200_version.restype = C.c_char_p
    lib.lbfgs_b200_last_error.restype = C.c_char_p
    lib.lbfgs_b200_last_error.argtypes = [vp]
    lib.lbfgs_b200_ctx_create.argtypes = [C.POINTER(vp), ci, vp]
    lib.lbfgs_b200_ctx_destroy.argtypes = [vp]
    lib.lbfgs_b200_ctx_destroy.restype = None
    lib.lbfgs_b200_stream.restype = vp
    lib.lbfgs_b200_stream.argtypes = [vp]
    lib.lbfgs_b200_sm_count.argtypes = [vp]
    lib.lbfgs_b200_launch_count.restype = C.c_uint64
    lib.lbfgs_b200_launch_count.argtypes = [vp]
    lib.lbfgs_b200_malloc.argtypes = [vp, C.POINTER(vp), sz]
    lib.lbfgs_b200_free.argtypes = [vp, vp]
    lib.lbfgs_b200_memcpy_h2d.argtypes = [vp, vp, vp, sz]
    lib.lbfgs_b200_memcpy_d2h.argtypes = [vp, vp, vp, sz]
    lib.lbfgs_b200_memcpy_d2d.argtypes = [vp, vp, vp, sz]
    lib.lbfgs_b200_memset_zero.argtypes = [vp, vp, sz]
    lib.lbfgs_b200_sync.argtypes = [vp]
    lib.lbfgs_b200_trim.argtypes = [vp]
    lib.lbfgs_b200_timer_start.argtypes = [vp]
    lib.lbfgs_b200_timer_stop.argtypes = [vp, C.POINTER(C.c_float)]
    lib.lbfgs_b200_set_index_offset.argtypes = [vp, i64]
    lib.lbfgs_b200_profile_enable.argtypes = [vp, ci]
    lib.lbfgs_b200_profile_read.argtypes = [vp, ci, C.POINTER(C.c_double), C.POINTER(C.c_uint64), ci]
    lib.lbfgs_b200_profile_bytes.argtypes = [vp, ci, C.POINTER(C.c_double), ci]
    lib.lbfgs_b200_comm_unique_id.argtypes = [vp]
    lib.lbfgs_b200_comm_init.argtypes = [vp, vp, ci, ci]
    lib.lbfgs_b200_comm_size.argtypes = [vp]
    lib.lbfgs_b200_hist_create.argtypes = [vp, C.POINTER(vp), i64, ci, ci]
    lib.lbfgs_b200_hist_destroy.argtypes = [vp]
    lib.lbfgs_b200_hist_destroy.restype = None
    lib.lbfgs_b200_hist_reset.argtypes = [vp]
    lib.lbfgs_b200_hist_ncorr.argtypes = [vp]
    lib.lbfgs_b200_hist_m.argtypes = [vp]
    lib.lbfgs_b200_hist_s_col.restype = vp
    lib.lbfgs_b200_hist_s_col.argtypes = [vp, ci]
    lib.lbfgs_b200_hist_y_col.restype = vp
    lib.lbfgs_b200_hist_y_col.argtypes = [vp, ci]
    for suf, ct in (("f64", C.c_double), ("f32", C.c_float)):
        pt = C.POINTER(ct)
        getattr(lib, "lbfgs_b200_dot_" + suf).argtypes = [vp, i64, vp, vp, pt]
        getattr(lib, "lbfgs_b200_dot3_" + suf).argtypes = [vp, i64, vp, vp, vp, pt]
        getattr(lib, "lbfgs_b200_axpy_out_" + suf).argtypes = [vp, i64, vp, ct, vp, vp]
        getattr(lib, "lbfgs_b200_scale_out_" + suf).argtypes = [vp, i64, ct, vp, vp]
        getattr(lib, "lbfgs_b200_objective_" + suf).argtypes = [vp, ci, vp, vp, i64, vp, vp, pt]
        getattr(lib, "lbfgs_b200_trial_" + suf).argtypes = [vp, ci, vp, vp, i64, vp, vp, ct, vp, vp, pt]
        getattr(lib, "lbfgs_b200_hist_update_" + suf).argtypes = [vp, vp, vp, vp, vp, ct, C.POINTER(ci), pt]
        getattr(lib, "lbfgs_b200_hist_add_" + suf).argtypes = [vp, vp, vp]
        getattr(lib, "lbfgs_b200_hist_apply_Hv_" + suf).argtypes = [vp, vp, ct, vp, ci, pt]
        getattr(lib, "lbfgs_b200_hist_update_apply_Hv_" + suf).argtypes = [vp, vp, vp, vp, vp, ct, ct, vp, ci, C.POINTER(ci), pt]
        getattr(lib, "lbfgs_b200_hist_scalars_" + suf).argtypes = [vp, pt, pt, pt]
        if hasattr(lib, "lbfgs_b200_owlqn_trial_" + suf):
            getattr(lib, "lbfgs_b200_owlqn_trial_" + suf).argtypes = [vp, ci, vp, vp, i64, vp, vp, vp, ct, ct, vp, vp, pt]
            getattr(lib, "lbfgs_b200_owlqn_project_" + suf).argtypes = [vp, i64, vp, vp, vp, ct, ct, vp, pt]
            getattr(lib, "lbfgs_b200_owlqn_sums_" + suf).argtypes = [vp, i64, vp, vp, ct, vp, pt]
            getattr(lib, "lbfgs_b200_owlqn_update_dir_" + suf).argtypes = [vp, vp, vp, vp, vp, ct, ct, vp, C.POINTER(ci), pt]
        if hasattr(lib, "lbfgs_b200_owlqn_weighted_trial_" + suf):
            getattr(lib, "lbfgs_b200_owlqn_weighted_trial_" + suf).argtypes = [vp, ci, vp, vp, i64, vp, vp, vp, ct, ct, vp, vp, vp, pt]
            getattr(lib, "lbfgs_b200_owlqn_weighted_project_" + suf).argtypes = [vp, i64, vp, vp, vp, ct, ct, vp, vp, pt]
            getattr(lib, "lbfgs_b200_owlqn_weighted_sums_" + suf).argtypes = [vp, i64, vp, vp, ct, vp, vp, pt]
            getattr(lib, "lbfgs_b200_owlqn_weighted_update_dir_" + suf).argtypes = [vp, vp, vp, vp, vp, ct, ct, vp, vp, C.POINTER(ci), pt]
    # bound-constrained path
    lib.lbfgs_b200_box_create.argtypes = [vp, C.POINTER(vp)]
    lib.lbfgs_b200_box_destroy.argtypes = [vp]
    lib.lbfgs_b200_box_destroy.restype = None
    for name in ("lbfgs_b200_box_xcp", "lbfgs_b200_box_classes"):
        getattr(lib, name).restype = vp
        getattr(lib, name).argtypes = [vp]
    lib.lbfgs_b200_box_vector.restype = vp
    lib.lbfgs_b200_box_vector.argtypes = [vp, ci]
    for suf, ct in (("f64", C.c_double), ("f32", C.c_float)):
        pt = C.POINTER(ct)
        getattr(lib, "lbfgs_b200_box_clamp_" + suf).argtypes = [vp, i64, vp, vp, vp]
        getattr(lib, "lbfgs_b200_box_proj_grad_norm_" + suf).argtypes = [vp, i64, vp, vp, vp, vp, pt]
        getattr(lib, "lbfgs_b200_box_dir_info_" + suf).argtypes = [vp, i64, vp, vp, vp, vp, vp, pt]
        getattr(lib, "lbfgs_b200_hist_wt_dot_" + suf).argtypes = [vp, vp, pt]
        getattr(lib, "lbfgs_b200_hist_gram_" + suf).argtypes = [vp, pt, pt, pt, pt, pt]
        getattr(lib, "lbfgs_b200_hist_lincomb_" + suf).argtypes = [vp, vp, ct, vp, pt, vp, ci, vp]
        getattr(lib, "lbfgs_b200_hist_masked_gram_" + suf).argtypes = [vp, vp, vp, ci, pt]
        if hasattr(lib, "lbfgs_b200_hist_wt_dot_multi_" + suf):   # the k-vector passes (a test double of the ABI may lack them)
            getattr(lib, "lbfgs_b200_hist_wt_dot_multi_" + suf).argtypes = [vp, ci, vp, i64, pt]
            getattr(lib, "lbfgs_b200_hist_lincomb_multi_" + suf).argtypes = [vp, ct, ci, vp, i64, pt, vp, i64]
        if hasattr(lib, "lbfgs_b200_hist_quad_diag_" + suf):      # the diagonal pass (a test double of the ABI may lack it)
            getattr(lib, "lbfgs_b200_hist_quad_diag_" + suf).argtypes = [vp, ct, pt, vp]
        if hasattr(lib, "lbfgs_b200_hist_wt_dot_normal_" + suf):  # the sampler's passes (a test double of the ABI may lack them)
            getattr(lib, "lbfgs_b200_hist_wt_dot_normal_" + suf).argtypes = [vp, C.c_uint64, C.c_uint32, C.c_uint32, ci, pt]
            getattr(lib, "lbfgs_b200_hist_lincomb_normal_" + suf).argtypes = [vp, ct, C.c_uint64, C.c_uint32, C.c_uint32, ci, vp, pt, vp, i64]
        if hasattr(lib, "lbfgs_b200_hist_s_dot_multi_" + suf):    # the whitening passes (a test double of the ABI may lack them)
            getattr(lib, "lbfgs_b200_hist_s_dot_multi_" + suf).argtypes = [vp, ci, vp, i64, pt]
            getattr(lib, "lbfgs_b200_hist_wt_dot_diff_" + suf).argtypes = [vp, ci, vp, i64, vp, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        if hasattr(lib, "lbfgs_b200_box_final_classes_" + suf):   # the free-set passes (a test double of the ABI may lack them)
            u64, u32, cls = C.c_uint64, C.c_uint32, C.POINTER(C.c_ubyte)
            getattr(lib, "lbfgs_b200_hist_wt_dot_multi_masked_" + suf).argtypes = [vp, vp, vp, ci, ci, vp, i64, pt]
            getattr(lib, "lbfgs_b200_hist_wt_dot_diff_masked_" + suf).argtypes = [vp, vp, vp, ci, ci, vp, i64, vp, C.POINTER(C.c_double),
                                                                                  C.POINTER(C.c_double)]
            getattr(lib, "lbfgs_b200_hist_wt_dot_normal_masked_" + suf).argtypes = [vp, vp, vp, ci, u64, u32, u32, ci, pt]
            getattr(lib, "lbfgs_b200_hist_lincomb_multi_masked_" + suf).argtypes = [vp, vp, vp, ci, ct, ci, vp, i64, pt, vp, i64]
            getattr(lib, "lbfgs_b200_hist_lincomb_normal_masked_" + suf).argtypes = [vp, vp, vp, ci, ct, u64, u32, u32, ci, vp, pt, vp, i64]
            getattr(lib, "lbfgs_b200_hist_quad_diag_masked_" + suf).argtypes = [vp, vp, vp, ci, ct, pt, vp]
            getattr(lib, "lbfgs_b200_box_final_classes_" + suf).argtypes = [vp, vp, vp, vp, ct, C.POINTER(i64)]
        getattr(lib, "lbfgs_b200_box_cauchy_breaks_" + suf).argtypes = [vp, vp, vp, vp, vp, pt]
        getattr(lib, "lbfgs_b200_box_cauchy_sweep_" + suf).argtypes = [vp, vp, pt, pt, ct, ct, i64, i64, pt]
        getattr(lib, "lbfgs_b200_box_cauchy_build_" + suf).argtypes = [vp, vp, vp, vp, ct, ct, pt]
        getattr(lib, "lbfgs_b200_box_sub_step_" + suf).argtypes = [vp, ci, ci, vp, vp, vp, vp, vp, ct, pt]
    # device-resident solve (persistent kernel; single problem or batch)
    lib.lbfgs_b200_solver_create.argtypes = [vp, i64, ci, ci, C.POINTER(vp)]
    lib.lbfgs_b200_solver_create_batch.argtypes = [vp, i64, ci, ci, ci, C.POINTER(vp)]
    lib.lbfgs_b200_solver_destroy.argtypes = [vp]
    lib.lbfgs_b200_solver_destroy.restype = None
    lib.lbfgs_b200_solver_batch.argtypes = [vp]
    lib.lbfgs_b200_solver_profile.argtypes = [vp, vp, vp, vp, vp, vp]
    for name in ("lbfgs_b200_solver_final_grad", "lbfgs_b200_solver_history"):
        getattr(lib, name).restype = vp
        getattr(lib, name).argtypes = [vp]
    for name in ("lbfgs_b200_solver_final_grad_of", "lbfgs_b200_solver_history_of"):
        getattr(lib, name).restype = vp
        getattr(lib, name).argtypes = [vp, ci]
    for suf in ("f64", "f32"):
        getattr(lib, "lbfgs_b200_solver_minimize_" + suf).argtypes = [vp, ci, vp, vp, vp, ci, vp, vp, C.c_longlong, vp]
        getattr(lib, "lbfgs_b200_solver_minimize_batch_" + suf).argtypes = [vp, ci, vp, vp, i64, vp, ci, vp, i64, vp]
    # small-batch solve (one thread block per problem; a test double of the ABI may lack it)
    if hasattr(lib, "lbfgs_b200_small_max_n"):
        lib.lbfgs_b200_small_max_n.restype = i64
        lib.lbfgs_b200_small_max_n.argtypes = [ci, ci, ci]
        for suf in ("f64", "f32"):
            getattr(lib, "lbfgs_b200_small_minimize_" + suf).argtypes = [vp, ci, vp, vp, i64, i64, i64, vp, ci, vp, i64, vp, vp]
    if hasattr(lib, "lbfgs_b200_small_hist_create"):
        lib.lbfgs_b200_small_hist_create.argtypes = [vp, i64, ci, ci, i64, C.POINTER(vp)]
        lib.lbfgs_b200_small_hist_destroy.argtypes = [vp]
        lib.lbfgs_b200_small_hist_destroy.restype = None
        for name in ("lbfgs_b200_small_hist_s_col", "lbfgs_b200_small_hist_y_col"):
            getattr(lib, name).restype = vp
            getattr(lib, name).argtypes = [vp, i64, ci]
        for suf in ("f64", "f32"):
            getattr(lib, "lbfgs_b200_small_minimize_keep_" + suf).argtypes = [vp, ci, vp, vp, i64, i64, i64, vp, ci, vp, i64, vp, vp, vp]
            getattr(lib, "lbfgs_b200_small_hist_info_" + suf).argtypes = [vp, vp, vp]
            getattr(lib, "lbfgs_b200_small_hist_times_" + suf).argtypes = [vp, ci, i64, i64, ci, vp, i64, i64, vp, i64, i64]
            getattr(lib, "lbfgs_b200_small_hist_diag_" + suf).argtypes = [vp, ci, i64, i64, vp, i64]
            if hasattr(lib, "lbfgs_b200_small_hist_sample_" + suf):
                getattr(lib, "lbfgs_b200_small_hist_factor_times_" + suf).argtypes = [vp, i64, i64, ci, vp, i64, i64, vp, i64, i64]
                getattr(lib, "lbfgs_b200_small_hist_sample_" + suf).argtypes = [vp, C.c_uint64, C.c_uint32, i64, i64, ci, vp, i64, vp, i64, i64]
                getattr(lib, "lbfgs_b200_small_hist_logdet_" + suf).argtypes = [vp, i64, i64, C.POINTER(C.c_double)]
            if hasattr(lib, "lbfgs_b200_small_hist_factor_apply_" + suf):
                getattr(lib, "lbfgs_b200_small_hist_factor_apply_" + suf).argtypes = [vp, ci, i64, i64, ci, vp, i64, i64, vp, i64, i64]
                getattr(lib, "lbfgs_b200_small_hist_log_density_" + suf).argtypes = [vp, i64, i64, ci, vp, i64, i64, vp, i64,
                                                                                     C.POINTER(C.c_double)]
    lib._typed = True
    return lib


class _DrvParam(C.Structure):
    _fields_ = [("m", C.c_int), ("epsilon", C.c_double), ("epsilon_rel", C.c_double), ("past", C.c_int),
                ("delta", C.c_double), ("max_iterations", C.c_int), ("linesearch", C.c_int),
                ("max_submin", C.c_int), ("max_linesearch", C.c_int), ("min_step", C.c_double),
                ("max_step", C.c_double), ("ftol", C.c_double), ("wolfe", C.c_double)]


class _BatchItem(C.Structure):
    _fields_ = [("status", C.c_int), ("niter", C.c_int), ("nfev", C.c_long), ("fx", C.c_double), ("gnorm", C.c_double)]


class _AbiParam(C.Structure):
    """lbfgs_b200_param"""
    _fields_ = [("m", C.c_int), ("epsilon", C.c_double), ("epsilon_rel", C.c_double), ("past", C.c_int), ("delta", C.c_double),
                ("max_iterations", C.c_int), ("linesearch", C.c_int), ("max_linesearch", C.c_int), ("min_step", C.c_double),
                ("max_step", C.c_double), ("ftol", C.c_double), ("wolfe", C.c_double)]


class _Outcome(C.Structure):
    """lbfgs_b200_outcome"""
    _fields_ = [("status", C.c_int), ("niter", C.c_int), ("nfev", C.c_longlong), ("fx", C.c_double), ("gnorm", C.c_double),
                ("rounds", C.c_longlong)]


class _SmallItem(C.Structure):
    _fields_ = [("code", C.c_int), ("kind", C.c_int), ("niter", C.c_int), ("nfev", C.c_long), ("fx", C.c_double), ("gnorm", C.c_double),
                ("rounds", C.c_long)]


class _DrvResult(C.Structure):
    _fields_ = [("status", C.c_int), ("msg", C.c_char * 200), ("niter", C.c_int), ("nfev", C.c_long),
                ("fx", C.c_double), ("gnorm", C.c_double), ("trace_len", C.c_long), ("seconds", C.c_double),
                ("seconds_e2e", C.c_double), ("launches", C.c_ulonglong), ("h2d_bytes", C.c_long),
                ("d2h_bytes", C.c_long)]


class _OwlqnResult(C.Structure):
    _fields_ = [("status", C.c_int), ("msg", C.c_char * 200), ("niter", C.c_int), ("nfev", C.c_long), ("fx", C.c_double),
                ("gnorm", C.c_double), ("seconds", C.c_double)]


def driver(lib=None):
    """liblbfgs_b200_driver.so, or `lib` (a library exporting the same entry points, e.g. built on a test double), typed."""
    if lib is not None:
        return _declare_driver(lib)
    abi()  # the driver links against the kernel library: load it first, globally
    return _declare_driver(_load("liblbfgs_b200_driver.so"))


def _declare_driver(lib):
    """Declare the argument and result types of every lbfgsb200_drv_* entry point on `lib` (any library exporting the driver)."""
    if getattr(lib, "_drv_typed", False):
        return lib
    vp, ci, cl, err, errlen = C.c_void_p, C.c_int, C.c_long, C.c_char_p, C.c_int
    dp, fp = C.POINTER(C.c_double), C.POINTER(C.c_float)
    prm, res, item = C.POINTER(_DrvParam), C.POINTER(_DrvResult), C.POINTER(_BatchItem)
    for suf, pt in (("f64", dp), ("f32", fp)):
        getattr(lib, "lbfgsb200_drv_lbfgs_" + suf).argtypes = [ci, ci, pt, pt, cl, ci, prm, ci, ci, pt, pt, dp, cl, res]
        getattr(lib, "lbfgsb200_drv_lbfgsb_" + suf).argtypes = [ci, ci, pt, pt, cl, prm, pt, pt, pt, pt, dp, cl, res]
    for name in ("ctx", "session_create", "batch_session_create"):
        getattr(lib, "lbfgsb200_drv_" + name).restype = vp
    for name in ("shutdown", "session_destroy", "batch_session_destroy", "phase_enable"):
        getattr(lib, "lbfgsb200_drv_" + name).restype = None
    lib.lbfgsb200_drv_ctx.argtypes = [ci]
    lib.lbfgsb200_drv_shutdown.argtypes = []
    lib.lbfgsb200_drv_session_create.argtypes = [ci, ci, dp, dp, cl, ci, prm, ci, dp, err, errlen, ci]
    lib.lbfgsb200_drv_session_destroy.argtypes = [vp]
    lib.lbfgsb200_drv_session_solve.argtypes = [vp, ci, ci, res]
    lib.lbfgsb200_drv_session_result.restype = dp
    lib.lbfgsb200_drv_session_result.argtypes = [vp]
    lib.lbfgsb200_drv_session_download.argtypes = [vp, dp]
    lib.lbfgsb200_drv_comm_init.argtypes = [ci, vp, ci, ci, C.c_longlong, err, errlen]
    lib.lbfgsb200_drv_p2p_export.argtypes = [ci, vp, err, errlen]
    lib.lbfgsb200_drv_p2p_attach.argtypes = [ci, vp, ci, ci, C.c_longlong, err, errlen]
    lib.lbfgsb200_drv_set_global_extent.argtypes = [ci, C.c_longlong, C.c_longlong, err, errlen]
    lib.lbfgsb200_drv_cauchy_f64.argtypes = [ci, cl, ci, ci, dp, dp, dp, dp, dp, dp, dp, C.POINTER(C.c_ubyte), dp, C.POINTER(cl), dp, err, errlen]
    lib.lbfgsb200_drv_batch_f64.argtypes = [ci, ci, cl, ci, dp, ci, prm, ci, ci, ci, item, dp, dp]
    lib.lbfgsb200_drv_batch_session_create.argtypes = [ci, ci, cl, ci, dp, ci, prm, err, errlen]
    lib.lbfgsb200_drv_batch_session_destroy.argtypes = [vp]
    lib.lbfgsb200_drv_batch_session_download.argtypes = [vp, dp]
    lib.lbfgsb200_drv_batch_session_upload.argtypes = [vp, dp, err, errlen]
    lib.lbfgsb200_drv_batch_session_solve.argtypes = [vp, item, C.POINTER(cl), dp, dp, err, errlen]
    for name in ("lbfgsb200_drv_session_profile", "lbfgsb200_drv_batch_session_profile"):
        getattr(lib, name).argtypes = [vp, dp, dp, C.POINTER(C.c_ulonglong), dp, dp]
    lib.lbfgsb200_drv_solve_dense_f64.argtypes = [ci, ci, cl, ci, prm, ci, dp, dp, dp, C.POINTER(ci), err, errlen]
    lib.lbfgsb200_drv_phase_enable.argtypes = [ci]
    lib.lbfgsb200_drv_phase_report.argtypes = [C.c_char_p, ci]
    lib.lbfgsb200_drv_dense_f64.argtypes = [ci, cl, ci, ci, dp, dp, ci, dp, err, errlen]
    # the operator form of the final approximation (csrc/driver_hessian_ops.cpp): a library built from driver.cpp alone lacks it
    if hasattr(lib, "lbfgsb200_drv_solve_hessian_times_f64"):
        lib.lbfgsb200_drv_solve_hessian_times_f64.argtypes = [ci, ci, cl, ci, prm, ci, dp, dp, cl, dp, dp, dp, C.POINTER(ci), err, errlen]
        lib.lbfgsb200_drv_batch_hessian_times_f64.argtypes = [ci, ci, cl, ci, dp, ci, prm, ci, dp, cl, dp, dp, dp, err, errlen]
        lib.lbfgsb200_drv_hist_times_f64.argtypes = [ci, cl, ci, ci, dp, dp, dp, cl, dp, dp, err, errlen]
    # the small-batch solve (csrc/driver_small_batch.cpp)
    if hasattr(lib, "lbfgsb200_drv_small_batch_f64"):
        for suf, pt in (("f64", dp), ("f32", fp)):
            getattr(lib, "lbfgsb200_drv_small_batch_" + suf).argtypes = [ci, ci, cl, cl, pt, pt, pt, cl, ci, prm, pt, pt,
                                                                         C.POINTER(_SmallItem), err, errlen]
    if hasattr(lib, "lbfgsb200_drv_small_batch_hessian_times_f64"):
        for suf, pt in (("f64", dp), ("f32", fp)):
            getattr(lib, "lbfgsb200_drv_small_batch_hessian_times_" + suf).argtypes = [ci, ci, cl, cl, pt, pt, pt, cl, ci, prm, pt, cl, ci, pt,
                                                                                      pt, pt, pt, C.POINTER(_SmallItem), err, errlen]
    # the diagonals of the final approximation (csrc/driver_hessian_diag.cpp)
    if hasattr(lib, "lbfgsb200_drv_solve_hessian_diag_f64"):
        lib.lbfgsb200_drv_solve_hessian_diag_f64.argtypes = [ci, ci, cl, ci, prm, ci, dp, dp, dp, C.POINTER(ci), err, errlen]
        lib.lbfgsb200_drv_batch_hessian_diag_f64.argtypes = [ci, ci, cl, ci, dp, ci, prm, ci, dp, dp, err, errlen]
        lib.lbfgsb200_drv_hist_diag_f64.argtypes = [ci, cl, ci, ci, dp, dp, dp, dp, err, errlen]
        for suf, pt in (("f64", dp), ("f32", fp)):
            getattr(lib, "lbfgsb200_drv_small_batch_hessian_diag_" + suf).argtypes = [ci, ci, cl, cl, pt, pt, pt, cl, ci, prm, pt, pt, pt,
                                                                                     C.POINTER(_SmallItem), err, errlen]
    # N(x*, H) from the final approximation (csrc/driver_hessian_sample.cpp)
    if hasattr(lib, "lbfgsb200_drv_solve_hessian_sample_f64"):
        u64, u32 = C.c_uint64, C.c_uint32
        lib.lbfgsb200_drv_solve_hessian_sample_f64.argtypes = [ci, ci, cl, ci, prm, ci, dp, ci, dp, dp, u64, u32, ci, dp, dp, C.POINTER(ci), err,
                                                               errlen]
        lib.lbfgsb200_drv_batch_hessian_sample_f64.argtypes = [ci, ci, cl, ci, dp, ci, prm, ci, ci, dp, dp, u64, u32, ci, dp, dp, dp, err, errlen]
        lib.lbfgsb200_drv_hist_sample_f64.argtypes = [ci, cl, ci, ci, dp, dp, ci, dp, dp, dp, u64, u32, u32, ci, dp, dp, err, errlen]
        for suf, pt in (("f64", dp), ("f32", fp)):
            getattr(lib, "lbfgsb200_drv_small_batch_hessian_sample_" + suf).argtypes = [ci, ci, cl, cl, pt, pt, pt, cl, ci, prm, pt, ci, pt, pt, u64,
                                                                                       u32, ci, pt, dp, C.POINTER(_SmallItem), err, errlen]
    # whitening and log densities under N(x*, H) (csrc/driver_hessian_whiten.cpp)
    if hasattr(lib, "lbfgsb200_drv_solve_hessian_whiten_f64"):
        lib.lbfgsb200_drv_solve_hessian_whiten_f64.argtypes = [ci, ci, cl, ci, prm, ci, dp, ci, ci, dp, dp, ci, dp, dp, dp, C.POINTER(ci), err,
                                                               errlen]
        lib.lbfgsb200_drv_batch_hessian_whiten_f64.argtypes = [ci, ci, cl, ci, dp, ci, prm, ci, ci, ci, dp, dp, ci, dp, dp, dp, dp, err, errlen]
        lib.lbfgsb200_drv_hist_whiten_f64.argtypes = [ci, cl, ci, ci, dp, dp, ci, ci, dp, dp, ci, dp, dp, dp, err, errlen]
        for suf, pt in (("f64", dp), ("f32", fp)):
            getattr(lib, "lbfgsb200_drv_small_batch_hessian_whiten_" + suf).argtypes = [ci, ci, cl, cl, pt, pt, pt, cl, ci, prm, pt, ci, ci, pt, pt,
                                                                                       ci, pt, pt, dp, cl, C.POINTER(_SmallItem), err, errlen]
    # the final approximation of a bound-constrained solve (csrc/driver_box_hessian.cpp)
    if hasattr(lib, "lbfgsb200_drv_box_hessian_f64"):
        u64, u32 = C.c_uint64, C.c_uint32
        for suf, pt in (("f64", dp), ("f32", fp)):
            getattr(lib, "lbfgsb200_drv_box_hessian_" + suf).argtypes = [ci, ci, cl, prm, pt, pt, pt, ci, C.c_double, ci, ci, pt, pt, C.c_ulonglong,
                                                                         C.c_uint, pt, dp, dp, C.POINTER(cl), C.POINTER(ci), err, errlen]
        lib.lbfgsb200_drv_box_hist_hessian_f64.argtypes = [ci, cl, ci, ci, dp, dp, ci, C.POINTER(C.c_ubyte), ci, ci, dp, dp, C.c_ulonglong,
                                                           C.c_uint, dp, dp, dp, C.POINTER(cl), err, errlen]
    # the L1-regularised solve (csrc/driver_owlqn.cpp)
    if hasattr(lib, "lbfgsb200_drv_owlqn_f64"):
        for suf, pt in (("f64", dp), ("f32", fp)):
            getattr(lib, "lbfgsb200_drv_owlqn_" + suf).argtypes = [ci, ci, pt, pt, cl, prm, C.c_double, pt, ci, pt, pt,
                                                                   C.POINTER(_OwlqnResult)]
    lib._drv_typed = True
    return lib


def _checked(what, call, failed=bool):
    """call(err, errlen) runs an entry point that reports failure as text in (err, errlen): its result, or
    RuntimeError("<what> failed: <text>") when failed(result)."""
    err = C.create_string_buffer(256)
    r = call(err, len(err))
    if failed(r):
        raise RuntimeError("%s failed: %s" % (what, err.value.decode()))
    return r


def _ls_id(linesearch):
    return LINE_SEARCHES[linesearch] if isinstance(linesearch, str) else int(linesearch)


def _ptr(a):
    """A pointer to the data of a float64 / float32 array, None for None."""
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_float if a.dtype == np.float32 else C.c_double))


# ------------------------------------------------------------------------------------------------------
# Python mirror of the reference's classes
# ------------------------------------------------------------------------------------------------------
class LBFGSParam:
    """Same fields and defaults as LBFGSpp::LBFGSParam<Scalar> (reference Param.h:171-182)."""

    def __init__(self, **kw):
        self.m = 6
        self.epsilon = 1e-5
        self.epsilon_rel = 1e-5
        self.past = 0
        self.delta = 0.0
        self.max_iterations = 0
        self.linesearch = LBFGS_LINESEARCH_BACKTRACKING_STRONG_WOLFE
        self.max_linesearch = 20
        self.min_step = 1e-20
        self.max_step = 1e20
        self.ftol = 1e-4
        self.wolfe = 0.9
        for k, v in kw.items():
            if not hasattr(self, k):
                raise AttributeError("LBFGSParam has no field %r" % k)
            setattr(self, k, v)

    def _c(self):
        return _DrvParam(self.m, self.epsilon, self.epsilon_rel, self.past, self.delta, self.max_iterations,
                         self.linesearch, 10, self.max_linesearch, self.min_step, self.max_step, self.ftol, self.wolfe)


class OWLQNSolver:
    """LBFGSpp::OWLQNSolver<Scalar> on the GPU (include/OWLQN.h): minimises f(x) + lam |x|_1, host buffers in and out.

    minimize(objective, x0) returns dict(status, msg, niter, nfev, fx = F(x), gnorm = ||pg||, x, grad = grad f(x), seconds = the
    synchronised minimize() alone); with
    raise_errors=True the exceptions come back as ValueError / ArithmeticError / RuntimeError as for LBFGSSolver.  plain=True runs the
    objective as a plain device functor (projection kernel -> objective -> sums kernel) instead of the fused projected trial.
    From param it uses m, epsilon, epsilon_rel, past, delta, max_iterations, max_linesearch, min_step, max_step and ftol.
    weights (n entries, or None): F = f(x) + lam sum_i w_i |x_i|, w_i >= 0; a coordinate with lam * w_i == 0 is not penalised.
    """

    def __init__(self, param=None, lam=1.0, weights=None, dtype=np.float64, device=0, lib=None):
        self.param = param if param is not None else LBFGSParam()
        self.lam = float(lam)
        self.weights = weights
        self.dtype = np.dtype(dtype)
        self.device = device
        self.lib = lib

    def minimize(self, objective, x0, data0=None, data1=None, plain=False, raise_errors=False):
        dt = self.dtype
        x = np.array(x0, dtype=dt, order="C").copy()
        w = None if self.weights is None else np.ascontiguousarray(self.weights, dtype=dt)
        if w is not None and w.shape != (x.size,):
            raise ValueError("weights must have one entry per coordinate of x0 (got %s for n = %d)" % (w.shape, x.size))
        drv = driver(self.lib)
        grad = np.zeros(x.size, dtype=dt)
        d0, d1 = (None if a is None else np.ascontiguousarray(a, dtype=dt) for a in (data0, data1))
        res = _OwlqnResult()
        p = self.param._c()
        fn = drv.lbfgsb200_drv_owlqn_f64 if dt == np.float64 else drv.lbfgsb200_drv_owlqn_f32
        fn(self.device, objective, _ptr(d0), _ptr(d1), x.size, C.byref(p), self.lam, _ptr(w), 0 if plain else 1, _ptr(x), _ptr(grad),
           C.byref(res))
        if res.status and raise_errors:
            raise _EXC.get(res.status, RuntimeError)(res.msg.decode())
        return dict(status=STATUS_NAMES[res.status], msg=res.msg.decode(), niter=res.niter, nfev=res.nfev, fx=res.fx, gnorm=res.gnorm,
                    x=x, grad=grad, seconds=res.seconds)


class LBFGSBParam:
    """Same fields and defaults as LBFGSpp::LBFGSBParam<Scalar> (reference Param.h:330-341)."""

    def __init__(self, **kw):
        self.m = 6
        self.epsilon = 1e-5
        self.epsilon_rel = 1e-5
        self.past = 1
        self.delta = 1e-10
        self.max_iterations = 0
        self.max_submin = 10
        self.max_linesearch = 20
        self.min_step = 1e-20
        self.max_step = 1e20
        self.ftol = 1e-4
        self.wolfe = 0.9
        for k, v in kw.items():
            if not hasattr(self, k):
                raise AttributeError("LBFGSBParam has no field %r" % k)
            setattr(self, k, v)

    def _c(self):
        return _DrvParam(self.m, self.epsilon, self.epsilon_rel, self.past, self.delta, self.max_iterations, 3, self.max_submin,
                         self.max_linesearch, self.min_step, self.max_step, self.ftol, self.wolfe)


_EXC = {1: ValueError, 2: ArithmeticError, 3: RuntimeError, 4: RuntimeError}
STATUS_NAMES = {0: "ok", 1: "invalid_argument", 2: "logic_error", 3: "runtime_error", 4: "other"}


def _solve_result(res, x, grad, trace, raise_errors):
    """The dict a host-buffer minimize() returns for its _DrvResult, or the reference's exception when raise_errors."""
    if res.status and raise_errors:
        raise _EXC.get(res.status, RuntimeError)(res.msg.decode())
    return dict(status=STATUS_NAMES[res.status], msg=res.msg.decode(), niter=res.niter, nfev=res.nfev, fx=res.fx,
                gnorm=res.gnorm, x=x, grad=grad, trace=trace[:res.trace_len].copy(), seconds=res.seconds,
                seconds_e2e=res.seconds_e2e, launches=res.launches)


class LBFGSSolver:
    """LBFGSpp::LBFGSSolver<Scalar, LineSearch> on the GPU, host buffers in and out.

    minimize(objective, x0) returns a dict(niter, nfev, fx, gnorm, x, grad, trace, status, msg, seconds, ...);
    with raise_errors=True the reference's exceptions come back as ValueError (std::invalid_argument),
    ArithmeticError (std::logic_error) or RuntimeError (std::runtime_error).
    lib: a library exporting the driver's entry points to use instead of liblbfgs_b200_driver.so.
    """

    def __init__(self, param=None, linesearch="NocedalWright", dtype=np.float64, device=0, hv_algo=HV_AUTO,
                 fused=True, resident=False, lib=None):
        self.param = param if param is not None else LBFGSParam()
        self.ls = _ls_id(linesearch)
        self.dtype = np.dtype(dtype)
        self.device = device
        self.hv_algo = hv_algo
        self.fused = 2 if resident else fused   # 2: device-resident solve (one persistent kernel launch per minimize)
        self.lib = lib

    def minimize(self, objective, x0, data0=None, data1=None, trace_cap=100000, raise_errors=False, want_grad=True):
        drv = driver(self.lib)
        dt = self.dtype
        x = np.array(x0, dtype=dt, order="C").copy()
        n = x.size
        grad = np.zeros(n, dtype=dt) if want_grad else None
        trace = np.zeros(trace_cap, dtype=np.float64)
        d0, d1 = (None if a is None else np.ascontiguousarray(a, dtype=dt) for a in (data0, data1))
        res = _DrvResult()
        p = self.param._c()
        fn = drv.lbfgsb200_drv_lbfgs_f64 if dt == np.float64 else drv.lbfgsb200_drv_lbfgs_f32
        fn(self.device, objective, _ptr(d0), _ptr(d1), n, self.ls, C.byref(p), self.hv_algo, int(self.fused), _ptr(x), _ptr(grad),
           _ptr(trace), trace_cap, C.byref(res))
        return dict(_solve_result(res, x, grad, trace, raise_errors), h2d_bytes=res.h2d_bytes, d2h_bytes=res.d2h_bytes)


class LBFGSBSolver:
    """LBFGSpp::LBFGSBSolver<Scalar> (More-Thuente line search) on the GPU, host buffers in and out; Scalar from `dtype`."""

    def __init__(self, param=None, device=0, dtype=np.float64):
        self.param = param if param is not None else LBFGSBParam()
        self.device = device
        self.dtype = np.dtype(dtype)

    def minimize(self, objective, x0, lb, ub, data0=None, data1=None, trace_cap=100000, raise_errors=False, lib=None):
        """lib: a library exporting the driver's entry points to use instead of liblbfgs_b200_driver.so."""
        drv = driver(lib)
        dt = self.dtype
        x = np.array(x0, dtype=dt, order="C").copy()
        n = x.size
        lbv = np.ascontiguousarray(np.broadcast_to(lb, n), dtype=dt)
        ubv = np.ascontiguousarray(np.broadcast_to(ub, n), dtype=dt)
        grad = np.zeros(n, dtype=dt)
        trace = np.zeros(trace_cap)
        d0, d1 = (None if a is None else np.ascontiguousarray(a, dtype=dt) for a in (data0, data1))
        res = _DrvResult()
        p = self.param._c()
        fn = drv.lbfgsb200_drv_lbfgsb_f64 if dt == np.float64 else drv.lbfgsb200_drv_lbfgsb_f32
        fn(self.device, objective, _ptr(d0), _ptr(d1), n, C.byref(p), _ptr(x), _ptr(lbv), _ptr(ubv), _ptr(grad), _ptr(trace), trace_cap,
           C.byref(res))
        return _solve_result(res, x, grad, trace, raise_errors)


# ------------------------------------------------------------------------------------------------------
# thin object wrappers over the raw C ABI (kernel-level tests, microbenchmarks)
# ------------------------------------------------------------------------------------------------------
class Context:
    """lib: a ctypes library exporting the C ABI to use instead of liblbfgs_b200.so (its types are declared on first use)."""

    def __init__(self, device=0, stream=None, lib=None):
        self.lib = abi() if lib is None else _declare(lib)
        self.h = C.c_void_p()
        st = self.lib.lbfgs_b200_ctx_create(C.byref(self.h), device, stream)
        if st:
            raise LbfgsB200Error(st, self.lib.lbfgs_b200_last_error(None).decode())

    @classmethod
    def borrow(cls, handle):
        """Non-owning wrapper around an existing lbfgs_b200_ctx* (e.g. driver_ctx(device), which may carry a communicator)."""
        self = cls.__new__(cls)
        self.lib = abi()
        self.h = handle if isinstance(handle, C.c_void_p) else C.c_void_p(handle)
        self.owned = False
        return self

    def check(self, st):
        if st:
            raise LbfgsB200Error(st, self.lib.lbfgs_b200_last_error(self.h).decode())

    def close(self):
        if self.h and getattr(self, "owned", True):
            self.lib.lbfgs_b200_ctx_destroy(self.h)
        self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def array(self, host, dtype=None):
        return DeviceArray(self, host, dtype)

    def empty(self, n, dtype=np.float64):
        return DeviceArray(self, None, dtype, n)

    def sync(self):
        self.check(self.lib.lbfgs_b200_sync(self.h))

    def trim(self):
        """Give the context's cached device blocks back to the driver (lbfgs_b200_trim)."""
        self.check(self.lib.lbfgs_b200_trim(self.h))

    def launches(self):
        return self.lib.lbfgs_b200_launch_count(self.h)

    def timer_start(self):
        self.check(self.lib.lbfgs_b200_timer_start(self.h))

    def timer_stop(self):
        ms = C.c_float(0)
        self.check(self.lib.lbfgs_b200_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def _fn(self, name, dtype):
        return getattr(self.lib, "lbfgs_b200_%s_%s" % (name, "f64" if np.dtype(dtype) == np.float64 else "f32"))

    def dot(self, a, b):
        out = (a.ct * 1)()
        self.check(self._fn("dot", a.dtype)(self.h, a.n, a.ptr, b.ptr, out))
        return out[0]

    def dot3(self, g, d, x):
        out = (g.ct * 3)()
        self.check(self._fn("dot3", g.dtype)(self.h, g.n, g.ptr, d.ptr, x.ptr, out))
        return list(out)

    def axpy_out(self, a, s, b, out):
        self.check(self._fn("axpy_out", a.dtype)(self.h, a.n, a.ptr, s, b.ptr, out.ptr))

    def scale_out(self, s, a, out):
        self.check(self._fn("scale_out", a.dtype)(self.h, a.n, s, a.ptr, out.ptr))

    def objective(self, kind, x, g, data0=None, data1=None):
        out = (x.ct * 4)()
        self.check(self._fn("objective", x.dtype)(self.h, kind, data0.ptr if data0 else None,
                                                  data1.ptr if data1 else None, x.n, x.ptr, g.ptr, out))
        return list(out)

    def trial(self, kind, xp, d, step, x, g, data0=None, data1=None):
        out = (x.ct * 4)()
        self.check(self._fn("trial", x.dtype)(self.h, kind, data0.ptr if data0 else None, data1.ptr if data1 else None,
                                              xp.n, xp.ptr, d.ptr, step, x.ptr, g.ptr, out))
        return list(out)


    # OWL-QN kernels (include/lbfgs_b200.h, lbfgs_b200_owlqn_*): F = f + lam |x|_1
    def owlqn_trial(self, kind, xp, d, gp, step, lam, x, g, data0=None, data1=None):
        """Fused projected trial of a built-in objective: writes x, g; -> [f, |x|_1, pgp.(x - xp), pg.pg, x.x]"""
        out = (x.ct * 5)()
        self.check(self._fn("owlqn_trial", x.dtype)(self.h, kind, data0.ptr if data0 else None, data1.ptr if data1 else None, xp.n,
                                                    xp.ptr, d.ptr, gp.ptr, step, lam, x.ptr, g.ptr, out))
        return list(out)

    def owlqn_project(self, xp, d, gp, step, lam, x):
        """x = pi(xp + step d; xi); -> [|x|_1, pgp.(x - xp)]"""
        out = (x.ct * 2)()
        self.check(self._fn("owlqn_project", x.dtype)(self.h, xp.n, xp.ptr, d.ptr, gp.ptr, step, lam, x.ptr, out))
        return list(out)

    def owlqn_sums(self, x, g, lam, d=None):
        """-> [|x|_1, pg.pg, x.x]; with d also writes d = -pg"""
        out = (x.ct * 3)()
        self.check(self._fn("owlqn_sums", x.dtype)(self.h, x.n, x.ptr, g.ptr, lam, d.ptr if d is not None else None, out))
        return list(out)

    # the same under per-coordinate weights w (F = f + lam sum_i w_i |x_i|; lbfgs_b200_owlqn_weighted_*)
    def owlqn_weighted_trial(self, kind, xp, d, gp, step, lam, w, x, g, data0=None, data1=None):
        """-> [f, sum w_i |x_i|, pgp.(x - xp), pg.pg, x.x]; writes x, g"""
        out = (x.ct * 5)()
        self.check(self._fn("owlqn_weighted_trial", x.dtype)(self.h, kind, data0.ptr if data0 else None, data1.ptr if data1 else None,
                                                             xp.n, xp.ptr, d.ptr, gp.ptr, step, lam, w.ptr if w is not None else None,
                                                             x.ptr, g.ptr, out))
        return list(out)

    def owlqn_weighted_project(self, xp, d, gp, step, lam, w, x):
        """-> [sum w_i |x_i|, pgp.(x - xp)]; writes x"""
        out = (x.ct * 2)()
        self.check(self._fn("owlqn_weighted_project", x.dtype)(self.h, xp.n, xp.ptr, d.ptr, gp.ptr, step, lam,
                                                               w.ptr if w is not None else None, x.ptr, out))
        return list(out)

    def owlqn_weighted_sums(self, x, g, lam, w, d=None):
        """-> [sum w_i |x_i|, pg.pg, x.x]; with d also writes d = -pg; refuses (LbfgsB200Error) any bad weight"""
        out = (x.ct * 3)()
        self.check(self._fn("owlqn_weighted_sums", x.dtype)(self.h, x.n, x.ptr, g.ptr, lam, w.ptr if w is not None else None,
                                                            d.ptr if d is not None else None, out))
        return list(out)


class DeviceArray:
    def __init__(self, ctx, host=None, dtype=None, n=None, offset_elems=0):
        self.ctx = ctx
        if host is not None:
            host = np.ascontiguousarray(host, dtype=dtype)
            n = host.size
            dtype = host.dtype
        self.dtype = np.dtype(dtype)
        self.ct = C.c_double if self.dtype == np.float64 else C.c_float
        self.n = int(n)
        self.base = C.c_void_p()
        self.offset = offset_elems * self.dtype.itemsize
        ctx.check(ctx.lib.lbfgs_b200_malloc(ctx.h, C.byref(self.base), self.n * self.dtype.itemsize + self.offset))
        self.ptr = C.c_void_p(self.base.value + self.offset)
        if host is not None:
            ctx.check(ctx.lib.lbfgs_b200_memcpy_h2d(ctx.h, self.ptr, host.ctypes.data_as(C.c_void_p), host.nbytes))
            ctx.sync()

    def get(self):
        out = np.empty(self.n, dtype=self.dtype)
        self.ctx.check(self.ctx.lib.lbfgs_b200_memcpy_d2h(self.ctx.h, out.ctypes.data_as(C.c_void_p), self.ptr, out.nbytes))
        return out

    def __del__(self):
        try:
            if self.base and self.ctx.h:
                self.ctx.lib.lbfgs_b200_free(self.ctx.h, self.base)
        except Exception:
            pass


class History:
    """The S/Y ring (BFGSMat) through the C ABI."""

    def __init__(self, ctx, n, m, dtype=np.float64):
        self.ctx, self.n, self.m, self.dtype = ctx, n, m, np.dtype(dtype)
        self.suf = "f64" if self.dtype == np.float64 else "f32"
        self.ct = C.c_double if self.dtype == np.float64 else C.c_float
        self.h = C.c_void_p()
        ctx.check(ctx.lib.lbfgs_b200_hist_create(ctx.h, C.byref(self.h), n, m, self.dtype.itemsize))

    def __del__(self):
        try:
            if self.h and self.ctx.h:
                self.ctx.lib.lbfgs_b200_hist_destroy(self.h)
            self.h = None   # a Box on this history checks it: finalisers of garbage cycles run in no particular order
        except Exception:
            pass

    def reset(self):
        self.ctx.check(self.ctx.lib.lbfgs_b200_hist_reset(self.h))

    @property
    def ncorr(self):
        return self.ctx.lib.lbfgs_b200_hist_ncorr(self.h)

    def add(self, s, y):
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_add_" + self.suf)(self.h, s.ptr, y.ptr))

    def update(self, x, xp, g, gp, eps=None):
        eps = np.finfo(self.dtype).eps if eps is None else eps
        acc = C.c_int(0)
        sy = (self.ct * 2)()
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_update_" + self.suf)(self.h, x.ptr, xp.ptr, g.ptr, gp.ptr,
                                                                                  eps, C.byref(acc), sy))
        return bool(acc.value), sy[0], sy[1]

    def update_apply_Hv(self, x, xp, g, gp, a, res, algo=HV_AUTO, eps=None):
        """hist_update(x, xp, g, gp) + apply_Hv(g, a, res) as one call (pair formed inside the dots pass); -> (accepted, g.res)"""
        eps = np.finfo(self.dtype).eps if eps is None else eps
        acc = C.c_int(0)
        out = (self.ct * 1)()
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_update_apply_Hv_" + self.suf)(
            self.h, x.ptr, xp.ptr, g.ptr, gp.ptr, eps, a, res.ptr, algo, C.byref(acc), out))
        return bool(acc.value), out[0]

    def owlqn_update_dir(self, x, xp, g, gp, lam, d, eps=None):
        """OWL-QN: pair update + d = the orthant-constrained -H pg(x, g); -> (accepted, pg.d)"""
        eps = np.finfo(self.dtype).eps if eps is None else eps
        acc = C.c_int(0)
        out = (self.ct * 1)()
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_owlqn_update_dir_" + self.suf)(
            self.h, x.ptr, xp.ptr, g.ptr, gp.ptr, eps, lam, d.ptr, C.byref(acc), out))
        return bool(acc.value), out[0]

    def owlqn_weighted_update_dir(self, x, xp, g, gp, lam, w, d, eps=None):
        """OWL-QN under per-coordinate weights w: pair update + the weighted constrained -H pg(x, g); -> (accepted, pg.d)"""
        eps = np.finfo(self.dtype).eps if eps is None else eps
        acc = C.c_int(0)
        out = (self.ct * 1)()
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_owlqn_weighted_update_dir_" + self.suf)(
            self.h, x.ptr, xp.ptr, g.ptr, gp.ptr, eps, lam, w.ptr if w is not None else None, d.ptr, C.byref(acc), out))
        return bool(acc.value), out[0]

    def apply_Hv(self, v, a, res, algo=HV_AUTO, want_dot=False):
        out = (self.ct * 1)()
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_apply_Hv_" + self.suf)(
            self.h, v.ptr, a, res.ptr, algo, out if want_dot else None))
        return out[0] if want_dot else None

    def scalars(self):
        theta = (self.ct * 1)()
        ys = (self.ct * (self.m + 1))()
        al = (self.ct * (self.m + 1))()
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_scalars_" + self.suf)(self.h, theta, ys, al))
        c = self.ncorr
        return theta[0], np.array(ys[:c]), np.array(al[:c])

    def wt_dot_multi(self, V, k, ldv):
        """[Y S]'V for the k columns of the DeviceArray V (leading dimension ldv): a (2c, k) array, rows y by age then s by age."""
        c = self.ncorr
        R = (self.ct * max(1, 2 * c * k))()
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_wt_dot_multi_" + self.suf)(self.h, k, V.ptr, ldv, R))
        return np.array(R[:2 * c * k], dtype=self.dtype).reshape(2 * c, k)

    def lincomb_multi(self, a0, V, k, ldv, C_coef, OUT, ldo):
        """OUT[:, j] = a0 V[:, j] + sum_a C[a, j] y_a + C[c + a, j] s_a (C: (2c, k), y by age then s by age)."""
        coef = np.ascontiguousarray(C_coef, dtype=self.dtype).reshape(-1)
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_lincomb_multi_" + self.suf)(
            self.h, a0, k, V.ptr, ldv, coef.ctypes.data_as(C.POINTER(self.ct)) if coef.size else None, OUT.ptr, ldo))

    def quad_diag(self, a0, K, out):
        """out_i = a0 + r_i' K r_i into the DeviceArray out (lbfgs_b200_hist_quad_diag): K (2c, 2c), symmetric, rows y by age then s by
        age; only its upper triangle is read."""
        Kc = np.ascontiguousarray(K, dtype=self.dtype).reshape(-1)
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_quad_diag_" + self.suf)(
            self.h, a0, Kc.ctypes.data_as(C.POINTER(self.ct)) if Kc.size else None, out.ptr))

    def wt_dot_normal(self, seed, stream, first, k):
        """[Y S]'Z for the draws first .. first+k-1 of stream `stream`, generated in the pass (lbfgs_b200_hist_wt_dot_normal): (2c, k)."""
        c = self.ncorr
        R = (self.ct * max(1, 2 * c * k))()
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_wt_dot_normal_" + self.suf)(self.h, seed, stream, first, k, R))
        return np.array(R[:2 * c * k], dtype=self.dtype).reshape(2 * c, k)

    def lincomb_normal(self, a0, seed, stream, first, k, mean, C_coef, OUT, ldo):
        """OUT[:, j] = mean + a0 z_j + sum_a C[c + a, j] s_a, z_j generated in the pass (lbfgs_b200_hist_lincomb_normal); mean: a
        DeviceArray or None."""
        coef = np.ascontiguousarray(C_coef, dtype=self.dtype).reshape(-1)
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_lincomb_normal_" + self.suf)(
            self.h, a0, seed, stream, first, k, mean.ptr if mean is not None else None,
            coef.ctypes.data_as(C.POINTER(self.ct)) if coef.size else None, OUT.ptr, ldo))

    def s_dot_multi(self, V, k, ldv):
        """S'V for the k columns of the DeviceArray V (lbfgs_b200_hist_s_dot_multi): a (c, k) array, rows s by age."""
        c = self.ncorr
        R = (self.ct * max(1, c * k))()
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_s_dot_multi_" + self.suf)(self.h, k, V.ptr, ldv, R))
        return np.array(R[:c * k], dtype=self.dtype).reshape(c, k)

    def wt_dot_diff(self, X, k, ldx, mean):
        """[Y S]'(X - mean) and |x_j - mean|^2 for the k columns of the DeviceArray X (lbfgs_b200_hist_wt_dot_diff): a (2c, k)
        float64 array and k float64 norms, as summed in fp64."""
        c = self.ncorr
        R = np.zeros(max(1, 2 * c * k))
        nrm = np.zeros(k)
        dp = C.POINTER(C.c_double)
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_hist_wt_dot_diff_" + self.suf)(self.h, k, X.ptr, ldx, mean.ptr, R.ctypes.data_as(dp),
                                                                                        nrm.ctypes.data_as(dp)))
        return R[:2 * c * k].reshape(2 * c, k), nrm

    # The masked forms (lbfgs_b200_hist_*_masked): the passes above on the rows whose class byte in `box` (a Box of this history)
    # intersects `mask`; the vector rows outside count as 0, output rows outside are 0 (mean_i for lincomb_normal_masked).
    def _masked(self, name):
        return getattr(self.ctx.lib, "lbfgs_b200_hist_%s_masked_%s" % (name, self.suf))

    def _cls(self, box):
        return box._ptr("cls")

    def wt_dot_multi_masked(self, box, mask, V, k, ldv):
        c = self.ncorr
        R = (self.ct * max(1, 2 * c * k))()
        self.ctx.check(self._masked("wt_dot_multi")(self.h, box.h, self._cls(box), mask, k, V.ptr, ldv, R))
        return np.array(R[:2 * c * k], dtype=self.dtype).reshape(2 * c, k)

    def wt_dot_diff_masked(self, box, mask, X, k, ldx, mean):
        c = self.ncorr
        R = np.zeros(max(1, 2 * c * k))
        nrm = np.zeros(k)
        dp = C.POINTER(C.c_double)
        self.ctx.check(self._masked("wt_dot_diff")(self.h, box.h, self._cls(box), mask, k, X.ptr, ldx, mean.ptr, R.ctypes.data_as(dp),
                                                   nrm.ctypes.data_as(dp)))
        return R[:2 * c * k].reshape(2 * c, k), nrm

    def wt_dot_normal_masked(self, box, mask, seed, stream, first, k):
        c = self.ncorr
        R = (self.ct * max(1, 2 * c * k))()
        self.ctx.check(self._masked("wt_dot_normal")(self.h, box.h, self._cls(box), mask, seed, stream, first, k, R))
        return np.array(R[:2 * c * k], dtype=self.dtype).reshape(2 * c, k)

    def lincomb_multi_masked(self, box, mask, a0, V, k, ldv, C_coef, OUT, ldo):
        coef = np.ascontiguousarray(C_coef, dtype=self.dtype).reshape(-1)
        self.ctx.check(self._masked("lincomb_multi")(self.h, box.h, self._cls(box), mask, a0, k, V.ptr, ldv,
                                                     coef.ctypes.data_as(C.POINTER(self.ct)) if coef.size else None, OUT.ptr, ldo))

    def lincomb_normal_masked(self, box, mask, a0, seed, stream, first, k, mean, C_coef, OUT, ldo):
        """OUT[:, j] = mean + a0 z_j + sum_a C[a, j] y_a + C[c + a, j] s_a on the rows of the mask, mean_i elsewhere."""
        coef = np.ascontiguousarray(C_coef, dtype=self.dtype).reshape(-1)
        self.ctx.check(self._masked("lincomb_normal")(self.h, box.h, self._cls(box), mask, a0, seed, stream, first, k,
                                                      mean.ptr if mean is not None else None,
                                                      coef.ctypes.data_as(C.POINTER(self.ct)) if coef.size else None, OUT.ptr, ldo))

    def quad_diag_masked(self, box, mask, a0, K, out):
        Kc = np.ascontiguousarray(K, dtype=self.dtype).reshape(-1)
        self.ctx.check(self._masked("quad_diag")(self.h, box.h, self._cls(box), mask, a0,
                                                 Kc.ctypes.data_as(C.POINTER(self.ct)) if Kc.size else None, out.ptr))

    def column(self, which, age):
        fn = self.ctx.lib.lbfgs_b200_hist_s_col if which == "s" else self.ctx.lib.lbfgs_b200_hist_y_col
        p = fn(self.h, age)
        out = np.empty(self.n, dtype=self.dtype)
        self.ctx.check(self.ctx.lib.lbfgs_b200_memcpy_d2h(self.ctx.h, out.ctypes.data_as(C.c_void_p), p, out.nbytes))
        return out


BOXV_VECC, BOXV_VECY, BOXV_LAMBDA, BOXV_MU, BOXV_TMP, BOXV_TMP2, BOXV_YFB, BOXV_DVEC, BOXV_BRK, BOXV_XCP = range(10)
CLS_FIXED, CLS_ACT, CLS_FREE, SUB_L, SUB_U, SUB_P, CLS_FINAL = 1, 2, 4, 8, 16, 32, 64


class Box:
    """The workspace of the bound-constrained path (lbfgs_b200_box) on a History: its n-vectors (BOXV_*) and class bytes."""

    def __init__(self, hist):
        self.hist, self.ctx, self.n, self.dtype = hist, hist.ctx, hist.n, hist.dtype
        self.h = C.c_void_p()
        self.ctx.check(self.ctx.lib.lbfgs_b200_box_create(hist.h, C.byref(self.h)))

    def __del__(self):
        try:
            if self.h and self.hist.h and self.ctx.h:   # lbfgs_b200_box_destroy reads its history
                self.ctx.lib.lbfgs_b200_box_destroy(self.h)
        except Exception:
            pass

    def _ptr(self, which):
        return self.ctx.lib.lbfgs_b200_box_classes(self.h) if which == "cls" else self.ctx.lib.lbfgs_b200_box_vector(self.h, which)

    def _spec(self, which):
        return (np.uint8, self.n) if which == "cls" else (self.dtype, self.n)

    def get(self, which):
        """Download BOXV_* vector `which`, or the class bytes for which = "cls"."""
        dt, n = self._spec(which)
        out = np.empty(n, dtype=dt)
        self.ctx.check(self.ctx.lib.lbfgs_b200_memcpy_d2h(self.ctx.h, out.ctypes.data_as(C.c_void_p), self._ptr(which), out.nbytes))
        return out

    def set(self, which, host):
        dt, n = self._spec(which)
        host = np.ascontiguousarray(host, dtype=dt)
        assert host.size == n
        self.ctx.check(self.ctx.lib.lbfgs_b200_memcpy_h2d(self.ctx.h, self._ptr(which), host.ctypes.data_as(C.c_void_p), host.nbytes))
        self.ctx.sync()

    def final_classes(self, x, lb, ub, tol=None):
        """CLS_FINAL on the free coordinates of the DeviceArray x against the DeviceArrays lb, ub (lbfgs_b200_box_final_classes);
        returns their number.  tol: 4 eps of the storage type by default."""
        tol = 4 * np.finfo(self.dtype).eps if tol is None else tol
        nf = C.c_int64(0)
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_box_final_classes_" + ("f64" if self.dtype == np.float64 else "f32"))(
            self.h, x.ptr, lb.ptr, ub.ptr, tol, C.byref(nf)))
        return nf.value


class Session:
    """A solver and its vectors kept resident on one GPU (bench.py): solve() repeats the same problem.
    lib: a library exporting the driver's entry points to use instead of liblbfgs_b200_driver.so."""

    def __init__(self, objective, x0, param, linesearch="MoreThuente", device=0, hv_algo=HV_AUTO, data0=None, data1=None,
                 resident=True, lib=None):
        self.drv = driver(lib)
        x0 = np.ascontiguousarray(x0, dtype=np.float64)
        self.n = x0.size
        d0, d1 = (None if a is None else np.ascontiguousarray(a, dtype=np.float64) for a in (data0, data1))
        p = param._c()
        self.h = _checked("session_create", lambda *err: self.drv.lbfgsb200_drv_session_create(
            device, objective, _ptr(d0), _ptr(d1), self.n, _ls_id(linesearch), C.byref(p), hv_algo, _ptr(x0), *err, int(resident)),
            failed=lambda h: not h)

    def solve(self, from_host=False, to_host=False):
        res = _DrvResult()
        self.drv.lbfgsb200_drv_session_solve(self.h, int(from_host), int(to_host), C.byref(res))
        if res.status:
            raise RuntimeError(res.msg.decode())
        return dict(niter=res.niter, nfev=res.nfev, fx=res.fx, gnorm=res.gnorm, launches=res.launches,
                    h2d_bytes=res.h2d_bytes, d2h_bytes=res.d2h_bytes)

    OPS = ("mixed", "first", "trial", "dots_form", "dots_plain", "combine", "combine_trial", "restore", "materialize", "-")   # slot 9 unused

    def profile(self):
        """Accounting of the last device-resident solve: dict(kernel_ms, sync_ms, ops={name: dict(ms, rounds, alg_bytes)}); None for
        the host-driven loop."""
        return _profile(self.drv.lbfgsb200_drv_session_profile, self.h)

    def result(self):
        p = self.drv.lbfgsb200_drv_session_result(self.h)
        return np.ctypeslib.as_array(p, shape=(self.n,)).copy()

    def solution(self):
        """x of the last solve(), copied from the device (the solve itself need not have asked for to_host)."""
        x = np.empty(self.n)
        if self.drv.lbfgsb200_drv_session_download(self.h, _ptr(x)):
            raise RuntimeError("session download failed")
        return x

    def close(self):
        if self.h:
            self.drv.lbfgsb200_drv_session_destroy(self.h)
            self.h = None


def _profile(fn, h):
    """The profile dict of Session.profile() from a *_profile entry point, or None when the solve ran no device-resident solver."""
    ms, rounds, nbytes = (C.c_double * 10)(), (C.c_ulonglong * 10)(), (C.c_double * 10)()
    kms, sync = C.c_double(0), (C.c_double * 3)()
    if fn(h, C.byref(kms), ms, rounds, nbytes, sync):
        return None
    return dict(kernel_ms=kms.value, sync_ms=sync[0], wait_last_cta_ms=sync[1], exchange_ms=sync[2],
                ops={Session.OPS[k]: dict(ms=ms[k], rounds=int(rounds[k]), alg_bytes=nbytes[k]) for k in range(10) if rounds[k]})


def solve_batch(objective, X0, param=None, linesearch="MoreThuente", device=0, hv_algo=HV_AUTO, threads=4, sharded=False,
                return_x=True, lib=None):
    """B independent problems (rows of X0) on one GPU: LBFGSSolver::minimize per problem, `threads` host threads each with
    its own context/stream.  sharded=True: run on the driver's communicator-attached context (n-sharded over ranks), one
    thread.  Returns (list of dicts, X, seconds)."""
    drv = driver(lib)
    X0 = np.ascontiguousarray(X0, dtype=np.float64)
    B, n = X0.shape
    param = param if param is not None else LBFGSParam()
    items = (_BatchItem * B)()
    X = np.empty_like(X0) if return_x else None
    secs = C.c_double(0)
    p = param._c()
    drv.lbfgsb200_drv_batch_f64(device, objective, n, B, _ptr(X0), _ls_id(linesearch), C.byref(p), hv_algo, threads, int(sharded), items,
                                _ptr(X), C.byref(secs))
    res = [dict(status=STATUS_NAMES[it.status], niter=it.niter, nfev=it.nfev, fx=it.fx, gnorm=it.gnorm) for it in items]
    return res, X, secs.value


class BatchSession:
    """B independent problems (rows of X0) minimised by ONE persistent kernel launch per solve() (LBFGSpp::LBFGSBatchSolver,
    include/LBFGSBatch.h).  The start points stay resident; with a communicator attached to the device's driver context the rows
    are this rank's blocks of n-sharded problems."""

    def __init__(self, objective, X0, param=None, linesearch="MoreThuente", device=0, lib=None):
        self.drv = driver(lib)
        X0 = np.ascontiguousarray(X0, dtype=np.float64)
        self.B, self.n = X0.shape
        param = param if param is not None else LBFGSParam()
        p = param._c()
        self.h = _checked("batch_session_create", lambda *err: self.drv.lbfgsb200_drv_batch_session_create(
            device, objective, self.n, self.B, _ptr(X0), _ls_id(linesearch), C.byref(p), *err), failed=lambda h: not h)

    def solve(self, return_x=True):
        items = (_BatchItem * self.B)()
        rounds = (C.c_long * self.B)()
        X = np.empty((self.B, self.n)) if return_x else None
        secs = C.c_double(0)
        _checked("batch solve", lambda *err: self.drv.lbfgsb200_drv_batch_session_solve(self.h, items, rounds, _ptr(X), C.byref(secs), *err),
                 failed=lambda bad: bad < 0)
        res = [dict(status=STATUS_NAMES[it.status], niter=it.niter, nfev=it.nfev, fx=it.fx, gnorm=it.gnorm, rounds=int(r))
               for it, r in zip(items, rounds)]
        return res, X, secs.value

    def upload(self, X0):
        """New start points (host array, B x n) for the following solves: the host -> device leg of the end-to-end path."""
        X0 = np.ascontiguousarray(X0, dtype=np.float64)
        assert X0.shape == (self.B, self.n)
        _checked("batch upload", lambda *err: self.drv.lbfgsb200_drv_batch_session_upload(self.h, _ptr(X0), *err))
        return X0.nbytes

    def solution(self):
        """X (B x n) of the last solve(), copied from the device (also after solve(return_x=False))."""
        X = np.empty((self.B, self.n))
        if self.drv.lbfgsb200_drv_batch_session_download(self.h, _ptr(X)):
            raise RuntimeError("batch session download failed")
        return X

    def profile(self):
        """Accounting of the last batched solve (one kernel launch for the whole batch): same dict as Session.profile()."""
        return _profile(self.drv.lbfgsb200_drv_batch_session_profile, self.h)

    def close(self):
        if self.h:
            self.drv.lbfgsb200_drv_batch_session_destroy(self.h)
            self.h = None


def solve_dense(objective, x0, param=None, linesearch="NocedalWright", resident=True, device=0, lib=None):
    """minimize() then final_approx_hessian() / final_approx_inverse_hessian() (small n).  Returns (niter, x, B, H)."""
    drv = driver(lib)
    x = np.array(x0, dtype=np.float64, order="C").copy()
    n = x.size
    param = param if param is not None else LBFGSParam()
    p = param._c()
    Bm, Hm = np.zeros((n, n)), np.zeros((n, n))
    niter = C.c_int(0)
    _checked("solve_dense", lambda *err: drv.lbfgsb200_drv_solve_dense_f64(device, objective, n, _ls_id(linesearch), C.byref(p), int(resident),
                                                                          _ptr(x), _ptr(Bm), _ptr(Hm), C.byref(niter), *err))
    return niter.value, x, Bm, Hm


def _hessian_products(call, V, n):
    """call(V, v_len, BV, HV, HBV, *err) runs a *_hessian_times entry point; V is (k, n) or a flat block of k n-vectors."""
    V = np.ascontiguousarray(V, dtype=np.float64).reshape(-1)
    shape = (V.size // n, n) if n and V.size % n == 0 else (V.size,)
    BV, HV, HBV = (np.zeros(V.size) for _ in range(3))
    call(V, V.size, BV, HV, HBV)
    return BV.reshape(shape), HV.reshape(shape), HBV.reshape(shape)


def solve_hessian_times(objective, x0, V, param=None, linesearch="NocedalWright", resident=True, device=0, lib=None):
    """minimize(), then the final approximation as an operator (LBFGSSolver::final_approx_hessian_times /
    final_approx_inverse_hessian_times) on the rows of V (k x n).  Returns (niter, x, B V, H V, H (B V))."""
    drv = driver(lib)
    x = np.array(x0, dtype=np.float64, order="C").copy()
    n = x.size
    p = (param if param is not None else LBFGSParam())._c()
    niter = C.c_int(0)
    BV, HV, HBV = _hessian_products(lambda v, vlen, bv, hv, hbv: _checked("solve_hessian_times", lambda *err: drv.lbfgsb200_drv_solve_hessian_times_f64(
        device, objective, n, _ls_id(linesearch), C.byref(p), int(resident), _ptr(x), _ptr(v), vlen, _ptr(bv), _ptr(hv), _ptr(hbv),
        C.byref(niter), *err)), V, n)
    return niter.value, x, BV, HV, HBV


def batch_hessian_times(objective, X0, b, V, param=None, linesearch="MoreThuente", device=0, lib=None):
    """A batch (rows of X0) minimised by LBFGSBatchSolver, then problem b's final approximation as an operator on the rows of V.
    Returns (B V, H V, H (B V))."""
    drv = driver(lib)
    X0 = np.ascontiguousarray(X0, dtype=np.float64)
    B, n = X0.shape
    p = (param if param is not None else LBFGSParam())._c()
    return _hessian_products(lambda v, vlen, bv, hv, hbv: _checked("batch_hessian_times", lambda *err: drv.lbfgsb200_drv_batch_hessian_times_f64(
        device, objective, n, B, _ptr(X0), _ls_id(linesearch), C.byref(p), b, _ptr(v), vlen, _ptr(bv), _ptr(hv), _ptr(hbv), *err)), V, n)


def solve_hessian_diagonal(objective, x0, param=None, linesearch="NocedalWright", resident=True, device=0, lib=None):
    """minimize(), then the diagonals of the final approximation (LBFGSSolver::final_approx_hessian_diagonal /
    final_approx_inverse_hessian_diagonal).  Returns (niter, x, diag B, diag H)."""
    drv = driver(lib)
    x = np.array(x0, dtype=np.float64, order="C").copy()
    n = x.size
    p = (param if param is not None else LBFGSParam())._c()
    niter = C.c_int(0)
    dB, dH = np.zeros(n), np.zeros(n)
    _checked("solve_hessian_diagonal", lambda *err: drv.lbfgsb200_drv_solve_hessian_diag_f64(
        device, objective, n, _ls_id(linesearch), C.byref(p), int(resident), _ptr(x), _ptr(dB), _ptr(dH), C.byref(niter), *err))
    return niter.value, x, dB, dH


def batch_hessian_diagonal(objective, X0, b, param=None, linesearch="MoreThuente", device=0, lib=None):
    """A batch (rows of X0) minimised by LBFGSBatchSolver, then the diagonals of problem b's final approximation.
    Returns (diag B, diag H)."""
    drv = driver(lib)
    X0 = np.ascontiguousarray(X0, dtype=np.float64)
    B, n = X0.shape
    p = (param if param is not None else LBFGSParam())._c()
    dB, dH = np.zeros(n), np.zeros(n)
    _checked("batch_hessian_diagonal", lambda *err: drv.lbfgsb200_drv_batch_hessian_diag_f64(
        device, objective, n, B, _ptr(X0), _ls_id(linesearch), C.byref(p), b, _ptr(dB), _ptr(dH), *err))
    return dB, dH


def hist_diagonal(S, Y, m=None, device=0, lib=None):
    """diag B and diag H of the history built by adding the pairs (S[k], Y[k]) in order to a ring of size m (default: all of them)."""
    drv = driver(lib)
    S = np.ascontiguousarray(S, dtype=np.float64)
    Y = np.ascontiguousarray(Y, dtype=np.float64)
    npairs, n = S.shape
    dB, dH = np.zeros(n), np.zeros(n)
    _checked("hist_diagonal", lambda *err: drv.lbfgsb200_drv_hist_diag_f64(device, n, npairs if m is None else m, npairs, _ptr(S), _ptr(Y),
                                                                          _ptr(dB), _ptr(dH), *err))
    return dB, dH


def solve_hessian_sample(objective, x0, V=None, seed=0, first=0, k=0, param=None, linesearch="NocedalWright", resident=True, device=0,
                         lib=None):
    """minimize(), then N(x*, H) from the final approximation (LBFGSSolver::final_approx_inverse_hessian_factor_times /
    final_approx_sample / final_approx_inverse_hessian_logdet): L V for the rows of V (H = L L'), the k draws x* + L z_j,
    j = first .. first+k-1 of stream 0, and log det H.  Returns (niter, x, LV, draws, logdet)."""
    drv = driver(lib)
    x = np.array(x0, dtype=np.float64, order="C").copy()
    n = x.size
    p = (param if param is not None else LBFGSParam())._c()
    v = None if V is None else np.ascontiguousarray(V, dtype=np.float64).reshape(-1, n)
    kv = 0 if v is None else v.shape[0]
    LV = None if v is None else np.zeros_like(v)
    D = np.zeros((k, n)) if k else None
    ld, niter = C.c_double(0.0), C.c_int(0)
    _checked("solve_hessian_sample", lambda *err: drv.lbfgsb200_drv_solve_hessian_sample_f64(
        device, objective, n, _ls_id(linesearch), C.byref(p), int(resident), _ptr(x), kv, _ptr(v), _ptr(LV), seed, first, k, _ptr(D),
        C.byref(ld), C.byref(niter), *err))
    return niter.value, x, LV, D, ld.value


def batch_hessian_sample(objective, X0, b, V=None, seed=0, first=0, k=0, param=None, linesearch="MoreThuente", device=0, lib=None):
    """A batch (rows of X0) minimised by LBFGSBatchSolver, then problem b's L V, draws X_b + L z_j from stream b and log det H.
    Returns (X, LV, draws, logdet)."""
    drv = driver(lib)
    X0 = np.ascontiguousarray(X0, dtype=np.float64)
    B, n = X0.shape
    p = (param if param is not None else LBFGSParam())._c()
    v = None if V is None else np.ascontiguousarray(V, dtype=np.float64).reshape(-1, n)
    kv = 0 if v is None else v.shape[0]
    LV = None if v is None else np.zeros_like(v)
    D = np.zeros((k, n)) if k else None
    X = np.zeros_like(X0)
    ld = C.c_double(0.0)
    _checked("batch_hessian_sample", lambda *err: drv.lbfgsb200_drv_batch_hessian_sample_f64(
        device, objective, n, B, _ptr(X0), _ls_id(linesearch), C.byref(p), b, kv, _ptr(v), _ptr(LV), seed, first, k, _ptr(D), C.byref(ld),
        _ptr(X), *err))
    return X, LV, D, ld.value


def hist_sample(S, Y, m=None, V=None, mean=None, seed=0, stream=0, first=0, k=0, device=0, lib=None):
    """BFGSMat's factor, sampler and log-determinant on the history built by adding the pairs (S[k], Y[k]) in order to a ring of size m
    (default: all of them).  Returns (LV, draws, logdet)."""
    drv = driver(lib)
    S = np.ascontiguousarray(S, dtype=np.float64)
    Y = np.ascontiguousarray(Y, dtype=np.float64)
    npairs, n = S.shape
    v = None if V is None else np.ascontiguousarray(V, dtype=np.float64).reshape(-1, n)
    kv = 0 if v is None else v.shape[0]
    LV = None if v is None else np.zeros_like(v)
    mu = None if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
    D = np.zeros((k, n)) if k else None
    ld = C.c_double(0.0)
    _checked("hist_sample", lambda *err: drv.lbfgsb200_drv_hist_sample_f64(device, n, npairs if m is None else m, npairs, _ptr(S), _ptr(Y), kv,
                                                                          _ptr(v), _ptr(LV), _ptr(mu), seed, stream, first, k, _ptr(D),
                                                                          C.byref(ld), *err))
    return LV, D, ld.value


def small_batch_hessian_sample(objective, X0, V=None, seed=0, first=0, k=0, param=None, linesearch="MoreThuente", dtype=np.float64, data0=None,
                               data1=None, ldd=0, device=0, lib=None):
    """solve_small_batch with every problem's final approximation kept, then for all problems at once (LBFGSSmallBatchSolver):
    L_b V_b (V: (B, kv, n)), the k draws X_b + L_b z_j from stream b, and log det H_b.  Returns (outcomes, X, LV, draws (B, k, n),
    logdet (B,))."""
    drv = driver(lib)
    X0 = np.ascontiguousarray(X0, dtype=dtype)
    B, n = X0.shape
    p = (param if param is not None else LBFGSParam())._c()
    d0 = None if data0 is None else np.ascontiguousarray(data0, dtype=dtype).reshape(-1)
    d1 = None if data1 is None else np.ascontiguousarray(data1, dtype=dtype).reshape(-1)
    v = None if V is None else np.ascontiguousarray(V, dtype=dtype).reshape(B, -1, n)
    kv = 0 if v is None else v.shape[1]
    LV = None if v is None else np.zeros_like(v)
    D = np.zeros((B, k, n), dtype=dtype) if k else None
    X = np.empty_like(X0)
    ld = np.zeros(B)
    items = (_SmallItem * B)()
    suf = "f32" if np.dtype(dtype) == np.float32 else "f64"
    err = C.create_string_buffer(256)
    r = getattr(drv, "lbfgsb200_drv_small_batch_hessian_sample_" + suf)(device, objective, n, B, _ptr(X0), _ptr(d0), _ptr(d1), int(ldd),
                                                                       _ls_id(linesearch), C.byref(p), _ptr(X), kv, _ptr(v), _ptr(LV), seed,
                                                                       first, k, _ptr(D), _ptr(ld), items, err, len(err))
    if r < 0:
        raise (ValueError if r == -1 else RuntimeError)("small_batch_hessian_sample failed: %s" % err.value.decode())
    res = [dict(status=STATUS_NAMES[it.kind], code=it.code, niter=it.niter, nfev=it.nfev, fx=it.fx, gnorm=it.gnorm, rounds=it.rounds)
           for it in items]
    return res, X, LV, D, ld


FACTOR_OPS = {"L": 0, "LT": 1, "LINV": 2, "LINVT": 3}   # LBFGS_B200_FACTOR_*: with H = L L', L, L', L^-1 and L^-T


def _op_id(op):
    return FACTOR_OPS[op] if isinstance(op, str) else int(op)


def _rows(A, n, dtype=np.float64):
    """A as contiguous rows of n values, its row count (0 for None)."""
    if A is None:
        return None, 0
    a = np.ascontiguousarray(A, dtype=dtype).reshape(-1, n)
    return a, a.shape[0]


def _solve_whiten(objective, x0, op, V, X, mean, param, linesearch, resident, device, lib):
    drv = driver(lib)
    x = np.array(x0, dtype=np.float64, order="C").copy()
    n = x.size
    p = (param if param is not None else LBFGSParam())._c()
    v, kv = _rows(V, n)
    P, kx = _rows(X, n)
    mu = None if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
    OV = None if v is None else np.zeros_like(v)
    lp = np.zeros(kx) if kx else None
    niter = C.c_int(0)
    _checked("solve_hessian_whiten", lambda *err: drv.lbfgsb200_drv_solve_hessian_whiten_f64(
        device, objective, n, _ls_id(linesearch), C.byref(p), int(resident), _ptr(x), _op_id(op), kv, _ptr(v), _ptr(OV), kx, _ptr(P), _ptr(mu),
        _ptr(lp), C.byref(niter), *err))
    return niter.value, x, OV, lp


def solve_hessian_factor(objective, x0, V, op="L", param=None, linesearch="NocedalWright", resident=True, device=0, lib=None):
    """minimize(), then op(L) V for the rows of V with H = L L' the final approximation (LBFGSSolver::final_approx_inverse_hessian_
    factor_times / _transpose_times / _solve / _transpose_solve; op one of FACTOR_OPS).  Returns (niter, x, OV)."""
    niter, x, OV, _ = _solve_whiten(objective, x0, op, V, None, None, param, linesearch, resident, device, lib)
    return niter, x, OV


def solve_hessian_log_density(objective, x0, X, mean=None, param=None, linesearch="NocedalWright", resident=True, device=0, lib=None):
    """minimize(), then log N(x; mean, H) at the rows of X (LBFGSSolver::final_approx_log_density; mean None: the solution).
    Returns (niter, x, logp)."""
    niter, x, _, lp = _solve_whiten(objective, x0, 0, None, X, mean, param, linesearch, resident, device, lib)
    return niter, x, lp


def _batch_whiten(objective, X0, b, op, V, X, mean, param, linesearch, device, lib):
    drv = driver(lib)
    X0 = np.ascontiguousarray(X0, dtype=np.float64)
    B, n = X0.shape
    p = (param if param is not None else LBFGSParam())._c()
    v, kv = _rows(V, n)
    P, kx = _rows(X, n)
    mu = None if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
    OV = None if v is None else np.zeros_like(v)
    lp = np.zeros(kx) if kx else None
    Xs = np.zeros_like(X0)
    _checked("batch_hessian_whiten", lambda *err: drv.lbfgsb200_drv_batch_hessian_whiten_f64(
        device, objective, n, B, _ptr(X0), _ls_id(linesearch), C.byref(p), b, _op_id(op), kv, _ptr(v), _ptr(OV), kx, _ptr(P), _ptr(mu), _ptr(lp),
        _ptr(Xs), *err))
    return Xs, OV, lp


def batch_hessian_factor(objective, X0, b, V, op="L", param=None, linesearch="MoreThuente", device=0, lib=None):
    """A batch (rows of X0) minimised by LBFGSBatchSolver, then problem b's op(L) V.  Returns (X, OV)."""
    Xs, OV, _ = _batch_whiten(objective, X0, b, op, V, None, None, param, linesearch, device, lib)
    return Xs, OV


def batch_hessian_log_density(objective, X0, b, X, mean=None, param=None, linesearch="MoreThuente", device=0, lib=None):
    """A batch minimised by LBFGSBatchSolver, then log N(x; mean, H_b) at the rows of X (mean None: problem b's solution).
    Returns (X_solutions, logp)."""
    Xs, _, lp = _batch_whiten(objective, X0, b, 0, None, X, mean, param, linesearch, device, lib)
    return Xs, lp


def _hist_whiten(S, Y, m, op, V, X, mean, device, lib):
    drv = driver(lib)
    S = np.ascontiguousarray(S, dtype=np.float64)
    Y = np.ascontiguousarray(Y, dtype=np.float64)
    npairs, n = S.shape
    v, kv = _rows(V, n)
    P, kx = _rows(X, n)
    mu = None if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
    OV = None if v is None else np.zeros_like(v)
    lp = np.zeros(kx) if kx else None
    _checked("hist_whiten", lambda *err: drv.lbfgsb200_drv_hist_whiten_f64(device, n, npairs if m is None else m, npairs, _ptr(S), _ptr(Y),
                                                                          _op_id(op), kv, _ptr(v), _ptr(OV), kx, _ptr(P), _ptr(mu), _ptr(lp),
                                                                          *err))
    return OV, lp


def hist_hessian_factor(S, Y, V, op="L", m=None, device=0, lib=None):
    """BFGSMat's op(L) V on the history built by adding the pairs (S[k], Y[k]) in order to a ring of size m (default: all of them)."""
    return _hist_whiten(S, Y, m, op, V, None, None, device, lib)[0]


def hist_hessian_log_density(S, Y, X, mean, m=None, device=0, lib=None):
    """BFGSMat::log_density at the rows of X on the history built from (S, Y) as hist_hessian_factor builds it."""
    return _hist_whiten(S, Y, m, 0, None, X, mean, device, lib)[1]


def _small_batch_whiten(objective, X0, op, V, X, means, param, linesearch, dtype, data0, data1, ldd, device, lib, b=None):
    drv = driver(lib)
    X0 = np.ascontiguousarray(X0, dtype=dtype)
    B, n = X0.shape
    per = B if b is None else 1     # problems whose vectors, points and means are given
    p = (param if param is not None else LBFGSParam())._c()
    d0 = None if data0 is None else np.ascontiguousarray(data0, dtype=dtype).reshape(-1)
    d1 = None if data1 is None else np.ascontiguousarray(data1, dtype=dtype).reshape(-1)
    v = None if V is None else np.ascontiguousarray(V, dtype=dtype).reshape(per, -1, n)
    kv = 0 if v is None else v.shape[1]
    P = None if X is None else np.ascontiguousarray(X, dtype=dtype).reshape(per, -1, n)
    kx = 0 if P is None else P.shape[1]
    mu = None if means is None else np.ascontiguousarray(means, dtype=dtype).reshape(per, n)
    OV = None if v is None else np.zeros_like(v)
    lp = np.zeros((per, kx)) if kx else None
    Xs = np.empty_like(X0)
    items = (_SmallItem * B)()
    suf = "f32" if np.dtype(dtype) == np.float32 else "f64"
    err = C.create_string_buffer(256)
    r = getattr(drv, "lbfgsb200_drv_small_batch_hessian_whiten_" + suf)(device, objective, n, B, _ptr(X0), _ptr(d0), _ptr(d1), int(ldd),
                                                                       _ls_id(linesearch), C.byref(p), _ptr(Xs), _op_id(op), kv, _ptr(v),
                                                                       _ptr(OV), kx, _ptr(P), _ptr(mu), _ptr(lp), -1 if b is None else int(b),
                                                                       items, err, len(err))
    if r < 0:
        raise (ValueError if r == -1 else RuntimeError)("small_batch_hessian_whiten failed: %s" % err.value.decode())
    res = [dict(status=STATUS_NAMES[it.kind], code=it.code, niter=it.niter, nfev=it.nfev, fx=it.fx, gnorm=it.gnorm, rounds=it.rounds)
           for it in items]
    if b is not None:
        OV, lp = None if OV is None else OV[0], None if lp is None else lp[0]
    return res, Xs, OV, lp


def small_batch_hessian_factor(objective, X0, V, op="L", param=None, linesearch="MoreThuente", dtype=np.float64, data0=None, data1=None,
                               ldd=0, device=0, lib=None, b=None):
    """solve_small_batch with every problem's final approximation kept, then op(L_b) V_b for all problems at once
    (LBFGSSmallBatchSolver; V: (B, kv, n)), or with b given for problem b alone through the one-problem forms (V: (kv, n)).
    Returns (outcomes, X, OV)."""
    res, Xs, OV, _ = _small_batch_whiten(objective, X0, op, V, None, None, param, linesearch, dtype, data0, data1, ldd, device, lib, b)
    return res, Xs, OV


def small_batch_hessian_log_density(objective, X0, X, means=None, param=None, linesearch="MoreThuente", dtype=np.float64, data0=None,
                                    data1=None, ldd=0, device=0, lib=None, b=None):
    """solve_small_batch with the final approximations kept, then log N(x; mean_b, H_b) at the points X (B, kx, n) for all problems at
    once (means (B, n); None: the solutions), or with b given for problem b alone through the one-problem forms (X: (kx, n), means: one
    mean or None).  Returns (outcomes, X_solutions, logp (B, kx) or (kx,))."""
    res, Xs, _, lp = _small_batch_whiten(objective, X0, 0, None, X, means, param, linesearch, dtype, data0, data1, ldd, device, lib, b)
    return res, Xs, lp


BOX_OPS = {"B": 0, "H": 1, "diagB": 2, "diagH": 3, "sample": 4, "log_density": 5, "logdet": 6, "L": 7, "LT": 8, "LINV": 9, "LINVT": 10,
           "denseB": 11, "denseH": 12}


def box_solve_hessian(objective, x0, lb, ub, op, V=None, mean=None, seed=0, first=0, k=0, free=True, tol=None, param=None, dtype=np.float64,
                      device=0, lib=None):
    """LBFGSBSolver<Scalar>::minimize on a built-in objective, then one operation (BOX_OPS) on the final approximation: on the free set at
    the solution (free=True: B_F, H_F, ...) or over the whole space.  V: (k, n) vectors for products and factor ops, points for the log
    density; mean: the draws' and densities' mean (None: the solution); k: the number of draws.  Returns a dict with x, niter, nfree
    (free only), logdet (log det H_F or H), and out: the (k, n) products or draws, the n-diagonal, the (n, n) matrix or the log densities."""
    drv = driver(lib)
    dt = np.dtype(dtype)
    opid = BOX_OPS[op] if isinstance(op, str) else int(op)
    x = np.array(x0, dtype=dt, order="C").copy()
    n = x.size
    lbv = np.ascontiguousarray(np.broadcast_to(lb, n), dtype=dt)
    ubv = np.ascontiguousarray(np.broadcast_to(ub, n), dtype=dt)
    Vr = None if V is None else np.ascontiguousarray(np.atleast_2d(V), dtype=dt)
    kv = k if opid == BOX_OPS["sample"] else (0 if Vr is None else Vr.shape[0])
    mu = None if mean is None else np.ascontiguousarray(mean, dtype=dt)
    out = np.zeros(n * n if opid >= BOX_OPS["denseB"] else max(kv, 1) * n, dtype=dt)
    dout = np.zeros(max(kv, 1))
    logdet, nfree, niter = C.c_double(0.0), C.c_long(-1), C.c_int(0)
    p = (param if param is not None else LBFGSBParam())._c()
    fn = drv.lbfgsb200_drv_box_hessian_f64 if dt == np.float64 else drv.lbfgsb200_drv_box_hessian_f32
    _checked("box_solve_hessian", lambda e, el: fn(device, objective, n, C.byref(p), _ptr(x), _ptr(lbv), _ptr(ubv), int(bool(free)),
                                                   -1.0 if tol is None else float(tol), opid, kv, _ptr(Vr), _ptr(mu), seed, first, _ptr(out),
                                                   _ptr(dout), C.byref(logdet), C.byref(nfree), C.byref(niter), e, el))
    if opid >= BOX_OPS["denseB"]:
        res = out.reshape(n, n)
    elif opid in (BOX_OPS["diagB"], BOX_OPS["diagH"]):
        res = out[:n]
    elif opid == BOX_OPS["log_density"]:
        res = dout[:kv]
    elif opid == BOX_OPS["logdet"]:
        res = logdet.value
    else:
        res = out[:kv * n].reshape(kv, n)
    return dict(x=x, niter=niter.value, nfree=nfree.value if free else None, logdet=logdet.value, out=res)


def box_solve_hessian_times(objective, x0, lb, ub, V, inverse=False, free=True, **kw):
    """B_F V or H_F V (free=False: B V or H V) after a bound-constrained solve; see box_solve_hessian."""
    return box_solve_hessian(objective, x0, lb, ub, "H" if inverse else "B", V=V, free=free, **kw)


def box_solve_hessian_diagonal(objective, x0, lb, ub, inverse=False, free=True, **kw):
    """diag B_F or diag H_F (free=False: diag B or diag H), 0 off the free set; see box_solve_hessian."""
    return box_solve_hessian(objective, x0, lb, ub, "diagH" if inverse else "diagB", free=free, **kw)


def box_solve_hessian_sample(objective, x0, lb, ub, k, seed=0, first=0, mean=None, free=True, **kw):
    """k draws of N(mean, H_F) on the free set, mean_i on the fixed coordinates (free=False: N(mean, H)), stream 0."""
    return box_solve_hessian(objective, x0, lb, ub, "sample", k=k, seed=seed, first=first, mean=mean, free=free, **kw)


def box_solve_hessian_log_density(objective, x0, lb, ub, X, mean=None, free=True, **kw):
    """log N(x_F; mean_F, H_F) of the rows of X (free=False: log N(x; mean, H)); see box_solve_hessian."""
    return box_solve_hessian(objective, x0, lb, ub, "log_density", V=X, mean=mean, free=free, **kw)


def box_solve_hessian_logdet(objective, x0, lb, ub, free=True, **kw):
    """log det H_F (free=False: log det H) and n_F; see box_solve_hessian."""
    return box_solve_hessian(objective, x0, lb, ub, "logdet", free=free, **kw)


def box_hist_hessian(S, Y, op, cls=None, m=None, V=None, mean=None, seed=0, first=0, k=0, device=0, lib=None):
    """The same operations on an explicit history (pairs S[k], Y[k] added in order to a ring of size m <= 20, fp64); cls: n class bytes
    whose CLS_FINAL bit marks the free set (None: the whole space).  Returns the dict of box_solve_hessian without x and niter."""
    drv = driver(lib)
    S = np.ascontiguousarray(np.atleast_2d(S), dtype=np.float64)
    Y = np.ascontiguousarray(np.atleast_2d(Y), dtype=np.float64)
    npairs, n = S.shape
    m = m if m is not None else max(1, npairs)
    opid = BOX_OPS[op] if isinstance(op, str) else int(op)
    Vr = None if V is None else np.ascontiguousarray(np.atleast_2d(V), dtype=np.float64)
    kv = k if opid == BOX_OPS["sample"] else (0 if Vr is None else Vr.shape[0])
    mu = None if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
    cb = None if cls is None else np.ascontiguousarray(cls, dtype=np.uint8)
    out = np.zeros(n * n if opid >= BOX_OPS["denseB"] else max(kv, 1) * n)
    dout = np.zeros(max(kv, 1))
    logdet, nfree = C.c_double(0.0), C.c_long(-1)
    _checked("box_hist_hessian", lambda e, el: drv.lbfgsb200_drv_box_hist_hessian_f64(
        device, n, m, npairs, _ptr(S), _ptr(Y), int(cb is not None), None if cb is None else cb.ctypes.data_as(C.POINTER(C.c_ubyte)), opid, kv,
        _ptr(Vr), _ptr(mu), seed, first, _ptr(out), _ptr(dout), C.byref(logdet), C.byref(nfree), e, el))
    if opid >= BOX_OPS["denseB"]:
        res = out.reshape(n, n)
    elif opid in (BOX_OPS["diagB"], BOX_OPS["diagH"]):
        res = out[:n]
    elif opid == BOX_OPS["log_density"]:
        res = dout[:kv]
    elif opid == BOX_OPS["logdet"]:
        res = logdet.value
    else:
        res = out[:kv * n].reshape(kv, n)
    return dict(nfree=nfree.value if cb is not None else None, logdet=logdet.value, out=res)


def small_max_n(m, objective, dtype=np.float64):
    """Largest n of a problem the small-batch solve takes for history size m and built-in objective `objective` (0 if none)."""
    return int(abi().lbfgs_b200_small_max_n(int(m), np.dtype(dtype).itemsize, int(objective)))


def solve_small_batch(objective, X0, param=None, linesearch="MoreThuente", dtype=np.float64, data0=None, data1=None, ldd=0,
                      want_grad=False, device=0, lib=None):
    """B independent small problems (rows of X0) minimised by LBFGSSmallBatchSolver (include/LBFGSSmallBatch.h): one launch, one
    thread block per problem.  data0/data1: one vector shared by all problems (ldd = 0) or problem b's at offset b*ldd of a flat
    array.  Returns (list of dicts with status / msg-free outcome, X, G or None).  A refused call (n above small_max_n, odd n for
    paired Rosenbrock, ...) raises ValueError; other failures RuntimeError."""
    drv = driver(lib)
    X0 = np.ascontiguousarray(X0, dtype=dtype)
    B, n = X0.shape
    p = (param if param is not None else LBFGSParam())._c()
    d0 = None if data0 is None else np.ascontiguousarray(data0, dtype=dtype).reshape(-1)
    d1 = None if data1 is None else np.ascontiguousarray(data1, dtype=dtype).reshape(-1)
    X = np.empty_like(X0)
    G = np.empty_like(X0) if want_grad else None
    items = (_SmallItem * B)()
    fn = drv.lbfgsb200_drv_small_batch_f32 if np.dtype(dtype) == np.float32 else drv.lbfgsb200_drv_small_batch_f64
    err = C.create_string_buffer(256)
    r = fn(device, objective, n, B, _ptr(X0), _ptr(d0), _ptr(d1), int(ldd), _ls_id(linesearch), C.byref(p), _ptr(X), _ptr(G), items, err, len(err))
    if r < 0:
        raise (ValueError if r == -1 else RuntimeError)("solve_small_batch failed: %s" % err.value.decode())
    res = [dict(status=STATUS_NAMES[it.kind], code=it.code, niter=it.niter, nfev=it.nfev, fx=it.fx, gnorm=it.gnorm, rounds=it.rounds)
           for it in items]
    return res, X, G


def small_batch_hessian_times(objective, X0, V, param=None, linesearch="MoreThuente", dtype=np.float64, data0=None, data1=None, ldd=0,
                              device=0, lib=None):
    """solve_small_batch with every problem's final approximation kept (LBFGSSmallBatchSolver::keep_final_approx), then its products
    with the vectors V: shape (k, n), shared by all problems, or (B, k, n).  Returns (outcomes, X, B V, H V, H (B V)), the products
    of shape (B, k, n)."""
    drv = driver(lib)
    X0 = np.ascontiguousarray(X0, dtype=dtype)
    B, n = X0.shape
    V = np.ascontiguousarray(V, dtype=dtype)
    shared = V.ndim == 2
    k = V.shape[-2]
    if V.shape[-1] != n or (not shared and (V.ndim != 3 or V.shape[0] != B)):
        raise ValueError("V must have shape (k, n) or (B, k, n)")
    p = (param if param is not None else LBFGSParam())._c()
    d0 = None if data0 is None else np.ascontiguousarray(data0, dtype=dtype).reshape(-1)
    d1 = None if data1 is None else np.ascontiguousarray(data1, dtype=dtype).reshape(-1)
    X = np.empty_like(X0)
    BV, HV, HBV = (np.empty((B, k, n), dtype=dtype) for _ in range(3))
    items = (_SmallItem * B)()
    suf = "f32" if np.dtype(dtype) == np.float32 else "f64"
    fn = getattr(drv, "lbfgsb200_drv_small_batch_hessian_times_" + suf)
    err = C.create_string_buffer(256)
    r = fn(device, objective, n, B, _ptr(X0), _ptr(d0), _ptr(d1), int(ldd), _ls_id(linesearch), C.byref(p), _ptr(V), k, int(shared), _ptr(X),
           _ptr(BV), _ptr(HV), _ptr(HBV), items, err, len(err))
    if r < 0:
        raise (ValueError if r == -1 else RuntimeError)("small_batch_hessian_times failed: %s" % err.value.decode())
    res = [dict(status=STATUS_NAMES[it.kind], code=it.code, niter=it.niter, nfev=it.nfev, fx=it.fx, gnorm=it.gnorm, rounds=it.rounds)
           for it in items]
    return res, X, BV, HV, HBV


def small_batch_hessian_diagonal(objective, X0, param=None, linesearch="MoreThuente", dtype=np.float64, data0=None, data1=None, ldd=0,
                                 device=0, lib=None):
    """solve_small_batch with every problem's final approximation kept (LBFGSSmallBatchSolver::keep_final_approx), then the diagonals
    of all of them, one launch each (final_approx_hessian_diagonal / final_approx_inverse_hessian_diagonal).  Returns (outcomes, X,
    diag B, diag H), the diagonals of shape (B, n)."""
    drv = driver(lib)
    X0 = np.ascontiguousarray(X0, dtype=dtype)
    B, n = X0.shape
    p = (param if param is not None else LBFGSParam())._c()
    d0 = None if data0 is None else np.ascontiguousarray(data0, dtype=dtype).reshape(-1)
    d1 = None if data1 is None else np.ascontiguousarray(data1, dtype=dtype).reshape(-1)
    X = np.empty_like(X0)
    dB, dH = np.empty((B, n), dtype=dtype), np.empty((B, n), dtype=dtype)
    items = (_SmallItem * B)()
    suf = "f32" if np.dtype(dtype) == np.float32 else "f64"
    fn = getattr(drv, "lbfgsb200_drv_small_batch_hessian_diag_" + suf)
    err = C.create_string_buffer(256)
    r = fn(device, objective, n, B, _ptr(X0), _ptr(d0), _ptr(d1), int(ldd), _ls_id(linesearch), C.byref(p), _ptr(X), _ptr(dB), _ptr(dH), items,
           err, len(err))
    if r < 0:
        raise (ValueError if r == -1 else RuntimeError)("small_batch_hessian_diagonal failed: %s" % err.value.decode())
    res = [dict(status=STATUS_NAMES[it.kind], code=it.code, niter=it.niter, nfev=it.nfev, fx=it.fx, gnorm=it.gnorm, rounds=it.rounds)
           for it in items]
    return res, X, dB, dH


class SmallHistory:
    """The kept final approximations of a small-batch solve (lbfgs_b200_small_hist) through the C ABI: create, minimize-keep, info,
    columns and products."""

    def __init__(self, ctx, n, m, B, dtype=np.float64):
        self.ctx, self.n, self.m, self.B, self.dtype = ctx, n, m, B, np.dtype(dtype)
        self.suf = "f64" if self.dtype == np.float64 else "f32"
        self.ct = C.c_double if self.dtype == np.float64 else C.c_float
        self.h = C.c_void_p()
        ctx.check(ctx.lib.lbfgs_b200_small_hist_create(ctx.h, n, m, self.dtype.itemsize, B, C.byref(self.h)))

    def __del__(self):
        try:
            if self.h and self.ctx.h:
                self.ctx.lib.lbfgs_b200_small_hist_destroy(self.h)
            self.h = None
        except Exception:
            pass

    def minimize(self, objective, X, param, linesearch="MoreThuente", data0=None, data1=None, ldd=0, ldx=None, G=None, keep=True):
        """lbfgs_b200_small_minimize_keep_* (keep=False: the plain lbfgs_b200_small_minimize_*) on DeviceArrays; returns the raw
        outcomes (a ctypes array of lbfgs_b200_outcome)."""
        outs = (_Outcome * self.B)()
        p = _AbiParam(*(getattr(param, f) for f, _ in _AbiParam._fields_))
        args = [self.ctx.h, objective, data0.ptr if data0 is not None else None, data1.ptr if data1 is not None else None, ldd, self.n, self.B,
                C.byref(p), _ls_id(linesearch), X.ptr, self.n if ldx is None else ldx, G.ptr if G is not None else None, outs]
        if keep:
            self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_small_minimize_keep_" + self.suf)(*args, self.h))
        else:
            self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_small_minimize_" + self.suf)(*args))
        return outs

    def info(self):
        """(c, theta): per-problem pair counts and theta, arrays of B."""
        c = np.zeros(self.B, dtype=np.int32)
        th = np.zeros(self.B, dtype=self.dtype)
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_small_hist_info_" + self.suf)(self.h, c.ctypes.data_as(C.c_void_p),
                                                                                        th.ctypes.data_as(C.c_void_p)))
        return c, th

    def column(self, which, b, age):
        fn = self.ctx.lib.lbfgs_b200_small_hist_s_col if which == "s" else self.ctx.lib.lbfgs_b200_small_hist_y_col
        p = fn(self.h, b, age)
        if not p:
            raise IndexError("no such column")
        out = np.empty(self.n, dtype=self.dtype)
        self.ctx.check(self.ctx.lib.lbfgs_b200_memcpy_d2h(self.ctx.h, out.ctypes.data_as(C.c_void_p), p, out.nbytes))
        return out

    def times(self, inverse, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop):
        """lbfgs_b200_small_hist_times_* on DeviceArrays (asynchronous)."""
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_small_hist_times_" + self.suf)(self.h, int(inverse), b0, count, k, V.ptr, ldv, ldvp,
                                                                                         OUT.ptr, ldo, ldop))

    def diagonal(self, inverse, b0, count, OUT, ldo):
        """lbfgs_b200_small_hist_diag_* into the DeviceArray OUT, problem b0 + p's diagonal at offset p*ldo (asynchronous)."""
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_small_hist_diag_" + self.suf)(self.h, int(inverse), b0, count, OUT.ptr, ldo))

    def factor_times(self, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop):
        """lbfgs_b200_small_hist_factor_times_*: OUT = L_b V with H_b = L_b L_b', on DeviceArrays (asynchronous)."""
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_small_hist_factor_times_" + self.suf)(self.h, b0, count, k, V.ptr, ldv, ldvp, OUT.ptr,
                                                                                                ldo, ldop))

    def sample(self, seed, first, b0, count, k, MEAN, ldm, OUT, ldo, ldop):
        """lbfgs_b200_small_hist_sample_*: OUT = MEAN_b + L_b z_j, z_j draw first + j of stream b; MEAN a DeviceArray or None."""
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_small_hist_sample_" + self.suf)(
            self.h, seed, first, b0, count, k, MEAN.ptr if MEAN is not None else None, ldm, OUT.ptr, ldo, ldop))

    def factor_apply(self, op, b0, count, k, V, ldv, ldvp, OUT, ldo, ldop):
        """lbfgs_b200_small_hist_factor_apply_*: OUT = op(L_b) V (op one of FACTOR_OPS), on DeviceArrays (asynchronous)."""
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_small_hist_factor_apply_" + self.suf)(self.h, _op_id(op), b0, count, k, V.ptr, ldv,
                                                                                                ldvp, OUT.ptr, ldo, ldop))

    def log_density(self, b0, count, k, X, ldx, ldxp, MEAN, ldm):
        """lbfgs_b200_small_hist_log_density_*: log N(x_pj; MEAN_p, H_b) for problems b0 .. b0+count-1, a (count, k) array."""
        out = np.zeros((count, k))
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_small_hist_log_density_" + self.suf)(
            self.h, b0, count, k, X.ptr, ldx, ldxp, MEAN.ptr, ldm, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def logdet(self, b0=0, count=None):
        """lbfgs_b200_small_hist_logdet_*: log det H_b for problems b0 .. b0+count-1 (NaN where the pairs fail the check)."""
        count = self.B - b0 if count is None else count
        out = np.zeros(count)
        self.ctx.check(getattr(self.ctx.lib, "lbfgs_b200_small_hist_logdet_" + self.suf)(self.h, b0, count,
                                                                                          out.ctypes.data_as(C.POINTER(C.c_double))))
        return out


def phase_clock(on=True):
    """Enable / disable (and clear) the wall-clock accounting of the host-driven L-BFGS-B loop's phases (LBFGSpp/PhaseClock.h)."""
    driver().lbfgsb200_drv_phase_enable(int(on))


def phase_report():
    import json
    buf = C.create_string_buffer(8192)
    driver().lbfgsb200_drv_phase_report(buf, 8192)
    return json.loads(buf.value.decode() or "{}")


def driver_ctx(device=0):
    """The lbfgs_b200_ctx* the driver uses for `device` (so that the raw ABI / profiling can address it)."""
    return C.c_void_p(driver().lbfgsb200_drv_ctx(device))


def comm_init(device, unique_id_bytes, rank, nranks, index_offset=0):
    """Attach an NCCL communicator to the driver's context of `device`: n is sharded over `nranks` GPUs."""
    buf = C.create_string_buffer(bytes(unique_id_bytes), 128)
    _checked("comm_init", lambda *err: driver().lbfgsb200_drv_comm_init(device, buf, rank, nranks, index_offset, *err))


def p2p_export(device):
    """64-byte cudaIpc handle of this rank's inbox for the in-kernel NVLink all-reduce."""
    buf = C.create_string_buffer(64)
    _checked("p2p_export", lambda *err: driver().lbfgsb200_drv_p2p_export(device, buf, *err))
    return buf.raw


def p2p_attach(device, all_handles, rank, nranks, index_offset=0):
    """all_handles: the nranks 64-byte handles concatenated in rank order."""
    buf = C.create_string_buffer(bytes(all_handles), 64 * nranks)
    _checked("p2p_attach", lambda *err: driver().lbfgsb200_drv_p2p_attach(device, buf, rank, nranks, index_offset, *err))


def set_global_extent(device, index_offset, n_global):
    """Declare this rank's block of the global vector (needed by the chained-Rosenbrock / tridiagonal objectives when sharded:
    they exchange one boundary coordinate per side with the neighbouring ranks before every evaluation)."""
    _checked("set_global_extent", lambda *err: driver().lbfgsb200_drv_set_global_extent(device, index_offset, n_global, *err))


def comm_unique_id():
    buf = C.create_string_buffer(128)
    st = abi().lbfgs_b200_comm_unique_id(buf)
    if st:
        raise RuntimeError("ncclGetUniqueId failed")
    return buf.raw


def build_all(force=False):
    return _build.build_all(force)
