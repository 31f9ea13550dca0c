"""OWLQNSolver(param, lam, w) (include/OWLQN.h) and the driver's weighted lbfgsb200_drv_owlqn_* on the host-memory test double
(tests/cpp/mock_abi_owlqn.cpp) against the C++ checker (tests/cpp/owlqn_oracle.hpp) with weights bit for bit: seeded runs of the four
built-in objectives, both routes, both precisions, under unit, mixed and all-zero weights; unit weights against the unweighted solver;
and the refusal of bad weights before any trial."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb
from test_owlqn_cpu import tridiag_data
from test_hessian_whiten_cpu import CXX, DRIVER_FLAGS, driver_on
from test_owlqn_front_cpu import CASES, CPP, ORC_SUM_SEQUENTIAL


def weighted_checker(tmp_path_factory):
    """liblbfgs-free build of the weighted C++ checker's entry points (owlqn_oracle_weighted_f64 / _f32), typed"""
    so = str(tmp_path_factory.mktemp("owlqn_oracle_weighted") / "owlqn_oracle_weighted.so")
    subprocess.run(CXX + ["-fPIC", "-shared", "-o", so, os.path.join(CPP, "owlqn_oracle_capi.cpp")], check=True)
    lib = C.CDLL(so)
    for suf, pt in (("f64", C.POINTER(C.c_double)), ("f32", C.POINTER(C.c_float))):
        getattr(lib, "owlqn_oracle_weighted_" + suf).argtypes = [C.c_int, pt, pt, C.c_long, C.POINTER(lb._DrvParam), C.c_double, pt, C.c_int,
                                                                 pt, pt, C.POINTER(lb._OwlqnResult)]
    return lib


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    return weighted_checker(tmp_path_factory)


@pytest.fixture(scope="module")
def front(tmp_path_factory):
    return driver_on(tmp_path_factory, os.path.join(CPP, "mock_abi_owlqn.cpp"), "front_on_owlqn_mock_weighted")


def checker_run_w(lib, obj, x0, lam, w, prm, dtype, d0=None, d1=None, mode=ORC_SUM_SEQUENTIAL):
    x = np.array(x0, dtype=dtype)
    g = np.zeros_like(x)
    w = np.ascontiguousarray(w, dtype=dtype)
    d0, d1 = (None if a is None else np.ascontiguousarray(a, dtype=dtype) for a in (d0, d1))
    res = lb._OwlqnResult()
    p = prm._c()
    fn = lib.owlqn_oracle_weighted_f64 if np.dtype(dtype) == np.float64 else lib.owlqn_oracle_weighted_f32
    fn(obj, lb._ptr(d0), lb._ptr(d1), x.size, C.byref(p), lam, lb._ptr(w), mode, lb._ptr(x), lb._ptr(g), C.byref(res))
    return dict(status=lb.STATUS_NAMES[res.status], msg=res.msg.decode(), niter=res.niter, nfev=res.nfev, fx=res.fx, gnorm=res.gnorm, x=x,
                grad=g)


def weights(kind, n, seed):
    if kind == "ones":
        return np.ones(n)
    if kind == "zeros":
        return np.zeros(n)
    rng = np.random.default_rng(seed + 1000)
    w = rng.choice([0.0, 0.5, 1.0, 3.0], n)
    w[[0, n - 1]] = 0.0                      # the first and last coordinate (the neighbours of the block's ends)
    w[3::4] = 0.0 if n > 8 else w[3::4]      # the last lane of every pack of 4
    return w


def start(n, seed):
    rng = np.random.default_rng(seed)
    x0 = rng.uniform(-2, 2, n)
    x0[rng.random(n) < 0.2] = 0.0
    return x0


def same(got, want):
    assert (got["status"], got["nfev"]) == (want["status"], want["nfev"]), (got["msg"], want["msg"])
    if want["status"] == "ok":
        assert got["niter"] == want["niter"]
        assert got["fx"] == want["fx"] and got["gnorm"] == want["gnorm"]
        assert np.array_equal(got["x"], want["x"]) and np.array_equal(got["grad"], want["grad"])
    else:
        assert got["msg"] == want["msg"]


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("plain", [False, True], ids=["fused", "unfused"])
@pytest.mark.parametrize("wkind", ["ones", "mixed", "zeros"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_weighted_front_matches_checker(front, checker, case, wkind, plain, dtype):
    _, obj, n, lam, kw, seed = case
    x0 = start(n, seed)
    w = weights(wkind, n, seed)
    d0, d1 = tridiag_data(n, seed) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
    prm = lb.LBFGSParam(**kw)
    got = lb.OWLQNSolver(prm, lam, weights=w, dtype=dtype, lib=front).minimize(obj, x0.astype(dtype), d0, d1, plain=plain)
    want = checker_run_w(checker, obj, x0.astype(dtype), lam, w, prm, dtype, d0, d1)
    same(got, want)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("plain", [False, True], ids=["fused", "unfused"])
@pytest.mark.parametrize("case", CASES[::3], ids=[c[0] for c in CASES[::3]])
def test_unit_weights_give_unweighted_bits(front, case, plain, dtype):
    """w = 1 reproduces OWLQNSolver(param, lam): iterations, evaluations, F, ||pg||, x, grad f, or the same exception"""
    _, obj, n, lam, kw, seed = case
    x0 = start(n, seed).astype(dtype)
    d0, d1 = tridiag_data(n, seed) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
    prm = lb.LBFGSParam(**kw)
    a = lb.OWLQNSolver(prm, lam, weights=np.ones(n), dtype=dtype, lib=front).minimize(obj, x0, d0, d1, plain=plain)
    b = lb.OWLQNSolver(prm, lam, dtype=dtype, lib=front).minimize(obj, x0, d0, d1, plain=plain)
    same(a, b)


def test_weighted_cases_cover_every_exit(checker):
    """The mixed-weight runs end by each stopping rule and by each search failure they name."""
    seen = set()
    for _, obj, n, lam, kw, seed in CASES:
        d0, d1 = tridiag_data(n, seed) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
        r = checker_run_w(checker, obj, start(n, seed), lam, weights("mixed", n, seed), lb.LBFGSParam(**kw), np.float64, d0, d1)
        seen.add(r["msg"] if r["status"] != "ok" else "ok")
    assert "ok" in seen
    assert "the line search routine reached the maximum number of iterations" in seen
    assert "the line search step became smaller than the minimum value allowed" in seen


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("plain", [False, True], ids=["fused", "unfused"])
def test_bad_weights_refused_before_any_trial(front, checker, plain, dtype):
    """A negative, NaN or infinite weight, or one with lam * w overflowing, is std::invalid_argument after the one evaluation at x0
    (the first sums pass finds it), before any trial; the checker refuses at the same point."""
    n = 16
    big = 1e308 if dtype == np.float64 else 1e38
    for bad in (-1.0, float("nan"), float("inf"), big):
        w = np.ones(n)
        w[5] = bad
        r = lb.OWLQNSolver(lb.LBFGSParam(), 10.0, weights=w, dtype=dtype, lib=front).minimize(lb.OBJ_QUAD_SHIFT, np.zeros(n, dtype),
                                                                                              plain=plain)
        assert r["status"] == "invalid_argument" and r["nfev"] == 1, r
        c = checker_run_w(checker, lb.OBJ_QUAD_SHIFT, np.zeros(n, dtype), 10.0, w, lb.LBFGSParam(), dtype)
        assert c["status"] == "invalid_argument" and c["nfev"] == 1, c


def test_front_refuses_weights_of_another_size_or_device(tmp_path_factory):
    """OWLQNSolver(param, lambda, w).minimize() throws std::invalid_argument before any evaluation when w's size or device is not x's."""
    so = str(tmp_path_factory.mktemp("owlqn_wcheck") / "owlqn_wcheck.so")
    subprocess.run(CXX + DRIVER_FLAGS + ["-o", so] + [os.path.join(CPP, "owlqn_weights_front_check.cpp"), os.path.join(CPP, "mock_abi_owlqn.cpp"),
                                                     "-pthread"], check=True)
    fn = C.CDLL(so).owlqn_weights_front_check
    fn.argtypes = [C.c_long, C.c_long, C.c_int]
    assert fn(16, 15, 0) == 1 and fn(16, 17, 0) == 1 and fn(16, 16, 1) == 1
    assert fn(16, 16, 0) == 0
