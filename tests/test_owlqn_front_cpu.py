"""OWLQNSolver (include/OWLQN.h) and the driver's lbfgsb200_drv_owlqn_* on the host-memory test double (tests/cpp/mock_abi_owlqn.cpp)
against the C++ checker (tests/cpp/owlqn_oracle.hpp) bit for bit: seeded runs of the four built-in objectives, both routes (fused
projected trial, and projection -> plain functor -> sums), both precisions: iterations, evaluations, F, x, and the exception type and
message of the runs that fail."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb
from test_hessian_whiten_cpu import CXX, driver_on
from test_owlqn_cpu import tridiag_data

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")
OBJS = [lb.OBJ_QUAD_SHIFT, lb.OBJ_ROSENBROCK_PAIRED, lb.OBJ_ROSENBROCK_CHAINED, lb.OBJ_QUAD_TRIDIAG]
ORC_SUM_SEQUENTIAL, ORC_SUM_LANES8 = 0, 1


def owlqn_checker(tmp_path_factory):
    """liblbfgs-free build of the C++ checker's entry points (owlqn_oracle_f64 / _f32)."""
    so = str(tmp_path_factory.mktemp("owlqn_oracle") / "owlqn_oracle.so")
    subprocess.run(CXX + ["-fPIC", "-shared", "-o", so, os.path.join(CPP, "owlqn_oracle_capi.cpp")], check=True)
    lib = C.CDLL(so)
    for suf, pt in (("f64", C.POINTER(C.c_double)), ("f32", C.POINTER(C.c_float))):
        getattr(lib, "owlqn_oracle_" + suf).argtypes = [C.c_int, pt, pt, C.c_long, C.POINTER(lb._DrvParam), C.c_double, C.c_int, pt, pt,
                                                        C.POINTER(lb._OwlqnResult)]
    return lib


def checker_run(lib, obj, x0, lam, prm, dtype, d0=None, d1=None, mode=ORC_SUM_SEQUENTIAL):
    x = np.array(x0, dtype=dtype)
    g = np.zeros_like(x)
    d0, d1 = (None if a is None else np.ascontiguousarray(a, dtype=dtype) for a in (d0, d1))
    res = lb._OwlqnResult()
    p = prm._c()
    fn = lib.owlqn_oracle_f64 if np.dtype(dtype) == np.float64 else lib.owlqn_oracle_f32
    fn(obj, lb._ptr(d0), lb._ptr(d1), x.size, C.byref(p), lam, mode, lb._ptr(x), lb._ptr(g), C.byref(res))
    return dict(status=lb.STATUS_NAMES[res.status], msg=res.msg.decode(), niter=res.niter, nfev=res.nfev, fx=res.fx, gnorm=res.gnorm, x=x,
                grad=g)


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    return owlqn_checker(tmp_path_factory)


@pytest.fixture(scope="module")
def front(tmp_path_factory):
    return driver_on(tmp_path_factory, os.path.join(CPP, "mock_abi_owlqn.cpp"), "front_on_owlqn_mock")


def seeded_cases():
    """(id, objective, n, lam, param kwargs, x0 seed): sparse and dense solutions, every stopping rule, and failing searches"""
    out = []
    for obj in OBJS:
        for n in (2, 7, 64, 301):
            if obj == lb.OBJ_ROSENBROCK_PAIRED and n % 2:
                continue
            lam = {lb.OBJ_QUAD_SHIFT: 0.4 * n, lb.OBJ_ROSENBROCK_PAIRED: 0.5, lb.OBJ_ROSENBROCK_CHAINED: 0.3, lb.OBJ_QUAD_TRIDIAG: 0.6}[obj]
            out.append(("obj%d_n%d" % (obj, n), obj, n, lam, dict(m=6, max_iterations=100), n))
        n = 64
        out.append(("obj%d_past" % obj, obj, n, 0.2, dict(m=3, past=2, delta=1e-6, max_iterations=100), 1))
        out.append(("obj%d_cap" % obj, obj, n, 0.2, dict(m=10, max_iterations=7), 2))
        out.append(("obj%d_one_trial" % obj, obj, n, 0.05, dict(max_linesearch=1, max_iterations=100), 3))
        out.append(("obj%d_min_step" % obj, obj, n, 0.05, dict(min_step=0.9, max_iterations=100), 4))
    return out


CASES = seeded_cases()


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("plain", [False, True], ids=["fused", "unfused"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_front_matches_checker(front, checker, case, plain, dtype):
    _, obj, n, lam, kw, seed = case
    rng = np.random.default_rng(seed)
    x0 = rng.uniform(-2, 2, n)
    x0[rng.random(n) < 0.2] = 0.0
    d0, d1 = tridiag_data(n, seed) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
    prm = lb.LBFGSParam(**kw)
    got = lb.OWLQNSolver(prm, lam, dtype=dtype, lib=front).minimize(obj, x0.astype(dtype), d0, d1, plain=plain)
    want = checker_run(checker, obj, x0.astype(dtype), lam, prm, dtype, d0, d1)
    assert (got["status"], got["msg"], got["nfev"]) == (want["status"], want["msg"], want["nfev"])
    if want["status"] == "ok":
        assert got["niter"] == want["niter"]
        assert got["fx"] == want["fx"] and got["gnorm"] == want["gnorm"]
        assert np.array_equal(got["x"], want["x"]) and np.array_equal(got["grad"], want["grad"])


def test_cases_cover_every_exit(front, checker):
    """The seeded cases end by each stopping rule and by each search failure they name."""
    seen = set()
    for _, obj, n, lam, kw, seed in CASES:
        rng = np.random.default_rng(seed)
        x0 = rng.uniform(-2, 2, n)
        x0[rng.random(n) < 0.2] = 0.0
        d0, d1 = tridiag_data(n, seed) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
        r = checker_run(checker, obj, x0, lam, lb.LBFGSParam(**kw), np.float64, d0, d1)
        seen.add(r["msg"] if r["status"] != "ok" else "ok")
    assert "ok" in seen
    assert "the line search routine reached the maximum number of iterations" in seen
    assert "the line search step became smaller than the minimum value allowed" in seen


def test_checker_sum_modes(checker):
    """The checker in both summation modes: QuadShift's closed form max(i - lam/2, 0) to 1e-8, with its zero pattern."""
    n, lam = 300, 100.0
    prm = lb.LBFGSParam(m=6, epsilon=1e-10, epsilon_rel=0.0, max_iterations=200)
    for mode in (ORC_SUM_SEQUENTIAL, ORC_SUM_LANES8):
        r = checker_run(checker, lb.OBJ_QUAD_SHIFT, np.zeros(n), lam, prm, np.float64, mode=mode)
        assert r["status"] == "ok", r["msg"]
        want = np.maximum(np.arange(n) - lam / 2, 0.0)
        assert np.max(np.abs(r["x"] - want)) <= 1e-8
        assert np.array_equal(r["x"] == 0, want == 0)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_front_refusals_on_double(front, dtype):
    """The C ABI refusals as the front meets them: a lambda that is not positive and finite is refused before any evaluation."""
    for lam in (0.0, -1.0, float("nan"), float("inf")):
        r = lb.OWLQNSolver(lb.LBFGSParam(), lam, dtype=dtype, lib=front).minimize(lb.OBJ_QUAD_SHIFT, np.zeros(8, dtype=dtype))
        assert r["status"] == "invalid_argument" and r["nfev"] == 0, r
