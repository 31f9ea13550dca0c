"""The product's header-only front on a CPU: include/LBFGS.h + LBFGSpp/*.h + lbfgspp_b200/csrc/driver.cpp compiled against
tests/cpp/mock_abi.cpp, a host-memory TEST DOUBLE of the C ABI that takes every sum left to right with the CPU checker's own
routines.  With rounding taken out of the picture, everything the front decides (solver loop, first step, line-search drivers
and state machines, snapshot swaps, curvature gate, convergence rules, evaluation counting, exception types and messages) must
reproduce the checker -- which is pinned to the unmodified reference headers -- bit for bit.  No GPU code runs here; the
kernels' own parity is the job of the -m gpu tests."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po
from util import LS, golden_cases, unhex

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "tests", "cpp", "front_on_mock.so")


@pytest.fixture(scope="module")
def front():
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-march=x86-64-v3", "-fPIC", "-shared", "-Wall",
                    "-Wno-unknown-pragmas", "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic", "-o", SO,
                    os.path.join(ROOT, "lbfgspp_b200", "csrc", "driver.cpp"), os.path.join(ROOT, "tests", "cpp", "mock_abi.cpp"),
                    "-pthread"], check=True)
    return C.CDLL(SO)


def cpu_param(orc, prm):
    return orc.default_param(**{k: getattr(prm, k) for k in ("m", "epsilon", "epsilon_rel", "past", "delta", "max_iterations",
                                                               "linesearch", "max_linesearch", "min_step", "max_step", "ftol", "wolfe")})


def assert_same(f, c, where):
    assert f["status"] == c["status"] and f["msg"].replace("lbfgs_b200: ", "") == c["msg"], (where, f["status"], f["msg"], c["status"], c["msg"])
    assert (f["niter"], f["nfev"]) == (c["niter"], c["nfev"]), where
    assert np.array_equal(f["trace"], c["trace"]), where
    if c["status"] == "ok":
        assert f["fx"] == c["fx"] and f["gnorm"] == c["gnorm"], where
        assert np.array_equal(f["x"].astype(np.float64), c["x"].astype(np.float64)), where
        assert np.array_equal(f["grad"].astype(np.float64), c["grad"].astype(np.float64)), where


@pytest.mark.parametrize("fused", [1, 0])
@pytest.mark.parametrize("case", [c for c in golden_cases("lbfgs")], ids=lambda c: c["name"])
def test_front_reproduces_golden_vectors_bit_for_bit(front, orc, case, fused):
    dtype = np.float64 if case["dtype"] == "f64" else np.float32
    prm = lb.LBFGSParam(**case["param"])
    d0, d1 = (unhex(case["data"][0]), unhex(case["data"][1])) if case["data"] else (None, None)
    f = lb.LBFGSSolver(prm, LS[case["ls"]], dtype=dtype, fused=fused, lib=front).minimize(case["objective"], unhex(case["x0"]), data0=d0, data1=d1)
    assert f["status"] == case["status"] and f["msg"].replace("lbfgs_b200: ", "") == case["msg"]
    assert (f["niter"], f["nfev"]) == (case["niter"], case["nfev"])
    assert np.array_equal(f["trace"], unhex(case["trace"]))
    if case["status"] == "ok":
        assert float(f["fx"]).hex() == case["fx"] and float(f["gnorm"]).hex() == case["gnorm"]
        assert np.array_equal(f["x"].astype(np.float64), unhex(case["x"]))
        assert np.array_equal(f["grad"].astype(np.float64), unhex(case["grad"]))


@pytest.mark.parametrize("ls", ["Backtracking", "Bracketing", "NocedalWright", "MoreThuente"])
def test_front_equals_checker_on_random_problems(front, orc, ls):
    rng = np.random.default_rng(5)
    for n in (2, 6, 24, 100, 2002):
        for t in range(5):
            x0 = rng.uniform(-1, 1, n)
            prm = lb.LBFGSParam(m=3 + t % 8, max_linesearch=int(rng.choice([20, 64, 256])), past=int(rng.choice([0, 0, 3])),
                                delta=1e-9, linesearch=int(rng.choice([1, 2, 3])) if ls != "NocedalWright" and ls != "MoreThuente" else 3)
            c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, LS[ls], cpu_param(orc, prm))
            for fused in (1, 0):
                assert_same(lb.LBFGSSolver(prm, LS[ls], fused=fused, lib=front).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0), c, (ls, n, t, fused))
    n = 3000
    d, b, _ = po.quad_tridiag_data(n)
    prm = lb.LBFGSParam(m=20)
    c = orc.lbfgs(po.OBJ_QUAD_TRIDIAG, np.zeros(n), LS[ls], cpu_param(orc, prm), data0=d, data1=b)
    assert_same(lb.LBFGSSolver(prm, LS[ls], lib=front).minimize(lb.OBJ_QUAD_TRIDIAG, np.zeros(n), data0=d, data1=b), c, (ls, "tridiag"))
    x0 = np.full(300, 1.3)
    c = orc.lbfgs(po.OBJ_ROSENBROCK_CHAINED, x0, LS[ls], cpu_param(orc, lb.LBFGSParam()))
    assert_same(lb.LBFGSSolver(lb.LBFGSParam(), LS[ls], lib=front).minimize(lb.OBJ_ROSENBROCK_CHAINED, x0), c, (ls, "chained"))


def test_front_error_paths_equal_the_checker(front, orc):
    """Parameter errors, a non-descent / exhausted line search, an already optimal start: same exception type and message."""
    cases = [(lb.LBFGSParam(m=0), "MoreThuente", np.zeros(4)), (lb.LBFGSParam(ftol=0.7), "Backtracking", np.zeros(4)),
             (lb.LBFGSParam(linesearch=1), "NocedalWright", np.zeros(4)), (lb.LBFGSParam(max_linesearch=1), "Backtracking", np.zeros(12)),
             (lb.LBFGSParam(max_linesearch=1), "Bracketing", np.zeros(12)), (lb.LBFGSParam(max_linesearch=1, max_iterations=3), "MoreThuente", np.zeros(12)),
             (lb.LBFGSParam(max_linesearch=1, max_iterations=3), "NocedalWright", np.zeros(12)), (lb.LBFGSParam(max_step=1e-3), "MoreThuente", np.zeros(8)),
             (lb.LBFGSParam(min_step=10.0, max_step=20.0), "Backtracking", np.zeros(8)), (lb.LBFGSParam(), "MoreThuente", np.ones(6)),
             (lb.LBFGSParam(max_iterations=4), "Bracketing", np.zeros(10)), (lb.LBFGSParam(epsilon=0.0, epsilon_rel=0.0, max_iterations=60), "MoreThuente", np.zeros(4))]
    for prm, ls, x0 in cases:
        c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, LS[ls], cpu_param(orc, prm))
        for fused in (1, 0):
            assert_same(lb.LBFGSSolver(prm, LS[ls], fused=fused, lib=front).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0), c, (ls, fused, c["status"], c["msg"]))


def test_front_float32_equals_checker(front, orc):
    for ls in ("Backtracking", "Bracketing", "NocedalWright", "MoreThuente"):
        prm = lb.LBFGSParam()
        c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, np.zeros(10), LS[ls], cpu_param(orc, prm), dtype=np.float32)
        assert_same(lb.LBFGSSolver(prm, LS[ls], dtype=np.float32, lib=front).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(10)), c, ls)


@pytest.mark.parametrize("ls", ["Backtracking", "Bracketing", "NocedalWright", "MoreThuente"])
def test_session_solve_equals_one_shot_minimize(front, ls):
    """A host-driven Session keeps one solver for its line search across solves: every solve, from the resident start point or from
    the host, reproduces a one-shot minimize() bit for bit."""
    n = 300
    d, b, _ = po.quad_tridiag_data(n)
    for objective, x0, data in ((lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n), {}), (lb.OBJ_QUAD_TRIDIAG, np.zeros(n), dict(data0=d, data1=b))):
        prm = lb.LBFGSParam(m=8)
        c = lb.LBFGSSolver(prm, ls, fused=True, lib=front).minimize(objective, x0, **data)
        assert c["status"] == "ok", c["msg"]
        s = lb.Session(objective, x0, prm, ls, resident=False, lib=front, **data)
        try:
            for from_host in (False, True):
                r = s.solve(from_host=from_host, to_host=from_host)
                assert (r["niter"], r["nfev"], r["fx"], r["gnorm"]) == (c["niter"], c["nfev"], c["fx"], c["gnorm"]), (ls, objective, from_host)
                assert np.array_equal(s.solution(), c["x"])
                if from_host:
                    assert np.array_equal(s.result(), c["x"])
            assert s.profile() is None   # the host-driven loop has no device-resident accounting
        finally:
            s.close()


def test_thread_batch_equals_lone_solves(front):
    """The thread-pool batch (host-driven loop: the two-loop recursion keeps built-in objectives off the device-resident solve) gives
    every problem exactly its lone solve, whichever worker thread ran it."""
    rng = np.random.default_rng(3)
    X0 = rng.uniform(-1, 1, (5, 40))
    prm = lb.LBFGSParam(m=5)
    for ls in ("Bracketing", "MoreThuente"):
        res, X, _ = lb.solve_batch(lb.OBJ_ROSENBROCK_PAIRED, X0, prm, ls, hv_algo=lb.HV_TWO_LOOP, threads=2, lib=front)
        for b in range(len(X0)):
            c = lb.LBFGSSolver(prm, ls, hv_algo=lb.HV_TWO_LOOP, lib=front).minimize(lb.OBJ_ROSENBROCK_PAIRED, X0[b])
            assert res[b] == {k: c[k] for k in ("status", "niter", "nfev", "fx", "gnorm")}, (ls, b)
            assert np.array_equal(X[b], c["x"]), (ls, b)


@pytest.mark.parametrize("bad", [4, -1])
def test_every_entry_point_rejects_an_unknown_line_search(front, bad):
    """No entry point that takes a line-search id falls back to a default search on an id it does not know."""
    x0, prm = np.zeros(8), lb.LBFGSParam()
    f = lb.LBFGSSolver(prm, bad, lib=front).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0)
    assert (f["status"], f["msg"]) == ("invalid_argument", "unknown line search id")
    with pytest.raises(RuntimeError, match="^session_create failed: unknown line search id$"):
        lb.Session(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, bad, resident=False, lib=front)
    with pytest.raises(RuntimeError, match="^batch_session_create failed: unknown line search id$"):
        lb.BatchSession(lb.OBJ_ROSENBROCK_PAIRED, np.zeros((2, 8)), prm, bad, lib=front)
    with pytest.raises(RuntimeError, match="^solve_dense failed: unknown line search id$"):
        lb.solve_dense(lb.OBJ_ROSENBROCK_PAIRED, x0, prm, bad, resident=False, lib=front)
    # the thread-pool batch on the host-driven loop (the test double has no device-resident solve): the same call solves every problem
    # with a known id, so "invalid_argument" can only come from the id
    for ls, status in (("MoreThuente", "ok"), (bad, "invalid_argument")):
        res, _, _ = lb.solve_batch(lb.OBJ_ROSENBROCK_PAIRED, np.zeros((5, 8)), prm, ls, hv_algo=lb.HV_TWO_LOOP, threads=2, lib=front)
        assert [r["status"] for r in res] == [status] * 5, ls


# ---- the reference's example programs (examples/*.cpp) against the test double: host-functor compatibility mode, dense B / H ----
@pytest.fixture(scope="module")
def example_bins(tmp_path_factory):
    out = tmp_path_factory.mktemp("examples_on_mock")
    mock_o = str(out / "mock_abi.o")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wno-unknown-pragmas", "-c", "-o", mock_o,
                    os.path.join(ROOT, "tests", "cpp", "mock_abi.cpp")], check=True)
    bins = {}
    for name in ("rosenbrock_host_functor", "quadratic_free_function", "line_search_comparison"):
        exe = str(out / name)
        subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-I", os.path.join(ROOT, "include"), "-o", exe,
                        os.path.join(ROOT, "examples", name + ".cpp"), mock_o], check=True)
        bins[name] = exe
    return bins


def test_examples_run_on_the_test_double(example_bins):
    """Same expectations as tests/test_gpu_examples.py (the reference's own self-checks), host logic only."""
    r = subprocess.run([example_bins["quadratic_free_function"]], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.startswith("2 iterations"), r.stdout + r.stderr
    r = subprocess.run([example_bins["rosenbrock_host_functor"]], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "iterations" in r.stdout and "max |B*H - I|" in r.stdout, r.stdout + r.stderr
    r = subprocess.run([example_bins["line_search_comparison"], "12", "host"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "FAILED" not in r.stdout and r.stdout.count("LineSearchMoreThuente") == 12, r.stdout + r.stderr


# ---- the bound-constrained front (include/LBFGSB.h, LBFGSpp/{Cauchy,SubspaceMin,BFGSMat,BKLDLT}.h) on the test double -------------
def check_box(f, c, lbv, ubv, iter_slack=0):
    """The product's Cauchy sweep (prefix sums over sorted breakpoints) and BOXCQP algebra re-associate sums, so this is parity
    to rounding, not bit for bit: same iterations, evaluations within one, fx to 1e-9, x to 1e-6 (the bar of the GPU tests)."""
    assert f["status"] == c["status"], (f["status"], f["msg"], c["status"], c["msg"])
    if c["status"] != "ok":
        assert f["msg"].replace("lbfgs_b200: ", "") == c["msg"]
        return
    assert abs(f["niter"] - c["niter"]) <= iter_slack, (f["niter"], c["niter"])
    assert abs(f["nfev"] - c["nfev"]) <= iter_slack + 1, (f["nfev"], c["nfev"])
    assert abs(f["fx"] - c["fx"]) <= 1e-9 * max(1.0, abs(c["fx"])), (f["fx"], c["fx"])
    assert np.max(np.abs(f["x"] - c["x"])) <= 1e-6 * max(1.0, np.max(np.abs(c["x"])))
    # feasible up to the rounding of x = xp + step*drt: like the reference, the solver does not clamp the final iterate (LBFGSB.h:208-216
    # return before force_bounds), and the checker shows the same <= 4e-16 excursions on these inputs
    lo, hi = np.broadcast_to(lbv, f["x"].size), np.broadcast_to(ubv, f["x"].size)
    slack = 4 * np.finfo(float).eps * np.maximum(1.0, np.abs(f["x"]))
    assert np.all(f["x"] >= lo - slack) and np.all(f["x"] <= hi + slack)


@pytest.mark.parametrize("case", golden_cases("lbfgsb"), ids=lambda c: c["name"])
def test_box_front_on_golden_vectors(front, case):
    prm = lb.LBFGSBParam(**case["param"])
    lbv, ubv = unhex(case["lb"]), unhex(case["ub"])
    f = lb.LBFGSBSolver(prm).minimize(case["objective"], unhex(case["x0"]), lbv, ubv, lib=front)
    c = dict(status=case["status"], msg=case["msg"], niter=case["niter"], nfev=case["nfev"], fx=float.fromhex(case["fx"]), x=unhex(case["x"]))
    check_box(f, c, lbv, ubv, iter_slack=0 if case["niter"] < 20 else 2)


def test_box_front_equals_checker_on_random_boxes(front, orc):
    rng = np.random.default_rng(8)
    for obj in (po.OBJ_ROSENBROCK_CHAINED, po.OBJ_ROSENBROCK_PAIRED, po.OBJ_QUAD_SHIFT, po.OBJ_QUAD_TRIDIAG):
        for n in (2, 4, 10, 26, 100, 1000):
            for trial in range(5):
                lo = rng.uniform(-2, 1, n)
                hi = lo + rng.uniform(0.1, 3, n)
                if trial == 0:
                    lo[:], hi[:] = 2.0, 4.0
                elif trial == 1:
                    lo[:], hi[:] = -np.inf, np.inf
                elif trial == 2:
                    hi[::3] = lo[::3]
                elif trial == 3:
                    lo[::2], hi[1::3] = -np.inf, np.inf
                x0 = rng.uniform(-3, 5, n)
                d0, d1 = po.quad_tridiag_data(n, seed=trial)[:2] if obj == po.OBJ_QUAD_TRIDIAG else (None, None)
                kw = dict(m=int(rng.choice([1, 3, 6, 10])), max_iterations=12, max_submin=int(rng.choice([0, 1, 10])))
                c = orc.lbfgsb(obj, x0, lo, hi, orc.default_param(lbfgsb=True, **kw), data0=d0, data1=d1)
                f = lb.LBFGSBSolver(lb.LBFGSBParam(**kw)).minimize(obj, x0, lo, hi, data0=d0, data1=d1, lib=front)
                # short runs (<= 12 iterations) keep the comparison in the regime where rounding has not yet moved the path
                check_box(f, c, lo, hi)


def test_box_front_parameter_and_size_errors(front, orc):
    f = lb.LBFGSBSolver(lb.LBFGSBParam(m=0)).minimize(po.OBJ_QUAD_SHIFT, np.zeros(4), 0.0, 1.0, lib=front)
    c = orc.lbfgsb(po.OBJ_QUAD_SHIFT, np.zeros(4), 0.0, 1.0, orc.default_param(lbfgsb=True, m=0))
    assert f["status"] == c["status"] == "invalid_argument" and f["msg"].replace("lbfgs_b200: ", "") == c["msg"]


def test_front_is_sanitizer_clean(tmp_path):
    """driver.cpp + the header-only front + the test double under ASan + UBSan (+ LeakSanitizer at exit) over 522 small solves:
    all line searches, fused / unfused trials, fp32, L-BFGS-B with mixed bounds, the exception paths."""
    exe = str(tmp_path / "front_selfcheck_san")
    r = subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                        "-fno-omit-frame-pointer", "-ffp-contract=off", "-Wno-unknown-pragmas", "-o", exe,
                        os.path.join(ROOT, "tests", "cpp", "front_selfcheck.cpp"), os.path.join(ROOT, "lbfgspp_b200", "csrc", "driver.cpp"),
                        os.path.join(ROOT, "tests", "cpp", "mock_abi.cpp"), "-pthread"], capture_output=True, text=True)
    if r.returncode != 0 and ("cannot find -lasan" in r.stderr or "cannot find -lubsan" in r.stderr):
        pytest.skip("sanitizer runtimes not installed")
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "front selfcheck ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
