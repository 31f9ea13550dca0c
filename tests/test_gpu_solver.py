"""GPU parity tests, solver level: LBFGSSolver<Scalar, LineSearch>::minimize on the H100 against the CPU checker.

Parity definition (SURVEY.md 8c): same return value (iterations), same number of objective evaluations,
|fx_gpu - fx_cpu| <= 1e-10 * max(1, |fx_cpu|), |x_gpu - x_cpu|_inf <= 1e-8 * max(1, |x|_inf), and the per-evaluation
trace of f equal to a relative tolerance that starts at 1e-10 and is allowed to grow with the evaluation index
(L-BFGS amplifies last-bit differences of the dot products; the CPU checker shows the same growth between two
summation orders of its own, see test_oracle_cpu.py::test_lanes_and_omp_modes_agree_with_sequential)."""
import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po
from util import LS, golden_cases, unhex

pytestmark = pytest.mark.gpu

LS_NAMES = ["Backtracking", "Bracketing", "NocedalWright", "MoreThuente"]


def check_parity(g, c, trace_rtol0=1e-10, growth=4.0, xtol=1e-8):
    assert g["status"] == c["status"], (g["status"], g["msg"], c["status"], c["msg"])
    assert g["msg"] == c["msg"]
    assert (g["niter"], g["nfev"]) == (c["niter"], c["nfev"])
    if c["status"] != "ok":
        return
    assert abs(g["fx"] - c["fx"]) <= 1e-10 * max(1.0, abs(c["fx"]))
    assert np.max(np.abs(g["x"] - c["x"])) <= xtol * max(1.0, np.max(np.abs(c["x"])))
    k = np.arange(len(c["trace"]))
    tol = np.minimum(trace_rtol0 * growth ** k, 1e-3) * np.maximum(np.abs(c["trace"]), 1e-6 * abs(c["trace"][0]) + 1e-300)
    assert np.all(np.abs(g["trace"] - c["trace"]) <= tol), np.max(np.abs(g["trace"] - c["trace"]) / tol)


def cpu_param(orc, prm):
    return orc.default_param(**{k: getattr(prm, k) for k in ("m", "epsilon", "epsilon_rel", "past", "delta", "max_iterations",
                                                               "linesearch", "max_linesearch", "min_step", "max_step", "ftol", "wolfe")})


@pytest.mark.parametrize("ls", LS_NAMES)
@pytest.mark.parametrize("fused", [True, False])
def test_config1_rosenbrock_n10(orc, ls, fused):
    """BASELINE config 1: example-rosenbrock.cpp (float -> double), default parameters."""
    prm = lb.LBFGSParam()
    g = lb.LBFGSSolver(prm, ls, fused=fused).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(10))
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, np.zeros(10), LS[ls], cpu_param(orc, prm))
    check_parity(g, c)
    assert g["launches"] > 0


@pytest.mark.parametrize("hv", [lb.HV_TWO_LOOP, lb.HV_AUTO])
@pytest.mark.parametrize("n", [1000, 100000, 1000000])
def test_config2_shape_rosenbrock_m10_more_thuente(orc, n, hv):
    """BASELINE config 2 at sizes the CPU checker finishes in seconds (the full n = 1e7 run is in bench.py)."""
    prm = lb.LBFGSParam(m=10)
    g = lb.LBFGSSolver(prm, "MoreThuente", hv_algo=hv).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n))
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, np.zeros(n), LS["MoreThuente"], cpu_param(orc, prm), sum_mode=po.SUM_LANES8)
    check_parity(g, c, xtol=1e-7)


def test_config3_shape_quadratic_m20_bracketing(orc):
    n = 20000
    d, b, xs = po.quad_tridiag_data(n, kappa=1e3, seed=0)
    prm = lb.LBFGSParam(m=20)
    g = lb.LBFGSSolver(prm, "Bracketing").minimize(lb.OBJ_QUAD_TRIDIAG, np.zeros(n), data0=d, data1=b)
    c = orc.lbfgs(po.OBJ_QUAD_TRIDIAG, np.zeros(n), LS["Bracketing"], cpu_param(orc, prm), data0=d, data1=b)
    assert g["status"] == "ok" and c["status"] == "ok"
    # a 100+-iteration run: demand the relative-on-fx parity and iteration counts within a few percent
    assert abs(g["fx"] - c["fx"]) <= 1e-9 * abs(c["fx"])
    assert abs(g["niter"] - c["niter"]) <= max(3, c["niter"] // 20)
    assert np.max(np.abs(g["x"] - xs)) <= 1e-3


def test_quadratic_example(orc):
    g = lb.LBFGSSolver(lb.LBFGSParam()).minimize(lb.OBJ_QUAD_SHIFT, np.zeros(10))
    assert g["niter"] == 2 and np.allclose(g["x"], np.arange(10.0), atol=1e-12)


@pytest.mark.parametrize("ls", LS_NAMES)
def test_random_starts_property(ls):
    """The self-checking examples' criterion (example-rosenbrock-comparison.cpp:44-51): |x - 1|_inf <= 1e-4."""
    rng = np.random.default_rng(11)
    prm = lb.LBFGSParam(max_linesearch=256)
    for n in (2, 8, 24):
        for _ in range(4):
            g = lb.LBFGSSolver(prm, ls).minimize(lb.OBJ_ROSENBROCK_PAIRED, rng.uniform(-1, 1, n))
            assert g["status"] == "ok" and np.max(np.abs(g["x"] - 1.0)) <= 1e-4


def test_float32_solver(orc):
    prm = lb.LBFGSParam()
    g = lb.LBFGSSolver(prm, "NocedalWright", dtype=np.float32).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(10))
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, np.zeros(10), LS["NocedalWright"], cpu_param(orc, prm), dtype=np.float32)
    assert g["status"] == "ok" and abs(g["niter"] - c["niter"]) <= 3 and np.max(np.abs(g["x"] - 1.0)) <= 1e-2


@pytest.mark.parametrize("case", [c for c in golden_cases("lbfgs") if c["dtype"] == "f64"], ids=lambda c: c["name"])
def test_golden_vectors_from_reference_headers(case):
    """Frozen outputs of the unmodified reference headers (tests/golden/make_golden.py)."""
    prm = lb.LBFGSParam(**case["param"])
    d0, d1 = (unhex(case["data"][0]), unhex(case["data"][1])) if case["data"] else (None, None)
    g = lb.LBFGSSolver(prm, case["ls"]).minimize(case["objective"], unhex(case["x0"]), data0=d0, data1=d1)
    c = dict(status=case["status"], msg=case["msg"], niter=case["niter"], nfev=case["nfev"], fx=float.fromhex(case["fx"]),
             x=unhex(case["x"]), trace=unhex(case["trace"]))
    long_run = case["niter"] > 60
    if long_run:  # chaotic regime: compare the optimum, not the path
        assert g["status"] == c["status"] and abs(g["fx"] - c["fx"]) <= 1e-9 * max(1.0, abs(c["fx"]))
    else:
        check_parity(g, c, xtol=1e-6)


def test_exceptions_map_to_python():
    with pytest.raises(ValueError):
        lb.LBFGSSolver(lb.LBFGSParam(m=0)).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(4), raise_errors=True)
    with pytest.raises(RuntimeError):
        lb.LBFGSSolver(lb.LBFGSParam(max_linesearch=1), "Backtracking").minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(4), raise_errors=True)
