"""OWL-QN on the H100: the new kernels against numpy (element-wise outputs bit for bit, sums to a stated tolerance), whole solves of the
four built-in objectives, fused and unfused, fp64 and fp32, against the float64 statement in test_owlqn_cpu, solves at n = 1e6, and the
error paths."""
import ctypes as C

import numpy as np
import pytest

import lbfgspp_b200 as lb
from test_owlqn_cpu import (constrain, kkt_violation, objective, orthant, owlqn, project, pseudo_grad, tridiag_data, two_loop)

pytestmark = pytest.mark.gpu
DT = [np.float64, np.float32]
IDS = ["f64", "f32"]
OBJS = [lb.OBJ_QUAD_SHIFT, lb.OBJ_ROSENBROCK_PAIRED, lb.OBJ_ROSENBROCK_CHAINED, lb.OBJ_QUAD_TRIDIAG]


def sparse_point(rng, n, dtype):
    x = rng.standard_normal(n)
    x[rng.random(n) < 0.3] = 0.0
    return x.astype(dtype)


@pytest.fixture(scope="module")
def owlqn_ctx():
    ctx = lb.Context(0)
    yield ctx
    ctx.close()


@pytest.mark.parametrize("dtype", DT, ids=IDS)
@pytest.mark.parametrize("obj", OBJS)
@pytest.mark.parametrize("n", [2, 6, 1026, 300_002, 300_003])
def test_trial_kernel(owlqn_ctx, dtype, obj, n):
    """The fused projected trial: x and g bit for bit against numpy, the five sums to a relative 1e-12 (fp64) / 1e-5 (fp32)."""
    if obj == lb.OBJ_ROSENBROCK_PAIRED and n % 2:
        pytest.skip("paired Rosenbrock needs an even n")
    rng = np.random.default_rng(n + obj)
    T = np.dtype(dtype).type
    lam, step = T(0.7), T(0.37)
    xp, d, gp = sparse_point(rng, n, dtype), rng.standard_normal(n).astype(dtype), rng.standard_normal(n).astype(dtype)
    gp[::7] = T(0.1)     # |gp| < lam at some zeros: pg = 0 there
    d0, d1 = tridiag_data(n) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
    c = owlqn_ctx
    D0 = c.array(d0.astype(dtype)) if d0 is not None else None
    D1 = c.array(d1.astype(dtype)) if d1 is not None else None
    X, G = c.empty(n, dtype), c.empty(n, dtype)
    out = c.owlqn_trial(obj, c.array(xp), c.array(d), c.array(gp), step, lam, X, G, D0, D1)
    pgp = pseudo_grad(xp, gp, lam)
    x = project(xp + step * d, orthant(xp, pgp))
    f, g = objective(obj, dtype, d0, d1)(x)
    assert np.array_equal(X.get(), x) and np.array_equal(G.get(), g)
    pg = pseudo_grad(x, g, lam).astype(np.float64)
    x64 = x.astype(np.float64)
    want = [f, np.sum(np.abs(x64)), pgp.astype(np.float64) @ (x64 - xp), pg @ pg, x64 @ x64]
    tol = 1e-12 if dtype == np.float64 else 1e-5
    scale = [abs(f), want[1], np.abs(pgp) @ np.abs(x64 - xp), want[3], want[4]]
    for k in range(5):
        assert abs(out[k] - want[k]) <= tol * max(scale[k], 1.0), (k, out[k], want[k])
    # the unfused route: projection kernel, then the sums at (x, g)
    X2 = c.empty(n, dtype)
    p = c.owlqn_project(c.array(xp), c.array(d), c.array(gp), step, lam, X2)
    assert np.array_equal(X2.get(), x)
    assert abs(p[0] - want[1]) <= tol * max(want[1], 1.0) and abs(p[1] - want[2]) <= tol * max(scale[2], 1.0)
    Dd = c.empty(n, dtype)
    s = c.owlqn_sums(X2, c.array(g), lam, Dd)
    assert np.array_equal(Dd.get(), -pseudo_grad(x, g, lam))
    for k, w in zip(range(3), [want[1], want[3], want[4]]):
        assert abs(s[k] - w) <= tol * max(w, 1.0)


@pytest.mark.parametrize("dtype", DT, ids=IDS)
@pytest.mark.parametrize("m", [3, 10, 20])
def test_update_dir_kernels(owlqn_ctx, dtype, m):
    """Pair-forming dots with pg and the constrained combination on random histories of c = 0..m pairs, with the curvature gate
    refusing the first pair (the combination at c = 0) and a later one (pg written into the spare column, then a second dots pass):
    d against the two-loop recursion on pg (1e-10 / 1e-4 of |d|), exactly 0 where the constraint holds with margin, dg = pg.d."""
    c = owlqn_ctx
    n = 5000 + m
    rng = np.random.default_rng(m)
    T = np.dtype(dtype).type
    lam = T(0.3)
    h = lb.History(c, n, m, dtype)
    S, Y = [], []
    x = sparse_point(rng, n, dtype)
    g = rng.standard_normal(n).astype(dtype)
    tol = 1e-10 if dtype == np.float64 else 1e-4
    for it in range(m + 2):
        xn = (x + T(0.1) * rng.standard_normal(n).astype(dtype)).astype(dtype)
        xn[rng.random(n) < 0.2] = 0
        curv = T(-2) if it in (0, 1, m // 2 + 1) else T(2)     # y = -2 s + noise: s'y < 0, the gate refuses the pair
        gn = (g + (xn - x) * curv + T(0.01) * rng.standard_normal(n).astype(dtype)).astype(dtype)
        Dd = c.empty(n, dtype)
        acc, dg = h.owlqn_update_dir(c.array(xn), c.array(x), c.array(gn), c.array(g), lam, Dd)
        s, y = (xn - x).astype(np.float64), (gn - g).astype(np.float64)
        assert acc == bool(s @ y > np.finfo(dtype).eps * (y @ y)) and acc == (curv > 0)
        if acc:
            S.append(s)
            Y.append(y)
            S, Y = S[-m:], Y[-m:]
        theta = (Y[-1] @ Y[-1]) / (S[-1] @ Y[-1]) if S else 1.0
        pg = pseudo_grad(xn, gn, lam).astype(np.float64)
        raw = two_loop(S, Y, pg, theta) if S else -pg / theta
        want = constrain(raw, pg)
        got = Dd.get().astype(np.float64)
        assert np.max(np.abs(got - want)) <= tol * np.max(np.abs(raw))
        clear = np.abs(raw * pg) > 1e-6 * np.max(np.abs(raw * pg))
        assert np.array_equal(got[clear] == 0, want[clear] == 0)
        assert abs(dg - pg @ got) <= tol * max(abs(dg), 1.0)
        x, g = xn, gn


def solve_pair(obj, n, lam, dtype, plain, **kw):
    rng = np.random.default_rng(obj * 100 + n)
    x0 = rng.uniform(-1.5, 1.5, n)
    d0, d1 = tridiag_data(n) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
    prm = lb.LBFGSParam(**kw)
    gpu = lb.OWLQNSolver(prm, lam, dtype=dtype).minimize(obj, x0.astype(dtype), d0, d1, plain=plain)
    ref = owlqn(objective(obj, np.float64, d0, d1), x0.astype(dtype).astype(np.float64), lam, **kw)
    return gpu, ref


@pytest.mark.parametrize("plain", [False, True], ids=["fused", "unfused"])
@pytest.mark.parametrize("obj", OBJS)
def test_solve_fp64_against_oracle(obj, plain):
    """Runs of up to 60 iterations take the oracle's iterations and evaluations; F to 1e-10, x to 1e-8, the same zero pattern."""
    n = 1001 if obj != lb.OBJ_ROSENBROCK_PAIRED else 1000
    lam = {lb.OBJ_QUAD_SHIFT: 40.0, lb.OBJ_ROSENBROCK_PAIRED: 0.5, lb.OBJ_ROSENBROCK_CHAINED: 0.5, lb.OBJ_QUAD_TRIDIAG: 0.8}[obj]
    gpu, ref = solve_pair(obj, n, lam, np.float64, plain, m=6, max_iterations=60)
    assert gpu["status"] == "ok", gpu["msg"]
    assert (gpu["niter"], gpu["nfev"]) == (ref["niter"], ref["nfev"])
    assert abs(gpu["fx"] - ref["fx"]) <= 1e-10 * max(abs(ref["fx"]), 1.0)
    assert np.max(np.abs(gpu["x"] - ref["x"])) <= 1e-8 * max(np.max(np.abs(ref["x"])), 1.0)
    assert np.array_equal(gpu["x"] == 0, ref["x"] == 0)
    assert 0 < np.count_nonzero(gpu["x"]) < n or obj == lb.OBJ_ROSENBROCK_PAIRED


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    from test_owlqn_front_cpu import owlqn_checker
    return owlqn_checker(tmp_path_factory)


@pytest.mark.parametrize("plain", [False, True], ids=["fused", "unfused"])
@pytest.mark.parametrize("obj", OBJS)
def test_solve_fp32_against_checker(checker, obj, plain):
    """fp32 runs of 8 iterations finish and take the C++ checker's fp32 iterations and evaluations; F to 1e-5 (relative), x to 1e-3,
    and the fused and unfused routes compute the same bits.  The runs stop before the decrease of F reaches the level of fp32
    rounding: there the sufficient-decrease test is decided by the order of the sums.  On the tridiagonal quadratic the checker's
    own two summation modes (left to right, eight lanes) take different evaluations from iteration 10 on."""
    from test_owlqn_front_cpu import checker_run
    n = 501 if obj != lb.OBJ_ROSENBROCK_PAIRED else 500
    lam = 0.8
    rng = np.random.default_rng(obj * 100 + n)
    x0 = rng.uniform(-1.5, 1.5, n).astype(np.float32)
    d0, d1 = tridiag_data(n) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
    prm = lb.LBFGSParam(m=6, max_iterations=8)
    gpu = lb.OWLQNSolver(prm, lam, dtype=np.float32).minimize(obj, x0, d0, d1, plain=plain)
    ref = checker_run(checker, obj, x0, lam, prm, np.float32, d0, d1)
    assert gpu["status"] == "ok" and ref["status"] == "ok", (gpu["msg"], ref["msg"])
    assert (gpu["niter"], gpu["nfev"]) == (ref["niter"], ref["nfev"])
    assert abs(gpu["fx"] - ref["fx"]) <= 1e-5 * max(abs(ref["fx"]), 1.0)
    assert np.max(np.abs(gpu["x"] - ref["x"])) <= 1e-3 * max(np.max(np.abs(ref["x"])), 1.0)
    other = lb.OWLQNSolver(prm, lam, dtype=np.float32).minimize(obj, x0, d0, d1, plain=not plain)
    assert (other["niter"], other["nfev"], other["fx"]) == (gpu["niter"], gpu["nfev"], gpu["fx"])
    assert np.array_equal(other["x"], gpu["x"])


@pytest.mark.parametrize("dtype", DT, ids=IDS)
def test_abi_refusals(owlqn_ctx, dtype):
    """Every OWL-QN entry refuses a lambda that is not positive and finite, and the history entry a history of the other precision."""
    c = owlqn_ctx
    n = 64
    v = [c.array(np.ones(n, dtype)) for _ in range(4)]
    out = c.empty(n, dtype)
    h = lb.History(c, n, 4, dtype)
    for lam in (0.0, -1.0, float("nan"), float("inf")):
        for call in (lambda: c.owlqn_trial(lb.OBJ_QUAD_SHIFT, v[0], v[1], v[2], 0.5, lam, out, v[3]),
                     lambda: c.owlqn_project(v[0], v[1], v[2], 0.5, lam, out),
                     lambda: c.owlqn_sums(v[0], v[1], lam, out),
                     lambda: h.owlqn_update_dir(v[0], v[1], v[2], v[3], lam, out)):
            with pytest.raises(lb.LbfgsB200Error, match="lambda"):
                call()
    other = np.float32 if dtype == np.float64 else np.float64
    w = [c.array(np.ones(n, other)) for _ in range(5)]
    fn = getattr(c.lib, "lbfgs_b200_owlqn_update_dir_" + ("f64" if other == np.float64 else "f32"))
    acc, dg = C.c_int(0), (C.c_double * 1)() if other == np.float64 else (C.c_float * 1)()
    st = fn(h.h, w[0].ptr, w[1].ptr, w[2].ptr, w[3].ptr, 1e-7, 0.5, w[4].ptr, C.byref(acc), dg)
    assert st == 1 and "element" in c.lib.lbfgs_b200_last_error(c.h).decode()


def test_quad_shift_at_scale():
    """n = 1e6: the closed form max(i - lam/2, 0), with the exact zeros."""
    n, lam = 1_000_000, 2e5
    r = lb.OWLQNSolver(lb.LBFGSParam(m=6, epsilon=1e-10, epsilon_rel=0.0, max_iterations=100), lam).minimize(lb.OBJ_QUAD_SHIFT, np.zeros(n))
    assert r["status"] == "ok", r["msg"]
    i = np.arange(n)
    assert np.max(np.abs(r["x"] - np.maximum(i - lam / 2, 0))) <= 1e-6
    assert np.all(r["x"][i <= lam / 2] == 0.0)


def test_tridiag_c3_kkt():
    """The C3 data (n = 1e6, m = 20): the KKT bar at the solution, which is sparse but not empty."""
    import pyoracle as po
    n, lam = 1_000_000, 0.5
    d, b, _ = po.quad_tridiag_data(n)
    # ||pg|| <= 1e-4: the sufficient decrease the search asks for beyond that is below the rounding of F (|F| ~ 1e5) at this n
    r = lb.OWLQNSolver(lb.LBFGSParam(m=20, epsilon=1e-4, epsilon_rel=0.0, max_iterations=3000), lam).minimize(
        lb.OBJ_QUAD_TRIDIAG, np.zeros(n), d, b)
    assert r["status"] == "ok", r["msg"]
    on, off = kkt_violation(r["x"], r["grad"], lam)
    assert on <= 1e-3 and off <= 1e-3
    assert 0 < np.count_nonzero(r["x"]) < n


@pytest.mark.parametrize("plain", [False, True], ids=["fused", "unfused"])
def test_max_linesearch_error(plain):
    """max_linesearch = 1 ends the solve with the oracle's exception type and message."""
    n = 10
    prm = dict(max_linesearch=1)
    with pytest.raises(RuntimeError) as e:
        owlqn(objective(lb.OBJ_ROSENBROCK_PAIRED), np.full(n, -1.2), 0.1, **prm)
    r = lb.OWLQNSolver(lb.LBFGSParam(**prm), 0.1).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.full(n, -1.2), plain=plain)
    assert r["status"] == "runtime_error" and r["msg"] == str(e.value)
