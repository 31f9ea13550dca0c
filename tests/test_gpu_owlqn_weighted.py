"""Weighted OWL-QN on the H100 (F = f + lam sum_i w_i |x_i|): the weighted kernels against numpy (element-wise outputs bit for bit,
sums to the tolerances of test_gpu_owlqn), the direction on histories of 0 to m pairs, w = 1 against the unweighted solver bit for
bit, mixed weights against the float64 statement (fp64) and the C++ checker (fp32), the closed form and the weighted KKT conditions at
n = 1e6, and the refusals at the C ABI."""

import numpy as np
import pytest

import lbfgspp_b200 as lb
from test_owlqn_cpu import objective, tridiag_data, two_loop
from test_owlqn_weighted_cpu import constrain_w, owlqn_w, point_w, pseudo_grad_w, weighted_kkt_violation

pytestmark = pytest.mark.gpu
DT = [np.float64, np.float32]
IDS = ["f64", "f32"]
OBJS = [lb.OBJ_QUAD_SHIFT, lb.OBJ_ROSENBROCK_PAIRED, lb.OBJ_ROSENBROCK_CHAINED, lb.OBJ_QUAD_TRIDIAG]


@pytest.fixture(scope="module")
def owlqn_ctx():
    ctx = lb.Context(0)
    yield ctx
    ctx.close()


def crossing_weights(xp, d, step, rng):
    """mixed weights, 0 at every coordinate whose trial xp + step d crosses zero (those must not be clamped) and at the ends"""
    n = xp.size
    w = rng.choice(np.array([0.0, 0.5, 1.0, 3.0]), n).astype(xp.dtype)
    z = xp + step * d
    w[(np.sign(z) != np.sign(xp)) & (rng.random(n) < 0.5)] = 0
    w[[0, n - 1]] = 0
    return w


@pytest.mark.parametrize("dtype", DT, ids=IDS)
@pytest.mark.parametrize("obj", OBJS)
@pytest.mark.parametrize("n", [2, 6, 1026, 300_002, 300_003])
def test_weighted_trial_kernels(owlqn_ctx, dtype, obj, n):
    """The weighted fused trial, projection and sums: x, g and d bit for bit against numpy, the sums to 1e-12 (fp64) / 1e-5 (fp32)."""
    if obj == lb.OBJ_ROSENBROCK_PAIRED and n % 2:
        pytest.skip("paired Rosenbrock needs an even n")
    rng = np.random.default_rng(n + obj + 7)
    T = np.dtype(dtype).type
    lam, step = T(0.7), T(0.37)
    xp = rng.standard_normal(n)
    xp[rng.random(n) < 0.3] = 0.0
    xp = xp.astype(dtype)
    d, gp = rng.standard_normal(n).astype(dtype), rng.standard_normal(n).astype(dtype)
    gp[::7] = T(0.1)
    w = crossing_weights(xp, d, step, rng)
    lw = (lam * w).astype(dtype)
    d0, d1 = tridiag_data(n) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
    c = owlqn_ctx
    D0 = c.array(d0.astype(dtype)) if d0 is not None else None
    D1 = c.array(d1.astype(dtype)) if d1 is not None else None
    W = c.array(w)
    X, G = c.empty(n, dtype), c.empty(n, dtype)
    out = c.owlqn_weighted_trial(obj, c.array(xp), c.array(d), c.array(gp), step, lam, W, X, G, D0, D1)
    pgp = pseudo_grad_w(xp, gp, lw)
    x = point_w(xp, d, pgp, step, lw)
    crossed = (w == 0) & (np.sign(xp + step * d) != np.sign(xp)) & (xp + step * d != 0)
    assert np.all(x[crossed] != 0)
    f, g = objective(obj, dtype, d0, d1)(x)
    assert np.array_equal(X.get(), x) and np.array_equal(G.get(), g)
    pg = pseudo_grad_w(x, g, lw).astype(np.float64)
    x64, w64 = x.astype(np.float64), w.astype(np.float64)
    want = [f, w64 @ np.abs(x64), pgp.astype(np.float64) @ (x64 - xp), pg @ pg, x64 @ x64]
    tol = 1e-12 if dtype == np.float64 else 1e-5
    scale = [abs(f), want[1], np.abs(pgp) @ np.abs(x64 - xp), want[3], want[4]]
    for k in range(5):
        assert abs(out[k] - want[k]) <= tol * max(scale[k], 1.0), (k, out[k], want[k])
    X2 = c.empty(n, dtype)
    p = c.owlqn_weighted_project(c.array(xp), c.array(d), c.array(gp), step, lam, W, X2)
    assert np.array_equal(X2.get(), x)
    assert abs(p[0] - want[1]) <= tol * max(want[1], 1.0) and abs(p[1] - want[2]) <= tol * max(scale[2], 1.0)
    Dd = c.empty(n, dtype)
    s = c.owlqn_weighted_sums(X2, c.array(g), lam, W, Dd)
    assert np.array_equal(Dd.get(), -pseudo_grad_w(x, g, lw))
    for k, v in zip(range(3), [want[1], want[3], want[4]]):
        assert abs(s[k] - v) <= tol * max(v, 1.0)
    # w = 1: the unweighted kernel's bits
    ones = c.array(np.ones(n, dtype))
    X3, G3, X4, G4 = (c.empty(n, dtype) for _ in range(4))
    o3 = c.owlqn_weighted_trial(obj, c.array(xp), c.array(d), c.array(gp), step, lam, ones, X3, G3, D0, D1)
    o4 = c.owlqn_trial(obj, c.array(xp), c.array(d), c.array(gp), step, lam, X4, G4, D0, D1)
    assert o3 == o4 and np.array_equal(X3.get(), X4.get()) and np.array_equal(G3.get(), G4.get())


@pytest.mark.parametrize("dtype", DT, ids=IDS)
@pytest.mark.parametrize("m", [3, 10])
def test_weighted_update_dir(owlqn_ctx, dtype, m):
    """Weighted pair-forming dots and constrained combination on histories of c = 0..m pairs with refused pairs (the pg column):
    d against the two-loop recursion on the weighted pg, unconstrained where lam_i == 0; dg = pg.d.  Tiles of 2048 elements: the
    zero weights fall on tile edges too."""
    c = owlqn_ctx
    n = 3 * 2048 + 5 + m
    rng = np.random.default_rng(m + 50)
    T = np.dtype(dtype).type
    lam = T(0.3)
    w = rng.choice(np.array([0.0, 0.5, 1.0, 2.0]), n).astype(dtype)
    w[[0, 2047, 2048, 4095, 4096, n - 1]] = 0
    lw = (lam * w).astype(dtype)
    W = c.array(w)
    h = lb.History(c, n, m, dtype)
    S, Y = [], []
    x = rng.standard_normal(n).astype(dtype)
    x[rng.random(n) < 0.3] = 0
    g = rng.standard_normal(n).astype(dtype)
    tol = 1e-10 if dtype == np.float64 else 1e-4
    for it in range(m + 2):
        xn = (x + T(0.1) * rng.standard_normal(n).astype(dtype)).astype(dtype)
        xn[rng.random(n) < 0.2] = 0
        curv = T(-2) if it in (0, 1, m // 2 + 1) else T(2)
        gn = (g + (xn - x) * curv + T(0.01) * rng.standard_normal(n).astype(dtype)).astype(dtype)
        Dd = c.empty(n, dtype)
        acc, dg = h.owlqn_weighted_update_dir(c.array(xn), c.array(x), c.array(gn), c.array(g), lam, W, Dd)
        s, y = (xn - x).astype(np.float64), (gn - g).astype(np.float64)
        assert acc == (curv > 0)
        if acc:
            S.append(s)
            Y.append(y)
            S, Y = S[-m:], Y[-m:]
        theta = (Y[-1] @ Y[-1]) / (S[-1] @ Y[-1]) if S else 1.0
        pg = pseudo_grad_w(xn, gn, lw).astype(np.float64)
        raw = two_loop(S, Y, pg, theta) if S else -pg / theta
        want = constrain_w(raw, pg, lw)
        got = Dd.get().astype(np.float64)
        assert np.max(np.abs(got - want)) <= tol * np.max(np.abs(raw))
        clear = np.abs(raw * pg) > 1e-6 * np.max(np.abs(raw * pg))
        assert np.array_equal(got[clear] == 0, want[clear] == 0)
        assert np.all(got[(w == 0) & clear] != 0)
        assert abs(dg - pg @ got) <= tol * max(abs(dg), 1.0)
        x, g = xn, gn


@pytest.mark.parametrize("dtype", DT, ids=IDS)
@pytest.mark.parametrize("plain", [False, True], ids=["fused", "unfused"])
@pytest.mark.parametrize("obj", OBJS)
def test_unit_weights_bit_identical(obj, plain, dtype):
    """w = 1: iterations, evaluations, F, x and grad f of OWLQNSolver(param, lam), bit for bit."""
    n = 4099 if obj != lb.OBJ_ROSENBROCK_PAIRED else 4100
    rng = np.random.default_rng(obj + 3)
    x0 = rng.uniform(-1.5, 1.5, n).astype(dtype)
    d0, d1 = tridiag_data(n) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
    prm = lb.LBFGSParam(m=6, max_iterations=40)
    a = lb.OWLQNSolver(prm, 0.8, weights=np.ones(n), dtype=dtype).minimize(obj, x0, d0, d1, plain=plain)
    b = lb.OWLQNSolver(prm, 0.8, dtype=dtype).minimize(obj, x0, d0, d1, plain=plain)
    assert a["status"] == b["status"] == "ok", (a["msg"], b["msg"])
    assert (a["niter"], a["nfev"], a["fx"], a["gnorm"]) == (b["niter"], b["nfev"], b["fx"], b["gnorm"])
    assert np.array_equal(a["x"], b["x"]) and np.array_equal(a["grad"], b["grad"])


def mixed(n, seed):
    rng = np.random.default_rng(seed)
    w = rng.choice(np.array([0.0, 0.5, 1.0, 3.0]), n)
    w[[0, 3, 4, n - 1]] = 0
    return w


@pytest.mark.parametrize("plain", [False, True], ids=["fused", "unfused"])
@pytest.mark.parametrize("obj", OBJS)
def test_mixed_weights_fp64_against_statement(obj, plain):
    """fp64, mixed weights: the float64 statement's iterations and evaluations; F to 1e-10, x to 1e-8, the same zero pattern."""
    n = 1001 if obj != lb.OBJ_ROSENBROCK_PAIRED else 1000
    lam = {lb.OBJ_QUAD_SHIFT: 40.0, lb.OBJ_ROSENBROCK_PAIRED: 0.5, lb.OBJ_ROSENBROCK_CHAINED: 0.5, lb.OBJ_QUAD_TRIDIAG: 0.8}[obj]
    rng = np.random.default_rng(obj * 100 + n)
    x0 = rng.uniform(-1.5, 1.5, n)
    w = mixed(n, obj)
    d0, d1 = tridiag_data(n) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
    kw = dict(m=6, max_iterations=60)
    gpu = lb.OWLQNSolver(lb.LBFGSParam(**kw), lam, weights=w).minimize(obj, x0, d0, d1, plain=plain)
    ref = owlqn_w(objective(obj, np.float64, d0, d1), x0, lam, w, **kw)
    assert gpu["status"] == "ok", gpu["msg"]
    assert (gpu["niter"], gpu["nfev"]) == (ref["niter"], ref["nfev"])
    assert abs(gpu["fx"] - ref["fx"]) <= 1e-10 * max(abs(ref["fx"]), 1.0)
    assert np.max(np.abs(gpu["x"] - ref["x"])) <= 1e-8 * max(np.max(np.abs(ref["x"])), 1.0)
    assert np.array_equal(gpu["x"] == 0, ref["x"] == 0)


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    from test_owlqn_weighted_front_cpu import weighted_checker
    return weighted_checker(tmp_path_factory)


@pytest.mark.parametrize("plain", [False, True], ids=["fused", "unfused"])
@pytest.mark.parametrize("obj", OBJS)
def test_mixed_weights_fp32_against_checker(checker, obj, plain):
    """fp32, mixed weights, 8 iterations: the C++ checker's fp32 iterations and evaluations; F to 1e-5, x to 1e-3."""
    from test_owlqn_weighted_front_cpu import checker_run_w
    n = 501 if obj != lb.OBJ_ROSENBROCK_PAIRED else 500
    rng = np.random.default_rng(obj * 100 + n)
    x0 = rng.uniform(-1.5, 1.5, n).astype(np.float32)
    w = mixed(n, obj)
    d0, d1 = tridiag_data(n) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
    prm = lb.LBFGSParam(m=6, max_iterations=8)
    gpu = lb.OWLQNSolver(prm, 0.8, weights=w, dtype=np.float32).minimize(obj, x0, d0, d1, plain=plain)
    ref = checker_run_w(checker, obj, x0, 0.8, w, prm, np.float32, d0, d1)
    assert gpu["status"] == "ok" and ref["status"] == "ok", (gpu["msg"], ref["msg"])
    assert (gpu["niter"], gpu["nfev"]) == (ref["niter"], ref["nfev"])
    assert abs(gpu["fx"] - ref["fx"]) <= 1e-5 * max(abs(ref["fx"]), 1.0)
    assert np.max(np.abs(gpu["x"] - ref["x"])) <= 1e-3 * max(np.max(np.abs(ref["x"])), 1.0)


def test_quad_shift_closed_form_at_scale():
    """n = 1e6, mixed weights: x_i = max(i - lam_i / 2, 0), exact zeros where i <= lam_i / 2, and i itself where w_i = 0."""
    n, lam = 1_000_000, 2e5
    w = np.array([0.0, 0.5, 1.0, 3.0])[np.arange(n) % 4]
    r = lb.OWLQNSolver(lb.LBFGSParam(m=6, epsilon=1e-10, epsilon_rel=0.0, max_iterations=100), lam, weights=w).minimize(
        lb.OBJ_QUAD_SHIFT, np.zeros(n))
    assert r["status"] == "ok", r["msg"]
    i = np.arange(n)
    want = np.maximum(i - lam * w / 2, 0)
    assert np.max(np.abs(r["x"] - want)) <= 1e-6
    assert np.array_equal(r["x"] == 0, want == 0)


def test_tridiag_c3_weighted_kkt():
    """The C3 data (n = 1e6, m = 20) with an unpenalised block and mixed weights: the weighted KKT conditions at the solution."""
    import pyoracle as po
    n, lam = 1_000_000, 0.5
    d, b, _ = po.quad_tridiag_data(n)
    w = np.array([0.5, 1.0, 2.0])[np.arange(n) % 3]
    w[:1000] = 0.0
    # ||pg|| <= 1e-3 bounds every violation below; under these weights a tighter bar asks for decreases below the rounding of F
    r = lb.OWLQNSolver(lb.LBFGSParam(m=20, epsilon=1e-3, epsilon_rel=0.0, max_iterations=3000), lam, weights=w).minimize(
        lb.OBJ_QUAD_TRIDIAG, np.zeros(n), d, b)
    assert r["status"] == "ok", r["msg"]
    on, off, smooth = weighted_kkt_violation(r["x"], r["grad"], lam * w)
    assert on <= 1e-3 and off <= 1e-3 and smooth <= 1e-3
    assert 0 < np.count_nonzero(r["x"]) < n


@pytest.mark.parametrize("dtype", DT, ids=IDS)
def test_weighted_abi_refusals(owlqn_ctx, dtype):
    """A NULL w, a bad lambda, a misaligned w at the direction entry, and bad weights at the sums entry (with their count)."""
    c = owlqn_ctx
    n = 64
    v = [c.array(np.ones(n, dtype)) for _ in range(4)]
    W = c.array(np.ones(n, dtype))
    out = c.empty(n, dtype)
    h = lb.History(c, n, 4, dtype)
    for call in (lambda w, lam: c.owlqn_weighted_trial(lb.OBJ_QUAD_SHIFT, v[0], v[1], v[2], 0.5, lam, w, out, v[3]),
                 lambda w, lam: c.owlqn_weighted_project(v[0], v[1], v[2], 0.5, lam, w, out),
                 lambda w, lam: c.owlqn_weighted_sums(v[0], v[1], lam, w, out),
                 lambda w, lam: h.owlqn_weighted_update_dir(v[0], v[1], v[2], v[3], lam, w, out)):
        with pytest.raises(lb.LbfgsB200Error, match="NULL weights"):
            call(None, 1.0)
        for lam in (0.0, -1.0, float("nan"), float("inf")):
            with pytest.raises(lb.LbfgsB200Error, match="lambda"):
                call(W, lam)
    odd = lb.DeviceArray(c, np.ones(n + 1, dtype), offset_elems=1)
    with pytest.raises(lb.LbfgsB200Error, match="boundary"):
        h.owlqn_weighted_update_dir(v[0], v[1], v[2], v[3], 1.0, odd, out)
    big = 1e308 if dtype == np.float64 else 1e38
    bad = np.ones(n, dtype)
    bad[[1, 5, 9, 63]] = [-1.0, np.nan, np.inf, big]
    with pytest.raises(lb.LbfgsB200Error, match="4 weights"):
        c.owlqn_weighted_sums(v[0], v[1], 10.0, c.array(bad))
