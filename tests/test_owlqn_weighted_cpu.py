"""Weighted OWL-QN (F = f + lam sum_i w_i |x_i|) without a GPU: a float64 numpy statement of the algorithm OWLQNSolver(param, lam, w)
runs (the oracle of the weighted GPU tests), checked against the QuadShift closed form, the weighted KKT conditions, the smooth
minimiser at all-zero weights, and the unweighted statement at w = 1."""
import numpy as np
import pytest

import lbfgspp_b200 as lb
from test_owlqn_cpu import EPS64, constrain, fail, objective, orthant, owlqn, project, tridiag_data, two_loop


# ---- the weighted expressions of include/LBFGSpp/OWLQNCore.h, lw = lam * w element by element (owlqn_lam_i)
def pseudo_grad_w(x, g, lw):
    lw = np.asarray(lw, dtype=x.dtype)
    right, left = g + lw, g - lw
    zero = np.where(right < 0, right, np.where(left > 0, left, 0)).astype(x.dtype)
    return np.where(x > 0, g + lw, np.where(x < 0, g - lw, zero)).astype(x.dtype)


def point_w(xp, d, pgp, step, lw):
    """owlqn_point_w: the projected trial coordinate where lam_i > 0, xp + step d where lam_i == 0"""
    z = xp + step * d
    return np.where(lw > 0, project(z, orthant(xp, pgp)), z).astype(xp.dtype)


def constrain_w(d, pg, lw):
    return np.where(lw > 0, constrain(d, pg), d).astype(d.dtype)


def weights_ok(lam, w):
    with np.errstate(over="ignore"):
        lw = lam * w
    return np.all((w >= 0) & np.isfinite(w) & np.isfinite(lw))


def owlqn_w(fg, x0, lam, w, m=6, epsilon=1e-5, epsilon_rel=1e-5, past=0, delta=0.0, max_iterations=0, max_linesearch=20, min_step=1e-20,
            max_step=1e20, ftol=1e-4):
    """Weighted OWL-QN as OWLQNSolver(param, lam, w) runs it, in float64: -> dict(niter, nfev, fx, x, grad, gnorm).  Raises the
    solver's exceptions; ValueError for a weight the solver refuses (after the first evaluation, as the solver's sums pass does)."""
    w = np.asarray(w, dtype=np.float64)
    with np.errstate(over="ignore"):      # an overflowing lambda * w is refused below
        lw = lam * w
    x = np.array(x0, dtype=np.float64)
    f, g = fg(x)
    nfev = 1
    if not weights_ok(lam, w):
        raise ValueError("a weight is negative, not finite, or makes lambda * w overflow")
    l1 = lambda v: np.sum(w * np.abs(v))
    pg = pseudo_grad_w(x, g, lw)
    F = f + lam * l1(x)
    fhist = [0.0] * past
    if past:
        fhist[0] = F
    gnorm = np.sqrt(pg @ pg)
    out = lambda k: dict(niter=k, nfev=nfev, fx=F, x=x, grad=g, gnorm=gnorm)
    if gnorm <= epsilon or gnorm <= epsilon_rel * np.sqrt(x @ x):
        return out(1)
    d, step, dg = -pg, 1.0 / gnorm, -(pg @ pg)
    S, Y, theta = [], [], 1.0
    k = 1
    while True:
        if dg > 0:
            fail("not_descent")
        xp, gp, Fp = x, g, F
        pgp = pseudo_grad_w(xp, gp, lw)
        trials = 0
        while True:
            x = point_w(xp, d, pgp, step, lw)
            f, g = fg(x)
            nfev += 1
            F = f + lam * l1(x)
            if not (F > Fp + ftol * (pgp @ (x - xp)) or F != F):
                break
            if step < min_step:
                fail("too_small")
            if step > max_step:
                fail("too_large")
            step *= 0.5
            trials += 1
            if trials >= max_linesearch:
                fail("max_trials")
        pg = pseudo_grad_w(x, g, lw)
        gnorm = np.sqrt(pg @ pg)
        if gnorm <= epsilon or gnorm <= epsilon_rel * np.sqrt(x @ x):
            return out(k)
        if past:
            fxd = fhist[k % past]
            if k >= past and abs(fxd - F) <= delta * max(abs(F), abs(fxd), 1.0):
                return out(k)
            fhist[k % past] = F
        if max_iterations and k >= max_iterations:
            return out(k)
        s, y = x - xp, g - gp
        if s @ y > EPS64 * (y @ y):
            S.append(s)
            Y.append(y)
            theta = (y @ y) / (s @ y)
            S, Y = S[-m:], Y[-m:]
        d = constrain_w(two_loop(S, Y, pg, theta) if S else -pg / theta, pg, lw)
        dg = pg @ d
        if not dg < 0:
            fail("not_descent")
        step = 1.0
        k += 1


def weighted_kkt_violation(x, g, lw):
    """-> (on, off, smooth): max |g_i + lam_i sign(x_i)| over the penalised support, max (|g_i| - lam_i) over the penalised zeros, and
    max |g_i| over the unpenalised coordinates"""
    pen = lw > 0
    nz = (x != 0) & pen
    z = (x == 0) & pen
    on = np.max(np.abs(g[nz] + lw[nz] * np.sign(x[nz])), initial=0.0)
    off = np.max(np.abs(g[z]) - lw[z], initial=-1.0)
    smooth = np.max(np.abs(g[~pen]), initial=0.0)
    return on, off, smooth


def mixed_weights(n, seed=0):
    """0, 0.5, 1, 3 and a huge weight in turn, with zeros at the first and last coordinate and at pack edges"""
    w = np.array([0.0, 0.5, 1.0, 3.0, 1e200])[np.arange(n) % 5]
    w[[0, 3, 4, n - 1]] = 0.0
    rng = np.random.default_rng(seed)
    w[rng.random(n) < 0.1] = 0.0
    return w


@pytest.mark.parametrize("lam", [0.5, 7.0])
def test_statement_quad_shift_closed_form(lam):
    """f = sum (x_i - i)^2: the minimiser is sign(c_i) max(|c_i| - lam_i/2, 0) with c_i = i, exactly 0 wherever i <= lam_i / 2, and
    exactly i where lam_i == 0 (w_i = 0 or lam * w_i underflowing)"""
    n = 60
    w = np.array([0.0, 0.5, 1.0, 3.0, 1e200])[np.arange(n) % 5]
    w[7] = 1e-320           # lam * w rounds to 0 only for lam < 1e-3; here it is subnormal but positive
    lw = lam * w
    r = owlqn_w(objective(lb.OBJ_QUAD_SHIFT), np.zeros(n), lam, w, epsilon=1e-12, epsilon_rel=0.0, max_iterations=300)
    c = np.arange(n, dtype=np.float64)
    want = np.sign(c) * np.maximum(np.abs(c) - lw / 2, 0.0)
    assert np.max(np.abs(r["x"] - want)) <= 1e-8
    assert np.array_equal(r["x"] == 0, want == 0)
    assert np.all(r["x"][w == 1e200] == 0.0)


def test_statement_underflowing_weight_is_unpenalised():
    """lam * w_i rounding to 0 leaves coordinate i smooth: it reaches c_i although w_i > 0"""
    n, lam = 20, 1e-5
    w = np.ones(n)
    w[[2, 9]] = 1e-320
    assert lam * w[2] == 0.0
    r = owlqn_w(objective(lb.OBJ_QUAD_SHIFT), np.zeros(n), lam, w, epsilon=1e-12, epsilon_rel=0.0, max_iterations=300)
    assert abs(r["x"][2] - 2.0) <= 1e-8 and abs(r["x"][9] - 9.0) <= 1e-8


def test_statement_weighted_kkt_tridiag():
    """The tridiagonal quadratic under mixed weights: g_i = -lam_i sign(x_i) on the penalised support, |g_i| <= lam_i at the penalised
    zeros, g_i ~ 0 where lam_i == 0"""
    n, lam = 400, 0.8
    d, b = tridiag_data(n)
    w = mixed_weights(n)
    w[w > 10] = 2.0
    r = owlqn_w(objective(lb.OBJ_QUAD_TRIDIAG, data0=d, data1=b), np.zeros(n), lam, w, m=10, epsilon=1e-10, epsilon_rel=0.0,
                max_iterations=3000)
    on, off, smooth = weighted_kkt_violation(r["x"], r["grad"], lam * w)
    assert on <= 1e-8 and off <= 1e-8 and smooth <= 1e-8
    pen = w > 0
    assert 0 < np.count_nonzero(r["x"][pen]) < np.count_nonzero(pen)
    assert np.all(r["x"][~pen] != 0)


def test_statement_zero_weights_reach_smooth_minimiser():
    """w = 0 everywhere: plain L-BFGS with the same search, ending at A^-1 b"""
    n, lam = 200, 0.8
    d, b = tridiag_data(n)
    A = np.diag(d + 1.0) - 0.5 * (np.eye(n, k=1) + np.eye(n, k=-1))
    r = owlqn_w(objective(lb.OBJ_QUAD_TRIDIAG, data0=d, data1=b), np.zeros(n), lam, np.zeros(n), m=10, epsilon=1e-10, epsilon_rel=0.0,
                max_iterations=2000)
    assert np.max(np.abs(r["x"] - np.linalg.solve(A, b))) <= 1e-8


@pytest.mark.parametrize("obj", [lb.OBJ_QUAD_SHIFT, lb.OBJ_ROSENBROCK_PAIRED, lb.OBJ_ROSENBROCK_CHAINED, lb.OBJ_QUAD_TRIDIAG])
def test_statement_unit_weights_are_unweighted(obj):
    """w = 1 takes the unweighted statement's path and bits"""
    n = 64
    rng = np.random.default_rng(obj)
    x0 = rng.uniform(-1.5, 1.5, n)
    d0, d1 = tridiag_data(n) if obj == lb.OBJ_QUAD_TRIDIAG else (None, None)
    fg = objective(obj, np.float64, d0, d1)
    a = owlqn_w(fg, x0, 0.5, np.ones(n), max_iterations=40)
    b = owlqn(fg, x0, 0.5, max_iterations=40)
    assert (a["niter"], a["nfev"], a["fx"]) == (b["niter"], b["nfev"], b["fx"])
    assert np.array_equal(a["x"], b["x"]) and np.array_equal(a["grad"], b["grad"])


@pytest.mark.parametrize("bad", [-1.0, np.nan, np.inf, 1e308])
def test_statement_refuses_bad_weights(bad):
    """A negative, NaN or infinite weight, or one with lam * w overflowing (lam = 10, w = 1e308), is refused after one evaluation"""
    w = np.ones(8)
    w[3] = bad
    with pytest.raises(ValueError):
        owlqn_w(objective(lb.OBJ_QUAD_SHIFT), np.zeros(8), 10.0, w)


def test_python_front_refuses_wrong_size():
    """The Python front refuses weights of another length before it reaches the driver."""
    with pytest.raises(ValueError, match="one entry per coordinate"):
        lb.OWLQNSolver(lb.LBFGSParam(), 1.0, weights=np.ones(7)).minimize(lb.OBJ_QUAD_SHIFT, np.zeros(8))
