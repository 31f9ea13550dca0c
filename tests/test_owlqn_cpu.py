"""OWL-QN (F = f + lam |x|_1) without a GPU: a float64 numpy statement of the algorithm OWLQNSolver runs (the oracle of the GPU tests),
checked against closed forms and the KKT conditions, and the solver's refusals of a bad lambda."""
import numpy as np
import pytest

import lbfgspp_b200 as lb

EPS64 = np.finfo(np.float64).eps
MESSAGES = {
    "not_descent": (ArithmeticError, "the moving direction increases the objective function value"),
    "too_small": (RuntimeError, "the line search step became smaller than the minimum value allowed"),
    "too_large": (RuntimeError, "the line search step became larger than the maximum value allowed"),
    "max_trials": (RuntimeError, "the line search routine reached the maximum number of iterations"),
}


def fail(kind):
    exc, msg = MESSAGES[kind]
    raise exc(msg)


# ---- the built-in objectives (csrc/objectives.cuh), element by element in the kernels' order
def objective(kind, dtype=np.float64, data0=None, data1=None):
    T = np.dtype(dtype).type

    def quad_shift(x):
        r = x - np.arange(x.size).astype(dtype)
        return T(np.sum(r * r)), T(2) * r

    def rosen_paired(x):
        x0, x1 = x[0::2], x[1::2]
        t1 = T(1) - x0
        t2 = T(10) * (x1 - x0 * x0)
        g = np.empty_like(x)
        g[1::2] = T(20) * t2
        g[0::2] = T(-2) * (x0 * g[1::2] + t1)
        return T(np.sum(t1 * t1 + t2 * t2)), g

    def rosen_chained(x):
        n = x.size
        xm = np.concatenate([[T(0)], x[:-1]]).astype(dtype)
        xn = np.concatenate([x[1:], [T(0)]]).astype(dtype)
        u = x - xm * xm
        f = T(4) * u * u
        g = T(8) * u + T(16) * (x * x - xn) * x
        g[n - 1] = T(8) * u[n - 1]
        f[0] = (x[0] - T(1)) * (x[0] - T(1))
        g[0] = T(2) * (x[0] - T(1)) + T(16) * (x[0] * x[0] - xn[0]) * x[0]
        return T(np.sum(f)), g

    def quad_tridiag(x):
        d, b = data0.astype(dtype), data1.astype(dtype)
        xm = np.concatenate([[T(0)], x[:-1]]).astype(dtype)
        xn = np.concatenate([x[1:], [T(0)]]).astype(dtype)
        ax = (d + T(1)) * x - T(0.5) * (xm + xn)
        return T(np.sum(x * (T(0.5) * ax - b))), ax - b

    return {lb.OBJ_QUAD_SHIFT: quad_shift, lb.OBJ_ROSENBROCK_PAIRED: rosen_paired, lb.OBJ_ROSENBROCK_CHAINED: rosen_chained,
            lb.OBJ_QUAD_TRIDIAG: quad_tridiag}[kind]


# ---- the expressions of include/LBFGSpp/OWLQNCore.h
def pseudo_grad(x, g, lam):
    lam = x.dtype.type(lam)
    right, left = g + lam, g - lam
    zero = np.where(right < 0, right, np.where(left > 0, left, 0)).astype(x.dtype)
    return np.where(x > 0, g + lam, np.where(x < 0, g - lam, zero)).astype(x.dtype)


def orthant(xp, pgp):
    return np.where(xp != 0, np.sign(xp), np.sign(-pgp))


def project(z, xi):
    return np.where(np.sign(z) == xi, z, 0).astype(z.dtype)


def constrain(d, pg):
    return np.where(d * pg >= 0, 0, d).astype(d.dtype)


def two_loop(S, Y, v, theta):
    """-H v by the two-loop recursion over the kept pairs (oldest first in S, Y)"""
    q = -v.astype(np.float64)
    alpha = []
    for s, y in reversed(list(zip(S, Y))):
        a = s @ q / (s @ y)
        alpha.append(a)
        q = q - a * y
    r = q / theta
    for (s, y), a in zip(zip(S, Y), reversed(alpha)):
        b = y @ r / (s @ y)
        r = r + (a - b) * s
    return r


def owlqn(fg, x0, lam, m=6, epsilon=1e-5, epsilon_rel=1e-5, past=0, delta=0.0, max_iterations=0, max_linesearch=20, min_step=1e-20,
          max_step=1e20, ftol=1e-4):
    """OWL-QN as OWLQNSolver runs it, in float64: -> dict(niter, nfev, fx, x, grad, gnorm).  Raises the solver's exceptions."""
    x = np.array(x0, dtype=np.float64)
    f, g = fg(x)
    nfev = 1
    pg = pseudo_grad(x, g, lam)
    F = f + lam * np.sum(np.abs(x))
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
        pgp = pseudo_grad(xp, gp, lam)
        xi = orthant(xp, pgp)
        trials = 0
        while True:
            x = project(xp + step * d, xi)
            f, g = fg(x)
            nfev += 1
            F = f + lam * np.sum(np.abs(x))
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
        pg = pseudo_grad(x, g, lam)
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
        d = constrain(two_loop(S, Y, pg, theta) if S else -pg / theta, pg)
        dg = pg @ d
        if not dg < 0:
            fail("not_descent")
        step = 1.0
        k += 1


def tridiag_data(n, seed=0):
    rng = np.random.default_rng(seed)
    return rng.uniform(0.5, 2.0, n), rng.standard_normal(n)


def kkt_violation(x, g, lam):
    """max over the nonzeros of |g_i + lam sign(x_i)| / lam, and over the zeros of (|g_i| - lam) / lam (<= 0 when satisfied)"""
    nz = x != 0
    a = np.max(np.abs(g[nz] + lam * np.sign(x[nz])), initial=0.0) / lam
    b = np.max(np.abs(g[~nz]) - lam, initial=-lam) / lam
    return a, b


@pytest.mark.parametrize("lam", [0.5, 7.0, 1e3])
def test_oracle_quad_shift_closed_form(lam):
    """f = sum (x_i - i)^2: the minimiser is max(i - lam/2, 0), exactly 0 wherever i <= lam/2."""
    n = 50
    r = owlqn(objective(lb.OBJ_QUAD_SHIFT), np.zeros(n), lam, epsilon=1e-12, epsilon_rel=0.0, max_iterations=200)
    want = np.maximum(np.arange(n) - lam / 2, 0.0)
    assert np.max(np.abs(r["x"] - want)) <= 1e-8
    assert np.all(r["x"][np.arange(n) <= lam / 2] == 0.0)


def test_oracle_kkt_tridiag():
    """The tridiagonal quadratic: |g_i + lam sign(x_i)| small on the nonzeros, |g_i| <= lam (1 + tol) on the zeros."""
    n, lam = 400, 0.8
    d, b = tridiag_data(n)
    r = owlqn(objective(lb.OBJ_QUAD_TRIDIAG, data0=d, data1=b), np.zeros(n), lam, m=10, epsilon=1e-10, epsilon_rel=0.0,
              max_iterations=2000)
    nz = int(np.count_nonzero(r["x"]))
    assert 0 < nz < n
    on, off = kkt_violation(r["x"], r["grad"], lam)
    assert on <= 1e-8 and off <= 1e-8


def test_oracle_raises_max_trials():
    """max_linesearch = 1: the first refused trial ends the solve with the backtracking search's exception."""
    with pytest.raises(RuntimeError, match="maximum number of iterations"):
        owlqn(objective(lb.OBJ_ROSENBROCK_PAIRED), np.full(10, -1.2), 0.1, max_linesearch=1)


@pytest.mark.parametrize("lam", [0.0, -1.0, float("nan"), float("inf")])
def test_solver_refuses_lambda(lam):
    """OWLQNSolver refuses a lambda that is not positive and finite before it touches a device."""
    r = lb.OWLQNSolver(lb.LBFGSParam(), lam).minimize(lb.OBJ_QUAD_SHIFT, np.zeros(8))
    assert r["status"] == "invalid_argument" and "lambda" in r["msg"]
