"""The device-resident solve of the neighbour-coupled objectives (chained Rosenbrock, tridiagonal quadratic).

Their passes are separate code from the element-wise objectives': the trials store their points and gradients and a search keeps its
best trial by swapping it into (x_lo, g_lo), a search that never improved on its start point restores it (RESTORE), the trial pass
stages tiles of 2016 elements with a 16-byte margin on either side, and the combination pass forms x1 of the element on either side of
a tile in two spare warps and hands a tile's last x1 to the next tile of the same CTA.  The dots pass forms their new pair from the
staged g, x, gp, xp (DOTS_FORM) or reads the staged g as it is (DOTS_PLAIN).  The runs here cross tiles and CTAs, in fp64 and fp32
(whose 16-byte units hold 4 elements instead of 2), at odd n (a ragged last unit), with short histories (the longest block) and with
histories past 24 pairs (the columns of the dots taken in two rounds).

The sharpest check: the library is built without FMA contraction, so a gradient the solve returns must equal the objective's gradient
expression (evaluated in the solve's dtype, one operation at a time as objectives.cuh does) at the returned x, bit for bit.  A wrong
neighbour at a tile edge, or another summation order in the margin warps, changes only the last bits of g at a few elements, which
the CPU checker's bars on fx and x do not see."""
import ctypes as C

import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po
from test_gpu_resident_implied_grad import quad_shift_grad, resident
from test_gpu_solver import check_parity, cpu_param
from util import LS

pytestmark = pytest.mark.gpu

CHAINED, TRIDIAG = lb.OBJ_ROSENBROCK_CHAINED, lb.OBJ_QUAD_TRIDIAG
DTYPES = [np.float64, np.float32]
N = 262147                 # odd, n mod 4 = 3: a ragged last unit in both dtypes
STAGE_BYTES = 196608       # the persistent kernel's staging ring (kPStageBytes, persist.cuh)


def neighbours(x):
    z = np.zeros(1, dtype=x.dtype)
    return np.concatenate((z, x[:-1])), np.concatenate((x[1:], z))


def chained_grad(x):
    """grad f of the chained Rosenbrock function, expression by expression as the kernels evaluate it (in x's dtype)."""
    T = x.dtype.type
    xm, xn = neighbours(x)
    u = x - xm * xm
    g = T(8) * u + T(16) * (x * x - xn) * x
    g[-1] = T(8) * u[-1]
    g[0] = T(2) * (x[0] - T(1)) + T(16) * (x[0] * x[0] - xn[0]) * x[0]
    return g


def tridiag_grad(x, d, b):
    """grad f of the tridiagonal quadratic (data0 = d, data1 = b), expression by expression as the kernels evaluate it."""
    T = x.dtype.type
    xm, xn = neighbours(x)
    return ((d + T(1)) * x - T(0.5) * (xm + xn)) - b


def problem(objective, n, dtype, seed=5, kappa=1e3):
    """(x0, d, b) in dtype: chained Rosenbrock from 1.3, the tridiagonal quadratic from 0."""
    if objective == CHAINED:
        return np.full(n, 1.3, dtype), None, None
    d, b, _ = po.quad_tridiag_data(n, kappa=kappa, seed=seed)
    return np.zeros(n, dtype), d.astype(dtype), b.astype(dtype)


def grad_of(objective, x, d, b):
    return chained_grad(x) if objective == CHAINED else tridiag_grad(x, d, b)


def block_length(m, itemsize):
    """solver_create's rule: the largest power of two <= 1024 for which two stages of 2m+4 rows fit the staging ring."""
    bt = 1024
    while bt > 32 and 2 * (2 * m + 4) * bt * itemsize > STAGE_BYTES:
        bt >>= 1
    return bt


def sm_count(ctx):
    """The device's SM count as the library reads it: the persistent kernel runs one CTA per SM."""
    return ctx.lib.lbfgs_b200_sm_count(ctx.h)


def owner(i, n, bt, sms):
    """(CTA, tile of that CTA, offset in the tile) of element i, as the persistent kernel splits n (Own, persist.cuh)."""
    units = -(-n // bt)
    K = min(units, sms)
    u = i // bt
    cta = next(c for c in range(K) if u < (units * (c + 1)) // K)
    return cta, u - (units * cta) // K, i % bt


def orders(orc, objective, x0, d, b, ls, prm, dtype):
    """The checker's run in its two summation orders: (lanes-of-8 run, sequential run)."""
    kw = dict(data0=d, data1=b, dtype=dtype)
    return (orc.lbfgs(objective, x0, LS[ls], cpu_param(orc, prm), sum_mode=po.SUM_LANES8, **kw),
            orc.lbfgs(objective, x0, LS[ls], cpu_param(orc, prm), sum_mode=po.SUM_SEQUENTIAL, **kw))


def spread_bar(a, b, key="x"):
    """32 times the checker's own spread between its two summation orders (at least 32 rounding units of the value)."""
    va, vb = np.asarray(a[key], dtype=np.float64), np.asarray(b[key], dtype=np.float64)
    eps = np.finfo(np.asarray(a[key]).dtype).eps
    return 32 * max(float(np.max(np.abs(va - vb))), eps * max(1.0, float(np.max(np.abs(va)))))


def across_ctas(ctx, m, dtype, r):
    """(n, BT, SMs, blocks per CTA) for n = 3 SMs BT + r: every CTA owns at least three blocks of the history."""
    bt = block_length(m, np.dtype(dtype).itemsize)
    sms = sm_count(ctx)
    n = 3 * sms * bt + r
    units = -(-n // bt)
    K = min(units, sms)
    tiles = [(units * (c + 1)) // K - (units * c) // K for c in range(K)]
    assert min(tiles) >= 3, tiles
    return n, bt, sms, tiles


def held_to_checker(ctx, orc, objective, x0, d, b, prm, ls, dtype, bt, sms):
    """A capped run: the front returns the C ABI's x and gradient, the gradient is grad f(x) bit for bit, the checker's two summation
    orders agree on the counts and the GPU matches them, x lies within spread_bar of the checker, and the run meets check_parity
    (fp64) or the host-driven loop takes the same counts (fp32).  Returns the rounds by pass."""
    n = x0.size
    outs, X, G, by_op = resident(ctx, objective, x0, prm, ls, data0=d, data1=b)
    g = lb.LBFGSSolver(prm, ls, dtype=dtype, resident=True).minimize(objective, x0, data0=d, data1=b)
    assert np.array_equal(np.asarray(g["x"], dtype=dtype), X[0]) and np.array_equal(np.asarray(g["grad"], dtype=dtype), G[0])
    gref = grad_of(objective, X[0], d, b)
    bad = np.flatnonzero(G[0] != gref)
    assert bad.size == 0, ("gradient differs from grad f(x) at %d elements, first %d (CTA, tile, offset) = %s"
                           % (bad.size, bad[0], owner(int(bad[0]), n, bt, sms)))
    c, c2 = orders(orc, objective, x0, d, b, ls, prm, dtype)
    assert c["status"] == "ok" and (c["niter"], c["nfev"]) == (c2["niter"], c2["nfev"])
    assert (outs[0].status, outs[0].niter, outs[0].nfev) == (0, c["niter"], c["nfev"])
    bar = spread_bar(c, c2)
    err = np.abs(X[0].astype(np.float64) - c["x"])
    worst = int(np.argmax(err))
    assert err[worst] <= bar, ("x off by %.3g > %.3g at %d (CTA, tile, offset) = %s" % (err[worst], bar, worst, owner(worst, n, bt, sms)))
    if dtype == np.float64:
        check_parity(g, c, xtol=bar / max(1.0, np.max(np.abs(c["x"]))))
    else:
        # the host-driven loop: a second driver of the same arithmetic
        h = lb.LBFGSSolver(prm, ls, dtype=dtype, resident=False).minimize(objective, x0, data0=d, data1=b)
        assert (h["status"], h["niter"], h["nfev"]) == ("ok", g["niter"], g["nfev"])
        assert abs(h["fx"] - g["fx"]) <= spread_bar(c, c2, "fx")
    return by_op


def batch_matches_lone_solves(ctx, objective, X0, d, b, prm, ls):
    """The rows of X0 solved in one launch (shared data d, b): every member bit for bit its lone solve."""
    outs, X, G, _ = resident(ctx, objective, X0, prm, ls, data0=d, data1=b)
    for k in range(len(X0)):
        lone, Xl, Gl, _ = resident(ctx, objective, X0[k], prm, ls, data0=d, data1=b)
        assert (outs[k].status, outs[k].niter, outs[k].nfev, outs[k].fx) == (lone[0].status, lone[0].niter, lone[0].nfev, lone[0].fx)
        assert np.array_equal(X[k], Xl[0]) and np.array_equal(G[k], Gl[0])


GEOMETRY = [(obj, dt, m) for obj in (CHAINED, TRIDIAG) for dt in DTYPES for m in (3, 10, 12)]


@pytest.mark.parametrize("objective,dtype,m", GEOMETRY,
                         ids=["%s-%s-m%d" % ("chained" if o == CHAINED else "tridiag", np.dtype(d).name, m) for o, d, m in GEOMETRY])
def test_tiles_and_ctas(gpu_ctx, orc, objective, dtype, m):
    """n = 3 SMs BT + r, r odd: every CTA owns at least three blocks of the history, every tile boundary of the combination pass
    and every 2016-element tile of the trial pass lies inside the vector.  m = 3 gives the longest block (fp64: 512 units per tile,
    one per thread), m = 12 a column for every warp of the pair-forming dots."""
    n, bt, sms, tiles = across_ctas(gpu_ctx, m, dtype, {3: 7, 10: 21, 12: 27}[m])
    x0, d, b = problem(objective, n, dtype)
    caps = (6,) if dtype == np.float64 else (1, 2, 3)
    for cap in caps:
        prm = lb.LBFGSParam(m=m, max_iterations=cap)
        by_op = held_to_checker(gpu_ctx, orc, objective, x0, d, b, prm, "MoreThuente", dtype, bt, sms)
        # the margin code ran: trials on staged tiles, the combination pass with its fused first trial, the pair-forming dots
        assert by_op.get("trial", 0) > 0 and (cap == 1 or (by_op.get("combine_trial", 0) > 0 and by_op.get("dots_form", 0) > 0)), by_op
        print("\n%s %s m=%d BT=%d n%%4=%d tiles/CTA=%d..%d cap=%d rounds=%s"
              % ("chained" if objective == CHAINED else "tridiag", np.dtype(dtype).name, m, bt, n % 4, min(tiles), max(tiles), cap, by_op))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_two_rounds_of_columns(gpu_ctx, orc, dtype):
    """m = 30 and a run past 25 accepted pairs: the pair-forming dots reach c = 10 (the new pair formed by the warps without a
    column), c = 12 (by the warps of column 0) and c > 24 (the columns taken in two rounds)."""
    m = 30
    n, bt, sms, _ = across_ctas(gpu_ctx, m, dtype, 13)
    # (seed 1: this far into a run the checker's spread between its two orders is a loose measure of where a third order lands;
    # at seed 5 the GPU's x lies at 2x the bar in fp64, at other seeds well inside it)
    x0, d, b = problem(TRIDIAG, n, dtype, seed=1)
    prm = lb.LBFGSParam(m=m, max_iterations=28)
    by_op = held_to_checker(gpu_ctx, orc, TRIDIAG, x0, d, b, prm, "MoreThuente", dtype, bt, sms)
    assert by_op.get("dots_form", 0) >= 26, by_op
    X0 = np.stack([x0, np.random.default_rng(11).uniform(-1, 1, n), np.full(n, 0.5)]).astype(dtype)
    batch_matches_lone_solves(gpu_ctx, TRIDIAG, X0, d, b, prm, "MoreThuente")


def indefinite_tridiag(n, dtype, seed=5):
    """(d, b) of a tridiagonal quadratic with d = -3 at 1 % of the elements: A is indefinite, and once the search directions pick up
    its negative curvature, backtracking to the Armijo condition accepts pairs with s'y < 0, which the curvature gate rejects."""
    d, b, _ = po.quad_tridiag_data(n, kappa=10.0, seed=seed)
    d[np.random.default_rng(seed).random(n) < 0.01] = -3.0
    return d.astype(dtype), b.astype(dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_plain_dots(gpu_ctx, orc, dtype):
    """The dots without a new pair (DOTS_PLAIN, after the curvature gate rejects a pair) of a neighbour-coupled objective: g is
    staged as it is, and every column, age 0 included, comes from the history."""
    m = 10
    n, bt, sms, _ = across_ctas(gpu_ctx, m, dtype, 21)
    d, b = indefinite_tridiag(n, dtype)
    x0 = np.zeros(n, dtype)
    prm = lb.LBFGSParam(m=m, linesearch=lb.LBFGS_LINESEARCH_BACKTRACKING_ARMIJO, max_iterations=8)
    by_op = held_to_checker(gpu_ctx, orc, TRIDIAG, x0, d, b, prm, "Backtracking", dtype, bt, sms)
    assert by_op.get("dots_plain", 0) > 0, by_op
    X0 = np.stack([x0, np.random.default_rng(12).uniform(-1, 1, n), np.full(n, 0.5)]).astype(dtype)
    batch_matches_lone_solves(gpu_ctx, TRIDIAG, X0, d, b, prm, "Backtracking")


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("objective", [CHAINED, TRIDIAG], ids=["chained", "tridiag"])
def test_converged(gpu_ctx, orc, objective, dtype):
    """Whole runs: chained Rosenbrock converges in 29 iterations, the tridiagonal quadratic at kappa = 10 in 21 (checker, fp64)."""
    x0, d, b = problem(objective, N, dtype, kappa=10.0)
    # (in fp32 the tridiagonal quadratic's gradient does not fall below the default epsilon: that run stops at the cap)
    prm = lb.LBFGSParam(m=6, max_iterations=200)
    outs, X, G, _ = resident(gpu_ctx, objective, x0, prm, "MoreThuente", data0=d, data1=b)
    assert outs[0].status == 0 and np.array_equal(G[0], grad_of(objective, X[0], d, b))
    g = lb.LBFGSSolver(prm, "MoreThuente", dtype=dtype, resident=True).minimize(objective, x0, data0=d, data1=b)
    assert np.array_equal(np.asarray(g["x"], dtype=dtype), X[0])
    c = orc.lbfgs(objective, x0, LS["MoreThuente"], cpu_param(orc, prm), data0=d, data1=b, dtype=dtype,
                  **({"sum_mode": po.SUM_LANES8} if dtype == np.float64 else {}))
    if dtype == np.float64:
        check_parity(g, c, xtol=1e-7)
    else:   # fp32 sums in another order than the checker's and whole runs part ways: the stop rule at the returned point
        assert g["status"] == c["status"] == "ok"
        if c["niter"] < prm.max_iterations:
            assert g["niter"] < prm.max_iterations
            assert g["gnorm"] <= max(prm.epsilon, prm.epsilon_rel * np.linalg.norm(np.asarray(g["x"], np.float64))) * (1 + 1e-6)
        else:
            assert g["niter"] == prm.max_iterations


# (id, line search, parameters, status): how each chained-Rosenbrock run from x0 = 1.3 at n = N ends, found with the CPU checker
EXITS = [
    ("converged", "MoreThuente", dict(), "ok"),
    ("iteration_cap", "MoreThuente", dict(max_iterations=7), "ok"),
    ("stall", "MoreThuente", dict(past=1, delta=1e-3, max_linesearch=2), "ok"),
    ("cap_on_start_point", "MoreThuente", dict(max_linesearch=1, ftol=0.4, max_iterations=4), "ok"),   # RESTORE ends the run
    ("cap_on_kept_trial", "MoreThuente", dict(max_linesearch=2, wolfe=0.1, max_iterations=5), "ok"),   # the last search keeps an earlier trial
    ("max_linesearch_backtracking", "Backtracking", dict(max_linesearch=2), "runtime_error"),
    ("max_linesearch_bracketing", "Bracketing", dict(max_linesearch=2), "runtime_error"),
    ("step_max_when_armed", "MoreThuente", dict(max_step=0.5), "invalid_argument"),
]


def ends_on(r):
    """Which point the last search of a successful run returned, from its trace of f: its last trial, or an earlier point."""
    return "last_trial" if r["trace"][-1] == r["fx"] else "earlier"


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("name,ls,kw,status", EXITS, ids=[e[0] for e in EXITS])
def test_exit_points(gpu_ctx, orc, name, ls, kw, status, dtype):
    prm = lb.LBFGSParam(**kw)
    x0 = np.full(N, 1.3, dtype)
    c = orc.lbfgs(CHAINED, x0, LS[ls], cpu_param(orc, prm), dtype=dtype, **({"sum_mode": po.SUM_LANES8} if dtype == np.float64 else {}))
    assert c["status"] == status, (c["status"], c["msg"])
    g = lb.LBFGSSolver(prm, ls, dtype=dtype, resident=True).minimize(CHAINED, x0)
    assert (g["status"], g["msg"]) == (c["status"], c["msg"])
    outs, X, G, by_op = resident(gpu_ctx, CHAINED, x0, prm, ls)
    assert np.array_equal(np.asarray(g["x"], dtype=dtype), X[0]) and outs[0].nfev == g["nfev"]
    assert np.array_equal(G[0], chained_grad(X[0]))
    if status == "ok":
        assert ends_on(g) == ends_on(c)
        if name.startswith("cap_on_"):   # f at the start of the last search: f where the run one iteration shorter ended
            prev = lb.LBFGSSolver(lb.LBFGSParam(**dict(kw, max_iterations=kw["max_iterations"] - 1)), ls, dtype=dtype, resident=True).minimize(CHAINED, x0)
            assert ends_on(g) == "earlier" and (g["fx"] == prev["fx"]) == (name == "cap_on_start_point")
            if name == "cap_on_start_point":
                assert by_op.get("restore", 0) > 0, by_op
    if dtype == np.float64:
        check_parity(g, c, xtol=1e-7)
        assert np.max(np.abs(g["x"] - c["x"])) <= 1e-7 * max(1.0, np.max(np.abs(c["x"])))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_chained_batch_matches_lone_solves(gpu_ctx, dtype):
    X0 = np.stack([np.full(N, 1.3), np.full(N, -0.7), np.random.default_rng(7).uniform(-1.5, 1.5, N)]).astype(dtype)
    prm = lb.LBFGSParam(m=6, max_iterations=40)
    outs, X, G, _ = resident(gpu_ctx, CHAINED, X0, prm, "MoreThuente")
    rounds = set()
    for k in range(len(X0)):
        lone, Xl, Gl, _ = resident(gpu_ctx, CHAINED, X0[k], prm, "MoreThuente")
        assert (outs[k].status, outs[k].niter, outs[k].nfev, outs[k].fx) == (lone[0].status, lone[0].niter, lone[0].nfev, lone[0].fx)
        assert np.array_equal(X[k], Xl[0]) and np.array_equal(G[k], Gl[0])
        assert np.array_equal(G[k], chained_grad(X[k]))
        rounds.add(outs[k].rounds)
    assert len(rounds) > 1   # the members finished in different rounds


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
def test_tridiag_batch_with_per_problem_data(gpu_ctx, orc, dtype):
    """Problem b's d and b at offset b*ldd of two flat buffers, ldd > n a multiple of 16 bytes; the elements between problems (and
    past the last one, up to the round_up(n, 32) the bulk copies read) hold NaN, which the solve must never use."""
    B, ldd = 3, N + 5
    assert ldd * np.dtype(dtype).itemsize % 16 == 0
    size = (B - 1) * ldd + -(-N // 32) * 32
    D, R = np.full(size, np.nan, dtype), np.full(size, np.nan, dtype)
    data = []
    for k in range(B):
        _, dk, bk = problem(TRIDIAG, N, dtype, seed=20 + k)
        D[k * ldd:k * ldd + N], R[k * ldd:k * ldd + N] = dk, bk
        data.append((dk, bk))
    prm = lb.LBFGSParam(m=10, max_iterations=25)
    X0 = np.zeros((B, N), dtype)
    outs, X, G, _ = resident(gpu_ctx, TRIDIAG, X0, prm, "MoreThuente", data0=D, data1=R, ldd=ldd)
    for k, (dk, bk) in enumerate(data):
        lone, Xl, Gl, _ = resident(gpu_ctx, TRIDIAG, X0[k], prm, "MoreThuente", data0=dk, data1=bk)
        assert (outs[k].status, outs[k].niter, outs[k].nfev, outs[k].fx) == (lone[0].status, lone[0].niter, lone[0].nfev, lone[0].fx)
        assert np.array_equal(X[k], Xl[0]) and np.array_equal(G[k], Gl[0])
        assert np.array_equal(G[k], tridiag_grad(X[k], dk, bk))
    if dtype == np.float64:
        c = orc.lbfgs(TRIDIAG, X0[0], LS["MoreThuente"], cpu_param(orc, prm), data0=data[0][0], data1=data[0][1], sum_mode=po.SUM_LANES8)
        assert (outs[0].status, outs[0].niter, outs[0].nfev) == (0, c["niter"], c["nfev"])
        assert abs(outs[0].fx - c["fx"]) <= 1e-10 * max(1.0, abs(c["fx"]))
        assert np.max(np.abs(X[0] - c["x"])) <= 1e-7 * max(1.0, np.max(np.abs(c["x"])))


def _pool_block(ctx, nbytes, fill):
    """A block of nbytes from the context's pool, filled with the byte `fill` and given back: the next allocation of that size gets it."""
    p = C.c_void_p()
    ctx.check(ctx.lib.lbfgs_b200_malloc(ctx.h, C.byref(p), nbytes))
    host = np.full(nbytes, fill, np.uint8)
    ctx.check(ctx.lib.lbfgs_b200_memcpy_h2d(ctx.h, p, host.ctypes.data_as(C.c_void_p), nbytes))
    ctx.sync()
    ctx.check(ctx.lib.lbfgs_b200_free(ctx.h, p))
    return p.value


def _solve_on_recycled(objective, x0, d, b, prm, fill):
    """The solve on a fresh context whose pool hands the solver recycled vector slabs filled with the byte `fill`: x, xp, g, gp, d
    ([5][vec_elems]) and, for a neighbour-coupled objective, x_lo, g_lo ([2][vec_elems]), vec_elems = n rounded up to whole 256-byte
    lines (DESIGN 2).  Such a block comes back from the pool as it was: its size is a whole number of lines, so nothing is cleared."""
    ctx = lb.Context(0)
    try:
        e = x0.dtype.itemsize
        line = -(-x0.size * e // 256) * 256
        slabs = [(5 * line, _pool_block(ctx, 5 * line, fill))]
        if objective in (CHAINED, TRIDIAG):
            slabs.append((2 * line, _pool_block(ctx, 2 * line, fill)))

        def held(s):
            gp = ctx.lib.lbfgs_b200_solver_final_grad_of(s, 0)
            assert any(a <= gp < a + size for size, a in slabs), "the solver did not get the recycled blocks"
            for size, a in slabs:   # both blocks are in use by the solver: the pool hands out another one of that size
                q = C.c_void_p()
                ctx.check(ctx.lib.lbfgs_b200_malloc(ctx.h, C.byref(q), size))
                ctx.check(ctx.lib.lbfgs_b200_free(ctx.h, q))
                assert q.value != a, "the solver did not get the recycled blocks"

        return resident(ctx, objective, x0, prm, "MoreThuente", data0=d, data1=b, on_solver=held)
    finally:
        ctx.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("objective", [lb.OBJ_QUAD_SHIFT, CHAINED], ids=["quad_shift", "chained"])
def test_dirty_padding_is_masked(objective, dtype):
    """Lanes past n are masked in the arithmetic: vectors whose padding holds NaN give the same bits as vectors whose padding is 0."""
    n = 100003
    x0 = np.full(n, 1.3, dtype)
    prm = lb.LBFGSParam(m=3, max_iterations=20)
    dirty = _solve_on_recycled(objective, x0, None, None, prm, 0xFF)   # all-ones bytes: NaN in both dtypes
    clean = _solve_on_recycled(objective, x0, None, None, prm, 0x00)
    (od, Xd, Gd, _), (oc, Xc, Gc, _) = dirty, clean
    assert (od[0].status, od[0].niter, od[0].nfev, od[0].fx) == (oc[0].status, oc[0].niter, oc[0].nfev, oc[0].fx)
    assert np.array_equal(Xd, Xc) and np.array_equal(Gd, Gc)
    assert np.all(np.isfinite(Xd)) and np.all(np.isfinite(Gd))
    gref = quad_shift_grad(Xd[0]) if objective == lb.OBJ_QUAD_SHIFT else chained_grad(Xd[0])
    assert np.array_equal(Gd[0], gref)
