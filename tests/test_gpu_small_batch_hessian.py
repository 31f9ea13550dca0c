"""The kept final approximations of the small-batch solve (LBFGSSmallBatchSolver::keep_final_approx, lbfgs_b200_small_hist_*): keeping
changes nothing of the solve, the kept history is the solve's history, the products B V / H V agree with a float64 restatement of the
reference's get_Bmat / get_Hmat built from the kept pairs, they are deterministic, and every refused call says why."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAXIT = 200
OBJECTIVES = [lb.OBJ_ROSENBROCK_PAIRED, lb.OBJ_QUAD_SHIFT, lb.OBJ_ROSENBROCK_CHAINED, lb.OBJ_QUAD_TRIDIAG]


def problem(objective, B, n, seed, dtype):
    """Seeded start points and (tridiagonal quadratic) per-problem data vectors."""
    rng = np.random.default_rng(seed)
    X0 = rng.uniform(-1.2, 1.2, (B, n)).astype(dtype)
    if objective != lb.OBJ_QUAD_TRIDIAG:
        return X0, None, None, 0
    d0 = rng.uniform(0.5, 2.0, B * n).astype(dtype)
    d1 = rng.standard_normal(B * n).astype(dtype)
    return X0, d0, d1, n


def solve_keep(ctx, objective, X0, prm, ls, d0=None, d1=None, ldd=0, keep=True):
    B, n = X0.shape
    h = lb.SmallHistory(ctx, n, prm.m, B, X0.dtype)
    X = ctx.array(X0.reshape(-1))
    G = ctx.empty(B * n, X0.dtype)
    D0 = ctx.array(d0) if d0 is not None else None
    D1 = ctx.array(d1) if d1 is not None else None
    outs = h.minimize(objective, X, prm, ls, D0, D1, ldd, G=G, keep=keep)
    return h, X.get().reshape(B, n), G.get().reshape(B, n), bytes(outs)


def kept(h, b):
    """Problem b's kept history read back: (S, Y by age (c x n), ys, SY, YY, SS (c x c by age), theta) as float64."""
    c_all, th = h.info()
    c, n, m, e = int(c_all[b]), h.n, h.m, h.dtype.itemsize
    S = np.array([h.column("s", b, a) for a in range(c)], dtype=np.float64).reshape(c, n)
    Y = np.array([h.column("y", b, a) for a in range(c)], dtype=np.float64).reshape(c, n)
    base = h.ctx.lib.lbfgs_b200_small_hist_s_col(h.h, b, 0)   # the record starts with s_0 (SmallHistLayout)
    rest = np.empty(m + 3 * m * m + 1, dtype=h.dtype)
    h.ctx.check(h.ctx.lib.lbfgs_b200_memcpy_d2h(h.ctx.h, rest.ctypes.data_as(C.c_void_p), C.c_void_p(base + e * 2 * m * n), rest.nbytes))
    ys = rest[:c].astype(np.float64)
    g = [rest[m + q * m * m: m + q * m * m + c * c].astype(np.float64).reshape(c, c) for q in range(3)]
    assert rest[m + 3 * m * m] == th[b]
    return S, Y, ys, g[0], g[1], g[2], float(th[b])


def dense_ref(S, Y, theta):
    """float64 restatement of the reference's get_Bmat / get_Hmat from pairs by age: W = [Y, theta S], Minv solved by partial-pivot LU
    (numpy.linalg.solve); H from R = triu(S'Y) in chronological order."""
    c, n = S.shape
    I = np.eye(n)
    if c == 0:
        return theta * I, I / theta
    W = np.hstack([Y.T, theta * S.T])
    SY = S @ Y.T
    L = np.triu(SY, 1)      # L(a, b) = s_a'y_b for pair a newer than pair b (a < b in age)
    Minv = np.block([[-np.diag(np.diag(SY)), L.T], [L, theta * (S @ S.T)]])
    Bm = theta * I - W @ np.linalg.solve(Minv, W.T)
    Sc, Yc = S[::-1], Y[::-1]
    R = np.triu(Sc @ Yc.T)
    A = np.linalg.solve(R, Sc)   # R^-1 S'
    D = np.diag(np.diag(R))
    Us = np.linalg.solve(R.T, (D + Yc @ Yc.T / theta) @ A - Yc / theta)
    Hm = I / theta + Sc.T @ Us - Yc.T @ A / theta
    return Bm, Hm


def rel(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300)


def products(ctx, h, V, inverse, b0=0, count=None, ldv=None, shared=True, ldo=None):
    """h.times on the host array V ((k, n) shared or (count, k, n)); returns (count, k, n)."""
    count = h.B - b0 if count is None else count
    n = h.n
    ldv = n if ldv is None else ldv
    ldo = n if ldo is None else ldo
    k = V.shape[-2]
    Vp = np.full(V.shape[:-1] + (ldv,), np.nan, dtype=h.dtype)   # padding past n is NaN: never read
    Vp[..., :n] = V
    Vd = ctx.array(Vp.reshape(-1))
    O = ctx.empty(count * k * ldo, h.dtype)
    h.times(inverse, b0, count, k, Vd, ldv, 0 if shared else k * ldv, O, ldo, k * ldo)
    return O.get().reshape(count, k, ldo)[..., :n]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("ls", ["MoreThuente", "Backtracking"])
@pytest.mark.parametrize("objective", OBJECTIVES)
def test_keeping_changes_nothing(gpu_ctx, objective, ls, dtype):
    X0, d0, d1, ldd = problem(objective, 64, 40, 7 + objective, dtype)
    prm = lb.LBFGSParam(m=5, max_iterations=MAXIT)
    _, Xa, Ga, oa = solve_keep(gpu_ctx, objective, X0, prm, ls, d0, d1, ldd, keep=False)
    _, Xb, Gb, ob = solve_keep(gpu_ctx, objective, X0, prm, ls, d0, d1, ldd, keep=True)
    assert Xa.tobytes() == Xb.tobytes() and Ga.tobytes() == Gb.tobytes() and oa == ob


def test_n2_history_is_the_batch_solvers(gpu_ctx):
    """At n = 2 the small batch and LBFGSBatchSolver are bit-identical: the kept pairs, c and theta equal lbfgs_b200_solver_history_of's."""
    lib, ctx = gpu_ctx.lib, gpu_ctx
    B, n, m = 16, 2, 3
    X0 = np.random.default_rng(5).uniform(-1.5, 1.5, (B, n))
    X0[3] = 1.0   # starts at the minimiser: c = 0
    prm = lb.LBFGSParam(m=m, max_iterations=MAXIT)
    h, X, _, _ = solve_keep(ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "MoreThuente")
    c_all, th = h.info()
    s = C.c_void_p()
    ctx.check(lib.lbfgs_b200_solver_create_batch(ctx.h, n, m, 8, B, C.byref(s)))
    try:
        Xd = ctx.array(X0.reshape(-1))
        p = lb._AbiParam(*(getattr(prm, f) for f, _ in lb._AbiParam._fields_))
        outs = (lb._Outcome * B)()
        ctx.check(lib.lbfgs_b200_solver_minimize_batch_f64(s, lb.OBJ_ROSENBROCK_PAIRED, None, None, 0, C.byref(p), 3, Xd.ptr, n, outs))
        assert np.array_equal(Xd.get().reshape(B, n), X)
        for b in range(B):
            hb = lib.lbfgs_b200_solver_history_of(s, b)
            c = lib.lbfgs_b200_hist_ncorr(hb)
            assert c == c_all[b]
            theta = (C.c_double * 1)()
            ys = (C.c_double * (m + 1))()
            al = (C.c_double * (m + 1))()
            ctx.check(lib.lbfgs_b200_hist_scalars_f64(hb, theta, ys, al))
            assert theta[0] == th[b] or c == 0
            for a in range(c):
                for which, fn in (("s", lib.lbfgs_b200_hist_s_col), ("y", lib.lbfgs_b200_hist_y_col)):
                    col = np.empty(n)
                    ctx.check(lib.lbfgs_b200_memcpy_d2h(ctx.h, col.ctypes.data_as(C.c_void_p), fn(hb, a), col.nbytes))
                    assert np.array_equal(col, h.column(which, b, a)), (b, a, which)
        assert c_all[3] == 0 and c_all.max() == m
    finally:
        lib.lbfgs_b200_solver_destroy(s)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_kept_history_is_consistent(gpu_ctx, dtype):
    """theta, ys and the Gram blocks agree with a float64 recomputation from the kept pairs; c = min(accepted pairs, m) covers c = 0,
    c < m and a wrapped ring; a chained Rosenbrock run from far away has its curvature gate reject pairs."""
    eps = np.finfo(dtype).eps
    n, m = 24, 4
    X0 = np.random.default_rng(11).uniform(-2, 2, (6, n)).astype(dtype)
    X0[0] = 1.0                                     # c = 0
    for its, want in ((2, 1), (3, 2), (MAXIT, m)):  # max_iterations = 2: one pair; 3: two; long: a wrapped ring
        prm = lb.LBFGSParam(m=m, max_iterations=its)
        h, _, _, outs = solve_keep(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "MoreThuente")
        c_all, th = h.info()
        assert c_all[0] == 0 and th[0] == 1
        assert all(c_all[1:] == want) if want < m else all(c_all[1:] == m)
        for b in range(1, 6):
            S, Y, ys, SY, YY, SS, theta = kept(h, b)
            tol = 50 * eps * max(1.0, np.max(np.abs(S @ Y.T)))
            assert abs(theta - Y[0] @ Y[0] / (S[0] @ Y[0])) <= 50 * eps * abs(theta)
            assert np.max(np.abs(ys - np.diag(S @ Y.T))) <= tol
            for got, ref in ((SY, S @ Y.T), (YY, Y @ Y.T), (SS, S @ S.T)):
                assert np.max(np.abs(got - ref)) <= 50 * eps * max(1.0, np.max(np.abs(ref))), (its, b)
    # the curvature gate: the small batch takes the chained Rosenbrock from far away through rejected pairs on some problems; the kept
    # ring then holds fewer pairs than the iterations would give, and it is still consistent
    Xc = np.random.default_rng(3).uniform(-3, 3, (32, 16)).astype(dtype)
    prm = lb.LBFGSParam(m=3, max_iterations=40)
    h, _, _, _ = solve_keep(gpu_ctx, lb.OBJ_ROSENBROCK_CHAINED, Xc, prm, "Backtracking")
    c_all, _ = h.info()
    assert c_all.max() <= 3
    for b in range(4):
        S, Y, ys, SY, _, _, theta = kept(h, b)
        assert np.all(np.diag(S @ Y.T) > eps * np.diag(Y @ Y.T))   # every kept pair passed the gate
        assert np.max(np.abs(SY - S @ Y.T)) <= 50 * eps * max(1.0, np.max(np.abs(S @ Y.T)))


def check_products(gpu_ctx, objective, n, m, dtype, ks=(1, 5, 16, 17, 40), per_problem=False, ldv_pad=0, B=3, its=MAXIT):
    X0, d0, d1, ldd = problem(objective, B, n, 100 + n + m, dtype)
    prm = lb.LBFGSParam(m=m, max_iterations=its)
    h, _, _, _ = solve_keep(gpu_ctx, objective, X0, prm, "MoreThuente", d0, d1, ldd)
    c_all, _ = h.info()
    rng = np.random.default_rng(n * 7 + m)
    eps = np.finfo(dtype).eps
    for b in range(B):
        S, Y, _, _, _, _, theta = kept(h, b)
        Bm, Hm = dense_ref(S, Y, theta)
        # fp64: 1e-10.  fp32: the coefficients come from 2c x 2c solves in fp32 whose error grows with the condition of Minv / R; bound
        # it by eps32 * cond(B) * 100 (at least 1e-3)
        tol = 1e-10 if dtype == np.float64 else max(1e-3, 100 * eps * np.linalg.cond(Bm))
        for k in ks:
            V = rng.standard_normal((B, k, n) if per_problem else (k, n))
            for inverse, ref in ((0, Bm), (1, Hm)):
                got = products(gpu_ctx, h, V.astype(dtype), inverse, ldv=n + ldv_pad, shared=not per_problem)[b].astype(np.float64)
                Vb = (V[b] if per_problem else V).astype(dtype).astype(np.float64)
                want = Vb @ ref.T
                assert rel(got, want) <= tol, (objective, n, m, k, b, inverse, rel(got, want), tol, int(c_all[b]))
    return h


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("objective", OBJECTIVES)
def test_products_match_the_reference(gpu_ctx, objective, dtype):
    for m in (1, 3, 10):
        check_products(gpu_ctx, objective, 30, m, dtype, ks=(1, 17) if m != 3 else (1, 5, 16, 17, 40))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_products_at_the_edges_of_the_budget(gpu_ctx, dtype):
    """n from 2 to small_max_n, the largest m small_max_n admits (its products' shared memory is sized from m), padded ldv, per-problem
    V.  Runs stop while the pairs are still independent (c <= n / 2), so that the reference's Minv is well conditioned."""
    obj = lb.OBJ_ROSENBROCK_PAIRED
    check_products(gpu_ctx, obj, 2, 1, dtype, ks=(1, 5))
    check_products(gpu_ctx, obj, lb.small_max_n(10, obj, dtype), 10, dtype, ks=(1, 16), B=2)
    m_big = max(m for m in range(1, 65) if lb.small_max_n(m, obj, dtype) >= 4)
    n_big = lb.small_max_n(m_big, obj, dtype)
    check_products(gpu_ctx, obj, n_big, m_big, dtype, ks=(1, 17), B=2, its=max(2, n_big // 2))
    check_products(gpu_ctx, obj, 50, 6, dtype, ks=(5, 17), per_problem=True, ldv_pad=3)


def test_secant_equations_and_inverse(gpu_ctx):
    n, m = 40, 6
    X0 = np.random.default_rng(2).uniform(-1.2, 1.2, (4, n))
    h, _, _, _ = solve_keep(gpu_ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, lb.LBFGSParam(m=m, max_iterations=MAXIT), "MoreThuente")
    for b in range(4):
        S, Y, _, _, _, _, _ = kept(h, b)
        Bs = products(gpu_ctx, h, S[:1], 0, b0=b, count=1)[0, 0]
        Hy = products(gpu_ctx, h, Y[:1], 1, b0=b, count=1)[0, 0]
        assert rel(Bs, Y[0]) <= 1e-8 and rel(Hy, S[0]) <= 1e-8
        V = np.random.default_rng(b).standard_normal((5, n))
        BV = products(gpu_ctx, h, V, 0, b0=b, count=1)[0]
        HBV = products(gpu_ctx, h, BV, 1, b0=b, count=1)[0]
        Bm, _ = dense_ref(S, Y, kept(h, b)[6])
        assert rel(HBV, V) <= 1e-10 * max(1.0, np.linalg.cond(Bm))


def test_determinism():
    """Problem b's products are the same bits at positions 0, 17 and B-1 of B = 100 000, in a sub-range and alone; a k = 40 call equals
    40 one-vector calls column by column."""
    ctx = lb.Context(0)
    n, B, m = 8, 100000, 3
    p = np.random.default_rng(1).uniform(-1, 1, n)
    X0 = np.random.default_rng(2).uniform(-1, 1, (B, n))
    for pos in (0, 17, B - 1):
        X0[pos] = p
    h, _, _, _ = solve_keep(ctx, lb.OBJ_ROSENBROCK_PAIRED, X0, lb.LBFGSParam(m=m, max_iterations=MAXIT), "MoreThuente")
    ha, _, _, _ = solve_keep(ctx, lb.OBJ_ROSENBROCK_PAIRED, p[None, :], lb.LBFGSParam(m=m, max_iterations=MAXIT), "MoreThuente")
    V = np.random.default_rng(3).standard_normal((40, n))
    for inverse in (0, 1):
        full = products(ctx, h, V, inverse)
        sub = products(ctx, h, V, inverse, b0=10, count=20)
        alone = products(ctx, ha, V, inverse)[0]
        for pos in (0, 17, B - 1):
            assert full[pos].tobytes() == alone.tobytes()
        assert sub[7].tobytes() == alone.tobytes()
        for j in range(40):
            one = products(ctx, h, V[j:j + 1], inverse, b0=17, count=1)[0, 0]
            assert one.tobytes() == full[17, j].tobytes()
    ctx.close()


def test_driver_entry_and_shared_vs_per_problem_V():
    X0 = np.random.default_rng(4).uniform(-1, 1, (5, 12))
    V = np.random.default_rng(5).standard_normal((3, 12))
    prm = lb.LBFGSParam(m=4, max_iterations=MAXIT)
    res, X, BV, HV, HBV = lb.small_batch_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, X0, V, prm)
    res2, X2, BV2, HV2, _ = lb.small_batch_hessian_times(lb.OBJ_ROSENBROCK_PAIRED, X0, np.broadcast_to(V, (5, 3, 12)), prm)
    _, Xs, _ = lb.solve_small_batch(lb.OBJ_ROSENBROCK_PAIRED, X0, prm)
    assert np.array_equal(X, Xs) and np.array_equal(X2, X) and res == res2
    assert np.array_equal(BV, BV2) and np.array_equal(HV, HV2)
    assert rel(HBV, np.broadcast_to(V, HBV.shape)) <= 1e-8


def test_front_errors_and_dense_matrices(tmp_path):
    libdir = os.path.join(ROOT, "lbfgspp_b200")
    exe = str(tmp_path / "small_batch_hessian_front")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-o", exe,
                    os.path.join(ROOT, "tests", "cpp", "small_batch_hessian_front.cpp"), "-L", libdir, "-l:liblbfgs_b200.so",
                    "-Wl,-rpath," + libdir, "-pthread"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.endswith("small batch hessian front done\n"), r.stdout + r.stderr
    out = dict(line.split(": ", 1) for line in r.stdout.splitlines()[:-1])
    not_kept = "logic_error: LBFGSSmallBatchSolver: no final approximation kept (call keep_final_approx(true) before minimize())"
    for case in ("before minimize, all", "before minimize, one", "before minimize, dense", "not kept"):
        assert out[case] == not_kept, case
    for case in ("all, not whole", "all, empty"):
        assert out[case] == "invalid_argument: V.size() must be a positive multiple of B * n", case
    for case in ("one, b = -1", "one, b = B", "dense, b = B"):
        assert out[case] == "invalid_argument: LBFGSSmallBatchSolver: problem index out of range", case
    assert out["one, not whole"] == "invalid_argument: V.size() must be a positive multiple of n"
    for case in ("kept, all", "kept, one"):
        assert out[case] == "ok"
    for b in range(3):
        assert float(out["dense %d asym B" % b]) <= 1e-12 and float(out["dense %d asym H" % b]) <= 1e-12
        assert float(out["dense %d BH - I" % b]) <= 1e-8
    assert out["dense 2 exact"] == "1"
    invalid = {"times before a solve": "no solve has filled", "keep, B differs": "history was made", "keep, n differs": "history was made",
               "keep, m differs": "history was made", "keep, precision differs": "history was made", "keep, NULL history": "NULL history",
               "times k=0": "k must be", "times ldv<n": "leading dimensions", "times ldo<n": "leading dimensions",
               "times b0<0": "problems [", "times past B": "problems [", "times count=0": "problems [", "times NULL V": "NULL argument",
               "times NULL OUT": "NULL argument", "times OUT=V other layout": "OUT may be V only", "times OUT=V shared": "OUT may be V only",
               "times wrong precision": "holds fp64 values", "create m=0": "small_hist_create: need", "create B=0": "small_hist_create: need",
               "create NULL out": "NULL argument"}
    for case, want in invalid.items():
        assert out[case].startswith("ERR_INVALID: ") and want in out[case], (case, out[case])
    for case in ("keep", "times OUT=V same layout", "times", "sync"):
        assert out[case].startswith("OK"), (case, out[case])
