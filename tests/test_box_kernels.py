"""The bound-constrained entry points of the C ABI (include/lbfgs_b200.h, LBFGS_B200_DECLARE_BOX), fp64 and fp32, one entry point at a
time against plain float64 numpy restatements of their contract (lbfgspp_b200/csrc/lbfgsb_kernels.cuh).

Every test runs on two backends through the same ctypes calls:
  "double"  tests/cpp/mock_abi.cpp compiled on its own: the host-memory test double of the ABI (sequential sums, no GPU).  It proves
            the references, the tolerances and the plumbing; tests/test_front_on_mock_cpu.py pins the double to the CPU checker.
  "gpu"     liblbfgs_b200.so on an H100: the kernels against the same references.
Inputs are rounded to the working precision T before anything else, so a reference and a backend see the same bits.

Tolerances (as in tests/test_gpu_kernels.py):
  - element-wise outputs (clamp, brk, d, xcp, every vector a sub-step writes): <= 2 ulp of the sum of the magnitudes of the
    operands, which admits FMA contraction and nothing else;
  - class bytes, counts, proj_grad_norm (a max) and dir_info's step (a min): exact;
  - sums: |err| <= 64 eps sum|terms| on the GPU (tree sums), K u sum|terms| on the double (K terms left to right); per row for
    lincomb (red_tol).
The bars of the breakpoint sweep are derived in test_cauchy_sweep's docstring.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [1, 2, 127, 128, 129, 2047, 2048, 2049, 100_003, (1 << 20) + 7]
DTYPES = [np.float64, np.float32]
SUF = {np.dtype(np.float64): "f64", np.dtype(np.float32): "f32"}
INF = np.inf
NAN_BITS = {np.dtype(np.float64): np.uint64(0x7FF8DEADBEEF0001), np.dtype(np.float32): np.uint32(0x7FC0BEEF)}
UINT = {np.dtype(np.float64): np.uint64, np.dtype(np.float32): np.uint32}


def _gxx(out, sources, hidden):
    """hidden: export only what is marked for export (the driver's entry points), as test_front_on_mock_cpu.py builds them."""
    vis = ["-fvisibility=hidden", "-fvisibility-inlines-hidden"] if hidden else []
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wno-unknown-pragmas"] + vis +
                   ["-Wl,-Bsymbolic", "-o", out] + sources + ["-pthread"], check=True)
    return out


@pytest.fixture(scope="module", params=["double", pytest.param("gpu", marks=pytest.mark.gpu)])
def backend(request, tmp_path_factory):
    """A Context on the test double (CPU) or on liblbfgs_b200.so (GPU)."""
    if request.param == "double":
        so = _gxx(str(tmp_path_factory.mktemp("box_double") / "mock_abi.so"), [os.path.join(ROOT, "tests", "cpp", "mock_abi.cpp")], False)
        ctx = lb.Context(0, lib=C.CDLL(so))
    else:
        ctx = lb.Context(0)
    ctx.kind = request.param
    yield ctx
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- helpers
def eps(dt):
    return float(np.finfo(dt).eps)


def red_tol(backend, terms, dt, axis=None):
    """Bar of a sum of `terms`: 64 eps sum|terms| for the kernels' tree-shaped sums; the double adds left to right, where only the
    recursive-summation bound K u sum|terms| (K terms, u = eps/2) holds."""
    a = np.abs(np.asarray(terms, dtype=np.float64))
    k = 64 * eps(dt) if backend.kind == "gpu" else max(64 * eps(dt), (a.size if axis is None else a.shape[axis]) * eps(dt) / 2)
    return k * np.sum(a, axis=axis) + 1e-300


def assert_ew(got, ref, scale, dt, what=""):
    """Element-wise result: equal, or within 2 ulp of `scale` (the sum of the operands' magnitudes)."""
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    with np.errstate(invalid="ignore"):   # inf - inf where both are inf: those are equal already
        diff = np.abs(got - ref)
    ok = (got == ref) | (np.isnan(got) & np.isnan(ref)) | (diff <= 2 * eps(dt) * np.asarray(scale, dtype=np.float64))
    assert np.all(ok), (what, np.flatnonzero(~ok)[:5], got[~ok][:5], ref[~ok][:5])


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return np.array_equal(a.view(UINT[a.dtype]), b.view(UINT[b.dtype]))


def fn(ctx, name, dt):
    return getattr(ctx.lib, "lbfgs_b200_%s_%s" % (name, SUF[np.dtype(dt)]))


def out_buf(dt, k):
    ct = C.c_double if np.dtype(dt) == np.float64 else C.c_float
    return (ct * max(k, 1))()


def host_ptr(a):
    ct = C.c_double if a.dtype == np.float64 else C.c_float
    return a.ctypes.data_as(C.POINTER(ct))


def dev(ctx, a, off=0):
    return lb.DeviceArray(ctx, a, offset_elems=off)


def make_history(ctx, n, m, dt, npairs, rng):
    h = lb.History(ctx, n, m, dt)
    for _ in range(npairs):
        s = rng.standard_normal(n).astype(dt)
        y = (s * rng.uniform(0.5, 2.0, n) + 0.1 * rng.standard_normal(n)).astype(dt)
        h.add(ctx.array(s), ctx.array(y))
    return h


def ring(h):
    """(S, Y) of the ring by age (newest first), float64, (c, n) each."""
    c = h.ncorr
    S = np.array([h.column("s", a) for a in range(c)], dtype=np.float64).reshape(c, h.n)
    Y = np.array([h.column("y", a) for a in range(c)], dtype=np.float64).reshape(c, h.n)
    return S, Y


# ---------------------------------------------------------------------------------------------------------------- clamp / pgnorm / dir_info
def bound_inputs(n, dt, rng):
    """x, g, d, lb, ub in T with every kind of coordinate: +-inf bounds, lb == ub, x on a bound, x outside the box."""
    x = rng.uniform(-2, 2, n)
    lo = x - rng.uniform(0.0, 1.0, n)
    hi = x + rng.uniform(0.0, 1.0, n)
    k = rng.integers(0, 9, n)
    lo[(k == 0) | (k == 2)] = -INF
    hi[(k == 1) | (k == 2)] = INF
    hi[k == 3] = lo[k == 3]
    x[k == 3] = lo[k == 3]
    x[k == 4] = lo[k == 4]
    x[k == 5] = hi[k == 5]
    x[k == 6] += 3 * rng.choice([-1.0, 1.0], int(np.sum(k == 6)))
    g = rng.standard_normal(n)
    d = rng.standard_normal(n)
    d[rng.random(n) < 0.2] = 0.0
    return tuple(v.astype(dt) for v in (x, g, d, lo, hi))


def ref_step(x, d, lo, hi):
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        s = np.where(d > 0, (hi - x) / d, np.where(d < 0, (lo - x) / d, np.asarray(INF, dtype=x.dtype)))
    return float(np.min(s)) if s.size else INF


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", SIZES)
def test_clamp_proj_grad_norm_dir_info(backend, n, dtype):
    dt = np.dtype(dtype)
    rng = np.random.default_rng(n + 7 * dt.itemsize)
    x, g, d, lo, hi = bound_inputs(n, dt, rng)
    cases = {"mixed": d, "d_zero": np.zeros(n, dt),
             "d_to_inf_bounds": np.where(np.isposinf(hi), np.abs(d) + 1, np.where(np.isneginf(lo), -np.abs(d) - 1, 0)).astype(dt)}
    for off in (0, 1):
        X, G, L, U = (dev(backend, v, off) for v in (x, g, lo, hi))
        # proj_grad_norm: max |clamp(x - g) - x|, computed in T like the kernel (exact: a max of exactly rounded values)
        o = out_buf(dt, 1)
        backend.check(fn(backend, "box_proj_grad_norm", dt)(backend.h, n, X.ptr, G.ptr, L.ptr, U.ptr, o))
        p = np.minimum(np.maximum(x - g, lo), hi) - x
        assert o[0] == max(0.0, float(np.max(np.abs(p)))), (off, o[0])
        for name, dd in cases.items():
            D = dev(backend, dd, off)
            o2 = out_buf(dt, 2)
            backend.check(fn(backend, "box_dir_info", dt)(backend.h, n, X.ptr, D.ptr, G.ptr, L.ptr, U.ptr, o2))
            terms = g.astype(np.float64) * dd.astype(np.float64)
            assert abs(o2[0] - np.sum(terms)) <= red_tol(backend, terms, dt), (name, off)
            step = ref_step(x, dd, lo, hi)
            assert o2[1] == step, (name, off, o2[1], step)
            if name != "mixed":
                assert step == INF
        # clamp last: it writes x in place
        backend.check(fn(backend, "box_clamp", dt)(backend.h, n, X.ptr, L.ptr, U.ptr))
        assert bits_equal(X.get(), np.minimum(np.maximum(x, lo), hi)), off


# ---------------------------------------------------------------------------------------------------------------- Cauchy: breaks and build
def breaks_inputs(n, dt, rng):
    """x in [lb, ub]: lb == ub with g != 0, x on a bound with g pointing out, g = 0 with finite bounds, +-inf bounds, and a tie group
    (identical x, lb, ub, g) that shares one breakpoint."""
    x = rng.uniform(-2, 2, n)
    lo = x - rng.uniform(0.1, 1.0, n)
    hi = x + rng.uniform(0.1, 1.0, n)
    g = rng.standard_normal(n)
    k = rng.integers(0, 10, n)
    hi[k == 0] = lo[k == 0]
    x[k == 0] = lo[k == 0]
    x[k == 1] = lo[k == 1]
    g[k == 1] = np.abs(g[k == 1]) + 0.5           # g > 0 at x = lb: d = -g points out, brk = +0
    x[k == 2] = hi[k == 2]
    g[k == 2] = -np.abs(g[k == 2]) - 0.5          # g < 0 at x = ub: brk = -0
    g[k == 3] = 0.0                                # finite bounds, never moves: FREE
    lo[k == 4] = -INF
    hi[k == 5] = INF
    lo[k == 6], hi[k == 6] = -INF, INF
    x[k == 7], lo[k == 7], hi[k == 7], g[k == 7] = 0.25, -1.0, 2.0, 0.75   # the tie group: brk = 5/3 for all
    return tuple(v.astype(dt) for v in (x, g, lo, hi))


def ref_breaks(x, g, lo, hi):
    dt = x.dtype
    with np.errstate(divide="ignore", invalid="ignore"):
        brk = np.where(lo == hi, dt.type(0), np.where(g < 0, (x - hi) / g, np.where(g > 0, (x - lo) / g, dt.type(INF)))).astype(dt)
    zero = brk == 0
    d = np.where(zero, dt.type(0), -g).astype(dt)
    cls = np.where(brk == INF, lb.CLS_FREE, np.where(zero, lb.CLS_FIXED, 0)).astype(np.uint8)
    ordv = brk[cls == 0]
    out5 = [np.sum(cls == lb.CLS_FIXED), np.sum(cls == lb.CLS_FREE), np.sum(cls == 0),
            np.sum((d * d).astype(np.float64)), float(np.min(ordv)) if ordv.size else INF]
    return brk, d, cls, out5, (d * d).astype(np.float64)


def ref_build(x, lo, hi, brk, d, cls, t_cross, tfinal):
    dt = x.dtype
    movable = cls != lb.CLS_FIXED
    crossed = movable & (cls != lb.CLS_FREE) & (brk <= t_cross)
    xcp = np.where(~movable, x, np.where(crossed, np.where(d > 0, hi, lo), x + dt.type(tfinal) * d)).astype(dt)
    cls1 = np.where(~movable, lb.CLS_FIXED, np.where(crossed, lb.CLS_ACT, lb.CLS_FREE)).astype(np.uint8)
    return xcp, cls1, [np.sum(crossed), np.sum(movable & ~crossed)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", SIZES)
def test_cauchy_breaks_and_build(backend, n, dtype):
    dt = np.dtype(dtype)
    rng = np.random.default_rng(3 * n + dt.itemsize)
    x, g, lo, hi = breaks_inputs(n, dt, rng)
    h = lb.History(backend, n, 3, dt)
    box = lb.Box(h)
    X, G, L, U = (dev(backend, v) for v in (x, g, lo, hi))
    brk, d, cls, out5, dd_terms = ref_breaks(x, g, lo, hi)
    tie = dt.type((0.25 - (-1.0)) / 0.75)
    ordv = np.sort(brk[cls == 0])
    t_choices = [-1.0, float(tie), float(ordv[ordv.size // 2]) if ordv.size else 1.0, float(ordv[-1]) if ordv.size else 2.0]
    for t_cross in t_choices:
        o5 = out_buf(dt, 5)
        backend.check(fn(backend, "box_cauchy_breaks", dt)(box.h, X.ptr, G.ptr, L.ptr, U.ptr, o5))
        assert list(o5)[:3] == out5[:3] and o5[4] == out5[4], (list(o5), out5)
        assert abs(o5[3] - out5[3]) <= red_tol(backend, dd_terms, dt)
        assert bits_equal(box.get(lb.BOXV_BRK), brk) and bits_equal(box.get(lb.BOXV_DVEC), d)
        assert np.array_equal(box.get("cls"), cls)
        tfinal = dt.type(max(t_cross, 0.0) + 0.37)
        c2 = out_buf(dt, 2)
        backend.check(fn(backend, "box_cauchy_build", dt)(box.h, X.ptr, L.ptr, U.ptr, dt.type(t_cross), tfinal, c2))
        xcp, cls1, counts = ref_build(x, lo, hi, brk, d, cls, dt.type(t_cross), tfinal)
        assert list(c2) == counts, (t_cross, list(c2), counts)
        assert np.array_equal(box.get("cls"), cls1), t_cross
        assert_ew(box.get(lb.BOXV_XCP), xcp, np.abs(x) + np.abs(tfinal * d), dt, t_cross)
        fixed = cls == lb.CLS_FIXED
        assert bits_equal(box.get(lb.BOXV_XCP)[fixed], x[fixed])          # FIXED rows: xcp = x, class unchanged
        if t_cross == float(tie) and n >= 64:
            grp = (x == dt.type(0.25)) & (g == dt.type(0.75)) & (lo == dt.type(-1.0))
            assert np.sum(grp) >= 2 and np.all(cls1[grp] == lb.CLS_ACT)   # the whole tie group is crossed at its own breakpoint
        if t_cross == -1.0:
            assert counts[0] == 0


# ---------------------------------------------------------------------------------------------------------------- W'v, lincomb, masked Gram
def class_bytes(n, rng):
    return rng.integers(0, 64, n).astype(np.uint8)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", SIZES)
def test_wt_dot_lincomb_masked_gram(backend, n, dtype):
    dt = np.dtype(dtype)
    rng = np.random.default_rng(11 * n + dt.itemsize)
    m = 3
    v = rng.standard_normal(n).astype(dt)
    v0 = rng.standard_normal(n).astype(dt)
    cls = class_bytes(n, rng)
    nan =np.full(n, NAN_BITS[dt], dtype=UINT[dt]).view(dt)
    for npairs in (0, 1, m, m + 2):              # c = 0, 1, m (the last wraps the ring)
        h = make_history(backend, n, m, dt, npairs, rng)
        box = lb.Box(h)
        box.set("cls", cls)
        clsp = box._ptr("cls")
        c = h.ncorr
        S, Y = ring(h)
        # hist_wt_dot, v aligned and offset by one element (the element-wise dots path)
        for off in (0, 1):
            raw = out_buf(dt, 2 * m)
            for k in range(2 * m):
                raw[k] = 7.0
            Vd = dev(backend, v, off)
            backend.check(fn(backend, "hist_wt_dot", dt)(h.h, Vd.ptr, raw))
            for j in range(c):
                assert abs(raw[j] - Y[j] @ v) <= red_tol(backend, Y[j] * v, dt), (c, off, j)
                assert abs(raw[c + j] - S[j] @ v) <= red_tol(backend, S[j] * v, dt), (c, off, j)
            assert all(raw[k] == 7.0 for k in range(2 * c, 2 * m))
        # hist_lincomb: every class bit, some unions, cls = NULL, v0 = NULL
        coef = rng.standard_normal(2 * c).astype(dt)
        a0 = dt.type(-0.75)
        for mask, use_cls, use_v0 in [(1, True, True), (2, True, True), (4, True, False), (8, True, True), (16, True, True),
                                      (32, True, True), (4 | 32, True, True), (1 | 2 | 4, True, False), (63, True, True),
                                      (0, False, True), (0, False, False)]:
            out, V0 = dev(backend, nan), dev(backend, v0)
            st = fn(backend, "hist_lincomb", dt)(h.h, box.h, a0, V0.ptr if use_v0 else None,
                                                  host_ptr(coef) if c else None, clsp if use_cls else None, mask, out.ptr)
            backend.check(st)
            terms = np.zeros((n, 2 * c + 1))
            if use_v0:
                terms[:, 0] = float(a0) * v0.astype(np.float64)
            terms[:, 1:1 + c] = (Y * coef[:c, None].astype(np.float64)).T
            terms[:, 1 + c:] = (S * coef[c:, None].astype(np.float64)).T
            sel = (cls & mask) != 0 if use_cls else np.ones(n, bool)
            got = out.get()
            assert bits_equal(got[~sel], nan[~sel]), (mask, "rows outside the mask were written")
            ref = np.sum(terms[sel], axis=1)
            assert np.all(np.abs(got[sel] - ref) <= red_tol(backend, terms[sel], dt, axis=1)), (c, mask, use_cls, use_v0)
        # hist_masked_gram
        R = np.vstack([Y, S])                        # (2c, n): y by age, then s by age
        for mask in (0, 4, 4 | 32, 63):
            G = out_buf(dt, 4 * m * m)
            backend.check(fn(backend, "hist_masked_gram", dt)(h.h, box.h, clsp, mask, G))
            sel = (cls & mask) != 0
            Rs = R[:, sel]
            for a in range(2 * c):
                for b_ in range(2 * c):
                    t = Rs[a] * Rs[b_]
                    assert abs(G[a * 2 * c + b_] - np.sum(t)) <= red_tol(backend, t, dt), (c, mask, a, b_)
            if mask == 0:
                assert all(G[e] == 0 for e in range(4 * c * c))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", [1, 6, 20])
@pytest.mark.parametrize("n", [1, 5, 127, 129, 300, 4097])
def test_masked_gram_shapes(backend, n, c, dtype):
    """Empty mask, a single selected row, n < 128 and n not a multiple of the 128-row strips, c up to 20 (fp64 c = 20 stages
    40 KB of rows in shared memory)."""
    dt = np.dtype(dtype)
    rng = np.random.default_rng(n + 100 * c + dt.itemsize)
    h = make_history(backend, n, c, dt, c, rng)
    box = lb.Box(h)
    S, Y = ring(h)
    R = np.vstack([Y, S])
    w = 2 * c
    one = np.zeros(n, np.uint8)
    one[rng.integers(0, n)] = lb.SUB_P
    for cls, mask in ((class_bytes(n, rng), 0), (one, lb.SUB_P), (class_bytes(n, rng), lb.CLS_FREE), (class_bytes(n, rng), 63)):
        box.set("cls", cls)
        G = out_buf(dt, w * w)
        backend.check(fn(backend, "hist_masked_gram", dt)(h.h, box.h, box._ptr("cls"), mask, G))
        sel = (cls & mask) != 0
        Rs = R[:, sel]
        ref = Rs @ Rs.T
        tol = 64 * eps(dt) * (np.abs(Rs) @ np.abs(Rs).T) + 1e-300
        got = np.array(G[:w * w]).reshape(w, w)
        assert np.all(np.abs(got - ref) <= tol), (mask, np.max(np.abs(got - ref) - tol))
        if not sel.any():
            assert np.all(got == 0)


# ---------------------------------------------------------------------------------------------------------------- the Gram blocks
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("m", [1, 2, 5, 20])
def test_gram_blocks_follow_the_history(backend, m, dtype):
    """hist_gram's SY, SS, YY, ys and theta and hist_wt_dot against float64 products of the ring's own columns after every step of
    a fixed script: add, update accepted / rejected, update_apply_Hv accepted / rejected, apply_Hv TWO_LOOP (leaves the new pair's
    Gram row pending), apply_Hv GRAM (folds it), back-to-back adds, reset; >= 3m pairs so the ring wraps several times.  Only
    L-BFGS-B reads SS (BFGSMat.h refresh_middle), so no apply_Hv parity test would see a stale SS block.  Reading the Gram blocks
    folds a pending pair, so the checks right after `update` and TWO_LOOP are skipped once per cycle to let GRAM's own fold run."""
    dt = np.dtype(dtype)
    n = 3001
    rng = np.random.default_rng(m + dt.itemsize)
    h = lb.History(backend, n, m, dt)
    x = rng.standard_normal(n).astype(dt)
    g = (2.0 * x).astype(dt)
    res = backend.empty(n, dt)
    v = dev(backend, rng.standard_normal(n).astype(dt))
    vh = v.get().astype(np.float64)

    def step_pair(accept):
        nonlocal x, g
        x1 = (x + 0.3 * rng.standard_normal(n)).astype(dt)
        g1 = (g + (1.5 if accept else -1.5) * (x1 - x) + 0.01 * rng.standard_normal(n)).astype(dt)
        args = [dev(backend, a) for a in (x1, x, g1, g)]
        if accept:
            x, g = x1, g1
        return args

    def check(where):
        c = h.ncorr
        S, Y = ring(h)
        SY, SS, YY, ys, th = out_buf(dt, c * c), out_buf(dt, c * c), out_buf(dt, c * c), out_buf(dt, c), out_buf(dt, 1)
        backend.check(fn(backend, "hist_gram", dt)(h.h, SY, SS, YY, ys, th))
        for i in range(c):
            for j in range(c):
                for blk, A, B in ((SY, S, Y), (SS, S, S), (YY, Y, Y)):
                    t = A[i] * B[j]
                    assert abs(blk[i * c + j] - np.sum(t)) <= red_tol(backend, t, dt), (where, c, i, j)
            assert abs(ys[i] - S[i] @ Y[i]) <= red_tol(backend, S[i] * Y[i], dt), (where, i)
        theta_ref = (Y[0] @ Y[0]) / (S[0] @ Y[0]) if c else 1.0
        assert abs(th[0] - theta_ref) <= 256 * eps(dt) * abs(theta_ref), (where, th[0], theta_ref)
        raw = out_buf(dt, 2 * c)
        backend.check(fn(backend, "hist_wt_dot", dt)(h.h, v.ptr, raw))
        for j in range(c):
            assert abs(raw[j] - Y[j] @ vh) <= red_tol(backend, Y[j] * vh, dt) and abs(raw[c + j] - S[j] @ vh) <= red_tol(backend, S[j] * vh, dt), where

    pairs, cycle = 0, 0
    while pairs < 3 * m + 2:
        s = rng.standard_normal(n).astype(dt)
        h.add(dev(backend, s), dev(backend, (1.2 * s + 0.05 * rng.standard_normal(n)).astype(dt)))
        pairs += 1
        check("add")
        assert h.update(*step_pair(True))[0]
        pairs += 1
        if cycle % 2:
            check("update")
        h.apply_Hv(dev(backend, g), dt.type(-1.0), res, lb.HV_TWO_LOOP)
        if cycle % 2:
            check("apply_Hv two-loop")
        h.apply_Hv(dev(backend, g), dt.type(-1.0), res, lb.HV_GRAM)
        check("apply_Hv gram")
        assert not h.update(*step_pair(False))[0]
        check("update rejected")
        assert h.update_apply_Hv(*step_pair(True), dt.type(-1.0), res, lb.HV_GRAM)[0]
        pairs += 1
        check("update_apply_Hv")
        assert not h.update_apply_Hv(*step_pair(False), dt.type(-1.0), res, lb.HV_GRAM)[0]
        check("update_apply_Hv rejected")
        for _ in range(2):
            s = rng.standard_normal(n).astype(dt)
            h.add(dev(backend, s), dev(backend, (0.8 * s + 0.05 * rng.standard_normal(n)).astype(dt)))
            pairs += 1
        check("back-to-back adds")
        if cycle == 1:
            h.reset()
            assert h.ncorr == 0
            check("reset")
            pairs = 0
        cycle += 1
    assert h.ncorr == m


# ---------------------------------------------------------------------------------------------------------------- the breakpoint sweep
def middle_matrix(S, Y, theta):
    """M = Minv^-1 of B = theta I - W M W', W = [Y, theta S] by age, as BFGSMat::refresh_middle builds it."""
    c = S.shape[0]
    SY, SS = S @ Y.T, S @ S.T
    Minv = np.zeros((2 * c, 2 * c))
    for a in range(c):
        Minv[a, a] = -SY[a, a]
        for b in range(c):
            if a < b:
                Minv[c + a, b] = SY[a, b]
                Minv[b, c + a] = SY[a, b]
            Minv[c + a, c + b] = theta * SS[a, b]
    return np.linalg.inv(Minv) if c else np.zeros((0, 0))


def sweep_reference(brk, cls, g, S, Y, theta, M, p0, gt, nfree_inf, dt, chunk=1 << 15):
    """Vectorised float64 restatement of the group-end rule (the double's sequential loop, mock_abi.cpp do_cauchy_sweep): prefix
    sums over the breakpoints sorted by (value, index) as long-double cumsums, the segment test at every tie-group end, the first
    qualifying end finalised.  Returns (out, info) with the float bars' scales and the rounding margins of the group ends up to the
    chosen one."""
    c = S.shape[0]
    w = 2 * c
    idx = np.flatnonzero(cls == 0)
    order = idx[np.lexsort((idx, brk[idx]))]
    t_all = brk[order].astype(np.float64)
    nord = order.size
    carry = np.zeros(1 + 2 * w, dtype=np.longdouble)
    carry_abs = np.zeros(1 + 2 * w)
    margins = []
    e_eps = float(np.finfo(dt).eps)
    for start in range(0, nord, chunk):
        sl = order[start:start + chunk]
        t = t_all[start:start + chunk]
        gi = g[sl].astype(np.float64)
        wy = Y[:, sl].T
        ws = theta * S[:, sl].T
        e = np.empty((sl.size, 1 + 2 * w))
        e[:, 0] = gi * gi
        e[:, 1:1 + c] = gi[:, None] * wy
        e[:, 1 + c:1 + w] = gi[:, None] * ws
        e[:, 1 + w:] = t[:, None] * e[:, 1:1 + w]
        pre = np.cumsum(e.astype(np.longdouble), axis=0) + carry
        pre_abs = np.cumsum(np.abs(e), axis=0) + carry_abs
        carry, carry_abs = pre[-1].copy(), pre_abs[-1].copy()
        k = np.arange(start, start + sl.size)
        tnext = np.where(k + 1 < nord, t_all[np.minimum(k + 1, nord - 1)], INF)
        ends = np.flatnonzero(tnext != t)
        if ends.size == 0:
            continue
        P = pre[ends]
        te, tn, ke = t[ends], tnext[ends], k[ends]
        rest = (gt - P[:, 0]).astype(np.float64)
        p = (p0 + P[:, 1:1 + w]).astype(np.float64)
        cv = (te[:, None] * (p0 + P[:, 1:1 + w]) - P[:, 1 + w:]).astype(np.float64)
        pMc = np.einsum("kr,rq,kq->k", p, M, cv) if w else np.zeros(ends.size)
        pMp = np.einsum("kr,rq,kq->k", p, M, p) if w else np.zeros(ends.size)
        fp = -rest * (1 - theta * te) - pMc
        fpp = theta * rest - pMp
        with np.errstate(divide="ignore", invalid="ignore"):
            dtmin = -fp / fpp
        dtv = tn - te
        all_crossed = (ke == nord - 1) & (nfree_inf == 0)
        sel = ~(dtmin >= dtv) | all_crossed
        first = int(np.argmax(sel)) if sel.any() else ends.size
        with np.errstate(divide="ignore", invalid="ignore"):
            rel = np.abs(dtmin - dtv) / np.maximum(np.abs(dtmin), np.abs(dtv))
        margins += [r for r, d_ in zip(rel[:first + 1], dtv[:first + 1]) if np.isfinite(d_)]
        if first == ends.size:
            continue
        j = first
        Pa = pre_abs[ends[j]]
        rest_abs = abs(gt) + Pa[0]
        p_abs = np.abs(p0) + Pa[1:1 + w]
        c_abs = abs(te[j]) * p_abs + Pa[1 + w:]
        Mabs = np.abs(M)
        fp_abs = rest_abs * (1 + abs(theta * te[j])) + (p_abs @ Mabs @ c_abs if w else 0.0)
        fpp_abs = theta * rest_abs + (p_abs @ Mabs @ p_abs if w else 0.0)
        dtm = dtmin[j]
        small = fpp[j] < e_eps
        if small:
            dtm = -fp[j] / e_eps
        unclamped = dtm
        dtm = max(dtm, 0.0)
        if all_crossed[j]:
            dtm = 0.0
        out = np.concatenate([[te[j], te[j] + dtm, fp[j], fpp[j], 1.0 if all_crossed[j] else 0.0], cv[j] + dtm * p[j]])
        info = dict(k=int(ke[j]), nord=nord, fp_abs=fp_abs, fpp_abs=fpp_abs, p=p[j], p_abs=p_abs, c_abs=c_abs, dtmin=dtm,
                    unclamped=unclamped, small_fpp=small, margins=np.array(margins), fp=fp[j], fpp=fpp[j])
        return out, info
    raise AssertionError("the reference found no segment")


def sweep_case(name, dt, rng, orc):
    """(n, c, x, g, lb, ub) of one sweep case."""
    f32 = dt == np.float32
    if name == "config4":
        # x0 = 3 in [2, 4], paired Rosenbrock: two giant tie groups (even and odd coordinates).  fp32 runs at a smaller n: sequential fp32
        # sums over 2^20 terms (the double) carry up to n*u = 6 % worst-case error, which would leave no margin for the segment test.
        n = (1 << 14) + 2 if f32 else (1 << 20) + 2
        x = np.full(n, 3.0)
        _, g = orc.objective(po.OBJ_ROSENBROCK_PAIRED, x)
        return n, 5, x, g, np.full(n, 2.0), np.full(n, 4.0)
    if name == "ties_straddle":
        # 13 (x, lb, ub, g) tuples spread over 20000 coordinates: tie groups of ~1500 positions straddle the 128-position scan blocks
        # and the 2048-pair sort tiles
        n = 20000
        tx = rng.uniform(0.1, 0.9, 13)
        tg = rng.choice([-1.0, 1.0], 13) * rng.uniform(0.05, 2.0, 13)
        k = rng.integers(0, 13, n)
        x, g = tx[k], tg[k]
        return n, 6, x, g, np.zeros(n), np.ones(n)
    if name == "keys_spread":
        # breakpoints from 1e-200 to 1e200 (fp32: 1e-30 to 1e30): the top radix digits decide.  brk = (x - 0) / 2^j = t exactly
        n = 5000
        e = 30 if f32 else 200
        j = rng.integers(-3, 4, n).astype(np.float64)
        t = (10.0 ** rng.uniform(-e, e, n)).astype(dt).astype(np.float64)
        return n, 7, t * 2.0 ** j, 2.0 ** j, np.zeros(n), np.full(n, INF)
    if name == "keys_ulp":
        # breakpoints one ulp apart around 1: the lowest digit decides (and, with the history's weights, which coordinates are crossed)
        n = 4099
        ulp = eps(dt)
        t = 1.0 + ulp * (rng.permutation(n) - n // 4)    # spacing of T just above 1; below 1 these fall on every second T
        j = rng.integers(-3, 4, n).astype(np.float64)
        return n, 6, t * 2.0 ** j, 2.0 ** j, np.zeros(n), np.full(n, INF)
    if name == "tie_first":
        # one giant tie group at t = 0.5, past the unconstrained minimiser (theta = 4 below), and never-bounded coordinates: the
        # segment test must look at the group's end only -- part-way through the group the slope is already positive
        n = 5000
        x, g = np.full(n, 0.5), np.ones(n)
        lo, hi = np.zeros(n), np.ones(n)
        lo[4000:], hi[4000:] = -INF, INF
        g[4000:] = rng.standard_normal(n - 4000)
        return n, 3, x, g, lo, hi
    if name == "nord1":
        n = 1000
        x, g = np.zeros(n), rng.standard_normal(n)
        lo, hi = np.full(n, -INF), np.full(n, INF)
        lo[17] = -0.4
        g[17] = 1.0
        return n, 4, x, g, lo, hi
    if name == "all_crossed":
        # every bound finite, g != 0, breakpoints far below the model's minimiser: the sweep crosses every group
        n = 3000
        g = rng.choice([-1.0, 1.0], n) * rng.uniform(0.5, 2.0, n)
        dist = rng.uniform(1e-4, 1e-3, n) * np.abs(g)
        return n, 5, np.zeros(n), g, -dist, dist
    if name == "fpp_small":
        # every ordinal breakpoint crossed early, one never-bounded coordinate with a tiny gradient g_f left: in the last segment
        # fpp = theta*g_f^2 - p'Mp < eps, so the finaliser takes dtmin = -fp/eps.  The whole gradient is small too: fpp is what is
        # left of prefix sums that cancel (rest = gt - G, p = p0 + A), and their rounding, ~eps*sum|g^2| and ~eps*sum|g w|, must stay
        # far below g_f^2 and g_f |w| for fpp and fp to be comparable between backends
        n = 3000
        scale, gf = (1e-4, 1e-5) if f32 else (1e-8, 1e-10)
        g = rng.choice([-1.0, 1.0], n) * rng.uniform(0.5, 2.0, n) * scale
        dist = rng.uniform(1e-4, 1e-3, n) * np.abs(g)
        lo, hi = -dist, dist
        lo[5], hi[5] = -INF, INF
        g[5] = gf
        return n, 5, np.zeros(n), g, lo, hi
    c = int(name.split("_")[1])   # "c_<c>": a mixed problem, c on both sides of each MAXV bound of the scan kernels
    n = 3001
    x = rng.uniform(-1, 1, n)
    g = rng.standard_normal(n)
    lo, hi = x - rng.uniform(0.05, 1.5, n), x + rng.uniform(0.05, 1.5, n)
    lo[::11], hi[::13] = -INF, INF
    return n, c, x, g, lo, hi


SWEEP_CASES = ["config4", "ties_straddle", "tie_first", "keys_spread", "keys_ulp", "nord1", "all_crossed", "fpp_small",
               "c_0", "c_1", "c_6", "c_7", "c_10", "c_11", "c_20"]


def sweep_inputs(backend, name, dt, seed, orc):
    rng = np.random.default_rng(seed)
    n, c, x, g, lo, hi = sweep_case(name, dt, rng, orc)
    x, g, lo, hi = (np.asarray(v, dtype=np.float64).astype(dt) for v in (x, g, lo, hi))
    h = make_history(backend, n, max(c, 1), dt, c, rng)
    S, Y = ring(h)
    theta = float(dt.type((Y[0] @ Y[0]) / (S[0] @ Y[0]))) if c else 1.0
    if name == "tie_first":
        theta = 4.0   # B0 = theta I: any theta > 0 gives a valid compact BFGS matrix
    M = middle_matrix(S, Y, theta).astype(dt)
    brk, d, cls, out5, _ = ref_breaks(x, g, lo, hi)
    dd = d.astype(np.float64)
    p0 = np.concatenate([Y @ dd, theta * (S @ dd)]).astype(dt)
    gt = float(dt.type(np.sum(dd * dd)))
    return dict(n=n, c=c, x=x, g=g, lo=lo, hi=hi, h=h, S=S, Y=Y, theta=theta, M=M, p0=p0, gt=gt, brk=brk, cls=cls,
                nord=int(out5[2]), ninf=int(out5[1]))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", SWEEP_CASES)
def test_cauchy_sweep(backend, orc, case, dtype):
    """box_cauchy_breaks then box_cauchy_sweep (radix sort, block scan, group-end test, finalise) against sweep_reference.

    Margin guard: rounding must not be able to flip which segment is chosen, so at every group end up to the chosen one
    |dtmin - dt| / max(|dtmin|, |dt|) must be >= 1e-6 (fp64) or 1e-2 (fp32); the fixed seeds are asserted to pass.  Given that,
    t_cross and the all-crossed flag must match exactly.

    Float bars.  Every output is built from prefix sums over at most K = nord sorted positions.  Recursive summation of K terms
    has |error| <= K u sum|terms| (u = eps/2; Higham, Accuracy and Stability, 4.2), which covers the double's left-to-right sums
    and the kernels' block scans alike; the 2c x 2c products with M add 4c u.  So with rel = (K + 4c + 8) u:
        |d fp|  <= rel * fp_abs,  |d fpp| <= rel * fpp_abs,
    fp_abs / fpp_abs being the same formulas evaluated on magnitudes (sum|g^2|, sum|g w|, sum|t g w|, |p0|, |M|).  Then, to first
    order, |d dtmin| <= rel (fp_abs + |dtmin| fpp_abs) / |fpp| (fpp < eps: rel fp_abs / eps), tfinal = t_cross + dtmin and
    W'(xcp - x0) = c + dtmin p inherit these.  fp64: K <= 2^20 + 2 gives rel <= 1.2e-10, inside 1e-9.  fp32: K <= 20000 gives
    rel <= 1.2e-3; the fp32 cases stay at that size (config4 at n = 2^14 + 2) because this worst-case bound grows with K."""
    dt = np.dtype(dtype)
    seed = SWEEP_CASES.index(case) * 10 + dt.itemsize
    I = sweep_inputs(backend, case, dt, seed, orc)
    if case == "fpp_small":
        # pick the sign of the small gradient that makes fp < 0 (otherwise dtmin clamps to 0 whatever the guard does)
        _, info = sweep_reference(I["brk"], I["cls"], I["g"], I["S"], I["Y"], I["theta"], I["M"].astype(np.float64),
                                  I["p0"].astype(np.float64), I["gt"], I["ninf"], dt)
        if info["fp"] >= 0:
            g = I["g"].copy()
            g[5] = -g[5]
            I.update(g=g)
            brk, d, cls, out5, _ = ref_breaks(I["x"], g, I["lo"], I["hi"])
            dd = d.astype(np.float64)
            I.update(brk=brk, cls=cls, p0=np.concatenate([I["Y"] @ dd, I["theta"] * (I["S"] @ dd)]).astype(dt),
                     gt=float(dt.type(np.sum(dd * dd))))
    n, c, w = I["n"], I["c"], 2 * I["c"]
    box = lb.Box(I["h"])
    X, G, L, U = (dev(backend, I[k]) for k in ("x", "g", "lo", "hi"))
    o5 = out_buf(dt, 5)
    backend.check(fn(backend, "box_cauchy_breaks", dt)(box.h, X.ptr, G.ptr, L.ptr, U.ptr, o5))
    assert int(o5[2]) == I["nord"] and int(o5[1]) == I["ninf"] and np.array_equal(box.get("cls"), I["cls"])
    M64, p064 = I["M"].astype(np.float64), I["p0"].astype(np.float64)
    ref, info = sweep_reference(I["brk"], I["cls"], I["g"], I["S"], I["Y"], I["theta"], M64, p064, I["gt"], I["ninf"], dt)
    guard = 1e-6 if dt == np.float64 else 1e-2
    assert info["margins"].size == 0 or np.min(info["margins"]) >= guard, ("seed fails the margin guard", np.min(info["margins"]))
    out = out_buf(dt, 5 + w)
    M = np.ascontiguousarray(I["M"])
    p0 = np.ascontiguousarray(I["p0"])
    backend.check(fn(backend, "box_cauchy_sweep", dt)(box.h, G.ptr, host_ptr(M) if c else None, host_ptr(p0) if c else None,
                                                       dt.type(I["theta"]), dt.type(I["gt"]), I["nord"], I["ninf"], out))
    got = np.array(out[:5 + w], dtype=np.float64)
    assert got[0] == float(dt.type(ref[0])) and got[4] == ref[4], (case, got[:5], ref[:5], info["k"])
    K = info["nord"]
    u = eps(dt) / 2
    rel = (K + 4 * c + 8) * u
    assert dt == np.float32 or rel <= 1e-9
    fpp_ref = ref[3]
    assert abs(got[2] - ref[2]) <= rel * info["fp_abs"], (case, got[2], ref[2])
    assert abs(got[3] - fpp_ref) <= rel * info["fpp_abs"], (case, got[3], fpp_ref)
    denom = eps(dt) if info["small_fpp"] else abs(fpp_ref)
    tol_dt = rel * (info["fp_abs"] + abs(info["unclamped"]) * info["fpp_abs"]) / denom + 2 * eps(dt) * abs(ref[1])
    assert abs(got[1] - ref[1]) <= tol_dt, (case, got[1], ref[1], tol_dt)
    tol_v = rel * (info["c_abs"] + abs(info["dtmin"]) * info["p_abs"]) + tol_dt * np.abs(info["p"]) + 2 * eps(dt) * np.abs(ref[5:])
    assert np.all(np.abs(got[5:] - ref[5:]) <= tol_v), (case, np.max(np.abs(got[5:] - ref[5:]) - tol_v))
    # the cases reach what they are named for
    if case in ("all_crossed", "config4"):
        assert info["k"] == K - 1 and ref[4] == (1.0 if case == "all_crossed" else ref[4])
    if case == "all_crossed":
        assert ref[4] == 1.0
    if case == "fpp_small":
        assert info["small_fpp"] and info["dtmin"] > 0 and abs(info["unclamped"]) < 0.5 * abs(info["fp"] / info["fpp"])
    if case in ("keys_spread", "ties_straddle"):
        assert 0 < info["k"] < K - 1, info["k"]        # the chosen segment lies inside the sorted order
    if case == "keys_ulp":
        assert info["k"] < K - 1                       # t_cross and dt come from the smallest keys, which only the lowest digit orders
    if case == "nord1":
        assert K == 1 and ref[4] == 0.0
    if case == "tie_first":
        assert info["k"] == 3999 and ref[0] == 0.5


# ---------------------------------------------------------------------------------------------------------------- subspace sub-steps
SUB_OPS = list(range(12))
VEC_NAMES = ["vecc", "vecy", "lambda", "mu", "tmp", "tmp2", "yfb", "dvec", "brk", "xcp"]


def sub_inputs(n, dt, rng):
    V = {k: rng.standard_normal(n).astype(dt) for k in VEC_NAMES}
    x0 = rng.uniform(-1, 1, n).astype(dt)
    lo = (x0 - rng.uniform(0.1, 1, n)).astype(dt)
    hi = (x0 + rng.uniform(0.1, 1, n)).astype(dt)
    lo[::7], hi[::9] = -INF, INF
    cls = class_bytes(n, rng)
    l_, u_ = lo - x0, hi - x0
    # CLASSIFY ties: y == l with lambda >= 0 and < 0, y == u with mu >= 0 and < 0
    k = rng.integers(0, 8, n)
    fin_l, fin_u = np.isfinite(l_), np.isfinite(u_)
    for sel, src, mult, sign in ((k == 0, l_, "lambda", 1.0), (k == 1, l_, "lambda", -1.0), (k == 2, u_, "mu", 1.0),
                                 (k == 3, u_, "mu", -1.0)):
        sel = sel & (fin_l if src is l_ else fin_u)
        V["vecy"][sel] = src[sel]
        V[mult][sel] = sign * np.abs(V[mult][sel])
    sel = (k == 4) & fin_l                            # y == l with lambda exactly 0: still L (the rule is lambda >= 0)
    V["vecy"][sel] = l_[sel]
    V["lambda"][sel] = 0.0
    g = rng.standard_normal(n).astype(dt)
    drt = rng.standard_normal(n).astype(dt)
    return V, cls, x0, g, lo, hi, drt


def sub_reference(op, flag, V, cls, x0, g, lo, hi, drt, theta):
    """The contract of k_sub_step (lbfgsb_kernels.cuh) in numpy, computed in T.  Returns (vectors, cls, drt, out3, scales)."""
    dt = x0.dtype
    z = dt.type(0)
    V = {k: v.copy() for k, v in V.items()}
    cls = cls.copy()
    drt = drt.copy()
    free = (cls & lb.CLS_FREE) != 0
    l_, u_ = lo - x0, hi - x0
    out3 = [0.0, 0.0, 0.0]
    sc = {}
    if op == 0:
        drt = (V["xcp"] - x0).astype(dt)
        sc["drt"] = np.abs(V["xcp"]) + np.abs(x0)
        for k in ("lambda", "mu", "vecc", "vecy"):
            V[k] = np.zeros_like(V[k])
    elif op == 1:
        V["tmp"] = np.where(cls & lb.CLS_ACT, V["xcp"] - x0, z).astype(dt)
        sc["tmp"] = np.abs(V["xcp"]) + np.abs(x0)
    elif op == 2:
        sc["vecc"] = np.abs(V["vecc"]) + np.abs(g)
        V["vecc"] = np.where(free, V["vecc"] + g, V["vecc"]).astype(dt)
    elif op == 3:
        V["tmp"] = np.where(free, -V["vecc"], z).astype(dt)
    elif op == 4:
        out3[0] = np.sum(free & ((V["vecy"] < l_) | (V["vecy"] > u_)))
    elif op == 5:
        y = V["vecy"]
        isL = free & ((y < l_) | ((y == l_) & (V["lambda"] >= 0)))
        isU = free & ~isL & ((y > u_) | ((y == u_) & (V["mu"] >= 0)))
        isP = free & ~isL & ~isU
        base = cls & np.uint8(~(lb.SUB_L | lb.SUB_U | lb.SUB_P) & 0xFF)
        cls = np.where(isL, base | lb.SUB_L, np.where(isU, base | lb.SUB_U, np.where(isP, base | lb.SUB_P, cls))).astype(np.uint8)
        V["vecy"] = np.where(isL, l_, np.where(isU, u_, y)).astype(dt)
        V["mu"] = np.where(isL | isP, z, V["mu"]).astype(dt)
        V["lambda"] = np.where(isU | isP, z, V["lambda"]).astype(dt)
        out3 = [np.sum(isL), np.sum(isU), np.sum(isP)]
    elif op == 6:
        V["tmp"] = np.where(cls & lb.SUB_L, l_, np.where(cls & lb.SUB_U, u_, z)).astype(dt)
        sc["tmp"] = np.abs(lo) + np.abs(hi) + np.abs(x0)
    elif op == 7:
        V["tmp"] = np.where(cls & lb.SUB_P, -(V["vecc"] + (V["tmp2"] if flag else z)), z).astype(dt)
        sc["tmp"] = np.abs(V["vecc"]) + np.abs(V["tmp2"])
    elif op == 8:
        V["tmp"] = np.where(free, V["vecy"], z).astype(dt)
    elif op == 9:
        r = (V["tmp2"] + V["vecc"] + dt.type(theta) * V["vecy"]).astype(dt)
        sc["lambda"] = sc["mu"] = np.abs(V["tmp2"]) + np.abs(V["vecc"]) + abs(theta) * np.abs(V["vecy"])
        V["lambda"] = np.where(cls & lb.SUB_L, r, V["lambda"]).astype(dt)
        V["mu"] = np.where(cls & lb.SUB_U, -r, V["mu"]).astype(dt)
    elif op == 10:
        out3 = [np.sum(free & ((cls & lb.SUB_L) != 0) & (V["lambda"] < 0)), np.sum(free & ((cls & lb.SUB_U) != 0) & (V["mu"] < 0)),
                np.sum(free & ((cls & lb.SUB_P) != 0) & ((V["vecy"] < l_) | (V["vecy"] > u_)))]
    elif op == 11:
        y = V["yfb"] if flag & 2 else V["vecy"]
        if flag & 1:
            y = np.minimum(np.maximum(y, l_), u_)
        drt = np.where(free, y, drt).astype(dt)
        sc["drt"] = np.abs(lo) + np.abs(hi) + np.abs(x0) + np.abs(y)
        out3[0] = drt.astype(np.float64) * g.astype(np.float64)   # terms of the reduced dot
    return V, cls, drt, out3, sc


SUB_CASES = [(op, 0) for op in range(12) if op not in (7, 11)] + [(7, 0), (7, 1), (11, 0), (11, 1), (11, 2), (11, 3)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", SIZES)
def test_sub_steps(backend, n, dtype):
    """All 12 sub-steps on a workspace prefilled with random values: every vector, the class bytes and drt compared, the ones an op
    must not write required to keep their bits."""
    dt = np.dtype(dtype)
    rng = np.random.default_rng(5 * n + dt.itemsize)
    h = lb.History(backend, n, 2, dt)
    box = lb.Box(h)
    V0, cls0, x0, g, lo, hi, drt0 = sub_inputs(n, dt, rng)
    theta = 1.7
    X0, G, L, U = (dev(backend, v) for v in (x0, g, lo, hi))
    for op, flag in SUB_CASES:
        for k, name in enumerate(VEC_NAMES):
            box.set(k, V0[name])
        box.set("cls", cls0)
        D = dev(backend, drt0)
        o3 = out_buf(dt, 3)
        for k in range(3):
            o3[k] = -5.0
        backend.check(fn(backend, "box_sub_step", dt)(box.h, op, flag, X0.ptr, G.ptr, L.ptr, U.ptr, D.ptr, dt.type(theta), o3))
        V, cls, drt, out3, sc = sub_reference(op, flag, V0, cls0, x0, g, lo, hi, drt0, theta)
        where = (op, flag)
        assert np.array_equal(box.get("cls"), cls), where
        for k, name in enumerate(VEC_NAMES):
            got = box.get(k)
            if name in sc:
                assert_ew(got, V[name], sc[name], dt, (where, name))
            else:
                assert bits_equal(got, V[name]), (where, name)
        if "drt" in sc:
            assert_ew(D.get(), drt, sc["drt"], dt, (where, "drt"))
        else:
            assert bits_equal(D.get(), drt), (where, "drt")
        if op in (4, 5, 10):
            assert list(o3) == out3, (where, list(o3), out3)
        elif op == 11:
            assert abs(o3[0] - np.sum(out3[0])) <= red_tol(backend, out3[0], dt) and o3[1] == 0 and o3[2] == 0, where
        if op == 5:
            y, l_, u_ = V0["vecy"], lo - x0, hi - x0
            free = (cls0 & lb.CLS_FREE) != 0
            if n >= 2048:   # the tie rules are exercised at this size
                assert np.any(free & (y == l_) & (V0["lambda"] >= 0)) and np.any(free & (y == l_) & (V0["lambda"] < 0))
                assert np.any(free & (y == u_) & (V0["mu"] >= 0) & (y > l_)) and np.any(free & (y == l_) & (V0["lambda"] == 0))


# ---------------------------------------------------------------------------------------------------------------- errors
@pytest.mark.parametrize("dtype", DTYPES)
def test_invalid_calls_return_status_1(backend, dtype):
    dt = np.dtype(dtype)
    other = np.float32 if dt == np.float64 else np.float64
    n = 64
    h = make_history(backend, n, 3, dt, 2, np.random.default_rng(0))
    box = lb.Box(h)
    x = dev(backend, np.zeros(n, dt))
    xo = dev(backend, np.zeros(n, other))
    o5 = out_buf(other, 5)
    # a call of the other precision on this box
    assert fn(backend, "box_cauchy_breaks", other)(box.h, xo.ptr, xo.ptr, xo.ptr, xo.ptr, o5) == 1
    # m = 21 is beyond the bound-constrained path's limit
    h21 = lb.History(backend, n, 21, dt)
    out = C.c_void_p()
    assert backend.lib.lbfgs_b200_box_create(h21.h, C.byref(out)) == 1 and not out.value
    # nord = 0
    o = out_buf(dt, 5 + 4)
    M = np.eye(4, dtype=dt)
    p0 = np.zeros(4, dt)
    assert fn(backend, "box_cauchy_sweep", dt)(box.h, x.ptr, host_ptr(M), host_ptr(p0), dt.type(1), dt.type(1), 0, 0, o) == 1
    # an unknown sub-step
    assert fn(backend, "box_sub_step", dt)(box.h, 12, 0, x.ptr, x.ptr, x.ptr, x.ptr, x.ptr, dt.type(1), None) == 1
    # lincomb with c > 0 and no coefficients
    assert fn(backend, "hist_lincomb", dt)(h.h, box.h, dt.type(1), x.ptr, None, None, 0, x.ptr) == 1


# ---------------------------------------------------------------------------------------------------------------- fp32 L-BFGS-B end to end
@pytest.fixture(scope="module")
def solver_lib(backend, tmp_path_factory):
    """The driver's entry points: on the double, driver.cpp + mock_abi.cpp; on the GPU, liblbfgs_b200_driver.so."""
    if backend.kind == "gpu":
        return None
    so = _gxx(str(tmp_path_factory.mktemp("front_on_double") / "front_on_mock.so"),
              [os.path.join(ROOT, "lbfgspp_b200", "csrc", "driver.cpp"), os.path.join(ROOT, "tests", "cpp", "mock_abi.cpp")], True)
    return C.CDLL(so)


@pytest.mark.parametrize("objective", [po.OBJ_ROSENBROCK_PAIRED, po.OBJ_ROSENBROCK_CHAINED])
@pytest.mark.parametrize("n", [1000, 100_000])
def test_lbfgsb_float32_end_to_end(backend, solver_lib, orc, objective, n):
    """LBFGSBSolver<float> on the config-4 shape (x0 = 3, bounds [2, 4]).  There is no fp32 L-BFGS-B reference, so the result is held
    to properties: status ok, x feasible, and at the returned x, recomputed in float64:
      - the projected-gradient stop rule max(epsilon, epsilon_rel |x|) within a factor 500.  An fp32 solve also stops through the
        past/delta test as soon as f stops changing in fp32; on these problems that leaves a float64 projected gradient up to 110x
        the threshold (chained Rosenbrock, n = 1000, on the test double), so the factor bounds how far short of the rule it stops;
      - fx within 1e-2 relative of the fp64 solve on the same backend: both stop wherever the rules first hold, and at n = 1e5
        (threshold ~1e-2) the two stopping points differ by 0.4 % in fx (paired Rosenbrock, test double)."""
    prm = lb.LBFGSBParam()
    x0 = np.full(n, 3.0)
    r64 = lb.LBFGSBSolver(prm).minimize(objective, x0, 2.0, 4.0, lib=solver_lib)
    r32 = lb.LBFGSBSolver(prm, dtype=np.float32).minimize(objective, x0, 2.0, 4.0, lib=solver_lib)
    assert r64["status"] == "ok" and r32["status"] == "ok", (r64["msg"], r32["msg"])
    x = r32["x"].astype(np.float64)
    assert r32["x"].dtype == np.float32 and np.all(x >= 2.0) and np.all(x <= 4.0)
    _, g = orc.objective(objective, x)
    pg = np.max(np.abs(np.clip(x - g, 2.0, 4.0) - x))
    thresh = max(prm.epsilon, prm.epsilon_rel * float(np.linalg.norm(x)))
    assert pg <= 500 * thresh, (pg, thresh, r32["niter"])
    assert abs(r32["fx"] - r64["fx"]) <= 1e-2 * abs(r64["fx"]), (r32["fx"], r64["fx"])
