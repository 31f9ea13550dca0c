"""The final approximation of a bound-constrained solve on a CPU: LBFGSBSolver's whole-space members and the free-set members
(B_F = Z'BZ, H_F = (Z'BZ)^-1 and its square root, include/LBFGSpp/CompactForm.h compact_free_*) through the driver built on the test
double tests/cpp/mock_abi_box_hessian.cpp, against float64 dense references formed in numpy from the same pairs."""
import os
import subprocess

import numpy as np
import pytest

import lbfgspp_b200 as lb
from test_hessian_sample_cpu import bfgs_dense_inverse, normals
from test_hessian_whiten_cpu import CXX, ROOT, driver_on, history, rel_err

MOCK = os.path.join(ROOT, "tests", "cpp", "mock_abi_box_hessian.cpp")
FINAL = lb.CLS_FINAL


@pytest.fixture(scope="module")
def front(tmp_path_factory):
    return driver_on(tmp_path_factory, MOCK, "front_on_box_hessian_mock")


def free_cls(n, F, rng):
    """Class bytes with CLS_FINAL on F and random other bits everywhere (the masked passes read only CLS_FINAL)."""
    cls = rng.integers(0, 64, n).astype(np.uint8)
    cls[F] |= FINAL
    return cls


def dense(S, Y):
    c = S.shape[0]
    theta = (Y[0] @ Y[0] / (S[0] @ Y[0])) if c else 1.0
    H = bfgs_dense_inverse(S, Y, theta)
    return np.linalg.inv(H), H, theta


def free_sets(n, rng):
    return {"none": np.array([], dtype=int), "one": np.array([n // 2]), "three": np.sort(rng.choice(n, 3, replace=False)),
            "half": np.sort(rng.choice(n, n // 2, replace=False)), "all": np.arange(n)}


@pytest.mark.parametrize("c", [0, 4, 12, 20])
@pytest.mark.parametrize("fset", ["none", "one", "three", "half", "all"])
def test_free_set_algebra_matches_dense(front, c, fset):
    """Products, diagonals, log det, log densities and the square root on F against B[F, F] and inv(B[F, F]) of the dense BFGS matrix,
    and H_F against the conditioning identity H_FF - H_FA H_AA^-1 H_AF."""
    stats = pytest.importorskip("scipy.stats")
    n = 30
    rng = np.random.default_rng(17 * c + len(fset))
    S, Y, _ = history(n, c, 40 + c)
    B, H, theta = dense(S, Y)
    F = free_sets(n, rng)[fset]
    A = np.setdiff1d(np.arange(n), F)
    cls = free_cls(n, F, rng)
    BF = B[np.ix_(F, F)]
    HF = np.linalg.inv(BF) if F.size else np.zeros((0, 0))
    if F.size and A.size:
        cond = H[np.ix_(F, F)] - H[np.ix_(F, A)] @ np.linalg.solve(H[np.ix_(A, A)], H[np.ix_(A, F)])
        assert rel_err(cond, HF) <= 1e-9 * np.linalg.cond(H)
    tol = 1e-11 * max(1.0, np.linalg.cond(BF) if F.size else 1.0)
    run = lambda op, **kw: lb.box_hist_hessian(S[::-1], Y[::-1], op, cls=cls, m=max(c, 1), lib=front, **kw)   # pairs oldest first
    V = rng.standard_normal((5, n))
    for op, M in (("B", BF), ("H", HF)):
        r = run(op, V=V)
        assert r["nfree"] == F.size
        want = np.zeros_like(V)
        want[:, F] = V[:, F] @ M.T
        assert np.all(r["out"][:, A] == 0.0), op
        assert rel_err(r["out"], want) <= tol if F.size else np.all(r["out"] == 0.0), op
    for op, M in (("diagB", BF), ("diagH", HF)):
        d = run(op)["out"]
        assert np.all(d[A] == 0.0) and np.allclose(d[F], np.diag(M), rtol=tol, atol=0), op
    r = run("logdet")
    want = np.linalg.slogdet(HF)[1] if F.size else 0.0
    assert abs(r["logdet"] - want) <= 1e-10 * max(1.0, abs(want)) * max(1.0, np.linalg.cond(BF) if F.size else 1.0)
    mean = rng.standard_normal(n)
    X = mean + 0.3 * rng.standard_normal((4, n))
    lp = run("log_density", V=X, mean=mean)["out"]
    if F.size:
        assert np.allclose(lp, stats.multivariate_normal(mean=mean[F], cov=HF).logpdf(X[:, F]), rtol=tol, atol=tol * n)
    else:
        assert np.all(lp == 0.0)
    k = max(F.size, 1)
    draws = run("sample", k=k, mean=mean, seed=99, first=3)["out"]
    assert np.all(draws[:, A] == mean[A])
    if F.size:
        Z = np.stack([normals(99, 0, 3 + j, n) for j in range(k)])[:, F]
        L = np.linalg.solve(Z, draws[:, F] - mean[F]).T       # draws_F - mean_F = L Z_F
        assert rel_err(L, L.T) <= 1e-9 * np.linalg.cond(BF)
        assert rel_err(L @ L, HF) <= 1e-9 * np.linalg.cond(BF)


@pytest.mark.parametrize("scale", [1e8, 1e-8])
@pytest.mark.parametrize("c", [4, 12, 20])
@pytest.mark.parametrize("fset", ["three", "half", "all"])
def test_square_root_and_logdet_at_extreme_curvature(front, scale, c, fset):
    """Y scaled by 1e8 or 1e-8 (the curvature of a log-likelihood summed over many observations): the y and s columns of W then differ
    in size by that factor, and L_F L_F = H_F, log det H_F and the log densities must still hold, also against the whole space."""
    stats = pytest.importorskip("scipy.stats")
    n = 30
    rng = np.random.default_rng(int(7 * c + len(fset) + (scale > 1)))
    S, Y, _ = history(n, c, 90 + c)
    Y = Y * scale
    B, H, theta = dense(S, Y)
    F = free_sets(n, rng)[fset]
    cls = free_cls(n, F, rng)
    BF = B[np.ix_(F, F)]
    HF = np.linalg.inv(BF)
    cnd = np.linalg.cond(BF)
    run = lambda op, **kw: lb.box_hist_hessian(S[::-1], Y[::-1], op, cls=cls, m=c, lib=front, **kw)
    want = np.linalg.slogdet(HF)[1]
    assert abs(run("logdet")["logdet"] - want) <= 1e-10 * max(1.0, abs(want)) * cnd
    if fset == "all":
        whole = lb.box_hist_hessian(S[::-1], Y[::-1], "logdet", m=c, lib=front)["logdet"]
        assert abs(run("logdet")["logdet"] - whole) <= 1e-10 * max(1.0, abs(whole)) * cnd
    mean = rng.standard_normal(n)
    X = mean + rng.standard_normal((3, n)) / np.sqrt(np.diag(B))
    lp = run("log_density", V=X, mean=mean)["out"]
    assert np.allclose(lp, stats.multivariate_normal(mean=mean[F], cov=HF).logpdf(X[:, F]), rtol=1e-10 * cnd, atol=1e-10 * cnd * n)
    k = F.size
    draws = run("sample", k=k, mean=mean, seed=5, first=0)["out"]
    Z = np.stack([normals(5, 0, j, n) for j in range(k)])[:, F]
    L = np.linalg.solve(Z, draws[:, F] - mean[F]).T
    assert rel_err(L, L.T) <= 1e-9 * cnd
    assert rel_err(L @ L, HF) <= 1e-9 * cnd


@pytest.mark.parametrize("c", [0, 3, 9])
def test_fully_free_set_equals_the_whole_space(front, c):
    n = 20
    rng = np.random.default_rng(c)
    S, Y, _ = history(n, c, 70 + c)
    Sa, Ya = S[::-1], Y[::-1]
    cls = np.full(n, FINAL, dtype=np.uint8)
    V = rng.standard_normal((3, n))
    mean = rng.standard_normal(n)
    X = mean + rng.standard_normal((3, n))
    for op, kw in (("B", dict(V=V)), ("H", dict(V=V)), ("diagB", {}), ("diagH", {}), ("log_density", dict(V=X, mean=mean)), ("logdet", {})):
        free = lb.box_hist_hessian(Sa, Ya, op, cls=cls, m=max(c, 1), lib=front, **kw)
        whole = lb.box_hist_hessian(Sa, Ya, op, m=max(c, 1), lib=front, **kw)
        assert rel_err(np.atleast_1d(free["out"]), np.atleast_1d(whole["out"])) <= 1e-12, op
        assert abs(free["logdet"] - whole["logdet"]) <= 1e-12 * max(1.0, abs(whole["logdet"])), op


BOUNDED = [("chained Rosenbrock in [2, 4]", lb.OBJ_ROSENBROCK_CHAINED, 12, 2.0, 4.0),
           ("paired Rosenbrock in [2, 4]", lb.OBJ_ROSENBROCK_PAIRED, 12, 2.0, 4.0),
           ("quadratic in [-0.5, 0.3]", lb.OBJ_QUAD_SHIFT, 16, -0.5, 0.3)]


@pytest.mark.parametrize("case", BOUNDED, ids=lambda c: c[0])
@pytest.mark.parametrize("m", [3, 8])
def test_solver_members_match_the_dense_matrices(front, case, m):
    """LBFGSBSolver on the test double: every whole-space member against the dense B and H of the same solve, and every free member
    against B[F, F] of it, with F from the classification rule applied to the returned x."""
    stats = pytest.importorskip("scipy.stats")
    name, obj, n, lo, hi = case
    prm = lb.LBFGSBParam(m=m)
    x0 = np.full(n, 0.5 * (lo + hi)) + np.linspace(-0.1, 0.1, n)
    call = lambda op, **kw: lb.box_solve_hessian(obj, x0, lo, hi, op, param=prm, lib=front, **kw)
    Bd, Hd = call("denseB", free=False)["out"], call("denseH", free=False)["out"]
    x = call("denseB", free=False)["x"]
    tol = 1e-10 * max(1.0, np.linalg.cond(Bd))
    assert rel_err(Bd @ Hd, np.eye(n)) <= tol
    V = np.random.default_rng(n + m).standard_normal((4, n))
    assert rel_err(call("B", V=V, free=False)["out"], V @ Bd.T) <= tol
    assert rel_err(call("H", V=V, free=False)["out"], V @ Hd.T) <= tol
    assert np.allclose(call("diagH", free=False)["out"], np.diag(Hd), rtol=tol, atol=0)
    r = call("L", V=np.eye(n), free=False)
    L = r["out"].T
    assert rel_err(L @ L.T, Hd) <= tol
    assert abs(r["logdet"] - np.linalg.slogdet(Hd)[1]) <= tol * n
    P = x + 0.05 * V
    assert np.allclose(call("log_density", V=P, free=False)["out"], stats.multivariate_normal(mean=x, cov=Hd).logpdf(P), rtol=tol, atol=tol * n)
    # the free set of the returned point
    eps = 4 * np.finfo(np.float64).eps
    fixed = (x <= lo + eps * max(1, abs(lo))) | (x >= hi - eps * max(1, abs(hi)))
    F = np.flatnonzero(~fixed)
    r = call("H", V=V)
    assert r["nfree"] == F.size and np.array_equal(r["x"], x)
    HF = np.linalg.inv(Bd[np.ix_(F, F)])
    want = np.zeros_like(V)
    want[:, F] = V[:, F] @ HF.T
    assert rel_err(r["out"], want) <= tol, name
    d = call("diagH")["out"]
    assert np.allclose(d[F], np.diag(HF), rtol=tol, atol=0) and np.all(d[fixed] == 0)
    assert abs(call("logdet")["logdet"] - np.linalg.slogdet(HF)[1]) <= tol * n


def test_classification_and_error_paths(tmp_path):
    """The free-set rule on the test double (exact bounds, one ulp inside, lb == ub, infinite bounds) and the exceptions of the front:
    std::logic_error before minimize() and before final_approx_free_set, std::invalid_argument for bad sizes."""
    src = tmp_path / "checks.cpp"
    src.write_text(r"""
#include <cmath>
#include <cstdio>
#include <limits>
#include <LBFGSB.h>
#include <LBFGSpp/DeviceObjectives.h>
using namespace LBFGSpp;
template <class T> int classify()
{
    const T inf = std::numeric_limits<T>::infinity(), e = std::numeric_limits<T>::epsilon();
    const T x[] = {T(2), std::nextafter(T(2), T(3)), T(2) + T(8) * e * T(2), T(4), std::nextafter(T(4), T(3)), T(1), T(1), T(-5), T(0.5)};
    const T l[] = {T(2), T(2), T(2), T(2), T(2), T(1), -inf, -inf, T(0)};
    const T u[] = {T(4), T(4), T(4), T(4), T(4), T(1), inf, inf, T(1)};
    lbfgs_b200_ctx* ctx = nullptr;
    lbfgs_b200_ctx_create(&ctx, 0, nullptr);
    lbfgs_b200_hist* h = nullptr;
    lbfgs_b200_hist_create(ctx, &h, 9, 2, int(sizeof(T)));
    lbfgs_b200_box* b = nullptr;
    lbfgs_b200_box_create(h, &b);
    int64_t nf = -1;
    detail::BoxAbi<T>::final_classes(b, x, l, u, T(4) * e, &nf);
    const unsigned char* cls = lbfgs_b200_box_classes(b);
    std::printf("%s:", sizeof(T) == 8 ? "f64" : "f32");
    for (int i = 0; i < 9; i++) std::printf(" %d", (cls[i] & LBFGS_B200_CLS_FINAL) ? 1 : 0);
    std::printf(" nfree %lld\n", (long long)nf);
    lbfgs_b200_box_destroy(b);
    lbfgs_b200_hist_destroy(h);
    lbfgs_b200_ctx_destroy(ctx);
    return 0;
}
template <class F> void expect(const char* what, F f)
{
    const char* got = "ok";
    try { f(); }
    catch (const std::invalid_argument&) { got = "invalid_argument"; }
    catch (const std::logic_error&) { got = "logic_error"; }
    catch (const std::runtime_error&) { got = "runtime_error"; }
    std::printf("%s: %s\n", what, got);
}
int main()
{
    classify<double>();
    classify<float>();
    Device dev(0);
    typedef DeviceVector<double> V;
    LBFGSBParam<double> prm;
    LBFGSBSolver<double> s(prm);
    V x(dev), lo(dev), hi(dev), O(dev), X(dev);
    std::vector<double> h0(6, 0.5), hl(6, 0.0), hh(6, 0.75);
    x.copy_from_host(h0.data(), 6); lo.copy_from_host(hl.data(), 6); hi.copy_from_host(hh.data(), 6); X.copy_from_host(h0.data(), 6);
    expect("before minimize, dense", [&] { s.final_approx_hessian(); });
    expect("before minimize, times", [&] { s.final_approx_inverse_hessian_times(X, O); });
    expect("before minimize, diagonal", [&] { s.final_approx_inverse_hessian_diagonal(O); });
    expect("before minimize, sample", [&] { s.final_approx_sample(x, 1, 0, 2, O); });
    expect("before minimize, logdet", [&] { s.final_approx_inverse_hessian_logdet(); });
    expect("before minimize, log density", [&] { s.final_approx_log_density(x, X); });
    expect("before minimize, free set", [&] { s.final_approx_free_set(x, lo, hi); });
    expect("before minimize, free times", [&] { s.final_approx_free_inverse_hessian_times(X, O); });
    BuiltinObjective<double> obj(LBFGS_B200_OBJ_ROSENBROCK_CHAINED);
    double fx = 0;
    s.minimize(obj, x, fx, lo, hi);
    expect("before free set, times", [&] { s.final_approx_free_hessian_times(X, O); });
    expect("before free set, diagonal", [&] { s.final_approx_free_inverse_hessian_diagonal(O); });
    expect("before free set, logdet", [&] { s.final_approx_free_inverse_hessian_logdet(); });
    expect("before free set, sample", [&] { s.final_approx_free_sample(x, 1, 0, 2, O); });
    expect("before free set, log density", [&] { s.final_approx_free_log_density(x, X); });
    expect("after minimize, whole times", [&] { s.final_approx_hessian_times(X, O); });
    expect("free set", [&] { s.final_approx_free_set(x, lo, hi); });
    expect("free times", [&] { s.final_approx_free_hessian_times(X, O); });
    expect("free log density", [&] { s.final_approx_free_log_density(x, X); });
    V Xbad(dev);
    Xbad.copy_from_host(h0.data(), 5);
    expect("free times, V of n - 1", [&] { s.final_approx_free_hessian_times(Xbad, O); });
    expect("free log density, mean of n - 1", [&] { s.final_approx_free_log_density(Xbad, X); });
    expect("free sample, k = 0", [&] { s.final_approx_free_sample(x, 1, 0, 0, O); });
    s.minimize(obj, x, fx, lo, hi);
    expect("after a new minimize, free times", [&] { s.final_approx_free_hessian_times(X, O); });
    std::printf("box hessian checks done\n");
}
""")
    exe = str(tmp_path / "checks")
    subprocess.run(CXX + ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "lbfgspp_b200", "csrc"), "-o", exe, str(src), MOCK,
                          "-pthread"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.endswith("box hessian checks done\n"), r.stdout + r.stderr
    lines = r.stdout.splitlines()
    # x on lb, one ulp inside lb (fixed by the tolerance), 16 eps inside (free), on ub, one ulp inside ub, lb == ub, free with
    # infinite bounds (twice), interior
    assert lines[0] == "f64: 0 0 1 0 0 0 1 1 1 nfree 4"
    assert lines[1] == "f32: 0 0 1 0 0 0 1 1 1 nfree 4"
    got = dict(line.split(": ", 1) for line in lines[2:-1])
    assert got == {
        "before minimize, dense": "logic_error", "before minimize, times": "logic_error", "before minimize, diagonal": "logic_error",
        "before minimize, sample": "logic_error", "before minimize, logdet": "logic_error", "before minimize, log density": "logic_error",
        "before minimize, free set": "logic_error", "before minimize, free times": "logic_error",
        "before free set, times": "logic_error", "before free set, diagonal": "logic_error", "before free set, logdet": "logic_error",
        "before free set, sample": "logic_error", "before free set, log density": "logic_error",
        "after minimize, whole times": "ok", "free set": "ok", "free times": "ok", "free log density": "ok",
        "free times, V of n - 1": "invalid_argument", "free log density, mean of n - 1": "invalid_argument",
        "free sample, k = 0": "invalid_argument", "after a new minimize, free times": "logic_error"}


def test_empty_history_after_a_reset_is_a_scaled_identity(front):
    """c = 0: B_F = theta I and H_F = I / theta on F (theta = 1 for an empty ring)."""
    n = 8
    cls = np.zeros(n, dtype=np.uint8)
    cls[[1, 4, 5]] = FINAL
    V = np.random.default_rng(3).standard_normal((2, n))
    want = np.zeros_like(V)
    want[:, [1, 4, 5]] = V[:, [1, 4, 5]]
    for op in ("B", "H"):
        assert np.array_equal(lb.box_hist_hessian(np.zeros((0, n)), np.zeros((0, n)), op, cls=cls, m=2, V=V, lib=front)["out"], want)


def test_nonpositive_curvature_is_reported(front):
    S, Y = np.ones((1, 4)), -np.ones((1, 4))
    cls = np.full(4, FINAL, dtype=np.uint8)
    with pytest.raises(RuntimeError, match="positive definite|singular"):
        lb.box_hist_hessian(S, Y, "sample", cls=cls, k=2, mean=np.zeros(4), lib=front)
    assert np.isnan(lb.box_hist_hessian(S, Y, "logdet", cls=cls, lib=front)["logdet"])
    assert np.all(np.isnan(lb.box_hist_hessian(S, Y, "log_density", cls=cls, V=np.eye(4), mean=np.zeros(4), lib=front)["out"]))
    for op, kw in (("H", dict(V=np.eye(4))), ("diagH", {})):    # H_F products and diag H_F refuse what the sampler refuses
        with pytest.raises(RuntimeError, match="positive definite"):
            lb.box_hist_hessian(S, Y, op, cls=cls, lib=front, **kw)


def test_driver_reports_the_missing_entry_points(tmp_path_factory):
    """Against the test double without the free-set passes the driver library loads and names them."""
    lib = driver_on(tmp_path_factory, os.path.join(ROOT, "tests", "cpp", "mock_abi_hessian_whiten.cpp"), "drv_on_whiten_mock")
    for dt in (np.float64, np.float32):
        with pytest.raises(RuntimeError, match="lbfgs_b200_box_final_classes_"):
            lb.box_solve_hessian(lb.OBJ_QUAD_SHIFT, np.zeros(4), -1.0, 1.0, "diagH", dtype=dt, lib=lib)
    with pytest.raises(RuntimeError, match="lbfgs_b200_hist_.*_masked_"):
        lb.box_hist_hessian(np.ones((1, 4)), np.ones((1, 4)), "H", cls=np.full(4, FINAL, np.uint8), V=np.eye(4), lib=lib)
    r = lb.box_solve_hessian(lb.OBJ_QUAD_SHIFT, np.zeros(4), -1.0, 1.0, "diagH", free=False, lib=lib)   # the whole space still works
    assert r["out"].shape == (4,)


def test_front_members_compile_with_werror(tmp_path):
    src = tmp_path / "front.cpp"
    src.write_text("""
#include <LBFGSB.h>
using namespace LBFGSpp;
template <class S> void f(LBFGSBSolver<S>& s, BFGSMat<S, true>& m, DeviceVector<S>& V, DeviceVector<S>& O, const unsigned char* cls)
{
    (void)s.final_approx_hessian(); (void)s.final_approx_inverse_hessian();
    s.final_approx_hessian_times(V, O); s.final_approx_inverse_hessian_times(V, O);
    s.final_approx_hessian_diagonal(O); s.final_approx_inverse_hessian_diagonal(O);
    s.final_approx_inverse_hessian_factor_times(V, O); s.final_approx_inverse_hessian_factor_transpose_times(V, O);
    s.final_approx_inverse_hessian_factor_solve(V, O); s.final_approx_inverse_hessian_factor_transpose_solve(V, O);
    s.final_approx_sample(V, 1ull, 0u, 2, O); (void)s.final_approx_inverse_hessian_logdet(); (void)s.final_approx_log_density(V, O);
    (void)s.final_approx_free_set(V, V, O); (void)s.final_approx_free_set(V, V, O, S(0));
    s.final_approx_free_hessian_times(V, O); s.final_approx_free_inverse_hessian_times(V, O);
    s.final_approx_free_hessian_diagonal(O); s.final_approx_free_inverse_hessian_diagonal(O);
    (void)s.final_approx_free_inverse_hessian_logdet(); s.final_approx_free_sample(V, 1ull, 0u, 2, O);
    (void)s.final_approx_free_log_density(V, O);
    (void)m.free_set(V, V, O, S(0)); (void)m.free_set_classes(cls); (void)m.free_count();
    m.free_hessian_times(V, 1, O); m.free_inverse_hessian_times(V, 1, O); m.free_hessian_diagonal(O); m.free_inverse_hessian_diagonal(O);
    (void)m.free_inverse_hessian_logdet(); m.free_sample(&V, 1ull, 0u, 0u, 1, O); (void)m.free_log_density(V, O, 1);
}
template void f<double>(LBFGSBSolver<double>&, BFGSMat<double, true>&, DeviceVector<double>&, DeviceVector<double>&, const unsigned char*);
template void f<float>(LBFGSBSolver<float>&, BFGSMat<float, true>&, DeviceVector<float>&, DeviceVector<float>&, const unsigned char*);
""")
    subprocess.run(CXX + ["-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", "-o", str(tmp_path / "front.o"), str(src)], check=True)
