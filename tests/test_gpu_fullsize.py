"""GPU checks at BASELINE config 2's full size (paired Rosenbrock n = 1e7, fp64, m = 10): the solve against the frozen CPU
run of the unmodified reference headers (tests/golden/c2_full.json, generator tests/golden/make_c2_full.py), and apply_Hv
through properties that need no CPU run of that size: the secant equation H y_new = s_new, linearity, agreement of the two
independent device algorithms (literal two-loop / Gram form) and run-to-run determinism."""
import json
import os

import numpy as np
import pytest

import lbfgspp_b200 as lb

pytestmark = pytest.mark.gpu

N, M = 10_000_000, 10
HERE = os.path.dirname(os.path.abspath(__file__))


def test_config2_full_size_solve_matches_reference_cpu_run():
    with open(os.path.join(HERE, "golden", "c2_full.json")) as fh:
        c = json.load(fh)
    assert (c["n"], c["m"]) == (N, M)
    g = lb.LBFGSSolver(lb.LBFGSParam(m=M), "MoreThuente").minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(N))
    assert g["status"] == "ok"
    assert (g["niter"], g["nfev"]) == (c["niter"], c["nfev"])
    fx_cpu = float.fromhex(c["fx"])
    assert abs(g["fx"] - fx_cpu) <= 1e-10 * max(1.0, abs(fx_cpu))
    x = g["x"]
    # x0 = 0 makes this a replicated 2-D problem: every pair must carry exactly the same two numbers
    assert np.all(x[0::2] == x[0]) and np.all(x[1::2] == x[1])
    assert abs(x[0] - float.fromhex(c["x_even"])) <= 1e-8 and abs(x[1] - float.fromhex(c["x_odd"])) <= 1e-8
    trace_cpu = np.array([float.fromhex(v) for v in c["trace"]])
    k = np.arange(trace_cpu.size)
    tol = np.minimum(1e-10 * 4.0 ** k, 1e-3) * np.maximum(np.abs(trace_cpu), 1e-6 * abs(trace_cpu[0]))
    assert np.all(np.abs(g["trace"] - trace_cpu) <= tol)


def test_apply_Hv_full_size_properties(gpu_ctx):
    rng = np.random.default_rng(0)
    hist = lb.History(gpu_ctx, N, M)
    s = y = None
    for _ in range(M + 2):  # two more than the ring holds: the oldest pairs are overwritten
        s = rng.standard_normal(N)
        y = s + 0.1 * rng.standard_normal(N)
        ds, dy = lb.DeviceArray(gpu_ctx, s), lb.DeviceArray(gpu_ctx, y)
        hist.add(ds, dy)
        del ds, dy
    assert hist.ncorr == M
    dy = lb.DeviceArray(gpu_ctx, y)
    res = gpu_ctx.empty(N)
    s_scale = np.max(np.abs(s))
    for algo in (lb.HV_TWO_LOOP, lb.HV_GRAM):
        hist.apply_Hv(dy, 1.0, res, algo)
        assert np.max(np.abs(res.get() - s)) <= 1e-10 * s_scale      # secant equation of the BFGS inverse update
    v1, v2 = rng.standard_normal(N), rng.standard_normal(N)
    a, b = 2.5, -0.75
    out = {}
    for algo in (lb.HV_TWO_LOOP, lb.HV_GRAM):
        h = []
        for v in (v1, v2, a * v1 + b * v2):
            dv = lb.DeviceArray(gpu_ctx, v)
            hist.apply_Hv(dv, -1.0, res, algo)
            h.append(res.get())
            del dv
        scale = np.max(np.abs(h[2])) + 1.0
        assert np.max(np.abs(h[2] - (a * h[0] + b * h[1]))) <= 1e-11 * scale   # linearity
        out[algo] = h[2]
    scale = np.max(np.abs(out[lb.HV_GRAM])) + 1.0
    assert np.max(np.abs(out[lb.HV_TWO_LOOP] - out[lb.HV_GRAM])) <= 1e-11 * scale  # two device algorithms agree
    dv = lb.DeviceArray(gpu_ctx, a * v1 + b * v2)
    hist.apply_Hv(dv, -1.0, res, lb.HV_GRAM)
    assert np.array_equal(res.get(), out[lb.HV_GRAM])                # bitwise repeatable


# ---------------------------------------------------------------------------------------------------------------------------------
# BASELINE configs 3, 4, 5 at their stated sizes against the frozen CPU runs of tests/golden/make_fullsize.py: the unmodified reference
# headers (sequential sums) and the restatement under two more summation orders.  Where the reference's own result depends on the
# summation order (C3's last line search, C5's 150-400-iteration random starts) the test holds the GPU to what is order-independent
# (the trace of f while it is well conditioned, the optimum, the error text) and to the spread the CPU columns show among
# themselves; with LBFGSPP_PARITY_REPORT=<file.json> set, every comparison is also written to that file.
# ---------------------------------------------------------------------------------------------------------------------------------
def _golden(name):
    with open(os.path.join(HERE, "golden", name)) as fh:
        return json.load(fh)


def _report(key, value):
    path = os.environ.get("LBFGSPP_PARITY_REPORT")
    if not path:
        return
    path = os.path.abspath(path)
    try:
        os.makedirs(os.path.dirname(path), exist_ok=True)
        data = {}
        if os.path.exists(path):
            with open(path) as fh:
                data = json.load(fh)
        data[key] = value
        with open(path, "w") as fh:
            json.dump(data, fh, indent=1)
    except OSError:
        pass


@pytest.mark.parametrize("loop", ["resident", "host"])
def test_config3_full_size_quadratic_m20_bracketing(loop):
    import pyoracle as po
    c = _golden("c3_full.json")
    n = c["n"]
    d, b, xs = po.quad_tridiag_data(n, kappa=1e3, seed=0)
    g = lb.LBFGSSolver(lb.LBFGSParam(m=c["m"]), "Bracketing", resident=(loop == "resident")).minimize(lb.OBJ_QUAD_TRIDIAG, np.zeros(n), data0=d, data1=b)
    cols = c["columns"]
    ref = cols["ref_headers"]
    tr_ref = np.array([float.fromhex(v) for v in ref["trace"]])
    tr = g["trace"]
    # (1) evaluation by evaluation while the run is well conditioned: the CPU columns agree to 1e-12 there
    k = min(150, tr.size, tr_ref.size)
    rel = np.abs(tr[:k] - tr_ref[:k]) / np.abs(tr_ref[:k])
    assert k == 150 and np.max(rel[1:]) <= 1e-10, np.max(rel[1:])
    # (2) the optimum: <= 1e-10 relative on f (north star), x* recovered like the CPU does
    f_best_ref = min(tr_ref)
    assert abs(min(tr) - f_best_ref) <= 1e-10 * abs(f_best_ref)
    assert np.max(np.abs(g["x"] - xs)) <= 2.0 * max(float.fromhex(v["x_err_inf"]) for v in cols.values())
    # (3) the end of the run.  Every CPU column ends in the reference's own LineSearchBracketing exception at the noise floor of f
    # (|f| = 7e7: the Armijo test compares differences of 1e-8) after 219..224 evaluations; which evaluation trips it depends on
    # the summation order.  The GPU must end the same way or converge, within the CPU columns' spread of evaluations +- 10 %.
    nfev_cpu = [v["nfev"] for v in cols.values()]
    assert g["status"] in ("ok", "runtime_error")
    if g["status"] == "runtime_error":
        assert g["msg"] == ref["msg"]
    assert 0.9 * min(nfev_cpu) <= g["nfev"] <= 1.1 * max(nfev_cpu), (g["nfev"], nfev_cpu)
    _report("C3_" + loop, dict(gpu=dict(status=g["status"], msg=g["msg"], niter=g["niter"], nfev=g["nfev"], f_best=float(min(tr)),
                                         x_err_inf=float(np.max(np.abs(g["x"] - xs))), trace_rel_err_first150=float(np.max(rel[1:]))),
                               cpu={k2: dict(status=v["status"], nfev=v["nfev"], f_best=min(float.fromhex(t) for t in v["trace"]),
                                             x_err_inf=float.fromhex(v["x_err_inf"])) for k2, v in cols.items()}))


@pytest.mark.parametrize("objective", ["paired", "chained"])
@pytest.mark.parametrize("tag", ["default", "epsrel0"])
def test_config4_full_size_box_2_4(objective, tag):
    c = _golden("c4_full.json")
    n = c["n"]
    cols = c["runs"][objective][tag]
    ref = cols["ref_headers"]
    assert all((v["niter"], v["nfev"], v["fx"]) == (ref["niter"], ref["nfev"], ref["fx"]) for v in cols.values())   # order-independent here
    kind = lb.OBJ_ROSENBROCK_PAIRED if objective == "paired" else lb.OBJ_ROSENBROCK_CHAINED
    prm = lb.LBFGSBParam() if tag == "default" else lb.LBFGSBParam(epsilon_rel=0.0)
    g = lb.LBFGSBSolver(prm).minimize(kind, np.full(n, 3.0), 2.0, 4.0)
    fx_ref = float.fromhex(ref["fx"])
    _report("C4_%s_%s" % (objective, tag), dict(gpu=dict(status=g["status"], niter=g["niter"], nfev=g["nfev"], fx=g["fx"],
                                                          n_at_lb=int(np.sum(g["x"] == 2.0)), n_at_ub=int(np.sum(g["x"] == 4.0))),
                                                 cpu=dict(niter=ref["niter"], nfev=ref["nfev"], fx=fx_ref, n_at_lb=ref["n_at_lb"], n_at_ub=ref["n_at_ub"])))
    assert g["status"] == ref["status"] == "ok"
    assert g["niter"] == ref["niter"]
    assert abs(g["nfev"] - ref["nfev"]) <= 1                                 # same bar as tests/test_gpu_lbfgsb.py
    assert abs(g["fx"] - fx_ref) <= 1e-9 * max(1.0, abs(fx_ref))
    x = g["x"]
    assert np.all(x >= 2.0) and np.all(x <= 4.0)
    assert (int(np.sum(x == 2.0)), int(np.sum(x == 4.0))) == (ref["n_at_lb"], ref["n_at_ub"])
    head = np.array([float.fromhex(v) for v in ref["x_head"]]); tail = np.array([float.fromhex(v) for v in ref["x_tail"]])
    assert np.max(np.abs(x[:8] - head)) <= 1e-6 and np.max(np.abs(x[-8:] - tail)) <= 1e-6
    assert abs(np.sum(x) - float.fromhex(ref["x_sum"])) <= 1e-6 * n


def test_config5_full_size_batch_of_64():
    """One persistent kernel launch for the 64 problems of BASELINE config 5 at n = 1e6.  These are 140-620-iteration runs from
    random starts in which the reference's own iteration count moves by 15 % on average (up to a factor 1.45) between summation
    orders, and the distance to x* at the stop by up to 50x (columns of c5_full.json: the stop rule gnorm <= 1e-5 |x| is met at
    different points of a flat valley).  So the per-seed table is reported (LBFGSPP_PARITY_REPORT) and the
    assertions are: (a) every problem stops on the reference's own criterion, near x* = 1; (b) per seed the GPU count lies within
    the CPU columns' range widened by the factor the columns show among themselves; (c) over the 64 seeds the mean count is
    within 8 % of the CPU columns' mean (2.7 % apart among themselves); (d) a batch member is bit-identical to the same problem
    solved alone."""
    c = _golden("c5_full.json")
    n, B = c["n"], c["B"]
    X0 = np.stack([np.random.default_rng(p["seed"]).uniform(-1, 1, n) for p in c["problems"]])
    bs = lb.BatchSession(lb.OBJ_ROSENBROCK_PAIRED, X0, lb.LBFGSParam(m=c["m"]), "MoreThuente")
    res, X, secs = bs.solve()
    bs.close()
    table = []
    cpu_means = []
    for b, p in enumerate(c["problems"]):
        cols = p["columns"]
        it_cpu = [v["niter"] for v in cols.values()]
        r = res[b]
        xerr = float(np.max(np.abs(X[b] - 1.0)))
        table.append(dict(seed=p["seed"], gpu=dict(status=r["status"], niter=r["niter"], nfev=r["nfev"], fx=r["fx"], gnorm=r["gnorm"], x_err_inf=xerr),
                          cpu={k: dict(niter=v["niter"], nfev=v["nfev"], fx=float.fromhex(v["fx"]), x_err_inf=float.fromhex(v["x_err_inf"]))
                               for k, v in cols.items()}))
        cpu_means.append(np.mean(it_cpu))
        assert r["status"] == "ok"
        assert r["gnorm"] <= 1e-5 * np.linalg.norm(X[b]) * (1 + 1e-12)            # LBFGS.h:137-140 with the default epsilon_rel
        assert xerr <= 0.05 and r["fx"] <= 1e-3, (p["seed"], xerr, r["fx"])
        assert min(it_cpu) / 1.5 <= r["niter"] <= 1.5 * max(it_cpu), (p["seed"], r["niter"], it_cpu)
    mean_gpu = np.mean([r["niter"] for r in res])
    _report("C5_batch64", dict(seconds=secs, mean_niter_gpu=float(mean_gpu), mean_niter_cpu_columns=float(np.mean(cpu_means)), problems=table))
    assert abs(mean_gpu - np.mean(cpu_means)) <= 0.08 * np.mean(cpu_means), (mean_gpu, np.mean(cpu_means))
    for b in (0, 17, 63):
        one = lb.LBFGSSolver(lb.LBFGSParam(m=c["m"]), "MoreThuente", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, X0[b])
        assert (one["niter"], one["nfev"], one["fx"]) == (res[b]["niter"], res[b]["nfev"], res[b]["fx"])
        assert np.array_equal(one["x"], X[b])
