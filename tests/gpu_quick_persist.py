"""Development check of the device-resident (persistent kernel) solve on a GPU: parity against the CPU checker at a few sizes,
timing at config 2's size, batch == lone solves.  Not collected by pytest (no test_ prefix); run: python tests/gpu_quick_persist.py"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import lbfgspp_b200 as lb  # noqa: E402
import pyoracle as po  # noqa: E402

orc = po.Oracle("orc")
LSN = {"Backtracking": 0, "Bracketing": 1, "NocedalWright": 2, "MoreThuente": 3}


def show(tag, g, c=None):
    line = "%-40s %s niter=%d nfev=%d fx=%.15e launches=%s" % (tag, g["status"], g["niter"], g["nfev"], g["fx"], g.get("launches"))
    if c is not None:
        line += "  | cpu %s niter=%d nfev=%d fx=%.15e dx=%.2e" % (c["status"], c["niter"], c["nfev"], c["fx"], np.max(np.abs(g["x"] - c["x"])))
    print(line, flush=True)


PERF_ONLY = "--perf" in sys.argv
if "--one" in sys.argv:   # under ncu: 3 warm solves + 1 at config 2's size, nothing else
    sess = lb.Session(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(10_000_000), lb.LBFGSParam(m=10), "MoreThuente", resident=True)
    for _ in range(4):
        r = sess.solve()
    print(r, sess.profile())
    sess.close()
    sys.exit(0)
for n in (() if PERF_ONLY else (10, 4098, 100000)):
    for ls in LSN:
        prm = lb.LBFGSParam(m=10 if n > 10 else 6)
        g = lb.LBFGSSolver(prm, ls, resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n))
        c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, np.zeros(n), LSN[ls], orc.default_param(m=prm.m))
        show("paired n=%d %s" % (n, ls), g, c)
if not PERF_ONLY:
    n = 5000
    d, b, _ = po.quad_tridiag_data(n, seed=1)
    g = lb.LBFGSSolver(lb.LBFGSParam(m=20), "Bracketing", resident=True).minimize(lb.OBJ_QUAD_TRIDIAG, np.zeros(n), data0=d, data1=b)
    c = orc.lbfgs(po.OBJ_QUAD_TRIDIAG, np.zeros(n), 1, orc.default_param(m=20), data0=d, data1=b)
    show("tridiag n=5000 m=20 Bracketing", g, c)
    g = lb.LBFGSSolver(lb.LBFGSParam(), "NocedalWright", resident=True).minimize(lb.OBJ_ROSENBROCK_CHAINED, np.full(300, 1.3))
    c = orc.lbfgs(po.OBJ_ROSENBROCK_CHAINED, np.full(300, 1.3), 2, orc.default_param())
    show("chained n=300 NW", g, c)
    g = lb.LBFGSSolver(lb.LBFGSParam(), "NocedalWright", resident=True).minimize(lb.OBJ_QUAD_SHIFT, np.zeros(10))
    show("quad_shift n=10", g)
    g = lb.LBFGSSolver(lb.LBFGSParam(max_linesearch=1), "Backtracking", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(12))
    show("error path (max_linesearch=1, BT)", g)
    print("   msg:", g["msg"])
    x0 = np.random.default_rng(3).uniform(-1, 1, 2000)
    g = lb.LBFGSSolver(lb.LBFGSParam(m=7, max_linesearch=64), "MoreThuente", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0)
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, 3, orc.default_param(m=7, max_linesearch=64))
    show("random start n=2000 MT", g, c)

# config 2 size: resident vs host-driven
for n in (1_000_000, 10_000_000):
    for resident in (True, False):
        sess = lb.Session(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n), lb.LBFGSParam(m=10), "MoreThuente", resident=resident)
        for _ in range(3):
            r = sess.solve()
        t0 = time.perf_counter()
        K = 10
        for _ in range(K):
            r = sess.solve()
        dt = (time.perf_counter() - t0) / K
        print("n=%d resident=%s: %d it / %d fev, fx=%.6e, %.3f ms per solve, %.1f it/s, launches=%d" % (
            n, resident, r["niter"], r["nfev"], r["fx"], dt * 1e3, r["niter"] / dt, r["launches"]), flush=True)
        prof = sess.profile()
        if prof:
            print('   kernel_ms=%.3f sync_ms=%.3f (waiting for the last CTA %.3f)' % (prof['kernel_ms'], prof['sync_ms'], prof['wait_last_cta_ms']))
            for k, v in prof['ops'].items():
                print('   %-14s rounds=%3d ms=%.3f  %.0f GB/s' % (k, v['rounds'], v['ms'], v['alg_bytes'] / max(v['ms'], 1e-9) / 1e6))
        sess.close()

# batch == lone solves
B, n = 8, 4096
X0 = np.stack([np.random.default_rng(1000 + b).uniform(-1, 1, n) for b in range(B)])
bs = lb.BatchSession(lb.OBJ_ROSENBROCK_PAIRED, X0, lb.LBFGSParam(m=10), "MoreThuente")
res, X, secs = bs.solve()
for b in range(B):
    one = lb.LBFGSSolver(lb.LBFGSParam(m=10), "MoreThuente", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, X0[b])
    print("batch b=%d: %s niter=%d nfev=%d fx=%.6e rounds=%d | lone niter=%d nfev=%d fx=%.6e identical=%s" % (
        b, res[b]["status"], res[b]["niter"], res[b]["nfev"], res[b]["fx"], res[b]["rounds"], one["niter"], one["nfev"], one["fx"],
        bool(res[b]["fx"] == one["fx"] and np.array_equal(X[b], one["x"]))), flush=True)
bs.close()
B, n = 8, 1_000_000
X0 = np.stack([np.random.default_rng(1000 + b).uniform(-1, 1, n) for b in range(B)])
bs = lb.BatchSession(lb.OBJ_ROSENBROCK_PAIRED, X0, lb.LBFGSParam(m=10), "MoreThuente")
res, _, secs = bs.solve(return_x=False)
res, _, secs = bs.solve(return_x=False)
print("batch B=8 n=1e6: %.1f ms, iterations %s, %.1f it/s" % (secs * 1e3, [r["niter"] for r in res], sum(r["niter"] for r in res) / secs), flush=True)
bs.close()
