"""Small whole solves for tests/gpu_sanitize.sh (compute-sanitizer target; not collected by pytest): both solver loops, all four line
searches, the neighbour-coupled objectives (staged tiles with margins, fp32 at odd n, a batch with per-problem data, plain dots rounds), fp32, a batch, the literal two-loop recursion, histories of 64 pairs, L-BFGS-B."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import lbfgspp_b200 as lb  # noqa: E402
import pyoracle as po  # noqa: E402  (only the deterministic data generator)

n = 6002
for resident in (False, True):
    for ls in ("Backtracking", "Bracketing", "NocedalWright", "MoreThuente"):
        g = lb.LBFGSSolver(lb.LBFGSParam(m=7), ls, resident=resident).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(n))
        print("lbfgs", "resident" if resident else "host", ls, g["status"], g["niter"], g["nfev"], g["fx"])
d, b, _ = po.quad_tridiag_data(5003, seed=2)
for resident in (False, True):
    g = lb.LBFGSSolver(lb.LBFGSParam(m=12, max_iterations=25), "Bracketing", resident=resident).minimize(lb.OBJ_QUAD_TRIDIAG, np.zeros(5003), data0=d, data1=b)
    print("tridiag", "resident" if resident else "host", g["status"], g["niter"], g["nfev"], g["fx"])
    g = lb.LBFGSSolver(lb.LBFGSParam(m=5), "NocedalWright", resident=resident).minimize(lb.OBJ_ROSENBROCK_CHAINED, np.full(3000, 1.3))
    print("chained", "resident" if resident else "host", g["status"], g["niter"], g["nfev"], g["fx"])
g = lb.LBFGSSolver(lb.LBFGSParam(), "MoreThuente", dtype=np.float32, resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(4096))
print("lbfgs f32 resident", g["status"], g["niter"], g["fx"])
g = lb.LBFGSSolver(lb.LBFGSParam(m=3, max_iterations=30), "MoreThuente", dtype=np.float32, resident=True).minimize(lb.OBJ_ROSENBROCK_CHAINED, np.full(6007, 1.3))
print("chained f32 resident odd n", g["status"], g["niter"], g["fx"])
# per-problem data through the C ABI: problem k's d and b at offset k*ldd, ldd > n (the bulk copies read up to round_up(n, 32))
from test_gpu_resident_implied_grad import resident  # noqa: E402
nb, ldd = 5003, 5004
D, R = np.zeros(2 * ldd + 5024), np.zeros(2 * ldd + 5024)
for k in range(3):
    D[k * ldd:k * ldd + nb], R[k * ldd:k * ldd + nb] = po.quad_tridiag_data(nb, seed=3 + k)[:2]
ctx = lb.Context(0)
outs, _, _, _ = resident(ctx, lb.OBJ_QUAD_TRIDIAG, np.zeros((3, nb)), lb.LBFGSParam(m=6, max_iterations=25), "MoreThuente", data0=D, data1=R, ldd=ldd)
print("tridiag batch per-problem data", [(o.status, o.niter) for o in outs])
# a neighbour-coupled solve with plain dots rounds: the curvature gate rejects pairs of an indefinite quadratic
from test_gpu_resident_coupled import indefinite_tridiag  # noqa: E402
d, b = indefinite_tridiag(6002, np.float64)
prm = lb.LBFGSParam(m=10, linesearch=lb.LBFGS_LINESEARCH_BACKTRACKING_ARMIJO, max_iterations=8)
outs, _, _, by_op = resident(ctx, lb.OBJ_QUAD_TRIDIAG, np.zeros(6002), prm, "Backtracking", data0=d, data1=b)
print("tridiag plain dots", outs[0].status, outs[0].niter, by_op)
ctx.close()
bs = lb.BatchSession(lb.OBJ_ROSENBROCK_PAIRED, np.stack([np.zeros(3000), np.full(3000, 0.5), np.ones(3000)]), lb.LBFGSParam(m=6), "MoreThuente")
res, _, _ = bs.solve()
bs.close()
print("batch", [(r["status"], r["niter"]) for r in res])
g = lb.LBFGSSolver(lb.LBFGSParam(m=5), "NocedalWright", hv_algo=lb.HV_TWO_LOOP).minimize(lb.OBJ_ROSENBROCK_CHAINED, np.full(3000, 1.3))
print("lbfgs two-loop chained", g["status"], g["niter"], g["fx"])
# long histories: a resident solve past c = 48 (the third round of columns, 64-element history blocks) and an m = 64 Gram apply_Hv
d, b, _ = po.quad_tridiag_data(6003, seed=1)
g = lb.LBFGSSolver(lb.LBFGSParam(m=64, max_iterations=52), "MoreThuente", resident=True).minimize(lb.OBJ_QUAD_TRIDIAG, np.zeros(6003), data0=d, data1=b)
print("tridiag resident m=64", g["status"], g["niter"], g["nfev"], g["fx"])
ctx = lb.Context(0)
rng = np.random.default_rng(64)
h = lb.History(ctx, 6003, 64)
for _ in range(70):
    s = rng.standard_normal(6003)
    h.add(ctx.array(s), ctx.array(s + 0.1 * rng.standard_normal(6003)))
res = ctx.empty(6003)
h.apply_Hv(ctx.array(rng.standard_normal(6003)), -1.0, res, lb.HV_GRAM)
print("apply_Hv gram m=64 c=%d" % h.ncorr, float(np.abs(res.get()).max()))
del h, res
ctx.close()
g = lb.LBFGSBSolver(lb.LBFGSBParam()).minimize(lb.OBJ_ROSENBROCK_CHAINED, np.full(5000, 3.0), 2.0, 4.0)
print("lbfgsb", g["status"], g["niter"], g["nfev"], g["fx"])
