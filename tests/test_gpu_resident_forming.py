"""The pair-forming dots pass of the device-resident solve forms each element once -- for objectives without neighbour coupling the
accepted point, its gradient and the new pair -- in the warps the dots geometry leaves without a column or, when every warp has a
column (c = 3, 6, 12, and every c > 24), in the warps of column 0.  These runs reach the geometries an m = 10 solve does not: c = 12
with two warps per column,
and c > 24 where one warp forms every tile and the columns take two rounds, on a vector whose last CTA holds a ragged tile of
fewer than 512 coordinates."""
import numpy as np
import pytest

import lbfgspp_b200 as lb
import pyoracle as po
from test_gpu_solver import check_parity, cpu_param
from util import LS

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("m,x0", [(12, np.zeros(1000)), (30, np.full(1000, -1.2))], ids=["m12", "m30"])
def test_forming_geometries_match_cpu_checker(orc, m, x0):
    prm = lb.LBFGSParam(m=m)
    g = lb.LBFGSSolver(prm, "MoreThuente", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, x0)
    c = orc.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, LS["MoreThuente"], cpu_param(orc, prm), sum_mode=po.SUM_LANES8)
    assert c["niter"] >= m       # the history (nearly) fills up: m = 30 reaches c > 24
    check_parity(g, c, xtol=1e-7)


@pytest.mark.parametrize("m", [12, 30])
def test_forming_batch_member_equals_lone_solve(m):
    n = 1000
    X0 = np.stack([np.zeros(n), np.full(n, -1.2), np.full(n, 0.5)])
    prm = lb.LBFGSParam(m=m)
    bs = lb.BatchSession(lb.OBJ_ROSENBROCK_PAIRED, X0, prm, "MoreThuente")
    res, X, _ = bs.solve()
    bs.close()
    for b in (1, 2):
        lone = lb.LBFGSSolver(prm, "MoreThuente", resident=True).minimize(lb.OBJ_ROSENBROCK_PAIRED, X0[b])
        assert (res[b]["niter"], res[b]["nfev"], res[b]["fx"]) == (lone["niter"], lone["nfev"], lone["fx"])
        assert np.array_equal(X[b], lone["x"])
