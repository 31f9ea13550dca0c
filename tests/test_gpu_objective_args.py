"""Both solver loops hold a built-in objective to the same argument rules: the host-driven loop's kernels (Context.objective /
Context.trial) and the device-resident solve (LBFGSSolver(resident=True)) reject the same malformed calls with
LBFGS_B200_ERR_INVALID (std::invalid_argument through the driver), and neither launches anything first."""
import numpy as np
import pytest

import lbfgspp_b200 as lb

pytestmark = pytest.mark.gpu

# (objective id, n, part of the message); no data vectors are passed
CASES = [
    pytest.param(7, 8, "unknown objective id 7", id="unknown_id"),
    pytest.param(lb.OBJ_ROSENBROCK_PAIRED, 5, "even n", id="paired_odd_n"),
    pytest.param(lb.OBJ_QUAD_TRIDIAG, 8, "data0", id="tridiag_no_data"),
    pytest.param(lb.OBJ_ROSENBROCK_CHAINED, 1, "n >= 2", id="chained_n1"),
]
DTYPES = [np.float64, np.float32]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind,n,msg", CASES)
def test_host_loop_rejects_before_launch(kind, n, msg, dtype):
    ctx = lb.Context(0)
    x, g = ctx.array(np.zeros(n, dtype)), ctx.empty(n, dtype)
    xp, d = ctx.array(np.zeros(n, dtype)), ctx.array(np.ones(n, dtype))
    before = ctx.launches()
    with pytest.raises(lb.LbfgsB200Error, match=msg) as e:
        ctx.objective(kind, x, g)
    assert e.value.status == 1
    with pytest.raises(lb.LbfgsB200Error, match=msg) as e:
        ctx.trial(kind, xp, d, 0.5, x, g)
    assert e.value.status == 1
    assert ctx.launches() == before


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind,n,msg", CASES)
def test_resident_solve_rejects_before_launch(kind, n, msg, dtype):
    dctx = lb.Context.borrow(lb.driver_ctx(0))
    before = dctx.launches()
    r = lb.LBFGSSolver(lb.LBFGSParam(), "MoreThuente", dtype=dtype, resident=True).minimize(kind, np.zeros(n, dtype))
    assert r["status"] == "invalid_argument" and msg in r["msg"], r["msg"]
    assert dctx.launches() == before
    with pytest.raises(ValueError, match=msg):
        lb.LBFGSSolver(lb.LBFGSParam(), "MoreThuente", dtype=dtype, resident=True).minimize(kind, np.zeros(n, dtype), raise_errors=True)
