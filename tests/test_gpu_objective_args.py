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


def _tridiag_batch(ctx, dtype, B, n, ldd, offset_elems=0):
    from test_gpu_resident_implied_grad import resident
    size = max(ldd, n) * B + 64
    d = lb.DeviceArray(ctx, np.ones(size, dtype), offset_elems=offset_elems)
    b = lb.DeviceArray(ctx, np.zeros(size, dtype))
    return resident(ctx, lb.OBJ_QUAD_TRIDIAG, np.zeros((B, n), dtype), lb.LBFGSParam(), "MoreThuente", data0=d, data1=b, ldd=ldd)


# (batch, n, ldd, data0 offset in elements, part of the message): the resident solve reads each problem's data with bulk copies
# that start on 16-byte boundaries of data + b*ldd
DATA_CASES = [
    pytest.param(2, 100, 50, 0, "at least n", id="ldd_below_n"),
    pytest.param(2, 100, -100, 0, "at least n", id="ldd_negative"),
    pytest.param(2, 100, 101, 0, "multiple of 16 bytes", id="ldd_misaligned"),
    pytest.param(1, 100, 0, 1, "16-byte boundary", id="data0_misaligned"),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,n,ldd,offset,msg", DATA_CASES)
def test_resident_solve_rejects_bad_data_layout_before_launch(gpu_ctx, B, n, ldd, offset, msg, dtype):
    before = gpu_ctx.launches()
    with pytest.raises(lb.LbfgsB200Error, match=msg) as e:
        _tridiag_batch(gpu_ctx, dtype, B, n, ldd, offset)
    assert e.value.status == 1
    assert gpu_ctx.launches() == before
