import hashlib
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LS = {"Backtracking": 0, "Bracketing": 1, "NocedalWright": 2, "MoreThuente": 3}


def unhex(xs):
    return np.array([float.fromhex(v) for v in xs], dtype=np.float64)


def golden_cases(kind=None):
    with open(os.path.join(HERE, "golden", "lbfgs_ref.json")) as fh:
        cases = json.load(fh)["cases"]
    return [c for c in cases if kind is None or c["kind"] == kind]


def same_run(a, b):
    """Bit-for-bit equality of two solver result dicts (status, counts, trace, x, grad)."""
    return (a["status"] == b["status"] and a["msg"] == b["msg"] and a["niter"] == b["niter"] and a["nfev"] == b["nfev"]
            and np.array_equal(a["trace"], b["trace"]) and np.array_equal(a["x"], b["x"])
            and np.array_equal(a["grad"], b["grad"]))


def array_digest(*arrays):
    """SHA-256 of the arrays' values as little-endian float64: equal digests mean bit-for-bit equal arrays."""
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a, dtype="<f8").tobytes())
    return h.hexdigest()


def run_digest(r):
    """A solver result reduced to what a bit-for-bit comparison needs: status, counts, and a digest of trace, x and grad."""
    return dict(status=r["status"], msg=r["msg"], niter=int(r["niter"]), nfev=int(r["nfev"]), sha256=array_digest(r["trace"], r["x"], r["grad"]))


def pin_runs(s, group):
    """Yield (key, result) for every seeded run of pin group `group`, solved by `s` (a pyoracle.Oracle).  The golden digests in
    golden/ref_pins.json come from the unmodified reference headers (oracle/_ref) running these same calls."""
    import pyoracle as po
    if group == "lbfgs":
        rng = np.random.default_rng(1)
        for n in (2, 6, 24, 100, 2002):
            for t in range(6):
                x0 = rng.uniform(-1, 1, n)
                for ls in range(4):
                    p = s.default_param(max_linesearch=256, m=3 + t % 8)
                    yield "n%d_t%d_ls%d" % (n, t, ls), s.lbfgs(po.OBJ_ROSENBROCK_PAIRED, x0, ls, p)
        d, b, _ = po.quad_tridiag_data(3000)
        for ls in range(4):
            yield "tridiag3000_ls%d" % ls, s.lbfgs(po.OBJ_QUAD_TRIDIAG, np.zeros(3000), ls, s.default_param(m=20), data0=d, data1=b)
    elif group == "lbfgs_f32":
        for ls in range(4):
            yield "ls%d" % ls, s.lbfgs(po.OBJ_ROSENBROCK_PAIRED, np.zeros(10), ls, s.default_param(), dtype=np.float32)
    elif group == "lbfgsb":
        rng = np.random.default_rng(3)
        for obj in (po.OBJ_ROSENBROCK_CHAINED, po.OBJ_ROSENBROCK_PAIRED, po.OBJ_QUAD_SHIFT, po.OBJ_QUAD_TRIDIAG):
            for n in (2, 4, 10, 25, 26, 100):
                if obj == po.OBJ_ROSENBROCK_PAIRED and n % 2:
                    continue
                for trial in range(6):
                    lo = rng.uniform(-2, 1, n)
                    hi = lo + rng.uniform(0, 3, n)
                    if trial == 0:
                        lo[:], hi[:] = 2.0, 4.0
                    elif trial == 1:
                        lo[:], hi[:] = -np.inf, np.inf
                    elif trial == 2:
                        hi[::3] = lo[::3]
                    elif trial == 3:
                        lo[::2], hi[1::3] = -np.inf, np.inf
                    x0 = rng.uniform(-3, 5, n)
                    d0, d1 = po.quad_tridiag_data(n, seed=trial)[:2] if obj == po.OBJ_QUAD_TRIDIAG else (None, None)
                    kw = dict(m=int(rng.choice([1, 2, 3, 6, 10])), max_iterations=int(rng.choice([0, 5, 50])),
                              max_submin=int(rng.choice([0, 1, 10])), past=int(rng.choice([0, 0, 2])))
                    if kw["past"]:
                        kw["delta"] = 1e-8
                    yield "obj%d_n%d_t%d" % (obj, n, trial), s.lbfgsb(obj, x0, lo, hi, s.default_param(lbfgsb=True, **kw), data0=d0, data1=d1)
    elif group == "lbfgsb_larger":
        for n, obj in ((2000, po.OBJ_ROSENBROCK_CHAINED), (5000, po.OBJ_ROSENBROCK_PAIRED)):
            yield "obj%d_n%d" % (obj, n), s.lbfgsb(obj, np.full(n, 3.0), 2.0, 4.0, s.default_param(lbfgsb=True))
    else:
        raise ValueError(group)


def apply_Hv_pin_runs(s):
    """Yield (key, res, theta) of the seeded apply_Hv calls pinned in golden/ref_pins.json."""
    rng = np.random.default_rng(3)
    n, m = 1000, 5
    for npairs in (0, 1, 4, 5, 6, 13):
        S = rng.standard_normal((npairs, n))
        Y = S + 0.1 * rng.standard_normal((npairs, n))
        v = rng.standard_normal(n)
        res, _, theta = s.apply_Hv(S, Y, v, -1.0, m)
        yield "npairs%d" % npairs, res, theta


def ref_pins():
    with open(os.path.join(HERE, "golden", "ref_pins.json")) as fh:
        return json.load(fh)
