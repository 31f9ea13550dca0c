"""Generate tests/golden/ref_pins.json: digests of the UNMODIFIED reference headers (oracle/_ref, built over minieigen) on the
seeded runs of tests/util.py:pin_runs / apply_Hv_pin_runs.

Needs oracle/_ref/libref_lbfgspp.so (make -C oracle ref REF=<LBFGSpp checkout>).  Run from the repository root:
    python tests/golden/make_ref_pins.py
Each solve is stored as status, message, counts and a SHA-256 of its trace, x and grad (float64 bytes), each apply_Hv result as a
SHA-256 of its float64 bytes and theta as a hex float: tests/test_oracle_cpu.py holds the restatement to these bit for bit on machines without the reference.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import pyoracle as po  # noqa: E402
from util import apply_Hv_pin_runs, array_digest, pin_runs, run_digest  # noqa: E402


def main():
    ref = po.Oracle("ref")
    out = {"source": "oracle/_ref (unmodified reference headers @ ebef584 over oracle/minieigen)",
           "generator": "tests/golden/make_ref_pins.py"}
    for group in ("lbfgs", "lbfgs_f32", "lbfgsb", "lbfgsb_larger"):
        out[group] = {k: run_digest(r) for k, r in pin_runs(ref, group)}
    out["apply_Hv"] = {k: dict(res_sha256=array_digest(res), theta=float(theta).hex()) for k, res, theta in apply_Hv_pin_runs(ref)}
    with open(os.path.join(HERE, "ref_pins.json"), "w") as fh:
        json.dump(out, fh, indent=0, sort_keys=True)
        fh.write("\n")
    print({k: len(v) for k, v in out.items() if isinstance(v, dict)})


if __name__ == "__main__":
    main()
