"""CPU tests of the boundary: the C-ABI library loads without a GPU, exports every symbol that include/lbfgs_b200.h
declares, and fails loudly (no silent CPU fallback) when no CUDA device is present."""
import ctypes as C
import os
import re

import pytest

import lbfgspp_b200 as lb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "lbfgs_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    names = set(re.findall(r"\b(lbfgs_b200_[a-z0-9_]+?)(?:_##SUF)?\s*\(", text))
    out = set()
    for nme in names:
        # functions declared through the DECLARE_* macros carry a _##SUF suffix in the header
        if re.search(r"\b" + nme + r"_##SUF", text):
            out.update({nme + "_f64", nme + "_f32"})
        else:
            out.add(nme)
    return sorted(out)


def test_library_exports_every_declared_symbol():
    lb.build_all()
    lib = C.CDLL(os.path.join(ROOT, "lbfgspp_b200", "liblbfgs_b200.so"))
    syms = declared_symbols()
    assert len(syms) >= 40
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing


def test_driver_library_loads_and_links_against_kernels():
    drv = lb.driver()
    assert hasattr(drv, "lbfgsb200_drv_lbfgs_f64") and hasattr(drv, "lbfgsb200_drv_lbfgs_f32")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback_context_creation_fails_loudly():
    with pytest.raises(lb.LbfgsB200Error) as e:
        lb.Context(0)
    assert "no CPU fallback" in str(e.value) or "CUDA" in str(e.value)


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback_solver_reports_runtime_error():
    import numpy as np
    r = lb.LBFGSSolver(lb.LBFGSParam()).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(10))
    assert r["status"] == "runtime_error" and r["niter"] == 0
    with pytest.raises(RuntimeError):
        lb.LBFGSSolver(lb.LBFGSParam()).minimize(lb.OBJ_ROSENBROCK_PAIRED, np.zeros(10), raise_errors=True)


def test_version_string():
    assert b"sm_90a" in lb.abi().lbfgs_b200_version()


def test_header_is_plain_c_and_links_from_c(tmp_path):
    """include/lbfgs_b200.h in a C99 translation unit (-pedantic -Werror), linked against the library, run without a GPU."""
    import subprocess
    lb.build_all()
    exe = str(tmp_path / "abi_is_plain_c")
    libdir = os.path.join(ROOT, "lbfgspp_b200")
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "c", "abi_is_plain_c.c"), "-o", exe, "-L", libdir, "-l:liblbfgs_b200.so",
                    "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode in (0, 3), (r.returncode, r.stdout, r.stderr)
    assert "lbfgs" in r.stdout.lower()
