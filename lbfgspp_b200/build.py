"""Build the two in-tree shared objects of the product (no JIT cache: the .so files travel with the snapshot).

  liblbfgs_b200.so         hand-written sm_90a kernels + C ABI  (nvcc; include/lbfgs_b200.h)
  liblbfgs_b200_driver.so  header-only C++ front (include/LBFGS.h ...) behind host-buffer entry points (g++)

`python -m lbfgspp_b200.build` or lbfgspp_b200.build.build_all().
"""
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "liblbfgs_b200.so")
DRV = os.path.join(PKG, "liblbfgs_b200_driver.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CXX = "/usr/bin/g++"

# -fmad=false: IEEE multiply/add without FMA contraction.  The scalar line-search cores then take bit-identical decisions on
# the device and on the host (g++ does not contract either), element-wise kernels reproduce the CPU checker bit for bit, and
# the streaming kernels stay HBM-bound (FP64 pipe < 30 % busy), so it costs nothing measurable.
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]     # H100 only: the kernels use sm_90a PTX (TMA bulk copies, mbarrier)
NVCC_FLAGS = ["-std=c++17"] + ARCH + ["-O3", "-lineinfo", "-fmad=false",
              "-Xcompiler", "-fPIC", "-shared", "-ccbin", CXX]


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _sources(*dirs, exts=(".cu", ".cuh", ".h", ".cpp", ".hpp")):
    out = []
    for d in dirs:
        for base, _, files in os.walk(d):
            out += [os.path.join(base, f) for f in files if f.endswith(exts)]
    return out


KERNEL_UNITS = ["lbfgs_b200.cu", "persist_f64.cu", "persist_f32.cu"]   # compiled in parallel, linked into one library


def build_kernels(force=False, verbose=False):
    srcs = _sources(CSRC, os.path.join(ROOT, "include"))
    if not force and _newer(LIB, srcs):
        return LIB
    objdir = os.path.join(PKG, "build")
    os.makedirs(objdir, exist_ok=True)
    flags = [f for f in NVCC_FLAGS if f != "-shared"]
    procs, objs = [], []
    for unit in KERNEL_UNITS:
        obj = os.path.join(objdir, unit.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [NVCC] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, os.path.join(CSRC, unit)]
        procs.append((cmd, subprocess.Popen(cmd)))
    for cmd, p in procs:
        if p.wait() != 0:
            raise subprocess.CalledProcessError(p.returncode, cmd)
    subprocess.run([NVCC, "-shared"] + ARCH + ["-ccbin", CXX, "-o", LIB] + objs + ["-lnccl"], check=True)
    return LIB


def build_driver(force=False):
    srcs = _sources(CSRC, os.path.join(ROOT, "include"))
    if not force and _newer(DRV, srcs + [LIB]):
        return DRV
    cmd = [CXX, "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-fvisibility=hidden", "-fvisibility-inlines-hidden",
           "-Wl,-Bsymbolic", "-o", DRV, os.path.join(CSRC, "driver.cpp"),
           "-L", PKG, "-l:liblbfgs_b200.so", "-Wl,-rpath,$ORIGIN", "-pthread"]
    subprocess.run(cmd, check=True)
    return DRV


def build_all(force=False, verbose=False):
    return build_kernels(force, verbose), build_driver(force)


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose="-v" in sys.argv))
