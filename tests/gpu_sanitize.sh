#!/bin/bash
# compute-sanitizer passes over a small end-to-end solve and the kernel-level tests (on a machine with an H100; not part of pytest):
#     bash tests/gpu_sanitize.sh > sanitize.log 2>&1
# memcheck: out-of-bounds / misaligned accesses; racecheck: shared-memory hazards (the TMA ring, the pair-forming tiles);
# synccheck: barrier misuse; initcheck: reads of uninitialised device memory.  Kernels run 10-100x slower under the tools,
# so the inputs are small; the multi-GPU exchange kernels spin on peer flags and are not run under the tools.
set -u
cd "$(dirname "$0")/.."
SAN=/usr/local/cuda/bin/compute-sanitizer
SEL='fused_update_apply_Hv or apply_Hv_gram or level1 or objective_and_fused_trial'
for tool in memcheck racecheck synccheck initcheck; do
    echo "=== $tool ==="
    timeout 600 $SAN --tool $tool --error-exitcode 9 --print-limit 20 \
        python -m pytest tests/test_gpu_kernels.py -m gpu -q -x -k "$SEL and not 1048" 2>&1 | tail -15
    echo "exit: $?"
done
# the bound-constrained kernels at n <= 4097 (initcheck would see reads of uninitialised radix padding or scan block sums)
BOX_SEL='gpu and not 100003 and not 1048583 and not 100000 and not config4 and not ties_straddle and not keys_spread and not keys_ulp'
for tool in memcheck racecheck synccheck initcheck; do
    echo "=== $tool: box kernels ==="
    timeout 900 $SAN --tool $tool --error-exitcode 9 --print-limit 20 \
        python -m pytest tests/test_box_kernels.py -m gpu -q -x -k "$BOX_SEL" 2>&1 | tail -15
    echo "exit: $?"
done
# whole solves: host-driven loop, the persistent kernel (its watchdog budget is scaled: everything runs 10-100x slower under the tools),
# neighbour-coupled objectives, a batch, L-BFGS-B.  racecheck covers the shared-memory staging rings (it does not model the
# async-proxy writes of bulk copies; generic-proxy hazards between the passes' phases are what it can see).
export LBFGS_B200_WATCHDOG_SCALE=2000
for tool in memcheck racecheck synccheck; do
    echo "=== $tool: whole solves ==="
    timeout 900 $SAN --tool $tool --error-exitcode 9 --print-limit 20 python tests/quick_sanitize_target.py 2>&1 | tail -25
    echo "exit: $?"
done
