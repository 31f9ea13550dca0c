"""n-sharded (multi-GPU) parity: launches tests/multi_gpu_check.py under torchrun on 2 GPUs of this box, once with the
in-kernel NVLink exchange and once with NCCL.  Skipped on a single-GPU machine (the host-side sharding logic is covered on CPU by
tests/test_sharding_cpu.py with the gloo backend)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize("mode,port", [("p2p", 29511), ("nccl", 29512)])
def test_two_gpu_sharded_parity(mode, port):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(HERE, "multi_gpu_check.py"), mode]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "MULTI_GPU_CHECK PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
