"""`pytest -m gpu` on a box with >= 2 GPUs: the batch-sharded int8 path (cross-rank DynamicQuantizeLinear range)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sharded_int8_resnet50_bit_exact():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29617", os.path.join(ROOT, "tools", "sharded_int8_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert "bit-identical to the unsharded oracle: True" in out.stdout
    # both forms of the exchange are exact: the NVLink peer-mailbox kernel (peer_minmax_kernel, the default) and the NCCL
    # fallback
    assert "NCCL fallback bit-identical: True" in out.stdout and "(timeouts 0)" in out.stdout, out.stdout[-1500:]
    print(out.stdout[-600:])
