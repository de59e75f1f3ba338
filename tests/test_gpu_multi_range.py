"""The range partitioner on >= 2 GPUs of one box (skipped on a single-GPU box): runs tests/multi_gpu_range_check.py
under torchrun, one rank per GPU."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.gpu
@pytest.mark.skipif(_ngpus() < 2, reason="needs >= 2 GPUs")
def test_range_partitioner_on_several_gpus():
    n = min(_ngpus(), 8)
    n = 8 if n >= 8 else 4 if n >= 4 else 2
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n),
                        "--master-addr", "127.0.0.1", "--master-port", "29521",
                        os.path.join(ROOT, "tests", "multi_gpu_range_check.py")],
                       capture_output=True, text=True, timeout=800)
    sys.stdout.write(r.stdout[-3000:])
    sys.stderr.write(r.stderr[-3000:])
    assert r.returncode == 0 and "MULTI_GPU_RANGE_CHECK_OK" in r.stdout
