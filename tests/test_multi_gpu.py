"""Multi-GPU parity (pytest -m gpu, needs >= 2 GPUs, skips otherwise): the frame-sharded / CFG-split step of
`bench.py --gpus N` (NCCL exchanges, eager and captured in a CUDA graph) against the unsharded native step on every
rank, through tools/gpu_shard_check.py under torchrun."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_step_matches_unsharded(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, found {torch.cuda.device_count()}")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(29500 + world), os.path.join(ROOT, "tools", "gpu_shard_check.py")]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=3600)
    assert r.returncode == 0 and "SHARD_CHECK OK" in r.stdout, (r.stdout[-4000:], r.stderr[-4000:])
