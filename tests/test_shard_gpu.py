"""-m gpu, needs >= 2 GPUs on the box (skipped otherwise): exact frame sharding (SURVEY 8e) of one clip over 2 ranks, launched the way
the driver launches bench.py (torchrun, one rank per GPU, NCCL): sharded forward vs the reference golden ('band': F = 96, window active)
and vs the single-GPU CUDA path, and the sharded DDIM sampler (distributed quantile, eager and graph-captured) vs the single-GPU
sampler.  The checks themselves live in tests/shard_ranks.py (they assert on rank 0)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("what,port", [("forward", 29611), ("ddim", 29612), ("ddim_graph", 29613)])
def test_two_rank_sharding_matches_single_gpu(what, port):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "shard_ranks.py"), what]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stderr[-3000:]
    assert "[band]" in r.stdout or "[ddim]" in r.stdout
