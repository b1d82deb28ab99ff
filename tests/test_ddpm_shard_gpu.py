"""-m gpu, needs >= 2 GPUs on the box (skipped otherwise): the ancestral (DDPM) sampler on one clip frame-sharded over 2 ranks
(torchrun, one rank per GPU, NCCL; clip-wide quantile through the all-reduced radix select, each rank's slice of one seeded
noise stream), eager and with the step graph, vs the single-GPU sampler.  The checks live in tests/ddpm_shard_ranks.py
(they assert on rank 0)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("mode,port", [("eager", 29621), ("graph", 29622)])
def test_two_rank_ancestral_sampler_matches_single_gpu(mode, port):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "ddpm_shard_ranks.py"), mode]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stderr[-3000:]
    assert "[ddpm]" in r.stdout
