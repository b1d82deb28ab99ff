"""-m gpu: a batch of two clips against the batch golden of the REAL reference (oracle/make_golden_batch.py, tests/golden/
batch_odd.npz): one UNet forward over both clips, and ddim_sample / p_sample_loop at b = 2, eager and as CUDA graphs.  Clip 1's
start image has 3x the amplitude of clip 0's, so a quantile shared by both clips would not reproduce the reference."""
import os

import numpy as np
import pytest
import torch

from oracle.make_golden_batch import batch_inputs, draw
from tests import gpu_common as G

pytestmark = pytest.mark.gpu


def golden():
    return np.load(os.path.join(G.ROOT, "tests", "golden", "batch_odd.npz"))


def test_batched_forward_matches_reference_golden():
    net = G.cuda_net()
    x, t, cond, _ = batch_inputs()
    net.update_num_frames(x.shape[2])
    with torch.no_grad():
        out = net.forward_with_cond_scale(x.cuda(), t.cuda(), cond=cond.cuda(), cond_scale=1.0).cpu()
    assert net.clip_count() == 2
    r = G.over_tol(out, torch.from_numpy(golden()["eps"]))
    print(f"b=2 forward vs reference: {r:.3f} x tol")
    assert r <= 1.0


def _diffusion(timesteps, sampling_timesteps):
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion
    D = DynamicNfGaussianDiffusion(denoise_fn=G.cuda_net(), num_frames=40, image_size=32, sampling_timesteps=sampling_timesteps,
                                   timesteps=timesteps, loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1,
                                   ddim_sampling_eta=1.0).cuda()
    return D


@pytest.mark.parametrize("kind", ["ddim", "ddpm"])
def test_batched_sampling_matches_reference_golden(kind):
    g = golden()
    x, _, cond, fea = batch_inputs()
    Fr, h, w = x.shape[2:]
    shape = (2, 3, Fr, h, w)
    if kind == "ddim":
        D, tag, ref = _diffusion(1000, int(g["ddim_steps"])), "batch_ddim", torch.from_numpy(g["ddim"])
        run = D.ddim_sample
    else:
        D, tag, ref = _diffusion(int(g["ddpm_t"]), None), "batch_ddpm", torch.from_numpy(g["ddpm"])
        run = D.p_sample_loop
    D.update_num_frames(Fr)
    res = {}
    for graph in (False, True):
        res[graph] = run(fea.cuda(), shape, cond=cond.cuda(), noise_fn=lambda k, s: draw(tag, k, s), use_graph=graph).cpu()
    assert D.denoise_fn.clip_count() == 2
    r_e, r_g = G.over_tol(res[False], ref), G.over_tol(res[True], ref)
    d = (res[True] - res[False]).abs().max().item()
    print(f"{kind} b=2: eager {r_e:.3f} x tol, graph {r_g:.3f} x tol, graph vs eager {d:.2e}")
    assert r_e <= 1.0 and r_g <= 1.0
    assert d <= 5e-5
