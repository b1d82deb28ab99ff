"""CPU: the oracle's ancestral step (oracle/ddpm_oracle.py ddpm_step, a restatement of U:1072-1121) against the REAL
reference's p_sample / p_sample_loop (tests/golden/ddpm_odd.npz, oracle/make_golden_ddpm.py, injected noise)."""
import os

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as DO
from oracle import unet_oracle as O
from oracle import weights as W

CASE = (23, 16, 16)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "ddpm_odd.npz"))


def test_single_steps_of_the_1000_step_schedule(gold):
    """Given the reference's own UNet output, the oracle's step reproduces p_sample at t = 999 (x0 = 64166 x - 64166 eps),
    998, 500, 1 and 0 (no noise) to fp32 rounding."""
    Fr, h, w = CASE
    x = torch.from_numpy(W.pseudo_normal("ddpm1000/x", (1, 3, Fr, h, w)))
    for j, t in enumerate(gold["single_t"].tolist()):
        noise = torch.from_numpy(W.pseudo_normal(f"ddpm1000/noise{t}", (1, 3, Fr, h, w)))
        y = DO.ddpm_step(torch.from_numpy(gold["single_eps"][j]), x, t, noise)
        d = (y - torch.from_numpy(gold["single_x_after"][j])).abs().max().item()
        assert d <= 1e-6, (t, d)


def test_six_step_loops(gold, synth_sd):
    """The whole p_sample_loop of a 6-step schedule (timesteps=6), with cond_scale 1 and 2, from the oracle's UNet."""
    Fr, h, w = CASE
    _, fea, cond = W.synth_inputs("odd", Fr, h, w)
    fea_rep = fea.unsqueeze(2).repeat(1, 1, Fr, 1, 1)
    T = int(gold["loop_t"])
    for scale in gold["loop_scales"].tolist():
        tag = f"ddpm6_cs{int(scale)}"
        img = torch.from_numpy(W.pseudo_normal(f"{tag}/noise-1", (1, 3, Fr, h, w)))
        for k in range(T):
            t = T - 1 - k
            with torch.no_grad():
                eps = O.forward_with_cond_scale(synth_sd, O.UnetCfg(), torch.cat([img, fea_rep], 1), torch.full((1,), t), cond,
                                                cond_scale=scale)
            img = DO.ddpm_step(eps, img, t, torch.from_numpy(W.pseudo_normal(f"{tag}/noise{k}", (1, 3, Fr, h, w))), timesteps=T)
        d = (img - torch.from_numpy(gold[f"loop_cs{int(scale)}"])).abs().max().item()
        print(f"oracle p_sample_loop T={T} cond_scale={scale}: max|d| {d:.2e}")
        assert d < 2e-4
