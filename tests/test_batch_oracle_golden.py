"""CPU: the oracle restatement (oracle/unet_oracle.py, oracle/ddpm_oracle.py) against the batch golden the REAL reference
produced (oracle/make_golden_batch.py): one forward over two clips, ddim_sample and p_sample_loop at b = 2.  The reference runs
the batch as one tensor; the restatement runs each clip's UNet alone and the updates over the batch (one quantile per clip)."""
import os

import numpy as np
import torch

from oracle import ddpm_oracle as DO
from oracle import unet_oracle as O
from oracle.make_golden_batch import DDIM_STEPS, DDPM_T, batch_inputs, draw


def over_tol(a, ref):
    return ((a - ref).abs() / (1e-4 + 1e-3 * ref.abs())).max().item()


def eps_of(sd, img, fea, t, cond):
    Fr = img.shape[2]
    x = torch.cat([img, fea.unsqueeze(2).expand(-1, -1, Fr, -1, -1)], dim=1)
    return torch.cat([O.unet_forward(sd, O.UnetCfg(), x[i:i + 1], torch.full((1,), t, dtype=torch.long), cond[i:i + 1])
                      for i in range(x.shape[0])])


def test_oracle_reproduces_batch_golden(golden_dir, synth_sd):
    g = np.load(os.path.join(golden_dir, "batch_odd.npz"))
    x, t, cond, fea = batch_inputs()
    with torch.no_grad():
        eps = torch.cat([O.unet_forward(synth_sd, O.UnetCfg(), x[i:i + 1], t[i:i + 1], cond[i:i + 1]) for i in range(2)])
        assert over_tol(eps, torch.from_numpy(g["eps"])) < 0.5
        shape = (2, 3) + tuple(x.shape[2:])
        img = draw("batch_ddim", -1, shape)
        for k, (tt, tn) in enumerate(O.ddim_time_pairs(1000, int(g["ddim_steps"]))):
            img = O.ddim_step(eps_of(synth_sd, img, fea, tt, cond), img, tt, tn, draw("batch_ddim", k, shape) if tn > 0 else None)
        assert over_tol(img, torch.from_numpy(g["ddim"])) < 0.5
        img = draw("batch_ddpm", -1, shape)
        T = int(g["ddpm_t"])
        for k in range(T):
            tt = T - 1 - k
            img = DO.ddpm_step(eps_of(synth_sd, img, fea, tt, cond), img, tt, draw("batch_ddpm", k, shape), timesteps=T)
        assert over_tol(img, torch.from_numpy(g["ddpm"])) < 0.5
    assert (DDIM_STEPS, DDPM_T) == (int(g["ddim_steps"]), T)
