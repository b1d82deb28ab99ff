"""TEST INFRASTRUCTURE — a batch of two clips through the REAL reference (batch dimension b = 2, U:892-956, 1156-1208, 1123-1134),
on the 'odd' geometry (23 f x 16^2) with injected noise (torch.randn / randn_like patched with W.pseudo_normal, as
make_golden_cfg.py):

  (a) one `forward_with_cond_scale(cond_scale=1)` over both clips: clip 0 = the 'odd' clip at t = 47, clip 1 = another clip
      ('odd_b') at t = 523 with 3x the amplitude in its noisy channels;
  (b) `ddim_sample` at b = 2, 3 steps, cond_scale 1: draw k (k = -1 the start image, U:1166; k >= 0 the randn_like of step k,
      U:1201) is pseudo_normal('batch_ddim/noise{k}') of shape (2, 3, F, h, w), the start image's clip 1 scaled by 3 so that one
      quantile shared by both clips would give another sample;
  (c) `p_sample_loop` at b = 2 on the 6-step schedule of ddpm_odd.npz (timesteps = 6), draws pseudo_normal('batch_ddpm/noise{k}'),
      the start image's clip 1 scaled by 3.

Run in the build container only:    python oracle/make_golden_batch.py"""
import importlib
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import weights as W          # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
U_MOD = 'DM_3.modules.video_flow_diffusion_multiGPU_v0_crema_plus_faceemb_ca_multi_test'
CASE = (23, 16, 16)                       # the 'odd' geometry
T_FWD = (47, 523)
DDIM_STEPS, DDPM_T, AMP = 3, 6, 3.0


def batch_inputs():
    """x (2, 275, F, h, w), t (2,), cond (2, F, 1032), fea (2, 272, h, w) of the two clips (shared with the tests)."""
    Fr, h, w = CASE
    xs, feas, conds = [], [], []
    for tag, amp in (('odd', 1.0), ('odd_b', AMP)):
        x_t, fea, cond = W.synth_inputs(tag, Fr, h, w)
        xs.append(torch.cat([x_t * amp, fea.unsqueeze(2).expand(-1, -1, Fr, -1, -1)], dim=1))
        feas.append(fea); conds.append(cond)
    return torch.cat(xs).contiguous(), torch.tensor(T_FWD, dtype=torch.long), torch.cat(conds), torch.cat(feas)


def draw(tag, k, shape):
    """draw k of a sampler run: the start image (k = -1) has clip 1 scaled by AMP"""
    x = torch.from_numpy(W.pseudo_normal(f"{tag}/noise{k}", tuple(shape)))
    if k == -1:
        x[1] *= AMP
    return x


class Injected:
    def __init__(self, tag):
        self.tag, self.k = tag, -1

    def one(self, shape):
        x = draw(self.tag, self.k, shape)
        self.k += 1
        return x

    def __enter__(self):
        self.real = torch.randn, torch.randn_like
        torch.randn = lambda *size, **kw: self.one(size[0] if len(size) == 1 and not isinstance(size[0], int) else size)
        torch.randn_like = lambda t, **kw: self.one(t.shape)
        return self

    def __exit__(self, *a):
        torch.randn, torch.randn_like = self.real


def main():
    sys.path.insert(0, os.path.join(HERE, 'shims'))
    sys.path.insert(0, '/root/reference')
    warnings.filterwarnings("ignore")
    U = importlib.import_module(U_MOD)
    with open(os.path.join(GOLD, 'state_dict_schema.json')) as f:
        schema = [(n, tuple(s)) for n, s in json.load(f)['entries']]
    net = U.DynamicNfUnet3D(dim=64, cond_dim=1032, cond_aud=1024, cond_pose=6, cond_eye=2, num_frames=40, channels=275, out_grid_dim=2,
                            out_conf_dim=1, dim_mults=(1, 2, 4, 8), use_hubert_audio_cond=True, learn_null_cond=False,
                            use_final_activation=False, use_deconv=True, padding_mode="zeros", win_width=40).eval()
    net.load_state_dict(W.synth_state_dict(schema), strict=True)
    Fr, h, w = CASE
    net.update_num_frames(Fr)
    x, t, cond, fea = batch_inputs()
    with torch.no_grad():
        eps = net.forward_with_cond_scale(x, t, cond=cond, cond_scale=1.)
    print("forward", tuple(eps.shape), float(eps.abs().max()))
    shape = (2, 3, Fr, h, w)

    def diffusion(T, S):
        D = U.DynamicNfGaussianDiffusion(denoise_fn=net, num_frames=40, image_size=32, sampling_timesteps=S, timesteps=T,
                                         loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0).eval()
        D.update_num_frames(Fr)
        return D

    with Injected("batch_ddim") as inj, torch.no_grad():
        ddim = diffusion(1000, DDIM_STEPS).ddim_sample(fea, shape, cond=cond, cond_scale=1.)
    assert inj.k == DDIM_STEPS - 1, inj.k             # start image + one draw per step but the last
    print("ddim_sample", float(ddim[0].abs().max()), float(ddim[1].abs().max()))
    D6 = diffusion(DDPM_T, None)
    assert not D6.is_ddim_sampling
    with Injected("batch_ddpm") as inj, torch.no_grad():
        ddpm = D6.p_sample_loop(fea, shape, cond=cond, cond_scale=1.)
    assert inj.k == DDPM_T, inj.k                     # start image + one draw per step, t = 0 included
    print("p_sample_loop", float(ddpm[0].abs().max()), float(ddpm[1].abs().max()))
    np.savez_compressed(os.path.join(GOLD, "batch_odd.npz"), t=t.numpy(), eps=eps.numpy(), ddim_steps=np.int64(DDIM_STEPS),
                        ddim=ddim.numpy(), ddpm_t=np.int64(DDPM_T), ddpm=ddpm.numpy())


if __name__ == "__main__":
    main()
