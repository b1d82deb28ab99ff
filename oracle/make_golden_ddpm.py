"""TEST INFRASTRUCTURE — ancestral (DDPM) sampling golden from the REAL reference, on the 'odd' clip (23 f x 16^2) with
injected noise (torch.randn / torch.randn_like patched with W.pseudo_normal, as make_golden_cfg.py):

  (a) `GaussianDiffusion.p_sample_loop` (U:1123-1134) of a 6-step schedule (timesteps=6), with cond_scale 1 and 2;
      draw k of the loop (k = 0 the start image, U:1128; k >= 1 the randn_like of step k-1, U:1118) is
      pseudo_normal('ddpm6_cs{scale}/noise{k-1}');
  (b) single `p_sample` steps (U:1112-1121) of the 1000-step schedule at t in {999, 998, 500, 1, 0}, each from the same x
      = pseudo_normal('ddpm1000/x') with noise pseudo_normal('ddpm1000/noise{t}'); the UNet output the reference
      computed at each t is stored beside the result.

Also stores the schedule buffers the step reads (both schedules), for the host-coefficient check.
Run in the build container only:    python oracle/make_golden_ddpm.py"""
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
LOOP_T, SCALES = 6, (1.0, 2.0)
SINGLE_T = (999, 998, 500, 1, 0)
BUFS = ('sqrt_recip_alphas_cumprod', 'sqrt_recipm1_alphas_cumprod', 'posterior_mean_coef1', 'posterior_mean_coef2',
        'posterior_log_variance_clipped')


class Injected:
    """torch.randn / torch.randn_like replaced by named pseudo-normal draws; counts the draws."""

    def __init__(self):
        self.names, self.k = None, 0

    def draw(self, shape):
        name = self.names(self.k)
        self.k += 1
        return torch.from_numpy(W.pseudo_normal(name, tuple(shape)))

    def __enter__(self):
        self.real = torch.randn, torch.randn_like
        torch.randn = lambda *size, **kw: self.draw(size[0] if len(size) == 1 and not isinstance(size[0], int) else size)
        torch.randn_like = lambda t, **kw: self.draw(t.shape)
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

    def diffusion(T):
        # sampling_timesteps=None selects p_sample_loop (U:1022-1024, 1150), as FlowDiffusion(sampling_timesteps=None) does
        D = U.DynamicNfGaussianDiffusion(denoise_fn=net, num_frames=40, image_size=32, sampling_timesteps=None, timesteps=T,
                                         loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0).eval()
        assert not D.is_ddim_sampling
        return D

    Fr, h, w = CASE
    shape = (1, 3, Fr, h, w)
    _, fea, cond = W.synth_inputs('odd', Fr, h, w)
    net.update_num_frames(Fr)
    out = {}

    D6 = diffusion(LOOP_T)
    D6.update_num_frames(Fr)
    for scale in SCALES:
        tag = f"ddpm6_cs{int(scale)}"
        with Injected() as inj, torch.no_grad():
            inj.names = lambda k, tag=tag: f"{tag}/noise{k - 1}"
            img = D6.p_sample_loop(fea, shape, cond=cond, cond_scale=scale)
        assert inj.k == LOOP_T + 1, inj.k            # the start image + one draw per step, t = 0 included
        out[f"loop_cs{int(scale)}"] = img.numpy()
        print(f"p_sample_loop T={LOOP_T} cond_scale={scale}: max|x| {float(img.abs().max()):.4f}")

    D1000 = diffusion(1000)
    D1000.update_num_frames(Fr)
    x = torch.from_numpy(W.pseudo_normal("ddpm1000/x", shape))
    fea_rep = fea.unsqueeze(2).repeat(1, 1, Fr, 1, 1)
    singles, epss = [], []
    for t in SINGLE_T:
        tt = torch.full((1,), t, dtype=torch.long)
        with torch.no_grad():
            eps = net.forward_with_cond_scale(torch.cat([x, fea_rep], dim=1), tt, cond=cond, cond_scale=1.)   # U:1089-1092
        with Injected() as inj, torch.no_grad():
            inj.names = lambda k, t=t: f"ddpm1000/noise{t}"
            y = D1000.p_sample(x, tt, fea, cond=cond, cond_scale=1.)
        assert inj.k == 1
        singles.append(y.numpy())
        epss.append(eps.numpy())
        print(f"p_sample t={t}: max|x| {float(y.abs().max()):.4f}")

    np.savez_compressed(os.path.join(GOLD, "ddpm_odd.npz"),
                        loop_t=np.int64(LOOP_T), loop_scales=np.array(SCALES, dtype=np.float32),
                        loop_cs1=out["loop_cs1"], loop_cs2=out["loop_cs2"],
                        single_t=np.array(SINGLE_T, dtype=np.int64), single_x_after=np.stack(singles), single_eps=np.stack(epss),
                        buf6=np.stack([getattr(D6, n).numpy() for n in BUFS]),
                        buf1000=np.stack([getattr(D1000, n).numpy() for n in BUFS]))


if __name__ == "__main__":
    main()
