"""TEST INFRASTRUCTURE — torch-CPU restatement of the reference's ancestral (DDPM) step, GaussianDiffusion.p_sample
(DM_3/modules/video_flow_diffusion_multiGPU_v0_crema_plus_faceemb_ca_multi_test.py — "U" — :1087-1134), beside the UNet
restatement in oracle/unet_oracle.py.  Pinned against the real reference by oracle/make_golden_ddpm.py
(tests/test_ddpm_oracle_golden.py).  Each function cites its lines."""
import torch
import torch.nn.functional as F


def ddpm_buffers(timesteps=1000, s=0.008):
    """U:975-985 + U:1012-1055: the fp32 buffers one ancestral step reads, as a dict of (timesteps,) tensors."""
    steps = timesteps + 1
    x = torch.linspace(0, timesteps, steps, dtype=torch.float64)
    ac = torch.cos(((x / timesteps) + s) / (1 + s) * torch.pi * 0.5) ** 2
    ac = ac / ac[0]
    betas = torch.clip(1 - (ac[1:] / ac[:-1]), 0, 0.9999)
    alphas = 1. - betas
    acp = torch.cumprod(alphas, dim=0)
    prev = F.pad(acp[:-1], (1, 0), value=1.)
    pv = betas * (1. - prev) / (1. - acp)                                              # U:1045
    return dict(sqrt_recip_alphas_cumprod=torch.sqrt(1. / acp).float(),                 # U:1040
                sqrt_recipm1_alphas_cumprod=torch.sqrt(1. / acp - 1).float(),           # U:1041
                posterior_log_variance_clipped=torch.log(pv.clamp(min=1e-20)).float(),  # U:1053
                posterior_mean_coef1=(betas * torch.sqrt(prev) / (1. - acp)).float(),   # U:1054
                posterior_mean_coef2=((1. - prev) * torch.sqrt(alphas) / (1. - acp)).float())   # U:1055


def ddpm_step(eps, img, t, noise, timesteps=1000, dynamic_thres=True, pct=0.9, clip_denoised=True):
    """U:1072-1121: one ancestral step of img (b, ...) at timestep t (one value for the batch) given the UNet's eps.
    noise: the torch.randn_like draw of U:1118 (multiplied by 0 at t = 0), or None for none."""
    B = ddpm_buffers(timesteps)
    b = img.shape[0]
    shp = (b,) + (1,) * (img.ndim - 1)

    def ext(name):                                                                      # extract(a, t, shape), U:969-972
        return B[name][torch.full((b,), t, dtype=torch.long)].reshape(shp)
    x0 = ext('sqrt_recip_alphas_cumprod') * img - ext('sqrt_recipm1_alphas_cumprod') * eps          # U:1072-1076
    if clip_denoised:                                                                   # U:1094-1107
        s = 1.
        if dynamic_thres:
            s = torch.quantile(x0.reshape(b, -1).abs(), pct, dim=-1)
            s.clamp_(min=1.)
            s = s.view(-1, *((1,) * (x0.ndim - 1)))
        x0 = x0.clamp(-s, s) / s
    mean = ext('posterior_mean_coef1') * x0 + ext('posterior_mean_coef2') * img        # U:1078-1082
    if noise is None:
        return mean
    nonzero_mask = (1 - (torch.full((b,), t) == 0).float()).reshape(shp)                # U:1120
    return mean + nonzero_mask * (0.5 * ext('posterior_log_variance_clipped')).exp() * noise       # U:1121
