"""torch-CPU fp32 restatement of the sampler updates that csrc/sampler.cu must repeat bit for bit: the DDIM update of ddim_sample
(U:1181-1205; U = DM_3/modules/video_flow_diffusion_multiGPU_v0_crema_plus_faceemb_ca_multi_test.py), the ancestral update of
p_sample (U:1072-1121) and the classifier-free-guided eps of forward_with_cond_scale (U:879-890), for one clip.

Each line is the reference's own fp32 torch operation, in its order.  Unlike oracle.unet_oracle.ddim_step and
oracle.ddpm_oracle.ddpm_step, which they equal where both apply (tests/test_sampler_ref_cpu.py), these take the update's
coefficients as given (the five floats DynamicNfGaussianDiffusion.ddim_coefficients / ddpm_table hand the kernels), the
no-clip variant (clip_denoised=False, q < 0) and an optional threshold s in place of torch.quantile's.

q selects the clip as the kernels do: q > 0 the dynamic threshold at quantile q, q = 0 the static clamp to [-1, 1]
(use_dynamic_thres=False), q < 0 none."""
import numpy as np
import torch

F32 = torch.float32


def _f(v):
    """a 0-d fp32 tensor: the reference's extract()-ed buffers and alpha scalars multiply as fp32 tensors"""
    return torch.as_tensor(v, dtype=F32).reshape(())


def guided_eps(e_cond, e_null, scale):
    """U:889-890: null_logits + (logits - null_logits) * cond_scale"""
    return e_null + (e_cond - e_null) * float(scale)


def quantile_s(x0, q):
    """U:1186-1192 / U:1097-1103: max(1, torch.quantile(|x0|, q)) over the clip; NaN stays NaN"""
    s = torch.quantile(x0.reshape(1, -1).abs(), q, dim=-1)
    s.clamp_(min=1.)
    return s


def clip_x0(x0, q, s=None):
    """U:1183-1196 / U:1094-1107; s (a float or 1-element tensor) replaces the torch.quantile threshold when given"""
    if q < 0:
        return x0
    if q == 0:
        return x0.clamp(-1., 1.) / 1.
    s = quantile_s(x0, q) if s is None else torch.as_tensor(s, dtype=F32).reshape(1)
    s = s.view(-1, *((1,) * (x0.ndim - 1))) if x0.ndim > 1 else s
    return x0.clamp(-s, s) / s


def ddim_step(x, e, noise, coef, q, s=None):
    """U:1181-1205 with coef = (ca, cb, sqrt(alpha_next), c, sigma).  noise None is the last step, which adds sigma * 0."""
    ca, cb, san, c, sigma = (_f(v) for v in coef)
    x0 = ca * x - cb * e                                                    # predict_start_from_noise, U:1072-1076
    x0 = clip_x0(x0, q, s)
    return x0 * san + c * e + sigma * (noise if noise is not None else 0.)


def ddpm_step(x, e, noise, coef, q, s=None):
    """U:1072-1121 with coef = (ca, cb, c1, c2, sigma), sigma = [t > 0] * exp(0.5 * posterior_log_variance_clipped[t]).
    noise None returns the posterior mean."""
    ca, cb, c1, c2, sigma = (_f(v) for v in coef)
    x0 = ca * x - cb * e
    x0 = clip_x0(x0, q, s)
    mean = c1 * x0 + c2 * x                                                 # q_posterior, U:1078-1082
    return mean if noise is None else mean + sigma * noise                 # U:1121


def order_stat_s(abs_keys, q, replicas=1):
    """float64 max(1, at::lerp(v[lo], v[hi], w)) of the q-quantile of `replicas` copies of the keys, with torch.quantile's fp32
    rank q (N - 1) and its NaN rule (any NaN key gives NaN).  Element r of the sorted copies is element r // replicas of the
    sorted keys.  Returns (s, lo, hi, w)."""
    keys = np.sort(np.asarray(abs_keys, dtype=np.float64).reshape(-1))     # NaN sorts last
    N = keys.size * replicas
    rank = np.float32(q) * np.float32(N - 1)
    lo, hi = int(np.floor(rank)), int(np.ceil(rank))
    w = float(rank - np.floor(rank))
    vlo, vhi = keys[lo // replicas], keys[hi // replicas]
    with np.errstate(invalid="ignore"):
        lerp = vlo + w * (vhi - vlo) if w < 0.5 else vhi - (vhi - vlo) * (1.0 - w)
    if np.isnan(keys).any() or np.isnan(lerp):
        return float("nan"), lo, hi, w
    return max(float(lerp), 1.0), lo, hi, w
