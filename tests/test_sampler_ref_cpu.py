"""CPU: the fp32 restatement of the sampler updates (tests/sampler_ref.py), which tests/test_sampler_kernels_gpu.py holds the update
kernels to bit for bit, against oracle.unet_oracle.ddim_step and oracle.ddpm_oracle.ddpm_step, which the goldens pin to the real
reference; the coefficients the sampler hands the kernels against the reference's buffers; and dawn_test_kernel's refusals of bad
sampler-step cases, which happen before any CUDA call and so need no GPU."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as DO
from oracle import unet_oracle as O
from tests import sampler_ref as S


def bits_equal(a, b):
    """bit for bit, NaN payloads aside"""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


def clip(seed, t, shape=(1, 3, 5, 8, 8)):
    """x_t = sqrt(ab) x0 + sqrt(1 - ab) e as in sampling (x0 ~ 1.5 N(0, 1)), so ca x - cb e cancels as it does there"""
    g = torch.Generator().manual_seed(seed)
    acp, _ = O.cosine_alphas_cumprod()
    x0, e, z = (torch.randn(shape, generator=g, dtype=torch.float64) for _ in range(3))
    x = (acp[t].double().sqrt() * 1.5 * x0 + (1 - acp[t].double()).sqrt() * e).float()
    return x, e.float(), z.float()


def diffusion(eta=1.0):
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion
    return DynamicNfGaussianDiffusion(denoise_fn=None, num_frames=40, image_size=32, sampling_timesteps=20, timesteps=1000,
                                      loss_type='l2', use_dynamic_thres=True, ddim_sampling_eta=eta)


def oracle_ddim_coef(t, tn, eta):
    """the five scalars oracle.unet_oracle.ddim_step forms, in its own fp32 arithmetic"""
    acp, prev = O.cosine_alphas_cumprod()
    alpha, alpha_next = prev[t], prev[tn]
    sigma = eta * ((1 - alpha / alpha_next) * (1 - alpha_next) / (1 - alpha)).sqrt()
    c = ((1 - alpha_next) - sigma ** 2).sqrt()
    return torch.sqrt(1. / acp)[t], torch.sqrt(1. / acp - 1)[t], alpha_next.sqrt(), c, sigma


PAIRS = [(999, 949), (952, 904), (500, 450), (47, 0), (1, 0)]


@pytest.mark.parametrize("t,tn", PAIRS)
@pytest.mark.parametrize("eta", [1.0, 0.0])
@pytest.mark.parametrize("thres", [True, False], ids=["dynamic", "static"])
@pytest.mark.parametrize("with_noise", [True, False], ids=["noise", "no_noise"])
def test_ddim_step_equals_oracle(t, tn, eta, thres, with_noise):
    x, e, z = clip(t + 7 * tn, t)
    z = z if with_noise else None
    want = O.ddim_step(e, x, t, tn, z, eta=eta, dynamic_thres=thres)
    got = S.ddim_step(x, e, z if tn > 0 else None, oracle_ddim_coef(t, tn, eta), 0.9 if thres else 0.0)
    assert bits_equal(got, want)


@pytest.mark.parametrize("t", [999, 998, 500, 1, 0])
@pytest.mark.parametrize("q", [0.9, 0.0, -1.0])
@pytest.mark.parametrize("with_noise", [True, False], ids=["noise", "no_noise"])
def test_ddpm_step_equals_oracle(t, q, with_noise):
    x, e, z = clip(3 * t + 1, t)
    z = z if with_noise else None
    want = DO.ddpm_step(e, x, t, z, dynamic_thres=q > 0, clip_denoised=q >= 0)
    coef = diffusion().ddpm_table()[t]
    assert bits_equal(S.ddpm_step(x, e, z, coef, q), want)


@pytest.mark.parametrize("t,tn", PAIRS)
def test_ddim_coefficients_are_the_reference_buffers(t, tn):
    """ddim_coefficients reads sqrt_recip(m1)_alphas_cumprod from the buffers the reference registers (fp64 then fp32), which the
    kernels get; the oracle re-derives them in fp32 and may differ in the last bit, so the restatement takes them as given"""
    D = diffusion()
    ca, cb, san, c, sigma = D.ddim_coefficients(t, tn)
    assert (ca, cb) == (D.sqrt_recip_alphas_cumprod[t].item(), D.sqrt_recipm1_alphas_cumprod[t].item())
    assert (san, c, sigma) == tuple(v.item() for v in oracle_ddim_coef(t, tn, 1.0)[2:])


@pytest.mark.parametrize("scale", [0.0, 1.0, 2.0, 7.5])
def test_guided_eps_equals_oracle_combine(scale):
    """the oracle's module-level guidance (unet_forward_with_cond_scale) combines as null + (logits - null) * cond_scale"""
    g = torch.Generator().manual_seed(int(scale * 10))
    ec, en = torch.randn(3, 4, 8, 8, generator=g), torch.randn(3, 4, 8, 8, generator=g)
    assert bits_equal(S.guided_eps(ec, en, scale), en + (ec - en) * scale)


@pytest.mark.parametrize("q", [0.9, 0.0, -1.0])
def test_no_noise_adds_sigma_times_zero(q):
    """the last DDIM step adds sigma * 0. (U:1201), which turns a -0 sum into +0"""
    x = torch.tensor([-0.0, 0.0, 1.0])
    e = torch.tensor([-0.0, -0.0, 0.0])
    out = S.ddim_step(x, e, None, (1.0, 0.0, 1.0, 0.0, 0.0), q)
    assert out.view(torch.int32).tolist() == [0, 0, torch.tensor(1.0).view(torch.int32).item()]


NONFINITE = {
    "nan_key": ([1.0, float("nan"), 2.0, 3.0, 0.5], 0.9),
    "inf_minus_inf": ([0.5, 3.0, float("inf"), 2.0, 1.5], 0.9),        # lerp(3, inf, 0.6) = inf - inf
    "inf_pair_w0": ([1.0, float("inf"), float("inf")], 1.0),           # inf + 0 * (inf - inf)
    "inf_above_w_small": ([1.0] * 10 + [float("inf")], 0.92),          # vlo + w * inf = inf
}


@pytest.mark.parametrize("name", list(NONFINITE))
def test_nonfinite_thresholds_follow_torch(name):
    keys, q = NONFINITE[name]
    x = torch.tensor(keys)
    s = S.quantile_s(x, q).item()
    ref, *_ = S.order_stat_s(np.abs(keys), q)
    assert (np.isnan(s) and np.isnan(ref)) or s == ref, (s, ref)
    out = S.clip_x0(x, q)
    assert bool(torch.isnan(out).all()) == np.isnan(s)


def test_order_stat_s_of_replicas_is_the_quantile_of_the_copies():
    g = torch.Generator().manual_seed(5)
    x = torch.tensor([1.5, 2.0, 3.0, 7.0, 9.0])[torch.randint(0, 5, (1001,), generator=g)] * torch.rand(1001, generator=g)
    for W in (1, 2, 3):
        for q in (0.9, 0.5, 0.37):
            s, *_ = S.order_stat_s(x.abs().numpy(), q, W)
            t = S.quantile_s(x.repeat(W), q).item()
            assert abs(s - t) <= np.spacing(np.float32(s)), (W, q, s, t)


# ------------------------------------------------------------------------------------------------------------------ refusals
FAKE = 0x10000                                                      # never dereferenced: every case below is refused first


def _run(**kw):
    from dawn_pytorch_b200 import _lib as L
    c = L.DawnKernelCase()
    for k, v in kw.items():
        setattr(c, k, v)
    rc = L.lib.dawn_test_kernel(ctypes.byref(c), None)
    return rc, L.lib.dawn_last_error().decode()


DDIM, DDPM = 13, 14
STEP = dict(xs=FAKE, e=FAKE, scratch=FAKE, n=1000)
REFUSED = [
    ("ddim no x", DDIM, dict(STEP, xs=None), "missing pointer"),
    ("ddim no eps", DDIM, dict(STEP, e=None), "missing pointer"),
    ("ddpm no scratch", DDPM, dict(STEP, scratch=None), "missing pointer"),
    ("ddpm table without slot", DDPM, dict(STEP, tab=FAKE, num_t=1000), "missing pointer"),
    ("ddim n 0", DDIM, dict(STEP, n=0), "bad geometry"),
    ("ddpm n -1", DDPM, dict(STEP, n=-1), "bad geometry"),
    ("ddim replicas -1", DDIM, dict(STEP, replicas=-1), "bad geometry"),
    ("ddim replicas x n = 2^32", DDIM, dict(STEP, n=1 << 22, replicas=1 << 10), "bad geometry"),
    ("ddpm replicas x n over 2^32", DDPM, dict(STEP, n=2457600, replicas=1748), "bad geometry"),
    ("ddpm table of 0 rows", DDPM, dict(STEP, tab=FAKE, t_slot=FAKE, num_t=0), "bad geometry"),
]


@pytest.mark.parametrize("name,kernel,kw,why", REFUSED, ids=[r[0] for r in REFUSED])
def test_sampler_step_refusals_without_gpu(name, kernel, kw, why):
    rc, msg = _run(kernel=kernel, **kw)
    assert rc == -1 and msg == f"dawn_test_kernel: {why}", (rc, msg)
