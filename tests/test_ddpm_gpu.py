"""-m gpu: the ancestral (DDPM) sampler on the CUDA UNet — single p_sample steps of the 1000-step schedule and whole 6-step
p_sample_loops against the REAL reference (tests/golden/ddpm_odd.npz, oracle/make_golden_ddpm.py, injected noise), the step graph
against the eager loop, the handle entry against the plain one and torch's arithmetic, and FlowDiffusion's ancestral path.

Error bound of one step.  x0 = ca*x - cb*eps with ca ~ cb ~ 64166 at t = 999, so an eps error d becomes an x0 error of cb*d.
The dynamic threshold divides it back out: s = max(1, quantile_0.9 |x0|) moves by at most cb*d (an order statistic is
1-Lipschitz in the max norm), and clamp(x0, -s, s)/s moves by at most cb*d*(1 + max|x0|/s)/s.  The sample moves by c1 times
that, since c2*x and the noise term are exact.  The tests compute this bound from the measured eps error of the CUDA UNet."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import weights as W
from tests import gpu_common as G

pytestmark = pytest.mark.gpu
CASE = (23, 16, 16)                          # the 'odd' clip


def _gold():
    return np.load(os.path.join(G.ROOT, "tests", "golden", "ddpm_odd.npz"))


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _diffusion(timesteps, sampling_timesteps=None):
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion
    D = DynamicNfGaussianDiffusion(denoise_fn=G.cuda_net(), num_frames=40, image_size=32, sampling_timesteps=sampling_timesteps,
                                   timesteps=timesteps, loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1,
                                   ddim_sampling_eta=1.0).cuda()
    D.update_num_frames(CASE[0])
    return D


def _loop_noise(tag):
    Fr, h, w = CASE

    def noise_fn(k, shape):
        v = torch.from_numpy(W.pseudo_normal(f"{tag}/noise{k}", (1, 3, Fr, h, w)))
        return v if k < 0 else v[0]
    return noise_fn


def test_single_steps_of_the_1000_step_schedule_match_reference_golden():
    """p_sample at t = 999, 998, 500, 1, 0 from one fixed x.  First the update kernel alone, fed the reference's own eps:
    it repeats the reference's fp32 roundings.  Then the whole step with the CUDA UNet, within the bound of the module
    docstring."""
    from dawn_pytorch_b200._lib import check, lib
    g = _gold()
    D = _diffusion(1000)
    net = D.denoise_fn
    Fr, h, w = CASE
    _, fea, cond = W.synth_inputs("odd", Fr, h, w)
    fea_c, cond_c = fea.cuda(), cond.cuda()
    x = torch.from_numpy(W.pseudo_normal("ddpm1000/x", (1, 3, Fr, h, w)))
    n = x.numel()
    scratch = torch.empty(n + 512, dtype=torch.int32, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for j, t in enumerate(g["single_t"].tolist()):
        noise = torch.from_numpy(W.pseudo_normal(f"ddpm1000/noise{t}", (1, 3, Fr, h, w)))
        ref, eps_ref = torch.from_numpy(g["single_x_after"][j]), torch.from_numpy(g["single_eps"][j])
        ca, cb, c1, c2, sigma = D.ddpm_coefficients(t)
        xa, ea, na = x[0].cuda().contiguous(), eps_ref[0].cuda().contiguous(), noise[0].cuda().contiguous()
        check(lib.dawn_ddpm_step(_ptr(xa), _ptr(ea), _ptr(na), n, ca, cb, c1, c2, sigma, 0.9, _ptr(scratch), st), "dawn_ddpm_step")
        torch.cuda.synchronize()
        d_kernel = (xa.cpu() - ref[0]).abs().max().item()
        y = D.p_sample(x.cuda(), torch.full((1,), t, device="cuda"), fea_c, cond=cond_c, noise=noise.cuda())
        net.set_clip_invariants(fea_c[0], cond_c[0])
        eps = net.forward_x3(x[0].cuda().contiguous(), torch.full((1,), t, dtype=torch.long, device="cuda"))
        torch.cuda.synchronize()
        d_eps = (eps.cpu() - eps_ref[0]).abs().max().item()
        x0 = ca * x - cb * eps_ref
        s = max(1.0, torch.quantile(x0.abs().reshape(-1), 0.9).item())
        bound = c1 * cb * d_eps * (1 + x0.abs().max().item() / s) / s * 1.01 + 2e-6
        d = (y.cpu() - ref).abs().max().item()
        print(f"p_sample t={t}: kernel on the reference eps max|d| {d_kernel:.2e}; CUDA UNet eps max|d| {d_eps:.2e} "
              f"-> sample max|d| {d:.2e} (bound {bound:.2e}, s = {s:.4g})")
        assert d_kernel <= 1e-6
        assert G.over_tol(eps, eps_ref[0]) <= 1.0
        assert d <= bound


@pytest.mark.parametrize("scale", [1.0, 2.0])
def test_six_step_loops_match_reference_golden(scale):
    """The whole p_sample_loop of a 6-step schedule, with cond_scale 1 and 2 (two hoisted forwards per step).  Each step adds
    at most the bound of the module docstring (at the UNet's 1e-4 eps tolerance <= ~1.5e-4 here, as cb/s <= 1/quantile(|x-eps|)
    and c1 < 0.75), and an error already in x is carried on by c1*ca/s + c2 < 1, so six steps stay under 1e-3."""
    g = _gold()
    D = _diffusion(int(g["loop_t"]))
    Fr, h, w = CASE
    _, fea, cond = W.synth_inputs("odd", Fr, h, w)
    img = D.p_sample_loop(fea.cuda(), (1, 3, Fr, h, w), cond=cond.cuda(), cond_scale=scale,
                          noise_fn=_loop_noise(f"ddpm6_cs{int(scale)}"))
    torch.cuda.synchronize()
    d = (img.cpu() - torch.from_numpy(g[f"loop_cs{int(scale)}"])).abs().max().item()
    print(f"p_sample_loop T=6 cond_scale={scale}: max|d| vs reference {d:.3e}")
    assert d < 1e-3
    if scale == 1.0:
        # sample() with sampling_timesteps=None runs this loop (U:1150) with the default noise
        out = D.sample(fea[:, :256].cuda(), fea[:, 256:].cuda(), cond=cond.cuda())
        assert out.shape == (1, 3, Fr, h, w) and bool(torch.isfinite(out).all())


def test_step_graph_equals_eager_loop_and_keeps_the_ddim_graph():
    """use_graph: one captured step (forward_x3 + update + slot advance) replayed T times == the eager loop; a second clip
    replays the cached graph; a DDIM whole-loop graph captured on the same UNet before it is still replayable after it."""
    Fr, h, w = CASE
    _, fea, cond = W.synth_inputs("odd", Fr, h, w)
    fea_c, cond_c = fea.cuda(), cond.cuda()
    D = _diffusion(6)
    Dd = _diffusion(1000, sampling_timesteps=20)
    pairs = [Dd.ddim_schedule()[i] for i in (0, 10, 19)]
    ddim_noise = _loop_noise("ddpmgraph/ddim")
    a = Dd.ddim_sample(fea_c, (1, 3, Fr, h, w), cond=cond_c, noise_fn=ddim_noise, pairs=pairs, use_graph=True).clone()
    gen_ddim = Dd._graph["gen"]
    noise_fn = _loop_noise("ddpm6_cs1")
    eager = D.p_sample_loop(fea_c, (1, 3, Fr, h, w), cond=cond_c, noise_fn=noise_fn).clone()
    graph = D.p_sample_loop(fea_c, (1, 3, Fr, h, w), cond=cond_c, noise_fn=noise_fn, use_graph=True).clone()
    torch.cuda.synchronize()
    n_launch = D.denoise_fn.last_launch_count()
    ref = torch.from_numpy(_gold()["loop_cs1"])
    print(f"ddpm step graph: vs eager {(graph - eager).abs().max():.3e}, vs golden {(graph.cpu() - ref).abs().max():.3e}, "
          f"{n_launch} UNet launches per replay")
    assert (graph - eager).abs().max().item() < 5e-5
    assert (graph.cpu() - ref).abs().max().item() < 1e-3
    assert n_launch >= 200
    gen0 = D._ddpm_graph["gen"]
    # the DDIM graph was not evicted by the DDPM capture: it replays without a re-capture and gives the same sample
    b = Dd.ddim_sample(fea_c, (1, 3, Fr, h, w), cond=cond_c, noise_fn=ddim_noise, pairs=pairs, use_graph=True).clone()
    assert Dd._graph["gen"] == gen_ddim and (a - b).abs().max().item() < 5e-5
    # a second clip (other conditioning) replays the cached step graph
    cond2 = cond.flip(1).contiguous().cuda()
    e2 = D.p_sample_loop(fea_c, (1, 3, Fr, h, w), cond=cond2, noise_fn=noise_fn).clone()
    g2 = D.p_sample_loop(fea_c, (1, 3, Fr, h, w), cond=cond2, noise_fn=noise_fn, use_graph=True).clone()
    torch.cuda.synchronize()
    assert D._ddpm_graph["gen"] == gen0
    assert (g2 - e2).abs().max().item() < 5e-5
    assert (g2 - graph).abs().max().item() > 1e-3
    with pytest.raises(NotImplementedError):
        D.p_sample_loop(fea_c, (1, 3, Fr, h, w), cond=cond_c, cond_scale=2.0, noise_fn=noise_fn, use_graph=True)


@pytest.mark.parametrize("q", [0.9, 0.0, -1.0])
def test_handle_ddpm_step_equals_plain_entry_unsharded(q):
    """dawn_unet_ddpm_step on an unsharded handle is dawn_ddpm_step; both equal torch's arithmetic of U:1072-1121 (dynamic
    threshold, static clamp to [-1, 1], no clip)."""
    from dawn_pytorch_b200._lib import check, lib
    net = G.cuda_net()
    net.update_num_frames(8)
    _, _, cond, _, fea = G.clip("smoke", 8, 8, 8, 500)
    net.set_clip_invariants(fea[0].cuda(), cond[0].cuda())          # makes sure the handle exists
    gen = torch.Generator().manual_seed(7)
    n = 3 * 37 * 16 * 16
    xr = torch.randn(n, generator=gen) * 1.5
    e, nz = torch.randn(n, generator=gen), torch.randn(n, generator=gen)
    xa, xb, eps, noise = xr.cuda(), xr.cuda(), e.cuda(), nz.cuda()
    scratch = torch.empty(n + 512, dtype=torch.int32, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ca, cb, c1, c2, sigma = 3.7, 3.5, 0.3, 0.6, 0.2
    args = (n, ca, cb, c1, c2, sigma, q, _ptr(scratch), st)
    check(lib.dawn_ddpm_step(_ptr(xa), _ptr(eps), _ptr(noise), *args), "dawn_ddpm_step")
    check(lib.dawn_unet_ddpm_step(net._handle, _ptr(xb), _ptr(eps), _ptr(noise), *args), "dawn_unet_ddpm_step")
    torch.cuda.synchronize()
    assert torch.equal(xa, xb)
    f = torch.float32
    x0 = torch.tensor(ca, dtype=f) * xr - torch.tensor(cb, dtype=f) * e
    if q >= 0:
        s = torch.quantile(x0.abs(), q).clamp(min=1.0) if q > 0 else torch.tensor(1.0)
        x0 = x0.clamp(-s, s) / s
    ref = torch.tensor(c1, dtype=f) * x0 + torch.tensor(c2, dtype=f) * xr + torch.tensor(sigma, dtype=f) * nz
    d = (xa.cpu() - ref).abs().max().item()
    print(f"ddpm step q={q}: max|d| vs torch {d:.2e}")
    assert d < 2e-6
    # noise = NULL: the t = 0 form
    xc = xr.cuda()
    check(lib.dawn_ddpm_step(_ptr(xc), _ptr(eps), None, *args), "dawn_ddpm_step")
    torch.cuda.synchronize()
    assert (xc.cpu() - (ref - torch.tensor(sigma, dtype=f) * nz)).abs().max().item() < 2e-6


def test_flow_diffusion_runs_the_ancestral_loop():
    """FlowDiffusion(sampling_timesteps=1000) (`sampling_step: 1000` in DAWN's configs) samples with p_sample_loop:
    sample_one_video == compute_fea + face-box embedding + p_sample_loop + decode_sample with the same noise."""
    from dawn_pytorch_b200 import FlowDiffusion
    from oracle import lfg_oracle as L
    from oracle.make_golden_e2e import e2e_inputs, face_sd
    m = FlowDiffusion(sampling_timesteps=1000, pose_dim=6, win_width=40, ddim_sampling_eta=1.0)
    assert not m.diffusion.is_ddim_sampling
    m.diffusion.load_state_dict({**{"denoise_fn." + k: v for k, v in G.synth_sd().items()},
                                 **{k: v for k, v in m.diffusion.state_dict().items() if not k.startswith("denoise_fn.")}}, strict=True)
    m.generator.load_state_dict(W.lfg_synth_state_dict(L.state_dict_schema()), strict=True)
    m.face_loc_emb.load_state_dict(face_sd(), strict=True)
    m = m.cuda()
    img, hubert, pose, eye, bbox, init_pose, init_eye = [t.cuda() for t in e2e_inputs()]
    nf, size = hubert.shape[1], img.shape[-1]
    m.update_num_frames(nf)

    def noise_fn(k, shape):
        return torch.from_numpy(W.pseudo_normal(f"ddpm_e2e/noise{k}", tuple(shape)))

    out = m.sample_one_video(sample_img=img, sample_audio_hubert=hubert, sample_pose=pose, sample_eye=eye, sample_bbox=bbox,
                             init_pose=init_pose, init_eye=init_eye, cond_scale=1.0, noise_fn=noise_fn)
    # the same pipeline from its pieces (FD:325-383)
    fea = m.generator.compute_fea(img)
    face = m.face_loc_emb(m.generate_bbox_mask(bbox, size=size))
    ref_pose, ref_eye = pose[:, :6].permute(0, 2, 1), eye.permute(0, 2, 1)
    ref_text = torch.cat([hubert, ref_pose - init_pose.unsqueeze(1).repeat(1, nf, 1), ref_eye - init_eye.unsqueeze(1).repeat(1, nf, 1)], -1)
    h, w = fea.shape[-2:]
    pred = m.diffusion.p_sample_loop(torch.cat([fea, face], 1), (1, 3, nf, h, w), cond=ref_text, cond_scale=1.0, noise_fn=noise_fn)
    vid, warped = m.generator.decode_sample(img, pred[0], need_deformed=True)
    torch.cuda.synchronize()
    d_grid = (out["sample_vid_grid"] - pred[:, :2]).abs().max().item()
    d_vid = (out["sample_out_vid"][0] - vid.permute(1, 0, 2, 3)).abs().max().item()
    d_warp = (out["sample_warped_vid"][0] - warped.permute(1, 0, 2, 3)).abs().max().item()
    print(f"FlowDiffusion ancestral (1000 steps, {nf} f): grid max|d| {d_grid:.2e}, video {d_vid:.2e}, warped {d_warp:.2e}")
    assert out["sample_out_vid"].shape == (1, 3, nf, size, size)
    assert d_grid < 1e-4 and d_vid < 1e-3 and d_warp < 1e-3
