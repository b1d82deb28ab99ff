"""-m gpu: sampling from a real clip on the device — `dawn_q_sample` and `dawn_motion_to_latent` bit for bit against torch's fp32
ops and the REAL reference (tests/golden/resample.npz, oracle/make_golden_resample.py), both captured into a CUDA graph, the
suffix samplers (`ddim_sample_from`, `p_sample_loop_from`, `interpolate`) against ddim_sample / the golden / each other, and
FlowDiffusion's `real_video_latent` and `resample_video` end to end.

Two runs of the UNet on the same inputs may differ in the last bits: its GroupNorm sums are accumulated with atomics, in an order
that changes from run to run.  Where a sampler path is compared with another that issues the same launches on the same values
(the CPU tests check the call sequences), the bound is the one the existing DDIM and DDPM graph tests use, 5e-5."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import lfg_motion_oracle as M
from oracle import weights as W
from oracle.make_golden_resample import x0_latent
from tests import gpu_common as G

pytestmark = pytest.mark.gpu
CASE = (23, 16, 16)                          # the 'odd' clip


def _gold():
    return np.load(os.path.join(G.ROOT, "tests", "golden", "resample.npz"))


def _diffusion(timesteps=1000, sampling_timesteps=20):
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion
    D = DynamicNfGaussianDiffusion(denoise_fn=G.cuda_net(), num_frames=40, image_size=32, sampling_timesteps=sampling_timesteps,
                                   timesteps=timesteps, loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1,
                                   ddim_sampling_eta=1.0).cuda()
    D.update_num_frames(CASE[0])
    return D


def _noise(tag):
    def noise_fn(k, shape):
        return torch.from_numpy(W.pseudo_normal(f"{tag}{k}", tuple(shape)))
    return noise_fn


def _odd():
    Fr, h, w = CASE
    _, fea, cond = W.synth_inputs("odd", Fr, h, w)
    return (1, 3, Fr, h, w), fea.cuda(), cond.cuda()


SAME = 5e-5                                 # two UNet runs on the same values (module docstring)


def _bits(a, b):
    a, b = torch.as_tensor(a).detach().cpu().contiguous(), torch.as_tensor(b).detach().cpu().contiguous()
    return int((a.view(torch.int32) != b.view(torch.int32)).sum())


def _same(a, b, what):
    d = (a - b).abs().max().item()
    print(f"{what}: max|d| {d:.3e}")
    assert d < SAME, what


def test_q_sample_is_bit_exact_with_torch_and_the_reference():
    """Per-clip t in a batch of 2 at t in {0, 1, 500, 998, 999}: the golden of the reference's q_sample, torch's CPU fp32 ops and
    the per-kernel test entry all agree to the bit."""
    from dawn_pytorch_b200 import _lib
    g = _gold()
    D = _diffusion()
    shape = tuple(int(v) for v in g["q_shape"])
    x0 = x0_latent(shape)
    z = torch.from_numpy(W.pseudo_normal("resample/q_noise", shape))
    a_cpu, b_cpu = D.sqrt_alphas_cumprod.cpu(), D.sqrt_one_minus_alphas_cumprod.cpu()
    for row, tt in enumerate(g["q_t"].tolist()):
        t = torch.tensor(tt)
        out = D.q_sample(x0.cuda(), t.cuda(), noise=z.cuda())
        torch_cpu = a_cpu[t].view(-1, 1, 1, 1, 1) * x0 + b_cpu[t].view(-1, 1, 1, 1, 1) * z
        assert _bits(out, g["q_out"][row]) == 0 and _bits(out, torch_cpu) == 0, tt
        case = _lib.DawnKernelCase()
        case.kernel, case.clips, case.n, case.num_t = _lib.KERNEL_Q_SAMPLE, shape[0], x0[0].numel(), D.num_timesteps
        xc, zc, tc, oc = x0.cuda(), z.cuda(), t.cuda(), torch.empty(shape, device="cuda")
        case.x, case.noise, case.t, case.out = xc.data_ptr(), zc.data_ptr(), tc.data_ptr(), oc.data_ptr()
        case.w, case.b = D.sqrt_alphas_cumprod.data_ptr(), D.sqrt_one_minus_alphas_cumprod.data_ptr()
        _lib.check(_lib.lib.dawn_test_kernel(ctypes.byref(case), _lib.stream()), "dawn_test_kernel")
        assert _bits(oc, torch_cpu) == 0
    # an int t serves every clip; the default noise is drawn on the device
    y = D.q_sample(x0.cuda(), 999)
    assert y.shape == shape and bool(torch.isfinite(y).all())


def test_motion_to_latent_is_bit_exact_and_fused_noising_equals_two_steps():
    from dawn_pytorch_b200 import _lib
    D = _diffusion()
    gen = torch.Generator().manual_seed(3)
    B, Fr, h, w = 3, 5, 8, 12
    flow = torch.randn(B * Fr, h, w, 2, generator=gen)
    occ = torch.rand(B * Fr, 1, h, w, generator=gen)
    ref = torch.cat([flow.view(B, Fr, h, w, 2).permute(0, 4, 1, 2, 3), occ.view(B, Fr, 1, h, w).permute(0, 2, 1, 3, 4) * 2 - 1], dim=1)
    x0 = D.motion_to_latent(flow.cuda(), occ.cuda(), Fr)
    assert x0.shape == (B, 3, Fr, h, w) and _bits(x0, ref) == 0
    t = torch.tensor([0, 500, 999])
    z = torch.randn(B, 3, Fr, h, w, generator=gen)
    fused = D.motion_to_latent(flow.cuda(), occ.cuda(), Fr, t=t.cuda(), noise=z.cuda())
    two = D.q_sample(x0, t.cuda(), noise=z.cuda())
    assert _bits(fused, two) == 0
    case = _lib.DawnKernelCase()
    case.kernel, case.clips, case.F, case.H, case.W = _lib.KERNEL_MOTION_TO_LATENT, B, Fr, h, w
    fc, oc, out = flow.cuda(), occ.cuda(), torch.empty(B, 3, Fr, h, w, device="cuda")
    case.x, case.y, case.out = fc.data_ptr(), oc.data_ptr(), out.data_ptr()
    _lib.check(_lib.lib.dawn_test_kernel(ctypes.byref(case), _lib.stream()), "dawn_test_kernel")
    assert _bits(out, ref) == 0


def test_q_sample_and_fused_pass_capture_into_a_cuda_graph():
    """Neither entry synchronises with the host: both are captured into one torch CUDA graph, and its replay on new inputs
    equals the eager calls."""
    D = _diffusion()
    gen = torch.Generator().manual_seed(4)
    B, Fr, h, w = 2, 4, 8, 8
    x0, z = torch.randn(B, 3, Fr, h, w, device="cuda"), torch.randn(B, 3, Fr, h, w, device="cuda")
    flow, occ = torch.randn(B * Fr, h, w, 2, device="cuda"), torch.rand(B * Fr, 1, h, w, device="cuda")
    t = torch.tensor([10, 900], device="cuda")
    D.q_sample(x0, t, noise=z)                                           # warm-up outside the capture
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g):
            y1 = D.q_sample(x0, t, noise=z)
            y2 = D.motion_to_latent(flow, occ, Fr, t=t, noise=z)
    torch.cuda.current_stream().wait_stream(side)
    x0.copy_(torch.randn(x0.shape, generator=gen))
    flow.copy_(torch.randn(flow.shape, generator=gen))
    t.copy_(torch.tensor([999, 0]))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y1, D.q_sample(x0, t, noise=z))
    assert torch.equal(y2, D.motion_to_latent(flow, occ, Fr, t=t, noise=z))


@pytest.mark.parametrize("path", ["eager", "graph", "guided_graph"])
def test_ddim_sample_from_start_zero_equals_ddim_sample(path):
    D = _diffusion()
    shape, fea, cond = _odd()
    x_t = torch.from_numpy(W.pseudo_normal("resample/start0", shape))
    noise = _noise("resample/start0_")

    def with_start(k, shp):
        return x_t.clone() if k < 0 else noise(k, shp)
    kw = dict(cond_scale=2.0 if path == "guided_graph" else 1.0, use_graph=path != "eager")
    a = D.ddim_sample(fea, shape, cond=cond, noise_fn=with_start, **kw).clone()
    b = D.ddim_sample_from(x_t, 0, fea, cond=cond, noise_fn=noise, **kw)
    torch.cuda.synchronize()
    _same(a, b, f"ddim_sample_from(start=0) vs ddim_sample, {path}")


def test_ddim_suffix_matches_golden_and_graph_matches_eager():
    g = _gold()
    D = _diffusion()
    shape, fea, cond = _odd()
    start = int(g["ddim_start"])
    pairs = D.ddim_schedule()
    assert [tuple(p) for p in g["ddim_pairs"].tolist()] == pairs[start:]
    x0 = x0_latent(shape)
    x_t = D.q_sample(x0.cuda(), torch.full((1,), pairs[start][0]), noise=torch.from_numpy(W.pseudo_normal("resample/ddim_q", shape)))
    noise = _noise("resample/ddim")
    eager = D.ddim_sample_from(x_t, start, fea, cond=cond, noise_fn=noise)
    graph = D.ddim_sample_from(x_t, start, fea, cond=cond, noise_fn=noise, use_graph=True)
    torch.cuda.synchronize()
    ref = torch.from_numpy(g["ddim_out"][-1])
    d_e, d_g, d_ge = (eager.cpu() - ref).abs().max().item(), (graph.cpu() - ref).abs().max().item(), (graph - eager).abs().max().item()
    print(f"ddim suffix from step {start}: eager vs golden {d_e:.3e}, graph vs golden {d_g:.3e}, graph vs eager {d_ge:.3e}")
    assert d_e < 2e-4 and d_g < 2e-4 and d_ge < 5e-5
    # the caller's x_t is not modified: a second run from it gives the same sample
    one = D.ddim_sample_from(x_t, start, fea, cond=cond, noise_fn=noise)
    _same(one, eager, "second eager run")


def test_p_sample_loop_from_matches_golden_and_graph_matches_eager():
    g = _gold()
    D = _diffusion(sampling_timesteps=None)
    shape, fea, cond = _odd()
    t = int(g["anc_t"])
    x_t = D.q_sample(x0_latent(shape).cuda(), t, noise=torch.from_numpy(W.pseudo_normal("resample/anc_q", shape)))
    noise = _noise("resample/anc")
    eager = D.p_sample_loop_from(x_t, t, fea, cond=cond, noise_fn=noise)
    graph = D.p_sample_loop_from(x_t, t, fea, cond=cond, noise_fn=noise, use_graph=True)
    torch.cuda.synchronize()
    ref = torch.from_numpy(g["anc_out"])
    d_e, d_ge = (eager.cpu() - ref).abs().max().item(), (graph - eager).abs().max().item()
    print(f"ancestral from t={t}: eager vs golden {d_e:.3e}, graph vs eager {d_ge:.3e}")
    assert d_e < 1e-3 and d_ge < 5e-5
    with pytest.raises(NotImplementedError):
        D.p_sample_loop_from(x_t, t, fea, cond=cond, cond_scale=2.0, use_graph=True)


def test_interpolate_lam_zero_is_q_sample_and_loop_of_x1():
    D = _diffusion(timesteps=6, sampling_timesteps=None)
    shape, fea, cond = _odd()
    x1, x2 = x0_latent(shape), torch.tanh(torch.from_numpy(W.pseudo_normal("resample/x2", shape)))
    noise = _noise("resample/interp")
    out = D.interpolate(x1, x2, fea, cond=cond, lam=0.0, noise_fn=noise)
    xt1 = D.q_sample(x1, D.num_timesteps - 1, noise=noise(-2, shape))
    ref = D.p_sample_loop_from(xt1, D.num_timesteps - 1, fea, cond=cond, noise_fn=noise)
    torch.cuda.synchronize()
    _same(out, ref, "interpolate(lam=0) vs q_sample + p_sample_loop_from")
    mixed = D.interpolate(x1, x2, fea, cond=cond, lam=0.5, noise_fn=noise, use_graph=True)
    assert bool(torch.isfinite(mixed).all()) and (mixed - out).abs().max().item() > 1e-3


def _flowae():
    import json
    from dawn_pytorch_b200 import FlowAE
    with open(os.path.join(G.ROOT, "tests", "golden", "lfg_motion_schema.json")) as f:
        sch = json.load(f)
    ae = FlowAE(is_train=False)
    for k in ("region_predictor", "bg_predictor", "generator"):
        getattr(ae, k).load_state_dict(M.motion_synth_state_dict([(n, tuple(s)) for n, s in sch[k]]))
    return ae.cuda()


def test_real_video_latent_matches_reference_golden():
    from dawn_pytorch_b200 import FlowDiffusion
    g = _gold()
    b, f, hw = (int(v) for v in g["motion"])
    real_vid = torch.stack([M.motion_synth_inputs(f"resample/clip{i}", f, hw, hw)[1].permute(1, 0, 2, 3) for i in range(b)]).cuda()
    ref_img = real_vid[:, :, 0].clone()
    ae = _flowae()
    m = FlowDiffusion(sampling_timesteps=20, pose_dim=6).cuda()
    n_keys = len(m.state_dict())
    x0 = m.real_video_latent(real_vid, ref_img, ae)
    x0_parts = m.real_video_latent(real_vid, ref_img, (ae.region_predictor, ae.bg_predictor, ae.generator))
    torch.cuda.synchronize()
    assert len(m.state_dict()) == n_keys and torch.equal(x0, x0_parts)
    ref = torch.from_numpy(g["motion_latent"])
    assert x0.shape == ref.shape
    r_grid = G.over_tol(x0[:, :2], ref[:, :2])
    r_occ = G.over_tol((x0[:, 2] + 1) * 0.5, (ref[:, 2] + 1) * 0.5)      # the occlusion map, at the motion tests' tolerance
    print(f"real_video_latent: grid {r_grid:.3f} x tol, occlusion {r_occ:.3f} x tol")
    assert r_grid <= 1.0 and r_occ <= 1.0


def test_resample_video_runs_end_to_end_and_its_latent_is_ddim_sample_from():
    from oracle.make_golden_e2e import e2e_inputs
    from tests.test_e2e_gpu import build_model
    g = np.load(os.path.join(G.ROOT, "tests", "golden", "e2e_sample_one_video.npz"))
    nf, size = int(g["frames"]), int(g["image"])
    m = build_model(20)
    m.update_num_frames(nf)
    img, hubert, pose, eye, bbox, init_pose, init_eye = [t.cuda() for t in e2e_inputs()]
    shape = (1, 3, nf, size // 4, size // 4)
    x0 = x0_latent(shape).cuda()
    noise = _noise("resample/video")
    start = 15
    out = m.resample_video(img, x0, hubert, pose, eye, bbox, 1.0, start, init_pose=init_pose, init_eye=init_eye, noise_fn=noise)
    D = m.diffusion
    fea272, ref_text = m._conditioning(img, hubert, pose, eye, bbox, init_pose, init_eye)
    x_t = D.q_sample(x0, D.ddim_schedule()[start][0], noise=noise(-1, shape))
    pred = D.ddim_sample_from(x_t, start, fea272, cond=ref_text, noise_fn=noise)
    torch.cuda.synchronize()
    _same(out["sample_vid_grid"], pred[:, :2], "resample_video grid vs ddim_sample_from")
    _same(out["sample_vid_conf"], (pred[:, 2].unsqueeze(1) + 1) * 0.5, "resample_video conf vs ddim_sample_from")
    assert out["sample_out_vid"].shape == out["sample_warped_vid"].shape == (1, 3, nf, size, size)
    assert all(bool(torch.isfinite(v).all()) for v in out.values())
    # the later the start, the closer the sample stays to the clip's own motion
    late = m.resample_video(img, x0, hubert, pose, eye, bbox, 1.0, 19, init_pose=init_pose, init_eye=init_eye, noise_fn=noise)
    d_late = (late["sample_vid_grid"] - x0[:, :2]).abs().mean().item()
    d_early = (m.resample_video(img, x0, hubert, pose, eye, bbox, 1.0, 0, init_pose=init_pose, init_eye=init_eye,
                                noise_fn=noise)["sample_vid_grid"] - x0[:, :2]).abs().mean().item()
    print(f"resample_video: mean |grid - x0 grid| start 19 {d_late:.4f}, start 0 {d_early:.4f}")
    assert d_late < d_early
