"""-m gpu: classifier-free-guided DDIM sampling as one CUDA graph (`ddim_sample(use_graph=True, cond_scale != 1)`): each step is
one UNet pass over the conditioned clips and their all-zero-cond twins plus one fused guided update
(`dawn_unet_sampler_capture_guided` / `dawn_unet_ddim_step_guided`).  Against the real reference's guided sampler (golden),
the eager guided loop, each clip sampled alone, torch's fp32 arithmetic of one update, and the plain graph held beside it."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dawn_pytorch_b200 import _lib
from oracle import weights as W
from tests import gpu_common as G

pytestmark = pytest.mark.gpu


def _sampler(steps, F):
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion
    net = G.cuda_net()
    D = DynamicNfGaussianDiffusion(denoise_fn=net, num_frames=40, image_size=32, sampling_timesteps=steps, timesteps=1000,
                                   loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0).cuda()
    D.update_num_frames(F)
    return D, net


def _cfg_golden():
    g = np.load(os.path.join(G.ROOT, "tests", "golden", "ddim_cfg2_odd.npz"))
    F, h, w, _ = G.CASES["odd"]
    _, fea, cond = W.synth_inputs("odd", F, h, w)
    D, net = _sampler(int(g["steps"]), F)

    def noise_fn(k, shape):
        return torch.from_numpy(W.pseudo_normal(f"cfg2/noise{k}", tuple(shape)))
    return g, D, net, (F, h, w), fea.cuda(), cond.cuda(), noise_fn


def test_guided_graph_matches_reference_golden_and_eager():
    g, D, net, (F, h, w), fea, cond, noise_fn = _cfg_golden()
    scale = float(g["cond_scale"])
    eager = D.ddim_sample(fea, (1, 3, F, h, w), cond=cond, cond_scale=scale, noise_fn=noise_fn).clone()
    graph = D.ddim_sample(fea, (1, 3, F, h, w), cond=cond, cond_scale=scale, noise_fn=noise_fn, use_graph=True).clone()
    torch.cuda.synchronize()
    assert net.clip_count() == 2                             # the clip and its null twin in one pass
    d = (graph.cpu() - torch.from_numpy(g["sample"])).abs().max().item()
    r = G.over_tol(graph, eager)
    print(f"guided graph (cond_scale {scale}): vs golden max|d| {d:.3e}, vs eager {r:.4f} x tol, "
          f"{net.last_launch_count()} kernel launches in one graph")
    assert d < 2e-4
    assert r <= 0.05


def test_one_capture_serves_every_cond_scale():
    g, D, net, (F, h, w), fea, cond, noise_fn = _cfg_golden()
    D.ddim_sample(fea, (1, 3, F, h, w), cond=cond, cond_scale=2.0, noise_fn=noise_fn, use_graph=True)
    captures, gen, graph_gen = D._guided_captures, D._guided_graph["gen"], net.graph_generation()
    y3 = D.ddim_sample(fea, (1, 3, F, h, w), cond=cond, cond_scale=3.0, noise_fn=noise_fn, use_graph=True).clone()
    torch.cuda.synchronize()
    assert D._guided_captures == captures and D._guided_graph["gen"] == gen and net.graph_generation() == graph_gen
    e3 = D.ddim_sample(fea, (1, 3, F, h, w), cond=cond, cond_scale=3.0, noise_fn=noise_fn).clone()
    r3 = G.over_tol(y3, e3)
    print(f"cond_scale 3 on the cached capture: vs eager {r3:.4f} x tol")
    assert r3 <= 0.05
    # cond_scale = 1 is the plain loop: its own graph, no guided capture
    D._graph = None
    y1 = D.ddim_sample(fea, (1, 3, F, h, w), cond=cond, cond_scale=1.0, noise_fn=noise_fn, use_graph=True).clone()
    assert D._graph is not None and D._guided_captures == captures
    e1 = D.ddim_sample(fea, (1, 3, F, h, w), cond=cond, cond_scale=1.0, noise_fn=noise_fn).clone()
    assert G.over_tol(y1, e1) <= 0.05
    assert (y1 - y3).abs().max().item() > 1e-3


def _two_clips(F, h, w):
    per = [G.clip(f"odd/sample{i}", F, h, w, 47) for i in range(2)]
    fea = torch.cat([p[4] for p in per]).cuda()
    cond = torch.cat([p[2] for p in per]).cuda()
    gen = torch.Generator().manual_seed(1)
    noise = {k: torch.randn(2, 3, F, h, w, generator=gen) for k in range(-1, 3)}
    noise[-1][1] *= 3.0                                      # the clips' quantiles differ
    return fea, cond, noise


def test_batched_guided_graph_equals_each_clip_alone():
    F, h, w, _ = G.CASES["odd"]
    D, net = _sampler(3, F)
    fea, cond, noise = _two_clips(F, h, w)
    yb = D.ddim_sample(fea, (2, 3, F, h, w), cond=cond, cond_scale=2.0, noise_fn=lambda k, s: noise[k].clone(), use_graph=True).cpu()
    assert net.clip_count() == 4 and D._guided_graph["key"][-1] == 2        # one 4-clip pass per step
    for i in range(2):
        yi = D.ddim_sample(fea[i:i + 1], (1, 3, F, h, w), cond=cond[i:i + 1], cond_scale=2.0,
                           noise_fn=lambda k, s: noise[k][i].reshape(s).clone(), use_graph=True).cpu()
        r = G.over_tol(yb[i:i + 1], yi)
        print(f"guided graph, clip {i}: batched vs alone {r:.4f} x tol")
        assert r <= 0.05


def test_guided_graph_keeps_the_plain_graph_of_the_same_geometry():
    """A plain graph over 2 clips and a guided graph over 1 clip both run B = 2: each has its own slot in the handle."""
    F, h, w, _ = G.CASES["odd"]
    D, net = _sampler(3, F)
    fea, cond, noise = _two_clips(F, h, w)
    a = D.ddim_sample(fea, (2, 3, F, h, w), cond=cond, noise_fn=lambda k, s: noise[k].clone(), use_graph=True).clone()
    plain, gen = D._graph, net.graph_generation()
    D.ddim_sample(fea[:1], (1, 3, F, h, w), cond=cond[:1], cond_scale=2.0, noise_fn=lambda k, s: noise[k][0].reshape(s).clone(),
                  use_graph=True)
    assert net.clip_count() == 2 and net.graph_generation() == gen
    b = D.ddim_sample(fea, (2, 3, F, h, w), cond=cond, noise_fn=lambda k, s: noise[k].clone(), use_graph=True).clone()
    torch.cuda.synchronize()
    assert D._graph is plain and D._graph["gen"] == gen                     # no re-capture
    assert (a - b).abs().max().item() < 5e-5


def _ref_update(x, ec, en, noise, s, coef, q):
    """torch fp32, one clip: forward_with_cond_scale (U:879-890) then the DDIM update (U:1169-1205)."""
    ca, cb, san, c, sigma = coef
    e = en + (ec - en) * s
    x0 = ca * x - cb * e
    if q > 0:
        t = torch.quantile(x0.reshape(-1).abs(), q).clamp(min=1.0)
        x0 = x0.clamp(-t, t) / t
    elif q == 0:
        x0 = x0.clamp(-1.0, 1.0)
    return x0 * san + c * e + sigma * noise


@pytest.mark.parametrize("q", [0.9, 0.0, -1.0])
def test_guided_update_against_torch(q):
    F, h, w = 8, 16, 16
    net = G.cuda_net()
    net.update_num_frames(F)
    per = [G.clip(f"guided/step{i}", F, h, w, 500) for i in range(2)]
    fea = torch.cat([p[4] for p in per] * 2).cuda()
    cond = torch.cat([p[2] for p in per] * 2).cuda()
    net.set_clip_invariants(fea, cond)                        # B = 4: two pairs
    n1 = 3 * F * h * w
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(4, 3, F, h, w, generator=gen) * 1.5
    x[1] *= 3.0
    eps = torch.randn(4, 3, F, h, w, generator=gen)
    noise = torch.randn(2, 3, F, h, w, generator=gen)
    coef, s = (1.3, 0.8, 0.9, 0.3, 0.2), 2.5
    xd, ed, nd = x.clone().cuda(), eps.cuda(), noise.cuda()
    scale = torch.tensor([s], device="cuda")
    scratch = torch.empty(n1 + 512, dtype=torch.int32, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    fp = lambda a: ctypes.c_void_p(a.data_ptr())             # noqa: E731
    _lib.check(_lib.lib.dawn_unet_ddim_step_guided(net._handle, fp(xd), fp(ed), fp(nd), n1, fp(scale), *coef, q, fp(scratch), st),
               "dawn_unet_ddim_step_guided")
    torch.cuda.synchronize()
    xd = xd.cpu()
    assert torch.equal(xd[:2], xd[2:])                       # both slots of a pair hold the new x
    for i in range(2):
        ref = _ref_update(x[i], eps[i], eps[2 + i], noise[i], s, coef, q)
        d = int((xd[i].view(torch.int32) != ref.view(torch.int32)).sum())
        print(f"q {q}, pair {i}: {d} elements differ from torch")
        assert d == 0
    # refusals: an odd clip count has no pairs
    net.set_clip_invariants(fea[:3], cond[:3])
    rc = _lib.lib.dawn_unet_ddim_step_guided(net._handle, fp(ed), fp(ed), fp(nd), n1, fp(scale), *coef, q, fp(scratch), st)
    assert rc == -1 and b"even clip count" in _lib.lib.dawn_last_error()


def test_guided_eps_is_rounded_as_three_ops():
    """With ca = 0, cb = -1, sqrt_an = 1, c = sigma = 0 and no clip the update returns the guided eps itself, which must equal
    torch's three rounded fp32 ops bit for bit (a fused multiply-add differs in the last bit of many elements)."""
    F, h, w = 8, 16, 16
    net = G.cuda_net()
    net.update_num_frames(F)
    _, _, cond, _, fea = G.clip("guided/exact", F, h, w, 500)
    net.set_clip_invariants(torch.cat([fea, fea]).cuda(), torch.cat([cond, cond]).cuda())     # B = 2: one pair
    n1 = 3 * F * h * w
    gen = torch.Generator().manual_seed(11)
    eps = torch.randn(2, 3, F, h, w, generator=gen)
    s = 2.7
    xd, ed = torch.randn(2, 3, F, h, w, generator=gen).cuda(), eps.cuda()
    scale = torch.tensor([s], device="cuda")
    scratch = torch.empty(n1 + 512, dtype=torch.int32, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    fp = lambda a: ctypes.c_void_p(a.data_ptr())             # noqa: E731
    _lib.check(_lib.lib.dawn_unet_ddim_step_guided(net._handle, fp(xd), fp(ed), None, n1, fp(scale), 0.0, -1.0, 1.0, 0.0, 0.0,
                                                   -1.0, fp(scratch), st), "dawn_unet_ddim_step_guided")
    torch.cuda.synchronize()
    ec, en = eps[0], eps[1]
    ref = en + (ec - en) * s
    assert torch.equal(xd[0].cpu(), ref) and torch.equal(xd[1].cpu(), ref)
    fused = ((ec - en).double() * s + en.double()).float()  # one rounding of the product and the sum
    assert not torch.equal(fused, ref)


def test_frame_sharded_handle_refuses_guidance():
    """Needs >= 2 GPUs (skipped otherwise): the checks run in tests/guided_shard_ranks.py, one rank per GPU."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29621", os.path.join(G.ROOT, "tests", "guided_shard_ranks.py")]
    r = subprocess.run(cmd, cwd=G.ROOT, capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stderr[-3000:]
    assert "[guided]" in r.stdout


def test_sample_one_video_with_guidance_on_the_graph():
    from dawn_pytorch_b200 import FlowDiffusion
    from oracle import lfg_oracle as L
    from oracle.make_golden_e2e import e2e_inputs, face_sd
    g = np.load(os.path.join(G.ROOT, "tests", "golden", "e2e_sample_one_video.npz"))
    steps, nf = int(g["steps"]), int(g["frames"])
    m = FlowDiffusion(sampling_timesteps=steps, pose_dim=6, win_width=40, ddim_sampling_eta=1.0)
    m.diffusion.load_state_dict({**{"denoise_fn." + k: v for k, v in G.synth_sd().items()},
                                 **{k: v for k, v in m.diffusion.state_dict().items() if not k.startswith("denoise_fn.")}}, strict=True)
    m.generator.load_state_dict(W.lfg_synth_state_dict(L.state_dict_schema()), strict=True)
    m.face_loc_emb.load_state_dict(face_sd(), strict=True)
    m = m.cuda()
    m.update_num_frames(nf)
    img, hubert, pose, eye, bbox, init_pose, init_eye = [t.cuda() for t in e2e_inputs()]

    def noise_fn(k, shape):
        return torch.from_numpy(W.pseudo_normal(f"guided_e2e/noise{k}", tuple(shape)))
    run = lambda graph: m.sample_one_video(sample_img=img, sample_audio_hubert=hubert, sample_pose=pose, sample_eye=eye,  # noqa: E731
                                           sample_bbox=bbox, init_pose=init_pose, init_eye=init_eye, cond_scale=2.0,
                                           noise_fn=noise_fn, use_graph=graph)
    eager = {k: v.cpu() for k, v in run(False).items() if torch.is_tensor(v)}
    graph = {k: v.cpu() for k, v in run(True).items() if torch.is_tensor(v)}
    torch.cuda.synchronize()
    r = G.over_tol(graph["sample_vid_grid"], eager["sample_vid_grid"])
    d_vid = (graph["sample_out_vid"] - eager["sample_out_vid"]).abs().max().item()
    print(f"sample_one_video cond_scale 2: grid {r:.4f} x tol, frames max|d| {d_vid:.2e}")
    assert r <= 0.05 and d_vid < 1e-3
