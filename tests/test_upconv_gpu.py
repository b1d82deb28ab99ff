"""-m gpu: the UNet's upconv variant (nearest x2 + 3x3 conv, U:165-172) in every padding mode and UNets without spatial linear
attention, against the REAL reference's goldens (tests/golden/upconv.npz), the CPU oracle at every sub-module boundary, a float64
reference of the upsample conv alone, each clip alone, the eager samplers and the kernels each mode launches.

Upsample conv bound (the split arithmetic of tests/test_contraction_gpu.py, u = 2^-24): the class taps are sums of 3x3 taps
folded in fp64 and rounded once (<= u S), the 3-term fp16 split leaves <= 3 * 2^-22 |a||b| per product, truncating adds
inside a drain interval of Kc products <= Kc 2^-23 S and the K / Kc round-to-nearest drains plus bias <= (K/Kc + 4) u S, with
S = sum |a||b| over the nine taps on the upsampled grid.  The bound takes the largest of the three paths the up conv may run on
(mma.sync Kc = 8, wgmma GEMM Kc = 256, halo conv Kc = 576) at K = 9 C; norm-wise ||d|| / ||R|| <= 2^-20 + 576 u."""
import collections
import json
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as TF

from oracle import weights as W
from tests import upconv_cases as UC

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SPLIT = 3 * 2.0 ** -22
_NETS = {}


def net_of(tag, **over):
    """one module per configuration for the session, synthetic weights loaded"""
    from dawn_pytorch_b200 import DynamicNfUnet3D
    key = (tag, tuple(sorted(over.items())))
    if key not in _NETS:
        net = DynamicNfUnet3D(**{**UC.ctor(tag), **over}).eval()
        net.load_state_dict(W.synth_state_dict([(k, list(v.shape)) for k, v in net.state_dict().items()]), strict=True)
        _NETS[key] = net.cuda()
    return _NETS[key]


def run(net, x, t, cond):
    net.update_num_frames(x.shape[2])
    with torch.no_grad():
        out = net.forward_with_cond_scale(x.cuda(), t.cuda(), cond=cond.cuda(), cond_scale=1.0)
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("tag", UC.TAGS)
def test_case_matches_reference_and_oracle_taps(tag):
    net = net_of(tag)
    x, t, cond, x_t, fea = UC.clip(tag)
    eps = run(net, x, t, cond)
    ref = torch.from_numpy(UC.golden()[f"eps/{tag}"])
    assert eps.shape == ref.shape
    r_eps = UC.over_tol(eps, ref)
    taps_o = {}
    UC.oracle(tag, x, t, cond, taps=taps_o)
    bufs = net.request_taps(list(taps_o), x.shape[2], x.shape[3], x.shape[4], torch.device("cuda"))
    try:
        run(net, x, t, cond)
    finally:
        got = {k: v.cpu() for k, v in bufs.items()}
        net.clear_taps()
    ratios = {name: UC.over_tol(got[name], want) for name, want in taps_o.items()}
    print(f"\n{tag}: eps {r_eps:.3f} x tol; worst tap {max(ratios.values()):.3f} x tol ({max(ratios, key=ratios.get)})")
    bad = {k: round(v, 3) for k, v in ratios.items() if v > 1.0}
    assert not bad, f"taps over tolerance (in forward order): {bad}"
    assert r_eps <= 1.0
    net.set_clip_invariants(fea[0].cuda(), cond[0].cuda())
    out = net.forward_x3(x_t[0].cuda(), t.cuda())
    torch.cuda.synchronize()
    r_x3 = UC.over_tol(out.cpu()[None], eps)
    print(f"    forward_x3 vs forward: {r_x3:.4f} x tol")
    assert r_x3 <= 0.05


@pytest.mark.parametrize("mode", UC.MODES)
def test_upsample_conv_alone_against_float64(mode):
    """Each up conv of a 32 x 64 latent (inputs 16 x 32 at 64 channels: the up2 halo conv in zeros mode; 8 x 16 at 128 and
    4 x 8 at 256 channels: the per-class GEMMs) from its own tapped input, against conv2d(pad(nearest(x))) in float64."""
    net = net_of("up_zeros", padding_mode=mode)
    F, h, w = 4, 32, 64
    x_t, fea, cond = W.synth_inputs(f"upconv_alone/{mode}", F, h, w)
    x = torch.cat([x_t, fea.unsqueeze(2).expand(-1, -1, F, -1, -1)], dim=1).contiguous()
    t = torch.full((1,), 400, dtype=torch.long)
    names = [f"ups.{K}.{j}" for K in range(3) for j in (3, 4)]
    net.update_num_frames(F)
    bufs = net.request_taps(names, F, h, w, torch.device("cuda"))
    try:
        run(net, x, t, cond)
    finally:
        got = {k: v[0].transpose(0, 1).double() for k, v in bufs.items()}     # (F, C, H, W)
        net.clear_taps()
    sd = net.state_dict()
    for K in range(3):
        xin, out = got[f"ups.{K}.3"], got[f"ups.{K}.4"]
        wt = sd[f"ups.{K}.4.1.weight"][:, :, 0].double().cuda()
        b = sd[f"ups.{K}.4.1.bias"].double().cuda()
        C = wt.shape[0]
        u = TF.interpolate(xin, scale_factor=2, mode="nearest")
        up = TF.pad(u, (1, 1, 1, 1), mode="constant" if mode == "zeros" else mode)
        ref = TF.conv2d(up, wt, b)
        S = TF.conv2d(up.abs(), wt.abs()) + b.abs().reshape(1, -1, 1, 1)
        R = TF.conv2d(up * up, wt * wt).sqrt()
        Kd = 9 * C
        c1 = SPLIT + U + max(kc * 2.0 ** -23 + (Kd / kc + 4) * U for kc in (8, 256, 576))
        tau = 2.0 ** -20 + 576 * U
        d = (out - ref).abs()
        el = (d / (c1 * S + 8 * U * ref.abs() + 2.0 ** -25 * S)).max().item()
        nr = (d.norm() / R.norm()).item()
        print(f"  {mode} ups.{K}.4 ({C} ch, {xin.shape[2]}x{xin.shape[3]}): elementwise max |d|/bound = {el:.3f}; "
              f"||d||/||R|| = {nr:.2e} ({nr / tau:.3f} of tau)")
        assert torch.isfinite(out).all()
        assert el <= 1.0 and nr <= tau


def test_two_clips_equal_each_clip_alone():
    tag = "upconv_nosla"
    net = net_of(tag)
    F = UC.report(tag)["F"]
    xa, ta, ca, _, _ = UC.clip(tag)
    xb, tb, cb, _, _ = UC.clip(tag, key=tag + "_b", amp=3.0, t=int(ta) // 2 + 7)
    xb[:, 3:] += 0.25 * torch.linspace(-1, 1, F).reshape(1, 1, F, 1, 1)
    ya, yb = run(net, xa, ta, ca), run(net, xb, tb, cb)
    y2 = run(net, torch.cat([xa, xb]), torch.cat([ta, tb]), torch.cat([ca, cb]))
    assert net.clip_count() == 2
    ra, rb = UC.over_tol(y2[0:1], ya), UC.over_tol(y2[1:2], yb)
    rob = UC.over_tol(yb, UC.oracle(tag, xb, tb, cb))
    print(f"\n{tag}: B=2 vs alone {ra:.4f} / {rb:.4f} x tol; second clip vs oracle {rob:.3f} x tol")
    assert ra <= 0.05 and rb <= 0.05 and rob <= 1.0
    assert (y2[0] - y2[1]).abs().max() > 1e-2


def test_ddim_graph_equals_eager():
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion
    tag = "upconv_nosla"
    net = net_of(tag)
    F, h, w = 8, 16, 16
    D = DynamicNfGaussianDiffusion(denoise_fn=net, num_frames=40, image_size=32, sampling_timesteps=3, timesteps=1000,
                                   loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0).cuda()
    D.update_num_frames(F)
    _, fea, cond = W.synth_inputs("upconv_ddim", F, h, w)

    def noise_fn(k, shape):
        return torch.from_numpy(W.pseudo_normal(f"upconv_ddim/noise{k}", tuple(shape)))
    eager = D.ddim_sample(fea.cuda(), (1, 3, F, h, w), cond=cond.cuda(), noise_fn=noise_fn).cpu()
    graph = D.ddim_sample(fea.cuda(), (1, 3, F, h, w), cond=cond.cuda(), noise_fn=noise_fn, use_graph=True).cpu()
    d = (graph - eager).abs().max().item()
    print(f"\nddim graph vs eager ({tag}): max|d| {d:.2e}")
    assert torch.isfinite(graph).all() and d < 1e-4


def test_flow_diffusion_upconv_samples_and_matches_eager():
    from dawn_pytorch_b200 import FlowDiffusion
    from oracle import lfg_oracle as L
    from oracle.make_golden_e2e import e2e_inputs, face_sd
    m = FlowDiffusion(sampling_timesteps=3, pose_dim=6, win_width=40, ddim_sampling_eta=1.0, use_deconv=False, padding_mode="reflect")
    unet = m.unet
    assert unet._cfg.upconv == 1 and unet._cfg.pad_mode == 1
    unet.load_state_dict(W.synth_state_dict([(k, list(v.shape)) for k, v in unet.state_dict().items()]), strict=True)
    m.generator.load_state_dict(W.lfg_synth_state_dict(L.state_dict_schema()), strict=True)
    m.face_loc_emb.load_state_dict(face_sd(), strict=True)
    m = m.cuda()
    img, hubert, pose, eye, bbox, init_pose, init_eye = [t.cuda() for t in e2e_inputs()]
    m.update_num_frames(hubert.shape[1])

    def noise_fn(k, shape):
        return torch.from_numpy(W.pseudo_normal(f"upconv_e2e/noise{k}", tuple(shape)))
    res = lambda graph: m.sample_one_video(sample_img=img, sample_audio_hubert=hubert, sample_pose=pose, sample_eye=eye,  # noqa: E731
                                           sample_bbox=bbox, init_pose=init_pose, init_eye=init_eye, cond_scale=1.0,
                                           noise_fn=noise_fn, use_graph=graph)
    eager = {k: v.cpu() for k, v in res(False).items() if torch.is_tensor(v)}
    graph = {k: v.cpu() for k, v in res(True).items() if torch.is_tensor(v)}
    torch.cuda.synchronize()
    assert all(torch.isfinite(v).all() for v in eager.values())
    d_grid = (graph["sample_vid_grid"] - eager["sample_vid_grid"]).abs().max().item()
    d_vid = (graph["sample_out_vid"] - eager["sample_out_vid"]).abs().max().item()
    print(f"\nFlowDiffusion upconv reflect: graph vs eager grid max|d| {d_grid:.2e}, frames {d_vid:.2e}")
    assert d_grid < 1e-4 and d_vid < 1e-3


def kernel_counts(mode):
    """{kernel name: launches} of one forward at 16 x 16 (deconv for mode None); run in a fresh process by the test below"""
    over = {"use_deconv": True} if mode is None else {"padding_mode": mode}
    net = net_of("up_zeros", **over)
    x, t, cond, _, _ = UC.clip("up_zeros")
    run(net, x, t, cond)                                                         # warm: workspace and attributes
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run(net, x, t, cond)
    c = collections.Counter(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                            and not e.name.startswith("Memcpy") and not e.name.startswith("Memset"))
    return dict(c), net.last_launch_count()


def test_border_pass_runs_only_for_clamp_and_wrap_modes():
    """The profile is taken in a new Python process: torch.profiler records no device events once a process is a few minutes
    old.  Zeros mode launches exactly what the ConvTranspose model launches; reflect, replicate and circular add one border pass
    per up conv (three at four levels)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import json; from tests import test_upconv_gpu as T; "
            "print(json.dumps({str(m): T.kernel_counts(m) for m in (None, 'zeros', 'reflect', 'replicate', 'circular')}))")
    r = subprocess.run([sys.executable, "-s", "-B", "-c", code], cwd=root, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    pat = re.compile(r"(?<!\w)pad_border_kernel(?!\w)")
    border = {m: sum(n for k, n in c.items() if pat.search(k)) for m, (c, _) in res.items()}
    print(f"\nborder passes per forward: {border}; launches: { {m: n for m, (_, n) in res.items()} }")
    assert border == {"None": 0, "zeros": 0, "reflect": 3, "replicate": 3, "circular": 3}
    assert res["zeros"][0] == res["None"][0] and res["zeros"][1] == res["None"][1]
    for m in ("reflect", "replicate", "circular"):
        assert res[m][0] == res["reflect"][0]
