"""-m gpu: the CUDA path at UNet configurations other than DAWN's own (tests/config_cases.py), against the REAL reference's goldens
(tests/golden/configs.npz) and, at every sub-module boundary, against the CPU oracle (which tests/test_config_oracle_golden.py pins
to the reference at the same configurations).

These configurations reach paths DAWN's own never runs: FiLM tables of 1024-channel blocks, the general init-conv kernel
(init_conv_x3_kernel: 3x3 / 5x5 kernels, 128 output channels), level-0 temporal attention on the general path (128 channels),
1x1 images at the deepest level, equal-width levels, the SIMT banded attention kernel for windows over 40 frames, and other
input / conditioning / output widths."""
import json
import os
import re
import subprocess
import sys

import pytest
import torch

from tests import config_cases as CC

pytestmark = pytest.mark.gpu

_NETS = {}


def net_of(tag):
    """one module per configuration for the session, synthetic weights loaded"""
    from dawn_pytorch_b200 import DynamicNfUnet3D
    if tag not in _NETS:
        net = DynamicNfUnet3D(**CC.ctor(tag)).eval()
        net.load_state_dict(CC.synth_sd(tag), strict=True)
        _NETS[tag] = net.cuda()
    return _NETS[tag]


def run(net, x, t, cond):
    net.update_num_frames(x.shape[2])
    with torch.no_grad():
        out = net.forward_with_cond_scale(x.cuda(), t.cuda(), cond=cond.cuda(), cond_scale=1.0)
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("tag", CC.TAGS)
def test_config_matches_reference_and_oracle_taps(tag):
    net = net_of(tag)
    x, t, cond, x_t, fea = CC.clip(tag)
    eps = run(net, x, t, cond)
    ref = torch.from_numpy(CC.golden()[f"eps/{tag}"])
    assert eps.shape == ref.shape
    r_eps = CC.over_tol(eps, ref)
    # every sub-module boundary against the oracle (B = 1)
    taps_o = {}
    CC.oracle(tag, x, t, cond, taps=taps_o)
    bufs = net.request_taps(list(taps_o), x.shape[2], x.shape[3], x.shape[4], torch.device("cuda"))
    try:
        run(net, x, t, cond)
    finally:
        got = {k: v.cpu() for k, v in bufs.items()}
        net.clear_taps()
    ratios = {}
    for name, want in taps_o.items():
        assert got[name].shape == want.shape, name
        ratios[name] = CC.over_tol(got[name], want)
    print(f"\n{tag}: eps {r_eps:.3f} x tol; worst tap {max(ratios.values()):.3f} x tol")
    for name, r in ratios.items():
        print(f"    {name:24s} {r:.3f}")
    bad = {k: round(v, 3) for k, v in ratios.items() if v > 1.0}
    assert not bad, f"taps over tolerance (in forward order): {bad}"
    assert r_eps <= 1.0
    # the hoisted entry (per-clip invariants once, then the 3 noisy channels) computes the same function
    net.set_clip_invariants(fea[0].cuda(), cond[0].cuda())
    out = net.forward_x3(x_t[0].cuda(), t.cuda())
    torch.cuda.synchronize()
    r_x3 = CC.over_tol(out.cpu()[None], eps)
    print(f"    forward_x3 vs forward: {r_x3:.4f} x tol")
    assert r_x3 <= 0.05


@pytest.mark.parametrize("tag", ["dim128", "l6"])
def test_two_clips_equal_each_clip_alone(tag):
    """B = 2 with its own amplitude and timestep per clip.  Clip 1's features vary over the frames, so the general entry runs the
    full init conv for both clips and then the general hoisted init-conv kernel rewrites clip 0 only (per-clip skip flag); the
    batched hoisted entry runs the same kernel on both clips at its own clip stride."""
    net = net_of(tag)
    F = CC.report(tag)["F"]
    xa, ta, ca, xta, fa = CC.clip(tag)
    xb, tb, cb, xtb, fb = CC.clip(tag, key=tag + "_b", amp=3.0, t=int(ta) // 2 + 7)
    xb[:, 3:] += 0.25 * torch.linspace(-1, 1, F).reshape(1, 1, F, 1, 1)          # frame-varying features
    ya, yb = run(net, xa, ta, ca), run(net, xb, tb, cb)
    y2 = run(net, torch.cat([xa, xb]), torch.cat([ta, tb]), torch.cat([ca, cb]))
    assert net.clip_count() == 2
    ra, rb = CC.over_tol(y2[0:1], ya), CC.over_tol(y2[1:2], yb)
    rob = CC.over_tol(yb, CC.oracle(tag, xb, tb, cb))
    print(f"\n{tag}: B=2 vs alone {ra:.4f} / {rb:.4f} x tol; varying clip vs oracle {rob:.3f} x tol")
    assert ra <= 0.05 and rb <= 0.05
    assert rob <= 1.0
    assert (y2[0] - y2[1]).abs().max() > 1e-2
    # batched hoisted entry: both clips frame-invariant
    net.set_clip_invariants(torch.cat([fa, fa]).cuda(), torch.cat([ca, cb]).cuda())
    o2 = net.forward_x3(torch.cat([xta, xtb]).cuda(), torch.cat([ta, tb]).cuda())
    torch.cuda.synchronize()
    xb0 = torch.cat([xtb, fa.unsqueeze(2).expand(-1, -1, F, -1, -1)], dim=1).contiguous()
    yb0 = run(net, xb0, tb, cb)
    r0, r1 = CC.over_tol(o2.cpu()[0:1], ya), CC.over_tol(o2.cpu()[1:2], yb0)
    print(f"    batched forward_x3 vs alone {r0:.4f} / {r1:.4f} x tol")
    assert r0 <= 0.05 and r1 <= 0.05


def kernel_names(tag):
    net = net_of(tag)
    x, t, cond, _, _ = CC.clip(tag)
    run(net, x, t, cond)                                                         # warm: workspace and attributes
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run(net, x, t, cond)
    return {e.name for e in prof.events()}


@pytest.mark.parametrize("tag,kernel", [("dim128", "init_conv_x3_kernel"), ("w120", "attention_kernel")])
def test_config_runs_the_path_it_is_for(tag, kernel):
    """dim128 runs the general hoisted init-conv kernel (not the 7x7 / 64-channel tiled one); w120's 120-frame window runs the
    SIMT banded attention kernel (the tensor-core one takes windows up to 40, the fused temporal one up to 64).  The profile is
    taken in a new Python process: torch.profiler records no device events once a process is a few minutes old."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = f"import json; from tests import test_configs_gpu as T; print(json.dumps(sorted(T.kernel_names({tag!r}))))"
    r = subprocess.run([sys.executable, "-s", "-B", "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    pat = re.compile(r"(?<!\w)" + kernel + r"(?!\w)")
    assert any(pat.search(n) for n in names), sorted(names)
