"""LFG flow decoder (SURVEY 8f N1) on the GPU, through the reference-facing module API -> C-ABI (include/dawn_lfg.h):
parity against golden vectors produced by the REAL reference `Generator` and against the CPU oracle on the same seeded inputs."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import lfg_oracle as L
from oracle import weights as W

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CASES = {'lfg_small': (3, 64, 64, 16, 16), 'lfg_rect': (2, 64, 96, 16, 24)}
RTOL, ATOL = 1e-3, 1e-4
PROBE_N = 4096
CTOR = dict(num_channels=3, num_regions=10, block_expansion=64, max_features=512, num_down_blocks=2, num_bottleneck_blocks=6,
            pixelwise_flow_predictor_params=None, skips=True, revert_axis_swap=True)          # config/hdtf128.yaml:82-93


def over_tol(a, ref):
    a, ref = a.detach().float().cpu(), ref.detach().float().cpu()
    return ((a - ref).abs() / (ATOL + RTOL * ref.abs())).max().item()


def probe_idx(name, numel):
    u = W.uniform01('probe/' + name, PROBE_N)
    return np.minimum((u.astype(np.float64) * numel).astype(np.int64), numel - 1)


_NET = None


def synth_sd():
    with open(os.path.join(GOLD, "lfg_state_dict_schema.json")) as f:
        sch = json.load(f)
    return W.lfg_synth_state_dict([(n, tuple(s)) for n, s in sch["entries"]])


def net():
    global _NET
    if _NET is None:
        from dawn_pytorch_b200 import LfgGenerator
        g = LfgGenerator(**CTOR)
        g.load_state_dict(synth_sd(), strict=True)
        _NET = g.cuda()
    return _NET


@pytest.mark.parametrize("case", list(CASES))
def test_decode_matches_reference_golden(case):
    g = net()
    nf, H, Wd, h, w = CASES[case]
    src, flow, occ = W.lfg_synth_inputs(case, nf, H, Wd, h, w)
    gold = np.load(os.path.join(GOLD, f"{case}.npz"))
    out = g.forward_with_flow(src.cuda(), flow.cuda(), occ.cuda())
    torch.cuda.synchronize()
    taps_o = {}
    with torch.no_grad():
        L.forward_with_flow(synth_sd(), L.LfgCfg(), src, flow, occ, taps=taps_o)
    for name in ("bottleneck", "up0", "up1"):
        print(f"{case} tap {name}: {over_tol(g.read_tap(name), taps_o[name]):.3f} x tol")
    d_def = (out["deformed"].cpu() - torch.from_numpy(gold["deformed"])).abs().max().item()
    r = over_tol(out["prediction"], torch.from_numpy(gold["prediction"]))
    print(f"{case}: prediction {r:.3f} x tol, deformed max|d| {d_def:.2e}, {g.last_launch_count()} launches")
    assert d_def < 1e-5
    for name in ("bottleneck", "up0", "up1"):
        assert over_tol(g.read_tap(name), taps_o[name]) <= 1.0, name      # unscaled north-star tolerance on the un-normalised activations
    assert r <= 1.0
    assert g.last_launch_count() > 30


def test_compute_fea_matches_reference_golden():
    g = net()
    for case, (nf, H, Wd, h, w) in CASES.items():
        src, _, _ = W.lfg_synth_inputs(case, nf, H, Wd, h, w)
        gold = np.load(os.path.join(GOLD, f"{case}.npz"))
        fea = g.compute_fea(src.cuda()).cpu()
        assert fea.shape == (1, 256, H // 4, Wd // 4)
        got = fea.flatten()[probe_idx(case + '/fea', fea.numel())].numpy()
        ref = gold["fea_probe"]
        assert (np.abs(got - ref) / (ATOL + RTOL * np.abs(ref))).max() <= 1.0
        assert abs(float(fea.abs().mean()) - float(gold["fea_absmean"])) < 1e-4


def test_128_probes_and_sampler_layout():
    """128x128 source with a 32x32 flow (config/hdtf128.yaml), probes from the reference; the (3, F, h, w) sampler layout with
    occlusion = (conf + 1) / 2 (FD:366-369) decodes to the same frames as the reference argument layout."""
    g = net()
    nf, H, Wd, h, w = 2, 128, 128, 32, 32
    src, flow, occ = W.lfg_synth_inputs('lfg_128', nf, H, Wd, h, w)
    gold = np.load(os.path.join(GOLD, "lfg_128.npz"))
    out = g.forward_with_flow(src.cuda(), flow.cuda(), occ.cuda())
    ip = probe_idx('lfg_128/pred', out["prediction"].numel())
    got = out["prediction"].cpu().flatten()[ip].numpy()
    ref = gold["prediction_probe"]
    r = (np.abs(got - ref) / (ATOL + RTOL * np.abs(ref))).max()
    print(f"lfg_128: {r:.3f} x tol")
    assert r <= 1.0
    assert np.abs(out["deformed"].cpu().flatten()[ip].numpy() - gold["deformed_probe"]).max() < 1e-5
    sample = torch.cat([flow.permute(3, 0, 1, 2), (occ * 2 - 1).permute(1, 0, 2, 3)], dim=0).contiguous()      # (3, F, h, w)
    pred2 = g.decode_sample(src.cuda(), sample.cuda())
    assert over_tol(pred2, out["prediction"]) <= 0.05


def test_cpu_tensors_fail_loudly():
    from dawn_pytorch_b200 import _lib
    with pytest.raises(_lib.DawnError):
        net().forward_with_flow(torch.rand(1, 3, 64, 64), torch.zeros(1, 16, 16, 2), torch.zeros(1, 1, 16, 16))
