"""GPU: the LFG decoder at every configuration of tests/lfg_config_cases.py against the real reference's probes and the oracle,
and at the benchmark's clip geometry (200 frames of 256x256 from 64x64 flows)."""
import numpy as np
import pytest
import torch

from tests import lfg_config_cases as CC

pytestmark = pytest.mark.gpu


def module(tag):
    from dawn_pytorch_b200 import LfgGenerator
    g = LfgGenerator(**CC.ctor(tag))
    g.load_state_dict(CC.synth_sd(tag), strict=True)
    return g.cuda()


@pytest.mark.parametrize("tag", CC.TAGS)
def test_config_matches_reference(tag):
    """prediction / deformed / fea against the reference's probes; every read_tap against the oracle (unscaled tolerance)"""
    g = module(tag)
    src, flow, occ = CC.inputs(tag)
    out = g.forward_with_flow(src.cuda(), flow.cuda(), occ.cuda())
    fea = g.compute_fea(src.cuda())
    torch.cuda.synchronize()
    got = {"prediction": out["prediction"], "deformed": out["deformed"], "fea": fea}
    ora = CC.oracle(tag)
    fails = []
    for name in ("prediction", "fea"):
        r = CC.over_tol(CC.probes(tag, name, got[name]), CC.ref_probes(tag, name)[0])
        print(f"{tag} {name}: {r:.4f} x tol (reference probes)")
        if r > 1.0:
            fails.append(f"{name} {r:.3f} x tol")
    d = np.abs(CC.probes(tag, "deformed", got["deformed"]) - CC.ref_probes(tag, "deformed")[0]).max()
    print(f"{tag} deformed: max|d| {d:.2e}")
    if d >= 1e-5:
        fails.append(f"deformed max|d| {d:.2e}")
    for name in CC.report(tag)["taps"]:
        t = g.read_tap(name)
        assert t.shape == ora[name].shape, (name, t.shape, ora[name].shape)
        r = CC.over_tol(t, ora[name])
        print(f"{tag} tap {name}: {r:.4f} x tol (oracle)")
        if r > 1.0:
            fails.append(f"tap {name} {r:.3f} x tol")
    r = CC.over_tol(out["prediction"], ora["prediction"])
    print(f"{tag} prediction: {r:.4f} x tol (oracle, every element)")
    if r > 1.0:
        fails.append(f"prediction vs oracle {r:.3f} x tol")
    assert not fails, f"{tag}: " + "; ".join(fails)


CLIP_FRAMES, PICK = 200, (0, 1, 100, 199)


def test_clip_geometry():
    """bench.py's clip decode: decode_sample of 200 frames of 256x256 from 64x64 flows with hdtf256's generator_params (level-0
    buffers of 3.4 GB, byte offsets above 2^31).  Frames 0, 1, 100, 199 against the oracle run on those frames alone (frames are
    independent given the source) and against the same frames decoded as a 4-frame batch: the kernels choose their paths and
    round each row independently of the frame count, so the two decodes must agree bit for bit."""
    tag = "dawn256"
    g = module(tag)
    src, _, _ = CC.inputs(tag)
    from oracle import weights as W
    _, flow, occ = W.lfg_synth_inputs("lfgcfg/clip", CLIP_FRAMES, 256, 256, 64, 64)
    sample = torch.cat([flow.permute(3, 0, 1, 2), (occ * 2 - 1).permute(1, 0, 2, 3)], dim=0).contiguous()   # (3, F, h, w)
    pick = list(PICK)
    full = g.decode_sample(src.cuda(), sample.cuda())[pick].cpu()
    assert g.workspace_bytes() > 2 ** 32                                # the multi-GB level-0 buffers really exist
    small = g.decode_sample(src.cuda(), sample[:, pick].contiguous().cuda()).cpu()
    torch.cuda.synchronize()
    ora = CC.oracle(tag, src, flow[pick], ((sample[2, pick] + 1) * 0.5)[:, None])["prediction"]
    r = CC.over_tol(full, ora)
    d = (full - small).abs().max().item()
    print(f"clip: 200-frame decode vs oracle {r:.4f} x tol; vs 4-frame decode max|d| {d:.1e}")
    assert r <= 1.0
    assert torch.equal(full, small), f"the 200-frame and 4-frame decodes differ by up to {d:.2e}"
