"""GPU: PBnet's pose / blink generator on the device (dawn_pytorch_b200/pbnet.py, include/dawn_pbnet.h).

* every golden case through get_model -> load_state_dict -> generate(z=...) matches the reference's output;
* 1500 frames (a minute of audio) for reemb5 and reemb6 match the float64 oracle run on the same GPU;
* the banded attention kernel on its own matches float64 for 1 to 1500 frames, 4 and 8 heads, bands 100 and 200, self and cross;
* padded frames are exactly zero; the default z is torch.randn as the reference draws it; two calls are bitwise equal;
* one generate is 7 num_layers + 1 launches; load_state_dict after a call reaches the library.
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import pbnet_oracle as P
from oracle import weights as W

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RTOL, ATOL = 1e-3, 1e-4


def over_tol(a, ref):
    a, ref = a.detach().double().cpu(), ref.detach().double().cpu()
    return ((a - ref).abs() / (ATOL + RTOL * ref.abs())).max().item()


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLD, "pbnet.npz"))


@pytest.fixture(scope="module")
def schema():
    with open(os.path.join(GOLD, "pbnet_schema.json")) as f:
        return {k: [(n, tuple(s)) for n, s in v] for k, v in json.load(f).items()}


def cuda_model(cfg, sd):
    from dawn_pytorch_b200.pbnet import get_model
    model = get_model(cfg.parameters("cuda:0"))
    model.load_state_dict(sd, strict=True)
    return model.eval()


def run(model, case, cfg, lengths, z=True):
    pose, audio, zz, lens = P.synth_inputs(case, cfg, lengths)
    return model.generate(pose, audio, lens, fact=1, z=zz.cuda() if z else None)


@pytest.mark.parametrize("case", list(P.CASES))
def test_golden_case_matches_reference(case, golden, schema):
    cfg, lengths = P.CASES[case]
    model = cuda_model(cfg, P.synth_state_dict(schema[case]))
    batch = run(model, case, cfg, lengths)
    ref = torch.from_numpy(golden[f"{case}/output"])
    out = batch["output"]
    assert out.shape == ref.shape and out.device.type == "cuda"
    r = over_tol(out, ref)
    print(f"{case}: max |d| / (atol + rtol |ref|) = {r:.3g}")
    assert r <= 1.0
    for k in ("x", "z", "y", "mask", "lengths"):
        assert k in batch
    if cfg.archiname == "transformerreemb5":
        assert torch.equal(batch["out_pose"], out[:, :, :6]) and torch.equal(batch["out_eye"], out[:, :, 6:])
    else:
        assert "out_pose" not in batch


@pytest.mark.parametrize("arch", ["transformerreemb5", "transformerreemb6"])
def test_a_minute_of_audio_matches_oracle(arch, schema):
    cfg = P.PbCfg(archiname=arch)
    sd = P.synth_state_dict(schema["reemb5_pose_250" if arch.endswith("5") else "reemb6_pose_150"])
    model = cuda_model(cfg, sd)
    case = f"{arch}_1500"
    pose, audio, z, lens = P.synth_inputs(case, cfg, [1500])
    out = model.generate(pose, audio, lens, z=z.cuda())["output"]
    ref = P.decoder_forward({k: v.cuda() for k, v in sd.items()}, cfg, pose.cuda(), audio.cuda(), z.cuda(), lens.cuda())
    r = over_tol(out, ref)
    print(f"{case}: max |d| / (atol + rtol |ref|) = {r:.3g}")
    assert r <= 1.0


def attention_case(bs, F, D, H, band, npairs, x_q, x_kv, wq, wk, wv, freqs, bias, out):
    from dawn_pytorch_b200 import _lib
    c = _lib.DawnPbnetAttentionCase(bs=bs, F=F, D=D, H=H, band=band, npairs=npairs, qscale=32 ** -0.5)
    for name, t in (("x_q", x_q), ("x_kv", x_kv), ("wq", wq), ("wk", wk), ("wv", wv), ("freqs", freqs), ("bias", bias), ("out", out)):
        setattr(c, name, t.data_ptr())
    _lib.check(_lib.lib.dawn_pbnet_test_attention(ctypes.byref(c), _lib.stream()), "dawn_pbnet_test_attention")


@pytest.mark.parametrize("F", [1, 63, 64, 65, 401, 1500])
@pytest.mark.parametrize("H", [4, 8])
@pytest.mark.parametrize("band", [100, 200])
@pytest.mark.parametrize("site", ["self", "cross"])
def test_attention_kernel_matches_float64(F, H, band, site):
    D, bs, hid = 64, 2, 32 * H
    tag = f"pbattn/{F}/{H}/{band}/{site}"
    t = lambda k, shape, bound: torch.from_numpy(W.symmetric(f"{tag}/{k}", shape, bound)).cuda()   # noqa: E731
    x_q = t("xq", (bs * F, D), 1.7)
    x_kv = x_q if site == "self" else t("xkv", (bs * F, D), 1.7)
    wq, wk, wv = (t(k, (D, hid), 0.25) for k in ("wq", "wk", "wv"))
    npairs = min(32, H) // 2
    freqs = 1. / (10000 ** (torch.arange(0, 2 * npairs, 2).float() / (2 * npairs)))
    table = t("bias", (H, 2 * band + 1), 1.7)
    out = torch.empty(bs * F, hid, device="cuda")
    attention_case(bs, F, D, H, band, npairs, x_q, x_kv, wq, wk, wv, freqs.cuda(), table, out)
    torch.cuda.synchronize()
    d = torch.float64
    pos = torch.arange(F, device="cuda")
    rel = pos[None, :] - pos[:, None]
    full = table.to(d)[:, (rel.clamp(-band, band) + band)].masked_fill((rel.abs() > band)[None], float("-inf"))
    xq, xkv = x_q.to(d).view(bs, F, D), x_kv.to(d).view(bs, F, D)
    ref = P.attention(xq @ wq.to(d), xkv @ wk.to(d), xkv @ wv.to(d), full, freqs.cuda(), H)
    r = over_tol(out.view(bs, F, hid), ref)
    assert r <= 0.25, r


def test_padded_rows_zero_default_z_determinism_and_launches(schema):
    cfg, lengths = P.CASES["reemb5_blink_bs2"]
    model = cuda_model(cfg, P.synth_state_dict(schema["reemb5_blink_bs2"]))
    pose, audio, _, lens = P.synth_inputs("reemb5_blink_bs2", cfg, lengths)
    torch.manual_seed(7)
    a = model.generate(pose, audio, lens)
    assert model.last_launch_count() == 7 * cfg.num_layers + 1 == 15
    torch.manual_seed(7)
    z = torch.randn(max(lengths), len(lengths), cfg.latent_dim, device="cuda")
    b = model.generate(pose, audio, lens, z=z)
    assert torch.equal(a["z"], z) and torch.equal(a["output"], b["output"])
    c = model.generate(pose, audio, lens, z=z)
    assert torch.equal(b["output"], c["output"])
    assert torch.count_nonzero(a["output"][1, 77:]) == 0 and torch.count_nonzero(a["output"][1, :77]) > 0
    assert torch.equal(a["mask"], CVAE_mask(lens))


def CVAE_mask(lens):
    from dawn_pytorch_b200.pbnet import CVAE
    return CVAE.lengths_to_mask(lens.cuda())


def test_load_state_dict_after_a_call_reaches_the_library(schema):
    cfg, lengths = P.CASES["reemb5_pose_250"]
    first = P.synth_state_dict(schema["reemb5_pose_250"])
    second = {k: v * 1.0625 for k, v in first.items()}
    model = cuda_model(cfg, first)
    a = run(model, "reemb5_pose_250", cfg, lengths)["output"]
    model.load_state_dict(second)
    b = run(model, "reemb5_pose_250", cfg, lengths)["output"]
    fresh = run(cuda_model(cfg, second), "reemb5_pose_250", cfg, lengths)["output"]
    assert not torch.equal(a, b) and torch.equal(b, fresh)

