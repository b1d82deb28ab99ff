"""GPU: PBnet's pose / blink generator on the device (dawn_pytorch_b200/pbnet.py, include/dawn_pbnet.h).

* every golden case through get_model -> load_state_dict -> generate(z=...) matches the reference's output, at DAWN's shape and
  at the other configurations of oracle/pbnet_oracle.CONFIG_CASES;
* 1500 frames (a minute of audio) for reemb5 and reemb6 match the float64 oracle run on the same GPU;
* 65 537 clips in one generate (more than a grid's 65 535 z-blocks) match the float64 oracle run on the same GPU;
* the banded attention kernel on its own matches float64 for 1 to 1500 frames, 4 and 8 heads, bands 100 and 200, self and cross;
  and against a banded float64 reference with a derived bound for 2 and 32 heads and 15 000 frames (ten minutes of audio);
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

U = 2.0 ** -24

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


@pytest.fixture(scope="module")
def config_golden():
    return np.load(os.path.join(GOLD, "pbnet_configs.npz"))


@pytest.fixture(scope="module")
def config_schema():
    with open(os.path.join(GOLD, "pbnet_configs_schema.json")) as f:
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


@pytest.mark.parametrize("case", list(P.CONFIG_CASES))
def test_other_configuration_matches_reference(case, config_golden, config_schema):
    cfg, lengths = P.CONFIG_CASES[case]
    model = cuda_model(cfg, P.synth_state_dict(config_schema[case]))
    out = run(model, case, cfg, lengths)["output"]
    ref = torch.from_numpy(config_golden[f"{case}/output"])
    assert out.shape == ref.shape
    r = over_tol(out, ref)
    print(f"{case}: max |d| / (atol + rtol |ref|) = {r:.3g}")
    assert r <= 1.0
    assert model.last_launch_count() >= 7 * cfg.num_layers + 1


def test_more_clips_than_a_grid_z_dimension_matches_oracle():
    cfg = P.PbCfg(audio_dim=64, pos_dim=0, eye_dim=2)
    lengths = [2] * 65537
    lengths[1::3] = [1] * len(lengths[1::3])
    from dawn_pytorch_b200.pbnet import get_model
    sd = P.synth_state_dict([(k, tuple(v.shape)) for k, v in get_model(cfg.parameters()).state_dict().items()])
    model = cuda_model(cfg, sd)
    pose, audio, z, lens = P.synth_inputs("pbnet_65537", cfg, lengths)
    out = model.generate(pose, audio, lens, z=z.cuda())["output"]
    ref = P.decoder_forward({k: v.cuda() for k, v in sd.items()}, cfg, pose.cuda(), audio.cuda(), z.cuda(), lens.cuda())
    r = over_tol(out, ref)
    print(f"65537 clips of 1-2 frames: max |d| / (atol + rtol |ref|) = {r:.3g}")
    assert r <= 1.0
    assert torch.count_nonzero(out[1::3, 1]) == 0 and torch.count_nonzero(out[0, 1]) > 0
    assert model.last_launch_count() == 7 * cfg.num_layers + 1 + (2 * cfg.num_layers - 1)   # each attention site: 2 launches


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


def banded_reference(q, k, v, table, band, freqs, heads, exact_angles=False, chunk=512):
    """float64 banded attention of (bs, F, 32 H) q (unscaled), k, v with the rotary of P.rotate (fp32 angles, or exact fp64 ones)
    and bias table (H, 2 band + 1), query chunk by query chunk over the keys within +-band, and the derived error bound of the
    kernel pipeline (see test_attention_kernel_banded_float64)"""
    bs, F, hid = q.shape
    d = torch.float64
    if exact_angles:
        ang = torch.arange(F, device=q.device, dtype=d)[:, None] * freqs.to(d)[None, :]
    else:
        ang = P.rotary_angles(F, freqs)
    cos, sin = ang.cos(), ang.sin()
    r = 2 * freqs.shape[0]
    split = lambda t: t.reshape(bs, F, heads, 32).transpose(1, 2)                  # noqa: E731

    def rot(t):
        a, b = t[..., 0:r:2], t[..., 1:r:2]
        out = t.clone()
        out[..., 0:r:2], out[..., 1:r:2] = a * cos - b * sin, b * cos + a * sin
        return out

    qs, ks, vs = rot(split(q) * 32 ** -0.5), rot(split(k)), split(v)
    out = torch.empty(bs, heads, F, 32, dtype=d, device=q.device)
    for i0 in range(0, F, chunk):
        i1 = min(F, i0 + chunk)
        j0, j1 = max(0, i0 - band), min(F, i1 + band)
        rel = torch.arange(j0, j1, device=q.device)[None, :] - torch.arange(i0, i1, device=q.device)[:, None]
        bias = table.to(d)[:, rel.clamp(-band, band) + band].masked_fill((rel.abs() > band)[None], float("-inf"))
        p = torch.softmax(qs[:, :, i0:i1] @ ks[:, :, j0:j1].transpose(-1, -2) + bias[None], -1)
        out[:, :, i0:i1] = p @ vs[:, :, j0:j1]
    return out.transpose(1, 2).reshape(bs, F, hid)


@pytest.mark.parametrize("F,H,band,site", [(65, 2, 200, "self"), (401, 32, 100, "cross"), (1500, 2, 100, "cross"),
                                           (1500, 32, 200, "self"), (15000, 4, 200, "cross"), (15000, 32, 100, "self")])
def test_attention_kernel_banded_float64(F, H, band, site):
    """q, k, v come from x @ w (D = 64 fmaf from 0), rotated in fp32 (2 roundings, cos / sin of the fp32 angle within 2 ulp);
    the score is a 32-term fmaf chain plus the bias; the online softmax's exp and rescale each within a few u of the score; the
    output sums up to 2 band + 1 weighted rows.  With E_s the largest score error over a query's keys:
        |out - ref| <= (2 E_s + (3 (2 band + 1) + 8) u) max |v| + max e_v
    (the row sum, the weighted sum and the rescales each round once per key)."""
    D, bs, hid = 64, 2, 32 * H
    tag = f"pbattn_banded/{F}/{H}/{band}/{site}"
    t = lambda k, shape, bound: torch.from_numpy(W.symmetric(f"{tag}/{k}", shape, bound)).cuda()   # noqa: E731
    x_q = t("xq", (bs * F, D), 1.7)
    x_kv = x_q if site == "self" else t("xkv", (bs * F, D), 1.7)
    wq, wk, wv = (t(k, (D, hid), 0.25) for k in ("wq", "wk", "wv"))
    npairs = min(32, H) // 2
    freqs = (1. / (10000 ** (torch.arange(0, 2 * npairs, 2).float() / (2 * npairs)))).cuda()
    table = t("bias", (H, 2 * band + 1), 1.7)
    out = torch.empty(bs * F, hid, device="cuda")
    attention_case(bs, F, D, H, band, npairs, x_q, x_kv, wq, wk, wv, freqs, table, out)
    torch.cuda.synchronize()
    d = torch.float64
    xq, xkv = x_q.to(d).view(bs, F, D), x_kv.to(d).view(bs, F, D)
    q, k, v = xq @ wq.to(d), xkv @ wk.to(d), xkv @ wv.to(d)
    ref = banded_reference(q, k, v, table, band, freqs, H)
    # magnitudes: |q|, |k| per feature within the projection's sum of |terms| (rotation mixes a pair: take the pair's sum)
    Q = (xq.abs() @ wq.to(d).abs()) * 32 ** -0.5
    K, V = xkv.abs() @ wk.to(d).abs(), xkv.abs() @ wv.to(d).abs()
    pair = lambda m: (m.view(bs, F, hid // 2, 2).sum(-1, keepdim=True)).expand(bs, F, hid // 2, 2).reshape(bs, F, hid)  # noqa: E731
    Qp, Kp = pair(Q), pair(K)
    e_q, e_k = (D + 8) * U * Qp, (D + 8) * U * Kp
    head = lambda m: m.view(bs, F, H, 32)                                              # noqa: E731
    # E_s <= sum_d (e_q |k| + |q| e_k) + 34 u sum_d |q k| + u |bias|, maximised over the query's band with |q|, |k| <= Qp, Kp
    qe, qm = head(e_q + Qp * 34 * U), head(Qp)
    kmax = head(Kp).amax(1, keepdim=True)
    kemax = head(e_k).amax(1, keepdim=True)
    E_s = (qe * kmax + qm * kemax).sum(-1) + U * table.abs().max().item()             # (bs, F, H)
    vmax = head(V).amax(1).amax(-1)                                                   # (bs, H)
    e_v = (D * U * head(V)).amax(1).amax(-1)
    bound = ((2 * E_s + (3 * (2 * band + 1) + 8) * U) * vmax[:, None, :] + e_v[:, None, :])[..., None].expand(bs, F, H, 32).reshape(bs, F, hid)
    got = out.view(bs, F, hid).double()
    dd = (got - ref).abs()
    el = (dd / bound).max().item()
    r = over_tol(got, ref)
    msg = f"attention F={F} H={H} band={band} {site}: max |d|/bound = {el:.3f}; north-star {r:.3f}"
    if F >= 10000:
        exact = banded_reference(q, k, v, table, band, freqs, H, exact_angles=True)
        msg += (f"; max |d| vs fp32-angle ref {dd.max().item():.3g}, vs fp64-angle ref {(got - exact).abs().max().item():.3g} "
                f"({over_tol(got, exact):.3f} x north-star)")
    print(msg)
    assert el <= 1.0 and r <= 1.0


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

