"""GPU: the HuBERT audio encoder on the device (dawn_pytorch_b200/hubert.py, include/dawn_hubert.h), at the north-star tolerance
|d| <= 1e-4 + 1e-3 |ref| unless a kernel's own bound is derived below.

* every golden case (made by transformers' HubertModel) matches: hubert-large on 1 s, an odd length and a batch of 2, two small
  configurations, and hubert_features on 21 s of speech (one segment boundary and the tail) and on 100 s (five full segments,
  more than one forward's worth, and the tail);
* hubert_features run 4 full segments to a forward equals it run one segment to a forward, bit for bit;
* the hidden state after the positional conv and after every encoder layer matches the float64 oracle run on the same GPU
  (hubert-large at 1 s, and at 3 s where every contraction runs on the wgmma GEMM), and so do the output and four boundaries of
  two full 20 s segments in one forward;
* a batch of 2 clips of 3 s equals each clip run alone, bit for bit;
* the attention, layer-0 conv and positional-conv kernel entries match float64 for T in {1, 49, 63, 64, 65, 1000, 3000};
* one forward is 2 n + G + 7 L + 3 launches; CPU tensors raise.
Transformers is not imported here.
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from dawn_pytorch_b200._lib import HUBERT_ATTENTION, HUBERT_CONV0, HUBERT_POS_CONV
from oracle import hubert_oracle as O
from oracle import weights as W

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RTOL, ATOL = 1e-3, 1e-4
TS = [1, 49, 63, 64, 65, 1000, 3000]
U = 2.0 ** -24                      # fp32 unit roundoff


def over_tol(a, ref):
    a, ref = a.detach().double().cpu(), ref.detach().double().cpu()
    return ((a - ref).abs() / (ATOL + RTOL * ref.abs())).max().item()


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLD, "hubert.npz"))


@pytest.fixture(scope="module")
def schema():
    with open(os.path.join(GOLD, "hubert_schema.json")) as f:
        return {k: [(n, tuple(s)) for n, s in v] for k, v in json.load(f).items()}


_MODELS = {}


def cuda_model(cname, schema):
    """one device model per configuration (hubert-large holds 1.2 GB of weights)"""
    if cname not in _MODELS:
        from dawn_pytorch_b200.hubert import HubertModel
        sd = O.synth_state_dict(schema[cname])
        model = HubertModel(O.CONFIGS[cname]).cuda()
        model.load_state_dict(sd, strict=True)
        _MODELS[cname] = (model.eval(), sd)
    return _MODELS[cname]


@pytest.mark.parametrize("case", [c for c, v in O.CASES.items() if v[1] == "model"])
def test_golden_case_matches_transformers(case, golden, schema):
    cname, _, lengths = O.CASES[case]
    model, _ = cuda_model(cname, schema)
    x = O.synth_input_values(case, lengths).cuda()
    out = model(x).last_hidden_state
    step = O.PROBE_STEP.get(case, 1)
    ref = torch.from_numpy(golden[f"{case}/out"])
    assert out[..., ::step].shape == ref.shape
    r = over_tol(out[..., ::step], ref)
    print(f"{case}: max |d| / tol = {r:.3f}")
    assert r <= 1.0


@pytest.mark.parametrize("case", [c for c, v in O.CASES.items() if v[1] == "features"])
def test_features_match_golden(case, golden, schema):
    from dawn_pytorch_b200.hubert import hubert_features
    cname, _, lengths = O.CASES[case]
    model, _ = cuda_model(cname, schema)
    feats = hubert_features(model, O.synth_speech(case, lengths[0]))
    assert feats.device.type == "cuda" and feats.dtype == torch.float32
    step = O.PROBE_STEP.get(case, 1)
    ref = torch.from_numpy(golden[f"{case}/out"])
    assert feats[:, ::step].shape == ref.shape
    r = over_tol(feats[:, ::step], ref)
    print(f"{case}: max |d| / tol = {r:.3f}")
    assert r <= 1.0


def test_capped_segment_batches_equal_one_segment_per_forward(schema, monkeypatch):
    # 9 full segments and a tail: forwards of 4, 4, 1 and the tail against ten forwards of one.  Every contraction has >= 128 rows
    # either way, so both take the same kernel paths and batching may not change a bit.
    from dawn_pytorch_b200 import hubert as HB
    model, _ = cuda_model("small_a", schema)
    speech = O.synth_speech("cap", 9 * HB.CLIP + 7000)
    assert [len(b) for b in HB.segment_batches(HB.segment_plan(speech.shape[0]))] == [4, 4, 1, 1]
    capped = HB.hubert_features(model, speech)
    monkeypatch.setattr(HB, "SEGMENTS_PER_CALL", 1)
    assert torch.equal(capped, HB.hubert_features(model, speech))


# cases without a golden: 3 s of hubert-large is 149 frames, so every contraction has >= 128 rows and runs on the wgmma GEMM
ORACLE_ONLY = {"large_3s": ("large", "model", [48000])}


@pytest.mark.parametrize("case", ["large_1s", "small_b", "large_3s"])
def test_every_layer_boundary_matches_oracle(case, golden, schema):
    cname, _, lengths = O.CASES[case] if case in O.CASES else ORACLE_ONLY[case]
    c = O.CONFIGS[cname]
    model, sd = cuda_model(cname, schema)
    x = O.synth_input_values(case, lengths).cuda()
    _, taps = O.forward(sd, c, x.double(), boundaries=True)
    worst = 0.0
    for layer, ref in enumerate(taps):
        r = over_tol(model.hidden_state(x, layer), ref)
        worst = max(worst, r)
        assert r <= 1.0, f"boundary {layer}: {r:.3f}"
    print(f"{case}: worst boundary max |d| / tol = {worst:.3f}")
    if case in O.CASES:
        # the goldens' per-frame mean |h| of every boundary, made by transformers, agree with the oracle's
        am = torch.stack([t.abs().mean(-1) for t in taps]).float().cpu()
        assert over_tol(am, torch.from_numpy(golden[f"{case}/absmean"])) <= 0.1


def test_two_full_segments_match_oracle(schema):
    # hubert_features' forward of two full 20 s segments (2 x 1000 rows, the production row counts of q|k|v, fc1 and fc2 on the
    # wgmma GEMM): the output and the boundaries after the positional conv and after layers 1, 12 and 24, against float64
    from dawn_pytorch_b200.hubert import SEGMENT
    model, sd = cuda_model("large", schema)
    c = O.CONFIGS["large"]
    x = O.synth_input_values("two_segments", [SEGMENT, SEGMENT]).cuda()
    out_ref, taps = O.forward(sd, c, x.double(), boundaries=True)
    assert out_ref.shape[:2] == (2, 1000)
    margins = {"out": over_tol(model(x).last_hidden_state, out_ref)}
    for layer in (0, 1, 12, 24):
        margins[f"layer {layer}"] = over_tol(model.hidden_state(x, layer), taps[layer])
    print("two 20 s segments: max |d| / tol " + ", ".join(f"{k} {v:.3f}" for k, v in margins.items()))
    assert max(margins.values()) <= 1.0


def test_batch_of_two_equals_each_clip_alone(schema):
    # 3 s: every contraction has >= 128 rows alone and batched, so both runs take the same kernel paths and batching may not
    # change a bit (shorter clips can cross the 128-row line of the wgmma path in one run and not the other)
    model, _ = cuda_model("large", schema)
    x = torch.cat([O.synth_input_values("large_1s", [48000]), O.synth_input_values("large_b2", [48000])]).cuda()
    both = model(x).last_hidden_state
    for b in range(2):
        assert torch.equal(both[b], model(x[b:b + 1]).last_hidden_state[0])


def test_launch_count_and_cpu_tensors_raise(schema):
    from dawn_pytorch_b200._lib import DawnError
    model, _ = cuda_model("large", schema)
    model(O.synth_input_values("large_1s", [16000]).cuda())
    c = O.CONFIGS["large"]
    n, G, L = len(c["conv_dim"]), c["num_conv_pos_embedding_groups"], c["num_hidden_layers"]
    assert model.last_launch_count() == 2 * n + G + 7 * L + 3
    with pytest.raises(DawnError):
        model(O.synth_input_values("large_1s", [16000]))


# ------------------------------------------------------------------------------------------------ kernel entries
def _case(**kw):
    from dawn_pytorch_b200 import _lib
    c = _lib.DawnHubertKernelCase()
    for k, v in kw.items():
        setattr(c, k, ctypes.c_void_p(v.data_ptr()) if torch.is_tensor(v) else v)
    _lib.check(_lib.lib.dawn_hubert_test_kernel(ctypes.byref(c), _lib.stream()), "dawn_hubert_test_kernel")


def _dev(key, shape, bound=1.0):
    return torch.from_numpy(W.symmetric(key, shape, bound)).cuda()


@pytest.mark.parametrize("T", TS)
def test_attention_kernel_matches_float64(T):
    B, H = 2, 3
    D = 64 * H
    qkv = _dev(f"hb_attn/{T}", (B * T, 3 * D), 2.0)
    qkv[:, :D] *= 0.125                                      # q arrives pre-scaled, as the q|k|v contraction writes it
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    out = torch.full((B * T, D), float("nan"), device="cuda")
    _case(kernel=HUBERT_ATTENTION, B=B, T=T, H=H, ld=3 * D, q=q, kk=k, v=v, out=out)
    heads = lambda t: t.double().view(B, T, H, 64).transpose(1, 2)  # noqa: E731
    qd, kd, vd = heads(q), heads(k), heads(v)
    ref = (torch.softmax(qd @ kd.transpose(-1, -2), -1) @ vd).transpose(1, 2).reshape(B * T, D)
    # FP16x3 products carry <= 2^-21 relative error each (hi / lo split, the dropped lo*lo term): on the scores that is
    # 2^-21 sum_d |q k| and after the softmax a relative weight error of twice that; P V adds 2^-21 max|v| and the fp32 sums
    # 64 + T roundings.  Bound: (2^-20 S + 2^-21 + (64 + T) 2^-24) max|v| with S = max_ij sum_d |q_id k_jd|, doubled.
    S = (qd.abs() @ kd.abs().transpose(-1, -2)).max().item()
    bound = 2 * (2.0 ** -20 * S + 2.0 ** -21 + (64 + T) * U) * vd.abs().max().item()
    err = (out.double() - ref).abs().max().item()
    print(f"T={T}: attention max |d| {err:.2e}, bound {bound:.2e}")
    assert err <= bound


@pytest.mark.parametrize("T", TS)
def test_conv0_kernel_matches_float64(T):
    B, C, k, s = 2, 512, 10, 5
    L = (T - 1) * s + k + 3
    x = _dev(f"hb_conv0/{T}/x", (B, L), 3.0)
    w, b = _dev("hb_conv0/w", (C, 1, k), 0.3), _dev("hb_conv0/b", (C,), 0.05)
    g, be = 1 + _dev("hb_conv0/g", (C,), 0.2), _dev("hb_conv0/be", (C,), 0.05)
    out = torch.full((B * T, C), float("nan"), device="cuda")
    _case(kernel=HUBERT_CONV0, B=B, L=L, C=C, k=k, s=s, eps=1e-5, x=x, w=w, bias=b, gamma=g, beta=be, out=out)
    y = Fn.conv1d(x.double()[:, None], w.double(), b.double(), stride=s).transpose(1, 2)
    ref = Fn.gelu(Fn.layer_norm(y, (C,), g.double(), be.double(), 1e-5))
    # Propagated fp32 error (u = 2^-24), per row:
    #   conv: k fused multiply-adds onto the bias:          e_y  <= (k + 1) u (|b| + sum_i |w_i x_i|)
    #   mean of C values (lane sums, then the warp tree):  e_mu <= max e_y + C u max|y|
    #   centred d = y - mu:                                 e_d  <= e_y + e_mu + u |d|
    #   variance: relative error of rstd                    r    <= sum_c |d| e_d / (C var) + (C + 2) u
    #   n = d rstd:                                         e_n  <= rstd e_d + |n| (r + 2 u)
    #   out = GELU(n gamma + beta), GELU slope <= 1.13 and erff within 4 u:  1.13 (|gamma| e_n + 2 u |n gamma + beta|) + 4 u (|ref| + 1)
    mag = Fn.conv1d(x.double().abs()[:, None], w.double().abs(), b.double().abs(), stride=s).transpose(1, 2)
    e_y = (k + 1) * U * mag
    e_mu = e_y.amax(-1, keepdim=True) + C * U * y.abs().amax(-1, keepdim=True)
    d = y - y.mean(-1, keepdim=True)
    e_d = e_y + e_mu + U * d.abs()
    var = d.pow(2).mean(-1, keepdim=True)
    rstd = (var + 1e-5).rsqrt()
    r = (d.abs() * e_d).sum(-1, keepdim=True) / (C * var) + (C + 2) * U
    n = d * rstd
    e_n = rstd * e_d + n.abs() * (r + 2 * U)
    bound = 1.13 * (g.double().abs() * e_n + 2 * U * (n * g.double() + be.double()).abs()) + 4 * U * (ref.abs() + 1)
    err = (out.double().view(B, T, C) - ref).abs()
    print(f"T={T}: conv0 max |d| {err.max().item():.2e}, max bound {bound.max().item():.2e}, north-star {over_tol(out, ref.reshape(B * T, C)):.3f}")
    assert (err <= bound).all()
    assert over_tol(out, ref.reshape(B * T, C)) <= 1.0


@pytest.mark.parametrize("T", TS)
def test_pos_conv_kernel_matches_float64(T):
    B, G, k = 1, 16, 128
    D = 64 * G
    x = _dev(f"hb_pos/{T}/x", (B, T, D), 2.0)
    g, v, b = 1 + _dev("hb_pos/g", (1, 1, k), 0.5), _dev("hb_pos/v", (D, 64, k)), _dev("hb_pos/b", (D,), 0.05)
    out = torch.full((B, T, D), float("nan"), device="cuda")
    _case(kernel=HUBERT_POS_CONV, B=B, T=T, G=G, k=k, x=x, g=g, w=v, bias=b, out=out)
    w = g.double() * v.double() / v.double().pow(2).sum(dim=(0, 1), keepdim=True).sqrt()
    xt = x.double().transpose(1, 2)
    conv = Fn.conv1d(xt, w, b.double(), padding=k // 2, groups=G)[:, :, :T]
    ref = x.double() + Fn.gelu(conv).transpose(1, 2)
    # Relative to sum |w x| over the K = 64 k window (u = 2^-24): a 3-term split product is within 2^-20 of w x (the dropped lo*lo
    # term and the fp16 rounding of the lo pieces).  Accumulation depends on the path the dispatcher takes:
    #   wgmma (>= 128 rows): the tensor core adds with truncation (<= 2 u per add) inside a chunk of 4 panels = 16 k16 steps x 3
    #     split terms, then each chunk is drained into fp32 with one rounded add: 48 * 2 u + K / 256 u;
    #   mma.sync (< 128 rows): each 8-wide k-step's 3 split MMAs land in a zeroed fragment (3 truncations) and are added to the
    #     running sum with one rounded add: 3 * 2 u + K / 8 u.
    # The bias, GELU (slope <= 1.13) and residual add a few roundings of |ref|.
    K = 64 * k
    acc = (48 * 2 + K / 256) * U if B * T >= 128 else (3 * 2 + K / 8) * U
    mag = Fn.conv1d(xt.abs(), w.abs(), None, padding=k // 2, groups=G)[:, :, :T].transpose(1, 2)
    bound = 1.13 * (2.0 ** -20 + acc) * mag + 4 * U * (ref.abs() + x.double().abs())
    err = (out.double() - ref).abs()
    r = over_tol(out, ref)
    print(f"T={T}: pos conv max |d| {err.max().item():.2e}, max bound {bound.max().item():.2e}, north-star {r:.3f}")
    assert (err <= bound).all()
    assert r <= 1.0
