"""TEST INFRASTRUCTURE — float64 functional restatement of transformers' HubertModel (stable-layer-norm variant, eval mode) and of
the generator's audio pipeline (unified_video_generator.py:229-242, 450-501), the deterministic synthetic weights and inputs of
the HuBERT parity cases, and the case list shared by oracle/make_golden_hubert.py and the tests.

Written from the model's documented semantics:
  feature extractor  per conv layer: Conv1d (bias) -> LayerNorm over channels (eps 1e-5) -> erf GELU
  feature projection LayerNorm(conv_dim[-1], layer_norm_eps) -> Linear
  positional conv    Conv1d(D, D, k, padding k // 2, groups G), weight norm over dim 2 (w = g v / ||v|| per tap), the last output
                     frame dropped when k is even, GELU, added to the hidden state
  encoder layers     h += out_proj(MHA(LN(h))) with q / sqrt(64); h += fc2(GELU(fc1(final_layer_norm(h)))); then encoder.layer_norm
"""
import math

import numpy as np
import torch
import torch.nn.functional as Fn

from oracle import weights as W

KERNEL, STRIDE = 400, 320
CLIP = STRIDE * 1000
SEGMENT = CLIP - STRIDE + KERNEL


def config(**over):
    """HubertConfig fields of hubert-large-ls960-ft, with overrides"""
    c = dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096, hidden_act="gelu",
             layer_norm_eps=1e-5, feat_extract_norm="layer", feat_extract_activation="gelu", conv_dim=[512] * 7,
             conv_stride=[5, 2, 2, 2, 2, 2, 2], conv_kernel=[10, 3, 3, 3, 3, 2, 2], conv_bias=True, num_conv_pos_embeddings=128,
             num_conv_pos_embedding_groups=16, do_stable_layer_norm=True, feat_proj_layer_norm=True, conv_pos_batch_norm=False,
             mask_time_prob=0.05, mask_feature_prob=0.0)
    c.update(over)
    return c


LARGE = config()
SMALL_A = config(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, intermediate_size=512, conv_dim=[256] * 7,
                 num_conv_pos_embeddings=16, num_conv_pos_embedding_groups=4)
SMALL_B = config(hidden_size=512, num_hidden_layers=3, num_attention_heads=8, intermediate_size=1024, conv_dim=[384] * 5,
                 conv_stride=[5, 2, 2, 2, 2], conv_kernel=[10, 3, 3, 2, 2], conv_bias=False, num_conv_pos_embeddings=31,
                 num_conv_pos_embedding_groups=8, layer_norm_eps=1e-6, mask_time_prob=0.0)

CONFIGS = {"large": LARGE, "small_a": SMALL_A, "small_b": SMALL_B}
# name -> (config name, kind, lengths): "model" cases run HubertModel on (len(lengths), max(lengths)) normalised noise; the
# "features" case runs hubert_features on that many samples of synthetic speech
CASES = {
    "large_1s": ("large", "model", [16000]),
    "large_odd": ("large", "model", [23457]),
    "large_b2": ("large", "model", [12000, 12000]),
    "small_a": ("small_a", "model", [9999]),
    "small_b": ("small_b", "model", [5000, 5000, 5000]),
    "features_21s": ("small_a", "features", [21 * 16000 + 3217]),
    "features_5seg": ("small_a", "features", [5 * 320000 + 6000]),      # 5 full segments and a tail: more than one batch
}
PROBE_STEP = {"large_1s": 4, "large_odd": 4, "large_b2": 4, "features_21s": 4, "features_5seg": 16}   # channels kept: [..., ::step]


# ------------------------------------------------------------------------------------------------ synthetic weights and inputs
def synth_value(name, shape):
    """LayerNorm gains 1 +- 0.2, biases +- 0.05, Linear / conv weights U(+-1/sqrt(fan_in)) (torch's default range); out_proj and
    fc2 at half that, so the residual stream of 24 layers stays O(1-10); weight-norm g in [0.5, 1.5], v U(+-1)"""
    shape = tuple(int(s) for s in shape)
    leaf = name.split('.')[-1]
    if name == "masked_spec_embed":
        return W.symmetric(name, shape, 1.0)
    if leaf == "original0":
        return np.float32(1.0) + W.symmetric(name, shape, 0.5)
    if leaf == "original1":
        return W.symmetric(name, shape, 1.0)
    if "layer_norm" in name and leaf == "weight":
        return np.float32(1.0) + W.symmetric(name, shape, 0.2)
    if leaf == "bias":
        return W.symmetric(name, shape, 0.05)
    if leaf == "weight":
        fan_in = int(np.prod(shape[1:]))
        gain = 0.5 if ("out_proj" in name or "output_dense" in name) else 1.0
        return W.symmetric(name, shape, gain / math.sqrt(fan_in))
    raise ValueError(f"no synthetic HuBERT rule for {name} {shape}")


def synth_state_dict(schema):
    return {n: torch.from_numpy(np.ascontiguousarray(synth_value(n, s))).float() for n, s in schema}


def synth_speech(tag, n):
    """n samples of a deterministic speech-like float32 signal: a few drifting tones under a syllable envelope, plus noise"""
    t = np.arange(n, dtype=np.float64) / 16000.0
    f = 120.0 + 40.0 * W.uniform01(f"{tag}/f0", 1)[0]
    env = 0.5 + 0.5 * np.sin(2 * np.pi * 3.7 * t) ** 2
    x = env * (np.sin(2 * np.pi * f * t) + 0.5 * np.sin(2 * np.pi * 2.7 * f * t + 0.3))
    x += 0.2 * W.pseudo_normal(f"{tag}/noise", (n,)).astype(np.float64)
    return (0.1 * x).astype(np.float32)


def synth_input_values(tag, lengths):
    """(B, L) float32 normalised noise-like input values, one row per length (all equal)"""
    return torch.from_numpy(W.pseudo_normal(f"{tag}/input", (len(lengths), max(lengths))))


def schema_of(c):
    """HubertModel's state_dict names and shapes for config c, in transformers' order"""
    D, I, k, G = c["hidden_size"], c["intermediate_size"], c["num_conv_pos_embeddings"], c["num_conv_pos_embedding_groups"]
    s = []
    if c["mask_time_prob"] > 0 or c["mask_feature_prob"] > 0:
        s.append(("masked_spec_embed", (D,)))
    for i, (co, kk) in enumerate(zip(c["conv_dim"], c["conv_kernel"])):
        p = f"feature_extractor.conv_layers.{i}."
        s.append((p + "conv.weight", (co, 1 if i == 0 else c["conv_dim"][i - 1], kk)))
        if c["conv_bias"]:
            s.append((p + "conv.bias", (co,)))
        s += [(p + "layer_norm.weight", (co,)), (p + "layer_norm.bias", (co,))]
    C = c["conv_dim"][-1]
    s += [("feature_projection.layer_norm.weight", (C,)), ("feature_projection.layer_norm.bias", (C,)),
          ("feature_projection.projection.weight", (D, C)), ("feature_projection.projection.bias", (D,)),
          ("encoder.pos_conv_embed.conv.bias", (D,)),
          ("encoder.pos_conv_embed.conv.parametrizations.weight.original0", (1, 1, k)),
          ("encoder.pos_conv_embed.conv.parametrizations.weight.original1", (D, D // G, k)),
          ("encoder.layer_norm.weight", (D,)), ("encoder.layer_norm.bias", (D,))]
    for l in range(c["num_hidden_layers"]):
        p = f"encoder.layers.{l}."
        for n in ("k_proj", "v_proj", "q_proj", "out_proj"):
            s += [(p + f"attention.{n}.weight", (D, D)), (p + f"attention.{n}.bias", (D,))]
        s += [(p + "layer_norm.weight", (D,)), (p + "layer_norm.bias", (D,)),
              (p + "feed_forward.intermediate_dense.weight", (I, D)), (p + "feed_forward.intermediate_dense.bias", (I,)),
              (p + "feed_forward.output_dense.weight", (D, I)), (p + "feed_forward.output_dense.bias", (D,)),
              (p + "final_layer_norm.weight", (D,)), (p + "final_layer_norm.bias", (D,))]
    return s


# ------------------------------------------------------------------------------------------------ the model
def output_length(c, L):
    for k, s in zip(c["conv_kernel"], c["conv_stride"]):
        L = (L - k) // s + 1
    return L


def _ln(x, sd, p, eps):
    return Fn.layer_norm(x, x.shape[-1:], sd[p + ".weight"], sd[p + ".bias"], eps)


def forward(sd, c, x, boundaries=False):
    """input values (B, L) -> last_hidden_state (B, T, D) in the dtype of x (float64 for the oracle).  boundaries: also return
    the hidden state after the positional conv and after every encoder layer (before encoder.layer_norm), as a list."""
    dt, dev = x.dtype, x.device
    sd = {k: v.to(dev, dt) for k, v in sd.items()}
    eps = c["layer_norm_eps"]
    h = x[:, None, :]
    for i, s in enumerate(c["conv_stride"]):
        p = f"feature_extractor.conv_layers.{i}."
        h = Fn.conv1d(h, sd[p + "conv.weight"], sd.get(p + "conv.bias"), stride=s)
        h = Fn.gelu(_ln(h.transpose(1, 2), sd, p + "layer_norm", 1e-5)).transpose(1, 2)
    h = h.transpose(1, 2)
    h = Fn.linear(_ln(h, sd, "feature_projection.layer_norm", eps), sd["feature_projection.projection.weight"],
                  sd["feature_projection.projection.bias"])
    g = sd["encoder.pos_conv_embed.conv.parametrizations.weight.original0"]
    v = sd["encoder.pos_conv_embed.conv.parametrizations.weight.original1"]
    w = g * v / v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt()
    k = v.shape[-1]
    pc = Fn.conv1d(h.transpose(1, 2), w, sd["encoder.pos_conv_embed.conv.bias"], padding=k // 2,
                   groups=c["num_conv_pos_embedding_groups"])
    if k % 2 == 0:
        pc = pc[:, :, :-1]
    h = h + Fn.gelu(pc).transpose(1, 2)
    taps = [h]
    B, T, D = h.shape
    H = c["num_attention_heads"]
    for l in range(c["num_hidden_layers"]):
        p = f"encoder.layers.{l}."
        a = _ln(h, sd, p + "layer_norm", eps)
        proj = lambda n: Fn.linear(a, sd[p + f"attention.{n}.weight"], sd[p + f"attention.{n}.bias"]).view(B, T, H, 64).transpose(1, 2)  # noqa: E731
        q, kk, vv = proj("q_proj") * 0.125, proj("k_proj"), proj("v_proj")
        o = torch.softmax(q @ kk.transpose(-1, -2), dim=-1) @ vv
        o = o.transpose(1, 2).reshape(B, T, D)
        h = h + Fn.linear(o, sd[p + "attention.out_proj.weight"], sd[p + "attention.out_proj.bias"])
        f = _ln(h, sd, p + "final_layer_norm", eps)
        f = Fn.gelu(Fn.linear(f, sd[p + "feed_forward.intermediate_dense.weight"], sd[p + "feed_forward.intermediate_dense.bias"]))
        h = h + Fn.linear(f, sd[p + "feed_forward.output_dense.weight"], sd[p + "feed_forward.output_dense.bias"])
        taps.append(h)
    out = _ln(h, sd, "encoder.layer_norm", eps)
    return (out, taps) if boundaries else out


# ------------------------------------------------------------------------------------------------ the generator's pipeline
def normalize(speech):
    x = np.asarray(speech, dtype=np.float32)
    return (x - x.mean()) / np.sqrt(x.var() + 1e-7)


def features(model_fn, speech, num_frames=None):
    """unified_video_generator.py:229-242, 450-501 with the model as a function (B, L) tensor -> (B, T, D) tensor"""
    n = speech.shape[0]
    if num_frames is None:
        num_frames = int((n / 16000) * 25)
    x = torch.from_numpy(normalize(speech))
    num_iter = n // CLIP
    res = [model_fn(x[CLIP * i:CLIP * i + SEGMENT][None])[0] for i in range(num_iter)]
    tail = x[CLIP * num_iter:]
    if tail.shape[0] >= KERNEL:
        res.append(model_fn(tail[None])[0])
    ret = torch.cat(res, 0)
    expected = (n - (KERNEL - STRIDE)) // STRIDE
    assert abs(ret.shape[0] - expected) <= 1
    ret = Fn.pad(ret, (0, 0, 0, expected - ret.shape[0])) if ret.shape[0] < expected else ret[:expected]
    y = ret.double().cpu().numpy()
    T = y.shape[0]
    xs, xn = np.arange(T), np.linspace(0, T - 1, num_frames)
    hi = np.searchsorted(xs, xn).clip(1, T - 1)
    lo = hi - 1
    return torch.from_numpy((((xn - xs[lo]) / (xs[hi] - xs[lo]))[:, None] * y[hi]
                             + ((xs[hi] - xn) / (xs[hi] - xs[lo]))[:, None] * y[lo]).astype(np.float32))
