"""TEST INFRASTRUCTURE — float64 restatement of PBnet's decoder as CAE.generate runs it (never shipped).

The decoder of transformerreemb5 / reemb6 (PBnet/src/models/architectures/transformerreemb5.py:311-378 and
transformerdecoder4.py:24-221), written out from the architecture, with every attention over all F x F frame pairs and the
eval-mode band (|j - i| > band weighs 0) applied as an exclusion.  Also: the configurations of the golden cases, their
deterministic synthetic weights (integer arithmetic only, oracle/weights.py) and inputs.
"""
import math
from dataclasses import dataclass

import numpy as np
import torch

from oracle import weights as W

BANDS = {"transformerreemb5": 200, "transformerreemb6": 100}


@dataclass(frozen=True)
class PbCfg:
    archiname: str = "transformerreemb5"
    pos_dim: int = 6
    eye_dim: int = 0
    audio_dim: int = 1024
    latent_dim: int = 256
    audio_latent_dim: int = 256
    pose_latent_dim: int = 64
    ff_size: int = 128
    num_layers: int = 2
    num_heads: int = 4
    num_buckets: int = 128
    max_distance: int = 128

    @property
    def band(self):
        return BANDS[self.archiname]

    @property
    def out_dim(self):
        return self.pos_dim + (0 if self.archiname == "transformerreemb6" else self.eye_dim)

    def parameters(self, device="cpu"):
        """the dict unified_video_generator.py:80-92 hands get_model: opt.yaml (parser defaults) + device, audio_dim, pos/eye_dim"""
        return dict(modeltype="cvae", archiname=self.archiname, device=device, lambdas={"rc": 1.0, "kl": 1.0, "reg": 0.1},
                    latent_dim=self.latent_dim, num_frames=200, audio_dim=self.audio_dim, pos_dim=self.pos_dim, eye_dim=self.eye_dim,
                    ff_size=self.ff_size, num_layers=self.num_layers, num_heads=self.num_heads,
                    audio_latent_dim=self.audio_latent_dim, pose_latent_dim=self.pose_latent_dim, max_distance=self.max_distance,
                    num_buckets=self.num_buckets, activation="gelu", dropout=0.1)


# name -> (cfg, lengths): the golden cases; F = max(lengths)
CASES = {
    "reemb5_pose_250": (PbCfg(), [250]),
    "reemb5_blink_37": (PbCfg(pos_dim=0, eye_dim=2), [37]),
    "reemb6_pose_150": (PbCfg(archiname="transformerreemb6"), [150]),
    "reemb5_blink_bs2": (PbCfg(pos_dim=0, eye_dim=2), [120, 77]),
    "reemb5_pose_1": (PbCfg(), [1]),
}

# name -> (cfg, lengths): the golden cases of other configurations the library accepts (tests/golden/pbnet_configs.npz).  Widths
# that are not multiples of 64 (d_model 32 and 96) run with bs x F rows on both sides of the contraction dispatcher's 128-row
# line; the reference's encoder needs (audio_latent_dim + 2 d_model) % num_heads == 0.
CONFIG_CASES = {
    "d96_h6_l3_reemb5": (PbCfg(pose_latent_dim=96, num_heads=6, num_layers=3, ff_size=100, audio_dim=128, latent_dim=42,
                               audio_latent_dim=42), [70, 33]),
    "d256_h32_l1_reemb6": (PbCfg(archiname="transformerreemb6", pos_dim=1, pose_latent_dim=256, num_heads=32, num_layers=1,
                                 ff_size=2048, audio_dim=64, latent_dim=96, audio_latent_dim=96), [230]),
    "d32_h2_l4_reemb5": (PbCfg(pos_dim=20, eye_dim=12, pose_latent_dim=32, num_heads=2, num_layers=4, ff_size=1, latent_dim=18,
                               audio_latent_dim=18), [9]),
    "d32_h4_l2_rows150": (PbCfg(pos_dim=3, eye_dim=2, pose_latent_dim=32, num_heads=4, num_layers=2, ff_size=64, audio_dim=192,
                                latent_dim=28, audio_latent_dim=28), [150]),
    "d96_h2_l1_rows80": (PbCfg(archiname="transformerreemb6", pose_latent_dim=96, num_heads=2, num_layers=1, ff_size=256,
                               audio_dim=256, latent_dim=8, audio_latent_dim=8), [40, 17]),
}


# ----------------------------------------------------------------------------- synthetic weights and inputs
def positional_encoding(d_model, max_len=20000):
    pe = torch.zeros(max_len, d_model)
    position = torch.arange(0, max_len, dtype=torch.float).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2).float() * (-math.log(10000.0) / d_model))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe.unsqueeze(0).transpose(0, 1).contiguous()


def synth_value(name, shape):
    shape = tuple(int(s) for s in shape)
    leaf = name.split('.')[-1]
    if leaf == 'pe':
        return positional_encoding(shape[2], shape[0]).numpy()
    if name.endswith('rotary_emb.freqs') or 'relative_attention_bias' in name:
        return W.synth_value(name, shape)
    if leaf == 'gamma' or (leaf == 'weight' and len(shape) == 1):          # LayerNorm gains
        return np.float32(1.0) + W.symmetric(name, shape, 0.2)
    if leaf in ('bias', 'in_proj_bias'):
        return W.symmetric(name, shape, 0.1 if 'norm' in name else 0.05)
    if leaf in ('weight', 'in_proj_weight') and len(shape) == 2:            # nn.Linear default init range
        return W.symmetric(name, shape, 1.0 / math.sqrt(shape[1]))
    raise ValueError(f"no synthetic PBnet rule for {name} {shape}")


def synth_state_dict(schema):
    return {n: torch.from_numpy(np.ascontiguousarray(synth_value(n, s))).float() for n, s in schema}


def synth_inputs(tag, cfg, lengths):
    """first pose (bs, 1, out_dim) in [-0.5, 0.5], audio features ~ N(0, 1) (bs, F, audio_dim), z ~ N(0, 1) (F, bs, latent_dim)"""
    bs, F = len(lengths), max(lengths)
    pose = torch.from_numpy(W.symmetric(f"{tag}/pose", (bs, 1, cfg.out_dim), 0.5))
    audio = torch.from_numpy(W.pseudo_normal(f"{tag}/audio", (bs, F, cfg.audio_dim)))
    z = torch.from_numpy(W.pseudo_normal(f"{tag}/z", (F, bs, cfg.latent_dim)))
    return pose, audio, z, torch.tensor(lengths, dtype=torch.long)


# ----------------------------------------------------------------------------- the decoder
def bucket(rel, num_buckets, max_distance):
    """T5 relative-position bucket of rel = j - i: half the buckets per sign, exact up to num_buckets / 4, then log-spaced up to
    max_distance (evaluated in fp32, as the bucket edges are defined)"""
    n = -rel
    nb = num_buckets // 2
    out = (n < 0).long() * nb
    n = n.abs()
    exact = nb // 2
    large = exact + (torch.log(n.float() / exact) / math.log(max_distance / exact) * (nb - exact)).long()
    large = torch.clamp(large, max=nb - 1)
    return out + torch.where(n < exact, n, large)


def rel_bias(table, F, band, num_buckets, max_distance, dtype):
    """(heads, F, F) bias of pair (i, j), -inf where |j - i| > band"""
    pos = torch.arange(F, device=table.device)
    rel = pos[None, :] - pos[:, None]
    b = table.to(dtype)[bucket(rel, num_buckets, max_distance)].permute(2, 0, 1)
    return b.masked_fill((rel.abs() > band)[None], float("-inf"))


def rotary_angles(F, freqs):
    """(F, len(freqs)) float64 angles f * freq, each rounded to fp32 as the reference's fp32 einsum (and the device's rotary
    table) form it: at 15 000 frames an exact product differs from that by up to half an fp32 ulp of 15 000, 4.9e-4 rad"""
    return (torch.arange(F, device=freqs.device, dtype=torch.float32)[:, None] * freqs.float()[None, :]).double()


def rotate(t, freqs):
    """rotary over the first 2 len(freqs) features of each head, interleaved pairs, position = frame index; the fp32 angle,
    then cos / sin in float64"""
    ang = rotary_angles(t.shape[-2], freqs)
    cos, sin = ang.cos().to(t.dtype), ang.sin().to(t.dtype)
    r = 2 * freqs.shape[0]
    a, b = t[..., 0:r:2], t[..., 1:r:2]
    out = t.clone()
    out[..., 0:r:2] = a * cos - b * sin
    out[..., 1:r:2] = b * cos + a * sin
    return out


def attention(q, k, v, bias, freqs, heads):
    """q (bs, F, 32 H) unscaled, k, v (bs, F, 32 H) -> (bs, F, 32 H): rotary on q * 32^-0.5 and k, + bias, softmax, @ v"""
    bs, F, _ = q.shape
    split = lambda t: t.reshape(bs, F, heads, 32).transpose(1, 2)                 # noqa: E731
    q, k, v = split(q) * 32 ** -0.5, split(k), split(v)
    q, k = rotate(q, freqs), rotate(k, freqs)
    p = torch.softmax(q @ k.transpose(-1, -2) + bias[None], dim=-1)
    return (p @ v).transpose(1, 2).reshape(bs, F, heads * 32)


def layer_norm(x, w, b=None, eps=1e-5):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    y = (x - mu) / torch.sqrt(var + eps) * w
    return y if b is None else y + b


def decoder_forward(sd, cfg, pose, audio, z, lengths, dtype=torch.float64):
    """CAE.generate(pose, audio, lengths)['output'] with the given z (F, bs, latent_dim), in `dtype` on audio's device"""
    dev = audio.device
    p = lambda k: sd["decoder." + k].to(device=dev, dtype=dtype)                  # noqa: E731
    lin = lambda x, name, bias=True: x @ p(name + ".weight").T + (p(name + ".bias") if bias else 0)   # noqa: E731
    bs, F = audio.shape[:2]
    H, band = cfg.num_heads, cfg.band
    x0 = pose.to(device=dev, dtype=dtype)[:, 0, :]
    first = lin(x0, "firstposeEmbedding")[:, None, :].expand(bs, F, -1)
    mem = lin(torch.cat([first, z.to(device=dev, dtype=dtype).permute(1, 0, 2), lin(audio.to(dtype), "audioEmbedding")], -1),
              "ztimelinear")
    tables = {s: rel_bias(sd[f"decoder.time_rel_pos_bias_{s}.relative_attention_bias.weight"].to(dev), F, band, cfg.num_buckets,
                          cfg.max_distance, dtype) for s in ("tgt", "mem")}
    hid = 32 * H
    x = lin(torch.zeros(bs, F, cfg.pose_latent_dim, device=dev, dtype=dtype), "init_proj")
    a = "init_temporal_attn.fn."
    qkv = lin(layer_norm(x, p(a + "norm.gamma")), a + "fn.to_qkv", bias=False)
    x = lin(attention(qkv[..., :hid], qkv[..., hid:2 * hid], qkv[..., 2 * hid:], tables["tgt"], p(a + "fn.rotary_emb.freqs"), H),
            a + "fn.to_out", bias=False) + x
    for l in range(cfg.num_layers):
        s = f"seqTransDecoder.decoder_layers.{l}."
        qkv = lin(x, s + "self_attn.to_qkv", bias=False)
        o = attention(qkv[..., :hid], qkv[..., hid:2 * hid], qkv[..., 2 * hid:], tables["tgt"], p(s + "self_attn.rotary_emb.freqs"), H)
        x = layer_norm(x + lin(o, s + "self_attn.to_out", bias=False), p(s + "layer_norm1.weight"), p(s + "layer_norm1.bias"))
        c = s + "multihead_attn."
        o = attention(lin(x, c + "to_q", bias=False), lin(mem, c + "to_k", bias=False), lin(mem, c + "to_v", bias=False),
                      tables["mem"], p(c + "rotary_emb.freqs"), H)
        x = layer_norm(x + lin(o, c + "to_out", bias=False), p(s + "layer_norm2.weight"), p(s + "layer_norm2.bias"))
        h = torch.nn.functional.gelu(lin(x, s + "ffn.linear1"))
        x = layer_norm(x + lin(h, s + "ffn.linear2"), p(s + "layer_norm3.weight"), p(s + "layer_norm3.bias"))
    out = lin(x, "finallayer")
    mask = torch.arange(F, device=dev)[None, :] < lengths.to(dev)[:, None]
    return out.masked_fill(~mask[..., None], 0.0)
