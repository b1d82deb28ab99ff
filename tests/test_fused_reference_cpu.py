"""CPU: the float64 references of tests/fused_ref.py, which the per-kernel GPU tests hold the fused kernels to, against the oracle
functions of oracle/unet_oracle.py, which the goldens pin to the real reference.  Each reference gets the oracle's inputs: the T5
bucket bias of rel = key - query laid out per (head, rel), and the rotary table of positions arange(F).  The references then
carry the project's semantics for the shapes the network does not run (bands 41-64, query windows q_lo > 0, SLA split
lengths), where only the per-kernel tests look.
"""
import math

import pytest
import torch
import torch.nn.functional as TF

from oracle import unet_oracle as O
from tests import fused_ref as R

DT = torch.float64


def rnd(shape, seed, scale=1.0, dtype=DT):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=DT) * scale).to(dtype)


def close(name, a, b, tol):
    err = ((a - b).abs().max() / b.abs().max()).item()
    print(f"  {name}: max |ref - oracle| / max |oracle| = {err:.2e}")
    assert err <= tol, f"{name}: {err:.2e} > {tol:.0e}"


def attn_sd(p, C, seed, conv=False):
    shape = (1, C, 1, 1, 1)
    qkv, out = rnd((768, C), seed + 1, 0.125), rnd((C, 256), seed + 2, 0.0625)
    sd = {p + ".norm.gamma": 1 + 0.2 * rnd(shape, seed)}
    if conv:                                                 # SpatialLinearAttention: 1x1 conv weights and an output bias
        sd.update({p + ".fn.to_qkv.weight": qkv[:, :, None, None], p + ".fn.to_out.weight": out[:, :, None, None],
                   p + ".fn.to_out.bias": rnd(C, seed + 3)})
    else:
        sd.update({p + ".fn.fn.to_qkv.weight": qkv, p + ".fn.fn.to_out.weight": out})
    return sd, sd[p + ".norm.gamma"].reshape(C), qkv, out


@pytest.mark.parametrize("Fr,band,q_lo,q_hi", [(30, 8, 0, 30), (50, 41, 0, 50), (70, 64, 0, 70), (80, 20, 30, 70), (12, 40, 0, 12)])
def test_temporal_against_oracle(Fr, band, q_lo, q_hi):
    C, H, W = 64, 2, 3
    sd, gamma, wqkv, wout = attn_sd("t", C, Fr + band)
    x = rnd((Fr, C, H, W), 7)
    emb = rnd((32, 8), 8)
    freqs = 1.0 / (10000 ** (torch.arange(0, 32, 2, dtype=DT) / 32))
    want = O.temporal_attention(sd, "t", x, O.rel_pos_bias(emb, Fr, band), freqs, band=band)     # (F, C, H, W)
    rel = torch.arange(-band, band + 1)
    bias = emb[O.rel_pos_bucket(rel, 32, 32)].t()                                               # (heads, 2 band + 1)
    ang = torch.arange(Fr, dtype=DT)[:, None] * freqs[None, :]
    rot = torch.stack((ang.cos(), ang.sin()), -1)
    seq = x.permute(2, 3, 0, 1).reshape(H * W, Fr, C)
    out, bound, _ = R.temporal(seq, seq[:, q_lo:q_hi], gamma, wqkv, wout, rot, bias, band, q_lo, q_hi)
    close("temporal", out, want.permute(2, 3, 0, 1).reshape(H * W, Fr, C)[:, q_lo:q_hi], 1e-12)
    assert torch.isfinite(bound).all() and (bound > 0).all()


@pytest.mark.parametrize("P", [64, 80])
def test_sla_against_oracle(P):
    C, Fr = 64, 3
    H, W = 8, P // 8
    sd, gamma, wqkv, wout = attn_sd("s", C, P, conv=True)
    x = rnd((Fr, C, H, W), 9)
    want = O.spatial_linear_attention(sd, "s", x)
    xs = x.permute(0, 2, 3, 1).reshape(Fr, P, C)
    Bf, _ = R.sla_ctx(xs, gamma, wqkv, wout)
    out, _ = R.sla_out(xs, gamma, wqkv, Bf, sd["s.fn.to_out.bias"])
    close("sla", out, want.permute(0, 2, 3, 1).reshape(Fr, P, C), 1e-12)


@pytest.mark.parametrize("H,W", [(3, 3), (8, 8), (10, 20)])
def test_full_attention_against_oracle(H, W):
    C, Fr = 128, 2
    sd, gamma, wqkv, wout = attn_sd("m", C, H * W)
    x = rnd((Fr, C, H, W), 10)
    want = O.mid_spatial_attention(sd, "m", x)
    tok = x.permute(0, 2, 3, 1).reshape(Fr, H * W, C)
    Wf = wqkv * gamma[None, :]
    Wf[:256] *= 32 ** -0.5
    qkv = R.layernorm(tok)[0] @ Wf.t()
    hd = lambda t: t.reshape(Fr, H * W, 8, 32).transpose(1, 2)
    q, k, v = hd(qkv[..., :256]), hd(qkv[..., 256:512]), hd(qkv[..., 512:])
    o, _ = R.attention(q, k, v, torch.arange(H * W), 1 << 30, None, 0.0, 0.0, full=True)
    out = tok + o.transpose(1, 2).reshape(Fr, H * W, 256) @ wout.t()
    close("mid attention", out, want.permute(0, 2, 3, 1).reshape(Fr, H * W, C), 1e-12)


def ca_tables(sd, p, ctx, co):
    """kq, nkq, G and T of one cross-attention, from its parameters (the per-clip tables the CA kernels consume)"""
    kv = ctx @ sd[p + ".to_kv.weight"].t()
    k, v = kv[:, :64].reshape(-1, 8, 8), kv[:, 64:].reshape(-1, 8, 8)
    nk, nv = sd[p + ".null_kv"][0], sd[p + ".null_kv"][1]
    sc = sd[p + ".k_scale"] * sd[p + ".q_scale"]
    kq = (TF.normalize(k, dim=-1) * sc).reshape(-1, 64)
    nkq = TF.normalize(nk, dim=-1) * sc
    Wo = sd[p + ".to_out.0.weight"].reshape(co, 8, 8)                                         # (c, head, dim)
    u = torch.cat(((Wo @ nv).sum(1)[None].expand(ctx.shape[0], co)[:, None],                 # (F, 9, co)
                   torch.einsum("chd,fhd->fhc", Wo, v - nv)), 1)
    u = u - u.mean(-1, keepdim=True)
    G = (u @ u.transpose(1, 2) / co).reshape(-1, 81)
    T = u * sd[p + ".to_out.1.g"]
    return kq, nkq, G, T


@pytest.mark.parametrize("ci,co", [(64, 64), (128, 256)])
def test_cross_attention_against_oracle(ci, co):
    Fr, n = 3, 20
    names = ["pose", "aud", "eye"]
    sd, g3, toq, ctxs = {}, [], [], []
    for a, nm in enumerate(names):
        p = "ca_" + nm
        s = 11 * a + ci
        sd.update({p + ".norm.g": 1 + 0.2 * rnd(ci, s), p + ".to_q.weight": rnd((64, ci), s + 1, ci ** -0.5),
                   p + ".to_kv.weight": rnd((128, 2 * co), s + 2, (2 * co) ** -0.5), p + ".null_kv": rnd((2, 8), s + 3),
                   p + ".q_scale": 1 + 0.3 * rnd(8, s + 4), p + ".k_scale": 1 + 0.3 * rnd(8, s + 5),
                   p + ".to_out.0.weight": rnd((co, 64), s + 6, 0.125), p + ".to_out.1.g": 1 + 0.2 * rnd(co, s + 7)})
        g3.append(sd[p + ".norm.g"]); toq.append(sd[p + ".to_q.weight"]); ctxs.append(rnd((Fr, 2 * co), s + 8))
    tok = rnd((Fr, n, ci), 99)
    tabs = [ca_tables(sd, "ca_" + nm, ctxs[a], co) for a, nm in enumerate(names)]
    kq = torch.stack([t[0] for t in tabs], 1)                                                  # (F, 3, 64)
    nkq = torch.stack([t[1] for t in tabs], 0)                                                 # (3, 8)
    G = torch.stack([t[2] for t in tabs], 1)                                                   # (F, 3, 81)
    T = torch.cat([t[3] for t in tabs], 1)                                                     # (F, 27, co)
    gates, _ = R.ca_gates(tok, torch.stack(g3), torch.stack(toq), kq, nkq)
    Wt, _ = R.ca_rstd(gates, G)
    for a, nm in enumerate(names):
        got = Wt[..., 9 * a:9 * (a + 1)] @ T[:, 9 * a:9 * (a + 1)]
        f32 = {k: v.float() for k, v in sd.items() if k.startswith("ca_" + nm)}
        want = O.cross_attention(f32, "ca_" + nm, tok.float(), ctxs[a].float())              # the oracle's softmax is fp32
        close(f"cross attention {nm}", got, want.double(), 1e-5)
