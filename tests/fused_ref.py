"""Float64 references of the fused attention and cross-attention kernels (csrc/temporal_fused.cu, attn_tc.cu, sla_fused.cu,
ca_fused.cu and their SIMT counterparts in kernels.cu), each written from the operation, with the elementwise error bound of the
kernel's arithmetic computed from absolute values of the same data.  The derivation is in tests/test_fused_gpu.py.
Device-agnostic: the CPU tests tie these references to the oracle, the GPU tests hold the kernels to them."""
import torch

U = 2.0 ** -24
TINY = 2.0 ** -25                          # absolute error of an fp16 lo piece in the subnormal range
SPLIT_RR = 3 * 2.0 ** -22                  # both operands split with a round-to-nearest hi (attn_tc.cu)
SPLIT_TR = 5 * 2.0 ** -22                  # truncated-hi activation x round-to-nearest weight image
SPLIT_TT = 8 * 2.0 ** -22                  # both operands split with a truncated hi
EXP2 = 2.0 ** -21                          # relative error of ex2.approx / __expf, as an absolute score error
LOG2E = 1.4426950408889634


def _d(t):
    return t.double()


def layernorm(x, g=None, eps=1e-5):
    """over the last dim, biased variance, gain only; returns (xhat * g, mean, rstd)"""
    mu = x.mean(-1, keepdim=True)
    rs = ((x - mu).pow(2).mean(-1, keepdim=True) + eps).rsqrt()
    y = (x - mu) * rs
    return (y * g if g is not None else y), mu, rs


def rotary(t, rot):
    """interleaved pairs (2i, 2i+1) rotated by rot[f, i] = (cos, sin); t (..., F, 2n), rot (F, n, 2)"""
    c, s = rot[..., 0], rot[..., 1]
    a, b = t[..., 0::2], t[..., 1::2]
    return torch.stack((a * c - b * s, b * c + a * s), -1).flatten(-2)


def rotary_err(E, y):
    """bound after the rotation of a pair whose parts carry errors E (and the rotation's own rounding)"""
    a = E[..., 0::2] + E[..., 1::2] + 2 * U * (y[..., 0::2].abs() + y[..., 1::2].abs())
    return torch.stack((a, a), -1).flatten(-2)


def attention(q, k, v, qpos, band, bias, c_qk, c_pv, Eq=None, Ek=None, Ev=None, e_exp=EXP2, bias_round=0.0, full=False):
    """softmax attention of queries at key positions qpos (|key - query| <= band unless band is None) with bias[h, rel + band],
    rel = key - query (full: every key attends, the bias still indexed rel + band).  q (B, H, Lq, d), k, v (B, H, Lk, d).
    Returns (o, bound).
    Score error  ds_ij = c_qk sum_d |q_d||k_d| + TINY (|q|_1 + |k|_1) + e_exp + 4u (|s_ij| + |m_i|) (+ propagated q, k errors);
    output error |do_i| <= max_j ds_ij * sum_j p_ij (|v_j| + |o_i|) + c_pv sum_j p_ij |v_j| + TINY (sum_j |v_j| / l_i + 1)
                           + (n_i + 8) u |o_i| (+ sum_j p_ij Ev_j)."""
    Lk = k.shape[-2]
    kpos = torch.arange(Lk, device=q.device)
    rel = kpos[None, :] - qpos[:, None]
    mask = torch.ones_like(rel, dtype=torch.bool) if full else rel.abs() <= band
    s = q @ k.transpose(-1, -2)
    bterm = 0.0
    if bias is not None:
        bmat = bias[:, (rel + band).clamp(0, bias.shape[1] - 1)]            # (H, Lq, Lk)
        s = s + bmat
        bterm = bias_round * bmat.abs()
    s = s.masked_fill(~mask, float("-inf"))
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    p = e / l
    o = p @ v
    aq, ak, av = q.abs(), k.abs(), v.abs()
    ds = c_qk * (aq @ ak.transpose(-1, -2)) + TINY * (aq.sum(-1, keepdim=True) + ak.sum(-1).unsqueeze(-2)) + e_exp
    ds = ds + 4 * U * (s.masked_fill(~mask, 0).abs() + m.abs()) + bterm
    if Eq is not None:
        ds = ds + Eq @ ak.transpose(-1, -2) + aq @ Ek.transpose(-1, -2) + Eq @ Ek.transpose(-1, -2)
    dsmax = ds.masked_fill(~mask, 0).amax(-1, keepdim=True)
    pv = p @ av
    n = mask.sum(-1, keepdim=True).double()
    bound = dsmax * (pv + o.abs()) + c_pv * pv + TINY * ((mask.double() @ av) / l + 1) + (n + 8) * U * o.abs()
    if Ev is not None:
        bound = bound + p @ Ev
    return o, bound


def projection_raw_split(x, Wf, wsum_abs):
    """y = LN(x) @ Wf^T with Wf gamma-folded, as the temporal kernel computes it: the raw row x is split, LayerNorm applied after
    the contraction (y = rstd (x @ Wf^T - mu wsum)).  Returns (y, bound), K = 64."""
    K = x.shape[-1]
    xh, mu, rs = layernorm(x)
    y = xh @ Wf.t()
    c1 = SPLIT_TR + K * 2.0 ** -23 + 8 * U
    ax = x.abs()
    S = ax @ Wf.abs().t()
    dmu = (K / 8 + 5) * U * ax.mean(-1, keepdim=True)
    bound = rs * (c1 * S + TINY * ax.sum(-1, keepdim=True) + dmu * wsum_abs) + (K / 8 + 6) * U * y.abs()
    return y, bound


def projection_ln_split(x, Wf):
    """y = LN(x) @ Wf^T with the normalised row split (sla_fused.cu, ca_fused.cu).  Returns (y, bound)."""
    K = x.shape[-1]
    xh, mu, rs = layernorm(x)
    y = xh @ Wf.t()
    c1 = SPLIT_TR + K * 2.0 ** -23 + 8 * U + (K / 8 + 6) * U
    dmu = (K / 8 + 3) * U * x.abs().mean(-1, keepdim=True)
    aW = Wf.abs()
    bound = c1 * (xh.abs() @ aW.t()) + TINY * xh.abs().sum(-1, keepdim=True) + rs * dmu * aW.sum(1)
    return y, bound


def temporal(x, res, gamma, wqkv, wout, rot, bias, band, q_lo, q_hi):
    """Residual(PreNorm(temporal attention)) of one pixel batch.  x (B, Fe, 64) on-chip sequence, res (B, q_hi - q_lo, 64).
    Returns (out, bound, y) with y = out - res."""
    x, res, gamma, wqkv, wout, rot, bias = map(_d, (x, res, gamma, wqkv, wout, rot, bias))
    Wf = wqkv * gamma[None, :]
    Wf[:256] *= 32 ** -0.5
    wsum = Wf.sum(1).abs()
    y, E = projection_raw_split(x, Wf, wsum)                               # (B, Fe, 768)
    B, Fe, _ = x.shape
    heads = lambda t: t.reshape(B, Fe, 8, 32).transpose(1, 2)             # (B, 8, Fe, 32)
    q, k, v = (heads(y[..., i * 256:(i + 1) * 256]) for i in range(3))
    Eq, Ek, Ev = (heads(E[..., i * 256:(i + 1) * 256]) for i in range(3))
    Eq, Ek = rotary_err(Eq, q), rotary_err(Ek, k)
    q, k = rotary(q, rot), rotary(k, rot)
    q, Eq = q[:, :, q_lo:q_hi], Eq[:, :, q_lo:q_hi]
    Eq = Eq + U * q.abs()                                                  # the scale to the log2 domain
    nk = min(Fe, 2 * band + 1)
    o, Eo = attention(q, k, v, torch.arange(q_lo, q_hi, device=x.device), band, bias,
                      SPLIT_TT + 32 * 2.0 ** -23 + 5 * U, SPLIT_TT + 32 * 2.0 ** -23 + (nk / 16 + 6) * U,
                      Eq, Ek, Ev, bias_round=2 * U)
    o = o.transpose(1, 2).reshape(B, q_hi - q_lo, 256)
    Eo = Eo.transpose(1, 2).reshape(B, q_hi - q_lo, 256)
    aW = wout.abs()
    yo = o @ wout.t()
    Ey = Eo @ aW.t() + (SPLIT_TR + 32 * 2.0 ** -23 + 10 * U) * (o.abs() @ aW.t()) + TINY * aW.sum(1)
    out = res + yo
    return out, Ey + U * out.abs(), yo


def sla_ctx(x, gamma, wqkv, wout):
    """Bf[f][h*32 + d][c] = sum_e softmax_px(k)[d] v[e] wout[c][h*32 + e] of (F, P, 64) rows x.  Returns (Bf (F, 256, C), bound)."""
    x, gamma, wqkv, wout = map(_d, (x, gamma, wqkv, wout))
    Fr, P, _ = x.shape
    Wf = wqkv * gamma[None, :]
    kv, E = projection_ln_split(x, Wf[256:])                               # (F, P, 512)
    hd = lambda t: t.reshape(Fr, P, 8, 32).permute(0, 2, 3, 1)            # (F, 8, 32, P)
    k, v, Ek, Ev = hd(kv[..., :256]), hd(kv[..., 256:]), hd(E[..., :256]), hd(E[..., 256:])
    m = k.amax(-1, keepdim=True)
    p = torch.exp(k - m)
    l = p.sum(-1, keepdim=True)
    p = p / l
    ctx = p @ v.transpose(-1, -2)                                          # (F, 8, d, e)
    ds = (Ek + EXP2 + 4 * U * (k.abs() + m.abs())).amax(-1, keepdim=True)
    pv = p @ v.abs().transpose(-1, -2)
    n = P / 16 + 48
    dctx = ds * (pv + ctx.abs()) + p @ Ev.transpose(-1, -2) + (SPLIT_TT + 16 * 2.0 ** -23 + 4 * U) * pv \
        + TINY * (v.abs().sum(-1).unsqueeze(-2) / l + 1) + n * U * ctx.abs()
    W = wout.t().reshape(8, 32, -1)                                        # (h, e, C)
    Bf = (ctx @ W).reshape(Fr, 256, -1)
    aW = W.abs()
    bound = (dctx @ aW + 34 * U * (ctx.abs() @ aW)).reshape(Fr, 256, -1)
    return Bf, bound


def sla_out(x, gamma, wqkv, Bf, bias):
    """out = x + bias + sum_h softmax_d(q_h) 32^-1/2 Bf[f][h]; x (F, P, 64), Bf (F, 256, 64).  Returns (out, bound)."""
    x, gamma, wqkv, Bf, bias = map(_d, (x, gamma, wqkv, Bf, bias))
    Fr, P, _ = x.shape
    q, Eq = projection_ln_split(x, wqkv[:256] * gamma[None, :])
    q, Eq = q.reshape(Fr, P, 8, 32).transpose(1, 2), Eq.reshape(Fr, P, 8, 32).transpose(1, 2)    # (F, 8, P, 32)
    p = torch.softmax(q, -1) * 32 ** -0.5
    Bh = Bf.reshape(Fr, 8, 32, -1)
    yh = p @ Bh                                                            # (F, 8, P, C)
    pB = p @ Bh.abs()
    dq = (Eq + EXP2 + 4 * U * (q.abs() + q.amax(-1, keepdim=True).abs())).amax(-1, keepdim=True)
    bound_h = dq * (pB + yh.abs()) + (SPLIT_TT + 32 * 2.0 ** -23 + 40 * U) * pB + TINY * (Bh.abs().sum(-2, keepdim=True) + 1)
    y = yh.sum(1)
    out = x + bias + y
    return out, bound_h.sum(1) + 8 * U * pB.sum(1) + 2 * U * (x + bias).abs() + 2 * U * out.abs()


def ca_gates(x, g3, toq3, kq, nkq):
    """gates (F, P, 3, 8) of the three cross-attentions: the frame key's weight in the softmax over {null key, frame key} of
    8 * normalize(q_h) . key, q = LayerNorm_img(x) @ to_q^T.  kq (F, 3, 64) and nkq (3, 8) carry the q/k scales.
    Returns (gates, bound)."""
    x, g3, toq3, kq, nkq = map(_d, (x, g3, toq3, kq, nkq))
    Fr, P, ci = x.shape
    gs, bs = [], []
    for a in range(3):
        q, Eq = projection_ln_split(x, toq3[a] * g3[a][None, :])
        q, Eq = q.reshape(Fr, P, 8, 8), Eq.reshape(Fr, P, 8, 8)
        k = kq[:, a].reshape(Fr, 1, 8, 8)
        nk = nkq[a].reshape(1, 1, 1, 8)
        nrm = q.norm(dim=-1).clamp_min(1e-12)
        z = 8 * (q * (k - nk)).sum(-1) / nrm
        g = torch.sigmoid(z)
        an = q.abs()
        dz = 8 / nrm * ((Eq * (k - nk).abs()).sum(-1) + (q * (k - nk)).sum(-1).abs() / nrm ** 2 * (an * Eq).sum(-1)
                        + 16 * U * (an * (k.abs() + nk.abs())).sum(-1)) + 4 * U * z.abs()
        gs.append(g)
        bs.append(g * (1 - g) * dz + EXP2)
    return torch.stack(gs, 2), torch.stack(bs, 2)


def ca_rstd(gates, G, dg=None):
    """Wt (M, 32): per cross-attention a, rs * [1, gates_a] with rs = (c^T G_a c + 1e-5)^-1/2, c = [1, gates_a]; columns 27-31
    are zero.  gates (F, P, 3, 8), G (F, 3, 81); dg the gates' own error bound.  Returns (Wt, bound)."""
    gates, G = _d(gates), _d(G)
    Fr, P = gates.shape[:2]
    c = torch.cat((torch.ones_like(gates[..., :1]), gates), -1)           # (F, P, 3, 9)
    Gm = G.reshape(Fr, 1, 3, 9, 9)
    var = torch.einsum("fpai,fpaij,fpaj->fpa", c, Gm.expand(Fr, P, 3, 9, 9), c)
    rs = (var.clamp_min(0) + 1e-5).rsqrt()
    Wt = torch.zeros(Fr, P, 32, dtype=torch.float64, device=gates.device)
    Wt[..., :27] = (rs[..., None] * c).reshape(Fr, P, 27)
    ac, aG = c.abs(), Gm.abs().expand(Fr, P, 3, 9, 9)
    dc = torch.zeros_like(c) if dg is None else torch.cat((torch.zeros_like(dg[..., :1]), dg), -1)
    q = lambda l, r: torch.einsum("fpai,fpaij,fpaj->fpa", l, aG, r)
    dvar = q(ac, dc) + q(dc, ac) + q(dc, dc) + 20 * U * q(ac, ac)         # Gram-form variance relative to sum |c_a c_b G_ab|
    drs = 0.5 * rs ** 3 * dvar + 3 * U * rs
    b = torch.zeros_like(Wt)
    b[..., :27] = (drs[..., None] * ac + rs[..., None] * dc + U * (rs[..., None] * ac)).reshape(Fr, P, 27)
    return Wt, b


def gn_hcond(Y, stats, count, cpg, w, b, film, Wt, T):
    """out = SiLU(FiLM(GroupNorm(Y))) + Wt_f @ T_f, GroupNorm from the given (sum, sum of squares) per group.
    Y (F, P, co), Wt (F, P, 32), T (F, 32, co).  Returns (out, bound)."""
    Y, stats, w, b, Wt, T = map(_d, (Y, stats, w, b, Wt, T))
    co = Y.shape[-1]
    grp = torch.arange(co, device=Y.device) // cpg
    mean = stats[0::2][grp] / count
    var = stats[1::2][grp] / count - mean * mean
    rstd = (var + 1e-5).rsqrt()
    al, be = rstd * w, b - mean * rstd * w
    aal, abe = al.abs(), b.abs() + (mean * al).abs()
    if film is not None:
        sc, sh = _d(film[:co]) + 1, _d(film[co:])
        al, be = al * sc, be * sc + sh
        aal, abe = aal * sc.abs(), abe * sc.abs() + sh.abs()
    t = Y * al + be
    dt = 6 * U * (Y.abs() * aal + abe)
    silu = t * torch.sigmoid(t)
    dsilu = 1.1 * dt + 4 * U * silu.abs() + TINY
    h = Wt @ T
    aWt, aT = Wt.abs(), T.abs()
    dh = (SPLIT_TT + 32 * 2.0 ** -23 + 4 * U) * (aWt @ aT) + TINY * (aT.sum(-2, keepdim=True) + aWt.sum(-1, keepdim=True))
    out = silu + h
    return out, dsilu + dh + 2 * U * out.abs()
