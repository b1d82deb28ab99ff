"""Float64 references of the UNet's per-clip and per-step glue kernels (csrc/kernels.cu), each with an elementwise error bound
built from absolute values of the same data.  tests/test_unet_kernels_gpu.py holds the kernels to them; the error model is in
that file's docstring.  Inputs are the fp32 values the kernel reads, as float64 tensors."""
import math

import numpy as np
import torch

U = 2.0 ** -24
DT = torch.float64


def ulp32(v):
    """one fp32 ulp of |v| (the spacing at v; 2^-149 at zero)"""
    a = v.abs().to(torch.float32).cpu().numpy()
    return torch.from_numpy(np.spacing(a).astype(np.float64)).to(v.device)


def silu(t):
    return t / (1 + torch.exp(-t))


def silu_err(t, dt):
    """|d SiLU| for an input error dt: |SiLU'| <= 1.1, and the fp32 exp, add and divide add 5u of the result"""
    return 1.1 * dt + 5 * U * silu(t).abs()


# ------------------------------------------------------------------------------------------------------------------ norms
def rowstats(x):
    """(mean, rstd) of each row of x (M, C), biased variance, eps 1e-5.  The kernel sums NV float4 per lane, then a 5-step
    butterfly: depth NV + 7."""
    M, C = x.shape
    nv = 8 if C <= 1024 else 16
    mu = x.mean(1)
    var = ((x - mu[:, None]) ** 2).mean(1)
    rstd = 1 / torch.sqrt(var + 1e-5)
    dmu = (nv + 9) * U * x.abs().mean(1) + U * mu.abs()
    # the mean's error only adds dmu^2 to the variance; each centred value and square rounds, the sum adds depth nv + 7
    dvar = (nv + 11) * U * var + dmu ** 2
    drstd = rstd * (0.5 * dvar / (var + 1e-5) + 3 * U)
    return mu, rstd, dmu, drstd


def gn_stats(y, P, clips, cpg, count=None):
    """fp64 (sum, sum of squares) per clip and group of y (M, C): [clips][8][2], with the number of values per group"""
    M, C = y.shape
    clip = (torch.arange(M, device=y.device) // P) % clips
    st = torch.zeros(clips, 8, 2, dtype=DT, device=y.device)
    for b in range(clips):
        yb = y[clip == b].reshape(-1, 8, cpg)
        st[b, :, 0] = yb.sum((0, 2))
        st[b, :, 1] = (yb * yb).sum((0, 2))
    n = (M // (P * clips)) * P * cpg if count is None else count
    return st, float(n)


def gn_apply(y, st, count, P, clips, cpg, w, b, res=None):
    """SiLU((y - mean) rstd w + b) (+ res) with mean / rstd from the fp64 sums as the kernel forms them"""
    M, C = y.shape
    clip = (torch.arange(M, device=y.device) // P) % clips
    mean = st[..., 0] / count
    var = st[..., 1] / count - mean * mean
    rstd = 1 / torch.sqrt(var + 1e-5)
    grp = torch.arange(C, device=y.device) // cpg
    m, r = mean[clip][:, grp], rstd[clip][:, grp]
    t = (y - m) * r * w + b
    o = silu(t)
    # mean and rstd round to fp32 (u each); y - mean, the two products and the add round once each
    dt = r * w.abs() * (U * m.abs() + 5 * U * (y - m).abs()) + 2 * U * (b.abs() + t.abs())
    do = silu_err(t, dt)
    if res is not None:
        o = o + res
        do = do + U * o.abs()
    return o, do


# ------------------------------------------------------------------------------------------------------------------ conditioning tables
def table_rows(F, clips):
    """cond row read by table frame i = f * clips + b: b * (F / clips) + f"""
    i = torch.arange(F)
    return (i % clips) * (F // clips) + i // clips


def cond_mlp(cond, off, K, W, b, F, clips):
    """ctx[i] = b + W SiLU(cond[src(i), off:off+K]) in table order; lane-strided sums of ceil(K/32) terms and a butterfly"""
    x = cond[table_rows(F, clips).to(cond.device), off:off + K]
    s = silu(x)
    out = s @ W.t() + b
    depth = math.ceil(K / 32) + 5
    bound = (depth + 7) * U * (s.abs() @ W.abs().t() + b.abs()) + U * out.abs()
    return out, bound


def cond_kv(ctx, Wkv):
    """kv = ctx Wkv^T (no bias, no activation)"""
    n1 = ctx.shape[1]
    out = ctx @ Wkv.t()
    return out, (math.ceil(n1 / 32) + 7) * U * (ctx.abs() @ Wkv.abs().t())


def normalize8(k, sc):
    """F.normalize over 8 dims (1e-12 clamp) times the folded scale; 8-term sum of squares, sqrt, divide, three products"""
    n = k.norm(dim=-1, keepdim=True)
    out = k / n.clamp(min=1e-12) * sc
    return out, 16 * U * out.abs()


def ca_tables(kv, nkv, qs, ks, Wout, gout):
    """per frame of kv (F, 128): kq (F, 64), nkq (8,), u-vector Gram G (F, 81) and gain-folded T (F, 9, co), with bounds"""
    Fr = kv.shape[0]
    co = Wout.shape[0]
    sc = qs * ks
    kq, dkq = normalize8(kv[:, :64].reshape(Fr, 8, 8), sc)
    nkq, dnkq = normalize8(nkv[0], sc)
    nv = nkv[1]
    Wo = Wout.reshape(co, 8, 8)
    vd = kv[:, 64:].reshape(Fr, 8, 8) - nv                                     # (F, h, d)
    u0 = (Wo @ nv).sum(1)                                                      # (co,)
    uh = torch.einsum("chd,fhd->fhc", Wo, vd)                                  # (F, 8, co)
    u = torch.cat((u0[None, None].expand(Fr, 1, co), uh), 1)                   # (F, 9, co)
    e0 = 66 * U * (Wo.abs() @ nv.abs()).sum(1)
    eh = 10 * U * torch.einsum("chd,fhd->fhc", Wo.abs(), kv[:, 64:].reshape(Fr, 8, 8).abs() + nv.abs())
    eu = torch.cat((e0[None, None].expand(Fr, 1, co), eh), 1)
    mean = u.mean(-1, keepdim=True)
    ut = u - mean
    depth = math.ceil(co / 32) + 5
    eut = eu + eu.mean(-1, keepdim=True) + (depth + 2) * U * u.abs().mean(-1, keepdim=True) + U * ut.abs()
    G = ut @ ut.transpose(1, 2) / co
    a = ut.abs()
    dG = (eut @ a.transpose(1, 2) + a @ eut.transpose(1, 2)) / co + (depth + 2) * U * (a @ a.transpose(1, 2)) / co
    T = ut * gout
    dT = (eut + U * a) * gout.abs() + U * T.abs()
    return (kq.reshape(Fr, 64), dkq.reshape(Fr, 64), nkq, dnkq, G.reshape(Fr, 81), dG.reshape(Fr, 81), T, dT,
            (a @ a.transpose(1, 2)).reshape(Fr, 81) / co)


# ------------------------------------------------------------------------------------------------------------------ time embedding
def sinusoid(t, freqs):
    """(sin, cos) of the fp32 product t * freqs (oracle.unet_oracle.sinusoidal), taken in float64; the bound allows CUDA's
    2-ulp sinf / cosf"""
    a = (t.to(torch.float32)[:, None] * freqs.to(torch.float32)[None, :]).double()
    e = torch.cat((a.sin(), a.cos()), -1)
    return e, 2 * ulp32(e)


def gelu(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def time_mlp(t, freqs, W1, b1, W2, b2):
    """SiLU(W2 GELU(W1 sin|cos + b1) + b2) per clip: sequential sums of dim and 4 dim terms"""
    emb, de = sinusoid(t, freqs)
    dim = emb.shape[1]
    h = emb @ W1.t() + b1
    dh = (dim + 2) * U * (emb.abs() @ W1.abs().t() + b1.abs()) + de @ W1.abs().t()
    g = gelu(h)
    dg = 1.13 * dh + 8 * U * h.abs()                                          # |GELU'| <= 1.13; erff 2 ulp, three roundings
    o = g @ W2.t() + b2
    do = (4 * dim + 2) * U * (g.abs() @ W2.abs().t() + b2.abs()) + dg @ W2.abs().t()
    return silu(o), silu_err(o, do)


def film(ts, W, b):
    """out[clip] = W ts[clip] + b, lane-strided sums of ceil(tdim/32) terms"""
    out = ts @ W.t() + b
    depth = math.ceil(ts.shape[1] / 32) + 5
    return out, (depth + 2) * U * (ts.abs() @ W.abs().t() + b.abs())


def rotary_table(freqs, F, pos0):
    """(F, 16, 2) cos / sin of the fp32 product (pos0 + f) * freqs[i]"""
    pos = torch.arange(pos0, pos0 + F, dtype=torch.float32)
    a = (pos[:, None] * freqs.to(torch.float32).cpu()[None, :]).double()
    out = torch.stack((a.cos(), a.sin()), -1)
    return out, 2 * ulp32(out)


# ------------------------------------------------------------------------------------------------------------------ fp16 split
def split_f16x2_rn(x):
    """numpy restatement of split_f16x2_rn (csrc/f16x3.cuh) on fp32 values: hi keeps 11 significant bits (round half up on the
    bit pattern), lo = fp16(x - hi); returns the fp16 bit patterns as uint16"""
    x = np.ascontiguousarray(x, dtype=np.float32)
    hb = ((x.view(np.uint32).astype(np.uint64) + 0x1000) & 0xFFFFE000).astype(np.uint32)
    h = hb.view(np.float32)
    with np.errstate(over="ignore"):                                         # beyond fp16's range both kernels give inf
        lo = (x - h).astype(np.float16)
        return h.astype(np.float16).view(np.uint16), lo.view(np.uint16)


# ------------------------------------------------------------------------------------------------------------------ layout / init conv / heads
def ncf_to_nhwc(x, clips, C, F, HW, Cpad, c0):
    """x (clips, C, F, HW) -> (F * clips, HW, Cpad) at channel c0, other channels zero"""
    out = torch.zeros(F * clips, HW, Cpad, dtype=x.dtype, device=x.device)
    xv = x.reshape(clips, C, F, HW).permute(2, 0, 3, 1).reshape(F * clips, HW, C)
    out[:, :, c0:c0 + C] = xv
    return out


def fea_shift(fr, k, Cpad, c0):
    """fr (clips, C, H, W) -> (k * clips, H * W, Cpad): copy s of clip b = the frame shifted by s - k // 2 rows, zero outside"""
    clips, C, H, W = fr.shape
    out = torch.zeros(k * clips, H * W, Cpad, dtype=fr.dtype, device=fr.device)
    for s in range(k):
        d = s - k // 2
        sh = torch.zeros_like(fr)
        if d >= 0:
            sh[:, :, :H - d] = fr[:, :, d:]
        else:
            sh[:, :, -d:] = fr[:, :, :H + d]
        out[s * clips:(s + 1) * clips, :, c0:c0 + C] = sh.permute(0, 2, 3, 1).reshape(clips, H * W, C)
    return out


def frame_invariance(x, c0):
    """x (clips, C, F, HW): per clip, whether any bit of channels [c0, C) differs from frame 0"""
    xb = x[:, c0:].contiguous().view(torch.int32)
    return [bool((xb[b] != xb[b, :, :1]).any()) for b in range(x.shape[0])]


def map_reduce_f32(part, bias, Co):
    """bias[i % Co] + part[0][i] + part[1][i] + ... in fp32, in that order (bit-exact restatement)"""
    p = part.to(torch.float32)
    n = p.shape[1]
    acc = bias.to(torch.float32).repeat(n // Co) if bias is not None else torch.zeros(n, dtype=torch.float32, device=p.device)
    for s in range(p.shape[0]):
        acc = acc + p[s]
    return acc


def init_conv_x3(xt, w3, mp, k):
    """xt (clips, 3, F, H, W), w3 (k*k*3, Co), mp (clips, H, W, Co) -> (F * clips, H * W, Co) = map + k x k conv (zero padding)"""
    clips, _, F, H, W = xt.shape
    Co = w3.shape[1]
    w = w3.reshape(k, k, 3, Co).permute(3, 2, 0, 1)                            # (Co, 3, k, k)
    x = xt.permute(2, 0, 1, 3, 4).reshape(F * clips, 3, H, W)                  # frame f of clip b at f * clips + b
    conv = torch.nn.functional.conv2d(x, w, padding=k // 2)
    cabs = torch.nn.functional.conv2d(x.abs(), w.abs(), padding=k // 2)
    m = mp.permute(0, 3, 1, 2).repeat(F, 1, 1, 1)                              # (F * clips, Co, H, W)
    out = (conv + m).permute(0, 2, 3, 1).reshape(F * clips, H * W, Co)
    bound = ((3 * k * k + 2) * U * (cabs + m.abs())).permute(0, 2, 3, 1).reshape(F * clips, H * W, Co)
    return out, bound


def heads_out(hf, ho, clips, HW, Wf, bf, Wo, bo):
    """rows m = (f * clips + b) * HW + p -> out (clips, ng + nc, F, HW)"""
    M, C = hf.shape
    Fc = M // (HW * clips)
    o = torch.cat((hf @ Wf.t() + bf, ho @ Wo.t() + bo), 1)                    # (M, ng + nc)
    a = torch.cat((hf.abs() @ Wf.abs().t() + bf.abs(), ho.abs() @ Wo.abs().t() + bo.abs()), 1)
    lay = lambda t: t.reshape(Fc, clips, HW, -1).permute(1, 3, 0, 2).contiguous()
    return lay(o), lay((C // 4 + 6) * U * a)
