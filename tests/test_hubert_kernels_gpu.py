"""GPU: each HuBERT kernel entry (include/dawn_hubert.h, dawn_hubert_test_kernel) against the same operation in float64, at the
shapes, strides and edges the network reaches: every entry runs the network's own packing and launch code on caller buffers.

* attention: hubert-large's 16 heads, 3 sequences, an output row wider than 64 H whose padding must keep its sentinel, and a
  sharp softmax (scores from -30 to +45) whose maximum key sits in the last key block, so the online rescale has to reach
  both the output and the row sum; T in {1, 65, 999, 1000};
* conv0 (feature-extractor layer 0): more than 132 * 16 * 8 = 16 896 rows, so the grid-stride row loop runs; k = 64 and other
  strides; C = 2048;
* the row LayerNorm (+ GELU) pass: C in {64, 512, 1024, 2048}, in place and out of place, strides wider than C, eps 1e-5 and
  1e-6, more than 16 896 rows, and rows whose mean is 30-300x their standard deviation (a one-pass variance fails there);
* a feature-extractor conv >= 1 (stride-2 k3 / k2 contraction, then LayerNorm + GELU), with and without the conv bias, on both
  sides of the dispatcher's 128-row line;
* a pre-LN projection through the commit-time fold, the row statistics and the dispatcher: q|k|v (three parts, q times 1/8)
  and fc1 (GELU), on both sides of 128 rows;
* the positional conv with B = 2 and 3 sequences of different content and k in {31, 127, 128}: each sequence's output equals
  that sequence run alone, bit for bit.

Error bounds are propagated from the fp32 unit roundoff u = 2^-24 through each kernel's own order of operations (see each
helper); every case also meets the north-star tolerance 1e-4 + 1e-3 |ref| (the pre-LN projection on its rows within 10
standard deviations of zero mean, see test_contraction_gpu.run_ln_bias) and prints its margins.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as Fn

from dawn_pytorch_b200._lib import (HUBERT_ATTENTION, HUBERT_CONV0, HUBERT_FE_CONV, HUBERT_LN_LINEAR, HUBERT_POS_CONV,
                                    HUBERT_ROW_LN)
from tests.test_contraction_gpu import c1_tau, ln_fold_bound, tiny_of

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
DEV = "cuda"
SENT = 1234.5
GUARD = 64
GELU_SLOPE = 1.13


def gen(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def big_mean_rows(M, C, seed):
    """normal rows; every 7th row is shifted by 30-300 standard deviations"""
    x = gen((M, C), seed)
    g = torch.Generator().manual_seed(seed + 1)
    shift = (30 + 270 * torch.rand(M, generator=g)).to(DEV)
    sel = torch.arange(M, device=DEV) % 7 == 3
    x[sel] += shift[sel, None]
    return x


def run(**kw):
    from dawn_pytorch_b200 import _lib
    c = _lib.DawnHubertKernelCase()
    for k, v in kw.items():
        setattr(c, k, ctypes.c_void_p(v.data_ptr()) if torch.is_tensor(v) else v)
    torch.cuda.synchronize()
    _lib.check(_lib.lib.dawn_hubert_test_kernel(ctypes.byref(c), _lib.stream()), "dawn_hubert_test_kernel")
    torch.cuda.synchronize()


def guarded(rows, ld):
    """a [GUARD + rows + GUARD][ld] sentinel buffer and its body view"""
    buf = torch.full((GUARD + rows + GUARD, ld), SENT, device=DEV)
    return buf, buf[GUARD:GUARD + rows]


def check_guarded(buf, rows, C):
    assert torch.all(buf[:GUARD] == SENT) and torch.all(buf[GUARD + rows:] == SENT), "store outside the output rows"
    assert torch.all(buf[GUARD:GUARD + rows, C:] == SENT), "store into the row padding"
    return buf[GUARD:GUARD + rows, :C]


def report(name, out, ref, bound, ns_rows=None):
    """elementwise |d| <= bound; north-star on ns_rows (bool mask, default all; the other rows' figure is printed only)"""
    out = out.double()
    assert torch.isfinite(out).all(), f"{name}: non-finite output"
    d = (out - ref).abs()
    el = (d / bound).max().item()
    nsr = d / (1e-4 + 1e-3 * ref.abs())
    ns = (nsr if ns_rows is None else nsr[ns_rows]).max().item()
    other = f" (other rows {nsr[~ns_rows].max().item():.3f}, not held)" if ns_rows is not None and (~ns_rows).any() else ""
    print(f"  {name}: elementwise max |d|/bound = {el:.3f}; north-star max |d|/tol = {ns:.3f}{other}")
    assert el <= 1.0, f"{name}: error {el:.2f}x the bound"
    assert ns <= 1.0, f"{name}: {ns:.2f}x the north-star tolerance"


def ln_bound(y, e_y, g, be, eps, gelu):
    """float64 LayerNorm(y) * g + be (then erf GELU) and the bound of ln_row_warp on fp32 rows known within e_y: lane sums of
    C / 64 pairs and a 5-level warp tree (mean, then centred squares), rstd = 1 / sqrtf(var + eps), (y - mu) rstd g + be"""
    C = y.shape[-1]
    depth = (C / 32 + 8) * U                                    # summation error of one row, relative to the sum of |terms|
    mu = y.mean(-1, keepdim=True)
    d = y - mu
    var = d.pow(2).mean(-1, keepdim=True)
    rstd = (var + eps).rsqrt()
    n = d * rstd
    e_mu = e_y.amax(-1, keepdim=True) + depth * y.abs().mean(-1, keepdim=True) + U * mu.abs()
    e_d = e_y + e_mu + U * d.abs()
    r = (d.abs() * e_d).sum(-1, keepdim=True) / (C * var) + depth + 3 * U      # relative error of rstd
    e_n = rstd * e_d + n.abs() * (r + 2 * U)
    g, be = g.double(), be.double()
    pre = n * g + be
    e_pre = g.abs() * e_n + 2 * U * pre.abs()
    if not gelu:
        return pre, e_pre + U * pre.abs()
    ref = Fn.gelu(pre)
    return ref, GELU_SLOPE * e_pre + 4 * U * (ref.abs() + 1)


# ------------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("T", [1, 65, 999, 1000])
def test_attention_large_heads_wide_rows_sharp_softmax(T):
    B, H = 3, 16
    D = 64 * H
    ld, ldo = 3 * D + 4, D + 8
    seed = 6000 + T
    qkv = torch.zeros(B * T, ld, device=DEV)
    qkv[:, :3 * D] = gen((B * T, 3 * D), seed, 0.3)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D]
    g = torch.Generator().manual_seed(seed + 1)
    for h in range(H):                                          # score ~ k[j, 64 h]: -30 .. 30, the last key of each sequence 45
        q[:, 64 * h] = 1.0
        k[:, 64 * h] = (60 * torch.rand(B * T, generator=g) - 30).to(DEV)
        k[T - 1::T, 64 * h] = 45.0
    buf, _ = guarded(B * T, ldo)
    run(kernel=HUBERT_ATTENTION, B=B, T=T, H=H, ld=ld, ldo=ldo, q=q, kk=k, v=v, out=buf[GUARD:])
    out = check_guarded(buf, B * T, D)
    heads = lambda t: t.double().reshape(B, T, H, 64).transpose(1, 2)  # noqa: E731
    qd, kd, vd = heads(q), heads(k), heads(v)
    ref = (torch.softmax(qd @ kd.transpose(-1, -2), -1) @ vd).transpose(1, 2).reshape(B * T, D)
    # as test_hubert_gpu.test_attention_kernel_matches_float64: FP16x3 products within 2^-21 relative, the softmax doubling the
    # score error, fp32 sums of 64 + T terms; S = max_ij sum_d |q_id k_jd|
    S = (qd.abs() @ kd.abs().transpose(-1, -2)).amax(-1).transpose(1, 2).reshape(B * T, H).repeat_interleave(64, 1)
    bound = 2 * (2.0 ** -20 * S + 2.0 ** -21 + (64 + T) * U) * vd.abs().max().item()
    report(f"attention B={B} H={H} T={T}", out, ref, bound)


# ------------------------------------------------------------------------------------------------ conv0
@pytest.mark.parametrize("B,T,C,k,s", [(2, 9000, 512, 10, 5), (1, 17000, 64, 64, 3), (2, 300, 2048, 64, 7), (3, 6000, 1024, 10, 5)])
def test_conv0_row_loop_wide_kernels(B, T, C, k, s):
    L = (T - 1) * s + k + 2
    seed = 6100 + B + T + C + k
    x = gen((B, L), seed, 0.5)
    w, b = gen((C, 1, k), seed + 1, 1 / math.sqrt(k)), gen((C,), seed + 2, 0.05)
    gam, be = 1 + gen((C,), seed + 3, 0.2), gen((C,), seed + 4, 0.05)
    out = torch.full((B * T, C), float("nan"), device=DEV)
    run(kernel=HUBERT_CONV0, B=B, L=L, C=C, k=k, s=s, eps=1e-5, x=x, w=w, bias=b, gamma=gam, beta=be, out=out)
    y = Fn.conv1d(x.double()[:, None], w.double(), b.double(), stride=s).transpose(1, 2).reshape(B * T, C)
    mag = Fn.conv1d(x.double().abs()[:, None], w.double().abs(), b.double().abs(), stride=s).transpose(1, 2).reshape(B * T, C)
    ref, bound = ln_bound(y, (k + 1) * U * mag, gam, be, 1e-5, True)       # k fused multiply-adds onto the bias
    report(f"conv0 B={B} T={T} C={C} k={k} s={s}", out, ref, bound)


# ------------------------------------------------------------------------------------------------ row LayerNorm
ROW_LN_CASES = [  # M, C, gelu, in place, ld, ldo, eps
    (20000, 64, 1, True, 64, 64, 1e-5), (17000, 512, 1, True, 512, 512, 1e-5), (16897, 512, 0, True, 520, 520, 1e-6),
    (17000, 1024, 0, False, 1040, 1032, 1e-5), (17001, 2048, 0, False, 2112, 2050, 1e-6), (300, 1024, 1, False, 1024, 1088, 1e-6),
    (999, 2048, 1, False, 2048, 2048, 1e-5),
]


@pytest.mark.parametrize("M,C,gelu,inplace,ld,ldo,eps", ROW_LN_CASES,
                         ids=[f"m{c[0]}-c{c[1]}-{'gelu' if c[2] else 'ln'}-{'inplace' if c[3] else 'out'}-ld{c[4]}-ldo{c[5]}-eps{c[6]:g}"
                              for c in ROW_LN_CASES])
def test_row_layernorm(M, C, gelu, inplace, ld, ldo, eps):
    seed = 6200 + M + C + gelu
    x = big_mean_rows(M, C, seed)
    gam, be = 1 + gen((C,), seed + 2, 0.2), gen((C,), seed + 3, 0.05)
    xbuf = torch.full((M, ld), float("nan"), device=DEV)
    xbuf[:, :C] = x
    if inplace:
        buf = None
        run(kernel=HUBERT_ROW_LN, M=M, C=C, ld=ld, ldo=ld, gelu=gelu, eps=eps, x=xbuf, gamma=gam, beta=be, out=xbuf)
        assert torch.isnan(xbuf[:, C:]).all(), "store into the row padding"
        out = xbuf[:, :C]
    else:
        buf, _ = guarded(M, ldo)
        run(kernel=HUBERT_ROW_LN, M=M, C=C, ld=ld, ldo=ldo, gelu=gelu, eps=eps, x=xbuf, gamma=gam, beta=be, out=buf[GUARD:])
        out = check_guarded(buf, M, C)
    ref, bound = ln_bound(x.double(), torch.zeros(M, C, dtype=torch.float64, device=DEV), gam, be, eps, gelu)
    report(f"row LN M={M} C={C} gelu={gelu} {'in place' if inplace else 'out of place'} eps={eps:g}", out, ref, bound)


# ------------------------------------------------------------------------------------------------ feature-extractor conv
FE_CASES = [  # B, L, C, N, k, bias: output rows on both sides of 128
    (2, 3199, 512, 512, 3, True), (3, 49, 512, 512, 3, True), (4, 1599, 512, 512, 2, True), (3, 1599, 384, 384, 2, False),
    (1, 101, 512, 512, 2, False), (2, 257, 512, 1024, 3, True),
]


@pytest.mark.parametrize("B,L,C,N,k,bias", FE_CASES, ids=[f"b{c[0]}-l{c[1]}-{c[2]}-{c[3]}-k{c[4]}-{'bias' if c[5] else 'nobias'}"
                                                            for c in FE_CASES])
def test_feature_extractor_conv(B, L, C, N, k, bias):
    s = 2
    T = (L - k) // s + 1
    M = B * T
    seed = 6300 + B + L + C + N + k
    x = gen((B, L, C), seed)
    w = gen((N, C, k), seed + 1, 1 / math.sqrt(C * k))
    b = gen((N,), seed + 2, 0.05) if bias else None
    gam, be = 1 + gen((N,), seed + 3, 0.2), gen((N,), seed + 4, 0.05)
    out = torch.full((M, N), float("nan"), device=DEV)
    run(kernel=HUBERT_FE_CONV, B=B, L=L, C=C, N=N, k=k, s=s, x=x, w=w, bias=b if bias else None, gamma=gam, beta=be, out=out)
    xt = x.double().transpose(1, 2)
    y = Fn.conv1d(xt, w.double(), b.double() if bias else None, stride=s).transpose(1, 2).reshape(M, N)
    S = Fn.conv1d(xt.abs(), w.double().abs(), b.double().abs() if bias else None, stride=s).transpose(1, 2).reshape(M, N)
    c1, _ = c1_tau("tc" if M >= 128 else "mma", k * C, C, 0)                  # the dispatcher's path
    B2d = w.permute(2, 1, 0).reshape(k * C, N)
    e_y = c1 * S + 8 * U * y.abs() + tiny_of(x, B2d, C)
    ref, bound = ln_bound(y, e_y, gam, be, 1e-5, True)
    report(f"fe conv B={B} L={L} {C}->{N} k={k} bias={bias} M={M}", out, ref, bound)


# ------------------------------------------------------------------------------------------------ pre-LN projections
LN_LINEAR_CASES = [  # M, C, N per part, parts, qscale, gelu, eps
    (100, 1024, 1024, 3, 0.125, 0, 1e-5), (1999, 1024, 1024, 3, 0.125, 0, 1e-5), (100, 1024, 4096, 1, 1.0, 1, 1e-5),
    (1999, 1024, 4096, 1, 1.0, 1, 1e-5), (77, 384, 512, 1, 1.0, 0, 1e-6), (333, 512, 512, 3, 0.125, 0, 1e-6),
]


@pytest.mark.parametrize("M,C,N,parts,qscale,gelu,eps", LN_LINEAR_CASES,
                         ids=[f"m{c[0]}-{c[1]}-{c[3]}x{c[2]}-{'gelu' if c[5] else 'lin'}-eps{c[6]:g}" for c in LN_LINEAR_CASES])
def test_ln_linear(M, C, N, parts, qscale, gelu, eps):
    seed = 6400 + M + C + N + parts
    x = big_mean_rows(M, C, seed)
    NT = parts * N
    w, b = gen((NT, C), seed + 1, 1 / math.sqrt(C)), gen((NT,), seed + 2, 0.05)
    gam, be = 1 + gen((C,), seed + 3, 0.2), gen((C,), seed + 4, 0.05)
    out = torch.full((M, NT), float("nan"), device=DEV)
    run(kernel=HUBERT_LN_LINEAR, M=M, C=C, N=N, parts=parts, qscale=qscale, gelu=gelu, eps=eps, x=x, w=w, bias=b, gamma=gam,
        beta=be, out=out)
    xd = x.double()
    sc = torch.ones(NT, dtype=torch.float64, device=DEV)
    sc[:N] = qscale
    Wf = (w.double() * gam.double()).t() * sc                     # the fold W' = W diag(gamma), per-part scale: (C, NT)
    bf = (b.double() + w.double() @ be.double()) * sc
    mu, var = xd.mean(1), xd.var(1, unbiased=False)
    rs = 1.0 / torch.sqrt(var + eps)
    v = ((xd - mu[:, None]) * rs[:, None]) @ Wf
    Sx = (xd.abs() @ Wf.abs()) * rs[:, None]
    c1, _ = c1_tau("tc" if M >= 128 else "mma", C, C, 0)          # the dispatcher's path
    pre = v + bf
    e = ln_fold_bound(c1, xd, mu, rs, Wf.sum(0).float(), Sx, v, tiny_of(x, Wf.float(), C)) \
        + U * Sx + 2 * U * (v.abs() + bf.abs())                  # fp32 rounding of W' and b' at commit, the bias add
    if gelu:
        ref = Fn.gelu(pre)
        bound = GELU_SLOPE * (e + 2 * U * pre.abs()) + 4 * U * (ref.abs() + 1)
    else:
        ref, bound = pre, e
    # the fold's error grows with |mu| / sigma (test_contraction_gpu.run_ln_bias): the north star is held on rows within 10 sigma
    report(f"ln linear M={M} {C}->{parts}x{N} gelu={gelu} eps={eps:g}", out, ref, bound, ns_rows=mu.abs() * rs < 10)


# ------------------------------------------------------------------------------------------------ positional conv
@pytest.mark.parametrize("B,T,k", [(2, 150, 128), (3, 200, 31), (2, 129, 127), (3, 333, 128)])
def test_pos_conv_batch_equals_each_sequence_alone(B, T, k):
    G = 4
    D = 64 * G
    seed = 6500 + B + T + k
    x = gen((B, T, D), seed, 2.0)
    g, v, bias = 1 + gen((1, 1, k), seed + 1, 0.3), gen((D, 64, k), seed + 2), gen((D,), seed + 3, 0.05)
    out = torch.full((B, T, D), float("nan"), device=DEV)
    run(kernel=HUBERT_POS_CONV, B=B, T=T, G=G, k=k, x=x, g=g, w=v, bias=bias, out=out)
    for b in range(B):                      # T >= 128: alone and batched take the same wgmma path, so no bit may change
        alone = torch.full((1, T, D), float("nan"), device=DEV)
        run(kernel=HUBERT_POS_CONV, B=1, T=T, G=G, k=k, x=x[b:b + 1].contiguous(), g=g, w=v, bias=bias, out=alone)
        assert torch.equal(out[b], alone[0]), f"sequence {b} differs from itself run alone"
    w = g.double() * v.double() / v.double().pow(2).sum(dim=(0, 1), keepdim=True).sqrt()
    xt = x.double().transpose(1, 2)
    conv = Fn.conv1d(xt, w, bias.double(), padding=k // 2, groups=G)[:, :, :T]
    ref = x.double() + Fn.gelu(conv).transpose(1, 2)
    # as test_hubert_gpu.test_pos_conv_kernel_matches_float64 on the wgmma path (>= 128 rows): 3-term split products within
    # 2^-20, truncating adds inside a chunk of 4 panels (48 * 2 u) and one rounded drain per 256 products
    K = 64 * k
    mag = Fn.conv1d(xt.abs(), w.abs(), None, padding=k // 2, groups=G)[:, :, :T].transpose(1, 2)
    bound = GELU_SLOPE * (2.0 ** -20 + (48 * 2 + K / 256) * U) * mag + 4 * U * (ref.abs() + x.double().abs())
    report(f"pos conv B={B} T={T} k={k}", out.reshape(B * T, D), ref.reshape(B * T, D), bound.reshape(B * T, D))
