"""GPU: every fused attention and cross-attention kernel, one at a time, against a float64 reference of the same operation.

`dawn_test_fused` (include/dawn_unet.h, csrc/fused_test.cu) runs one kernel with the weight folds (`fold_linear`, `fold_ca_q`)
and fp16 packers the network's upload runs, after the kernel's own shape predicate; a refused geometry returns -1 and launches
nothing.  Rotary and relative-bias tables, cross-attention keys and Gram forms, GroupNorm sums and FiLM vectors are inputs, so
a case does not depend on the per-clip table kernels.  The bias is one random value per (head, rel = key - query), not the
bucket table, whose neighbouring rel share values; the rotary table holds random angles per (frame, pair).  The references
(tests/fused_ref.py) are written from the operation in float64 and return an elementwise bound computed from absolute
values of the same data, so the bound follows the conditioning of each case.

Error model (u = 2^-24):

* Split products.  A round-to-nearest 11-bit hi leaves |x - hi| <= 2^-11 |x|, a truncated hi (split_f16x2_trunc) <= 2^-10 |x|; lo is
  the fp16 rounding of the rest (2^-11 of it).  With the lo*lo term dropped, one product is off by at most
  3 * 2^-22 |a||b| (both round-to-nearest: attn_tc.cu), 5 * 2^-22 (truncated activation x weight image: projections,
  out-projections) or 8 * 2^-22 (both truncated: the temporal kernel's Q K^T and P V, the SLA context and output products,
  gn_hcond's Wt T).  An fp16 lo in the subnormal range adds 2^-25 times the other operand (TINY terms).
* Accumulation.  mma.sync adds with truncation inside the instruction chain: at most K * 2^-23 of sum |a||b| over the chain
  (K = 32 for scores and for P V blocks, 64 for the 64-channel projections); the round-to-nearest adds outside the
  tensor core (across key blocks, heads, pixel groups) add one u each.
* Scores.  ds_ij <= c_qk sum_d |q_d||k_d| + TINY (|q|_1 + |k|_1) + 2^-21 + 4u (|s_ij| + |m_i|) + (propagated q, k errors
  sum_d (Eq_d |k_d| + |q_d| Ek_d + Eq_d Ek_d)), c_qk = split + 32 * 2^-23 + O(u).  The 2^-21 is the relative error of
  ex2.approx / __expf, which acts as an absolute score error; the 4u terms cover the rounding of s - m, of the scale to the
  log2 domain and of the bias add.
* Softmax output.  With p the exact weights and o_i = sum_j p_ij v_j, a score perturbation ds moves o_i by
  sum_j p_ij ds_ij (v_j - o_i), so |do_i| <= max_j ds_ij * sum_j p_ij (|v_j| + |o_i|) + c_pv sum_j p_ij |v_j| + sum_j p_ij Ev_j
  + (n_i + 8) u |o_i| (the sum l of n_i weights and the normalisation) + TINY terms.
* LayerNorm-folded projections.  The temporal kernel splits the raw row and applies LayerNorm after the contraction:
  y = rstd (x W'^T - mu wsum), so its error is rstd (c1 sum |x||W'| + (K/8 + 5) u mean|x| |wsum|) + (K/8 + 6) u |y|
  (a stable fp32 mean / variance of K values is within (K/8 + 3) u), c1 = 5 * 2^-22 + 64 * 2^-23 + 8u.  That bound follows
  rows whose mean is 30-100x their standard deviation, where x W'^T cancels.  The SLA and CA kernels split the normalised
  row: c1 sum |x^||W| + rstd (K/8 + 3) u mean|x| sum |W|.  Rotary adds the errors of a pair.  The out-projections propagate
  |do| through |Wout| and add (5 * 2^-22 + 32 * 2^-23 + 10u) sum |o||Wout|.
* Cross-attention gates.  z = 8 q.(k - k_null) / |q|; dz from the q bound and 16u sum |q|(|k| + |k_null|); the gate moves by
  g (1 - g) dz + 2^-21.  Gram-form variance c^T G c, c = [1, gates]: its error is bounded relative to sum |c_a c_b G_ab|
  (20u of it plus the gates' errors through |G|), not relative to the variance, which cancels; rstd moves by 1/2 rs^3 dvar.
* GroupNorm from sums.  t = y al + be in fp32 (al, be from the fp64 statistics): 6u (|y al| + |be|); SiLU adds 1.1 dt
  + 4u |SiLU|; Wt T_f adds (8 * 2^-22 + 32 * 2^-23 + 4u) sum |Wt||T|.
* These bounds are worst cases: for the temporal kernel, where the projection bound is carried through the attention, the
  measured error sits 10^3 to 10^4 below it (on an H100 80GB HBM3 at 400 W), so an index error that moves one key's weight
  can pass it.  The norm-wise check is what such an error fails.
* Norm-wise, on every case.  ||out - ref|| / ||ref|| <= tau (over the attention / context part, without the residual): 2^-16
  for every tensor-core kernel except the ones whose inputs are themselves rounded to fp32 products (SLA, CA: 2^-15).  For
  the temporal kernel tau is multiplied by the largest |mean| / std of the case's rows (1 for zero-mean rows), because the
  raw-row split loses that factor to the LayerNorm fold's cancellation.  A 2-term split
  leaves 2^-11..2^-10 of every product, about 2^-12 rms after cancellation: 8-16x above tau.

Every case fills guard rows, ldo padding and the rows outside [q_lo, q_hi) with a sentinel and checks that they keep it.

Coverage: kernel x variant -> test.
  kernel                 variant                                                        test
  temporal_fused_kernel  (the norm-wise check is the binding one: see above)
                         F 200 x P 4096 band 40 (benchmark shape)                       test_temporal[bench]
                         F 1, 15, 16, 17 at P 131; two-stage F 224, one-stage F 225      test_temporal[f*], [stage*]
                         F 256 band 64; bands 1, 8, 41, 64 and >= F                       test_temporal[band*]
                         windows [0,40) [40,80) of 80, [40,80) of 120, [40,248) of 288   test_temporal[win*]
                         padded ldx / ldr / ldo, out aliasing res, mean 30-100x std      test_temporal[pad], [alias], [bigmean]
  attention_tc_kernel    band 40 at L 200, bands 1 / 8, L 50; pb 16 / 9 / strides;       test_attention[tc-*]
                         window [40,240) of 280; full mode with bias (L 23, band 40);
                         full without bias L 9, 64, 200, 400
  attention_kernel       bands 41, 64, 120 with L > band; a window                        test_attention[simt-*]
  sla_ctx + sla_merge    P 64, 576, 4096 and 80, 208, 400 (split lengths); F 1, 8          test_sla_ctx
  sla_out_kernel         P 64, 80, 4096, in place and not                                test_sla_out
  sla_context_kernel     P 36, 4096                                                      test_sla_ctx_unfused
  ca_wt_kernel<64/128>   P 128, 144, 1024, 4096; saturated and nearly tied gates         test_ca_wt
  ca_rstd_kernel         given gates                                                     test_ca_rstd
  gn_hcond_kernel        co 64..512, P 16 / 144 / 4096, FiLM or not, fp32 or planes      test_gn_hcond
  all                    refused geometries                                              test_refusals
  both attention cores   row strides that are not a multiple of 4                       test_attention_misaligned_rows
"""
import ctypes
import math

import pytest
import torch

from tests import fused_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = 1234.5
GUARD = 16
TAU = 2.0 ** -16


def _lib():
    from dawn_pytorch_b200 import _lib
    return _lib


def gen(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def guarded(rows, ld, tail=0):
    """[GUARD + rows + GUARD + tail][ld] sentinel buffer; returns (buffer, pointer to row 0)"""
    buf = torch.full((GUARD + rows + GUARD + tail, ld), SENT, dtype=torch.float32, device=DEV)
    return buf, buf.data_ptr() + GUARD * ld * 4


def body(buf, rows, width):
    assert torch.all(buf[:GUARD] == SENT) and torch.all(buf[GUARD + rows:] == SENT), "store outside the output rows"
    b = buf[GUARD:GUARD + rows]
    assert torch.all(b[:, width:] == SENT), "store into the row padding"
    return b[:, :width]


def run(**kw):
    L = _lib()
    c = L.DawnFusedCase()
    keep = []
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            keep.append(v)
            v = v.data_ptr()
        setattr(c, k, v)
    torch.cuda.synchronize()
    rc = L.lib.dawn_test_fused(ctypes.byref(c), None)
    torch.cuda.synchronize()
    return rc


def check(name, out, ref, bound, y_ref=None, tau=TAU, norm=True):
    out = out.double()
    assert torch.isfinite(out).all(), f"{name}: non-finite output"
    d = (out - ref).abs()
    el = (d / bound).max().item()
    yr = ref if y_ref is None else y_ref
    nr = (d.norm() / yr.norm()).item()
    print(f"  {name}: max |d|/bound = {el:.3f}; ||d||/||ref|| = {nr:.2e} ({nr / tau:.3f} tau)")
    assert el <= 1.0, f"{name}: elementwise error {el:.2f}x the bound"
    if norm:
        assert nr <= tau, f"{name}: norm-wise error {nr:.2e} > {tau:.2e}"
    return el


def attn_weights(seed):
    gamma = 1 + 0.2 * gen(64, seed)
    wqkv = gen((768, 64), seed + 1, 0.125)
    wout = gen((64, 256), seed + 2, 0.0625)
    return gamma, wqkv, wout


# ------------------------------------------------------------------------------------------------ temporal fused
TEMPORAL = {   # id: (Fe, P, band, q_lo, q_hi, options)
    "bench": (200, 4096, 40, 0, 200, {}),
    "f1": (1, 131, 40, 0, 1, {}), "f15": (15, 131, 40, 0, 15, {}), "f16": (16, 131, 40, 0, 16, {}),
    "f17": (17, 131, 40, 0, 17, {}),
    "stage2-f224": (224, 24, 40, 0, 224, {}), "stage1-f225": (225, 24, 40, 0, 225, {}),
    "band64-f256": (256, 16, 64, 0, 256, {}),
    "band1": (100, 24, 1, 0, 100, {}), "band8": (100, 24, 8, 0, 100, {}), "band41": (100, 24, 41, 0, 100, {}),
    "band64": (150, 24, 64, 0, 150, {}), "band-ge-f": (30, 24, 40, 0, 30, {}),
    "win0-80": (80, 24, 40, 0, 40, {}), "win40-80": (80, 24, 40, 40, 80, {}), "win40-120": (120, 24, 40, 40, 80, {}),
    "win40-288": (288, 16, 40, 40, 248, {}),
    "pad": (48, 40, 8, 0, 48, {"ldx": 72, "ldr": 68, "ldo": 76}),
    "alias": (48, 40, 8, 0, 48, {"alias": True}),
    "bigmean": (64, 40, 40, 0, 64, {"mean": True}),
}


@pytest.mark.parametrize("cid", list(TEMPORAL))
def test_temporal(cid):
    Fe, P, band, q_lo, q_hi, o = TEMPORAL[cid]
    seed = sum(map(ord, cid))
    ldx, ldr, ldo = o.get("ldx", 64), o.get("ldr", 64), o.get("ldo", 64)
    Fq = q_hi - q_lo
    x = gen((Fe * P, 64), seed)
    if o.get("mean"):
        x = x * 0.5 + (30 + 70 * torch.rand(Fe * P, 1, generator=torch.Generator().manual_seed(seed))).to(DEV) * 0.5
    xb = torch.full((Fe * P, ldx), SENT, device=DEV)
    xb[:, :64] = x
    gamma, wqkv, wout = attn_weights(seed)
    rot_ang = gen((Fe, 16), seed + 3, 3.0)
    rot = torch.stack((rot_ang.cos(), rot_ang.sin()), -1).contiguous()
    bias = gen((8, 2 * band + 1), seed + 4)
    res = gen((Fq * P, 64), seed + 5)
    # q_lo * P sentinel rows after the output and residual: an output row indexed by the on-chip frame f instead of f - q_lo
    # lands there
    tail = q_lo * P
    if o.get("alias"):
        obuf, optr = guarded(Fq * P, ldo, tail)
        obuf[GUARD:GUARD + Fq * P, :64] = res
        rptr, ldr = optr, ldo
    else:
        rbuf = torch.full((Fq * P + tail, ldr), SENT, device=DEV)
        rbuf[:Fq * P, :64] = res
        rptr = rbuf
        obuf, optr = guarded(Fq * P, ldo, tail)
    rc = run(kernel=_lib().FUSED_TEMPORAL, F=Fe, P=P, C=64, band=band, q_lo=q_lo, q_hi=q_hi, ldx=ldx, ldr=ldr, ldo=ldo,
             x=xb, res=rptr, out=optr, gamma=gamma, w_qkv=wqkv, w_out=wout, rot=rot, bias=bias)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    out = body(obuf, Fq * P, 64).reshape(Fq, P, 64)
    xs, rs = x.reshape(Fe, P, 64), res.reshape(Fq, P, 64)
    worst, dn, yn = 0.0, 0.0, 0.0
    for p0 in range(0, P, 128):
        sl = slice(p0, min(P, p0 + 128))
        ref, bnd, y = R.temporal(xs[:, sl].transpose(0, 1), rs[:, sl].transpose(0, 1), gamma, wqkv, wout, rot, bias, band,
                                 q_lo, q_hi)
        d = (out[:, sl].transpose(0, 1).double() - ref).abs()
        assert torch.isfinite(d).all()
        worst = max(worst, (d / bnd).max().item())
        dn += d.pow(2).sum().item()
        yn += y.pow(2).sum().item()
    nr = math.sqrt(dn / yn)
    # the raw-row split carries the conditioning of the LayerNorm fold: rows whose mean is r times their standard deviation
    # lose a factor r, so tau scales with the largest r of the case (1 for zero-mean rows)
    r = max(1.0, (xs.mean(-1).abs() / xs.std(-1, unbiased=False)).max().item())
    tau = TAU * r
    print(f"  temporal {cid}: max |d|/bound = {worst:.3f}; ||d||/||y|| = {nr:.2e} ({nr / tau:.3f} tau, mean/std {r:.0f})")
    assert worst <= 1.0, f"elementwise error {worst:.2f}x the bound"
    assert nr <= tau, f"norm-wise error {nr:.2e} > {tau:.2e}"


# ------------------------------------------------------------------------------------------------ attention cores
ATTN = {   # id: (kernel, nseq, L, band, q_lo, q_hi, layout, bias)
    "tc-band40-L200": ("tc", 32, 200, 40, 0, 200, "pb16", True),
    "tc-band1": ("tc", 16, 100, 1, 0, 100, "pb16", True),
    "tc-band8": ("tc", 18, 100, 8, 0, 100, "pb9", True),
    "tc-L50": ("tc", 18, 50, 40, 0, 50, "pb9", True),
    "tc-strided": ("tc", 6, 70, 20, 0, 70, "stride", True),
    "tc-win40-240": ("tc", 16, 280, 40, 40, 240, "pb16", True),
    "tc-full-bias-L23": ("tc", 16, 23, 40, 0, 23, "pb16", True),
    "tc-full-L9": ("tc", 4, 9, 1 << 30, 0, 9, "frames", False),
    "tc-full-L64": ("tc", 4, 64, 1 << 30, 0, 64, "frames", False),
    "tc-full-L200": ("tc", 3, 200, 1 << 30, 0, 200, "frames", False),
    "tc-full-L400": ("tc", 2, 400, 1 << 30, 0, 400, "frames", False),
    "simt-band41": ("simt", 16, 100, 41, 0, 100, "pb16", True),
    "simt-band64": ("simt", 16, 150, 64, 0, 150, "pb16", True),
    "simt-band120": ("simt", 9, 200, 120, 0, 200, "pb9", True),
    "simt-win": ("simt", 16, 180, 60, 50, 130, "pb16", True),
}


def seq_rows(layout, nseq, L):
    """row index of element e of sequence s, (nseq, L), and the AttnArgs layout fields"""
    s, e = torch.arange(nseq)[:, None], torch.arange(L)[None, :]
    if layout.startswith("pb"):
        pb = int(layout[2:])
        return ((s // pb) * L + e) * pb + s % pb, dict(pb=pb)
    if layout == "frames":                       # mid spatial attention: sequences are frames of L tokens
        return s * L + e, dict(seq_base_stride=L, elem_stride=1)
    return s + e * nseq, dict(seq_base_stride=1, elem_stride=nseq)


@pytest.mark.parametrize("cid", list(ATTN))
def test_attention(cid):
    kern, nseq, L, band, q_lo, q_hi, layout, has_bias = ATTN[cid]
    seed = sum(map(ord, cid))
    rows = nseq * L
    qkv = gen((rows, 768), seed, 0.6)
    bias = gen((8, 2 * band + 1), seed + 1) if has_bias else None
    idx, lay = seq_rows(layout, nseq, L)
    obuf, optr = guarded(rows, 264)
    kw = dict(kernel=_lib().FUSED_ATTN_TC if kern == "tc" else _lib().FUSED_ATTN_SIMT, nseq=nseq, L=L, band=band, q_lo=q_lo,
              q_hi=q_hi, ld=768, ldo=264, qkv=qkv, out=optr, **lay)
    if bias is not None:
        kw["bias"] = bias
    rc = run(**kw)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    out = body(obuf, rows, 256)
    idx = idx.to(DEV)
    owned = torch.zeros(rows, dtype=torch.bool, device=DEV)
    owned[idx[:, q_lo:q_hi].reshape(-1)] = True
    assert torch.all(out[~owned] == SENT), "store into a row outside [q_lo, q_hi)"
    t = qkv.double()[idx]                                                  # (nseq, L, 768)
    hd = lambda a: a.reshape(nseq, L, 8, 32).transpose(1, 2)
    q, k, v = hd(t[..., :256])[:, :, q_lo:q_hi], hd(t[..., 256:512]), hd(t[..., 512:])
    full = band >= L
    nk = L if full else min(L, 2 * band + 1)
    if kern == "tc":
        c_qk, c_pv = R.SPLIT_RR + 32 * 2.0 ** -23 + 4 * R.U, R.SPLIT_RR + 32 * 2.0 ** -23 + (nk / 32 + 6) * R.U
    else:
        c_qk, c_pv = 34 * R.U, (nk + 2) * R.U
    o, bnd = R.attention(q, k, v, torch.arange(q_lo, q_hi, device=DEV), band, None if bias is None else bias.double(), c_qk,
                         c_pv, e_exp=R.EXP2 if kern == "tc" else 4 * R.U, full=full)
    got = out[idx[:, q_lo:q_hi]].double().reshape(nseq, q_hi - q_lo, 8, 32).transpose(1, 2)
    check(f"attention {cid}", got, o, bnd)


# ------------------------------------------------------------------------------------------------ SLA
def sla_weights(seed):
    gamma = 1 + 0.2 * gen(64, seed)
    wqkv = gen((768, 64), seed + 1, 0.3)
    wout = gen((64, 256), seed + 2, 0.0625)
    return gamma, wqkv, wout


SLA_CTX = [(64, 1), (576, 8), (4096, 8), (80, 1), (80, 8), (208, 8), (400, 1)]


@pytest.mark.parametrize("P,Fr", SLA_CTX, ids=[f"P{p}-F{f}" for p, f in SLA_CTX])
def test_sla_ctx(P, Fr):
    seed = 7 * P + Fr
    x = gen((Fr * P, 64), seed)
    gamma, wqkv, wout = sla_weights(seed)
    ldb = 72
    bbuf, bptr = guarded(Fr * 256, ldb)
    rc = run(kernel=_lib().FUSED_SLA_CTX, F=Fr, P=P, C=64, ldx=64, ldb=ldb, x=x, gamma=gamma, w_qkv=wqkv, w_out=wout, Bf=bptr)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    Bf = body(bbuf, Fr * 256, 64).reshape(Fr, 256, 64)
    ref, bnd = R.sla_ctx(x.reshape(Fr, P, 64), gamma, wqkv, wout)
    check(f"sla_ctx P{P} F{Fr}", Bf, ref, bnd, tau=2 * TAU)


@pytest.mark.parametrize("P,inplace", [(64, True), (80, False), (4096, True), (4096, False)])
def test_sla_out(P, inplace):
    Fr = 3
    seed = 11 * P + inplace
    x = gen((Fr * P, 64), seed)
    gamma, wqkv, _ = sla_weights(seed)
    Bf = gen((Fr * 256, 64), seed + 3, 0.05)
    bias = gen(64, seed + 4)
    obuf, optr = guarded(Fr * P, 68)
    if inplace:
        obuf[GUARD:GUARD + Fr * P, :64] = x
        xptr, ldx = optr, 68
    else:
        xptr, ldx = x, 64
    rc = run(kernel=_lib().FUSED_SLA_OUT, F=Fr, P=P, C=64, ldx=ldx, ldo=68, ldb=64, x=xptr, out=optr, gamma=gamma, w_qkv=wqkv,
             Bf=Bf, out_bias=bias)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    out = body(obuf, Fr * P, 64).reshape(Fr, P, 64)
    ref, bnd = R.sla_out(x.reshape(Fr, P, 64), gamma, wqkv, Bf.reshape(Fr, 256, 64), bias)
    check(f"sla_out P{P} inplace={inplace}", out, ref, bnd, y_ref=ref - (x.reshape(Fr, P, 64).double() + bias.double()),
          tau=2 * TAU)


@pytest.mark.parametrize("P", [36, 4096])
def test_sla_ctx_unfused(P):
    Fr, C = 2, 128
    seed = 13 * P
    qkv = gen((Fr * P, 768), seed)
    wout = gen((C, 256), seed + 1, 0.0625)
    ldb = 136
    bbuf, bptr = guarded(Fr * 256, ldb)
    rc = run(kernel=_lib().FUSED_SLA_CTX_UNFUSED, F=Fr, P=P, C=C, ld=768, ldb=ldb, qkv=qkv, w_out=wout, Bf=bptr)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    Bf = body(bbuf, Fr * 256, C).reshape(Fr, 256, C)
    t = qkv.double().reshape(Fr, P, 3, 8, 32)
    k, v = t[:, :, 1].permute(0, 2, 3, 1), t[:, :, 2].permute(0, 2, 3, 1)   # (F, 8, 32, P)
    p = torch.softmax(k, -1)
    ctx = p @ v.transpose(-1, -2)
    W = wout.double().t().reshape(8, 32, C)
    ref = (ctx @ W).reshape(Fr, 256, C)
    pv = p @ v.abs().transpose(-1, -2)
    dctx = (4 * R.U * (k.abs() + k.amax(-1, keepdim=True).abs()) + 4 * R.U).amax(-1, keepdim=True) * (pv + ctx.abs()) \
        + (P + 8) * R.U * (pv + ctx.abs())
    bnd = (dctx @ W.abs() + 34 * R.U * (ctx.abs() @ W.abs())).reshape(Fr, 256, C)
    check(f"sla_context P{P}", Bf, ref, bnd)


# ------------------------------------------------------------------------------------------------ cross-attention gates
def ca_inputs(ci, Fr, P, seed):
    x = gen((Fr * P, ci), seed)
    g3 = 1 + 0.2 * gen((3, ci), seed + 1)
    toq = gen((3, 64, ci), seed + 2, ci ** -0.5)
    kq = gen((Fr, 3, 64), seed + 3)
    nkq = gen((3, 8), seed + 4)
    kq[0, 0] *= 40                               # frame 0, pose: saturated gates
    kq[-1, 1] = nkq[1].repeat(8) + 1e-3 * kq[-1, 1]   # last frame, audio: nearly tied logits
    B = gen((Fr, 3, 9, 24), seed + 5, 0.3)
    G = (B @ B.transpose(-1, -2)).reshape(Fr, 3, 81).contiguous()
    return x, g3, toq, kq, nkq, G


@pytest.mark.parametrize("ci,P", [(64, 128), (64, 144), (128, 1024), (64, 4096), (128, 144), (128, 4096)])
def test_ca_wt(ci, P):
    Fr = 2
    x, g3, toq, kq, nkq, G = ca_inputs(ci, Fr, P, 17 * P + ci)
    wbuf, wptr = guarded(Fr * P, 32)
    rc = run(kernel=_lib().FUSED_CA_WT, F=Fr, P=P, C=ci, ldx=ci, x=x, gamma=g3, w_qkv=toq, kq=kq, nkq=nkq, G=G, Wt=wptr)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    Wt = body(wbuf, Fr * P, 32)
    assert torch.all(Wt[:, 27:] == 0), "Wt columns 27-31 must be zero"
    gates, dg = R.ca_gates(x.reshape(Fr, P, ci), g3, toq, kq, nkq)
    assert (gates < 1e-6).any() and (gates > 1 - 1e-6).any() and ((gates - 0.5).abs() < 1e-2).any()
    ref, bnd = R.ca_rstd(gates, G, dg)
    check(f"ca_wt ci{ci} P{P}", Wt.reshape(Fr, P, 32)[..., :27], ref[..., :27], bnd[..., :27], tau=2 * TAU)


def test_ca_rstd():
    Fr, P = 3, 100
    g = torch.sigmoid(gen((Fr * P, 24), 5, 3.0))
    B = gen((Fr, 3, 9, 24), 6, 0.3)
    G = (B @ B.transpose(-1, -2)).reshape(Fr, 3, 81).contiguous()
    wbuf, wptr = guarded(Fr * P, 32)
    rc = run(kernel=_lib().FUSED_CA_RSTD, F=Fr, P=P, gates=g, G=G, Wt=wptr)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    Wt = body(wbuf, Fr * P, 32)
    assert torch.all(Wt[:, 27:] == 0)
    ref, bnd = R.ca_rstd(g.reshape(Fr, P, 3, 8), G)
    check("ca_rstd", Wt.reshape(Fr, P, 32), ref, bnd + (ref == 0))


# ------------------------------------------------------------------------------------------------ gn_hcond
GN = [(co, P, film, planes) for co, P in [(64, 16), (128, 144), (256, 4096), (512, 144), (64, 4096), (512, 16)]
      for film, planes in [(False, False), (True, True), (True, False), (False, True)]]


@pytest.mark.parametrize("co,P,film,planes", GN, ids=[f"co{c}-P{p}-{'film' if f else 'nofilm'}-{'planes' if s else 'fp32'}"
                                                      for c, p, f, s in GN])
def test_gn_hcond(co, P, film, planes):
    Fr = 2
    seed = co + P + 2 * film + planes
    M = Fr * P
    Y = gen((M, co), seed, 2.0) + 0.5
    cpg = co // 8
    yd = Y.double().reshape(M, 8, cpg)
    stats = torch.stack((yd.sum((0, 2)), (yd * yd).sum((0, 2))), 1).reshape(16).contiguous()
    gw, gb = 1 + 0.3 * gen(co, seed + 1), 0.3 * gen(co, seed + 2)
    fv = gen(2 * co, seed + 3, 0.5) if film else None
    Wt = gen((M, 32), seed + 4, 0.5)
    Wt[:, 27:] = 0
    ldbT = co + 64 if co % 128 else co
    T = gen((Fr * 32, ldbT), seed + 5, 0.3)
    kw = dict(kernel=_lib().FUSED_GN_HCOND, F=Fr, P=P, C=co, ldy=co, ldbT=ldbT, Y=Y, Wt=Wt, T=T, gn_stats=stats,
              gn_count=float(M * cpg), cpg=cpg, gn_w=gw, gn_b=gb)
    if fv is not None:
        kw["film"] = fv
    if planes:
        pl = torch.full((2 * GUARD + 2 * M, co), 0x7BFF, dtype=torch.int16, device=DEV)   # sentinel: fp16 65504
        hi, lo = pl[GUARD:GUARD + M], pl[GUARD + M:GUARD + 2 * M]
        kw.update(out16h=hi.data_ptr(), out16l=lo.data_ptr())
    else:
        obuf, optr = guarded(M, co + 8)
        kw.update(out=optr, ldo=co + 8)
    rc = run(**kw)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    ref, bnd = R.gn_hcond(Y.reshape(Fr, P, co), stats, float(M * cpg), cpg, gw, gb, fv, Wt.reshape(Fr, P, 32),
                          T.reshape(Fr, 32, ldbT)[..., :co])
    name = f"gn_hcond co{co} P{P} film={film} planes={planes}"
    if planes:
        assert torch.all(pl[:GUARD] == 0x7BFF) and torch.all(pl[GUARD + 2 * M:] == 0x7BFF), "store outside the planes"
        h, l = hi.view(torch.float16).float(), lo.view(torch.float16).float()
        nrm = h.abs() >= 2.0 ** -14                                        # fp16 normal range: hi holds all 11 bits
        assert nrm.float().mean() > 0.99
        half_ulp = torch.ldexp(torch.ones_like(h), torch.frexp(h).exponent - 12)     # of hi's 11-bit significand
        assert torch.all(l.abs()[nrm] <= half_ulp[nrm]), f"{name}: hi is not the value rounded to 11 significant bits"
        assert torch.all(l.abs()[nrm] <= 2.0 ** -11 * h.abs()[nrm]), f"{name}: |lo| > 2^-11 |hi|"
        check(name, (h.double() + l.double()).reshape(Fr, P, co), ref,
              bnd + 2.0 ** -22 * ref.abs() + R.TINY)
    else:
        check(name, body(obuf, M, co).reshape(Fr, P, co), ref, bnd)


# ------------------------------------------------------------------------------------------------ refusals
REFUSE = [
    ("temporal band 65", dict(kernel=0, F=100, P=4, C=64, band=65, q_lo=0, q_hi=100)),
    ("temporal band 0", dict(kernel=0, F=100, P=4, C=64, band=0, q_lo=0, q_hi=100)),
    ("temporal C 128", dict(kernel=0, F=100, P=4, C=128, band=40, q_lo=0, q_hi=100)),
    ("temporal 17 query tiles", dict(kernel=0, F=288, P=4, C=64, band=40, q_lo=8, q_hi=272)),
    ("temporal window past F", dict(kernel=0, F=100, P=4, C=64, band=40, q_lo=40, q_hi=101)),
    ("temporal F 400 (shared memory)", dict(kernel=0, F=400, P=4, C=64, band=8, q_lo=0, q_hi=200)),
    ("attention tc band 41", dict(kernel=1, nseq=4, L=100, band=41, q_lo=0, q_hi=100, ld=768, ldo=256)),
    ("sla P 48", dict(kernel=3, F=1, P=48, C=64, ldx=64, ldb=64)),
    ("sla P 72", dict(kernel=3, F=1, P=72, C=64, ldx=64, ldb=64)),
    ("sla 17 splits", dict(kernel=3, F=1, P=1088, C=64, ldx=64, ldb=64)),
    ("sla C 128", dict(kernel=4, F=1, P=64, C=128, ldx=128, ldb=64, ldo=128)),
    ("ca P 112", dict(kernel=6, F=1, P=112, C=64, ldx=64)),
    ("ca ci 96", dict(kernel=6, F=1, P=128, C=96, ldx=96)),
    ("gn_hcond co 48", dict(kernel=8, F=1, P=16, C=48, cpg=6, ldy=48, ldbT=64, ldo=48)),
    ("gn_hcond P 24", dict(kernel=8, F=1, P=24, C=64, cpg=8, ldy=64, ldbT=64, ldo=64)),
    ("gn_hcond co 544", dict(kernel=8, F=1, P=16, C=544, cpg=68, ldy=544, ldbT=576, ldo=544)),
]


@pytest.mark.parametrize("name,geo", REFUSE, ids=[r[0] for r in REFUSE])
def test_refusals(name, geo):
    """each kernel's own predicate refuses the geometry: -1, and the output stays untouched"""
    big = torch.zeros(1 << 16, device=DEV)
    out = torch.full((1 << 16,), SENT, device=DEV)
    ptrs = {k: big for k in ("x", "res", "gamma", "w_qkv", "w_out", "rot", "bias", "qkv", "out_bias", "kq", "nkq", "G",
                             "gates", "T", "Y", "gn_w", "gn_b")}
    ptrs["gn_stats"] = torch.zeros(16, dtype=torch.float64, device=DEV)
    for k in ("out", "Bf", "Wt"):
        ptrs[k] = out
    base = dict(ldx=64, ldr=64, ldo=256, ld=768, ldb=64, ldy=64, ldbT=64)
    base.update(geo)
    rc = run(**base, **ptrs)
    assert rc == -1, f"{name}: accepted"
    assert "refuses" in _lib().lib.dawn_last_error().decode()
    assert torch.all(out == SENT)


@pytest.mark.parametrize("kern,ld,ldo", [(2, 770, 256), (2, 768, 258), (1, 770, 256)])
def test_attention_misaligned_rows(kern, ld, ldo):
    """both attention cores read and write rows as float4: a row stride that is not a multiple of 4 is refused"""
    qkv = torch.zeros(16 * 40 * ld, device=DEV)
    out = torch.full((16 * 40 * ldo,), SENT, device=DEV)
    rc = run(kernel=kern, nseq=16, L=40, band=8, q_lo=0, q_hi=40, pb=16, ld=ld, ldo=ldo, qkv=qkv, out=out)
    assert rc == -1 and "bad geometry" in _lib().lib.dawn_last_error().decode()
    assert torch.all(out == SENT)
