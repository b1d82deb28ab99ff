"""GPU: the UNet's per-clip and per-step glue kernels (csrc/kernels.cu), one at a time, against a float64 reference of the same
operation, and the sampler's exact quantile select against a float64 sort.

`dawn_test_kernel` (include/dawn_unet.h, csrc/kernels_test.cu) runs one kernel through the launcher unet.cu calls, on the test's
buffers; it builds the CondDesc / FilmDesc arrays on the device and refuses a bad geometry before any CUDA call.  The references
(tests/unet_kernel_ref.py) are written from the operation in float64 and return an elementwise bound computed from absolute values
of the same data.  Multi-stage kernels are checked stage by stage: each stage's reference starts from what the kernel's previous
stage wrote, so the bounds do not have to carry errors through.

Error model (u = 2^-24):

* Sums.  A sum of n fp32 terms accumulated in a chain of depth d is within (d + 1) u sum |terms| (FMA chains included); the
  lane-strided warp sums have depth ceil(n / 32) + 5, the sequential ones n.  Each further fp32 operation adds u of its result.
* Row statistics.  The mean is within (NV + 9) u mean|x|; the mean's error only adds its square to the variance, each centred
  square and the sum add (NV + 11) u var, and rstd moves by 1/2 dvar / (var + eps) + 3u of itself.
* GroupNorm apply.  mean and rstd come from the fp64 sums exactly as the reference forms them and round to fp32: the output
  moves by rstd |w| (u |mean| + 5u |y - mean|) + 2u (|b| + |t|) before SiLU, so rows whose mean is far above their spread are
  bounded by the rounding of the mean.  SiLU: |SiLU'| <= 1.1 plus 5u of the result (expf is within 2 ulp).
* Transcendentals.  sinf / cosf / erff / expf are within 2 ulp (CUDA C Programming Guide, Mathematical Functions).  The
  sinusoid and rotary angles are the fp32 products the kernels and the oracle form; sin and cos are then taken in float64.
* Cross-attention tables.  Normalised keys: 16u of |kq|.  u vectors: 66u sum |Wout||nv| (u_0), 10u sum |Wout|(|v| + |nv|)
  (u_h).  Centring adds the mean's error.  G is bounded relative to sum_c |u_a||u_b| / co, not to G, which cancels.
* Norm-wise, on every rounding case: ||out - ref|| / ||ref|| <= tau = 2^-18 (times mean / std where rows are offset), so an
  error of 1e-5 relative everywhere fails even where the elementwise bound allows it.
* Bit-exact: ncf_to_nhwc, fea_shift, frame_invariance, split_rows (against a numpy restatement of split_f16x2_rn), map_reduce
  (against the same fixed-order fp32 sum) and the select's order statistics.

Every output buffer has sentinel guard rows and padding columns that must keep the sentinel.

Coverage: kernel x variant -> test.
  kernel                    variant                                                         test
  rowstats_kernel<8/16>     C 64, 192, 1024, 1536, 2048; M 37; ld > C; mean 100x std        test_rowstats
  gn_apply_kernel           co 64..1024; clips 1, 2, 3, 16; res off / on / in place;        test_gn_apply
                            padded ldy / ldr / ldo; offset groups
  cond_mlp / cond_kv /      co 64..512 in one launch (early returns), co 1024 (64 KB smem);  test_cond_tables
  ca_tables_batched         K 1024 / 6 / 2; F 23, 46, 69 with clips 1, 2, 3; zero key head
  time_mlp_kernel           dim 64, 128; t 0, 1, 47, 999; clips 1, 16; t_stride 0, 1          test_time_mlp
  film_kernel               n 128..2048 in one launch; clips 1, 3, 16                      test_film
  rotary_table_kernel       F 1, 200, 288; pos0 0, 40, 4000                                  test_rotary
  split_rows_kernel         zeros, -0, subnormals, ties, overflow; ld > C                    test_split_rows
  ncf_to_nhwc_kernel        C 275 -> Cpad 288 at c0 3; HW 17x9; clips 1, 3; skip flag        test_ncf_to_nhwc
  frame_invariance_kernel   last element; +0 / -0; NaN; F 1; 16 clips                        test_frame_invariance
  fea_shift / map_reduce    k 3, 5, 7; clips 1, 3; skip flag                                 test_fea_shift_map_reduce
  init_conv_x3_tiled<7>     W 8, 24, 64, 65, 100; H 1, 3, 8, 9; both clip strides; skip      test_init_conv_x3[tiled*]
  init_conv_x3_kernel       k 3, 5 at Co 64, k 7 at Co 128; skip                             test_init_conv_x3[gen*]
  heads_out_kernel          C 64, 128; (ng, nc) (2, 1), (2, 2); clips 1, 2, 3                test_heads_out
  all                       refused geometries (tests/test_unet_kernel_reference_cpu.py too) test_refusals
  radix select (DDIM/DDPM)  n 1 .. 2 457 600; ties; lo + 1 / lo + 2 keys <= v; clamp to 1;    test_select
                            zeros, -0, subnormals; 1e-30 .. 1e30; q 0.5, 1, 0.9, 1e-6
  ddim_update_kernel        first step of the 20-, 250-, 500-, 999-step schedules, bit-exact test_ddim_schedule
                            (every update variant: tests/test_sampler_kernels_gpu.py)
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests import unet_kernel_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = 1234.5
GUARD = 16
TAU = 2.0 ** -18
DT = torch.float64


def _lib():
    from dawn_pytorch_b200 import _lib
    return _lib


def gen(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def guarded(rows, ld, dtype=torch.float32, sent=SENT):
    """[GUARD + rows + GUARD][ld] sentinel buffer; returns (buffer, pointer to row 0)"""
    buf = torch.full((GUARD + rows + GUARD, ld), sent, dtype=dtype, device=DEV)
    return buf, buf.data_ptr() + GUARD * ld * buf.element_size()


def body(buf, rows, width, sent=SENT):
    assert torch.all(buf[:GUARD] == sent) and torch.all(buf[GUARD + rows:] == sent), "store outside the output rows"
    b = buf[GUARD:GUARD + rows]
    assert torch.all(b[:, width:] == sent), "store into the row padding"
    return b[:, :width]


def run(descs=(), **kw):
    L = _lib()
    c = L.DawnKernelCase()
    keep = []

    def ptr(v):
        if isinstance(v, torch.Tensor):
            keep.append(v)
            return v.data_ptr()
        return v
    for k, v in kw.items():
        setattr(c, k, ptr(v))
    for i, d in enumerate(descs):
        for k, v in d.items():
            setattr(c.desc[i], k, ptr(v))
    c.ndesc = len(descs) if descs else c.ndesc
    torch.cuda.synchronize()
    rc = L.lib.dawn_test_kernel(ctypes.byref(c), None)
    torch.cuda.synchronize()
    return rc


def ok(**kw):
    rc = run(**kw)
    assert rc == 0, _lib().lib.dawn_last_error().decode()


def check(name, out, ref, bound, tau=TAU, norm=True):
    out = out.double()
    assert torch.isfinite(out).all(), f"{name}: non-finite output"
    d = (out - ref).abs()
    el = torch.where(d == 0, 0.0, d / bound).max().item()           # exact zeros (a zero key head) have a zero bound
    nr = (d.norm() / ref.norm()).item() if ref.norm() > 0 else d.norm().item()
    print(f"  {name}: max |d|/bound = {el:.3f}; ||d||/||ref|| = {nr:.2e} ({nr / tau:.3f} tau)")
    assert el <= 1.0, f"{name}: elementwise error {el:.2f}x the bound"
    if norm:
        assert nr <= tau, f"{name}: norm-wise error {nr:.2e} > {tau:.2e}"
    return el


def padded(rows, C, ld, seed, scale=1.0, offset=None):
    """(rows, ld) fp32 rows with C live channels; padding columns hold 1e30 so that a read of them shows"""
    x = torch.full((rows, ld), 1e30, dtype=torch.float32, device=DEV)
    v = gen((rows, C), seed, scale)
    if offset is not None:
        v = v + offset
    x[:, :C] = v
    return x


# ================================================================================================================= rowstats
@pytest.mark.parametrize("C,ld,big", [(64, 64, False), (192, 196, False), (1024, 1024, False), (1536, 1540, False), (2048, 2048, False),
                                      (2048, 2052, True), (1024, 1028, True), (192, 192, True)])
def test_rowstats(C, ld, big):
    M = 37
    off = (100 * gen((M, 1), C + 1)) if big else None
    x = padded(M, C, ld, C, 1.0, off)
    buf, p = guarded(M, 2)
    ok(kernel=_lib().KERNEL_ROWSTATS, x=x, ld=ld, C=C, M=M, eps=1e-5, out=p)
    o = body(buf, M, 2)
    mu, rstd, dmu, drstd = R.rowstats(x[:, :C].double())
    check(f"mean C={C}", o[:, 0], mu, dmu, norm=not big)
    check(f"rstd C={C}", o[:, 1], rstd, drstd)


# ================================================================================================================= gn_apply
GN_CASES = [  # co, clips, P, Fc, res ("none" | "sep" | "inplace"), pad, offset
    (64, 1, 64, 3, "none", 0, 0.0), (128, 2, 36, 2, "sep", 4, 0.0), (256, 3, 16, 2, "inplace", 0, 0.0),
    (512, 16, 4, 1, "sep", 8, 0.0), (1024, 2, 4, 3, "none", 4, 0.0), (64, 3, 100, 1, "sep", 0, 50.0),
    (256, 16, 9, 2, "inplace", 4, 30.0)]


@pytest.mark.parametrize("co,clips,P,Fc,res,pad,offset", GN_CASES)
def test_gn_apply(co, clips, P, Fc, res, pad, offset):
    M, cpg = Fc * clips * P, co // 8
    ld = co + pad
    clip = (torch.arange(M, device=DEV) // P) % clips
    y = padded(M, co, ld, co + clips, 1.0)
    # every clip and group gets its own offset and spread, so a wrong clip or group index moves the output
    shift = offset + gen((clips, 8), 5, 2.0)
    spread = 0.5 + gen((clips, 8), 6).abs()
    grp = torch.arange(co, device=DEV) // cpg
    y[:, :co] = y[:, :co] * spread[clip][:, grp] + shift[clip][:, grp]
    st, count = R.gn_stats(y[:, :co].double(), P, clips, cpg)
    w, b = 1 + 0.3 * gen(co, 7), 0.5 * gen(co, 8)
    r = padded(M, co, ld, 9) if res != "none" else None
    if res == "inplace":
        obuf, op = None, r.data_ptr()
        rref = r[:, :co].double().clone()
    else:
        obuf, op = guarded(M, ld)
        rref = r[:, :co].double() if r is not None else None
    ok(kernel=_lib().KERNEL_GN_APPLY, y=y, ldy=ld, C=co, M=M, stats=st.contiguous(), count=count, cpg=cpg, P=P, clips=clips,
       w=w, b=b, res=r if r is not None else None, ldr=ld, out=op, ldo=ld)
    out = body(obuf, M, co) if obuf is not None else r[:, :co]
    if obuf is not None:
        assert torch.all(obuf[GUARD:GUARD + M, co:] == SENT)
    else:
        assert torch.all(r[:, co:] == 1e30), "store into the row padding"
    ref, bound = R.gn_apply(y[:, :co].double(), st, count, P, clips, cpg, w.double(), b.double(), rref)
    tau = TAU * max(1.0, offset / 2)
    check(f"gn_apply co={co} clips={clips} res={res}", out, ref, bound, tau=tau)


# ================================================================================================================= cond tables
COND_OFF = {0: (1024, 6), 1: (0, 1024), 2: (1030, 2)}          # pose, aud, eye slices of the 1032-wide cond (ca slot order)


def cond_block(co, F, seed, zero_head=None):
    """one conditioned block's parameters and caller-owned outputs"""
    n1 = 2 * co
    ldbT = co + 8
    blk = dict(co=co, ldbT=ldbT, kq=guarded(F, 192), nkq=guarded(1, 24), T=guarded(F * 32, ldbT), G=guarded(F, 243), slots=[])
    for ca in range(3):
        off, K = COND_OFF[ca]
        s = seed + 31 * ca
        Wkv = gen((128, n1), s + 2, n1 ** -0.5)
        if zero_head is not None and ca == 1:
            Wkv[8 * zero_head:8 * zero_head + 8] = 0                            # that head's key is 0: F.normalize's clamp
        sl = dict(off=off, K=K, ca=ca, mW=gen((n1, K), s, K ** -0.5), mB=0.1 * gen(n1, s + 1), Wkv=Wkv,
                  nkv=gen((2, 8), s + 3), qs=1 + 0.3 * gen(8, s + 4), ks=1 + 0.3 * gen(8, s + 5),
                  Wout=gen((co, 64), s + 6, 0.125), gout=1 + 0.2 * gen(co, s + 7), ctx=guarded(F, n1), kv=guarded(F, 128))
        blk["slots"].append(sl)
    return blk


def desc_of(blk, sl):
    d = {k: sl[k] for k in ("off", "K", "ca", "mW", "mB", "Wkv", "nkv", "qs", "ks", "Wout", "gout")}
    d.update(co=blk["co"], ldbT=blk["ldbT"], ctx=sl["ctx"][1], kv=sl["kv"][1], kq=blk["kq"][1], nkq=blk["nkq"][1],
             T=blk["T"][1], G=blk["G"][1])
    return d


@pytest.mark.parametrize("cos,F,clips", [((64, 128, 256, 512), 23, 1), ((64, 256), 46, 2), ((128, 512), 69, 3), ((1024,), 23, 1)],
                         ids=["co64-512-F23", "clips2-F46", "clips3-F69", "co1024"])
def test_cond_tables(cos, F, clips):
    cond = gen((F, 1032), 11, 2.0)
    blocks = [cond_block(co, F, 100 * i + co, zero_head=(2 if i == 0 else None)) for i, co in enumerate(cos)]
    descs = [desc_of(b, s) for b in blocks for s in b["slots"]]
    ok(descs=descs, kernel=_lib().KERNEL_COND_TABLES, x=cond, cond_ld=1032, F=F, clips=clips)
    worst = 0.0
    for blk in blocks:
        co, ldbT = blk["co"], blk["ldbT"]
        kq, nkq = body(blk["kq"][0], F, 192), body(blk["nkq"][0], 1, 24)
        G = body(blk["G"][0], F, 243)
        T = body(blk["T"][0], F * 32, co).reshape(F, 32, co)
        assert torch.all(blk["T"][0][GUARD:GUARD + F * 32].reshape(F, 32, ldbT)[:, 27:] == SENT), "T rows 27..31 written"
        for sl in blk["slots"]:
            ca = sl["ca"]
            tag = f"co={co} ca={ca}"
            ctx = body(sl["ctx"][0], F, 2 * co)
            ref, bd = R.cond_mlp(cond.double(), sl["off"], sl["K"], sl["mW"].double(), sl["mB"].double(), F, clips)
            worst = max(worst, check(f"ctx {tag}", ctx, ref, bd))
            kv = body(sl["kv"][0], F, 128)
            ref, bd = R.cond_kv(ctx.double(), sl["Wkv"].double())
            worst = max(worst, check(f"kv {tag}", kv, ref, bd, norm=ref.norm() > 0))
            kq_r, dkq, nkq_r, dnkq, G_r, dG, T_r, dT, gabs = R.ca_tables(kv.double(), sl["nkv"].double(), sl["qs"].double(),
                                                                         sl["ks"].double(), sl["Wout"].double(),
                                                                         sl["gout"].double())
            k_got = kq[:, 64 * ca:64 * ca + 64]
            check(f"kq {tag}", k_got, kq_r, dkq + 1e-30)
            if sl["Wkv"][16:24].abs().sum() == 0:
                assert torch.all(k_got[:, 16:24] == 0), "zero key must normalise to zero"
            check(f"nkq {tag}", nkq[0, 8 * ca:8 * ca + 8], nkq_r, dnkq)
            g_got = G[:, 81 * ca:81 * ca + 81].double()
            el = ((g_got - G_r).abs() / dG).max().item()
            rel = ((g_got - G_r).abs() / gabs).max().item()
            print(f"  G {tag}: max |d|/bound = {el:.3f}; max |d| / (sum|u_a||u_b|/co) = {rel:.2e}")
            assert el <= 1.0
            worst = max(worst, check(f"T {tag}", T[:, 9 * ca:9 * ca + 9], T_r, dT))
    print(f"  worst {worst:.3f}")


# ================================================================================================================= time MLP / FiLM
def time_freqs(dim):
    half = dim // 2
    e = math.log(10000) / (half - 1)
    return torch.exp(torch.arange(half) * -e).float()


@pytest.mark.parametrize("dim", [64, 128])
@pytest.mark.parametrize("clips,t_stride", [(1, 0), (1, 1), (16, 0), (16, 1)])
def test_time_mlp(dim, clips, t_stride):
    tdim = 4 * dim
    ts = [0, 1, 47, 999]
    t = torch.tensor([ts[i % 4] if i < 4 else (i * 61) % 1000 for i in range(clips)] if t_stride else [999], dtype=torch.int64)
    freqs = time_freqs(dim)
    W1, b1 = gen((tdim, dim), dim, dim ** -0.5), 0.1 * gen(tdim, dim + 1)
    W2, b2 = gen((tdim, tdim), dim + 2, tdim ** -0.5), 0.1 * gen(tdim, dim + 3)
    buf, p = guarded(clips, tdim)
    ok(kernel=_lib().KERNEL_TIME_MLP, t=t.to(DEV), t_stride=t_stride, clips=clips, freqs=freqs.to(DEV), dim=dim, w=W1, b=b1,
       w2=W2, b2=b2, out=p)
    tt = t.repeat(clips) if t_stride == 0 else t
    ref, bound = R.time_mlp(tt, freqs.double(), W1.double().cpu(), b1.double().cpu(), W2.double().cpu(), b2.double().cpu())
    check(f"time_mlp dim={dim} clips={clips} stride={t_stride}", body(buf, clips, tdim).cpu(), ref, bound)


@pytest.mark.parametrize("tdim,clips", [(256, 1), (512, 3), (256, 16)])
def test_film(tdim, clips):
    ts = gen((clips, tdim), tdim + clips)
    ns = [128, 2048, 256, 512, 1024, 128]
    descs, outs = [], []
    for i, n in enumerate(ns):
        W, b = gen((n, tdim), 10 * i + 1, tdim ** -0.5), 0.1 * gen(n, 10 * i + 2)
        o = guarded(clips, n)
        descs.append(dict(W=W, b=b, out=o[1], n=n))
        outs.append((o, W, b, n))
    ok(descs=descs, kernel=_lib().KERNEL_FILM, x=ts, C=tdim, clips=clips)
    for (o, W, b, n) in outs:
        ref, bound = R.film(ts.double(), W.double(), b.double())
        check(f"film n={n} clips={clips}", body(o[0], clips, n), ref, bound)


# ================================================================================================================= rotary
@pytest.mark.parametrize("F", [1, 200, 288])
@pytest.mark.parametrize("pos0", [0, 40, 4000])
def test_rotary(F, pos0):
    freqs = (1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32))).float()
    buf, p = guarded(F, 32)
    ok(kernel=_lib().KERNEL_ROTARY, freqs=freqs.to(DEV), F=F, pos0=pos0, out=p)
    ref, bound = R.rotary_table(freqs, F, pos0)
    check(f"rotary F={F} pos0={pos0}", body(buf, F, 32).cpu().reshape(F, 16, 2), ref, bound)


# ================================================================================================================= split_rows
def test_split_rows():
    M, C, ld = 41, 196, 200
    x = padded(M, C, ld, 3)
    v = x[:, :C]
    v[0, :8] = torch.tensor([0.0, -0.0, 1e-40, -1e-42, 6e-8, 65504.0, 70000.0, -1e9])
    # exact rounding ties of the 11-bit hi: bit 12 set, bits below clear
    tie = torch.tensor([1.0 + 2.0 ** -11, 3.0 + 2.0 ** -10, -(1.5 + 2.0 ** -12)], dtype=torch.float32)
    v[1, :3] = tie
    v[2] = gen(C, 4, 1e-6)
    v[3] = gen(C, 5, 1e4)
    hb, hp = guarded(M, C, torch.int16, -1)
    lb, lp = guarded(M, C, torch.int16, -1)
    ok(kernel=_lib().KERNEL_SPLIT_ROWS, x=x, ld=ld, C=C, M=M, out_hi=hp, out_lo=lp)
    h_ref, l_ref = R.split_f16x2_rn(v.cpu().numpy())
    h = body(hb, M, C, -1).cpu().numpy().view(np.uint16)
    lo = body(lb, M, C, -1).cpu().numpy().view(np.uint16)
    assert np.array_equal(h, h_ref), f"hi plane differs at {np.argwhere(h != h_ref)[:5]}"
    assert np.array_equal(lo, l_ref), f"lo plane differs at {np.argwhere(lo != l_ref)[:5]}"


# ================================================================================================================= layout
@pytest.mark.parametrize("clips", [1, 3])
@pytest.mark.parametrize("skip", [None, "equal", "other"])
def test_ncf_to_nhwc(clips, skip):
    C, Cpad, c0, F, HW = 275, 288, 3, 5, 17 * 9
    x = gen((clips, C, F, HW), clips)
    flag = torch.tensor([1 if skip == "equal" else 0], dtype=torch.int32, device=DEV)
    buf, p = guarded(F * clips * HW, Cpad)
    ok(kernel=_lib().KERNEL_NCF_TO_NHWC, x=x, C=C, F=F, P=HW, Cpad=Cpad, c0=c0, out=p, clips=clips,
       skip_flag=flag if skip else None, skip_if=1)
    if skip == "equal":
        assert torch.all(buf == SENT), "a skipped launch wrote"
        return
    got = body(buf, F * clips * HW, Cpad).reshape(F * clips, HW, Cpad)
    assert torch.equal(got, R.ncf_to_nhwc(x, clips, C, F, HW, Cpad, c0))


def frame_case(name):
    clips, C, F, HW = 1, 275, 4, 17 * 9
    x = gen((clips, C, 1, HW), 3).expand(clips, C, F, HW).contiguous()
    want = None
    if name == "last":
        x[0, -1, -1, -1] = torch.nextafter(x[0, -1, -1, -1], torch.tensor(1e30, device=DEV))
    elif name == "signed_zero":
        x[0, 100, :, 7] = 0.0
        x[0, 100, 2, 7] = -0.0
    elif name == "nan_vs_finite":
        x[0, 50, 3, 9] = float("nan")
    elif name == "same_nan":
        x[0, 50, :, 9] = float("nan")
    elif name == "channel_below_c0":
        x[0, 2, 3, 0] += 1                                                     # the noisy channels are not compared
        want = [False]
    elif name == "f1":
        x = gen((2, C, 1, HW), 4)
        want = [False, False]
    elif name == "clips16":
        x = gen((16, C, 1, HW), 5).expand(16, C, F, HW).contiguous()
        x[15, 200, 1, 100] += 1
    return x, want


@pytest.mark.parametrize("name", ["invariant", "last", "signed_zero", "nan_vs_finite", "same_nan", "channel_below_c0", "f1",
                                  "clips16"])
def test_frame_invariance(name):
    x, want = frame_case(name)
    clips, C, F, HW = x.shape
    buf, p = guarded(1, clips + 1, torch.int32, -7)
    ok(kernel=_lib().KERNEL_FRAME_INVARIANCE, x=x, c0=3, C=C, F=F, P=HW, clips=clips, flag=p)
    got = body(buf, 1, clips + 1, -7)[0].tolist()
    if want is None:
        want = R.frame_invariance(x, 3)
    if name in ("last", "signed_zero", "nan_vs_finite"):
        assert want == [True]
    if name == "same_nan":
        assert want == [False]
    if name == "clips16":
        assert want == [False] * 15 + [True]
    assert got == [int(v) for v in want] + [sum(want)], f"{name}: flags {got}, want {want}"


@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("clips", [1, 3])
@pytest.mark.parametrize("skip", [None, "equal", "other"])
def test_fea_shift_map_reduce(k, clips, skip):
    Cf, Cpad, c0, F, H, W, Co = 272, 288, 3, 2, 17, 9, 64
    HW = H * W
    x = gen((clips, 275, F, HW), k + clips)                                     # the general entry's input: clip stride 275 F HW
    fea = x[:, 3:]
    flag = torch.tensor([1 if skip == "equal" else 0], dtype=torch.int32, device=DEV)
    sk = dict(skip_flag=flag if skip else None, skip_if=1)
    buf, p = guarded(k * clips * HW, Cpad)
    ok(kernel=_lib().KERNEL_FEA_SHIFT, x=fea.data_ptr(), cstride=F * HW, clip_stride=275 * F * HW, clips=clips, C=Cf, H=H, W=W,
       Cpad=Cpad, c0=c0, k=k, out=p, **sk)
    n = clips * HW * Co
    part = gen((k, n), 7 * k)
    bias = gen(Co, 8)
    mbuf, mp = guarded(1, n)
    ok(kernel=_lib().KERNEL_MAP_REDUCE, x=part, k=k, n=n, b=bias, C=Co, out=mp, **sk)
    if skip == "equal":
        assert torch.all(buf == SENT) and torch.all(mbuf == SENT), "a skipped launch wrote"
        return
    got = body(buf, k * clips * HW, Cpad).reshape(k * clips, HW, Cpad)
    assert torch.equal(got, R.fea_shift(fea[:, :, 0].reshape(clips, Cf, H, W), k, Cpad, c0))
    m = body(mbuf, 1, n)[0]
    assert torch.equal(m, R.map_reduce_f32(part, bias, Co)), "map_reduce is not the fixed-order fp32 sum"
    ref = bias.double().repeat(n // Co) + part.double().sum(0)
    check(f"map_reduce k={k}", m, ref, (k + 1) * R.U * (bias.double().abs().repeat(n // Co) + part.double().abs().sum(0)),
          tau=TAU)


# ================================================================================================================= init conv
IC_CASES = [  # tag, k, Co, H, W, clips, F, full stride (275 channels), skip clip
    ("tiled-8x1", 7, 64, 1, 8, 1, 2, False, None), ("tiled-24x3", 7, 64, 3, 24, 2, 2, True, None),
    ("tiled-64x8", 7, 64, 8, 64, 1, 2, False, None), ("tiled-65x9", 7, 64, 9, 65, 3, 1, True, 1),
    ("tiled-100x9", 7, 64, 9, 100, 2, 2, False, 0), ("tiled-100x1", 7, 64, 1, 100, 1, 3, False, None),
    ("gen-k3", 3, 64, 9, 65, 2, 2, True, None), ("gen-k5", 5, 64, 8, 24, 3, 1, False, 2),
    ("gen-k7-co128", 7, 128, 9, 33, 2, 2, False, None)]


@pytest.mark.parametrize("tag,k,Co,H,W,clips,F,full,skip", IC_CASES, ids=[c[0] for c in IC_CASES])
def test_init_conv_x3(tag, k, Co, H, W, clips, F, full, skip):
    HW = H * W
    nch = 275 if full else 3
    x = gen((clips, nch, F, H, W), k * W + H)
    w3 = gen((k * k * 3, Co), 3, 0.2)
    mp = gen((clips, H, W, Co), 4)
    flag = torch.zeros(clips, dtype=torch.int32, device=DEV)
    if skip is not None:
        flag[skip] = 1
    buf, p = guarded(F * clips * HW, 2 * Co)
    ok(kernel=_lib().KERNEL_INIT_CONV_X3, x=x, clip_stride=nch * F * HW, F=F, H=H, W=W, clips=clips, w=w3, map=mp, C=Co,
       out=p + Co * 4, ldo=2 * Co, k=k, skip_flag=flag if skip is not None else None, skip_if=1)
    rows = body(buf, F * clips * HW, 2 * Co).reshape(F * clips, HW, 2 * Co)
    assert torch.all(rows[..., :Co] == SENT), "columns [0, dim) of the cat(x, r) rows were written"
    got = rows[..., Co:]
    ref, bound = R.init_conv_x3(x[:, :3].double(), w3.double(), mp.double(), k)
    live = torch.ones(F * clips, dtype=torch.bool)
    if skip is not None:
        fo = torch.arange(F * clips)
        live = fo % clips != skip
        assert torch.all(got[~live] == SENT), "a skipped clip was written"
    check(f"init_conv {tag}", got[live], ref[live], bound[live])


# ================================================================================================================= heads
@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("ng,nc", [(2, 1), (2, 2)])
@pytest.mark.parametrize("clips", [1, 2, 3])
def test_heads_out(C, ng, nc, clips):
    F, HW = 3, 40
    M = F * clips * HW
    hf, ho = gen((M, C), C + clips), gen((M, C), C + clips + 1)
    Wf, bf = gen((ng, C), 1, C ** -0.5), gen(ng, 2)
    Wo, bo = gen((nc, C), 3, C ** -0.5), gen(nc, 4)
    n = M * (ng + nc)
    buf, p = guarded(1, n)
    ok(kernel=_lib().KERNEL_HEADS_OUT, x=hf, y=ho, C=C, M=M, P=HW, clips=clips, w=Wf, b=bf, ng=ng, w2=Wo, b2=bo, nc=nc, out=p)
    ref, bound = R.heads_out(hf.double(), ho.double(), clips, HW, Wf.double(), bf.double(), Wo.double(), bo.double())
    check(f"heads C={C} ({ng},{nc}) clips={clips}", body(buf, 1, n)[0].reshape(ref.shape), ref, bound)


# ================================================================================================================= refusals
def test_refusals():
    L = _lib()
    x = torch.zeros(64, 2052 + 8, device=DEV)
    o = torch.zeros(64, 2, device=DEV)
    for C, ld in [(2052, 2052), (66, 68), (64, 66)]:
        assert run(kernel=L.KERNEL_ROWSTATS, x=x, ld=ld, C=C, M=8, eps=1e-5, out=o) == -1
        assert L.lib.dawn_last_error().decode().startswith("dawn_test_kernel:")
    assert torch.all(o == 0), "a refused case launched"


# ================================================================================================================= sampler select
def _select(keys_f32, q, ddpm, n_extra_check=True):
    """runs dawn_ddim_step / dawn_ddpm_step with x = keys (signed), eps = 0 and unit coefficients, so the keys are |x| and the
    output is clamp(x, -s, s) / s; returns (x out, s, state words)"""
    L = _lib()
    x = keys_f32.to(DEV).contiguous().clone()
    n = x.numel()
    eps = torch.zeros_like(x)
    scratch = torch.zeros(n + 512, dtype=torch.int32, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    if ddpm:
        rc = L.lib.dawn_ddpm_step(p(x), p(eps), None, n, 1.0, 0.0, 1.0, 0.0, 0.0, q, p(scratch), None)
    else:
        rc = L.lib.dawn_ddim_step(p(x), p(eps), None, n, 1.0, 0.0, 1.0, 0.0, 0.0, q, p(scratch), None)
    assert rc == 0, L.lib.dawn_last_error().decode()
    torch.cuda.synchronize()
    sc = scratch[:264].cpu()
    return x.cpu(), sc[263:264].view(torch.float32).item(), sc


def _select_case(name):
    g = torch.Generator().manual_seed(hash(name) % 1000)
    rn = lambda n, s=3.0: torch.randn(n, generator=g) * s
    if name.startswith("n"):
        return rn(int(name[1:])), 0.9
    if name == "all_equal":
        return torch.full((1000,), -2.5), 0.9
    if name == "five_values":
        return torch.tensor([1.5, 2.0, 3.0, 7.0, 9.0])[torch.randint(0, 5, (10007,), generator=g)], 0.9
    if name == "le_lo_plus_1":        # 900 keys <= v[lo = 899]: v[hi] is the smallest key above it (the min_gt path)
        return torch.cat((torch.full((900,), 2.0), torch.full((100,), -5.0)))[torch.randperm(1000, generator=g)], 0.9
    if name == "le_lo_plus_2":        # 901 keys <= v[lo]: v[hi] = v[lo]
        return torch.cat((torch.full((901,), 2.0), torch.full((99,), 5.0)))[torch.randperm(1000, generator=g)], 0.9
    if name == "below_one":
        return torch.rand(5000, generator=g) * 1.98 - 0.99, 0.9
    if name == "zeros_subnormals":
        v = rn(4099)
        v[::3] = 0.0
        v[1::3] = -0.0
        v[2::7] = torch.tensor(1e-40) * torch.sign(v[2::7])
        return v, 0.9
    if name == "wide_range":
        return torch.exp(torch.rand(20011, generator=g) * 138.2 - 69.1) * torch.sign(rn(20011)), 0.9
    if name == "q_half_odd":
        return rn(10001), 0.5
    if name == "q_one":
        return rn(30000), 1.0
    if name == "q_tiny":
        return torch.exp(torch.rand(303105, generator=g) * 20) * torch.sign(rn(303105)), 1e-6
    raise KeyError(name)


SELECT_CASES = ["n1", "n2", "n255", "n256", "n257", "n28416", "n303105", "n2457600", "all_equal", "five_values", "le_lo_plus_1",
                "le_lo_plus_2", "below_one", "zeros_subnormals", "wide_range", "q_half_odd", "q_one", "q_tiny"]


@pytest.mark.parametrize("ddpm", [False, True], ids=["ddim", "ddpm"])
@pytest.mark.parametrize("name", SELECT_CASES)
def test_select(name, ddpm):
    x, q = _select_case(name)
    x = x.float()
    n = x.numel()
    out, s, sc = _select(x, q, ddpm)
    keys = np.sort(x.abs().numpy().astype(np.float64))
    rank = np.float32(q) * np.float32(n - 1)
    lo, hi = int(np.floor(rank)), int(np.ceil(rank))
    w = float(rank - np.floor(rank))
    vlo = sc[0:1].view(torch.float32).item()
    assert vlo == keys[lo], f"order statistic {lo}: {vlo!r} != {keys[lo]!r}"
    count_le = int(sc[260].item() & 0xFFFFFFFF) | (int(sc[261].item() & 0xFFFFFFFF) << 32)
    min_gt = sc[262:263].view(torch.float32).item()
    assert count_le == int(np.sum(keys <= keys[lo])), "count of keys <= v[lo]"
    vhi = vlo if (hi == lo or count_le >= lo + 2) else min_gt
    assert vhi == keys[hi], f"order statistic {hi}: {vhi!r} != {keys[hi]!r}"
    ref = max(keys[lo] + w * (keys[hi] - keys[lo]), 1.0)
    tq = max(torch.quantile(x.abs().double() if n > 16_000_000 else x.abs(), q).item(), 1.0)
    if w == 0:
        assert s == np.float32(ref), f"s {s!r} != {ref!r} at w = 0"
    else:
        assert abs(s - ref) <= np.spacing(np.float32(ref)), f"s {s!r} more than 1 ulp from {ref!r}"
    print(f"  {name}: n {n} lo {lo} hi {hi} w {w:.4g}: s {s!r}, float64 lerp {ref!r}, torch.quantile bit-equal: {s == tq}")
    want = torch.clamp(x, -s, s) / torch.tensor(s, dtype=torch.float32)
    # the update adds c * e = 0 * 0 (DDIM) or c2 * x = 0 * x (DDPM): a -0.0 quotient becomes +0.0 in DDIM as in torch
    want = want + 0.0 * x if ddpm else want * 1.0 + 0.0 * torch.zeros_like(x)
    assert torch.equal(out.view(torch.int32), want.view(torch.int32)), "clamp(x, -s, s) / s is not bit-exact"


@pytest.mark.parametrize("steps", [20, 250, 500, 999])
def test_ddim_schedule(steps):
    """first update of a real schedule (t = 952, 996, 998, 999): x = sqrt(ab) x0 + sqrt(1 - ab) e, so x0 = ca x - cb e cancels as
    in sampling; the kernel repeats torch's fp32 arithmetic bit for bit"""
    from oracle import unet_oracle as O
    L = _lib()
    t, tn = O.ddim_time_pairs(1000, steps)[0]
    acp, prev = O.cosine_alphas_cumprod()
    ca, cb = torch.sqrt(1.0 / acp)[t].item(), torch.sqrt(1.0 / acp - 1)[t].item()
    alpha, alpha_next = prev[t], prev[tn]
    sigma = ((1 - alpha / alpha_next) * (1 - alpha_next) / (1 - alpha)).sqrt()
    c = ((1 - alpha_next) - sigma ** 2).sqrt()
    sqrt_an = alpha_next.sqrt()
    n = 3 * 8 * 32 * 32
    g = torch.Generator().manual_seed(steps)
    x0 = torch.randn(n, generator=g) * 1.5
    e = torch.randn(n, generator=g)
    noise = torch.randn(n, generator=g)
    x = (torch.sqrt(acp[t]) * x0 + torch.sqrt(1 - acp[t]) * e).float()
    xd, ed, nd = x.to(DEV), e.to(DEV), noise.to(DEV)
    scratch = torch.zeros(n + 512, dtype=torch.int32, device=DEV)
    p = lambda v: ctypes.c_void_p(v.data_ptr())
    rc = L.lib.dawn_ddim_step(p(xd), p(ed), p(nd), n, ca, cb, sqrt_an.item(), c.item(), sigma.item(), 0.9, p(scratch), None)
    assert rc == 0, L.lib.dawn_last_error().decode()
    torch.cuda.synchronize()
    f = lambda v: torch.tensor(v, dtype=torch.float32)
    xr = f(ca) * x - f(cb) * e
    s = torch.quantile(xr.abs(), 0.9).clamp(min=1.0)
    ref = (xr.clamp(-s, s) / s) * f(sqrt_an.item()) + f(c.item()) * e + f(sigma.item()) * noise
    nd = int((xd.cpu().view(torch.int32) != ref.view(torch.int32)).sum())
    print(f"  ddim {steps} steps t={t}->{tn}: {nd} of {n} elements differ from torch fp32 (s = {s.item():.4g})")
    assert nd == 0
