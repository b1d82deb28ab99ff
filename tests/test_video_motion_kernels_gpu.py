"""GPU: every new kernel of the LFG motion estimator (csrc/lfg_motion_kernels.cu), one at a time, against a float64 reference.

`dawn_lfg_motion_test_kernel` (include/dawn_lfg.h) runs one kernel on the test's buffers.  The references below evaluate the
reference modules' operations in float64 on the same fp32 inputs and return an elementwise bound built from absolute values of
the same data, in the manner of tests/test_lfg_kernels_gpu.py.

Error model (u = 2^-24):

* Anti-alias downsample.  169 fp32 products and sums per value: 170 u sum |w||x|.
* Region softmax and moments.  v = logit / T rounds u |v|; expf(v - m) is within 2 ulp, so each exponential carries a relative
  error e_rel = u (2 |v| + |m| + 4); the sums are fp64.  heat = e / S: 2 e_rel + u, plus 2^-126 where expf underflows.  shift = sum heat g: 2 e_rel sum heat |g|
  + u |shift|.  covar = sum heat d d^T about the fp64 mean: 2 e_rel sum heat |d_i d_j| + 2 |shift err| sum heat |d| + u |covar|.
* Flow input.  The 2x2 inverses and A_s inv(A_d) are fp64, rounded once (u of each entry).  The quadratic form
  e = (s_x i00 + s_y i10) s_x + (s_x i01 + s_y i11) s_y rounds 8 u of its absolute terms, plus the subtraction g - mu (u (|g| + |mu|)
  times the slope); exp(-e / 2) moves by G |de| / 2 + 2 u G + 2^-126 (fp32 underflow far from a region); the difference of two Gaussians adds u |heat|.  A motion coordinate
  A (g - mu_d) + mu_s rounds 8 u of its absolute terms; the background coordinate h_x / h_z rounds 6 u (sum |b||g|) / |h_z| + the same
  relative error of h_z times |h_x / h_z|.  A sample moves by the coordinate error times (W / 2 + 1) times twice the largest step
  between neighbouring source values (zeros outside), plus 8 u of sum |w||v|; far outside the image it must be exactly 0.
* Flow combine.  softmax weights carry u (|l - m| + 4) relative error each, twice; flow = sum_k mask_k m_k rounds (R + 3) u of
  sum |mask_k m_k| plus those weights' errors times |m_k|; sigmoid: s (1 - s) u |x| + 4 u s.
* Background head.  fp64 means and dot products, rounded once each: u |mean| per channel, so 2 u sum |w||mean| + 2 u |b| + u |out|.
* Norm-wise, every case: ||out - ref|| / ||ref|| <= 2^-18, 2^-15 for the sampled channels (fp32 coordinates, as warp_blend).

Every output lives in a sentinel-filled buffer with guard rows and, where the kernel takes a row stride, padding columns.

Coverage: aa_down (N 1 / 3, 128x128 / 64x192, channels written at an offset inside a wider row, cw 3 / 4 / 32); region_moments
(R 10 / 3, logits at temperature 0.1 and sharpened x8, strided logit rows, heatmap written or not); flow_input (identity-ish
and near-singular but valid covariances, affines that push grids outside [-1, 1] and far outside, bg affine / none, revert on /
off, offset rows); flow_combine (R 10 / 2, strided logits, saturated sigmoid); bg_head (C 1024 / 64, fc / identity); refusals.

The file sorts after tests/test_temporal_wg_gpu.py on purpose: that module reads kernel names from torch.profiler, which records
no device events once a pytest process is a few minutes old, so the motion tests run after it rather than before.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = 1234.5
GUARD = 8
U = 2.0 ** -24
TAU, TAU_SAMPLE = 2.0 ** -18, 2.0 ** -15


def _lib():
    from dawn_pytorch_b200 import _lib
    return _lib


def gen(shape, seed, scale=1.0, lo=None):
    g = torch.Generator().manual_seed(seed)
    if lo is not None:
        return (lo + (scale - lo) * torch.rand(shape, generator=g)).to(DEV)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def guarded(rows, ld):
    buf = torch.full((GUARD + rows + GUARD, ld), SENT, dtype=torch.float32, device=DEV)
    return buf, buf.data_ptr() + GUARD * ld * 4


def body(buf, rows, lo, hi):
    assert torch.all(buf[:GUARD] == SENT) and torch.all(buf[GUARD + rows:] == SENT), "store outside the output rows"
    b = buf[GUARD:GUARD + rows]
    assert torch.all(b[:, :lo] == SENT) and torch.all(b[:, hi:] == SENT), "store outside the row's channel range"
    return b[:, lo:hi]


def run(kernel, **kw):
    L = _lib()
    c = L.DawnLfgMotionKernelCase()
    c.kernel = kernel
    for k, v in kw.items():
        setattr(c, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    torch.cuda.synchronize()
    rc = L.lib.dawn_lfg_motion_test_kernel(ctypes.byref(c), None)
    torch.cuda.synchronize()
    return rc


def ok(rc):
    assert rc == 0, _lib().lib.dawn_last_error().decode()


WORST = {}


def check(name, out, ref, bound, tau=TAU):
    out = out.detach().double().cpu().reshape(ref.shape)
    assert torch.isfinite(out).all(), f"{name}: non-finite output"
    d = (out - ref).abs()
    el = torch.where(d == 0, torch.zeros_like(d), d / bound).max().item()
    nr = (d.norm() / ref.norm().clamp_min(1e-300)).item()
    print(f"  {name}: max |d|/bound = {el:.3g}; ||d||/||ref|| = {nr:.2e} ({nr / tau:.3g} tau)")
    WORST[name] = max(el, nr / tau)
    assert el <= 1.0, f"{name}: elementwise error {el:.2f}x the bound"
    assert nr <= tau, f"{name}: norm-wise error {nr:.2e} > {tau:.2e}"


def grid64(h, w):
    x = 2 * (torch.arange(w, dtype=torch.float32) / (w - 1)) - 1
    y = 2 * (torch.arange(h, dtype=torch.float32) / (h - 1)) - 1
    return x.double().view(1, -1).expand(h, w), y.double().view(-1, 1).expand(h, w)


def gauss_weight():
    from oracle import lfg_motion_oracle as M
    return M.anti_alias_weight().to(DEV)


# ----------------------------------------------------------------------------------------------------------- anti-alias downsample
@pytest.mark.parametrize("N,H,W,ld,off,cw", [(1, 128, 128, 4, 0, 4), (3, 64, 192, 64, 32, 32), (2, 128, 128, 8, 2, 3)])
def test_aa_down(N, H, W, ld, off, cw):
    L = _lib()
    x = gen((N, 3, H, W), 1, 1.0, lo=0.0)
    wt = gauss_weight()
    h, w = H // 4, W // 4
    buf, ptr = guarded(N * h * w, ld)
    ok(run(L.LFGM_AA_DOWN, N=N, H=H, W=W, ld=ld, off=off, cw=cw, x=x, weight=wt, out=ptr))
    got = body(buf, N * h * w, off, off + cw)
    xd, wd = x.double().cpu(), wt.double().cpu()
    pad = torch.nn.functional.pad
    ref = torch.nn.functional.conv2d(pad(xd, (6, 6, 6, 6)), wd, groups=3)[:, :, ::4, ::4]
    mag = torch.nn.functional.conv2d(pad(xd.abs(), (6, 6, 6, 6)), wd.abs(), groups=3)[:, :, ::4, ::4]
    ref = ref.permute(0, 2, 3, 1).reshape(-1, 3)
    mag = mag.permute(0, 2, 3, 1).reshape(-1, 3)
    check(f"aa_down[{N}x{H}x{W}]", got[:, :3], ref, 170 * U * mag + 1e-300)
    if cw > 3:
        assert torch.all(got[:, 3:] == 0), "padding channels must be zero"


# ----------------------------------------------------------------------------------------------------------- region moments
def moments_ref(lg, T):
    """lg (N, P, R) float32 logits -> float64 heat (N, R, P), shift, covar and their bounds"""
    N, P, R = lg.shape
    v = (lg.double() / T)
    m = v.max(dim=1, keepdim=True).values
    e = torch.exp(v - m)
    heat = (e / e.sum(dim=1, keepdim=True)).permute(0, 2, 1)
    erel = (U * (2 * v.abs() + m.abs() + 4)).permute(0, 2, 1)
    return heat, erel


@pytest.mark.parametrize("R,h,w,ldl,sharpen,with_heat", [(10, 64, 64, 16, 1.0, True), (10, 32, 32, 16, 8.0, False),
                                                         (3, 16, 48, 7, 1.0, True)])
def test_region_moments(R, h, w, ldl, sharpen, with_heat):
    L = _lib()
    N, P, T = 3, h * w, 0.1
    # smooth blobs plus noise: peaked, well-spread regions as the region predictor produces
    gx, gy = grid64(h, w)
    cx, cy = gen((N, R), 2, 0.6), gen((N, R), 3, 0.6)
    blob = -((gx.to(DEV).float()[None, None] - cx[..., None, None]) ** 2 + (gy.to(DEV).float()[None, None] - cy[..., None, None]) ** 2) * 3
    lg = ((blob + 0.05 * gen((N, R, h, w), 4)) * sharpen).permute(0, 2, 3, 1).reshape(N, P, R).contiguous()
    logits = torch.full((N, P, ldl), SENT, device=DEV)
    logits[..., :R] = lg
    sbuf, sptr = guarded(N * R, 2)
    cbuf, cptr = guarded(N * R, 4)
    hbuf, hptr = guarded(N * R, P)
    ok(run(L.LFGM_REGION_MOMENTS, N=N, h=h, w=w, R=R, ldl=ldl, temperature=T, logits=logits, out=sptr, out2=cptr,
           out3=hptr if with_heat else None))
    heat, erel = moments_ref(lg.cpu(), T)
    g = torch.stack([gx.reshape(-1), gy.reshape(-1)], dim=-1)                    # (P, 2)
    shift = torch.einsum("nrp,pk->nrk", heat, g)
    sb = 2 * torch.einsum("nrp,nrp,pk->nrk", heat, erel, g.abs()) + U * shift.abs() + 1e-300
    d = g[None, None] - shift[:, :, None]                                        # (N, R, P, 2)
    covar = torch.einsum("nrp,nrpi,nrpj->nrij", heat, d, d)
    cb = (2 * torch.einsum("nrp,nrp,nrpi,nrpj->nrij", heat, erel, d.abs(), d.abs())
          + 2 * torch.einsum("nrp,nrpi->nri", heat, d.abs())[..., None] * sb[:, :, None, :].amax(-1, keepdim=True)
          + U * covar.abs() + 1e-300)
    tag = f"R{R}_{h}x{w}_s{sharpen:g}"
    check(f"region_moments.shift[{tag}]", body(sbuf, N * R, 0, 2), shift.reshape(-1, 2), sb.reshape(-1, 2))
    check(f"region_moments.covar[{tag}]", body(cbuf, N * R, 0, 4), covar.reshape(-1, 4), cb.reshape(-1, 4))
    if with_heat:
        check(f"region_moments.heatmap[{tag}]", body(hbuf, N * R, 0, P), heat.reshape(-1, P), ((2 * erel + U) * heat).reshape(-1, P) + 2.0 ** -126)
    else:
        assert torch.all(hbuf == SENT)


# ----------------------------------------------------------------------------------------------------------- flow input
def spd(N, R, seed, lo, hi, near_singular=False):
    """symmetric positive definite (N, R, 2, 2) with eigenvalues in [lo, hi]; near_singular: condition number ~1e3"""
    th = gen((N, R), seed, 3.14159, lo=0.0).cpu().double()
    l1 = gen((N, R), seed + 1, hi, lo=lo).cpu().double()
    l2 = l1 * (1e-3 if near_singular else gen((N, R), seed + 2, 1.0, lo=0.3).cpu().double())
    c, s = torch.cos(th), torch.sin(th)
    Q = torch.stack([torch.stack([c, -s], -1), torch.stack([s, c], -1)], -2)
    D = torch.diag_embed(torch.stack([l1, l2], -1))
    return (Q @ D @ Q.transpose(-1, -2)).float()


def svd_affine(covar):
    u, s, _ = torch.svd(covar.reshape(-1, 2, 2))
    return (u @ torch.diag_embed(s ** 0.5)).reshape(covar.shape)


@pytest.mark.parametrize("tag,bg,revert,near,scale_aff", [("plain", True, True, False, 1.0), ("nobg", False, False, False, 1.0),
                                                          ("singular", True, True, True, 1.0), ("outside", True, True, False, 6.0)])
def test_flow_input(tag, bg, revert, near, scale_aff):
    L = _lib()
    N, R, h, w, ld, off, cw = 2, 10, 32, 48, 80, 8, 48
    src = gen((h, w, 4), 11, 1.0, lo=0.0)
    src[..., 3] = 0
    sh_s, sh_d = gen((N, R, 2), 12, 0.5).cpu(), gen((N, R, 2), 13, 0.5).cpu()
    cov_s, cov_d = spd(N, R, 14, 0.004, 0.08, near), spd(N, R, 17, 0.004, 0.08)
    aff_s, aff_d = svd_affine(cov_s) * scale_aff, svd_affine(cov_d)
    bgm = torch.eye(3).repeat(N, 1, 1)
    bgm[:, :2, :] += gen((N, 2, 3), 20, 0.1).cpu()
    bgm[:, 2, :2] = gen((N, 2), 21, 0.05).cpu()                                  # exercises the homogeneous division
    t = {k: v.to(DEV).contiguous() for k, v in dict(ss=sh_s, cs=cov_s, as_=aff_s, sd=sh_d, cd=cov_d, ad=aff_d, bg=bgm).items()}
    obuf, optr = guarded(N * h * w, ld)
    mbuf, mptr = guarded(N * h * w, 2 * (R + 1))
    ok(run(L.LFGM_FLOW_INPUT, N=N, h=h, w=w, R=R, ld=ld, off=off, cw=cw, revert=int(revert), source=src,
           src_shift=t["ss"], src_covar=t["cs"], src_affine=t["as_"], drv_shift=t["sd"], drv_covar=t["cd"], drv_affine=t["ad"],
           bg=t["bg"] if bg else None, out=optr, out2=mptr))
    got = body(obuf, N * h * w, off, off + cw).reshape(N, h * w, cw).cpu().double()
    mot = body(mbuf, N * h * w, 0, 2 * (R + 1)).reshape(N, h * w, R + 1, 2).cpu().double()
    assert torch.all(got[..., 4 * (R + 1):] == 0)
    gx, gy = grid64(h, w)
    g = torch.stack([gx.reshape(-1), gy.reshape(-1)], -1)                       # (P, 2)
    # Gaussians and heat
    heat, hb = [], []
    parts = {}
    for side, sh, cv in (("d", sh_d, cov_d), ("s", sh_s, cov_s)):
        inv = torch.inverse(cv.double())
        s_ = g[None, None] - sh.double()[:, :, None]                             # (N, R, P, 2)
        e = torch.einsum("nrpi,nrij,nrpj->nrp", s_, inv, s_)
        eabs = torch.einsum("nrpi,nrij,nrpj->nrp", s_.abs(), inv.abs(), s_.abs())
        slope = 2 * torch.einsum("nrpi,nrij->nrpj", s_.abs(), inv.abs()).sum(-1)    # |de/ds| times |s| scale
        G = torch.exp(-0.5 * e)
        de = 10 * U * eabs + slope * U * (g.abs().sum(-1)[None, None] + sh.double().abs().sum(-1)[..., None])
        parts[side] = (G, 0.5 * G * de + 2 * U * G)
    ref_heat = parts["d"][0] - parts["s"][0]
    hbound = parts["d"][1] + parts["s"][1] + U * ref_heat.abs() + 2 * 2.0 ** -126       # expf underflows below 2^-126
    check(f"flow_input.heat[{tag}]", got[..., 4:4 * (R + 1):4].permute(0, 2, 1), ref_heat, hbound)
    assert torch.all(got[..., 0] == 0)
    # motion grids
    A = aff_s.double() @ torch.inverse(aff_d.double())
    if revert:
        A = A * torch.sign(A[:, :, 0:1, 0:1])
    c = g[None, None] - sh_d.double()[:, :, None]                                # (N, R, P, 2)
    m = torch.einsum("nrij,nrpj->nrpi", A, c) + sh_s.double()[:, :, None]
    mb = 8 * U * (torch.einsum("nrij,nrpj->nrpi", A.abs(), c.abs() + g.abs()[None, None] + sh_d.double().abs()[:, :, None])
                  + sh_s.double().abs()[:, :, None]) + 1e-300
    hom = torch.cat([g, torch.ones_like(g[:, :1])], -1)                          # (P, 3)
    B = bgm.double() if bg else torch.eye(3, dtype=torch.float64).repeat(N, 1, 1)
    hh = torch.einsum("nij,pj->npi", B, hom)
    mbg = hh[..., :2] / hh[..., 2:3]
    habs = torch.einsum("nij,pj->npi", B.abs(), hom.abs())
    mbgb = 6 * U * (habs[..., :2] + mbg.abs() * habs[..., 2:3]) / hh[..., 2:3].abs() + 1e-300
    ref_m = torch.cat([mbg[:, None], m], 1).permute(0, 2, 1, 3)                  # (N, P, R + 1, 2)
    ref_mb = torch.cat([mbgb[:, None], mb], 1).permute(0, 2, 1, 3)
    check(f"flow_input.motion[{tag}]", mot, ref_m, ref_mb)
    # samples of the source at the kernel's own grids (bilinear, zeros, align_corners=False), the error of the grids propagated
    s3 = src[..., :3].permute(2, 0, 1).double().cpu()[None].expand(N * (R + 1), -1, -1, -1)
    samp = torch.nn.functional.grid_sample(s3, ref_m.permute(0, 2, 1, 3).reshape(N * (R + 1), h * w, 1, 2), mode="bilinear",
                                           padding_mode="zeros", align_corners=False)
    samp = samp.reshape(N, R + 1, 3, h * w).permute(0, 3, 1, 2)                   # (N, P, R + 1, 3)
    sp = torch.nn.functional.pad(src[..., :3].double().cpu(), (0, 0, 1, 1, 1, 1))
    step = max((sp[1:] - sp[:-1]).abs().max().item(), (sp[:, 1:] - sp[:, :-1]).abs().max().item())
    coord_err = ref_mb.sum(-1, keepdim=True) + 4 * U * (ref_m.abs().sum(-1, keepdim=True) + 2)
    sb = coord_err * (max(h, w) / 2 + 1) * 2 * step + 8 * U * src.abs().max().item() + 1e-300
    got_s = got[..., :4 * (R + 1)].reshape(N, h * w, R + 1, 4)[..., 1:]
    check(f"flow_input.sample[{tag}]", got_s, samp, sb.expand_as(samp), tau=TAU_SAMPLE)
    if scale_aff > 1:
        far = ref_m.abs().amax(-1) > 1 + 2.0 / min(h, w)
        assert far.any(), "the case must put grids outside [-1, 1]"
        assert torch.all(got_s[far] == 0), "samples off the image must be exactly zero"


# ----------------------------------------------------------------------------------------------------------- flow combine
@pytest.mark.parametrize("R,ldl,scale", [(10, 16, 1.0), (2, 5, 1.0), (10, 12, 40.0)])
def test_flow_combine(R, ldl, scale):
    L = _lib()
    N, h, w = 2, 24, 40
    M = N * h * w
    logits = torch.full((M, ldl), SENT, device=DEV)
    logits[:, :R + 2] = gen((M, R + 2), 30, 2.0 * scale)
    motion = gen((M, 2 * (R + 1)), 31, 1.5)
    fbuf, fptr = guarded(M, 2)
    obuf, optr = guarded(M, 1)
    ok(run(L.LFGM_FLOW_COMBINE, N=N, h=h, w=w, R=R, ldl=ldl, logits=logits, motion=motion, out=fptr, out2=optr))
    lg = logits[:, :R + 1].double().cpu()
    mx = lg.max(-1, keepdim=True).values
    e = torch.exp(lg - mx)
    mask = e / e.sum(-1, keepdim=True)
    mrel = 2 * U * ((lg - mx).abs() + 4)
    mo = motion.double().cpu().view(M, R + 1, 2)
    flow = torch.einsum("mk,mkc->mc", mask, mo)
    fb = torch.einsum("mk,mkc->mc", mask * (mrel + (R + 3) * U), mo.abs()) + 1e-300
    check(f"flow_combine.flow[R{R}_x{scale:g}]", body(fbuf, M, 0, 2), flow, fb)
    x = logits[:, R + 1].double().cpu()
    s = torch.sigmoid(x)
    ob = s * (1 - s) * U * x.abs() + 4 * U * s + 2.0 ** -126
    check(f"flow_combine.occ[R{R}_x{scale:g}]", body(obuf, M, 0, 1).reshape(-1), s, ob)


# ----------------------------------------------------------------------------------------------------------- background head
@pytest.mark.parametrize("C,h,w,ld,fc", [(1024, 8, 8, 1024, True), (64, 4, 4, 96, True), (64, 4, 4, 64, False)])
def test_bg_head(C, h, w, ld, fc):
    L = _lib()
    N, P = 3, h * w
    x = torch.full((N * P, ld), SENT, device=DEV)
    x[:, :C] = gen((N * P, C), 40, 1.0).clamp_min(0)
    fw, fb = gen((6, C), 41, C ** -0.5), gen((6,), 42, 0.1)
    buf, ptr = guarded(N, 9)
    ok(run(L.LFGM_BG_HEAD, N=N, h=h, w=w, ld=ld, cw=C, x=x, fc_w=fw if fc else None, fc_b=fb if fc else None, out=ptr))
    got = body(buf, N, 0, 9)
    ref = torch.eye(3, dtype=torch.float64).repeat(N, 1, 1)
    bound = torch.full((N, 3, 3), 1e-300, dtype=torch.float64)
    if fc:
        mean = x[:, :C].double().cpu().view(N, P, C).mean(1)
        p = mean @ fw.double().cpu().T + fb.double().cpu()
        ref[:, :2, :] = p.view(N, 2, 3)
        bound[:, :2, :] = (2 * U * (mean.abs() @ fw.double().cpu().abs().T + fb.double().cpu().abs()) + U * p.abs()).view(N, 2, 3)
    else:
        assert torch.equal(got.cpu().view(N, 3, 3).double(), ref)
        return
    check(f"bg_head[C{C}]", got, ref.reshape(N, 9), bound.reshape(N, 9))


def test_refusals():
    L = _lib()
    x = torch.zeros(64, device=DEV)
    assert run(L.LFGM_AA_DOWN, N=1, H=64, W=64, ld=4, off=2, cw=4, x=x, weight=x, out=x) == -1     # off + cw > ld
    assert run(L.LFGM_REGION_MOMENTS, N=1, h=8, w=8, R=10, ldl=8, temperature=0.1, logits=x, out=x, out2=x) == -1
    assert run(L.LFGM_FLOW_COMBINE, N=1, h=8, w=8, R=20, ldl=32, logits=x, motion=x, out=x, out2=x) == -1
    assert run(L.LFGM_FLOW_INPUT, N=1, h=8, w=8, R=10, ld=40, off=0, cw=40, source=x) == -1
    assert run(99) == -1
    assert "unknown kernel" in L.lib.dawn_last_error().decode()


def test_print_worst():
    if WORST:
        print(f"worst over the per-kernel cases: {max(WORST.values()):.3g} x bound ({max(WORST, key=WORST.get)})")
