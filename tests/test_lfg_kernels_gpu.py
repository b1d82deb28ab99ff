"""GPU: every non-GEMM kernel of the LFG flow decoder (csrc/lfg_kernels.cu), one at a time, against a float64 reference.

`dawn_lfg_test_kernel` (include/dawn_lfg.h, csrc/lfg_test.cu) runs one kernel on the test's buffers; the final conv's weight goes
through the same packer as dawn_lfg_commit_params.  `dawn_conv3x3_s2_relu` is exported already and is called directly.  The
references (tests/lfg_ref.py) run the torch operations the reference decoder uses in float64 on the same fp32 inputs and return
an elementwise bound built from absolute values of the same data.

Error model (u = 2^-24):

* Motion resize.  The kernel forms src = scale (dst + 0.5) - 0.5 and the weights in fp32: each weight is off by at most
  4u (n_in + 1), which moves a resized value by that times the largest step between neighbouring source values; the two-level
  lerp rounds 6u of the largest |value|.  Equal sizes are an exact copy.
* Grid un-normalisation.  ix = ((gx + 1) W - 1) / 2 in fp32 is off by W/2 dgx + 4u (|ix| + W).
* Sampling.  Bilinear sampling with zero padding is continuous and bilinear inside each cell, so a coordinate error d moves the
  output by at most d times the slope of every cell that [ix - d, ix + d] touches; cells off the image have slope 0, so a
  sample far outside (|g| = 10, 1e4, 1e30: the saturating int conversion) must be exactly 0.  The four weighted taps round
  8u of sum |w||v|.
* Blend.  out = s o + p (1 - o): o's error times |s| + |p|, s's error times |o|, and 4u of |s o| + |p (1 - o)|.
* Final 7x7 conv.  K = 49 Cin fp32 products and the bias: (K + 2) u sum |x||w| + u |b| on the logit, s (1 - s) of it after the
  sigmoid plus 4u s for expf and the division, plus 2^-126 where expf(-logit) overflows (logit < -88.7) and s flushes to 0;
  then the blend above with the warped source.
* Elementwise passes.  x s + t: 2u (|x s| + |t|) (ReLU is 1-Lipschitz); y + x: u |y + x|; the 2x2 mean: 3u of the mean of
  |relu(x)|; the layout transforms and motion_pack layout 0 are copies and must be exact; layout 1's (c + 1) / 2 rounds
  u (|c| + 1) / 2.
* Face_loc conv.  (9 Ci + 2) u sum |x||w| + u |b|.
* Norm-wise, on every rounding case: ||out - ref|| / ||ref|| <= 2^-18, and 2^-15 for the kernels that sample at fp32
  coordinates (warp_blend, final_conv): on white-noise features a coordinate error of a few ulp of W moves the output by a
  few ulp of W times the O(1) slope between pixels, and a non-integer resize (20x28 -> 64x96) reaches 2^-17 in an fp32
  evaluation.  An index error that moves a tap by one pixel fails both checks by orders of magnitude.

Every output lives in a sentinel-filled buffer with guard rows and, where the kernel takes a row stride, padding columns; a
case checks that they keep the sentinel.

Coverage: kernel x variant -> test.
  warp_blend        grids on pixel centres, exactly +-1, half a pixel outside, floors on -1 / 0 / W-1 / W,
                    far outside (+-10, +-1e4, +-1e30)                                        test_warp_blend[centres|pm1|edges|far]
                    occlusion 0 / 1 and outside [0, 1]                                       test_warp_blend[occ01|occ-out]
                    flow -> level: equal, 16->64, 64->256, 24->64, 20x28->64x96, 32->16      test_warp_blend[eq|up4|up2|...]
                    C 64 / 128 / 256 / 512, prev with ldp / ldo > C, F 1 / 3, a grid-stride
                    loop that wraps 5x                                                        test_warp_blend[c*|prev*|wrap]
  motion_pack       layouts 0 and 1                                                          test_motion_pack
  final_conv        40x72, Cin 64 / 128, blend on / off, deformed or not, ldx > Cin,
                    resized motion, saturated sigmoid                                        test_final_conv
  affine_relu       scale or not, in place, strided                                          test_affine_relu
  residual_bn_relu  with and without z                                                       test_residual_bn_relu
  relu_avgpool2     one frame, strided output rows (ldo > C), several frames               test_relu_avgpool2
  chw_to_hwc (padding), hwc_to_chw (strided rows)                                            test_layouts
  conv3x3_s2_relu   odd / even H, W incl. 1x1 and 127x129, Ci 1 / 3, Co 1 / 16              test_conv3x3_s2_relu
  all               refused arguments                                                        test_refusals
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from tests import lfg_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = 1234.5
GUARD = 16
TAU = 2.0 ** -18
TAU_SAMPLE = 2.0 ** -15          # kernels that sample at fp32 coordinates (see the error model)


def _lib():
    from dawn_pytorch_b200 import _lib
    return _lib


def gen(shape, seed, scale=1.0, lo=None):
    g = torch.Generator().manual_seed(seed)
    if lo is not None:
        return (lo + (scale - lo) * torch.rand(shape, generator=g)).to(DEV)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def guarded(rows, ld):
    """[GUARD + rows + GUARD][ld] sentinel buffer; returns (buffer, pointer to row 0)"""
    buf = torch.full((GUARD + rows + GUARD, ld), SENT, dtype=torch.float32, device=DEV)
    return buf, buf.data_ptr() + GUARD * ld * 4


def body(buf, rows, width):
    assert torch.all(buf[:GUARD] == SENT) and torch.all(buf[GUARD + rows:] == SENT), "store outside the output rows"
    b = buf[GUARD:GUARD + rows]
    assert torch.all(b[:, width:] == SENT), "store into the row padding"
    return b[:, :width]


def run(kernel, **kw):
    L = _lib()
    c = L.DawnLfgKernelCase()
    c.kernel = kernel
    for k, v in kw.items():
        setattr(c, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    torch.cuda.synchronize()
    rc = L.lib.dawn_lfg_test_kernel(ctypes.byref(c), None)
    torch.cuda.synchronize()
    return rc


def ok(rc):
    assert rc == 0, _lib().lib.dawn_last_error().decode()


def check(name, out, ref, bound, norm=True, tau=TAU):
    out = out.detach().double().cpu()
    assert torch.isfinite(out).all(), f"{name}: non-finite output"
    d = (out - ref).abs()
    el = torch.where(d == 0, torch.zeros_like(d), d / bound).max().item()
    nr = (d.norm() / ref.norm().clamp_min(1e-300)).item()
    print(f"  {name}: max |d|/bound = {el:.3g}; ||d||/||ref|| = {nr:.2e} ({nr / tau:.3g} tau)")
    assert el <= 1.0, f"{name}: elementwise error {el:.2f}x the bound"
    if norm:
        assert nr <= tau, f"{name}: norm-wise error {nr:.2e} > {tau:.2e}"
    return el


# ------------------------------------------------------------------------------------------------ warp_blend
def level_grid(F_, h, w, seed, mode):
    """(F, h, w, 2) sampling grid of a named kind, on the (h, w) motion grid"""
    g = torch.Generator().manual_seed(seed)
    xs = (torch.arange(w) + 0.5) / w * 2 - 1
    ys = (torch.arange(h) + 0.5) / h * 2 - 1
    ident = torch.stack(torch.meshgrid(xs, ys, indexing="xy"), -1)[None].expand(F_, h, w, 2)
    if mode == "random":
        return ident + 0.35 * (2 * torch.rand(F_, h, w, 2, generator=g) - 1)
    size = torch.tensor([w, h], dtype=torch.float32)
    if mode == "centres":                                      # integer ix: exactly on a pixel centre of the level
        return (2 * (torch.randint(0, 10 ** 6, (F_, h, w, 2), generator=g) % size) + 1) / size - 1
    if mode == "pm1":
        return torch.where(torch.rand(F_, h, w, 2, generator=g) < 0.5, -1.0, 1.0)
    if mode == "edges":                                        # ix = k + frac, floors on -2, -1, 0, W-1, W
        k = torch.tensor([-2.0, -1.0, 0.0, -1.0, 0.0])[torch.randint(0, 5, (F_, h, w, 2), generator=g)]
        hi = torch.rand(F_, h, w, 2, generator=g) < 0.5
        k = torch.where(hi, size + k, k)
        frac = torch.tensor([0.0, 0.25, 0.5, 0.75])[torch.randint(0, 4, (F_, h, w, 2), generator=g)]
        return (2 * (k + frac) + 1) / size - 1
    if mode == "far":                                          # one coordinate far outside, the other anywhere
        far = torch.tensor([10.0, -10.0, 1e4, -1e4, 1e30, -1e30])[torch.randint(0, 6, (F_, h, w, 2), generator=g)]
        near = ident + 0.35 * (2 * torch.rand(F_, h, w, 2, generator=g) - 1)
        which = torch.randint(0, 3, (F_, h, w, 1), generator=g)
        return torch.where(torch.cat([which == 0, which == 1], -1) | (which == 2), far, near)
    raise ValueError(mode)


def occlusion(F_, h, w, seed, mode):
    g = torch.Generator().manual_seed(seed)
    u = torch.rand(F_, h, w, 1, generator=g)
    return {"uniform": u, "binary": (u < 0.5).float(), "outside": u * 2 - 0.5}[mode]


WARP = {   # id: (C, H, W, h, w, F, grid, occ, prev, ldp, ldo)
    "eq": (64, 16, 16, 16, 16, 3, "random", "uniform", False, 0, 64),
    "centres": (64, 24, 20, 24, 20, 2, "centres", "uniform", False, 0, 64),
    "pm1": (64, 16, 24, 16, 24, 2, "pm1", "uniform", True, 64, 64),
    "edges": (64, 16, 24, 16, 24, 3, "edges", "uniform", True, 64, 64),
    "far": (64, 16, 16, 16, 16, 2, "far", "uniform", True, 64, 64),
    "occ01": (64, 32, 32, 16, 16, 2, "random", "binary", True, 64, 64),
    "occ-out": (64, 32, 32, 16, 16, 2, "random", "outside", True, 64, 64),
    "up4": (64, 64, 64, 16, 16, 2, "random", "uniform", True, 64, 64),
    "up2": (64, 256, 256, 128, 128, 1, "random", "uniform", True, 64, 64),
    "up4-256": (64, 256, 256, 64, 64, 1, "edges", "uniform", True, 64, 64),
    "ratio-24-64": (128, 64, 64, 24, 24, 2, "random", "uniform", True, 128, 128),
    "rect-20x28": (64, 64, 96, 20, 28, 2, "random", "uniform", True, 64, 64),
    "down-32-16": (256, 16, 16, 32, 32, 2, "random", "uniform", False, 0, 256),
    "c128": (128, 16, 16, 16, 16, 1, "random", "uniform", True, 128, 128),
    "c256": (256, 16, 16, 8, 8, 3, "random", "uniform", False, 0, 256),
    "c512": (512, 8, 8, 8, 8, 3, "random", "uniform", True, 512, 512),
    "prev-ld": (64, 32, 32, 16, 16, 3, "random", "uniform", True, 72, 80),
    "noprev-ld": (128, 16, 16, 16, 16, 1, "random", "uniform", False, 0, 136),
    "wrap": (256, 128, 128, 64, 64, 3, "random", "outside", True, 260, 264),       # 3.1M threads over a 606k-thread grid
}


@pytest.mark.parametrize("cid", list(WARP))
def test_warp_blend(cid):
    C, H, W, h, w, F_, gmode, omode, has_prev, ldp, ldo = WARP[cid]
    seed = sum(map(ord, cid))
    skip = gen((H * W, C), seed)
    motion = torch.cat([level_grid(F_, h, w, seed + 1, gmode), occlusion(F_, h, w, seed + 2, omode),
                        torch.zeros(F_, h, w, 1)], -1).contiguous().to(DEV)
    prev = None
    kw = {}
    if has_prev:
        pbuf = torch.full((F_ * H * W, ldp), SENT, device=DEV)
        prev = gen((F_ * H * W, C), seed + 3)
        pbuf[:, :C] = prev
        kw = dict(prev=pbuf, ldp=ldp)
    obuf, optr = guarded(F_ * H * W, ldo)
    ok(run(_lib().LFG_WARP_BLEND, x=skip, C=C, H=H, W=W, motion=motion, F=F_, h=h, w=w, out=optr, ldo=ldo, **kw))
    out = body(obuf, F_ * H * W, C).reshape(F_, H, W, C)
    ref, bound = R.warp_blend(skip.reshape(H, W, C), motion, H, W, None if prev is None else prev.reshape(F_, H, W, C))
    check(f"warp_blend[{cid}]", out, ref, bound, tau=TAU_SAMPLE)


def test_motion_pack():
    F_, h, w = 3, 20, 28
    flow = gen((F_, h, w, 2), 11)
    occ = gen((F_, 1, h, w), 12, 1.0, lo=0.0)
    mbuf, mptr = guarded(F_ * h * w, 4)
    ok(run(_lib().LFG_MOTION_PACK, flow=flow, occ=occ, layout=0, F=F_, h=h, w=w, out=mptr))
    m = body(mbuf, F_ * h * w, 4).reshape(F_, h, w, 4)
    assert torch.equal(m[..., :2], flow) and torch.equal(m[..., 2], occ[:, 0]) and torch.all(m[..., 3] == 0)
    sample = gen((3, F_, h, w), 13)                                            # (grid_x, grid_y, conf) as the sampler writes it
    mbuf, mptr = guarded(F_ * h * w, 4)
    ok(run(_lib().LFG_MOTION_PACK, flow=sample, layout=1, F=F_, h=h, w=w, out=mptr))
    m = body(mbuf, F_ * h * w, 4).reshape(F_, h, w, 4)
    assert torch.equal(m[..., 0], sample[0]) and torch.equal(m[..., 1], sample[1]) and torch.all(m[..., 3] == 0)
    conf = sample[2].double().cpu()
    check("motion_pack[layout 1] occlusion", m[..., 2], (conf + 1) / 2, R.U * (conf.abs() + 1) / 2 + 1e-300, norm=False)


# ------------------------------------------------------------------------------------------------ final conv
FINAL = {   # id: (Cin, ldx, F, H, W, h, w, blend, deformed, logit scale)
    "c64-blend-def": (64, 64, 2, 40, 72, 40, 72, 1, True, 1.0),
    "c128-plain": (128, 128, 1, 40, 72, 40, 72, 0, False, 1.0),
    "c64-def-only": (64, 72, 2, 40, 72, 20, 36, 0, True, 1.0),
    "c128-blend-resized": (128, 136, 2, 48, 48, 12, 12, 1, False, 1.0),
    "saturated": (64, 64, 1, 24, 40, 24, 40, 0, True, 40.0),
}


@pytest.mark.parametrize("cid", list(FINAL))
def test_final_conv(cid):
    Cin, ldx, F_, H, W, h, w, blend, want_def, scale = FINAL[cid]
    seed = sum(map(ord, cid))
    x = gen((F_ * H * W, Cin), seed, 1.0, lo=0.0)                        # post-ReLU activations
    xb = torch.full((F_ * H * W, ldx), SENT, device=DEV)
    xb[:, :Cin] = x
    weight = gen((3, Cin, 7, 7), seed + 1, scale * (3.0 / (49 * Cin)) ** 0.5)
    bias = gen(3, seed + 2, 0.1)
    source = gen((3, H, W), seed + 3, 1.0, lo=0.0)
    motion = torch.cat([level_grid(F_, h, w, seed + 4, "random"), occlusion(F_, h, w, seed + 5, "uniform"),
                        torch.zeros(F_, h, w, 1)], -1).contiguous().to(DEV)
    pbuf, pptr = guarded(F_ * 3 * H, W)
    kw = {}
    if want_def:
        dbuf, dptr = guarded(F_ * 3 * H, W)
        kw["out2"] = dptr
    ok(run(_lib().LFG_FINAL_CONV, x=xb, ldx=ldx, C=Cin, F=F_, H=H, W=W, weight=weight, bias=bias, source=source, motion=motion,
           h=h, w=w, blend=blend, out=pptr, **kw))
    pred = body(pbuf, F_ * 3 * H, W).reshape(F_, 3, H, W)
    ref, bound, dref, dbound = R.final_conv(x.reshape(F_, H, W, Cin), weight, bias, source, motion, blend, want_def)
    if scale > 1:
        sat = ((ref < 1e-6) | (ref > 1 - 1e-6)).double().mean().item()
        print(f"  {sat:.0%} of the logits saturate the sigmoid")
        assert sat > 0.2
    check(f"final_conv[{cid}] prediction", pred, ref, bound, tau=TAU_SAMPLE)
    if want_def:
        check(f"final_conv[{cid}] deformed", body(dbuf, F_ * 3 * H, W).reshape(F_, 3, H, W), dref, dbound, tau=TAU_SAMPLE)


# ------------------------------------------------------------------------------------------------ elementwise passes
@pytest.mark.parametrize("variant", ["scale-strided", "scale-inplace", "relu-inplace"])
def test_affine_relu(variant):
    C, M, ld = 128, 3001, (136 if variant == "scale-strided" else 128)
    seed = sum(map(ord, variant))
    x = gen((M, C), seed)
    s, t = (gen(C, seed + 1), gen(C, seed + 2)) if variant.startswith("scale") else (None, None)
    xb, xptr = guarded(M, ld)
    xb[GUARD:GUARD + M, :C] = x
    kw = dict(scale=s, shift=t) if s is not None else {}
    if variant.endswith("inplace"):
        ok(run(_lib().LFG_AFFINE_RELU, x=xptr, ldx=ld, C=C, M=M, out=xptr, ldo=ld, **kw))
        out = body(xb, M, C)
    else:
        obuf, optr = guarded(M, 132)
        ok(run(_lib().LFG_AFFINE_RELU, x=xptr, ldx=ld, C=C, M=M, out=optr, ldo=132, **kw))
        out = body(obuf, M, C)
        assert torch.all(body(xb, M, ld)[:, C:] == SENT)
    xd = x.double().cpu()
    if s is None:
        assert torch.equal(out.cpu(), F.relu(x).cpu())
        return
    sd, td = s.double().cpu(), t.double().cpu()
    check(f"affine_relu[{variant}]", out, F.relu(xd * sd + td), 2 * R.U * ((xd * sd).abs() + td.abs()) + 1e-300)


@pytest.mark.parametrize("with_z", [True, False])
def test_residual_bn_relu(with_z):
    C, M = 256, 2049
    y, x = gen((M, C), 21), gen((M, C), 22)
    s, t = gen(C, 23), gen(C, 24)
    nbuf, nptr = guarded(M, C)
    kw = {}
    if with_z:
        zbuf, zptr = guarded(M, C)
        kw = dict(scale=s, shift=t, out2=zptr)
    ok(run(_lib().LFG_RESIDUAL_BN_RELU, y=y, x=x, C=C, M=M, out=nptr, **kw))
    xn = y.double().cpu() + x.double().cpu()
    check("residual", body(nbuf, M, C), xn, R.U * xn.abs() + 1e-300)
    if with_z:
        sd, td = s.double().cpu(), t.double().cpu()
        bound = sd.abs() * R.U * xn.abs() + 2 * R.U * ((xn * sd).abs() + td.abs()) + 1e-300
        check("residual_bn_relu z", body(zbuf, M, C), F.relu(xn * sd + td), bound)


# (H, W, C, ldo, frames): one frame into dense rows; a strided output (the skip half of an Hourglass level); frames * H rows of
# several frames, as the motion estimator pools a batch
@pytest.mark.parametrize("shape", [(16, 16, 64, 64, 1), (40, 72, 128, 128, 1), (2, 2, 512, 512, 1), (8, 12, 64, 136, 1),
                                   (8, 12, 128, 256, 3)])
def test_relu_avgpool2(shape):
    H, W, C, ldo, n = shape
    x = gen((n * H * W, C), n * H * W + C)
    obuf, optr = guarded(n * H * W // 4, ldo)
    ok(run(_lib().LFG_RELU_AVGPOOL2, x=x, H=n * H, W=W, C=C, out=optr, ldo=ldo))
    xd = x.double().cpu().reshape(n, H, W, C).permute(0, 3, 1, 2)
    ref = F.avg_pool2d(F.relu(xd), 2).permute(0, 2, 3, 1).reshape(-1, C)
    check(f"relu_avgpool2{shape}", body(obuf, n * H * W // 4, C), ref, 3 * R.U * ref + 1e-300)


def test_layouts():
    C, H, W, Cpad = 3, 40, 72, 32
    x = gen((C, H, W), 31)
    obuf, optr = guarded(H * W, Cpad)
    ok(run(_lib().LFG_CHW_TO_HWC, x=x, C=C, H=H, W=W, Cpad=Cpad, out=optr))
    out = body(obuf, H * W, Cpad)
    assert torch.equal(out[:, :C], x.reshape(C, -1).T) and torch.all(out[:, C:] == 0)
    M, C, ld = 1000, 64, 72
    xb = gen((M, ld), 32)
    obuf, optr = guarded(C, M)
    ok(run(_lib().LFG_HWC_TO_CHW, x=xb, ldx=ld, C=C, M=M, out=optr))
    assert torch.equal(body(obuf, C, M), xb[:, :C].T)


# ------------------------------------------------------------------------------------------------ Face_loc_Encoder layer
@pytest.mark.parametrize("Ci,Co,H,W", [(1, 16, 1, 1), (3, 1, 1, 1), (1, 16, 2, 2), (3, 16, 127, 129), (1, 1, 127, 129),
                                       (3, 16, 64, 64), (1, 16, 5, 4)])
def test_conv3x3_s2_relu(Ci, Co, H, W):
    seed = Ci * 1000 + Co * 100 + H + W
    x = gen((Ci, H, W), seed, 1.0, lo=0.0)
    wgt, b = gen((Co, Ci, 3, 3), seed + 1, 0.5), gen(Co, seed + 2, 0.1)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    obuf, optr = guarded(Co * Ho, Wo)
    _lib().check(_lib().lib.dawn_conv3x3_s2_relu(x.data_ptr(), Ci, H, W, wgt.data_ptr(), b.data_ptr(), Co, optr, None),
                 "dawn_conv3x3_s2_relu")
    torch.cuda.synchronize()
    ref, bound = R.conv3x3_s2_relu(x, wgt, b)
    check(f"conv3x3_s2_relu[{Ci},{Co},{H}x{W}]", body(obuf, Co * Ho, Wo).reshape(Co, Ho, Wo), ref, bound + 1e-300)


def test_refusals():
    L = _lib()
    t = torch.zeros(4096, device=DEV)
    cases = [
        (L.LFG_WARP_BLEND, dict(x=t, C=64, H=4, W=4, F=1, h=4, w=4, out=t, ldo=64)),                 # no motion
        (L.LFG_WARP_BLEND, dict(x=t, motion=t, C=66, H=4, W=4, F=1, h=4, w=4, out=t, ldo=66)),       # C % 4
        (L.LFG_WARP_BLEND, dict(x=t, motion=t, C=64, H=4, W=4, F=1, h=4, w=4, out=t, ldo=60)),       # ldo < C
        (L.LFG_WARP_BLEND, dict(x=t, motion=t, prev=t, ldp=62, C=64, H=4, W=4, F=1, h=4, w=4, out=t, ldo=64)),
        (L.LFG_FINAL_CONV, dict(x=t, ldx=60, C=60, F=1, H=4, W=4, h=4, w=4, weight=t, bias=t, out=t)),  # Cin % 8
        (L.LFG_FINAL_CONV, dict(x=t, ldx=64, C=64, F=1, H=4, W=4, h=4, w=4, weight=t, bias=t, out=t, blend=1)),  # no source
        (L.LFG_AFFINE_RELU, dict(x=t, ldx=64, C=64, M=4, out=t, ldo=64, scale=t)),                   # scale without shift
        (L.LFG_RELU_AVGPOOL2, dict(x=t, H=1, W=4, C=64, out=t, ldo=64)),
        (L.LFG_RELU_AVGPOOL2, dict(x=t, H=4, W=4, C=64, out=t, ldo=60)),                             # ldo < C
        (L.LFG_CHW_TO_HWC, dict(x=t, C=8, H=4, W=4, Cpad=4, out=t)),
        (L.LFG_MOTION_PACK, dict(flow=t, layout=0, F=1, h=4, w=4, out=t)),                          # layout 0 without occ
        (L.LFG_MOTION_PACK, dict(flow=t, occ=t, layout=2, F=1, h=4, w=4, out=t)),
        (99, {}),
    ]
    for k, kw in cases:
        assert run(k, **kw) == -1, (k, kw)
        assert "dawn_lfg_test_kernel" in L.lib.dawn_last_error().decode()
    assert L.lib.dawn_lfg_test_kernel(None, None) == -1
