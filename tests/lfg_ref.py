"""Float64 references of the LFG decoder's non-GEMM kernels (csrc/lfg_kernels.cu), for tests/test_lfg_kernels_gpu.py.

Each reference runs the torch operation the reference decoder uses (F.interpolate, F.grid_sample, F.conv2d, F.avg_pool2d,
torch.sigmoid) in float64 on the CPU, fed the same fp32 inputs as the kernel, and returns an elementwise bound on the kernel's
error computed from absolute values of the same data (the error model is in the test module's docstring).  Tensors are
channels-last (frames, H, W, C) like the kernels' unless noted; motion is (F, h, w, 4) = (grid_x, grid_y, occlusion, 0).
"""
import torch
import torch.nn.functional as F

U = 2.0 ** -24
TINY = 2.0 ** -126               # the smallest normal fp32


def _d(t):
    return t.detach().to("cpu", torch.float64)


def lerp_err(n_in):
    """bound on the fp32 error of one interpolation weight: src = scale * (dst + 0.5) - 0.5 has |src| <= n_in"""
    return 4 * U * (n_in + 1)


def resize_motion(motion, H, W):
    """F.interpolate(bilinear, align_corners=False) of the (F, h, w, 3) motion channels to (H, W) in float64, and a bound
    on the kernel's error per channel: the weights' rounding moves a value by at most their error times the largest step
    between neighbouring source values, and the two-level lerp rounds 6u of the largest |value|."""
    m = _d(motion)[..., :3]
    h, w = m.shape[1:3]
    if (h, w) == (H, W):
        return m, torch.zeros_like(m)
    r = F.interpolate(m.permute(0, 3, 1, 2), size=(H, W), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    step = torch.zeros(m.shape[0], 1, 1, 3, dtype=torch.float64)
    if w > 1:
        step = torch.maximum(step, (m[:, :, 1:] - m[:, :, :-1]).abs().amax(dim=(1, 2), keepdim=True))
    if h > 1:
        step = torch.maximum(step, (m[:, 1:] - m[:, :-1]).abs().amax(dim=(1, 2), keepdim=True))
    err = (lerp_err(h) + lerp_err(w)) * step + 6 * U * m.abs().amax(dim=(1, 2), keepdim=True)
    return r, err.expand_as(r).clone()


def _cell_slope(img, x0, y0):
    """max |v(x0 + 1, y) - v(x0, y)| over y in {y0, y0 + 1} of the zero-padded (H, W, C) image, per cell (..., C): the slope of the
    bilinear interpolant in x inside cell (x0, y0).  x0 / y0 are integer tensors of any value; cells off the image are 0."""
    H, W, C = img.shape
    pad = F.pad(img.permute(2, 0, 1), (2, 2, 2, 2)).permute(1, 2, 0)           # index p = coordinate + 2
    xs, ys = x0.clamp(-2, W) + 2, y0.clamp(-2, H) + 2
    a = (pad[ys, (xs + 1)] - pad[ys, xs]).abs()
    b = (pad[ys + 1, (xs + 1)] - pad[ys + 1, xs]).abs()
    return torch.maximum(a, b)


def sample_bound(img, gx, gy, dg_x, dg_y):
    """grid_sample(bilinear, zeros, align_corners=False) of one (H, W, C) image at grid points gx, gy (any shape S, fp32 values
    in float64), with grid errors dg: returns (sample (S, C), bound (S, C)).  The kernel un-normalises ix = ((gx + 1) W - 1) / 2
    in fp32 (error W / 2 dg + 4u (|ix| + W)); bilinear sampling with zero padding is continuous and piecewise bilinear, so the
    coordinate error moves the output by at most dix times the slope of every cell the error interval touches (0 off the
    image, so far-away samples get no slack); the four weighted taps round 8u of sum |w||v|."""
    H, W, C = img.shape
    ix = ((gx + 1) * W - 1) / 2
    iy = ((gy + 1) * H - 1) / 2
    dix = W / 2 * dg_x + 4 * U * (ix.abs() + W)
    diy = H / 2 * dg_y + 4 * U * (iy.abs() + H)
    out = F.grid_sample(img.permute(2, 0, 1)[None], torch.stack([gx, gy], -1).reshape(1, -1, 1, 2), mode="bilinear",
                        padding_mode="zeros", align_corners=False)[0, :, :, 0].T.reshape(*gx.shape, C)

    def fl(v):                                                                  # floor, saturated far outside the image
        return torch.floor(v.clamp(-1e6, 1e6)).long()

    xa, xb, ya, yb = fl(ix - dix), fl(ix + dix), fl(iy - diy), fl(iy + diy)
    assert ((xb - xa <= 2) | (xa >= W) | (xb < -1)).all() and ((yb - ya <= 2) | (ya >= H) | (yb < -1)).all()
    imgT = img.permute(1, 0, 2).contiguous()
    sx = torch.zeros(*gx.shape, C, dtype=torch.float64)
    sy = torch.zeros_like(sx)
    for x0 in (xa, xa + 1, xb):
        for y0 in (ya, ya + 1, yb):
            sx = torch.maximum(sx, _cell_slope(img, x0.clamp(max=xb), y0.clamp(max=yb)))
            sy = torch.maximum(sy, _cell_slope(imgT, y0.clamp(max=yb), x0.clamp(max=xb)))
    # sum |w||v| over the four taps
    x0, y0 = fl(ix), fl(iy)
    dx, dy = ix - torch.floor(ix), iy - torch.floor(iy)
    pad = F.pad(img.permute(2, 0, 1), (2, 2, 2, 2)).permute(1, 2, 0)
    absum = torch.zeros_like(sx)
    for ox, wx in ((0, 1 - dx), (1, dx)):
        for oy, wy in ((0, 1 - dy), (1, dy)):
            v = pad[(y0 + oy).clamp(-2, H + 1) + 2, (x0 + ox).clamp(-2, W + 1) + 2].abs()
            absum += (wx * wy).unsqueeze(-1).abs() * v
    bound = dix.unsqueeze(-1) * sx + diy.unsqueeze(-1) * sy + 8 * U * absum
    return out, bound


def warp_blend(skip, motion, H, W, prev=None):
    """apply_optical on one level (generator.py:71-90): out[f] = grid_sample(skip, g_f) * o_f + prev[f] * (1 - o_f), (g, o) the
    motion resized to (H, W).  skip (H, W, C); prev (F, H, W, C) or None.  Returns (out, bound)."""
    img = _d(skip)
    m, dm = resize_motion(motion, H, W)
    acc, eacc = sample_bound(img, m[..., 0], m[..., 1], dm[..., 0], dm[..., 1])
    oc, doc = m[..., 2:3], dm[..., 2:3]
    out = acc * oc
    bound = oc.abs() * eacc + doc * acc.abs() + 2 * U * out.abs()
    if prev is not None:
        p = _d(prev)
        out = out + p * (1 - oc)
        bound = bound + doc * p.abs() + 4 * U * ((acc * oc).abs() + (p * (1 - oc)).abs())
    return out, bound


def final_conv(x, weight, bias, source, motion, blend, want_deformed):
    """generator.py:163-167 and :152: 7x7 conv (Cin -> 3) + sigmoid, blended with the warped source image.  x (F, H, W, Cin);
    weight (3, Cin, 7, 7); source (3, H, W).  Returns (prediction (F, 3, H, W), bound, deformed or None, its bound).
    The fp32 accumulation of K = 49 Cin products and the bias rounds at most (K + 2) u sum |x||w| + u |b| (a worst case: the
    norm-wise check is the tight one); the sigmoid moves that by s (1 - s) and adds 4u s (expf and the division), and below a
    logit of -88.7 expf(-logit) overflows and s is 0 instead of a value under 2^-126 (TINY)."""
    xd = _d(x).permute(0, 3, 1, 2)
    wd, bd = _d(weight), _d(bias)
    K = wd.shape[1] * 49
    logit = F.conv2d(xd, wd, bd, padding=3)
    absum = F.conv2d(xd.abs(), wd.abs(), padding=3)
    s = torch.sigmoid(logit)
    es = s * (1 - s) * ((K + 2) * U * absum + U * bd.abs()[None, :, None, None]) + 4 * U * s + TINY
    deformed = edef = None
    pred, epred = s, es
    if blend or want_deformed:
        H, W = x.shape[1:3]
        m, dm = resize_motion(motion, H, W)
        img = _d(source).permute(1, 2, 0)
        deformed, edef = sample_bound(img, m[..., 0], m[..., 1], dm[..., 0], dm[..., 1])
        deformed, edef = deformed.permute(0, 3, 1, 2), edef.permute(0, 3, 1, 2)
        if blend:
            oc, doc = m[..., 2][:, None], dm[..., 2][:, None]
            pred = deformed * oc + s * (1 - oc)
            epred = (oc.abs() * edef + (1 - oc).abs() * es + doc * (deformed - s).abs()
                     + 4 * U * ((deformed * oc).abs() + (s * (1 - oc)).abs()))
    return pred, epred, deformed, edef


def conv3x3_s2_relu(x, weight, bias):
    """Face_loc_Encoder layer: relu(conv3x3 stride 2 pad 1 (x) + b), planar (Ci, H, W) -> (Co, ceil(H/2), ceil(W/2))."""
    xd, wd, bd = _d(x)[None], _d(weight), _d(bias)
    K = wd.shape[1] * 9
    y = F.relu(F.conv2d(xd, wd, bd, stride=2, padding=1))[0]
    bound = (K + 2) * U * F.conv2d(xd.abs(), wd.abs(), stride=2, padding=1)[0] + U * bd.abs()[:, None, None]
    return y, bound
