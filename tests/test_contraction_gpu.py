"""GPU: every wgmma / mma.sync contraction path, one kernel at a time, against a float64 reference of the same operation.

`dawn_test_contraction` (include/dawn_unet.h) runs one contraction through exactly one kernel path with the weight image and
accumulator scale the network builds; a path that refuses the geometry returns -1 and launches nothing.  Each reference is
defined from the operation (conv2d, conv_transpose2d, LayerNorm, rotary, softmax, cosine-similarity gate, GroupNorm) in
float64, on the GPU for the large cases and on the CPU for the small ones.

Tolerance, derived from the split arithmetic (u = 2^-24, the fp32 unit roundoff):

* Split.  A is split into hi = x rounded to 11 significant bits and lo = fp16(x - hi); B (pre-scaled by a power of two) into
  hi = fp16(w), lo = fp16(w - hi).  |x - hi - lo| <= 2^-11 |x - hi| <= 2^-22 |x|, the same for w.  The products hi*hi, hi*lo,
  lo*hi are exact in fp32; the dropped lo*lo and the two lo roundings leave |ab - sum| <= 3 * 2^-22 |a||b| per product.
  (fp16 subnormal lo pieces add at most 2^-25 |b| per product: the `tiny` term.)
* Accumulation.  Inside a drain interval of Kc products the tensor core adds with truncation, at most one ulp of the partial
  sum per product: <= Kc * 2^-23 * S, S = sum |a||b|.  The K/Kc drains and the epilogue's bias / residual adds round to
  nearest: <= (K/Kc + 4) u S.  The mma.sync kernel drains every 8 products (Kc = 8).
  => elementwise:  |d| <= c1 * S + c2 * |ref| + tiny,  c1 = 3 * 2^-22 + Kc * 2^-23 + (K/Kc + 4) * 2^-24,  c2 = 8u.
  A wrong tap, row, window or chunk gives an error of order |ref| ~ S / sqrt(K), 30x to 1000x above c1 * S for K <= 9216.
* Norm-wise.  With R = sqrt(sum a^2 b^2) (for zero-mean operands ||R|| = ||ref|| up to sampling), independent per-product
  errors of rms rho give ||d|| / ||R|| ~ rho.  The 3-term split has rho <= 2^-22; truncation inside a drain interval adds a
  bias of at most about Kc * 2^-24 of the partial sums.  Bound:  ||d|| / ||R|| <= tau = 2^-20 + Kc * 2^-24
  (1.6e-5 at the GEMM's default Kc = 256, 3.5e-5 at the halo conv's Kc = 576).  A 2-term split (one cross term missing)
  leaves |x - hi| ~ 2^-12 |x| in every product, rho ~ 1.5e-4, and 1xTF32 / 1xFP16 rho ~ 2.5e-4: both miss tau by 4x to 15x.
  Measured on an H100 80GB HBM3 (400 W): ||d|| / ||R|| = 2.6e-7 (Kc = 64), 9.3e-7 (Kc = 256), 2.0e-6 (Kc = 576), about
  0.06 tau; with the hi*lo term removed from the wgmma issue loops every wgmma case fails this check.
  The norm is taken over R rather than ref so that a LayerNorm fold over rows whose mean is many standard deviations
  (where the contraction cancels) is held to the conditioning of the data, not to a smaller number it cannot meet.
* Accumulation bias.  All-positive operands at K = 9216: truncation shrinks every partial sum, so the mean signed relative error
  grows with the drain interval.  The one-ulp-per-product model above gives -Kc * 2^-24 (1.5e-5 at the GEMM's default Kc = 256)
  and -K * 2^-24 (5.5e-4) without drains; on an H100 80GB HBM3 (400 W) the truncation was ~8x smaller: -1.7e-6 (GEMM, default
  drain), -3.6e-6 (halo conv, default drain) and -7.6e-5 with the GEMM's drains removed.  The check is |mean| <= 2^-16 (1.5e-5),
  4x above the default drains and 5x below no drain.
* LayerNorm statistics.  A numerically stable fp32 mean / variance of a row of K values is within (K/8 + 3) u of the float64
  value, relative to mean |x| (mean) and to the variance (rstd, halved); the bound adds the resulting |mu error| * |wsum| * rstd
  and (K/8 + 3) u |ref|.  One-pass E[x^2] - mu^2 in fp32 loses (mu / sigma)^2 u of the variance: at mu = 100 sigma that is
  far above this bound, which is what the large-mean rows test.  (The wgmma producers' inline statistics were one-pass and
  reached 0.995 of this bound at K = 64; they now sum each row shifted by its first element and sit at 0.14.)
* GroupNorm partial sums: the sum of the elementwise bounds plus 72 u sum |ref| (the kernels add <= 72 fp32 partials
  before the fp64 atomics); a tile that is missed or counted twice is off by a whole tile's sum.

Coverage: path x epilogue x producer -> test.
  path              epilogue            producer / variant                      test
  MMA_SYNC          PLAIN               gather, M < 128, stats, per-frame B      test_plain[mma-*], test_sla_outproj_per_frame_b
  MMA_SYNC          GN_APPLY            gather, per-frame B, FiLM               test_gn_apply_mma
  MMA_SYNC          QKV_TEMPORAL/SLA/MID/CA_GATE  rowstats                      test_layernorm_epilogues[mma-*]
  TC_GEMM           PLAIN               gather; 1x1, kxk, down, up parities,    test_plain[tc-*], test_transposed_conv_parities,
                                        perm_out, residual, stats, drain          test_perm_out_drops_halo_frames, test_gemm_drain
  TC_GEMM_PRESPLIT  PLAIN               cp.async, 3x3 at 8x8, K 4608 / 9216      test_plain[presplit-*]
  TC_GEMM           QKV_TEMPORAL/SLA/MID/CA_GATE  inline stats / rowstats      test_layernorm_epilogues[tc-*]
  TC_GEMM_PRESPLIT  QKV_TEMPORAL/SLA/MID  rowstats (N 768)                     test_layernorm_epilogues[presplit-*]
  TC_CONV3          PLAIN               gather, stats deferred / per tile, up2   test_conv3[gather-*], test_conv3_up2
  TC_CONV3_TMA      PLAIN               TMA, stats deferred / per tile, up2      test_conv3[tma-*], test_conv3_up2
  all               PLAIN               all-positive K = 9216                    test_accumulation_bias
  all               -                   refused geometries                       test_refusals
"""
import ctypes
import math
import zlib

import pytest
import torch
import torch.nn.functional as TF

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SPLIT = 3 * 2.0 ** -22
SENT = 1234.5                     # sentinel in Out padding columns and guard rows
GUARD = 64                        # guard rows before and after the output region
DEV = "cuda"


def _lib():
    from dawn_pytorch_b200 import _lib
    return _lib


def kc_of(path, K, Cin, drain):
    """products accumulated inside the tensor core before a round-to-nearest drain"""
    if path == "mma":
        return 8
    if path in ("conv3", "tma"):
        return (drain if drain in (1, 3) else 9) * 64                # taps of one 64-channel chunk
    return (drain if 0 < drain < 4 else 4) * 64


def c1_tau(path, K, Cin, drain):
    kc = min(kc_of(path, K, Cin, drain), K)
    c1 = SPLIT + kc * 2.0 ** -23 + (K / kc + 4) * U
    tau = 2.0 ** -20 + kc * U
    return c1, tau


PATHS = {"mma": 0, "tc": 1, "presplit": 2, "conv3": 3, "tma": 4}


# ------------------------------------------------------------------------------------------------ operands and the entry
def gen(shape, seed, dist="normal", device=DEV):
    g = torch.Generator().manual_seed(seed)
    if dist == "normal":
        t = torch.randn(shape, generator=g)
    else:                                             # all positive
        t = 0.5 + 0.5 * torch.rand(shape, generator=g)
    return t.to(device)


def padded(x2d, ld, fill):
    """rows of x2d (float32) in a [rows][ld] buffer, columns >= x2d.shape[1] set to fill"""
    buf = torch.full((x2d.shape[0], ld), fill, dtype=torch.float32, device=DEV)
    buf[:, :x2d.shape[1]] = x2d.float()
    return buf


def run_case(path, epi, geo, A2d, Bkn, N, out_rows, ldo, **kw):
    """fill a dawn_contraction_case, guard the output, run; returns (rc, out view [out_rows][N], buffers)"""
    L = _lib()
    c = L.DawnContractionCase()
    c.path, c.epi = PATHS[path], epi
    for k, v in geo.items():
        if k in ("dy", "dx"):
            for i, d in enumerate(v):
                getattr(c, k)[i] = d
        else:
            setattr(c, k, v)
    c.ntaps = len(geo["dy"])
    c.N, c.ldb, c.ldo = N, Bkn.shape[1], ldo
    c.A, c.B = A2d.data_ptr(), Bkn.data_ptr()
    obuf = torch.full((GUARD + out_rows + GUARD, ldo), SENT, dtype=torch.float32, device=DEV)
    c.Out = obuf.data_ptr() + GUARD * ldo * 4
    keep = []
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            keep.append(v)
            setattr(c, k, v.data_ptr())
        else:
            setattr(c, k, v)
    if c.q_post_scale == 0:
        c.q_post_scale = 1.0
    torch.cuda.synchronize()
    rc = L.lib.dawn_test_contraction(ctypes.byref(c), None)
    torch.cuda.synchronize()
    return rc, obuf, c


def check_guards(obuf, out_rows, N, written_rows=None):
    """padding columns and guard rows keep the sentinel; `written_rows` (bool mask) are the rows the kernel owns"""
    body = obuf[GUARD:GUARD + out_rows]
    assert torch.all(obuf[:GUARD] == SENT) and torch.all(obuf[GUARD + out_rows:] == SENT), "store outside the output rows"
    assert torch.all(body[:, N:] == SENT), "store into the ldo padding"
    if written_rows is not None:
        assert torch.all(body[~written_rows] == SENT), "store into a dropped row"
    return body[:, :N]


def check(name, out, ref, S, R, c1, tau, tiny=0.0, c2=8 * U, extra=None, norm=True):
    """elementwise |d| <= c1 S + c2 |ref| + tiny (+ extra); norm-wise ||d|| / ||R|| <= tau; prints the margins"""
    out = out.double()
    assert torch.isfinite(out).all(), f"{name}: non-finite output"
    d = (out - ref).abs()
    bound = c1 * S + c2 * ref.abs() + tiny
    if extra is not None:
        bound = bound + extra
    el = (d / bound).max().item()
    nr = (d.norm() / R.norm()).item()
    print(f"  {name}: elementwise max |d|/bound = {el:.3f}; ||d||/||R|| = {nr:.2e} (tau {tau:.1e}, {nr / tau:.3f} of it); "
          f"||d||/||ref|| = {(d.norm() / ref.norm()).item():.2e}")
    assert el <= 1.0, f"{name}: elementwise error {el:.2f}x the bound"
    if norm:
        assert nr <= tau, f"{name}: norm-wise error {nr:.2e} > {tau:.2e}"


def check_stats(name, stats, ref, bnd, cpg):
    """GroupNorm partial sums (double[16]) against float64 group sums of ref within the summed elementwise bound"""
    N = ref.shape[1]
    G = N // cpg
    want = torch.zeros(16, dtype=torch.float64, device=ref.device)
    tol = torch.zeros(16, dtype=torch.float64, device=ref.device)
    for g in range(G):
        r, b = ref[:, g * cpg:(g + 1) * cpg], bnd[:, g * cpg:(g + 1) * cpg]
        want[2 * g], want[2 * g + 1] = r.sum(), (r * r).sum()
        tol[2 * g] = b.sum() + 72 * U * r.abs().sum()
        tol[2 * g + 1] = (2 * r.abs() * b + b * b).sum() + 72 * U * (r * r).sum()
    err = ((stats.to(want.device) - want).abs() / tol)[:2 * G].max().item()
    print(f"  {name}: GroupNorm sums max |d|/bound = {err:.3f}")
    assert err <= 1.0, f"{name}: GroupNorm partial sums off by {err:.1f}x the bound"
    assert torch.all(stats[2 * G:] == 0)


# ------------------------------------------------------------------------------------------------ conv geometry helpers
def square_taps(k):
    p = k // 2
    return [ky - p for ky in range(k) for kx in range(k)], [kx - p for ky in range(k) for kx in range(k)]


def conv_weight_to_B(Wc, ldb):
    """conv2d weight (N, Cin, kh, kw) -> [(ky*kw + kx)*Cin + c][ldb]"""
    N, Cin, kh, kw = Wc.shape
    B = torch.zeros(kh * kw * Cin, ldb, dtype=torch.float32, device=Wc.device)
    B[:, :N] = Wc.permute(2, 3, 1, 0).reshape(kh * kw * Cin, N)
    return B


def up_taps(parity):
    """ConvTranspose2d(4, stride 2, padding 1): output 2i + parity takes input i + d through kernel row k, 2(i + d) - 1 + k = 2i + parity"""
    return [(k, (parity + 1 - k) // 2) for k in range(4) if (parity + 1 - k) % 2 == 0]


def conv_ref(x, w, op, **kw):
    """float64 op(x, w), S = op(|x|, |w|), R = sqrt(op(x^2, w^2)) for an op linear in both operands"""
    x, w = x.double(), w.double()
    return op(x, w, **kw), op(x.abs(), w.abs(), **kw), op(x * x, w * w, **kw).sqrt()


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def plain_problem(F, H, W, Cin, N, ksize, seed, lda=None, ref_dev=DEV, dist="normal"):
    """k x k same conv (1x1 = GEMM) on an (F, H, W, Cin) activation; returns A2d (lda padding NaN), B, ref pieces"""
    lda = lda or Cin
    x = gen((F, H, W, Cin), seed, dist)
    Wc = gen((N, Cin, ksize, ksize), seed + 1, dist) / math.sqrt(Cin * ksize * ksize)
    A2d = padded(x.reshape(-1, Cin), lda, float("nan"))
    B = conv_weight_to_B(Wc, (N + 63) // 64 * 64)
    ref, S, R = conv_ref(x.to(ref_dev).permute(0, 3, 1, 2), Wc.to(ref_dev), TF.conv2d, padding=ksize // 2)
    return A2d, B, nhwc(ref), nhwc(S), nhwc(R)


def tiny_of(A2d, B, Cin):
    """fp16-subnormal lo pieces: <= 2^-25 |b| per product (activations), <= 2^-36 max|B| |a| (scaled weights)"""
    return 2.0 ** -24 * B.double().abs().sum(0).max().item() + 2.0 ** -35 * B.abs().max().item() * Cin * 4


# ------------------------------------------------------------------------------------------------ PLAIN: GEMM / conv paths
PLAIN_CASES = [
    # id, path, F, H, W, Cin, N, k, extras
    ("tc-1x1-64-64-m128", "tc", 2, 8, 8, 64, 64, 1, {}),
    ("tc-1x1-64-64-m243-res-lda-ldo", "tc", 3, 9, 9, 64, 64, 1, dict(lda=96, ldo=72, res=True, stats=True)),
    ("tc-1x1-256-512", "tc", 4, 16, 16, 256, 512, 1, dict(stats=True)),
    ("tc-1x1-64-64-many-tiles", "tc", 1, 152064 + 100, 1, 64, 64, 1, dict(stats=True, res=True)),
    ("tc-1x1-64-128-many-tiles", "tc", 1, 9 * 132 * 128 * 2 + 17, 1, 64, 128, 1, dict(stats=True)),
    ("tc-3x3-8x8-512", "tc", 8, 8, 8, 512, 512, 3, dict(stats=True)),
    ("tc-3x3-8x8-1024", "tc", 4, 8, 8, 1024, 512, 3, {}),
    ("presplit-3x3-8x8-512", "presplit", 8, 8, 8, 512, 512, 3, dict(stats=True)),
    ("presplit-3x3-8x8-1024", "presplit", 4, 8, 8, 1024, 512, 3, dict(stats=True)),
    ("tc-3x3-gn-192", "tc", 3, 9, 9, 64, 192, 3, dict(stats=True)),
    ("tc-3x3-gn-128-ragged", "tc", 3, 9, 9, 128, 128, 3, dict(stats=True, res=True)),
    ("tc-7x7-16x16", "tc", 2, 16, 16, 64, 64, 7, dict(stats=True)),
    ("mma-1x1-m100", "mma", 1, 100, 1, 64, 64, 1, dict(stats=True, res=True, lda=68, ldo=66)),
    ("mma-3x3-96", "mma", 2, 9, 9, 96, 128, 3, dict(stats=True)),
    ("mma-3x3-8x8-1024", "mma", 2, 8, 8, 1024, 256, 3, dict(stats=True)),
]


@pytest.mark.parametrize("cid,path,F,H,W,Cin,N,k,ex", PLAIN_CASES, ids=[c[0] for c in PLAIN_CASES])
def test_plain(cid, path, F, H, W, Cin, N, k, ex):
    seed = zlib.crc32(cid.encode()) % 100000
    lda, ldo = ex.get("lda", Cin), ex.get("ldo", N)
    A2d, B, ref, S, R = plain_problem(F, H, W, Cin, N, k, seed, lda=lda)
    M = F * H * W
    ref, S, R = ref.reshape(M, N), S.reshape(M, N), R.reshape(M, N)
    bias = gen((B.shape[1],), seed + 2)
    ref = ref + bias[:N].double()
    kw = dict(bias=bias)
    if ex.get("res"):
        res = gen((M, N), seed + 3)
        resb = padded(res, ldo + 4, float("nan"))
        kw.update(Res=resb, ldr=ldo + 4)
        ref = ref + res.double()
    stats = None
    if ex.get("stats"):
        stats = torch.zeros(16, dtype=torch.float64, device=DEV)
        kw.update(stats=stats, cpg=N // 8)
    dy, dx = square_taps(k)
    geo = dict(F=F, IH=H, IW=W, Cin=Cin, lda=lda, dy=dy, dx=dx, in_stride=1, OHs=H, OWs=W, OH=H, OW=W, out_stride=1)
    rc, obuf, _ = run_case(path, 0, geo, A2d, B, N, M, ldo, **kw)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    out = check_guards(obuf, M, N)
    K = k * k * Cin
    c1, tau = c1_tau(path, K, Cin, 0)
    tiny = tiny_of(A2d, B, Cin)
    check(cid, out, ref, S, R, c1, tau, tiny)
    if stats is not None:
        check_stats(cid, stats, ref, c1 * S + 8 * U * ref.abs() + tiny, N // 8)


@pytest.mark.parametrize("drain", [1, 3, 0, 7])
def test_gemm_drain(drain):
    """the drain interval (1, 3, the default 4 panels; 7 means the default) with K = 2304 on a ragged M"""
    F, H, W, Cin, N = 5, 7, 7, 256, 64
    A2d, B, ref, S, R = plain_problem(F, H, W, Cin, N, 3, 40 + drain)
    M = F * H * W
    ref, S, R = ref.reshape(M, N), S.reshape(M, N), R.reshape(M, N)
    dy, dx = square_taps(3)
    geo = dict(F=F, IH=H, IW=W, Cin=Cin, lda=Cin, dy=dy, dx=dx, in_stride=1, OHs=H, OWs=W, OH=H, OW=W, out_stride=1, drain=drain)
    rc, obuf, _ = run_case("tc", 0, geo, A2d, B, N, M, N)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    c1, tau = c1_tau("tc", 9 * Cin, Cin, drain)
    check(f"drain={drain}", check_guards(obuf, M, N), ref, S, R, c1, tau, tiny_of(A2d, B, Cin))


@pytest.mark.parametrize("path,H", [("tc", 16), ("tc", 24), ("mma", 24), ("presplit", 32)])
def test_down_conv(path, H):
    """Downsample: 4x4 stride-2 conv, padding 1 (H = 24: odd number of 8-row output blocks)"""
    F, W, Cin, N = 3, H, 128, 128
    x = gen((F, H, W, Cin), 7 + H)
    Wc = gen((N, Cin, 4, 4), 8 + H) / math.sqrt(16 * Cin)
    A2d, B = x.reshape(-1, Cin).contiguous(), conv_weight_to_B(Wc, N)
    ref, S, R = (nhwc(t).reshape(-1, N) for t in conv_ref(x.permute(0, 3, 1, 2), Wc, TF.conv2d, stride=2, padding=1))
    bias = gen((N,), 9)
    ref = ref + bias.double()
    dy = [ky - 1 for ky in range(4) for kx in range(4)]
    dx = [kx - 1 for ky in range(4) for kx in range(4)]
    OH = H // 2
    geo = dict(F=F, IH=H, IW=W, Cin=Cin, lda=Cin, dy=dy, dx=dx, in_stride=2, OHs=OH, OWs=OH, OH=OH, OW=OH, out_stride=1)
    stats = torch.zeros(16, dtype=torch.float64, device=DEV)
    rc, obuf, _ = run_case(path, 0, geo, A2d, B, N, F * OH * OH, N, bias=bias, stats=stats, cpg=N // 8)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    c1, tau = c1_tau(path, 16 * Cin, Cin, 0)
    tiny = tiny_of(A2d, B, Cin)
    out = check_guards(obuf, F * OH * OH, N)
    check(f"down {path} H={H}", out, ref, S, R, c1, tau, tiny)
    check_stats(f"down {path} H={H}", stats, ref, c1 * S + 8 * U * ref.abs() + tiny, N // 8)


def up_problem(F, H, W, C, seed):
    x = gen((F, H, W, C), seed)
    Wt = gen((C, C, 4, 4), seed + 1) / math.sqrt(4 * C)          # ConvTranspose2d weight (in, out, kh, kw)
    bias = gen((C,), seed + 2)
    ref, S, R = (nhwc(t) for t in conv_ref(x.permute(0, 3, 1, 2), Wt, TF.conv_transpose2d, stride=2, padding=1))
    return x, Wt, bias, ref + bias.double(), S, R


@pytest.mark.parametrize("path", ["tc", "mma"])
def test_transposed_conv_parities(path):
    """ConvTranspose2d(4, 2, 1) as four 2x2-tap GEMMs, one per output parity class, interleaved into one output (out_stride 2)"""
    F, H, W, C = 4, 12, 16, 128
    x, Wt, bias, ref, S, R = up_problem(F, H, W, C, 77)
    A2d = x.reshape(-1, C).contiguous()
    obuf = None
    out_rows = F * 2 * H * 2 * W
    for py in range(2):
        for px in range(2):
            ty, tx = up_taps(py), up_taps(px)
            dy = [d for (_, d) in ty for _ in tx]
            dx = [d for _ in ty for (_, d) in tx]
            B = torch.zeros(4 * C, C, device=DEV)
            for t, ((ky, _), (kx, _)) in enumerate((a, b) for a in ty for b in tx):
                B[t * C:(t + 1) * C] = Wt[:, :, ky, kx]
            geo = dict(F=F, IH=H, IW=W, Cin=C, lda=C, dy=dy, dx=dx, in_stride=1, OHs=H, OWs=W, OH=2 * H, OW=2 * W,
                       out_stride=2, oy0=py, ox0=px)
            rc, ob, _ = run_case(path, 0, geo, A2d, B, C, out_rows, C, bias=bias)
            assert rc == 0, _lib().lib.dawn_last_error().decode()
            cls = torch.zeros(F, 2 * H, 2 * W, dtype=torch.bool, device=DEV)
            cls[:, py::2, px::2] = True
            body = check_guards(ob, out_rows, C, written_rows=cls.reshape(-1))
            obuf = body.clone() if obuf is None else torch.where(cls.reshape(-1, 1), body, obuf)
    c1, tau = c1_tau(path, 4 * C, C, 0)
    check(f"up parities {path}", obuf, ref.reshape(out_rows, C), S.reshape(out_rows, C), R.reshape(out_rows, C), c1, tau,
          tiny_of(A2d, Wt.reshape(C, -1).t(), C))


# ------------------------------------------------------------------------------------------------ sequence-blocked order
def seq_blocked_rows(F, P, pb):
    """pixel f * P + p of each row m, where row m = ((p // pb) * F + f) * pb + p % pb  (from the definition, not the kernel)"""
    pix = torch.empty(F * P, dtype=torch.long)
    for f in range(F):
        p = torch.arange(P)
        m = ((p // pb) * F + f) * pb + p % pb
        pix[m] = f * P + p
    return pix


def seq_block(P):
    return next(b for b in range(16, 0, -1) if P % b == 0)


@pytest.mark.parametrize("path,P,Fe,hl,F", [("tc", 4096, 12, 2, 8), ("tc", 36, 50, 20, 10), ("tc", 9, 90, 40, 10),
                                             ("mma", 36, 50, 20, 10), ("presplit", 4096, 6, 1, 4)])
def test_perm_out_drops_halo_frames(path, P, Fe, hl, F):
    """attention out-projection: rows in sequence-blocked order over Fe frames, scattered to the F own frames (+ residual);
    rows of the halo frames are dropped"""
    pb = seq_block(P)
    assert pb == {4096: 16, 36: 12, 9: 9}[P]
    Me, C, N = Fe * P, 256, 64
    o = gen((Me, C), P + Fe)
    Wl = gen((C, N), P + Fe + 1) / math.sqrt(C)
    bias, res = gen((N,), 5), gen((F * P, N), 6)
    pix = seq_blocked_rows(Fe, P, pb).to(DEV)                     # input pixel (f * P + p over Fe frames) of row m
    f_of = pix // P
    keep = (f_of >= hl) & (f_of < hl + F)
    dst = (pix - hl * P)[keep]
    ref_rows, S_rows, R_rows = conv_ref(o, Wl, torch.matmul)
    ref = torch.empty(F * P, N, dtype=torch.float64, device=DEV)
    S, R = torch.empty_like(ref), torch.empty_like(ref)
    ref[dst], S[dst], R[dst] = ref_rows[keep], S_rows[keep], R_rows[keep]
    ref = ref + bias.double() + res.double()
    ldo = 72
    geo = dict(F=1, IH=Me, IW=1, Cin=C, lda=C, dy=[0], dx=[0], in_stride=1, OHs=Me, OWs=1, OH=Me, OW=1, out_stride=1,
               perm_pb=pb, perm_F=Fe, perm_in=0, perm_out=1, perm_f_lo=hl, perm_f_hi=hl + F, P=P)
    rc, obuf, _ = run_case(path, 0, geo, o, Wl.contiguous(), N, F * P, ldo, bias=bias, Res=padded(res, ldo, float("nan")), ldr=ldo)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    c1, tau = c1_tau(path, C, C, 0)
    check(f"perm_out {path} P={P}", check_guards(obuf, F * P, N), ref, S, R, c1, tau, tiny_of(o, Wl, C))


# ------------------------------------------------------------------------------------------------ halo-tile 3x3 conv
CONV3_CASES = [  # path, F, H, W, Cin, N, drain
    ("conv3", 40, 64, 64, 64, 64, 0), ("tma", 40, 64, 64, 64, 64, 0),
    ("conv3", 6, 48, 40, 128, 128, 3), ("tma", 6, 48, 40, 128, 128, 1),
    ("conv3", 24, 16, 8, 256, 256, 0), ("tma", 24, 16, 8, 512, 256, 9),
    ("conv3", 12, 16, 16, 512, 512, 1), ("tma", 12, 16, 16, 128, 512, 3),
    ("conv3", 30, 16, 16, 64, 128, 9), ("tma", 10, 48, 40, 64, 256, 0),
]


@pytest.mark.parametrize("path,F,H,W,Cin,N,drain", CONV3_CASES,
                         ids=[f"{'gather' if c[0] == 'conv3' else 'tma'}-{c[2]}x{c[3]}-{c[4]}-{c[5]}-d{c[6]}" for c in CONV3_CASES])
def test_conv3(path, F, H, W, Cin, N, drain):
    seed = F * 7 + H + Cin + N + drain
    A2d, B, ref, S, R = plain_problem(F, H, W, Cin, N, 3, seed, lda=Cin if path == "tma" else Cin + 4)
    M = F * H * W
    ref, S, R = ref.reshape(M, N), S.reshape(M, N), R.reshape(M, N)
    bias = gen((N,), seed + 2)
    ref = ref + bias.double()
    stats = torch.zeros(16, dtype=torch.float64, device=DEV)
    dy, dx = square_taps(3)
    geo = dict(F=F, IH=H, IW=W, Cin=Cin, lda=A2d.shape[1], dy=dy, dx=dx, in_stride=1, OHs=H, OWs=W, OH=H, OW=W, out_stride=1,
               drain=drain)
    rc, obuf, _ = run_case(path, 0, geo, A2d, B, N, M, N + 8, bias=bias, stats=stats, cpg=N // 8)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    c1, tau = c1_tau(path, 9 * Cin, Cin, drain)
    tiny = tiny_of(A2d, B, Cin)
    name = f"{path} {H}x{W} {Cin}->{N} drain {drain}"
    check(name, check_guards(obuf, M, N), ref, S, R, c1, tau, tiny)
    check_stats(name, stats, ref, c1 * S + 8 * U * ref.abs() + tiny, N // 8)


@pytest.mark.parametrize("path", ["conv3", "tma"])
def test_conv3_up2(path):
    """ConvTranspose2d(4, 2, 1) at 64 channels as one 3x3 halo conv: 64-column block j is parity class j = 2 py + px"""
    F, H, W, C = 6, 32, 16, 64
    x, Wt, bias, ref, S, R = up_problem(F, H, W, C, 91)
    B = torch.zeros(9 * C, 4 * C, device=DEV)
    for py in range(2):
        for px in range(2):
            for ky, dy in up_taps(py):
                for kx, dx in up_taps(px):
                    t = (dy + 1) * 3 + dx + 1
                    B[t * C:(t + 1) * C, (2 * py + px) * C:(2 * py + px + 1) * C] = Wt[:, :, ky, kx]
    dy, dx = square_taps(3)
    geo = dict(F=F, IH=H, IW=W, Cin=C, lda=C, dy=dy, dx=dx, in_stride=1, OHs=H, OWs=W, OH=H, OW=W, out_stride=1, up2=1)
    out_rows = F * 4 * H * W
    rc, obuf, _ = run_case(path, 0, geo, x.reshape(-1, C).contiguous(), B, 4 * C, out_rows, 68, bias=bias.repeat(4))
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    out = obuf[GUARD:GUARD + out_rows]
    assert torch.all(obuf[:GUARD] == SENT) and torch.all(obuf[GUARD + out_rows:] == SENT)
    assert torch.all(out[:, C:] == SENT), "store into the ldo padding"
    c1, tau = c1_tau(path, 9 * C, C, 0)
    check(f"up2 {path}", out[:, :C], ref.reshape(-1, C), S.reshape(-1, C), R.reshape(-1, C), c1, tau,
          tiny_of(x, B, C))


# ------------------------------------------------------------------------------------------------ LayerNorm epilogues
def ln_rows(M, C, seed, big_mean_rows=True):
    """activation rows; every 7th row has a mean 30-100x its standard deviation"""
    x = gen((M, C), seed)
    if big_mean_rows:
        g = torch.Generator().manual_seed(seed + 1)
        scale = (30 + 70 * torch.rand(M, generator=g)).to(DEV)
        sel = torch.arange(M, device=DEV) % 7 == 3
        x[sel] = x[sel] + scale[sel, None]
    return x


def rot_table(nframes, seed):
    ang = gen((nframes, 16), seed) * 3.0
    return torch.stack([ang.cos(), ang.sin()], -1).contiguous()      # [frames][16][(cos, sin)]


def ln_reference(epi, xr, Bm, mu, rs, fr, rot=None, qps=1.0, kq=None, nkq=None):
    """float64 LayerNorm fold + epilogue on rows xr (already in row order m); returns ref, elementwise bound pieces"""
    y = (xr - mu[:, None]) * rs[:, None]
    v = y @ Bm
    Sx = (xr.abs() @ Bm.abs()) * rs[:, None]                    # the contraction runs on the raw rows
    Rx = ((xr * xr) @ (Bm * Bm)).sqrt() * rs[:, None]
    return v, Sx, Rx


def apply_rotary(v, e, fr, rot):
    v, e = v.clone(), e.clone()
    cs = rot[fr].double()                                       # [rows][16][2]
    for hcol in range(0, 512, 32):
        c, s = cs[:, :, 0], cs[:, :, 1]
        x0, x1 = v[:, hcol:hcol + 32:2], v[:, hcol + 1:hcol + 32:2]
        e0, e1 = e[:, hcol:hcol + 32:2], e[:, hcol + 1:hcol + 32:2]
        v[:, hcol:hcol + 32:2], v[:, hcol + 1:hcol + 32:2] = x0 * c - x1 * s, x1 * c + x0 * s
        e[:, hcol:hcol + 32:2] = c.abs() * e0 + s.abs() * e1 + 4 * U * (x0.abs() + x1.abs())
        e[:, hcol + 1:hcol + 32:2] = c.abs() * e1 + s.abs() * e0 + 4 * U * (x0.abs() + x1.abs())
    return v, e


def apply_sla(v, e, qps):
    v, e = v.clone(), e.clone()
    for h in range(8):
        blk = v[:, 32 * h:32 * h + 32]
        sm = torch.softmax(blk, 1)
        eb = e[:, 32 * h:32 * h + 32]
        v[:, 32 * h:32 * h + 32] = sm * qps
        e[:, 32 * h:32 * h + 32] = sm * qps * (eb + (sm * eb).sum(1, keepdim=True) + 48 * U)
    return v, e


def apply_gate(v, e, fr, kq, nkq):
    M = v.shape[0]
    g = torch.empty(M, 24, dtype=torch.float64, device=v.device)
    eg = torch.empty_like(g)
    for ca in range(3):
        for hd in range(8):
            q = v[:, ca * 64 + hd * 8: ca * 64 + hd * 8 + 8]
            eq = e[:, ca * 64 + hd * 8: ca * 64 + hd * 8 + 8].norm(dim=1)
            k = kq.double()[fr, ca, hd * 8:hd * 8 + 8]
            nk = nkq.double()[ca]
            qn = q.norm(dim=1).clamp_min(1e-12)
            sr, sn = 8 * (q * k).sum(1) / qn, 8 * (q * nk).sum(1) / qn
            g[:, ca * 8 + hd] = torch.sigmoid(sr - sn)
            dsr = 16 * k.norm(dim=1) * eq / qn
            dsn = 16 * nk.norm() * eq / qn
            eg[:, ca * 8 + hd] = 0.25 * (dsr + dsn) + 64 * U * (sr.abs() + sn.abs() + 1)
    return g, eg


LN_CASES = [  # path, epi, Cin, N, stats source ('inline' | 'rows')
    ("tc", 1, 256, 768, "inline"), ("tc", 1, 256, 768, "rows"), ("presplit", 1, 256, 768, "rows"), ("mma", 1, 256, 768, "rows"),
    ("tc", 2, 128, 768, "inline"), ("tc", 2, 128, 768, "rows"), ("presplit", 2, 128, 768, "rows"), ("mma", 2, 128, 768, "rows"),
    ("tc", 3, 512, 768, "inline"), ("tc", 3, 512, 768, "rows"), ("presplit", 3, 512, 768, "rows"), ("mma", 3, 512, 768, "rows"),
    ("tc", 3, 64, 64, "inline"),
    ("tc", 4, 256, 192, "inline"), ("tc", 4, 256, 192, "rows"), ("mma", 4, 256, 192, "rows"),
]
EPI_NAME = {1: "temporal", 2: "sla", 3: "mid", 4: "gate"}


@pytest.mark.parametrize("path,epi,Cin,N,src", LN_CASES, ids=[f"{c[0]}-{EPI_NAME[c[1]]}-{c[2]}-{c[3]}-{c[4]}" for c in LN_CASES])
def test_layernorm_epilogues(path, epi, Cin, N, src):
    seed = 1000 + epi * 10 + Cin + (src == "inline")
    P = 64 if epi != 3 or N != 64 else 1
    if epi == 1:                                               # temporal qkv: sequence-blocked rows over Fe frames
        Fe, P = 24, 48
        M = Fe * P
    elif N == 64:                                              # many row tiles per CTA: the s_ln / row-table rings wrap
        M = 9 * 132 * 128 + 77
    else:
        M = 20 * P + 33
    x = ln_rows(M, Cin, seed)
    Wl = gen((Cin, N), seed + 2) / math.sqrt(Cin)
    wsum = Wl.double().sum(0).float()                          # float64 column sums rounded to fp32
    xd = x.double()
    mu, var = xd.mean(1), xd.var(1, unbiased=False)
    rs = 1.0 / torch.sqrt(var + 1e-5)
    rowstats = torch.stack([mu, rs], 1).float().contiguous()
    kw = dict(wsum=wsum, P=P, q_post_scale=1.0)
    if src == "inline":
        kw["ln_inline"] = 1
    else:
        kw["rowstats"] = rowstats
    geo = dict(F=1, IH=M, IW=1, Cin=Cin, lda=Cin, dy=[0], dx=[0], in_stride=1, OHs=M, OWs=1, OH=M, OW=1, out_stride=1)
    rows = torch.arange(M, device=DEV)
    if epi == 1:
        pb = seq_block(P)
        pix = seq_blocked_rows(Fe, P, pb).to(DEV)
        rows = pix
        geo.update(perm_pb=pb, perm_F=Fe, perm_in=1)
        rot = rot_table(Fe, seed + 3)
        kw["rot"] = rot
    fr = rows // P
    v, Sx, Rx = ln_reference(epi, xd[rows], Wl.double(), mu[rows], rs[rows], fr)
    K = Cin
    c1, tau = c1_tau(path, K, Cin, 0)
    # LayerNorm fold: contraction error on the raw rows, fp32 (mu, wsum) products, statistics of a stable fp32 mean / variance
    kst = (K / 8 + 3) * U
    mu_err = kst * xd[rows].abs().mean(1) + U * mu[rows].abs()
    e = c1 * Sx + (mu_err[:, None] + 4 * U * mu[rows].abs()[:, None]) * wsum.double().abs() * rs[rows][:, None] \
        + (4 * U + kst) * v.abs() + tiny_of(x, Wl, Cin) * rs[rows][:, None]
    R = Rx
    if epi == 1:
        v, e = apply_rotary(v, e, fr, rot)
    elif epi == 2:
        kw["q_post_scale"] = 1.0 / math.sqrt(32.0)
        v, e = apply_sla(v, e, 1.0 / math.sqrt(32.0))
    name = f"{path} {EPI_NAME[epi]} {Cin}->{N} {src}"
    if epi == 4:
        kq = gen((M // P + 1, 3, 64), seed + 4)
        kq = kq / kq.reshape(-1, 8, 8).norm(dim=2).reshape(kq.shape[0], 3, 8).repeat_interleave(8, 2)
        nkq = gen((3, 8), seed + 5)
        gates = torch.full((M + GUARD, 24), SENT, device=DEV)
        kw.update(kq=kq, nkq=nkq, gates=gates)
        rc, _, _ = run_case(path, epi, geo, x, Wl.contiguous(), N, M, N, **kw)
        assert rc == 0, _lib().lib.dawn_last_error().decode()
        assert torch.all(gates[M:] == SENT), "gate store past the last row"
        g, eg = apply_gate(v, e, fr, kq, nkq)
        out = gates[:M].double()
        assert torch.isfinite(out).all()
        err = ((out - g).abs() / (eg + 8 * U)).max().item()
        print(f"  {name}: gates max |d|/bound = {err:.3f}")
        assert err <= 1.0
        return
    ldo = N + 4
    rc, obuf, _ = run_case(path, epi, geo, x, Wl.contiguous(), N, M, ldo, **kw)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    out = check_guards(obuf, M, N)
    # the softmax block is not a linear function of the contraction: its error is held elementwise only
    cols = slice(256, N) if epi == 2 else slice(0, N)
    check(name, out[:, cols], v[:, cols], torch.zeros_like(v[:, cols]), R[:, cols], 1.0, tau, extra=e[:, cols], c2=0.0)
    if epi == 2:
        d = (out[:, :256].double() - v[:, :256]).abs()
        el = (d / (e[:, :256] + 8 * U * v[:, :256].abs() + 1e-30)).max().item()
        print(f"  {name} (softmax block): elementwise max |d|/bound = {el:.3f}")
        assert el <= 1.0


# ------------------------------------------------------------------------------------------------ mma.sync-only epilogues
def test_sla_outproj_per_frame_b():
    """per-frame B (spatial linear attention out-projection): rows_per_batch = P, b_batch_stride = 256 * ldb, + bias + residual"""
    F, P, C, N = 5, 100, 256, 128
    M = F * P
    q = gen((M, C), 11)
    Bf = gen((F, C, N), 12) / math.sqrt(C)
    bias, res = gen((N,), 13), gen((M, N), 14)
    ref = torch.empty(M, N, dtype=torch.float64, device=DEV)
    S, R = torch.empty_like(ref), torch.empty_like(ref)
    for f in range(F):
        r, s, rr = conv_ref(q[f * P:(f + 1) * P], Bf[f], torch.matmul)
        ref[f * P:(f + 1) * P], S[f * P:(f + 1) * P], R[f * P:(f + 1) * P] = r, s, rr
    ref = ref + bias.double() + res.double()
    geo = dict(F=1, IH=M, IW=1, Cin=C, lda=C, dy=[0], dx=[0], in_stride=1, OHs=M, OWs=1, OH=M, OW=1, out_stride=1,
               rows_per_batch=P, b_batch_stride=C * N)
    rc, obuf, _ = run_case("mma", 0, geo, q, Bf.reshape(F * C, N), N, M, N, bias=bias, Res=res, ldr=N)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    c1, tau = c1_tau("mma", C, C, 0)
    check("sla out-projection per-frame B", check_guards(obuf, M, N), ref, S, R, c1, tau, tiny_of(q, Bf[0], C))
    for path in ("tc", "presplit"):                            # the wgmma GEMM has one B for all rows
        rc, obuf, _ = run_case(path, 0, geo, q, Bf.reshape(F * C, N), N, M, N, bias=bias, Res=res, ldr=N)
        assert rc == -1 and torch.all(obuf == SENT)


def test_gn_apply_mma():
    """Out = SiLU(FiLM(GroupNorm(Y))) + Wt @ T_f: per-frame B (K = 32), 8 groups over all rows"""
    F, P, N = 4, 150, 128
    M, cpg = F * P, N // 8
    wt = gen((M, 32), 21)
    T = gen((F, 32, N), 22) / math.sqrt(32)
    Y = gen((M, N), 23) * 3 + 1
    gw, gb, film = gen((N,), 24), gen((N,), 25), gen((2 * N,), 26) * 0.5
    Yd = Y.double()
    gsum = torch.stack([Yd[:, g * cpg:(g + 1) * cpg].sum() for g in range(8)])
    gsq = torch.stack([(Yd[:, g * cpg:(g + 1) * cpg] ** 2).sum() for g in range(8)])
    gn_stats = torch.stack([gsum, gsq], 1).reshape(16).contiguous()
    count = float(M * cpg)
    mean = (gsum / count).repeat_interleave(cpg)
    rstd = 1.0 / torch.sqrt(gsq / count - (gsum / count) ** 2 + 1e-5).repeat_interleave(cpg)
    t = (Yd - mean) * rstd * gw.double() + gb.double()
    t = t * (film[:N].double() + 1) + film[N:].double()
    silu = t * torch.sigmoid(t)
    acc = torch.empty(M, N, dtype=torch.float64, device=DEV)
    S, R = torch.empty_like(acc), torch.empty_like(acc)
    for f in range(F):
        a, s, r = conv_ref(wt[f * P:(f + 1) * P], T[f], torch.matmul)
        acc[f * P:(f + 1) * P], S[f * P:(f + 1) * P], R[f * P:(f + 1) * P] = a, s, r
    ref = silu + acc
    geo = dict(F=1, IH=M, IW=1, Cin=32, lda=32, dy=[0], dx=[0], in_stride=1, OHs=M, OWs=1, OH=M, OW=1, out_stride=1,
               rows_per_batch=P, b_batch_stride=32 * N)
    rc, obuf, _ = run_case("mma", 5, geo, wt, T.reshape(F * 32, N), N, M, N + 4, Y=Y, ldy=N, gn_stats=gn_stats,
                           gn_count=count, gn_w=gw, gn_b=gb, film=film, cpg=cpg)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    c1, tau = c1_tau("mma", 32, 32, 0)
    tabs = ((Yd - mean).abs() * rstd * gw.double().abs() + gb.double().abs()) * (film[:N].double().abs() + 1) + film[N:].double().abs()
    check("gn_apply", check_guards(obuf, M, N), ref, S, R, c1, 1.0, tiny_of(wt, T[0], 32), extra=32 * U * tabs + 2 ** -20 * tabs,
          norm=False)


# ------------------------------------------------------------------------------------------------ accumulation bias
@pytest.mark.parametrize("path,drain", [("tc", 0), ("tc", 1), ("presplit", 0), ("conv3", 0), ("tma", 3), ("mma", 0)])
def test_accumulation_bias(path, drain):
    """all-positive operands at K = 9216: truncating adds inside the tensor core shrink every sum; the drains bound the bias"""
    if path in ("conv3", "tma"):
        F, H, W, Cin, k = 2, 16, 8, 1024, 3
    else:
        F, H, W, Cin, k = 1, 256, 1, 9216, 1
    N = 64
    A2d, B, ref, S, R = plain_problem(F, H, W, Cin, N, k, 4242, dist="pos")
    M = F * H * W
    ref = ref.reshape(M, N)
    dy, dx = square_taps(k)
    geo = dict(F=F, IH=H, IW=W, Cin=Cin, lda=Cin, dy=dy, dx=dx, in_stride=1, OHs=H, OWs=W, OH=H, OW=W, out_stride=1, drain=drain)
    rc, obuf, _ = run_case(path, 0, geo, A2d, B, N, M, N)
    assert rc == 0, _lib().lib.dawn_last_error().decode()
    out = check_guards(obuf, M, N).double()
    bias_rel = ((out - ref) / ref).mean().item()
    print(f"  {path} drain {drain}: mean signed relative error {bias_rel:.2e} (bound {2 ** -16:.1e})")
    assert abs(bias_rel) <= 2.0 ** -16, f"{path} drain {drain}: accumulation bias {bias_rel:.2e}"
    c1, _ = c1_tau(path, k * k * Cin, Cin, drain)
    assert ((out - ref).abs() <= c1 * S.reshape(M, N) + 8 * U * ref.abs()).all()


# ------------------------------------------------------------------------------------------------ refusals
def _refusal_cases():
    dy3, dx3 = square_taps(3)
    base = dict(F=2, IH=16, IW=16, Cin=64, lda=64, dy=dy3, dx=dx3, in_stride=1, OHs=16, OWs=16, OH=16, OW=16, out_stride=1)
    one = dict(base, dy=[0], dx=[0])
    return [
        ("tc-m127", "tc", 0, dict(one, F=1, IH=127, IW=1, OHs=127, OWs=1, OH=127, OW=1), 64, {}),
        ("presplit-m127", "presplit", 0, dict(one, F=1, IH=127, IW=1, OHs=127, OWs=1, OH=127, OW=1), 64, {}),
        ("tc-cin96", "tc", 0, dict(one, Cin=96, lda=96), 64, {}),
        ("tc-n96", "tc", 0, one, 96, {}),
        ("tc-gn-apply", "tc", 5, one, 64, {}),
        ("tc-lda-odd", "tc", 0, dict(one, lda=66), 64, {}),
        ("presplit-ln-inline", "presplit", 3, one, 64, dict(ln_inline=1)),
        ("mma-ln-inline", "mma", 3, one, 64, dict(ln_inline=1)),
        ("tc-ln-inline-3x3", "tc", 3, base, 64, dict(ln_inline=1)),
        ("mma-cin48", "mma", 0, dict(one, Cin=48, lda=48), 64, {}),
        ("conv3-h24", "conv3", 0, dict(base, IH=24, OHs=24, OH=24), 64, {}),
        ("tma-w12", "tma", 0, dict(base, IW=12, OWs=12, OW=12), 64, {}),
        ("conv3-cin96", "conv3", 0, dict(base, Cin=96, lda=96), 64, {}),
        ("conv3-ntaps4", "conv3", 0, dict(base, dy=[0, 0, 1, 1], dx=[0, 1, 0, 1]), 64, {}),
        ("conv3-taps-transposed", "conv3", 0, dict(base, dy=dx3, dx=dy3), 64, {}),
        ("conv3-up2-stats", "conv3", 0, dict(base, up2=1), 256, dict(stats=True)),
        ("conv3-up2-n128", "conv3", 0, dict(base, up2=1), 128, {}),
        ("conv3-residual", "conv3", 0, base, 64, dict(res=True)),
        ("conv3-stride2", "conv3", 0, dict(base, in_stride=2, OHs=8, OWs=8, OH=8, OW=8), 64, {}),
        ("conv3-qkv", "conv3", 3, base, 64, {}),
        ("tma-lda-pad", "tma", 0, dict(base, lda=72), 64, {}),
        ("conv3-perm", "conv3", 0, dict(base, perm_pb=16, perm_F=2, perm_out=1, perm_f_lo=0, perm_f_hi=2, P=256), 64, {}),
    ]


REFUSALS = _refusal_cases()


@pytest.mark.parametrize("cid,path,epi,geo,N,ex", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_refusals(cid, path, epi, geo, N, ex):
    M = geo["F"] * geo["OHs"] * geo["OWs"]
    nin = geo["F"] * geo["IH"] * geo["IW"]
    A = gen((nin, geo["lda"]), 3)
    B = gen((len(geo["dy"]) * geo["Cin"], (N + 63) // 64 * 64), 4)
    kw = {}
    if ex.get("stats"):
        kw.update(stats=torch.zeros(16, dtype=torch.float64, device=DEV), cpg=N // 8)
    if ex.get("res"):
        kw.update(Res=gen((M * 4, N), 5), ldr=N)
    if ex.get("ln_inline"):
        kw.update(ln_inline=1)
    if epi in (1, 2, 3, 4):
        kw.update(wsum=torch.zeros(B.shape[1], device=DEV), rowstats=None if ex.get("ln_inline") else torch.zeros(M, 2, device=DEV))
        kw = {k: v for k, v in kw.items() if v is not None}
    out_rows = M * 4 if geo.get("up2") else M
    rc, obuf, _ = run_case(path, epi, geo, A, B, N, out_rows, max(N, 64), **kw)
    assert rc == -1, f"{cid}: rc = {rc}"
    assert torch.all(obuf == SENT), f"{cid}: Out was written"
    if "stats" in kw:
        assert torch.all(kw["stats"] == 0)
