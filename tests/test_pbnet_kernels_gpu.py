"""GPU: each PBnet decoder row kernel (include/dawn_pbnet.h, dawn_pbnet_test_kernel) against the same operation in float64, at
the shapes the library accepts beyond DAWN's (d_model 64, 4 heads, ff 128, 2 layers): every entry runs the launch code generate
uses on caller buffers.

* memory rows: T = bs F in {1, 7, 8, 9, 33} across the 8-row blocks, D in {32, 96, 256}, Lz in {1, 18, 42, 256}, pose_dim in
  {1, 32} and none, z in CAE.generate's (F, bs, Lz) layout;
* projection: H in {2, 6, 32} (npairs 1, 3, 16: at 32 heads the rotary covers the whole head), 1, 3 and 8 column groups with the
  decoder's flag patterns (q alone; q | k | v; k | v of 4 layers), ldx = 0 (one row for every frame), frames wrapping at F;
* to_out + LayerNorm: hid 64 to 1024, ldr = 0, the residual being the output (in place), rows whose mean is 30-300 sigma;
* FFN + LayerNorm: ff in {1, 33, 2048}, in place, and with finallayer (nout in {1, 32}) and the length mask of bs >= 2 clips of
  unequal lengths: masked rows must be exactly 0 and x untouched.

Every output has sentinel guard rows before and after its T rows.  Error bounds are propagated from the fp32 unit roundoff
u = 2^-24 through each kernel's own order of operations: an fmaf chain of n terms from 0 is within n u sum |terms|; the
two-pass LayerNorm (lane sums of D / 32 values, a 5-level warp tree) as tests/test_hubert_kernels_gpu.ln_bound; the erf GELU
within 1.13 (its largest slope) times its input's error plus 4 u (|gelu| + |a|).  Every case also meets the north-star
tolerance 1e-4 + 1e-3 |ref| and prints both margins.
"""
import ctypes
import math

import pytest
import torch

from dawn_pytorch_b200._lib import PBNET_FFN_LN, PBNET_MEMORY, PBNET_OUT_LN, PBNET_PROJ
from tests.test_hubert_kernels_gpu import GELU_SLOPE, GUARD, SENT, U, big_mean_rows, check_guarded, gen, guarded, ln_bound, report

pytestmark = pytest.mark.gpu

DEV = "cuda"
QSCALE = 32 ** -0.5                      # dim_head ** -0.5 as an fp32 value, the one generate passes
SCALE, ROTARY = 1, 2


def run(**kw):
    from dawn_pytorch_b200 import _lib
    c = _lib.DawnPbnetKernelCase()
    for k, v in kw.items():
        if k == "flags":
            for i, f in enumerate(v):
                c.flags[i] = f
        else:
            setattr(c, k, ctypes.c_void_p(v.data_ptr()) if torch.is_tensor(v) else v)
    torch.cuda.synchronize()
    rc = _lib.lib.dawn_pbnet_test_kernel(ctypes.byref(c), _lib.stream())
    torch.cuda.synchronize()
    return rc


def run_ok(**kw):
    from dawn_pytorch_b200 import _lib
    _lib.check(run(**kw), "dawn_pbnet_test_kernel")


def rotary_table(F, npairs):
    """(F, npairs, 2) fp32 (cos, sin) of the fp32 angle f * freq, as the decoder's rotary table holds them"""
    freqs = 1. / (10000 ** (torch.arange(0, 2 * npairs, 2).float() / (2 * npairs)))
    ang = torch.arange(F, dtype=torch.float32)[:, None] * freqs[None, :]
    return torch.stack([ang.cos(), ang.sin()], -1).contiguous().to(DEV)


# ------------------------------------------------------------------------------------------------ memory rows
MEMORY_CASES = [  # bs, F, D, Lz, PE
    (1, 1, 32, 1, 1), (1, 7, 96, 18, 32), (2, 4, 256, 256, 1), (3, 3, 64, 42, 0), (3, 11, 32, 256, 32), (1, 33, 256, 42, 6),
]


@pytest.mark.parametrize("bs,F,D,Lz,PE", MEMORY_CASES, ids=[f"bs{c[0]}-f{c[1]}-d{c[2]}-lz{c[3]}-pe{c[4]}" for c in MEMORY_CASES])
def test_memory_rows(bs, F, D, Lz, PE):
    T = bs * F
    seed = 7000 + T + D + Lz + PE
    aud, z = gen((T, D), seed), gen((F, bs, Lz), seed + 1)
    wz = gen((Lz, D), seed + 2, 1 / math.sqrt(Lz))
    xref, wp = gen((bs, max(PE, 1)), seed + 3, 0.5), gen((max(PE, 1), D), seed + 4, 0.5)
    buf, out = guarded(T, D)
    run_ok(kernel=PBNET_MEMORY, bs=bs, F=F, D=D, Lz=Lz, PE=PE, x=aud, z=z, w=wz, xref=xref, w2=wp, out=out)
    got = check_guarded(buf, T, D)
    zr = z.double().permute(1, 0, 2).reshape(T, Lz)                       # row m = b F + f reads z[f][b]
    xr = xref.double()[:, :PE].repeat_interleave(F, 0)
    acc = zr @ wz.double() + xr @ wp.double()[:PE]
    S = zr.abs() @ wz.double().abs() + xr.abs() @ wp.double()[:PE].abs()
    ref = aud.double() + acc
    bound = (Lz + PE) * U * S + U * ref.abs()                             # Lz + PE fmaf from 0, then aud + acc
    report(f"memory bs={bs} F={F} D={D} Lz={Lz} PE={PE}", got, ref, bound)


# ------------------------------------------------------------------------------------------------ projection
PROJ_CASES = [  # T, F, D, H, flags (one per group), ldx 0
    (1, 1, 32, 2, [SCALE | ROTARY], False),
    (7, 7, 96, 6, [SCALE | ROTARY, ROTARY, 0], False),
    (8, 4, 256, 32, [SCALE | ROTARY], False),
    (9, 9, 32, 2, [ROTARY, 0] * 4, False),
    (33, 11, 96, 6, [ROTARY, 0] * 4, False),
    (33, 33, 256, 32, [SCALE | ROTARY, ROTARY, 0], False),
    (9, 3, 64, 6, [SCALE | ROTARY], True),
    (33, 33, 32, 32, [SCALE | ROTARY], True),
]


@pytest.mark.parametrize("T,F,D,H,flags,ldx0", PROJ_CASES,
                         ids=[f"t{c[0]}-f{c[1]}-d{c[2]}-h{c[3]}-g{len(c[4])}{'-ldx0' if c[5] else ''}" for c in PROJ_CASES])
def test_projection(T, F, D, H, flags, ldx0):
    hid, G = 32 * H, len(flags)
    N, npairs = G * hid, min(32, H) // 2
    seed = 7100 + T + D + H + G
    x = gen((1 if ldx0 else T, D), seed, 1.7)
    w = gen((D, N), seed + 1, 0.25)
    rot = rotary_table(F, npairs)
    buf, out = guarded(T, N)
    run_ok(kernel=PBNET_PROJ, T=T, F=F, D=D, ldx=0 if ldx0 else D, hid=hid, ngroups=G, flags=flags, qscale=QSCALE, npairs=npairs,
           x=x, w=w, rot=rot, out=out)
    got = check_guarded(buf, T, N)
    xd = x.double().expand(T, D)
    v, S = xd @ w.double(), xd.abs() @ w.double().abs()
    e = D * U * S                                                          # D fmaf from 0
    qs = torch.tensor(QSCALE, dtype=torch.float32).item()
    cs = rot.double()[torch.arange(T, device=DEV) % F]                     # (T, npairs, 2): row m's frame is m % F
    ref, bound = v.clone(), e.clone()
    for g, fl in enumerate(flags):
        for h in range(H):
            c0 = g * hid + 32 * h
            vv, ee = v[:, c0:c0 + 32].clone(), e[:, c0:c0 + 32].clone()
            if fl & SCALE:
                vv, ee = vv * qs, ee * qs + U * (vv * qs).abs()
            if fl & ROTARY:
                a, b = vv[:, 0:2 * npairs:2], vv[:, 1:2 * npairs:2]
                ea, eb = ee[:, 0:2 * npairs:2], ee[:, 1:2 * npairs:2]
                c, s = cs[..., 0], cs[..., 1]
                err = ea * c.abs() + eb * s.abs() + ea * s.abs() + eb * c.abs() + 2 * U * (a.abs() + b.abs())
                ra, rb = a * c - b * s, b * c + a * s
                vv[:, 0:2 * npairs:2], vv[:, 1:2 * npairs:2] = ra, rb
                ee[:, 0:2 * npairs:2], ee[:, 1:2 * npairs:2] = err, err
            ref[:, c0:c0 + 32], bound[:, c0:c0 + 32] = vv, ee
    report(f"proj T={T} F={F} D={D} H={H} groups={flags}{' ldx=0' if ldx0 else ''}", got, ref, bound)


# ------------------------------------------------------------------------------------------------ to_out + LayerNorm
OUT_LN_CASES = [  # T, D, H, residual: "rows" (ldr = D), "one" (ldr = 0), "inplace" (res is the output)
    (1, 32, 2, "rows"), (7, 96, 6, "inplace"), (8, 256, 32, "rows"), (9, 32, 32, "one"), (33, 96, 2, "inplace"),
    (33, 256, 6, "one"), (9, 64, 4, "inplace"),
]


@pytest.mark.parametrize("T,D,H,resmode", OUT_LN_CASES, ids=[f"t{c[0]}-d{c[1]}-h{c[2]}-{c[3]}" for c in OUT_LN_CASES])
def test_out_layernorm(T, D, H, resmode):
    hid = 32 * H
    seed = 7200 + T + D + H
    o = gen((T, hid), seed)
    wo = gen((hid, D), seed + 1, 1 / math.sqrt(hid))
    gam, be = 1 + gen((D,), seed + 2, 0.2), gen((D,), seed + 3, 0.05)
    res = big_mean_rows(1 if resmode == "one" else T, D, seed + 4)
    buf, out = guarded(T, D)
    if resmode == "inplace":
        out.copy_(res)
        run_ok(kernel=PBNET_OUT_LN, T=T, D=D, hid=hid, ldr=D, x=o, w=wo, res=out, gamma=gam, beta=be, out=out)
    else:
        run_ok(kernel=PBNET_OUT_LN, T=T, D=D, hid=hid, ldr=0 if resmode == "one" else D, x=o, w=wo, res=res, gamma=gam, beta=be,
               out=out)
    got = check_guarded(buf, T, D)
    y = res.double().expand(T, D) + o.double() @ wo.double()
    e_y = hid * U * (o.double().abs() @ wo.double().abs()) + U * y.abs()   # hid fmaf from 0, then res + acc
    ref, bound = ln_bound(y, e_y, gam, be, 1e-5, False)
    report(f"out+LN T={T} D={D} hid={hid} res={resmode}", got, ref, bound)


# ------------------------------------------------------------------------------------------------ FFN + LayerNorm (+ finallayer)
FFN_CASES = [  # lengths (bs clips of F = max frames; T = bs F), D, ff, nout (0: in place, no finallayer)
    ([1], 32, 1, 0), ([7], 96, 33, 0), ([8], 256, 2048, 0), ([9], 32, 2048, 32), ([5, 2], 96, 1, 1), ([11, 4, 7], 256, 33, 32),
    ([3, 1], 64, 128, 6), ([33], 32, 33, 1),
]


@pytest.mark.parametrize("lengths,D,ff,nout", FFN_CASES, ids=[f"len{'-'.join(map(str, c[0]))}-d{c[1]}-ff{c[2]}-nout{c[3]}"
                                                              for c in FFN_CASES])
def test_ffn_layernorm(lengths, D, ff, nout):
    bs, F = len(lengths), max(lengths)
    T = bs * F
    seed = 7300 + T + D + ff + nout
    x = big_mean_rows(T, D, seed)
    w1, b1 = gen((D, ff), seed + 1, 1 / math.sqrt(D)), gen((ff,), seed + 2, 0.05)
    w2, b2 = gen((ff, D), seed + 3, 1 / math.sqrt(ff)), gen((D,), seed + 4, 0.05)
    gam, be = 1 + gen((D,), seed + 5, 0.2), gen((D,), seed + 6, 0.05)
    xd = x.double()
    a = xd @ w1.double() + b1.double()
    e_a = D * U * (xd.abs() @ w1.double().abs()) + U * a.abs()            # D fmaf from 0, then + b1
    h = torch.nn.functional.gelu(a)
    e_h = GELU_SLOPE * e_a + 4 * U * (h.abs() + a.abs())
    t = h @ w2.double() + b2.double()
    y = xd + t
    e_y = e_h @ w2.double().abs() + ff * U * (h.abs() @ w2.double().abs()) + U * t.abs() + U * y.abs()
    ref, e_ln = ln_bound(y, e_y, gam, be, 1e-5, False)
    xbuf, xb = guarded(T, D)
    xb.copy_(x)
    if nout == 0:
        run_ok(kernel=PBNET_FFN_LN, T=T, D=D, ff=ff, x=xb, w=w1, b1=b1, w2=w2, b2=b2, gamma=gam, beta=be)
        got = check_guarded(xbuf, T, D)
        report(f"ffn+LN T={T} D={D} ff={ff} in place", got, ref, e_ln)
        return
    wf, bf = gen((D, nout), seed + 7, 1 / math.sqrt(D)), gen((nout,), seed + 8, 0.05)
    mask = (torch.arange(F)[None, :] < torch.tensor(lengths)[:, None]).reshape(T).to(device=DEV, dtype=torch.uint8)
    buf, out = guarded(T, nout)
    run_ok(kernel=PBNET_FFN_LN, T=T, D=D, ff=ff, nout=nout, x=xb, w=w1, b1=b1, w2=w2, b2=b2, gamma=gam, beta=be, wf=wf, bf=bf,
           mask=mask, out=out)
    assert torch.equal(check_guarded(xbuf, T, D), x), "finallayer's call must leave x as it was"
    got = check_guarded(buf, T, nout)
    live = mask.bool()
    assert torch.all(got[~live] == 0) and not torch.signbit(got[~live]).any(), "masked rows must be exactly +0"
    fin = ref @ wf.double() + bf.double()
    e_f = e_ln @ wf.double().abs() + D * U * (ref.abs() @ wf.double().abs()) + U * fin.abs()
    report(f"ffn+LN+final T={T} lengths={lengths} D={D} ff={ff} nout={nout}", got[live], fin[live], e_f[live])


# ------------------------------------------------------------------------------------------------ refusals
def test_bad_geometry_is_refused_before_any_launch():
    t = torch.zeros(64, device=DEV)
    ok = dict(T=1, bs=1, F=1, D=32, Lz=1, PE=0, hid=32, ngroups=1, ff=1, x=t, z=t, xref=t, w=t, w2=t, b1=t, b2=t, gamma=t, beta=t,
              res=t, rot=t, out=t)
    bad = [dict(kernel=PBNET_MEMORY, D=48), dict(kernel=PBNET_MEMORY, D=288), dict(kernel=PBNET_MEMORY, bs=0),
           dict(kernel=PBNET_MEMORY, bs=1 << 13, F=1 << 12), dict(kernel=PBNET_PROJ, ngroups=9), dict(kernel=PBNET_PROJ, hid=48),
           dict(kernel=PBNET_PROJ, ldx=16), dict(kernel=PBNET_PROJ, flags=[ROTARY], npairs=0), dict(kernel=PBNET_PROJ, npairs=17),
           dict(kernel=PBNET_PROJ, flags=[4]), dict(kernel=PBNET_OUT_LN, ldr=16), dict(kernel=PBNET_OUT_LN, hid=2048),
           dict(kernel=PBNET_FFN_LN, ff=2049), dict(kernel=PBNET_FFN_LN, ff=0), dict(kernel=PBNET_FFN_LN, wf=t, bf=t, mask=t, nout=33),
           dict(kernel=PBNET_FFN_LN, wf=t, nout=1), dict(kernel=4), dict(kernel=PBNET_PROJ, x=None),
           dict(kernel=PBNET_MEMORY, out=None), dict(kernel=PBNET_FFN_LN, wf=t, bf=t, mask=t, nout=1, out=None)]
    for b in bad:
        kw = {**ok, **b}
        kw = {k: v for k, v in kw.items() if v is not None}
        assert run(**kw) == -1, b
    assert torch.count_nonzero(t) == 0
