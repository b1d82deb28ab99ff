"""GPU: the warpgroup-MMA spatial linear attention kernels (sla_ctx_kernel + sla_merge_kernel, sla_out_kernel) against the float64
references and bounds of tests/fused_ref.py, at the shapes tests/test_fused_gpu.py does not run: the benchmark's layers (P 4096
and 1024 at F 200), last 64-pixel tiles holding 16, 32 or 48 pixels, one and sixteen context splits, two clips stacked as 2F
frames, and padded row strides, in place and not.  Every case keeps the sentinels around the output and in its row padding.

Context splits (sla_fused_run): P 512 is one split of 512; P 1008 sixteen of 64, the last 48 pixels; P 8192 sixteen of 512.
Output CTAs own 128 to 512 pixels, 64 per warpgroup step: P 80, 96, 112 end inside the second warpgroup's tile, P 176 inside
the first warpgroup's tile of the second CTA.  The float64 references run a few frames at a time."""
import pytest
import torch

from tests import fused_ref as R
from tests import test_fused_gpu as TF

pytestmark = pytest.mark.gpu

FCHUNK = 25          # frames per reference call


def clip_input(Fr, P, seed, clips):
    """(Fr * P, 64) rows; with clips = 2 the second half of the frames is a second clip with other statistics"""
    x = TF.gen((Fr * P, 64), seed)
    if clips == 2:
        x[Fr // 2 * P:] = 3.0 * x[Fr // 2 * P:] + 1.5
    return x


CTX = {   # id: (P, F, ldx, clips)
    "bench-l0": (4096, 200, 64, 1), "bench-l1": (1024, 200, 64, 1),
    "tail16": (592, 2, 64, 1), "tail32": (96, 3, 64, 1), "tail48": (112, 3, 64, 1),
    "split1": (512, 3, 64, 1), "split16-tail48": (1008, 2, 64, 1), "split16": (8192, 1, 64, 1),
    "clips2": (1024, 16, 64, 2), "ldx72": (208, 4, 72, 1),
}


@pytest.mark.parametrize("cid", list(CTX))
def test_sla_ctx_wg(cid):
    P, Fr, ldx, clips = CTX[cid]
    seed = 17 * P + Fr
    x = clip_input(Fr, P, seed, clips)
    xs = torch.full((Fr * P, ldx), TF.SENT, device=TF.DEV)
    xs[:, :64] = x
    gamma, wqkv, wout = TF.sla_weights(seed)
    ldb = 72
    bbuf, bptr = TF.guarded(Fr * 256, ldb)
    rc = TF.run(kernel=TF._lib().FUSED_SLA_CTX, F=Fr, P=P, C=64, ldx=ldx, ldb=ldb, x=xs, gamma=gamma, w_qkv=wqkv, w_out=wout,
                Bf=bptr)
    assert rc == 0, TF._lib().lib.dawn_last_error().decode()
    Bf = TF.body(bbuf, Fr * 256, 64).reshape(Fr, 256, 64)
    xr = x.reshape(Fr, P, 64)
    parts = [R.sla_ctx(xr[f0:f0 + FCHUNK], gamma, wqkv, wout) for f0 in range(0, Fr, FCHUNK)]
    ref, bnd = torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
    TF.check(f"sla_ctx {cid}", Bf, ref, bnd, tau=2 * TF.TAU)


OUT = {   # id: (P, F, ldx, ldo, in place, clips)
    "bench-l0": (4096, 200, 64, 64, True, 1), "bench-l1": (1024, 200, 64, 64, True, 1),
    "tail16": (80, 3, 64, 68, False, 1), "tail32": (96, 3, 64, 68, False, 1), "tail48": (112, 3, 68, 68, True, 1),
    "cta-tail48": (176, 3, 64, 68, False, 1), "cta16": (8192, 1, 64, 64, True, 1),
    "clips2": (1024, 16, 64, 64, True, 2), "inplace-ld72": (208, 4, 72, 72, True, 1), "ldx80": (208, 4, 80, 68, False, 1),
}


@pytest.mark.parametrize("cid", list(OUT))
def test_sla_out_wg(cid):
    P, Fr, ldx, ldo, inplace, clips = OUT[cid]
    seed = 19 * P + Fr
    x = clip_input(Fr, P, seed, clips)
    gamma, wqkv, _ = TF.sla_weights(seed)
    Bf = TF.gen((Fr * 256, 64), seed + 3, 0.05)
    bias = TF.gen(64, seed + 4)
    obuf, optr = TF.guarded(Fr * P, ldo)
    if inplace:
        assert ldx == ldo
        obuf[TF.GUARD:TF.GUARD + Fr * P, :64] = x
        xarg = optr
    else:
        xarg = torch.full((Fr * P, ldx), TF.SENT, device=TF.DEV)
        xarg[:, :64] = x
    rc = TF.run(kernel=TF._lib().FUSED_SLA_OUT, F=Fr, P=P, C=64, ldx=ldx, ldo=ldo, ldb=64, x=xarg, out=optr, gamma=gamma,
                w_qkv=wqkv, Bf=Bf, out_bias=bias)
    assert rc == 0, TF._lib().lib.dawn_last_error().decode()
    out = TF.body(obuf, Fr * P, 64).reshape(Fr, P, 64)
    xr, Bfr = x.reshape(Fr, P, 64), Bf.reshape(Fr, 256, 64)
    parts = [R.sla_out(xr[f0:f0 + FCHUNK], gamma, wqkv, Bfr[f0:f0 + FCHUNK], bias) for f0 in range(0, Fr, FCHUNK)]
    ref, bnd = torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
    TF.check(f"sla_out {cid}", out, ref, bnd, y_ref=ref - (xr.double() + bias.double()), tau=2 * TF.TAU)
