"""GPU: the warpgroup-MMA fused temporal attention (temporal_fused_wg_kernel) against the float64 reference and against the
mma.sync kernel (temporal_fused_kernel) on the same input.

`launch_temporal_fused` runs the warpgroup kernel for every sequence of at most 256 frames; `DAWN_FUSED_TEMPORAL_MMA_SYNC`
forces the mma.sync kernel for the same case.  Each case checks the warpgroup kernel with the bounds of
tests/test_fused_gpu.py (elementwise bound of tests/fused_ref.py, norm-wise tau scaled by the rows' largest |mean| / std), checks
that the two kernels agree within tau of each other, and keeps the sentinels around the output, in its row padding and in the
rows an output indexed by the on-chip frame instead of f - q_lo would reach.  Which kernel ran is read from the profiler's
kernel names: F 256 runs the warpgroup kernel, F 257 the mma.sync one.  That check runs in a new process, where the profiler
still records device events."""
import math
import os
import subprocess
import sys

import pytest
import torch

from tests import fused_ref as R
from tests import test_fused_gpu as TF

pytestmark = pytest.mark.gpu

CASES = {   # id: (F, P, band, q_lo, q_hi, mean-shifted rows)
    **{f"f{f}": (f, 131, 40, 0, f, False) for f in (1, 16, 17, 64, 199, 200, 208, 209, 255, 256)},
    "bench": (200, 4096, 40, 0, 200, False),
    "band1": (200, 131, 1, 0, 200, False), "band8": (200, 131, 8, 0, 200, False),
    "band64-f256": (256, 131, 64, 0, 256, False),
    "win0-40-of-80": (80, 64, 40, 0, 40, False), "win40-120-of-200": (200, 64, 40, 40, 120, False),
    "win17-239-of-256": (256, 64, 64, 17, 239, False), "win250-256-of-256": (256, 64, 8, 250, 256, False),
    "bigmean": (200, 64, 40, 0, 200, True),
}


def inputs(F, P, band, q_lo, q_hi, mean, seed):
    x = TF.gen((F * P, 64), seed)
    if mean:
        x = x * 0.5 + (30 + 70 * torch.rand(F * P, 1, generator=torch.Generator().manual_seed(seed))).to(TF.DEV) * 0.5
    gamma, wqkv, wout = TF.attn_weights(seed)
    ang = TF.gen((F, 16), seed + 3, 3.0)
    rot = torch.stack((ang.cos(), ang.sin()), -1).contiguous()
    bias = TF.gen((8, 2 * band + 1), seed + 4)
    res = TF.gen(((q_hi - q_lo) * P, 64), seed + 5)
    return dict(x=x, gamma=gamma, w_qkv=wqkv, w_out=wout, rot=rot, bias=bias), res


def launch(kernel, F, P, band, q_lo, q_hi, tensors, res):
    """one kernel on the case; returns the owned output rows (q_hi - q_lo, P, 64) after the sentinel checks"""
    Fq = q_hi - q_lo
    ldo = 68
    obuf, optr = TF.guarded(Fq * P, ldo, q_lo * P)
    rbuf = torch.full((Fq * P + q_lo * P, 64), TF.SENT, device=TF.DEV)
    rbuf[:Fq * P] = res
    rc = TF.run(kernel=kernel, F=F, P=P, C=64, band=band, q_lo=q_lo, q_hi=q_hi, ldx=64, ldr=64, ldo=ldo, res=rbuf, out=optr,
                **tensors)
    assert rc == 0, TF._lib().lib.dawn_last_error().decode()
    return TF.body(obuf, Fq * P, 64).reshape(Fq, P, 64)


@pytest.mark.parametrize("cid", list(CASES))
def test_wg_matches_reference_and_mma_sync(cid):
    F, P, band, q_lo, q_hi, mean = CASES[cid]
    L = TF._lib()
    t, res = inputs(F, P, band, q_lo, q_hi, mean, sum(map(ord, cid)))
    wg = launch(L.FUSED_TEMPORAL, F, P, band, q_lo, q_hi, t, res)
    ms = launch(L.FUSED_TEMPORAL_MMA_SYNC, F, P, band, q_lo, q_hi, t, res)
    xs, rs = t["x"].reshape(F, P, 64), res.reshape(q_hi - q_lo, P, 64)
    worst, dn, dd, yn = 0.0, 0.0, 0.0, 0.0
    for p0 in range(0, P, 128):
        sl = slice(p0, min(P, p0 + 128))
        ref, bnd, y = R.temporal(xs[:, sl].transpose(0, 1), rs[:, sl].transpose(0, 1), t["gamma"], t["w_qkv"], t["w_out"],
                                 t["rot"], t["bias"], band, q_lo, q_hi)
        a, b = wg[:, sl].transpose(0, 1).double(), ms[:, sl].transpose(0, 1).double()
        assert torch.isfinite(a).all()
        d = (a - ref).abs()
        worst = max(worst, (d / bnd).max().item())
        dn += d.pow(2).sum().item()
        dd += (a - b).pow(2).sum().item()
        yn += y.pow(2).sum().item()
    r = max(1.0, (xs.mean(-1).abs() / xs.std(-1, unbiased=False)).max().item())
    tau = TF.TAU * r
    nr, nd = math.sqrt(dn / yn), math.sqrt(dd / yn)
    print(f"  {cid}: max |d|/bound = {worst:.3f}; ||d||/||y|| = {nr:.2e} ({nr / tau:.3f} tau); "
          f"||wg - mma.sync||/||y|| = {nd:.2e} ({nd / tau:.3f} tau)")
    assert worst <= 1.0, f"elementwise error {worst:.2f}x the bound"
    assert nr <= tau, f"norm-wise error {nr:.2e} > {tau:.2e}"
    assert nd <= tau, f"the two kernels differ by {nd:.2e} > {tau:.2e}"


def kernels_run(kernel, F, P, band, q_lo, q_hi):
    t, res = inputs(F, P, band, q_lo, q_hi, False, F)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = launch(kernel, F, P, band, q_lo, q_hi, t, res)
    names = {e.name for e in prof.events() if "temporal_fused" in e.name}
    return out, names


def dispatch_check():
    """F 256 runs the warpgroup kernel; F 257 (frames [8, 248) of it produce output: 16 query tiles) is refused by its predicate
    and runs the mma.sync kernel, bit for bit as when forced"""
    L = TF._lib()
    _, names = kernels_run(L.FUSED_TEMPORAL, 256, 8, 40, 0, 256)
    assert any("temporal_fused_wg_kernel" in n for n in names), names
    out, names = kernels_run(L.FUSED_TEMPORAL, 257, 8, 40, 8, 248)
    assert names and not any("temporal_fused_wg_kernel" in n for n in names), names
    forced, _ = kernels_run(L.FUSED_TEMPORAL_MMA_SYNC, 257, 8, 40, 8, 248)
    assert torch.equal(out, forced)


def test_dispatch_by_sequence_length():
    """dispatch_check in a new Python process: torch.profiler records no device events once a process is a few minutes old, so
    in a long pytest run the kernel names would come back empty whichever kernel ran"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-s", "-B", "-c", "from tests import test_temporal_wg_gpu as T; T.dispatch_check()"],
                       cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
