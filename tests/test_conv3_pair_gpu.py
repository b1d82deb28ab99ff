"""The halo conv's pair mode: 8 x 8 images, two frames of one clip per 128-row tile (rows 0-63 frame a, 64-127 frame b).

GPU cases check the same float64 reference and bounds as test_contraction_gpu.test_conv3, at the shapes of the UNet's 8 x 8 level
(Cin 256 / 512 / 1024 -> N 256 / 512 with GroupNorm statistics) and where the pair schedule has edges (H100: 132 SMs):

  * an odd frame count ends in a one-frame tile, whose second half must not be stored, counted in the GroupNorm sums or read
    outside the image (the output guard rows and the sentinel check catch a stray store);
  * fewer tiles than SMs, and many tiles per CTA (at N = 64 the epilogue warpgroup keeps its statistics over 8-tile runs);
  * both producers (gather from fp32, TMA from fp16 planes) and drains every 1, 3 and 9 taps;
  * a 64-channel transposed conv run as one 3x3 pair-mode conv with 4 x 64 columns.

The contraction entry point runs one clip, so a tile spanning two clips is not exercised here; the pairing is clip-major (images
f * clips + b and (f + 1) * clips + b), as the GroupNorm sums of the UNet's batched clips require.

CPU cases are static checks of the pair-mode kernels in the built library, as test_wgmma_schedule_cpu.py and test_sass_cpu.py do
for the 16 x 8 instantiations: no local memory, no ptxas-injected wgmma wait (C7517), the warpgroup MMAs in place and TMA loads
in the TMA-fed kernel."""
import collections
import os
import re
import shutil
import subprocess

import pytest

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dawn_pytorch_b200")
LIB = os.path.join(PKG, "libdawn_unet.so")
KERNEL = "tc_conv3_pair_kernel"

CASES = [  # path, F, H, W, Cin, N, drain
    ("conv3", 24, 8, 8, 256, 256, 0), ("tma", 24, 8, 8, 256, 512, 1),           # even, 48 / 96 tiles
    ("conv3", 23, 8, 8, 512, 512, 3), ("tma", 23, 8, 8, 512, 256, 0),           # odd: one-frame last tile
    ("conv3", 23, 8, 8, 1024, 256, 1), ("tma", 23, 8, 8, 1024, 512, 9),         # the decoder's concat conv
    ("conv3", 200, 8, 8, 512, 512, 9), ("tma", 200, 8, 8, 512, 512, 0),         # 800 tiles: the benchmark's mid-block convs
    ("tma", 201, 8, 8, 1024, 256, 3),                                            # 404 tiles, odd
    ("conv3", 2499, 8, 8, 64, 64, 0), ("tma", 2500, 8, 8, 64, 64, 1),           # one n-tile, 9-10 tiles per CTA, deferred sums
]


@pytest.mark.gpu
@pytest.mark.parametrize("path,F,H,W,Cin,N,drain", CASES,
                         ids=[f"{'gather' if c[0] == 'conv3' else 'tma'}-F{c[1]}-{c[4]}-{c[5]}-d{c[6]}" for c in CASES])
def test_conv3_pair(path, F, H, W, Cin, N, drain):
    from tests import test_contraction_gpu as TC
    TC.test_conv3(path, F, H, W, Cin, N, drain)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["conv3", "tma"])
def test_conv3_pair_up2(path):
    """ConvTranspose2d(4, 2, 1) at 64 channels from 8 x 8 images, odd frame count: parity class j = 2 py + px is column block j"""
    import torch
    from tests import test_contraction_gpu as TC
    F, H, W, C = 7, 8, 8, 64
    x, Wt, bias, ref, S, R = TC.up_problem(F, H, W, C, 93)
    B = torch.zeros(9 * C, 4 * C, device=TC.DEV)
    for py in range(2):
        for px in range(2):
            for ky, dy in TC.up_taps(py):
                for kx, dx in TC.up_taps(px):
                    t = (dy + 1) * 3 + dx + 1
                    B[t * C:(t + 1) * C, (2 * py + px) * C:(2 * py + px + 1) * C] = Wt[:, :, ky, kx]
    dy, dx = TC.square_taps(3)
    geo = dict(F=F, IH=H, IW=W, Cin=C, lda=C, dy=dy, dx=dx, in_stride=1, OHs=H, OWs=W, OH=H, OW=W, out_stride=1, up2=1)
    out_rows = F * 4 * H * W
    rc, obuf, _ = TC.run_case(path, 0, geo, x.reshape(-1, C).contiguous(), B, 4 * C, out_rows, 68, bias=bias.repeat(4))
    assert rc == 0, TC._lib().lib.dawn_last_error().decode()
    out = TC.check_guards(obuf, out_rows, C)
    c1, tau = TC.c1_tau(path, 9 * C, C, 0)
    TC.check(f"pair up2 {path}", out, ref.reshape(-1, C), S.reshape(-1, C), R.reshape(-1, C), c1, tau, TC.tiny_of(x, B, C))


# ------------------------------------------------------------------------------------------------ static checks (no GPU)
@pytest.fixture(scope="module")
def sass_counts():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or the built library is not available")
    out = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, timeout=600).stdout
    cur, cnt = None, {}
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            cnt[cur] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ln) if cur else None
        if m:
            op = m.group(1)
            for key in ("STL", "LDL", "HGMMA", "UBLKCP", "UTMALDG", "BRA.U.ANY"):
                if op == key or op.startswith(key + "."):
                    cnt[cur][key] += 1
    return {k: v for k, v in cnt.items() if KERNEL in k}


def test_pair_kernels_are_built(sass_counts):
    assert len(sass_counts) == 2, sorted(sass_counts)        # gather- and TMA-fed


def test_pair_kernels_do_not_spill(sass_counts):
    for k, c in sass_counts.items():
        assert c["STL"] == 0 and c["LDL"] == 0, (k, dict(c))


def test_pair_kernels_keep_their_mma_issue_loop_free(sass_counts):
    for k, c in sass_counts.items():
        assert c["HGMMA"] >= 24 and c["UBLKCP"] > 0, (k, dict(c))
        assert c["BRA.U.ANY"] <= c["UBLKCP"] + c["UTMALDG"], (k, dict(c))
    assert sum(c["UTMALDG"] > 0 for c in sass_counts.values()) == 1


def test_pair_kernels_have_no_injected_wgmma_wait():
    log = os.path.join(PKG, "build", "tc_conv3.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("no ptxas log (the library was not built in this tree)")
    with open(log) as fh:
        text = fh.read()
    entries = re.split(r"(?=ptxas info\s+: Compiling entry function)", text)
    pair = [e for e in entries if KERNEL in e.split("\n", 1)[0]]
    assert len(pair) == 2, "pair-mode kernels missing from the ptxas log"
    for e in pair:
        assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", e), e
    assert "C7517" not in text, [ln for ln in text.splitlines() if "C7517" in ln]
