"""CPU: static check of the built library's SASS (cuobjdump, no GPU needed).  The GEMM and halo-conv kernels must contain warpgroup
MMAs (HGMMA: 2 row halves x 3 split terms x 4 k-steps), and their MMA paths must stay free of the per-lane uniform-register loops
(`BRA.U.ANY`) that ptxas emits when an operand is not provably warp-uniform.  The loaders (cp.async.bulk / TMA, one thread) may keep
theirs: at most one loop per bulk copy / tensor load."""
import collections
import os
import re
import shutil
import subprocess

import pytest

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dawn_pytorch_b200", "libdawn_unet.so")


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
            for key in ("HGMMA", "UTCHMMA", "UBLKCP", "UTMALDG", "BRA.U.ANY"):
                if m.group(1).startswith(key):
                    cnt[cur][key] += 1
    return cnt


def kernels(cnt, name):
    return {k: v for k, v in cnt.items() if name in k}


@pytest.mark.parametrize("name", ["tc_gemm_kernel", "tc_conv3_kernel"])
def test_gemm_and_halo_conv_kernels_keep_their_mma_issue_loop_free(sass_counts, name):
    ks = kernels(sass_counts, name)
    assert ks
    for k, c in ks.items():
        assert c["HGMMA"] >= 24 and c["UTCHMMA"] == 0 and c["UBLKCP"] > 0, (k, dict(c))
        assert c["BRA.U.ANY"] <= c["UBLKCP"] + c["UTMALDG"], (k, dict(c))      # only the loaders' copies; none per MMA


def test_tma_fed_halo_conv_uses_tensor_loads(sass_counts):
    assert any(c["UTMALDG"] > 0 for c in kernels(sass_counts, "tc_conv3_kernel").values())
