"""CPU: static checks of the warpgroup-MMA spatial linear attention kernels in the built library (no GPU needed).  The context
kernel's K/V projection and the output kernel's q projection and Bf product are warpgroup MMAs (HGMMA); the context product
k^T v stays on mma.sync (HMMA), the output kernel has none left.  Neither touches local memory, and ptxas reports no spills and
no injected wgmma wait (C7517) for them."""
import collections
import os
import re
import shutil
import subprocess

import pytest

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dawn_pytorch_b200")
LIB = os.path.join(PKG, "libdawn_unet.so")
KERNELS = ("sla_ctx_kernel", "sla_out_kernel")


@pytest.fixture(scope="module")
def sass():
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
            cnt[cur][m.group(1).split(".")[0]] += 1
    return cnt


def one(sass, kernel):
    found = {k: v for k, v in sass.items() if kernel in k}
    assert len(found) == 1, list(found)
    return next(iter(found.values()))


def test_context_kernel_sass(sass):
    c = one(sass, "sla_ctx_kernel")
    assert c["HGMMA"] >= 48 and c["HMMA"] > 0, dict(c)     # 4 weight tiles x 4 k-steps x 3 split terms; k^T v on mma.sync
    assert c["LDL"] == 0 and c["STL"] == 0, dict(c)


def test_output_kernel_sass(sass):
    c = one(sass, "sla_out_kernel")
    assert c["HGMMA"] >= 18 and c["HMMA"] == 0, dict(c)    # q: 4 k-steps x 3, Bf: 2 k-steps x 3
    assert c["LDL"] == 0 and c["STL"] == 0, dict(c)


@pytest.mark.parametrize("kernel", KERNELS)
def test_ptxas_report(kernel):
    log = os.path.join(PKG, "build", "sla_fused.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("no ptxas log (the library was not built in this tree)")
    with open(log) as fh:
        lines = fh.read().splitlines()
    assert not [ln for ln in lines if "C7517" in ln]
    start = [i for i, ln in enumerate(lines) if "Compiling entry function" in ln and kernel in ln]
    assert len(start) == 1, "no ptxas -v report for the kernel"
    block = []
    for ln in lines[start[0] + 1:]:
        if "Compiling entry function" in ln:
            break
        block.append(ln)
    spill = [ln for ln in block if "spill stores" in ln]
    assert spill and all(re.search(r"\b0 bytes spill stores, 0 bytes spill loads", ln) for ln in spill), block
