"""CPU: static checks of the wgmma kernels' register schedule in the built library (no GPU needed).

* The halo conv holds its 64 accumulators per row half in registers next to the operand descriptors; the producer, loader, MMA
  and epilogue warpgroups get their own register budgets (setmaxnreg), and no instantiation may touch local memory.
* ptxas injects a full `warpgroup.wait` (C7517) where it cannot prove that accumulator registers are left alone while a wgmma
  group is in flight.  That wait serialises the taps / K panels, so its message must not appear in the build logs."""
import collections
import os
import re
import shutil
import subprocess

import pytest

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dawn_pytorch_b200")
LIB = os.path.join(PKG, "libdawn_unet.so")


@pytest.fixture(scope="module")
def local_memory_ops():
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
        if m and m.group(1).split(".")[0] in ("STL", "LDL"):
            cnt[cur][m.group(1).split(".")[0]] += 1
    return cnt


def test_halo_conv_does_not_spill(local_memory_ops):
    ks = {k: v for k, v in local_memory_ops.items() if "tc_conv3_kernel" in k}
    assert len(ks) == 4
    for k, c in ks.items():
        assert c["STL"] == 0 and c["LDL"] == 0, (k, dict(c))


@pytest.mark.parametrize("unit", ["tc_conv3", "tc_gemm"])
def test_no_injected_wgmma_wait(unit):
    log = os.path.join(PKG, "build", unit + ".ptxas.log")
    if not os.path.exists(log):
        pytest.skip("no ptxas log (the library was not built in this tree)")
    with open(log) as fh:
        text = fh.read()
    assert "Compiling entry function" in text, "not a ptxas -v log"
    assert "C7517" not in text, [ln for ln in text.splitlines() if "C7517" in ln]
