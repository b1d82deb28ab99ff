"""GPU: tensor-core attention core vs the SIMT fp32 kernel on random q/k/v; each case in its own time-boxed subprocess."""
import ctypes
import subprocess
import sys

ATT_CASES = [(64, 16, 1), (16, 96, 1), (7, 23, 1), (256, 200, 1), (64, 400, 1), (8, 64, 0), (5, 16, 0), (3, 300, 0)]


def one_att(args):
    sys.path.insert(0, ".")
    from dawn_pytorch_b200 import _lib
    md, mr = ctypes.c_float(), ctypes.c_float()
    rc = _lib.lib.dawn_selftest_attention(*args, ctypes.byref(md), ctypes.byref(mr))
    print(f"attention (nseq, L, temporal)={args}: rc={rc} max|diff|={md.value:.3e} max|ref|={mr.value:.3f}"
          + ("" if rc == 0 else " ERR " + _lib.lib.dawn_last_error().decode()), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1:
        one_att(tuple(int(a) for a in sys.argv[1:]))
    else:
        for c in ATT_CASES:
            try:
                r = subprocess.run([sys.executable, __file__, *map(str, c)], timeout=90, capture_output=True, text=True)
                print(r.stdout.strip() or ("NO OUTPUT rc=%d %s" % (r.returncode, r.stderr[-300:])), flush=True)
            except subprocess.TimeoutExpired:
                print(f"attention {c}: TIMEOUT (hang)", flush=True)
