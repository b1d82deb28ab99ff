"""GPU: wgmma GEMM vs mma.sync GEMM on random convs; each case in its own time-boxed subprocess."""
import ctypes
import subprocess
import sys

CASES = [  # F, H, W, Cin, N, k, stats
    (2, 16, 16, 64, 64, 1, 0),
    (2, 16, 16, 64, 64, 3, 1),
    (3, 9, 9, 64, 64, 3, 1),        # M = 243: ragged last tile
    (8, 32, 32, 64, 64, 3, 1),
    (4, 16, 16, 128, 128, 3, 1),
    (2, 16, 16, 256, 512, 1, 0),
    (16, 8, 8, 1024, 256, 3, 1),
    (40, 64, 64, 64, 64, 3, 1),     # 1280 tiles: persistent loop over many tiles per CTA
    (100, 64, 64, 64, 64, 3, 1),
    (100, 32, 32, 128, 128, 3, 1),
    (100, 64, 64, 64, 768, 1, 0),
]


def one(args):
    sys.path.insert(0, ".")
    from dawn_pytorch_b200 import _lib
    md, mr = ctypes.c_float(), ctypes.c_float()
    rc = _lib.lib.dawn_selftest_tc_gemm(*args, ctypes.byref(md), ctypes.byref(mr))
    print(f"case {args}: rc={rc} max|diff|={md.value:.3e} max|ref|={mr.value:.3f} rel={md.value / max(mr.value, 1e-9):.2e}"
          + ("" if rc == 0 else " ERR " + _lib.lib.dawn_last_error().decode()), flush=True)


ATT_CASES = [(64, 16, 1), (16, 96, 1), (7, 23, 1), (256, 200, 1), (64, 400, 1), (8, 64, 0), (5, 16, 0), (3, 300, 0)]


def one_att(args):
    sys.path.insert(0, ".")
    from dawn_pytorch_b200 import _lib
    md, mr = ctypes.c_float(), ctypes.c_float()
    rc = _lib.lib.dawn_selftest_attention(*args, ctypes.byref(md), ctypes.byref(mr))
    print(f"attention (nseq, L, temporal)={args}: rc={rc} max|diff|={md.value:.3e} max|ref|={mr.value:.3f}"
          + ("" if rc == 0 else " ERR " + _lib.lib.dawn_last_error().decode()), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "att":
        if len(sys.argv) > 2:
            one_att(tuple(int(a) for a in sys.argv[2:]))
        else:
            for c in ATT_CASES:
                try:
                    r = subprocess.run([sys.executable, __file__, "att", *map(str, c)], timeout=90, capture_output=True, text=True)
                    print(r.stdout.strip() or ("NO OUTPUT rc=%d %s" % (r.returncode, r.stderr[-300:])), flush=True)
                except subprocess.TimeoutExpired:
                    print(f"attention {c}: TIMEOUT (hang)", flush=True)
    elif len(sys.argv) > 1:
        one(tuple(int(a) for a in sys.argv[1:]))
    else:
        for c in CASES:
            try:
                r = subprocess.run([sys.executable, __file__, *map(str, c)], timeout=90, capture_output=True, text=True)
                print(r.stdout.strip() or ("NO OUTPUT rc=%d %s" % (r.returncode, r.stderr[-300:])), flush=True)
            except subprocess.TimeoutExpired:
                print(f"case {c}: TIMEOUT (hang)", flush=True)
