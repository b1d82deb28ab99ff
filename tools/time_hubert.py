"""Time the generator's audio stage, `hubert_features` (unified_video_generator.py:229-242, 450-501: normalisation, 20 s segments
through hubert-large, length fix-up, interpolation to 25 fps) with CUDA events, at 8 s (DAWN's 200 frames) and 60 s of audio:
the library against the float64 oracle's functional HubertModel run as eager torch fp32 on the same GPU with TF32 off, through
the same pipeline.  Synthetic hubert-large weights (oracle/hubert_oracle.py).  Prints the card's name and power limit, then one
line per length: median and range of the calls, and the largest difference between the two in units of the tolerance.

    python tools/time_hubert.py [--seconds 8 60] [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import hubert_oracle as O   # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except FileNotFoundError:
        return torch.cuda.get_device_name()


def timed(fn, reps):
    """per-call milliseconds of `reps` calls after one warm-up call, each bracketed by CUDA events"""
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return sorted(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, nargs="+", default=[8, 60])
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_hubert.py measures on the GPU"
    from dawn_pytorch_b200.hubert import HubertModel, hubert_features
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    with open(os.path.join(ROOT, "tests", "golden", "hubert_schema.json")) as f:
        schema = [(n, tuple(s)) for n, s in json.load(f)["large"]]
    sd = O.synth_state_dict(schema)
    model = HubertModel(O.LARGE).cuda()
    model.load_state_dict(sd)
    model.eval()
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    print(f"card: {card()}")
    for sec in args.seconds:
        speech = O.synth_speech(f"time/{sec}", int(sec * 16000))

        def lib_call():
            return hubert_features(model, speech)

        def oracle_call():
            return O.features(lambda v: O.forward(sd_dev, O.LARGE, v.cuda()), speech)

        with torch.no_grad():
            mine, ref = lib_call().cpu(), oracle_call()
            diff = ((mine.double() - ref.double()).abs() / (1e-4 + 1e-3 * ref.double().abs())).max().item()
            t_lib, t_ora = timed(lib_call, args.reps), timed(oracle_call, args.reps)
        med = lambda t: t[len(t) // 2]                                          # noqa: E731
        print(f"{sec:g} s ({mine.shape[0]} frames): hubert_features  library {med(t_lib):.2f} ms (range {t_lib[0]:.2f}-{t_lib[-1]:.2f}, "
              f"{model.last_launch_count()} launches in the last forward)  |  eager fp32 oracle {med(t_ora):.2f} ms "
              f"(range {t_ora[0]:.2f}-{t_ora[-1]:.2f})  |  speed-up {med(t_ora) / med(t_lib):.2f}x  |  "
              f"max |d| / (1e-4 + 1e-3 |ref|) = {diff:.3f}")


if __name__ == "__main__":
    main()
