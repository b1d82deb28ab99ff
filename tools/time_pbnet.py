"""Time PBnet's pose + blink generation (the two CVAE.generate calls of unified_video_generator.py:290-291) with CUDA events, at
200 frames and at 1500 frames (a minute of audio at 25 fps): the library against the oracle (oracle/pbnet_oracle.py) run as eager
torch fp32 on the same GPU with TF32 off, which computes every attention over all F x F frame pairs as the reference does.
Synthetic weights (oracle/pbnet_oracle.py).  Prints the card's name and power limit, then one line per length: median and range.

    python tools/time_pbnet.py [--frames 200 1500] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pbnet_oracle as P   # noqa: E402


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
    ap.add_argument("--frames", type=int, nargs="+", default=[200, 1500])
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_pbnet.py measures on the GPU"
    from dawn_pytorch_b200.pbnet import get_model
    torch.backends.cuda.matmul.allow_tf32 = False
    with open(os.path.join(ROOT, "tests", "golden", "pbnet_schema.json")) as f:
        schema = json.load(f)
    models = []
    for case in ("reemb5_pose_250", "reemb5_blink_37"):                     # DAWN's pose (6, 0) and blink (0, 2) models
        cfg, _ = P.CASES[case]
        sd = P.synth_state_dict([(n, tuple(s)) for n, s in schema[case]])
        m = get_model(cfg.parameters("cuda:0"))
        m.load_state_dict(sd)
        models.append((cfg, m, {k: v.cuda() for k, v in sd.items()}))
    print(f"card: {card()}")
    for F in args.frames:
        inputs = [tuple(t.cuda() for t in P.synth_inputs(f"time/{F}/{i}", cfg, [F])) for i, (cfg, _, _) in enumerate(models)]

        def lib_call():
            return [m.generate(pose, audio, lens, z=z)["output"] for (cfg, m, _), (pose, audio, z, lens) in zip(models, inputs)]

        def oracle_call():
            return [P.decoder_forward(sd, cfg, pose, audio, z, lens, dtype=torch.float32)
                    for (cfg, _, sd), (pose, audio, z, lens) in zip(models, inputs)]

        with torch.no_grad():
            mine, ref = lib_call(), oracle_call()
            diff = max(((a - b).abs() / (1e-4 + 1e-3 * b.abs())).max().item() for a, b in zip(mine, ref))
            t_lib, t_ora = timed(lib_call, args.reps), timed(oracle_call, args.reps)
        med = lambda t: t[len(t) // 2]                                          # noqa: E731
        print(f"F={F}: pose + blink generate  library {med(t_lib):.3f} ms (range {t_lib[0]:.3f}-{t_lib[-1]:.3f}, "
              f"{models[0][1].last_launch_count()} launches per model)  |  eager fp32 oracle {med(t_ora):.3f} ms "
              f"(range {t_ora[0]:.3f}-{t_ora[-1]:.3f})  |  speed-up {med(t_ora) / med(t_lib):.1f}x  |  "
              f"library vs fp32 oracle {diff:.3g} x tol")


if __name__ == "__main__":
    main()
