"""Step time of the UNet's up-path variants at DAWN's size: forward_x3 over one 200-frame 64 x 64 clip with the ConvTranspose
(deconv), and with nearest x2 + 3x3 conv in zeros and in reflect padding.  CUDA events after warm-up; the variants are timed
round-robin in one process (each round times every variant once), so drift of the card affects all of them alike.  Prints the
card's name, power limit and SM clocks beside the table, and the up convs' share (conv_other category of the per-kernel profile,
which also holds the init, down and 1x1 convs) from one profiled step per variant.

    python tools/time_upconv.py [--rounds 5] [--iters 5] [--frames 200] [--size 64]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import weights as W  # noqa: E402
from tests import gpu_common as G  # noqa: E402

VARIANTS = {"deconv": dict(use_deconv=True), "upconv-zeros": dict(use_deconv=False, padding_mode="zeros"),
            "upconv-reflect": dict(use_deconv=False, padding_mode="reflect")}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name() + " (nvidia-smi unavailable: power limit and clocks not read)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--size", type=int, default=64)
    a = ap.parse_args()
    from dawn_pytorch_b200 import DynamicNfUnet3D
    print(f"card before: {card()}")
    F, s = a.frames, a.size
    _, t, cond, x_t, fea = G.clip("time_upconv", F, s, s, 500)
    x_t, t, cond, fea = x_t[0].cuda(), t.cuda(), cond[0].cuda(), fea[0].cuda()
    nets = {}
    for name, kw in VARIANTS.items():
        net = DynamicNfUnet3D(**{**G.CTOR, **kw}).eval()
        net.load_state_dict(W.synth_state_dict([(k, list(v.shape)) for k, v in net.state_dict().items()]), strict=True)
        net = net.cuda()
        net.update_num_frames(F)
        net.set_clip_invariants(fea, cond)
        for _ in range(3):                                            # warm-up: workspace, attributes, first launches
            net.forward_x3(x_t, t)
        nets[name] = net
    torch.cuda.synchronize()
    times = {n: [] for n in nets}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        for _ in range(a.rounds):
            for n, net in nets.items():
                e0.record()
                for _ in range(a.iters):
                    net.forward_x3(x_t, t)
                e1.record()
                torch.cuda.synchronize()
                times[n].append(e0.elapsed_time(e1) / a.iters)
        prof = {}
        for n, net in nets.items():
            net.profile(True)
            net.forward_x3(x_t, t)
            p = net.profile_read()
            net.profile(False)
            prof[n] = p["conv_other"]
    print(f"card after:  {card()}")
    print(f"forward_x3, {F} frames x {s}^2, {a.rounds} rounds x {a.iters} steps per variant")
    print(f"{'variant':>15} {'median ms':>10} {'min':>8} {'max':>8} {'conv_other ms':>14} {'launches':>9}")
    for n in nets:
        v = sorted(times[n])
        print(f"{n:>15} {v[len(v) // 2]:10.3f} {v[0]:8.3f} {v[-1]:8.3f} {prof[n]['ms']:14.3f} {prof[n]['count']:9d}")


if __name__ == "__main__":
    main()
