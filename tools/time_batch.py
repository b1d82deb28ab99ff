"""Per-clip time of a batched device-resident forward_x3 (B clips in one UNet pass) against B = 1, CUDA events after warm-up.

The configurations are measured round-robin in one process (each round times every configuration once), so drift of the
card affects all of them alike.  Every timed size also checks that each clip of the batched eps equals that clip's own B = 1
eps.  Prints the card name and power limit beside the table.

    python tools/time_batch.py [--rounds 3] [--iters 10]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import gpu_common as G  # noqa: E402

SHAPES = [(16, 32, 32, [1, 2, 4, 8]), (200, 32, 32, [1, 2, 4]), (200, 64, 64, [1, 2])]


def inputs(F, h, w, B):
    per = [G.clip(f"time_batch/{F}x{h}/{i}", F, h, w, 500) for i in range(B)]
    x_t = torch.cat([p[3] for p in per]).cuda().contiguous()
    fea = torch.cat([p[4] for p in per]).cuda().contiguous()
    cond = torch.cat([p[2] for p in per]).cuda().contiguous()
    t = torch.tensor([(500 + 97 * i) % 1000 for i in range(B)], dtype=torch.long, device="cuda")
    return x_t, fea, cond, t


def run(net, F, h, w, B, x_t, fea, cond, t, iters):
    net.update_num_frames(F)
    net.set_clip_invariants(fea, cond)
    out = net.forward_x3(x_t, t)                 # warm-up (and the eps that is checked)
    net.forward_x3(x_t, t)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        net.forward_x3(x_t, t)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / max(iters, 1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        card = torch.cuda.get_device_name()
    print(f"card: {card}")
    net = G.cuda_net()
    cfgs = [(F, h, w, B) for F, h, w, Bs in SHAPES for B in Bs]
    data = {c: inputs(*c) for c in cfgs}
    times = {c: [] for c in cfgs}
    with torch.no_grad():
        for _ in range(a.rounds):
            for c in cfgs:
                F, h, w, B = c
                x_t, fea, cond, t = data[c]
                inv = (fea, cond) if B > 1 else (fea[0], cond[0])
                xin = x_t if B > 1 else x_t[0]
                ms, _ = run(net, F, h, w, B, xin, *inv, t, a.iters)
                times[c].append(ms)
        # each clip of the batch equals its own single-clip pass
        worst = {}
        for c in cfgs:
            F, h, w, B = c
            if B == 1:
                continue
            x_t, fea, cond, t = data[c]
            _, yb = run(net, F, h, w, B, x_t, fea, cond, t, 0)
            r = 0.0
            for i in range(B):
                _, yi = run(net, F, h, w, 1, x_t[i], fea[i], cond[i], t[i:i + 1], 0)
                r = max(r, G.over_tol(yb[i], yi))
            worst[c] = r
    print(f"{'shape':>14} {'B':>2} {'ms/pass':>9} {'ms/clip':>9} {'spread':>7} {'vs B=1':>7} {'batched vs own (x tol)':>22}")
    base = {}
    for c in cfgs:
        F, h, w, B = c
        med = sorted(times[c])[len(times[c]) // 2]
        spread = max(times[c]) - min(times[c])
        if B == 1:
            base[(F, h, w)] = med
        gain = base[(F, h, w)] / (med / B)
        chk = f"{worst[c]:.4f}" if c in worst else "-"
        print(f"{F:>5} f x {h:>2}^2 {B:>2} {med:9.3f} {med / B:9.3f} {spread:7.3f} {gain:6.2f}x {chk:>22}")
    assert all(v <= 0.05 for v in worst.values()), worst


if __name__ == "__main__":
    main()
