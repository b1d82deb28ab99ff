"""Classifier-free-guided DDIM sampling (cond_scale = 2, 20 steps): the eager loop (two UNet passes per step, conditioning
tables rebuilt before each) against the guided CUDA graph (one pass over the clip and its null twin per step, fused update).

CUDA events around whole `ddim_sample` calls after one warm-up call of each path (the graph's capture happens there); the
two paths alternate over the rounds and the median is reported.  Each path has its own UNet module (same weights), so the
alternation never switches a handle between the eager B = 1 and the guided B = 2 geometry, which would reallocate the
workspace and drop the captured graph; the tool asserts that neither handle changed geometry and that the graph was captured
once.  Both paths draw the same noise, and the max |d| between their samples is printed.  Prints the card name and power
limit beside the table.

    python tools/time_guided.py [--rounds 3] [--steps 20]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import gpu_common as G  # noqa: E402

SHAPES = [(16, 32, 32), (200, 64, 64)]


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--cond-scale", type=float, default=2.0)
    a = ap.parse_args()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        card = torch.cuda.get_device_name()
    print(f"card: {card}")
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion, DynamicNfUnet3D
    nets = {False: G.cuda_net()}                                  # eager: B = 1
    nets[True] = DynamicNfUnet3D(**G.CTOR).eval()                 # guided graph: B = 2, its own handle
    nets[True].load_state_dict(G.synth_sd(), strict=True)
    nets[True] = nets[True].cuda()
    rows = []
    for F, h, w in SHAPES:
        Ds = {g: DynamicNfGaussianDiffusion(denoise_fn=nets[g], num_frames=F, image_size=h, sampling_timesteps=a.steps, timesteps=1000,
                                            loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0).cuda()
              for g in (False, True)}
        for D in Ds.values():
            D.update_num_frames(F)
        _, _, cond, _, fea = G.clip(f"time_guided/{F}x{h}", F, h, w, 500)
        fea, cond = fea.cuda(), cond.cuda()
        gen = torch.Generator(device="cuda").manual_seed(0)
        noise = {k: torch.randn(3, F, h, w, device="cuda", generator=gen) for k in range(-1, a.steps)}

        def sample(graph):
            return Ds[graph].ddim_sample(fea, (1, 3, F, h, w), cond=cond, cond_scale=a.cond_scale,
                                         noise_fn=lambda k, s: noise[k].reshape(s), use_graph=graph)
        with torch.no_grad():
            out = {g: timed(lambda: sample(g))[1].clone() for g in (False, True)}          # warm-up, capture
            gens = {g: nets[g].graph_generation() for g in (False, True)}
            times = {False: [], True: []}
            for _ in range(a.rounds):
                for g in (False, True):
                    ms, _ = timed(lambda: sample(g))
                    times[g].append(ms)
        # the timed calls neither re-sized a workspace nor re-captured the graph
        assert all(nets[g].graph_generation() == gens[g] for g in (False, True)), "a handle changed geometry while timed"
        assert nets[False].clip_count() == 1 and nets[True].clip_count() == 2
        assert Ds[True]._guided_captures == 1, Ds[True]._guided_captures
        med = {g: sorted(v)[len(v) // 2] for g, v in times.items()}
        spread = {g: max(v) - min(v) for g, v in times.items()}
        rows.append((F, h, w, med, spread, (out[True] - out[False]).abs().max().item()))
    print(f"cond_scale {a.cond_scale}, {a.steps} DDIM steps, median of {a.rounds} alternating rounds")
    print(f"{'shape':>14} {'eager ms':>10} {'spread':>8} {'graph ms':>10} {'spread':>8} {'graph/eager':>11} {'max|d|':>9}")
    for F, h, w, med, spread, d in rows:
        print(f"{F:>5} f x {h:>2}^2 {med[False]:10.1f} {spread[False]:8.1f} {med[True]:10.1f} {spread[True]:8.1f} "
              f"{med[True] / med[False]:10.3f}x {d:9.2e}")


if __name__ == "__main__":
    main()
