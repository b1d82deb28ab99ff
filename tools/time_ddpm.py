"""Wall time of one whole ancestral (DDPM) sampling loop, eager against the step graph, on one GPU:
   python tools/time_ddpm.py [--frames 16] [--size 32] [--timesteps 1000]
Synthetic weights and inputs; the default noise with one seed for both loops, so the two samples must agree.
Prints one JSON line with the GPU's name and power limit beside the times."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import weights as W            # noqa: E402
from tests import gpu_common as G          # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--size", type=int, default=32)
    ap.add_argument("--timesteps", type=int, default=1000)
    args = ap.parse_args()
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion
    Fr, hw, T = args.frames, args.size, args.timesteps
    D = DynamicNfGaussianDiffusion(denoise_fn=G.cuda_net(), num_frames=40, image_size=32, sampling_timesteps=None, timesteps=T,
                                   loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0).cuda()
    D.update_num_frames(Fr)
    _, fea, cond = W.synth_inputs("ddpm_timing", Fr, hw, hw)
    fea, cond = fea.cuda(), cond.cuda()
    shape = (1, 3, Fr, hw, hw)

    def run(use_graph):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = D.p_sample_loop(fea, shape, cond=cond, use_graph=use_graph, seed=0)
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0

    x = torch.randn(shape, device="cuda")
    for t in (T - 1, T // 2, 0):                   # warm the eager step's kernels and allocations
        D.p_sample(x, t, fea, cond=cond)
    eager, s_eager = run(False)
    _, s_first_graph = run(True)                   # includes the capture of the step graph
    graph, s_graph = run(True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"workload": f"p_sample_loop, {T} steps, {Fr} frames, {hw}x{hw} latent, one clip",
                      "eager_s": round(s_eager, 3), "graph_s": round(s_graph, 3), "graph_first_call_s": round(s_first_graph, 3),
                      "eager_ms_per_step": round(1e3 * s_eager / T, 3), "graph_ms_per_step": round(1e3 * s_graph / T, 3),
                      "max_abs_diff_graph_vs_eager": (graph - eager).abs().max().item(),
                      "gpu": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}))


if __name__ == "__main__":
    main()
