"""Wall time of re-sampling a real clip's motion against sampling it from noise, on one GPU:
   python tools/time_resample.py [--frames 200] [--size 128] [--steps 20] [--start 10] [--graph]
DAWN-128 by default: FlowDiffusion.resample_video (q_sample at step `start`, then steps start..steps-1 of the DDIM schedule, then
the decode) against sample_one_video (all steps, then the decode), and on their own the q_sample of the clip's latent and the
motion -> latent pass (flow and occlusion of every frame -> x0, plain and fused with the noising), timed with CUDA events.
Synthetic weights and inputs.  Prints one JSON line with the GPU's name and power limit beside the times."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import lfg_oracle as L        # noqa: E402
from oracle import weights as W           # noqa: E402
from oracle.make_golden_e2e import face_sd   # noqa: E402
from tests import gpu_common as G         # noqa: E402


def build_model(steps):
    from dawn_pytorch_b200 import FlowDiffusion
    m = FlowDiffusion(sampling_timesteps=steps, pose_dim=6, win_width=40, ddim_sampling_eta=1.0)
    m.diffusion.load_state_dict({**{"denoise_fn." + k: v for k, v in G.synth_sd().items()},
                                 **{k: v for k, v in m.diffusion.state_dict().items() if not k.startswith("denoise_fn.")}}, strict=True)
    m.generator.load_state_dict(W.lfg_synth_state_dict(L.state_dict_schema()), strict=True)
    m.face_loc_emb.load_state_dict(face_sd(), strict=True)
    return m.cuda()


def event_ms(fn, reps=20):
    fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--size", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--start", type=int, default=10)
    ap.add_argument("--graph", action="store_true", help="run both samplers as CUDA graphs")
    args = ap.parse_args()
    nf, S, ns, start = args.frames, args.size, args.steps, args.start
    m = build_model(ns)
    m.update_num_frames(nf)
    img = torch.from_numpy(W.uniform01("time_resample/img", 3 * S * S).reshape(1, 3, S, S)).cuda()
    hubert = torch.from_numpy(W.pseudo_normal("time_resample/hubert", (1, nf, 1024))).cuda()
    pose = torch.from_numpy(W.symmetric("time_resample/pose", (1, 7, nf), 0.3)).cuda()
    eye = torch.from_numpy(W.uniform01("time_resample/eye", 2 * nf).reshape(1, 2, nf)).cuda()
    bbox = torch.tensor([[20., 44., 16., 50., 64., 64.]]).unsqueeze(-1).repeat(1, 1, nf).cuda()
    h = S // 4
    flow = torch.tanh(torch.from_numpy(W.pseudo_normal("time_resample/flow", (nf, h, h, 2)))).cuda()
    occ = torch.from_numpy(W.uniform01("time_resample/occ", nf * h * h).reshape(nf, 1, h, h)).cuda()
    D = m.diffusion
    x0 = D.motion_to_latent(flow, occ, nf)
    t = torch.full((1,), D.ddim_schedule()[start][0], dtype=torch.long, device="cuda")
    z = torch.randn_like(x0)
    gen = dict(sample_img=img, sample_audio_hubert=hubert, sample_pose=pose, sample_eye=eye, sample_bbox=bbox, cond_scale=1.0,
               use_graph=args.graph)

    def wall(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    full = lambda: m.sample_one_video(**gen)                            # noqa: E731
    part = lambda: m.resample_video(x0=x0, start=start, **gen)          # noqa: E731
    full(), part()                                                      # warm-up (and graph captures)
    s_full = [wall(full) for _ in range(3)]
    s_part = [wall(part) for _ in range(3)]
    ms_q = event_ms(lambda: D.q_sample(x0, t, noise=z))
    ms_m = event_ms(lambda: D.motion_to_latent(flow, occ, nf))
    ms_mq = event_ms(lambda: D.motion_to_latent(flow, occ, nf, t=t, noise=z))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"workload": f"DAWN-{S}, {nf} frames, {h}x{h} latent, {ns}-step DDIM, resample from step {start}, one clip, "
                                  f"{'graph' if args.graph else 'eager'} sampler",
                      "sample_one_video_s": round(float(np.median(s_full)), 3), "resample_video_s": round(float(np.median(s_part)), 3),
                      "resample_over_sample": round(float(np.median(s_part) / np.median(s_full)), 3),
                      "q_sample_ms": round(ms_q, 4), "motion_to_latent_ms": round(ms_m, 4), "motion_to_xt_fused_ms": round(ms_mq, 4),
                      "latent_mb": round(x0.numel() * 4 / 2 ** 20, 2),
                      "gpu": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}))


if __name__ == "__main__":
    main()
