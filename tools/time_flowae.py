"""Time FlowAE reconstructing a 256x256 clip (default 200 frames, the source repeated per frame as
LFG/test_flowautoenc_hdtf_video_256.py feeds it) per stage with CUDA events: regions (source and driving RegionPredictor calls,
including the host SVD), bg, flow and decode; against the oracle (oracle/lfg_motion_oracle.py) in eager torch fp32 on the same GPU
with TF32 off.  Synthetic weights (oracle/lfg_motion_oracle.py).  Prints one line per measurement and the card's name and power limit.

    python tools/time_flowae.py [--frames 200] [--reps 3] [--oracle-frames 50]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import lfg_motion_oracle as M   # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except FileNotFoundError:
        return torch.cuda.get_device_name()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-frames", type=int, default=50, help="frames of the oracle run (its time is scaled to --frames)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_flowae.py measures on the GPU"
    from dawn_pytorch_b200 import FlowAE
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "lfg_motion_schema.json")) as f:
        import json
        sch = json.load(f)
    sds = {k: M.motion_synth_state_dict([(n, tuple(s)) for n, s in v]) for k, v in sch.items()}
    ae = FlowAE()
    for k, sd in sds.items():
        getattr(ae, k).load_state_dict(sd)
    ae = ae.cuda()
    n = args.frames
    src1, drv = M.motion_synth_inputs("time_flowae", n, 256, 256)
    src, drv = src1.expand(n, -1, -1, -1).contiguous().cuda(), drv.cuda()
    print(f"card: {card()}")
    stages = {}
    for rep in range(args.reps + 1):                      # rep 0 warms up every shape
        t = {}
        (sp, dp), t["regions"] = timed(lambda: (ae.region_predictor(src), ae.region_predictor(drv)))
        bg, t["bg"] = timed(lambda: ae.bg_predictor(src, drv))
        g = ae.generator
        m, t["flow"] = timed(lambda: g.flow(src[:1], dp, sp, bg))
        _, t["decode"] = timed(lambda: (g.forward_with_flow(src[:1], m["optical_flow"], m["occlusion_map"]), g.compute_fea(src[:1])))
        if rep:
            for k, v in t.items():
                stages.setdefault(k, []).append(v)
    total = 0.0
    for k, v in stages.items():
        best = min(v)
        total += best
        print(f"flowae {n} frames 256x256: {k:8s} {best:9.1f} ms  (best of {len(v)}; {best / n:.3f} ms/frame)")
    print(f"flowae {n} frames 256x256: total    {total:9.1f} ms  ({total / n:.3f} ms/frame)")
    no = min(args.oracle_frames, n)
    sd = {k: {n_: t_.cuda() for n_, t_ in v.items()} for k, v in sds.items()}
    cfg = M.MotionCfg()
    with torch.no_grad():
        for rep in range(2):
            o = {}
            (sp, dp), o["regions"] = timed(lambda: (M.region_predictor(sd["region_predictor"], cfg, src[:no]),
                                                    M.region_predictor(sd["region_predictor"], cfg, drv[:no])))
            bg, o["bg"] = timed(lambda: M.bg_predictor(sd["bg_predictor"], cfg, src[:no], drv[:no]))
            m, o["flow"] = timed(lambda: M.flow_predictor(sd["generator"], cfg, src[:no], dp, sp, bg))
            from oracle import lfg_oracle as L
            _, o["decode"] = timed(lambda: L.forward_with_flow(M.decode_sd(sd["generator"]), L.LfgCfg(), src[:1], m["optical_flow"],
                                                               m["occlusion_map"]))
    ototal = 0.0
    for k, v in o.items():
        scaled = v * n / no
        ototal += scaled
        print(f"oracle eager fp32 (TF32 off), {no} frames scaled to {n}: {k:8s} {scaled:9.1f} ms")
    print(f"oracle eager fp32 (TF32 off), {no} frames scaled to {n}: total    {ototal:9.1f} ms  -> library {ototal / total:.2f}x faster")


if __name__ == "__main__":
    main()
