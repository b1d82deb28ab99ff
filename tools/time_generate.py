"""Time the talking-head generator (dawn_pytorch_b200/generate.py) at DAWN-128 and DAWN-256: 8 s of speech, 200 frames, 20 DDIM
steps, synthetic weights at the shipped shapes (hubert-large, PBnet reemb5 with 4 layers and ff 1024, the sample_one_video UNet,
the hdtf LFG decoder).  Prints the card's name and power limit, each handle's workspace bytes, and per resolution:

* the whole call, including the copy of the frames to the host (host clock around a call that ends in a synchronise);
* its stages one after the other with CUDA events: audio, pose/blink, resize, sampling, decode (8-bit RGB), copy to host;
* the fp32 decode and UVG:383-392 / 544-548's per-frame numpy conversion on the same clip, next to the rgb8 decode + copy.

Each number is the median and range of --reps repeats after one warm-up call.

    python tools/time_generate.py [--sizes 128 256] [--reps 3] [--frames 200] [--steps 20]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import hubert_oracle as HO    # noqa: E402
from oracle import lfg_oracle as L        # noqa: E402
from oracle import pbnet_oracle as P      # noqa: E402
from oracle import weights as W           # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except FileNotFoundError:
        return torch.cuda.get_device_name()


def stats(ms):
    ms = sorted(ms)
    return f"{ms[len(ms) // 2]:9.1f} ms [{ms[0]:.1f}, {ms[-1]:.1f}]"


def build(size, steps):
    from dawn_pytorch_b200 import FlowDiffusion, HubertModel, TalkingHeadGenerator, get_pbnet_model
    from oracle.make_golden_e2e import face_sd
    from tests import gpu_common as G
    fd = FlowDiffusion(sampling_timesteps=steps, pose_dim=6, win_width=40, ddim_sampling_eta=1.0)
    fd.diffusion.load_state_dict({**{"denoise_fn." + k: v for k, v in G.synth_sd().items()},
                                  **{k: v for k, v in fd.diffusion.state_dict().items() if not k.startswith("denoise_fn.")}})
    fd.generator.load_state_dict(W.lfg_synth_state_dict(L.state_dict_schema()))
    fd.face_loc_emb.load_state_dict(face_sd())
    hub = HubertModel(HO.LARGE)
    hub.load_state_dict(HO.synth_state_dict(HO.schema_of(HO.LARGE)))

    def pbnet(cfg):
        m = get_pbnet_model(cfg.parameters("cuda:0"))
        m.load_state_dict(P.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()]))
        return m.eval()
    pose = pbnet(P.PbCfg(pos_dim=6, eye_dim=0, ff_size=1024, num_layers=4))
    blink = pbnet(P.PbCfg(pos_dim=0, eye_dim=2, ff_size=1024, num_layers=4))
    vc = dict(input_size=size, max_n_frames=200, mean=[0.0, 0.0, 0.0], cond_scale=1.0)
    return TalkingHeadGenerator(fd.cuda(), hub.cuda().eval(), pose, blink, vc)


def staged(gen, portrait, speech, n_all, F):
    """the call's stages one after the other (as __call__ runs them), each bracketed by CUDA events -> {stage: ms}"""
    from dawn_pytorch_b200.generate import finish_pose_blink, pbnet_initial_states, portrait_resize
    from dawn_pytorch_b200.hubert import hubert_features
    dev = torch.device("cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(7)]
    ev[0].record()
    feats = hubert_features(gen.hubert, speech)
    ev[1].record()
    p0, b0 = pbnet_initial_states(None, None, dev)
    dur = torch.tensor([n_all])
    out_p = gen.pose_model.generate(p0, feats.unsqueeze(0), dur, fact=1)["output"]
    out_b = gen.blink_model.generate(b0, feats.unsqueeze(0), dur, fact=1)["output"]
    pose, blink = finish_pose_blink(out_p, out_b, p0, b0)
    ev[2].record()
    source = portrait_resize(portrait.to(dev), gen.video_config["input_size"])
    ev[3].record()
    fd = gen.flow_diffusion
    fd.update_num_frames(F)
    bbox = torch.tensor([[64., 192., 64., 192., 256., 256.]], device=dev).reshape(1, 6, 1)
    pred = fd._sample_latent(source[None], feats[:F][None], pose[:F].T[None], blink[:F].T[None], bbox, 1.0,
                             torch.zeros(1, 7, device=dev), torch.full((1, 2), 0.3, device=dev), None, True)
    ev[4].record()
    frames = fd.generator.decode_sample_rgb8(source[None], pred[0], gen.video_config["mean"])
    ev[5].record()
    host = frames.cpu()
    ev[6].record()
    torch.cuda.synchronize()
    names = ["audio", "pose/blink", "resize", "sampling", "decode rgb8", "copy to host"]
    return {n: ev[i].elapsed_time(ev[i + 1]) for i, n in enumerate(names)}, (source, pred, host)


def fp32_path(gen, source, pred, mean):
    """sample_one_video's fp32 decode, then UVG:383-392 / 544-548: each frame to the host and to 8 bits in numpy"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    vid = gen.flow_diffusion.generator.decode_sample(source[None], pred[0])
    frames = []
    for f in range(vid.shape[0]):
        frame = vid[f].permute(1, 2, 0).data.cpu().numpy().copy()
        frame += np.array(mean) / 255.0
        frame = np.clip(frame, 0, 1)
        frames.append((frame * 255).astype(np.uint8))
    return (time.perf_counter() - t0) * 1e3, np.stack(frames)


def rgb8_path(gen, source, pred, mean):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    frames = gen.flow_diffusion.generator.decode_sample_rgb8(source[None], pred[0], mean).cpu().numpy()
    return (time.perf_counter() - t0) * 1e3, frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_generate.py measures on the GPU"
    print(f"card: {card()}")
    n = int(args.frames / 25 * 16000)                                  # 8 s of speech for 200 frames
    speech = HO.synth_speech("time_generate", n)
    portrait = torch.from_numpy((W.uniform01("time_generate/portrait", 720 * 540 * 3).reshape(720, 540, 3) * 255).astype(np.uint8))
    for size in args.sizes:
        gen = build(size, args.steps)
        n_all = int(n / 16000 * 25)

        def whole():
            out = gen(portrait, speech, seed=0)
            return out["frames"].cpu()
        whole()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            whole()
            torch.cuda.synchronize()
            ms.append((time.perf_counter() - t0) * 1e3)
        staged(gen, portrait, speech, n_all, args.frames)
        per = {}
        for _ in range(args.reps):
            st, keep = staged(gen, portrait, speech, n_all, args.frames)
            for k, v in st.items():
                per.setdefault(k, []).append(v)
        source, pred, _ = keep
        mean = [0.0, 0.0, 0.0]
        fp32_path(gen, source, pred, mean)
        rgb8_path(gen, source, pred, mean)
        t32, t8 = [], []
        for _ in range(args.reps):
            a, f32 = fp32_path(gen, source, pred, mean)
            b, f8 = rgb8_path(gen, source, pred, mean)
            t32.append(a)
            t8.append(b)
        assert np.array_equal(f32, f8), "the rgb8 decode differs from the fp32 decode's numpy conversion"
        fd = gen.flow_diffusion
        print(f"DAWN-{size}: {args.frames} frames, {args.steps} steps, {n / 16000:.1f} s of speech")
        print(f"  whole call + frames to host {stats(ms)}")
        for k, v in per.items():
            print(f"  {k:<28s}{stats(v)}")
        print(f"  fp32 decode + numpy 8-bit   {stats(t32)}")
        print(f"  rgb8 decode + copy to host  {stats(t8)}")
        print(f"  workspace bytes: unet {fd.unet.workspace_bytes()}, lfg {fd.generator.workspace_bytes()}, "
              f"hubert {gen.hubert.workspace_bytes()}, pbnet pose {gen.pose_model.workspace_bytes()}, "
              f"blink {gen.blink_model.workspace_bytes()}; peak allocated by torch {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
        del gen, fd
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
