"""DAWN's talking-head generator in one call: a portrait and 16 kHz speech -> the clip's 8-bit RGB frames on the device.

`TalkingHeadGenerator` computes what the reference's unified_video_generator.py ("UVG") computes between reading its inputs and
writing its video (`process_audio`, `generate_pose_blink`, `generate_final_video`, UVG:202-400), without the `.npy` cache, the
host-side resize and the per-frame numpy conversion:

  audio       hubert_features: HuBERT, the 20 s segments and the 25 fps interpolation (UVG:229-242, 433-501)
  pose/blink  PBnet's pose and blink generators over all frames of the audio, then the inverse normalisation (UVG:252-302)
  source      the portrait resized to `input_size` by Pillow's bilinear resampler and scaled as ToTensor / * 255 / / 255 do
              (UVG:320-325, 372), on the device (`dawn_portrait_resize`, include/dawn_video.h)
  sampling    FlowDiffusion's conditioning and sampling loop (the code sample_one_video runs, FD:327-365)
  frames      the LFG decoder storing 8-bit RGB straight from its last kernel (UVG:544-548; `dawn_lfg_decode_sample_rgb8`)

Face detection and the 3DDFA initial states, audio decoding / resampling, and video writing stay with the caller: the initial
pose and eye / face box are inputs (UVG's fallbacks when absent), and the result holds the frames and the frame rate.
"""
import os

import numpy as np
import torch

from ._lib import DawnError, check, lib, ptr, stream
from .flow_diffusion import FlowDiffusion
from .hubert import KERNEL, HubertModel, hubert_features
from .pbnet import get_model as get_pbnet_model

FPS = 25
# PBnet's pose normalisation (UVG:95-98): yaw, pitch, roll, scale, tx, ty
POSE_MAX = (90., 90., 90., 1., 720., 1080.)
POSE_MIN = (-90., -90., -90., 0., 0., 0.)
# UVG's fallbacks when 3DDFA found no initial state: the PBnet stage's (UVG:276-279) differ from the video stage's (UVG:338-341)
PBNET_FALLBACK_POSE = [[0, 0, 0, 4.79e-04, 5.65e+01, 6.49e+01]]
PBNET_FALLBACK_BLINK = [[0.3, 0.3]]
VIDEO_FALLBACK_EYE_BBOX = [[0.3, 0.3, 64, 64, 192, 192, 256, 256]]
# the release tree's PBnet checkpoints and HuBERT directory (UVG:69-75)
POSE_CKPT = os.path.join("pretrain_models", "pbnet_seperate", "pose", "checkpoint_40000.pth.tar")
BLINK_CKPT = os.path.join("pretrain_models", "pbnet_seperate", "blink", "checkpoint_95000.pth.tar")
HUBERT_DIR = os.path.join("pretrain_models", "hubert-large-ls960-ft")


def inv_transform(x, min_vals, max_vals):
    """UVG:31-32"""
    return x * (max_vals - min_vals) + min_vals


def portrait_array(portrait):
    """A path, a PIL image, or an (H, W, 3) uint8 RGB array / tensor -> (H, W, 3) uint8 tensor on the host.  Files are decoded and
    converted to RGB by PIL, as UVG:320 does."""
    from PIL import Image
    if isinstance(portrait, (str, os.PathLike)):
        with Image.open(portrait) as im:
            portrait = im.convert("RGB")
    elif isinstance(portrait, Image.Image):
        portrait = portrait.convert("RGB")
    if isinstance(portrait, Image.Image):
        return torch.from_numpy(np.array(portrait, dtype=np.uint8))
    t = portrait if torch.is_tensor(portrait) else torch.from_numpy(np.asarray(portrait))
    if t.dim() != 3 or t.shape[2] != 3 or t.dtype != torch.uint8 or t.shape[0] < 1 or t.shape[1] < 1:
        raise ValueError(f"portrait must be an (H, W, 3) uint8 RGB image, got {tuple(t.shape)} {t.dtype}")
    return t


def portrait_resize(img, size, with_resized=False):
    """(H0, W0, 3) uint8 RGB on a CUDA device -> source (3, size, size) fp32 = ToTensor(img.resize((size, size), BILINEAR)) * 255
    / 255, bit for bit as PIL and torch compute it on the host (UVG:320-325, 372); with_resized also returns the resized (size,
    size, 3) uint8 image."""
    if img.device.type != "cuda":
        raise DawnError("dawn_portrait_resize runs on CUDA (sm_90a) only; there is no CPU path")
    img = img.contiguous()
    H0, W0, _ = img.shape
    source = torch.empty((3, size, size), device=img.device, dtype=torch.float32)
    resized = torch.empty((size, size, 3), device=img.device, dtype=torch.uint8) if with_resized else None
    with torch.cuda.device(img.device):
        check(lib.dawn_portrait_resize(ptr(img), H0, W0, size, ptr(source), ptr(resized), stream()), "dawn_portrait_resize")
    return (source, resized) if with_resized else source


def _state(value, shape, what):
    """an initial state as the reference loads it from its .npy file: a float32 tensor of `shape` on the host"""
    t = value if torch.is_tensor(value) else torch.from_numpy(np.asarray(value))
    if tuple(t.shape) != shape:
        raise ValueError(f"{what} must have shape {shape} (what the reference's 3DDFA stage saves), got {tuple(t.shape)}")
    return t.detach().cpu()


def _pose_range(device):
    return (torch.tensor(POSE_MIN, dtype=torch.float32, device=device).reshape(1, 1, 6),
            torch.tensor(POSE_MAX, dtype=torch.float32, device=device).reshape(1, 1, 6))


def pbnet_initial_states(init_pose, init_eye_bbox, device):
    """PBnet's first pose (1, 1, 6), normalised, and first blink (1, 1, 2) on `device` (UVG:270-282): from init_pose (1, 7) and
    init_eye_bbox (1, 8) when both are given, otherwise UVG's fallback, built in float64 and cast.  One torch op per reference op,
    in fp32: the result does not depend on the device."""
    if init_pose is not None and init_eye_bbox is not None:                          # UVG:272-273
        pose, blink = torch.as_tensor(init_pose), torch.as_tensor(init_eye_bbox)
    else:                                                                             # UVG:277-278
        pose, blink = torch.from_numpy(np.array(PBNET_FALLBACK_POSE)), torch.from_numpy(np.array(PBNET_FALLBACK_BLINK))
    pose = pose[:, :6].unsqueeze(0).to(torch.float32).to(device)
    blink = blink[:, :2].unsqueeze(0).to(torch.float32).to(device)
    min_vals, max_vals = _pose_range(device)
    return (pose - min_vals) / (max_vals - min_vals), blink                          # UVG:282


def finish_pose_blink(out_p, out_b, p0, b0):
    """PBnet's outputs (1, F, 6) / (1, F, 2) -> the driving pose (F, 6) and blink (F, 2) UVG:294-302 saves: the initial state
    added back and the pose's normalisation inverted, in the reference's fp32 operation order"""
    min_vals, max_vals = _pose_range(out_p.device)
    out_p = out_p + p0
    out_p = inv_transform(out_p, min_vals, max_vals)
    out_b = out_b + b0
    return out_p[0], out_b[0]


class TalkingHeadGenerator:
    """DAWN's generator (UVG:202-400) over this package's modules: `flow_diffusion` a FlowDiffusion, `hubert` a HubertModel,
    `pose_model` / `blink_model` PBnet CVAEs (get_pbnet_model), `video_config` the dict of config/DAWN_{128,256}.yaml (input_size,
    max_n_frames, mean and cond_scale are read).  All modules on one CUDA device."""

    def __init__(self, flow_diffusion, hubert, pose_model, blink_model, video_config):
        self.flow_diffusion, self.hubert = flow_diffusion, hubert
        self.pose_model, self.blink_model = pose_model, blink_model
        self.video_config = dict(video_config)

    @classmethod
    def from_release(cls, root, resolution=128, device="cuda"):
        """Everything UVG:60-124 and 504-531 load, from a DAWN release tree at `root` (every path relative to it):
        config/DAWN_{resolution}.yaml and the LFG config, LFG and diffusion checkpoints its model_config names; the PBnet pose and
        blink checkpoints with their opt.yaml (audio_dim 1024, pos_dim 6 / 0, eye_dim 0 / 2, as UVG:81-92 set); and
        pretrain_models/hubert-large-ls960-ft.  As in the reference, FlowDiffusion's `face_loc_emb` is never loaded from a
        checkpoint: it keeps its default (seeded by torch's global RNG) initialisation, as the reference's does."""
        import yaml
        rel = lambda p: os.path.normpath(os.path.join(root, p))            # noqa: E731
        cfg_path = rel(os.path.join("config", f"DAWN_{int(resolution)}.yaml"))
        if not os.path.isfile(cfg_path):
            raise FileNotFoundError(f"DAWN release file missing: {cfg_path}")
        with open(cfg_path) as f:
            video_config = yaml.safe_load(f)
        mc = video_config["model_config"]
        hubert_dir = rel(HUBERT_DIR)
        needed = [rel(mc["config_pth"]), rel(mc["ae_pretrained_pth"]), rel(mc["diffusion_pretrained_pth"]), rel(POSE_CKPT),
                  os.path.join(os.path.dirname(rel(POSE_CKPT)), "opt.yaml"), rel(BLINK_CKPT),
                  os.path.join(os.path.dirname(rel(BLINK_CKPT)), "opt.yaml"), os.path.join(hubert_dir, "config.json")]
        for p in needed:
            if not os.path.isfile(p):
                raise FileNotFoundError(f"DAWN release file missing: {p}")
        if not any(os.path.isfile(os.path.join(hubert_dir, w)) for w in ("model.safetensors", "pytorch_model.bin")):
            raise FileNotFoundError(f"DAWN release file missing: {os.path.join(hubert_dir, 'model.safetensors')}")
        fd = FlowDiffusion(is_train=mc["is_train"], sampling_timesteps=video_config["sampling_step"],
                           ddim_sampling_eta=video_config["ddim_sampling_eta"], pose_dim=mc["pose_dim"],
                           config_pth=rel(mc["config_pth"]), pretrained_pth=rel(mc["ae_pretrained_pth"]),
                           win_width=video_config["win_width"])                                          # UVG:504-524
        fd.diffusion.load_state_dict(torch.load(rel(mc["diffusion_pretrained_pth"]), map_location="cpu")["diffusion"])   # :527-528
        fd = fd.to(device).eval()
        hubert = HubertModel.from_pretrained(hubert_dir).to(device).eval()                                # UVG:69-72

        def pbnet(ckpt, pos_dim, eye_dim):                                                               # UVG:79-112
            with open(os.path.join(os.path.dirname(ckpt), "opt.yaml"), "rb") as f:
                params = yaml.load(f, Loader=yaml.Loader)            # the reference's load_args (UVG:34-37)
            params.update(device=device, audio_dim=1024, pos_dim=pos_dim, eye_dim=eye_dim)
            model = get_pbnet_model(params)
            model.load_state_dict(torch.load(ckpt, map_location="cpu"))
            return model.eval()

        return cls(fd, hubert, pbnet(rel(POSE_CKPT), 6, 0), pbnet(rel(BLINK_CKPT), 0, 2), video_config)

    def _device(self):
        devs = {next(self.flow_diffusion.parameters()).device, next(self.hubert.parameters()).device,
                self.pose_model.decoder.finallayer.weight.device, self.blink_model.decoder.finallayer.weight.device}
        if any(d.type != "cuda" for d in devs):
            raise DawnError("TalkingHeadGenerator runs on CUDA (sm_90a) only: move its modules to a CUDA device")
        if len(devs) != 1:
            raise DawnError(f"TalkingHeadGenerator's modules must share one device, found {sorted(map(str, devs))}")
        return devs.pop()

    @torch.no_grad()
    def __call__(self, portrait, speech_16k, init_pose=None, init_eye_bbox=None, max_frames=None, seed=None, use_graph=True, *,
                 pose_z=None, blink_z=None, noise_fn=None):
        """portrait: a path, a PIL image or an (H, W, 3) uint8 RGB array / tensor; speech_16k: 16 kHz samples, (N,) or (N, channels)
        (channel 0 is used); init_pose (1, 7) and init_eye_bbox (1, 8): the reference's 3DDFA outputs (yaw, pitch, roll, scale, tx,
        ty, _ and left / right eye ratio, face box x0, x1, y0, y1, image width, height), UVG's fallbacks when None; max_frames caps
        the clip below video_config's max_n_frames; seed seeds PBnet's draws and the sampler noise on the device (torch's global
        RNG otherwise); use_graph replays the sampling loop as one CUDA graph.

        Returns a dict: frames (F, H, W, 3) uint8 RGB on the device, fps 25, num_frames F, and what UVG caches: audio_features
        (F_all, 1024), drive_pose (F_all, 6), drive_blink (F_all, 2) over the whole audio."""
        vc = self.video_config
        img = portrait_array(portrait)
        speech = speech_16k.detach().cpu().numpy() if torch.is_tensor(speech_16k) else np.asarray(speech_16k)
        if speech.ndim not in (1, 2) or speech.shape[0] < KERNEL:
            raise ValueError(f"speech_16k must hold at least {KERNEL} samples (HuBERT's receptive field) as (N,) or (N, channels), "
                             f"got shape {speech.shape}")
        n_all = int((speech.shape[0] / 16000) * FPS)                                     # UVG:229
        if n_all < 1:
            raise ValueError(f"{speech.shape[0]} samples at 16 kHz make no video frame at {FPS} fps")
        pose_in = None if init_pose is None else _state(init_pose, (1, 7), "init_pose")
        eye_in = None if init_eye_bbox is None else _state(init_eye_bbox, (1, 8), "init_eye_bbox")
        dev = self._device()
        gen = None
        if seed is not None:
            gen = torch.Generator(device=dev)
            gen.manual_seed(int(seed))
        draw = (lambda shape: torch.randn(shape, generator=gen, device=dev)) if gen is not None else (lambda shape: None)  # noqa: E731

        # 1. audio features (UVG:229-242)
        audio_features = hubert_features(self.hubert, speech)                         # (F_all, 1024) on dev

        # 2. pose and blink over all frames of the audio (UVG:266-302)
        p0, b0 = pbnet_initial_states(pose_in, eye_in, dev)
        audio = audio_features.unsqueeze(0)
        durations = torch.tensor([n_all])
        pz = pose_z if pose_z is not None else draw((n_all, 1, self.pose_model.latent_dim))
        bz = blink_z if blink_z is not None else draw((n_all, 1, self.blink_model.latent_dim))
        out_p = self.pose_model.generate(p0, audio, durations, fact=1, z=pz)["output"]
        out_b = self.blink_model.generate(b0, audio, durations, fact=1, z=bz)["output"]
        drive_pose_all, drive_blink_all = finish_pose_blink(out_p, out_b, p0, b0)

        # 3. the clip: frame cap (UVG:328-333) and the video stage's initial states (UVG:335-350)
        F = min(max_frames or vc["max_n_frames"], n_all)
        if F < 1:
            raise ValueError(f"max_frames must be positive, got {max_frames}")
        hub = audio_features[:F]
        drive_poses, drive_blink = drive_pose_all[:F], drive_blink_all[:F]
        real_poses = pose_in.to(torch.float32) if pose_in is not None and eye_in is not None else torch.zeros(1, 7)
        real_blink_bbox = (eye_in.to(torch.float32) if pose_in is not None and eye_in is not None
                           else torch.tensor(VIDEO_FALLBACK_EYE_BBOX).reshape(1, -1).to(torch.float32))
        real_poses, real_blink_bbox = real_poses.to(dev), real_blink_bbox.to(dev)
        ip = real_poses[0].unsqueeze(0)
        ie = real_blink_bbox[0, :2].unsqueeze(0)
        drive_poses, drive_blink, real_blink_bbox = drive_poses.permute(1, 0), drive_blink.permute(1, 0), real_blink_bbox.permute(1, 0)

        # 4. source image (UVG:320-325, 372) on the device
        size = int(vc["input_size"])
        source = portrait_resize(img.to(dev), size)

        # 5. sampling (UVG:369-380 -> FD:327-365) and 6. 8-bit frames (UVG:383-392, 544-548)
        fd = self.flow_diffusion
        fd.update_num_frames(F)
        if noise_fn is None and gen is not None:
            noise_fn = lambda k, shape: torch.randn(shape, generator=gen, device=dev)  # noqa: E731
        pred = fd._sample_latent(source.unsqueeze(0), hub.unsqueeze(0), drive_poses.unsqueeze(0), drive_blink[:2].unsqueeze(0),
                                 real_blink_bbox[2:].unsqueeze(0), vc["cond_scale"], ip, ie, noise_fn, use_graph)
        frames = fd.generator.decode_sample_rgb8(source.unsqueeze(0), pred[0], vc["mean"])
        return {"frames": frames, "fps": FPS, "num_frames": F, "audio_features": audio_features, "drive_pose": drive_pose_all,
                "drive_blink": drive_blink_all, "source": source, "latent": pred[0]}
