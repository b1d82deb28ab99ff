"""Whole pipeline on the GPU — `FlowDiffusion.sample_one_video` (source encoder -> face-box embedding -> conditioning -> 3-step
DDIM over the CUDA UNet -> batched LFG decode) against a golden produced by the REAL reference `sample_one_video`
(oracle/make_golden_e2e.py: the reference's own classes and method bodies on the CPU, injected noise)."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import lfg_oracle as L
from oracle import weights as W
from tests import gpu_common as G

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAG, PROBE_N = 'e2e', 4096


def probe_idx(name, numel):
    u = W.uniform01('probe/' + name, PROBE_N)
    return np.minimum((u.astype(np.float64) * numel).astype(np.int64), numel - 1)


def build_model(steps):
    from dawn_pytorch_b200 import FlowDiffusion
    from oracle.make_golden_e2e import face_sd
    m = FlowDiffusion(sampling_timesteps=steps, pose_dim=6, win_width=40, ddim_sampling_eta=1.0)
    m.diffusion.load_state_dict({**{"denoise_fn." + k: v for k, v in G.synth_sd().items()},
                                 **{k: v for k, v in m.diffusion.state_dict().items() if not k.startswith("denoise_fn.")}}, strict=True)
    m.generator.load_state_dict(W.lfg_synth_state_dict(L.state_dict_schema()), strict=True)
    m.face_loc_emb.load_state_dict(face_sd(), strict=True)
    return m.cuda()


def test_sample_one_video_matches_reference_golden():
    from oracle.make_golden_e2e import e2e_inputs
    g = np.load(os.path.join(ROOT, "tests", "golden", "e2e_sample_one_video.npz"))
    steps, nf, size = int(g["steps"]), int(g["frames"]), int(g["image"])
    m = build_model(steps)
    m.update_num_frames(nf)
    img, hubert, pose, eye, bbox, init_pose, init_eye = [t.cuda() for t in e2e_inputs()]

    def noise_fn(k, shape):
        return torch.from_numpy(W.pseudo_normal(f"{TAG}/noise{k}", tuple(shape)))

    # pieces first (cheap to localise a failure): face-box mask and its embedding
    mask = m.generate_bbox_mask(bbox, size=size)
    assert float(mask.sum()) == float(g["bbox_mask_sum"])
    face = m.face_loc_emb(mask)
    assert (face.cpu() - torch.from_numpy(g["face_emb"])).abs().max().item() < 1e-5
    out = m.sample_one_video(sample_img=img, sample_audio_hubert=hubert, sample_pose=pose, sample_eye=eye, sample_bbox=bbox,
                             init_pose=init_pose, init_eye=init_eye, cond_scale=1.0, noise_fn=noise_fn)
    torch.cuda.synchronize()
    grid, conf, vid, warped = out["sample_vid_grid"].cpu(), out["sample_vid_conf"].cpu(), out["sample_out_vid"].cpu(), out["sample_warped_vid"].cpu()
    assert grid.shape == (1, 2, nf, size // 4, size // 4) and conf.shape == (1, 1, nf, size // 4, size // 4)
    assert vid.shape == warped.shape == (1, 3, nf, size, size)
    d_grid = (grid - torch.from_numpy(g["sample_vid_grid"])).abs().max().item()
    d_conf = (conf - torch.from_numpy(g["sample_vid_conf"])).abs().max().item()
    ip = probe_idx(TAG + '/vid', vid.numel())
    ref = torch.from_numpy(g["out_vid_probe"])
    d_vid = (vid.flatten()[ip] - ref).abs()
    r_vid = (d_vid / (1e-4 + 1e-3 * ref.abs())).max().item()
    d_warp = (warped.flatten()[ip] - torch.from_numpy(g["warped_vid_probe"])).abs().max().item()
    print(f"e2e sample_one_video: grid max|d| {d_grid:.2e}, conf {d_conf:.2e}, frames {r_vid:.3f} x tol (max|d| {d_vid.max():.2e}), warped {d_warp:.2e}")
    # the sampled latent passes through {steps} UNet forwards and quantile thresholds: same bar as the sampler golden test
    assert d_grid < 2e-4 and d_conf < 2e-4
    # frames: the north-star tolerance on the decoded video (measured 0.154 x); the warped source inherits the latent's error
    # times the image gradient of a bilinear warp (measured 8.7e-5)
    assert r_vid <= 1.0 and d_warp < 1e-3
    assert abs(float(vid.abs().mean()) - float(g["out_vid_absmean"])) < 1e-4
    # the graph-captured sampler gives the same video
    out2 = m.sample_one_video(sample_img=img, sample_audio_hubert=hubert, sample_pose=pose, sample_eye=eye, sample_bbox=bbox,
                              init_pose=init_pose, init_eye=init_eye, cond_scale=1.0, noise_fn=noise_fn, use_graph=True)
    torch.cuda.synchronize()
    assert (out2["sample_out_vid"].cpu() - vid).abs().max().item() < 1e-3
