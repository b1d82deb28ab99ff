"""TEST INFRASTRUCTURE — golden of sampling from a real clip (tests/golden/resample.npz) from the REAL reference, on the CPU:

  (a) `GaussianDiffusion.q_sample` (U:1226-1232) of a batch of 2 small latents with per-clip timesteps: the rows of Q_T pair
      t in {0, 1, 500, 998, 999} with a second timestep for the second clip; fixed noise pseudo_normal('resample/q_noise');
  (b) an ancestral run from a q-sampled image, as the reference's interpolate runs it (U:1218-1221): x_t = q_sample(x0, ANC_T),
      then `p_sample(img, i, fea, cond=cond)` for i = ANC_T - 1 .. 0 with fea passed (interpolate itself omits it and raises) and
      the randn_like of step k injected as pseudo_normal('resample/anc{k}');
  (c) a DDIM run from a q-sampled image over the suffix ddim_schedule()[DDIM_START:] of the 20-step schedule: x_t =
      q_sample(x0, pairs[DDIM_START][0]), each step the reference UNet's eps and the reference's step arithmetic (U:1169-1205)
      through its oracle restatement (oracle/unet_oracle.py ddim_step, pinned by tests/test_oracle_golden.py), noise of step
      k of the whole schedule pseudo_normal('resample/ddim{k}');
  (d) FD:248-262 + FD:281-282 on the real LFG modules (RegionPredictor, BGMotionPredictor, Generator with the synthetic weights of
      oracle/lfg_motion_oracle.py): the latent cat(grid, occlusion * 2 - 1) of MOTION_B clips of MOTION_F frames at 128 x 128
      (FD:248 fixes 128), each clip's first frame as its source image.

(b) and (c) run on the 'odd' clip (23 f x 16^2) with the UNet of oracle/weights.py, x0 = tanh(pseudo_normal('resample/x0')).
Run in the build container only:    python oracle/make_golden_resample.py"""
import importlib
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import weights as W          # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
U_MOD = 'DM_3.modules.video_flow_diffusion_multiGPU_v0_crema_plus_faceemb_ca_multi_test'
CASE = (23, 16, 16)                       # the 'odd' geometry
Q_SHAPE = (2, 3, 5, 8, 8)
Q_T = ((0, 999), (1, 998), (500, 500), (998, 1), (999, 0))
ANC_T = 3
DDIM_START = 17
MOTION_B, MOTION_F, MOTION_HW = 2, 2, 128


def x0_latent(shape):
    return torch.tanh(torch.from_numpy(W.pseudo_normal("resample/x0", shape)))


def main():
    sys.path.insert(0, os.path.join(HERE, 'shims'))
    sys.path.insert(0, '/root/reference')
    warnings.filterwarnings("ignore")
    from einops import rearrange
    from oracle import lfg_motion_oracle as M
    from oracle import unet_oracle as O
    U = importlib.import_module(U_MOD)
    with open(os.path.join(GOLD, 'state_dict_schema.json')) as f:
        schema = [(n, tuple(s)) for n, s in json.load(f)['entries']]
    net = U.DynamicNfUnet3D(dim=64, cond_dim=1032, cond_aud=1024, cond_pose=6, cond_eye=2, num_frames=40, channels=275, out_grid_dim=2,
                            out_conf_dim=1, dim_mults=(1, 2, 4, 8), use_hubert_audio_cond=True, learn_null_cond=False,
                            use_final_activation=False, use_deconv=True, padding_mode="zeros", win_width=40).eval()
    net.load_state_dict(W.synth_state_dict(schema), strict=True)
    D = U.DynamicNfGaussianDiffusion(denoise_fn=net, num_frames=40, image_size=32, sampling_timesteps=20, timesteps=1000,
                                     loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0).eval()
    out = {}

    # (a) q_sample with one timestep per clip
    xq = x0_latent(Q_SHAPE)
    zq = torch.from_numpy(W.pseudo_normal("resample/q_noise", Q_SHAPE))
    with torch.no_grad():
        out["q_out"] = np.stack([D.q_sample(xq, torch.tensor(tt, dtype=torch.long), noise=zq).numpy() for tt in Q_T])

    Fr, h, w = CASE
    shape = (1, 3, Fr, h, w)
    _, fea, cond = W.synth_inputs('odd', Fr, h, w)
    net.update_num_frames(Fr)
    D.update_num_frames(Fr)
    x0 = x0_latent(shape)

    # (b) ancestral steps ANC_T - 1 .. 0 from q_sample(x0, ANC_T)
    counter = {"k": 0}
    real_randn_like = torch.randn_like

    def injected(t, **kw):
        k = counter["k"]
        counter["k"] += 1
        return torch.from_numpy(W.pseudo_normal(f"resample/anc{k}", tuple(t.shape)))
    with torch.no_grad():
        img = D.q_sample(x0, torch.full((1,), ANC_T, dtype=torch.long),
                         noise=torch.from_numpy(W.pseudo_normal("resample/anc_q", shape)))
    torch.randn_like = injected
    try:
        for i in reversed(range(0, ANC_T)):                                         # U:1220-1221, fea and cond passed
            img = D.p_sample(img, torch.full((1,), i, dtype=torch.long), fea, cond=cond)
    finally:
        torch.randn_like = real_randn_like
    assert counter["k"] == ANC_T
    out["anc_out"] = img.numpy()
    print(f"ancestral from t={ANC_T}: max|x| {float(img.abs().max()):.4f}")

    # (c) DDIM over the schedule's suffix from q_sample(x0, pairs[DDIM_START][0])
    pairs = O.ddim_time_pairs()
    suffix = pairs[DDIM_START:]
    fea_rep = fea.unsqueeze(2).repeat(1, 1, Fr, 1, 1)
    with torch.no_grad():
        img = D.q_sample(x0, torch.full((1,), suffix[0][0], dtype=torch.long),
                         noise=torch.from_numpy(W.pseudo_normal("resample/ddim_q", shape)))
        traj = []
        for j, (t, tn) in enumerate(suffix):
            k = DDIM_START + j
            noise = torch.from_numpy(W.pseudo_normal(f"resample/ddim{k}", shape))
            eps = net.forward_with_cond_scale(torch.cat([img, fea_rep], dim=1), torch.full((1,), t, dtype=torch.long), cond=cond,
                                              cond_scale=1.0)
            img = O.ddim_step(eps, img, t, tn, noise)
            traj.append(img.numpy().copy())
            print(f"ddim step {k} (t={t}->{tn}): max|x| {float(img.abs().max()):.4f}")
    out["ddim_out"] = np.stack(traj)

    # (d) FD:248-262 latent of real clips
    from LFG.modules.bg_motion_predictor import BGMotionPredictor
    from LFG.modules.generator import Generator
    from LFG.modules.region_predictor import RegionPredictor
    import yaml
    with open('/root/reference/config/hdtf128.yaml') as f:
        mp = yaml.safe_load(f)['model_params']
    gen = Generator(num_regions=mp['num_regions'], num_channels=mp['num_channels'], revert_axis_swap=mp['revert_axis_swap'],
                    **mp['generator_params']).eval()
    rp = RegionPredictor(num_regions=mp['num_regions'], num_channels=mp['num_channels'], estimate_affine=mp['estimate_affine'],
                         **mp['region_predictor_params']).eval()
    bgp = BGMotionPredictor(num_channels=mp['num_channels'], **mp['bg_predictor_params']).eval()
    cfg = M.MotionCfg(bg_type=mp['bg_predictor_params']['bg_type'], revert_axis_swap=mp['revert_axis_swap'])
    for mod, sch in ((rp, M.region_predictor_schema(cfg)), (bgp, M.bg_predictor_schema(cfg)), (gen, M.generator_schema(cfg))):
        mod.load_state_dict(M.motion_synth_state_dict(sch), strict=True)
    vids = []
    for i in range(MOTION_B):
        _, drv = M.motion_synth_inputs(f"resample/clip{i}", MOTION_F, MOTION_HW, MOTION_HW)
        vids.append(drv.permute(1, 0, 2, 3))
    real_vid = torch.stack(vids)                                                    # (b, 3, f, H, W) in [0, 1]
    ref_img = real_vid[:, :, 0].clone()                                             # FD:222 with ref_id = 0
    b, c, f, H, Wd = real_vid.shape
    with torch.no_grad():                                                           # FD:248-260
        real_vid_tmp = rearrange(real_vid, 'b c f h w -> (b f) c h w')
        ref_img_tmp = ref_img.unsqueeze(1).repeat(1, f, 1, 1, 1).reshape(-1, 3, MOTION_HW, MOTION_HW)
        source_region_params = rp(ref_img_tmp)
        driving_region_params = rp(real_vid_tmp)
        bg_params = bgp(ref_img_tmp, real_vid_tmp)
        generated = gen(ref_img_tmp, source_region_params=source_region_params, driving_region_params=driving_region_params,
                        bg_params=bg_params)
        grid = rearrange(generated["optical_flow"], '(b f) h w c -> b c f h w', b=b, f=f)
        conf = rearrange(generated["occlusion_map"], '(b f) c h w -> b c f h w', b=b, f=f)
        latent = torch.cat((grid, conf * 2 - 1), dim=1)                            # FD:281-282
    eig, gap = M.conditioning(torch.cat([source_region_params["covar"], driving_region_params["covar"]]))
    print(f"motion latent {tuple(latent.shape)}: covariance min eigenvalue {eig:.3e}, min gap {gap:.3f}")
    assert eig > 1e-3 and gap > 0.05, "ill-conditioned covariances: SVD column signs would not be meaningful"
    out["motion_latent"] = latent.numpy()

    # np.savez (uncompressed) writes no timestamps: the file is byte-reproducible
    np.savez(os.path.join(GOLD, "resample.npz"), q_shape=np.array(Q_SHAPE, dtype=np.int64), q_t=np.array(Q_T, dtype=np.int64),
             anc_t=np.int64(ANC_T), ddim_start=np.int64(DDIM_START), ddim_pairs=np.array(suffix, dtype=np.int64),
             motion=np.array([MOTION_B, MOTION_F, MOTION_HW], dtype=np.int64), **out)


if __name__ == "__main__":
    main()
