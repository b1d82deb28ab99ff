"""TEST INFRASTRUCTURE — generate tests/golden/lfg_motion_*.npz by running the REAL reference motion estimator.

Run in the build container only (needs /root/reference):    python oracle/make_golden_lfg_motion.py
Imports the unmodified `RegionPredictor`, `BGMotionPredictor` and `Generator` (shims for the un-installed, irrelevant
imports under oracle/shims), loads the deterministic synthetic weights of oracle/lfg_motion_oracle.py (each module keeps its own
Gaussian `down.weight` buffer), runs FlowAE.forward's sequence (flow_autoenc.py:37-46) on the CPU, checks
oracle/lfg_motion_oracle.py against it, prints the conditioning of every case's covariances, and stores the reference outputs.
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, 'shims'))
sys.path.insert(0, '/root/reference')
warnings.filterwarnings("ignore")

from oracle import lfg_motion_oracle as M   # noqa: E402
from oracle import weights as W            # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
# name -> (driving frames, H, W); every output of the small case is stored, a fixed sample of the large images
CASES = {'lfg_motion_128': (3, 128, 128), 'lfg_motion_256': (2, 256, 256)}
PROBE_N = 4096
MIN_EIG, MIN_GAP = 1e-3, 0.05           # conditioning every case must keep for SVD sign parity to be meaningful


def build_reference(mp):
    from LFG.modules.bg_motion_predictor import BGMotionPredictor
    from LFG.modules.generator import Generator
    from LFG.modules.region_predictor import RegionPredictor
    gen = Generator(num_regions=mp['num_regions'], num_channels=mp['num_channels'], revert_axis_swap=mp['revert_axis_swap'],
                    **mp['generator_params']).eval()                                               # FD:116-121
    rp = RegionPredictor(num_regions=mp['num_regions'], num_channels=mp['num_channels'],
                         estimate_affine=mp['estimate_affine'], **mp['region_predictor_params']).eval()   # FD:124-130
    bg = BGMotionPredictor(num_channels=mp['num_channels'], **mp['bg_predictor_params']).eval()     # FD:132-136
    return gen, rp, bg


def check_schema(module, schema):
    ref = module.state_dict()
    assert [n for n, _ in schema] == list(ref), "oracle schema must list the reference's keys in order"
    for n, s in schema:
        assert tuple(ref[n].shape) == tuple(s), n
    sd = M.motion_synth_state_dict(schema)
    for n in sd:
        if n.endswith("down.weight"):
            assert torch.equal(sd[n], ref[n]), "the restated Gaussian must equal the module's own buffer"
    module.load_state_dict(sd, strict=True)
    return sd


def margin(a, ref):
    return ((a - ref).abs() / (1e-4 + 1e-3 * ref.abs())).max().item()


def main():
    import yaml
    with open('/root/reference/config/hdtf256.yaml') as f:
        mp = yaml.safe_load(f)['model_params']
    gen, rp, bgp = build_reference(mp)
    cfg = M.MotionCfg(bg_type=mp['bg_predictor_params']['bg_type'], revert_axis_swap=mp['revert_axis_swap'])
    rp_sd = check_schema(rp, M.region_predictor_schema(cfg))
    bg_sd = check_schema(bgp, M.bg_predictor_schema(cfg))
    gen_sd = check_schema(gen, M.generator_schema(cfg))
    with open(os.path.join(GOLD, 'lfg_motion_schema.json'), 'w') as f:
        json.dump({"region_predictor": [[n, list(s)] for n, s in M.region_predictor_schema(cfg)],
                   "bg_predictor": [[n, list(s)] for n, s in M.bg_predictor_schema(cfg)],
                   "generator": [[n, list(s)] for n, s in M.generator_schema(cfg)]}, f, indent=0)
    worst = 0.0
    for name, (nf, H, Wd) in CASES.items():
        src1, drv = M.motion_synth_inputs(name, nf, H, Wd)
        src = src1.expand(nf, -1, -1, -1).contiguous()                 # test_flowautoenc_hdtf_video_256.py: source per frame
        with torch.no_grad():
            s_ref, d_ref = rp(src), rp(drv)                            # flow_autoenc.py:38-41
            bg_ref = bgp(src, drv)
            g_ref = gen(src, source_region_params=s_ref, driving_region_params=d_ref, bg_params=bg_ref)
            mine = M.flowae_forward(rp_sd, bg_sd, gen_sd, cfg, src, drv)
        eig, gap = M.conditioning(torch.cat([s_ref["covar"], d_ref["covar"]]))
        m = {}
        for side, a, b in (("source", mine["source_region_params"], s_ref), ("driving", mine["driving_region_params"], d_ref)):
            for k in ("shift", "covar", "affine"):
                m[f"{side}.{k}"] = margin(a[k], b[k])
            m[f"{side}.heatmap"] = margin(a["heatmap"], b["heatmap"])
        m["bg"] = margin(mine["bg_params"], bg_ref)
        for k in ("optical_flow", "occlusion_map", "prediction", "deformed", "bottle_neck_feat"):
            m[k] = margin(mine[k], g_ref[k])
        w = max(m.values())
        worst = max(worst, w)
        print(f"{name}: {nf} frames {H}x{Wd}; covariance min eigenvalue {eig:.3e}, min (s1 - s2) / s1 {gap:.3f}; "
              f"|bg - I| max {(bg_ref - torch.eye(3)).abs().max():.3f}; |flow| max {g_ref['optical_flow'].abs().max():.3f}")
        print("   oracle vs reference (x tol): " + ", ".join(f"{k} {v:.3g}" for k, v in m.items()))
        assert eig > MIN_EIG and gap > MIN_GAP, "ill-conditioned covariances: SVD column signs would not be meaningful"
        assert w < 0.2, m
        out = {}
        for side, p in (("source", s_ref), ("driving", d_ref)):
            for k in ("shift", "covar", "affine", "u", "d"):
                out[f"{side}_{k}"] = p[k].numpy()
            hm = p["heatmap"]
            out[f"{side}_heatmap_probe"] = hm.flatten()[W.probe_indices(f"{name}/{side}/heatmap", hm.numel(), PROBE_N)].numpy()
        out["bg"] = bg_ref.numpy()
        for k in ("optical_flow", "occlusion_map"):
            out[k] = g_ref[k].numpy()
        for k in ("prediction", "deformed", "bottle_neck_feat"):
            t = g_ref[k]
            out[f"{k}_probe"] = t.flatten()[W.probe_indices(f"{name}/{k}", t.numel(), PROBE_N)].numpy()
        # np.savez (uncompressed) writes no timestamps: the files are byte-reproducible
        np.savez(os.path.join(GOLD, f"{name}.npz"), **out)
    print("worst oracle-vs-reference:", worst, "x tol")


if __name__ == "__main__":
    main()
