"""CPU: the motion-estimator oracle (oracle/lfg_motion_oracle.py) against golden vectors produced by the REAL reference
RegionPredictor / BGMotionPredictor / Generator.forward (oracle/make_golden_lfg_motion.py), on the same seeded inputs and weights."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import lfg_motion_oracle as M
from oracle import weights as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CASES = {'lfg_motion_128': (3, 128, 128), 'lfg_motion_256': (2, 256, 256)}
PROBE_N = 4096


def over_tol(a, ref):
    a, ref = torch.as_tensor(a).double(), torch.as_tensor(np.asarray(ref)).double()
    return ((a - ref).abs() / (1e-4 + 1e-3 * ref.abs())).max().item()


def sds():
    with open(os.path.join(GOLD, "lfg_motion_schema.json")) as f:
        sch = json.load(f)
    return {k: M.motion_synth_state_dict([(n, tuple(s)) for n, s in v]) for k, v in sch.items()}, sch


def test_schema_is_the_oracle_schema():
    _, sch = sds()
    assert [(n, tuple(s)) for n, s in sch["region_predictor"]] == M.region_predictor_schema()
    assert [(n, tuple(s)) for n, s in sch["bg_predictor"]] == M.bg_predictor_schema()
    assert [(n, tuple(s)) for n, s in sch["generator"]] == M.generator_schema()
    assert (len(sch["region_predictor"]), len(sch["bg_predictor"]), len(sch["generator"])) == (73, 37, 196)


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_reference_golden(case):
    sd, _ = sds()
    n, H, Wd = CASES[case]
    src1, drv = M.motion_synth_inputs(case, n, H, Wd)
    src = src1.expand(n, -1, -1, -1).contiguous()
    g = np.load(os.path.join(GOLD, f"{case}.npz"))
    with torch.no_grad():
        out = M.flowae_forward(sd["region_predictor"], sd["bg_predictor"], sd["generator"], M.MotionCfg(), src, drv)
    for side in ("source", "driving"):
        p = out[f"{side}_region_params"]
        for k in ("shift", "covar", "affine", "u", "d"):
            assert over_tol(p[k], g[f"{side}_{k}"]) <= 0.2, (side, k)
        hm = p["heatmap"].flatten()[W.probe_indices(f"{case}/{side}/heatmap", p["heatmap"].numel(), PROBE_N)]
        assert over_tol(hm, g[f"{side}_heatmap_probe"]) <= 0.2
    assert over_tol(out["bg_params"], g["bg"]) <= 0.2
    for k in ("optical_flow", "occlusion_map"):
        assert over_tol(out[k], g[k]) <= 0.2, k
    for k in ("prediction", "deformed", "bottle_neck_feat"):
        t = out[k].flatten()[W.probe_indices(f"{case}/{k}", out[k].numel(), PROBE_N)]
        assert over_tol(t, g[f"{k}_probe"]) <= 0.2, k
    # the cases are well conditioned: the SVD's column signs, which reach the flow through A_s inv(A_d), are meaningful
    eig, gap = M.conditioning(torch.cat([torch.from_numpy(g["source_covar"]), torch.from_numpy(g["driving_covar"])]))
    assert eig > 1e-3 and gap > 0.05
    assert out["optical_flow"].shape == (n, H // 4, Wd // 4, 2) and g["optical_flow"].std() > 0.1
