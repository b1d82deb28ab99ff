"""CPU: the motion-estimator oracle (oracle/lfg_motion_oracle.py) against the REAL reference on the cases beyond DAWN's own
configuration (tests/golden/lfg_motion_configs.npz, oracle/make_golden_lfg_motion_configs.py); the report's premises (the
revert cases reach the revert branch, the FlowAE cases are well conditioned, the schemas are the oracle's); the bg_type 'zero'
module's state_dict; and the rule that picks the frames per motion stage call."""
import pytest
import torch

from oracle import lfg_motion_oracle as M
from tests import lfg_motion_config_cases as C


@pytest.mark.parametrize("case", C.CASES)
def test_oracle_matches_reference_golden(case):
    sd = C.state_dicts(case)
    cfg = C.cfg(case)
    worst = {}
    with torch.no_grad():
        if case in C.FLOWAE:
            src, drv = C.flowae_inputs(case)
            out = M.flowae_forward(sd["region_predictor"], sd["bg_predictor"], sd["generator"], cfg, src, drv)
            for side in ("source", "driving"):
                p = out[f"{side}_region_params"]
                for k in ("shift", "covar", "affine", "u", "d", "heatmap"):
                    worst[f"{side}_{k}"] = C.over_tol(C.probe(case, f"{side}_{k}", p[k]), C.golden(case, f"{side}_{k}"))
            worst["bg"] = C.over_tol(out["bg_params"], C.golden(case, "bg"))
        else:
            src, dp, sp, bg = C.generator_inputs(case)
            out = M.generator_forward(sd["generator"], cfg, src, dp, sp, bg)
    for k in C.FLOWAE_OUTPUTS:
        worst[k] = C.over_tol(C.probe(case, k, out[k]), C.golden(case, k))
    assert max(worst.values()) <= 0.2, worst
    n, H, Wd = C.geometry(case)
    assert out["optical_flow"].shape == (n, H // 4, Wd // 4, 2) and out["prediction"].shape == (n, 3, H, Wd)


@pytest.mark.parametrize("case", C.CASES)
def test_report_premises(case):
    r = C.report(case)
    n, H, Wd = C.geometry(case)
    assert (r["frames"], r["H"], r["W"]) == (n, H, Wd)
    assert r["revert_axis_swap"] == C.cfg(case).revert_axis_swap
    sch = C.schemas(case)
    assert r["schema_digest"] == C.schema_digest(sch), "the reference's state_dict schema is not the oracle's"
    assert r["schema_entries"] == {k: len(v) for k, v in sch.items()}
    assert max(r["oracle_margins"].values()) < 0.2
    if case in C.FLOWAE:
        assert r["bg_type"] == C.FLOWAE[case][3] and r["input_tag"] == C.FLOWAE[case][4]
        assert r["min_eig"] > C.MIN_EIG and r["min_gap"] > C.MIN_GAP, "SVD column signs would not be meaningful"
    else:
        # every frame reaches the revert branch: A[0, 0] < 0 in several regions, well away from 0
        assert min(r["a00_negative_per_frame"]) >= 3 and r["a00_min_abs"] > 0.01
        _, dp, sp, bg = C.generator_inputs(case)
        a00 = C.composed_affine(dp, sp)[..., 0, 0]
        assert [int(v) for v in (a00 < 0).sum(dim=1)] == r["a00_negative_per_frame"]
        assert torch.linalg.eigvalsh(torch.cat([sp["covar"], dp["covar"]]).double()).min() > 0
        if C.GENERATOR[case][1] == 'perspective':
            assert bg[:, 2, :2].abs().min() > 0.01
        elif bg is not None:
            assert torch.equal(bg[:, 2], torch.tensor([0.0, 0.0, 1.0]).expand(n, 3))


def test_revert_pair_differs():
    """revert_on and revert_off share their inputs; the reference flows differ by far more than the tolerance"""
    assert C.report("revert_off")["flow_vs_revert_on"] > 100
    assert C.over_tol(C.golden("revert_on", "optical_flow"), C.golden("revert_off", "optical_flow")) > 100
    assert C.over_tol(C.golden("revert_on", "optical_flow"), C.golden("bg_persp", "optical_flow")) > 100


def test_bgzero_schema_is_the_module_state_dict():
    from dawn_pytorch_b200 import BGMotionPredictor
    bg = BGMotionPredictor(block_expansion=32, num_channels=3, max_features=1024, num_blocks=5, bg_type='zero')
    assert [(k, tuple(v.shape)) for k, v in bg.state_dict().items()] == C.schemas("bgzero")["bg_predictor"] == []
    assert C.report("bgzero")["schema_entries"]["bg_predictor"] == 0


@pytest.mark.parametrize("n,H,W,frames", [
    (1, 128, 128, 1),
    (49, 128, 128, 49),
    (50, 256, 256, 50),
    (120, 128, 256, 50),
    (200, 256, 256, 50),
    (43, 1024, 768, 42),            # 42 x 1024 x 768 x 64 = 2 113 929 216 < 2^31 <= 43 x ...
    (33, 1024, 1024, 31),
    (1000, 1024, 1024, 31),
    (5, 1024, 1024, 5),
    (10, 4096, 4096, 1),            # 1 x 4096 x 4096 x 64 = 2^30
    (3, 8192, 4096, 1),             # over the bound at one frame: set_geometry refuses it with its own message
])
def test_motion_frames_per_call(n, H, W, frames):
    from dawn_pytorch_b200.lfg import MOTION_CHUNK, motion_frames_per_call
    got = motion_frames_per_call(n, H, W)
    assert got == frames
    assert 1 <= got <= min(n, MOTION_CHUNK)
    if H * W * 64 < 2 ** 31:
        assert got * H * W * 64 < 2 ** 31 and (got == min(n, MOTION_CHUNK) or (got + 1) * H * W * 64 >= 2 ** 31)
