"""CPU: the LFG motion estimator's module boundary.  dawn_lfg_motion_create accepts DAWN's shipped configuration (both bg_type
values the library runs, revert_axis_swap either way) and refuses every other with a message (it needs no GPU); the modules'
state_dict keys are the reference's (tests/golden/lfg_motion_schema.json, dumped from the reference modules); a checkpoint-shaped
dict loads with strict=True; and Generator, the decoder alone, is unchanged."""
import ctypes
import json
import os

import pytest
import torch

from oracle import lfg_motion_oracle as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def create(**over):
    from dawn_pytorch_b200 import _lib
    from dawn_pytorch_b200.lfg import _motion_cfg
    cfg = _motion_cfg(**over)
    h = ctypes.c_void_p()
    rc = _lib.lib.dawn_lfg_motion_create(ctypes.byref(cfg), ctypes.byref(h))
    if rc == 0:
        _lib.lib.dawn_lfg_motion_destroy(h)
    return rc, _lib.lib.dawn_last_error().decode()


def schema(part):
    with open(os.path.join(GOLD, "lfg_motion_schema.json")) as f:
        return [(n, tuple(s)) for n, s in json.load(f)[part]]


@pytest.mark.parametrize("kw", [{}, dict(bg_type=0), dict(revert_axis_swap=0)])
def test_create_accepts_dawn_config(kw):
    rc, err = create(**kw)
    assert rc == 0, err


@pytest.mark.parametrize("kw,msg", [
    (dict(num_regions=5), "num_regions must be 10"),
    (dict(num_channels=1), "num_channels must be 3"),
    (dict(estimate_affine=0), "PCA-based"),
    (dict(pca_based=0), "PCA-based"),
    (dict(fast_svd=1), "fast_svd"),
    (dict(rp_block_expansion=64), "region predictor must have"),
    (dict(rp_num_blocks=4), "region predictor must have"),
    (dict(rp_temperature=0.2), "temperature 0.1"),
    (dict(rp_scale_factor=0.5), "scale_factor 0.25"),
    (dict(bg_type=2), "bg_type"),
    (dict(bg_max_features=512), "bg predictor must have"),
    (dict(pw_block_expansion=32), "flow predictor must have"),
    (dict(pw_scale_factor=1.0), "flow predictor must have"),
    (dict(use_covar_heatmap=0), "use_covar_heatmap"),
    (dict(use_deformed_source=0), "use_deformed_source"),
    (dict(estimate_occlusion_map=0), "estimate_occlusion_map"),
    (dict(revert_axis_swap=2), "revert_axis_swap"),
])
def test_create_refuses_unsupported(kw, msg):
    rc, err = create(**kw)
    assert rc == -1 and msg in err, err


def test_modules_refuse_unsupported_configs():
    from dawn_pytorch_b200 import BGMotionPredictor, RegionPredictor, _lib
    with pytest.raises(_lib.DawnError, match="PCA-based"):
        RegionPredictor(block_expansion=32, num_regions=10, num_channels=3, max_features=1024, num_blocks=5, temperature=0.1,
                        estimate_affine=True, scale_factor=0.25, pca_based=False)
    with pytest.raises(_lib.DawnError, match="bg_type"):
        BGMotionPredictor(block_expansion=32, num_channels=3, max_features=1024, num_blocks=5, bg_type='perspective')


def test_state_dict_keys_equal_the_reference():
    from dawn_pytorch_b200 import FlowAE
    ae = FlowAE(is_train=False)
    for part in ("region_predictor", "bg_predictor", "generator"):
        mine = [(k, tuple(v.shape)) for k, v in getattr(ae, part).state_dict().items()]
        assert mine == schema(part), part
    assert [len(schema(p)) for p in ("region_predictor", "bg_predictor", "generator")] == [73, 37, 196]


def test_checkpoint_shaped_dict_loads_strict():
    """the three load_state_dict calls of test_flowautoenc_hdtf_video_256.py:135-137"""
    from dawn_pytorch_b200 import FlowAE
    ae = FlowAE(is_train=False)
    checkpoint = {p: M.motion_synth_state_dict(schema(p)) for p in ("region_predictor", "bg_predictor", "generator")}
    for part in ("generator", "region_predictor", "bg_predictor"):
        res = getattr(ae, part).load_state_dict(checkpoint[part], strict=True)
        assert not res.missing_keys and not res.unexpected_keys
    assert torch.equal(ae.generator.state_dict()["pixelwise_flow_predictor.mask.weight"],
                       checkpoint["generator"]["pixelwise_flow_predictor.mask.weight"])
    assert torch.equal(ae.region_predictor.state_dict()["down.weight"], M.anti_alias_weight())
    assert not ae.training
    with pytest.raises(NotImplementedError):
        ae.train()


def test_generator_is_unchanged():
    """Generator (the decoder alone) still drops the flow predictor's entries and refuses forward"""
    from dawn_pytorch_b200 import LfgGenerator
    with open(os.path.join(GOLD, "lfg_state_dict_schema.json")) as f:
        sch = json.load(f)
    g = LfgGenerator(num_channels=3, num_regions=10, block_expansion=64, max_features=512, num_down_blocks=2, num_bottleneck_blocks=6,
                     pixelwise_flow_predictor_params={"block_expansion": 64}, skips=True, revert_axis_swap=True)
    assert [(k, list(v.shape)) for k, v in g.state_dict().items()] == [(k, list(s)) for k, s in sch["entries"]]
    assert not any(k.startswith("pixelwise_flow_predictor.") for k in g.state_dict())
    with pytest.raises(NotImplementedError):
        g.forward()


def test_flowae_refuses_cpu_tensors():
    from dawn_pytorch_b200 import FlowAE, _lib
    ae = FlowAE(is_train=False)
    ae.set_train_input(torch.rand(1, 3, 128, 128), torch.rand(1, 3, 128, 128))
    with pytest.raises(_lib.DawnError):
        ae.forward()
