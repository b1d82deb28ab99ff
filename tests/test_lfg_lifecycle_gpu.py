"""GPU: the native-handle lifecycle the LFG modules share (dawn_pytorch_b200/lfg.py: _Handle, _LfgModule).

* load_state_dict after a first call reaches the library: Generator.forward_with_flow, RegionPredictor, BGMotionPredictor and
  MotionGenerator.flow then return, bit for bit, what fresh modules built with the new weights return.
* .to() of the device a MotionGenerator is already on marks both of its handles (decoder and flow predictor) dirty.
"""
import json
import os

import pytest
import torch

from oracle import lfg_motion_oracle as M

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N, H, W = 2, 128, 128


def weight_sets():
    """the synthetic weights of the motion golden cases, and a second set: every floating-point entry scaled by 1.0625"""
    with open(os.path.join(GOLD, "lfg_motion_schema.json")) as f:
        schema = json.load(f)
    first = {k: M.motion_synth_state_dict([(n, tuple(s)) for n, s in schema[k]])
             for k in ("region_predictor", "bg_predictor", "generator")}
    second = {k: {n: t * 1.0625 if t.is_floating_point() else t for n, t in sd.items()} for k, sd in first.items()}
    return first, second


def modules(sds):
    """(decoder Generator, RegionPredictor, BGMotionPredictor, MotionGenerator) of FlowAE's configuration, loaded with sds"""
    from dawn_pytorch_b200 import FlowAE, LfgGenerator
    from dawn_pytorch_b200.lfg import _default_model_params
    ae = FlowAE(is_train=False)
    for k, sd in sds.items():
        getattr(ae, k).load_state_dict(sd)
    mp = _default_model_params()
    gp = {k: v for k, v in mp["generator_params"].items() if k != "pixelwise_flow_predictor_params"}
    dec = LfgGenerator(num_regions=mp["num_regions"], num_channels=mp["num_channels"], **gp)
    dec.load_state_dict(M.decode_sd(sds["generator"]))
    return dec.cuda(), ae.region_predictor.cuda(), ae.bg_predictor.cuda(), ae.generator.cuda()


def outputs(dec, rp, bg, mg):
    src, drv = (t.cuda() for t in M.motion_synth_inputs("lfg_lifecycle", N, H, W))
    srcp, drvp = rp(src), rp(drv)
    b = bg(src, drv)
    m = mg.flow(src, drvp, srcp, b)
    d = dec.forward_with_flow(src, m["optical_flow"], m["occlusion_map"])
    dm = mg.forward_with_flow(src, m["optical_flow"], m["occlusion_map"])
    out = {f"regions.{k}": drvp[k] for k in ("shift", "covar", "heatmap")}
    out.update(bg=b, optical_flow=m["optical_flow"], occlusion_map=m["occlusion_map"], prediction=d["prediction"],
               deformed=d["deformed"], motion_generator_prediction=dm["prediction"])
    return {k: v.clone() for k, v in out.items()}


def test_load_state_dict_after_a_call_reaches_the_library():
    first_sds, second_sds = weight_sets()
    mods = modules(first_sds)
    first = outputs(*mods)
    dec, rp, bg, mg = mods
    dec.load_state_dict(M.decode_sd(second_sds["generator"]))
    rp.load_state_dict(second_sds["region_predictor"])
    bg.load_state_dict(second_sds["bg_predictor"])
    mg.load_state_dict(second_sds["generator"])
    reloaded = outputs(*mods)
    fresh = outputs(*modules(second_sds))
    same_as_first = [k for k in fresh if torch.equal(fresh[k], first[k])]
    assert not same_as_first, f"the second weight set leaves {same_as_first} unchanged: the test would not see a stale upload"
    differ = {k: (reloaded[k] - fresh[k]).abs().max().item() for k in fresh if not torch.equal(reloaded[k], fresh[k])}
    assert not differ, f"reloaded modules differ from fresh ones (max |d|): {differ}"


def test_to_the_same_device_marks_every_handle_dirty():
    first_sds, _ = weight_sets()
    dec, rp, bg, mg = modules(first_sds)
    outputs(dec, rp, bg, mg)
    assert not mg._lfg.dirty and not mg._motion.dirty
    mg.to(torch.device("cuda", torch.cuda.current_device()))
    assert mg._lfg.dirty and mg._motion.dirty
