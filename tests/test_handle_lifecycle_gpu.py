"""GPU: the native-handle lifecycle every module shares (dawn_pytorch_b200/_lib.py: _Handle, _NativeModule).

* load_state_dict after a first call reaches the library: Generator.forward_with_flow, RegionPredictor, BGMotionPredictor,
  MotionGenerator.flow and the PBnet decoder then return, bit for bit, what fresh modules built with the new weights return; the
  UNet (16 frames of a 32 x 32 latent, BASELINE.json configs[0]) returns it to within the spread of two identical calls.
* .to() of the device a module is already on marks its handles dirty: both of a MotionGenerator's, the UNet's, the PBnet decoder's.
* del frees the device memory of every handle type: dawn_live_bytes returns to where it was.
"""
import gc
import json
import os

import pytest
import torch

from oracle import lfg_motion_oracle as M
from oracle import pbnet_oracle as P
from tests import gpu_common as G

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


# ---------------------------------------------------------------------------------------------------------------- the UNet
def unet_sds():
    first = G.synth_sd()
    return first, {n: t * 1.0625 if t.is_floating_point() else t for n, t in first.items()}


def unet(sd):
    from dawn_pytorch_b200 import DynamicNfUnet3D
    net = DynamicNfUnet3D(**G.CTOR).eval()
    net.load_state_dict(sd, strict=True)
    return net.cuda()


def unet_eps(net):
    x, t, cond, _, _ = G.clip("cfg1")
    net.update_num_frames(x.shape[2])
    with torch.no_grad():
        return net.forward_with_cond_scale(x.cuda(), t.cuda(), cond=cond.cuda(), cond_scale=1.0).clone()


# The UNet's GroupNorm statistics are summed by fp64 atomics in a run-dependent order, so two identical calls differ in the last
# bits (max |d| about 1.4e-6 on the benchmark clip); a stale upload differs by orders of magnitude more.
UNET_SPREAD = 1e-5


def test_unet_load_state_dict_after_a_call_reaches_the_library():
    first_sd, second_sd = unet_sds()
    net = unet(first_sd)
    first = unet_eps(net)
    net.load_state_dict(second_sd)
    reloaded = unet_eps(net)
    fresh = unet_eps(unet(second_sd))
    stale, d = (fresh - first).abs().max().item(), (reloaded - fresh).abs().max().item()
    assert stale > 1e3 * UNET_SPREAD and d <= UNET_SPREAD, f"max |d|: first vs fresh {stale:.2e}, reloaded vs fresh {d:.2e}"


def test_unet_to_the_same_device_marks_its_handle_dirty():
    net = unet(unet_sds()[0])
    unet_eps(net)
    assert not net._unet.dirty
    net.to(torch.device("cuda", torch.cuda.current_device()))
    assert net._unet.dirty


# ---------------------------------------------------------------------------------------------------------------- PBnet
PB_CASE = "reemb5_pose_250"


def pbnet_sds():
    with open(os.path.join(GOLD, "pbnet_schema.json")) as f:
        first = P.synth_state_dict([(n, tuple(s)) for n, s in json.load(f)[PB_CASE]])
    return first, {k: v * 1.0625 for k, v in first.items()}


def pbnet(sd):
    from dawn_pytorch_b200.pbnet import get_model
    model = get_model(P.CASES[PB_CASE][0].parameters("cuda:0"))
    model.load_state_dict(sd, strict=True)
    return model.eval()


def pbnet_output(model):
    cfg, lengths = P.CASES[PB_CASE]
    pose, audio, z, lens = P.synth_inputs(PB_CASE, cfg, lengths)
    return model.generate(pose, audio, lens, fact=1, z=z.cuda())["output"].clone()


def test_pbnet_load_state_dict_after_a_call_reaches_the_library():
    first_sd, second_sd = pbnet_sds()
    model = pbnet(first_sd)
    first = pbnet_output(model)
    model.load_state_dict(second_sd)
    reloaded = pbnet_output(model)
    fresh = pbnet_output(pbnet(second_sd))
    assert not torch.equal(fresh, first) and torch.equal(reloaded, fresh)


def test_pbnet_to_the_same_device_marks_its_handle_dirty():
    model = pbnet(pbnet_sds()[0])
    pbnet_output(model)
    assert not model.decoder._pbnet.dirty
    model.to(torch.device("cuda", torch.cuda.current_device()))
    assert model.decoder._pbnet.dirty


# ---------------------------------------------------------------------------------------------------------------- memory
def run_unet():
    net = unet(unet_sds()[0])
    unet_eps(net)
    return [net]


def run_lfg():
    mods = modules(weight_sets()[0])
    outputs(*mods)
    return list(mods)


def run_pbnet():
    model = pbnet(pbnet_sds()[0])
    pbnet_output(model)
    return [model]


def test_del_frees_the_device_memory():
    """for the UNet, the LFG decoder and motion estimator, and PBnet in turn"""
    from dawn_pytorch_b200._lib import lib
    for run in (run_unet, run_lfg, run_pbnet):
        gc.collect()
        base = lib.dawn_live_bytes()
        mods = run()
        ws = [m.workspace_bytes() for m in mods]
        assert min(ws) > 0 and lib.dawn_live_bytes() >= base + sum(ws), run.__name__
        del mods
        gc.collect()
        assert lib.dawn_live_bytes() == base, run.__name__
