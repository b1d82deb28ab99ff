"""GPU: the LFG motion estimator (RegionPredictor, BGMotionPredictor, MotionGenerator, FlowAE) through the reference-facing
module API -> C-ABI (include/dawn_lfg.h, dawn_lfg_motion_*), against golden vectors of the REAL reference modules
(oracle/make_golden_lfg_motion.py) and against the oracle (oracle/lfg_motion_oracle.py) run on the same GPU in fp32.
The file sorts after tests/test_temporal_wg_gpu.py on purpose: that module reads kernel names from torch.profiler, which records
no device events once a pytest process is a few minutes old, so the motion tests run after it rather than before.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import lfg_motion_oracle as M
from oracle import weights as W

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CASES = {'lfg_motion_128': (3, 128, 128), 'lfg_motion_256': (2, 256, 256)}
RTOL, ATOL = 1e-3, 1e-4
PROBE_N = 4096


def over_tol(a, ref):
    a, ref = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(ref).detach().double().cpu()
    return ((a - ref).abs() / (ATOL + RTOL * ref.abs())).max().item()


def schema(part):
    with open(os.path.join(GOLD, "lfg_motion_schema.json")) as f:
        return [(n, tuple(s)) for n, s in json.load(f)[part]]


_AE, _SD = None, None


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """the module's FlowAE holds workspaces sized for the 200-frame clip: give them back before the next test module runs"""
    yield
    global _AE
    _AE = None
    import gc
    gc.collect()
    torch.cuda.empty_cache()


def sds():
    global _SD
    if _SD is None:
        _SD = {k: M.motion_synth_state_dict(schema(k)) for k in ("region_predictor", "bg_predictor", "generator")}
    return _SD


def flowae():
    global _AE
    if _AE is None:
        from dawn_pytorch_b200 import FlowAE
        ae = FlowAE(is_train=False)
        for k, sd in sds().items():
            getattr(ae, k).load_state_dict(sd)                          # test_flowautoenc_hdtf_video_256.py:135-137
        _AE = ae.cuda()
    return _AE


def run(case, nf=None):
    n, H, Wd = CASES[case]
    src1, drv = M.motion_synth_inputs(case, n, H, Wd)
    src = src1.expand(n, -1, -1, -1).contiguous()
    ae = flowae()
    ae.set_train_input(src.cuda(), drv.cuda())
    ae.forward()
    torch.cuda.synchronize()
    return ae, src, drv


def probes(name, t):
    t = t.detach().cpu().flatten()
    return t[W.probe_indices(name, t.numel(), PROBE_N)]


@pytest.mark.parametrize("case", list(CASES))
def test_flowae_matches_reference_golden(case):
    ae, src, drv = run(case)
    g = np.load(os.path.join(GOLD, f"{case}.npz"))
    out = ae.generated
    worst = {}
    for side, p in (("source", out["source_region_params"]), ("driving", out["driving_region_params"])):
        for k in ("shift", "covar", "affine", "u", "d"):
            worst[f"{side}.{k}"] = over_tol(p[k], g[f"{side}_{k}"])
        worst[f"{side}.heatmap"] = over_tol(probes(f"{case}/{side}/heatmap", p["heatmap"]), g[f"{side}_heatmap_probe"])
    n = src.shape[0]
    bg = ae.bg_predictor(src.cuda(), drv.cuda())
    worst["bg"] = over_tol(bg, g["bg"])
    for k in ("optical_flow", "occlusion_map"):
        worst[k] = over_tol(out[k], g[k])
    for k in ("prediction", "deformed", "bottle_neck_feat"):
        worst[k] = over_tol(probes(f"{case}/{k}", out[k]), g[f"{k}_probe"])
    # the Hourglass / Encoder outputs against the oracle on the same inputs (sub-module parity)
    sd = sds()
    cfg = M.MotionCfg()
    taps = {}
    with torch.no_grad():
        M.region_predictor(sd["region_predictor"], cfg, drv, taps=taps)
        M.bg_predictor(sd["bg_predictor"], cfg, src, drv, taps=taps)
    ae.region_predictor(drv.cuda())
    worst["tap.region_predictor"] = over_tol(ae.region_predictor.read_tap("region_predictor"), taps["predictor"])
    worst["tap.bg_encoder"] = over_tol(ae.bg_predictor.read_tap("bg_encoder"), taps["encoder"])
    srcp = M.region_predictor(sd["region_predictor"], cfg, src)
    drvp = M.region_predictor(sd["region_predictor"], cfg, drv)
    bgo = M.bg_predictor(sd["bg_predictor"], cfg, src, drv)
    ptaps = {}
    with torch.no_grad():
        M.flow_predictor(sd["generator"], cfg, src, drvp, srcp, bgo, taps=ptaps)
    ae.generator.flow(src[:1].cuda(), {k: v.cuda() for k, v in drvp.items()}, {k: v.cuda() for k, v in srcp.items()}, bgo.cuda())
    worst["tap.flow_hourglass"] = over_tol(ae.generator.read_tap("flow_hourglass"), ptaps["pixelwise_flow_predictor.hourglass"])
    print(f"{case}: worst x tol " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    print(f"{case}: worst {max(worst.values()):.3g} x tol over {n} frames")
    assert max(worst.values()) <= 1.0, worst


def test_batch_is_bit_identical_to_single_frames():
    """4 frames in one call equal the same frames run one at a time, bit for bit, through every stage"""
    ae = flowae()
    src1, drv = M.motion_synth_inputs("lfg_motion_batch", 4, 128, 128)
    src = src1.expand(4, -1, -1, -1).contiguous().cuda()
    drv = drv.cuda()

    def flat(g):
        out = {k: v.clone() for k, v in g.items() if torch.is_tensor(v)}
        for side in ("source_region_params", "driving_region_params"):
            for k in ("shift", "covar", "affine", "heatmap"):
                out[f"{side}.{k}"] = g[side][k].clone()
        return out

    ae.set_train_input(src, drv)
    ae.forward()
    full = flat(ae.generated)
    full["bg"] = ae.bg_predictor(src, drv)
    bad = {}
    for i in range(4):
        ae.set_train_input(src[i:i + 1], drv[i:i + 1])
        ae.forward()
        one = flat(ae.generated)
        one["bg"] = ae.bg_predictor(src[i:i + 1], drv[i:i + 1])
        for k, v in one.items():
            if not torch.equal(v, full[k][i:i + 1]):
                bad[k] = max(bad.get(k, 0.0), (v - full[k][i:i + 1]).abs().max().item())
    print("batch of 4 vs one at a time, max |d| of the outputs that differ:", bad or "none")
    assert not bad


def test_200_frame_clip_256():
    """reconstruct a 200-frame 256x256 clip (test_flowautoenc_hdtf_video_256.py's source-per-frame layout, in one call); frames 0,
    1, 100 and 199 against the oracle in fp32 on the same GPU (TF32 off).  The region parameters, flow and occlusion are compared
    with the oracle's; the frames with the oracle decoder run on this flow and occlusion: on the white-noise synthetic source a
    flow difference d moves a warped pixel by d W / 2 times a unit-size slope, so the frames of two independent fp32 runs of the
    whole chain differ by more than the flow does (the golden cases above pin the chain end to end)."""
    from oracle import lfg_oracle as L
    ae = flowae()
    n = 200
    src1, drv = M.motion_synth_inputs("lfg_motion_clip", n, 256, 256)
    src = src1.expand(n, -1, -1, -1).contiguous().cuda()
    ae.set_train_input(src, drv.cuda())
    ae.forward()
    out = ae.generated
    assert out["prediction"].shape == (n, 3, 256, 256) and out["optical_flow"].shape == (n, 64, 64, 2)
    sel = [0, 1, 100, 199]
    sd = {k: {n_: t.cuda() for n_, t in v.items()} for k, v in sds().items()}
    flags = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            ref = M.flowae_forward(sd["region_predictor"], sd["bg_predictor"], sd["generator"], M.MotionCfg(), src[sel],
                                   drv[sel].cuda())
            dec = L.forward_with_flow(M.decode_sd(sd["generator"]), L.LfgCfg(), src[:1], out["optical_flow"][sel],
                                      out["occlusion_map"][sel])
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags
    worst = {k: over_tol(out[k][sel], ref[k]) for k in ("optical_flow", "occlusion_map")}
    for side in ("source_region_params", "driving_region_params"):
        for k in ("shift", "covar", "affine"):
            worst[f"{side}.{k}"] = over_tol(out[side][k][sel], ref[side][k])
    worst["prediction"] = over_tol(out["prediction"][sel], dec["prediction"])
    worst["deformed"] = over_tol(out["deformed"][sel], dec["deformed"])
    print("200-frame clip, frames 0/1/100/199 vs oracle: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    print(f"200-frame clip: worst {max(worst.values()):.3g} x tol")
    assert max(worst.values()) <= 1.0, worst


def test_cpu_tensors_fail_loudly():
    from dawn_pytorch_b200 import _lib
    ae = flowae()
    ae.set_train_input(torch.rand(1, 3, 128, 128), torch.rand(1, 3, 128, 128))
    with pytest.raises(_lib.DawnError):
        ae.forward()
    with pytest.raises(_lib.DawnError):
        ae.region_predictor(torch.rand(1, 3, 128, 128))
