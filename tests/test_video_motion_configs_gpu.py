"""GPU: the LFG motion estimator beyond DAWN's own configuration, through the reference-facing modules (FlowAE, RegionPredictor,
BGMotionPredictor, MotionGenerator) -> C-ABI (include/dawn_lfg.h, dawn_lfg_motion_*):
  - every case of tests/golden/lfg_motion_configs.npz (non-square frames, bg_type 'zero', one source image per frame,
    revert_axis_swap on and off, a perspective bg and bg_params=None) against the REAL reference at the north-star tolerance,
    and the hourglass / encoder taps against the oracle run on the same GPU;
  - batch independence on non-square frames and with per-frame sources, and across the 50-frame stage-call boundaries;
  - the geometry refusals, and frames whose size caps the frames per stage call below 50 (the int32 bound).
The file sorts after tests/test_temporal_wg_gpu.py for the reason tests/test_video_motion_gpu.py gives.
"""
import gc

import pytest
import torch
import yaml

from oracle import lfg_motion_oracle as M
from tests import lfg_motion_config_cases as C

pytestmark = pytest.mark.gpu

_AE = None


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """the modules here hold workspaces for up to 50 frames of 128x256 and 42 of 1024x768: give them back afterwards"""
    yield
    global _AE
    _AE = None
    gc.collect()
    torch.cuda.empty_cache()


def load(ae, case):
    for part, sd in C.state_dicts(case).items():
        getattr(ae, part).load_state_dict(sd, strict=True)
    return ae.cuda()


def flowae_from_yaml(case, tmp_path):
    """FlowAE(config_pth=...) from a YAML with the case's bg_type and revert_axis_swap"""
    from dawn_pytorch_b200 import FlowAE
    from dawn_pytorch_b200.lfg import _default_model_params
    cfg = C.cfg(case)
    mp = _default_model_params()
    mp['bg_predictor_params']['bg_type'] = cfg.bg_type
    mp['revert_axis_swap'] = cfg.revert_axis_swap
    path = tmp_path / f"{case}.yaml"
    path.write_text(yaml.safe_dump({'model_params': mp}))
    ae = FlowAE(is_train=False, config_pth=str(path))
    assert ae.bg_predictor.bg_type == cfg.bg_type
    return load(ae, case)


def default_flowae():
    global _AE
    if _AE is None:
        from dawn_pytorch_b200 import FlowAE
        _AE = load(FlowAE(is_train=False), "wide")
    return _AE


class _NoTF32:
    def __enter__(self):
        self.flags = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = self.flags


def cuda(p):
    return {k: v.cuda() for k, v in p.items()}


@pytest.mark.parametrize("case", C.CASES)
def test_matches_reference_golden(case, tmp_path):
    cfg = C.cfg(case)
    sd = {k: cuda(v) for k, v in C.state_dicts(case).items()}
    worst, taps = {}, {}
    if case in C.FLOWAE:
        ae = flowae_from_yaml(case, tmp_path)
        src, drv = (t.cuda() for t in C.flowae_inputs(case))
        ae.set_train_input(src, drv)
        ae.forward()
        out = ae.generated
        for side in ("source", "driving"):
            p = out[f"{side}_region_params"]
            for k in ("shift", "covar", "affine", "u", "d", "heatmap"):
                worst[f"{side}_{k}"] = C.over_tol(C.probe(case, f"{side}_{k}", p[k]), C.golden(case, f"{side}_{k}"))
        worst["bg"] = C.over_tol(ae.bg_predictor(src, drv), C.golden(case, "bg"))
        # the Hourglass / Encoder outputs against the oracle on the same inputs, on this GPU
        with torch.no_grad(), _NoTF32():
            M.region_predictor(sd["region_predictor"], cfg, drv, taps=taps)
            M.bg_predictor(sd["bg_predictor"], cfg, src, drv, taps=taps)
            srcp = M.region_predictor(sd["region_predictor"], cfg, src)
            drvp = M.region_predictor(sd["region_predictor"], cfg, drv)
            bgo = M.bg_predictor(sd["bg_predictor"], cfg, src, drv)
        ae.region_predictor(drv)
        worst["tap.region_predictor"] = C.over_tol(ae.region_predictor.read_tap("region_predictor"), taps["predictor"])
        if cfg.bg_type == 'affine':
            ae.bg_predictor(src, drv)
            worst["tap.bg_encoder"] = C.over_tol(ae.bg_predictor.read_tap("bg_encoder"), taps["encoder"])
        gen = ae.generator
    else:
        from dawn_pytorch_b200 import MotionGenerator
        from dawn_pytorch_b200.lfg import _default_model_params
        gen = MotionGenerator(num_regions=10, num_channels=3, revert_axis_swap=cfg.revert_axis_swap,
                              **_default_model_params()['generator_params'])
        gen.load_state_dict(C.state_dicts(case)["generator"], strict=True)
        gen = gen.cuda()
        src, drvp, srcp, bgo = C.generator_inputs(case)
        src, drvp, srcp = src.cuda(), cuda(drvp), cuda(srcp)
        bgo = bgo.cuda() if bgo is not None else None
        out = gen(src, driving_region_params=drvp, source_region_params=srcp, bg_params=bgo)
    for k in C.FLOWAE_OUTPUTS:
        worst[k] = C.over_tol(C.probe(case, k, out[k]), C.golden(case, k))
    # the flow predictor's hourglass on the frames of the first source image, from the same region parameters
    m = next((i for i in range(1, src.shape[0]) if not torch.equal(src[i], src[0])), src.shape[0])
    first = lambda p: {k: v[:m] for k, v in p.items()}                    # noqa: E731
    ptaps = {}
    with torch.no_grad(), _NoTF32():
        M.flow_predictor(sd["generator"], cfg, src[:m], first(drvp), first(srcp), bgo[:m] if bgo is not None else None,
                         taps=ptaps)
    gen.flow(src[:1], first(drvp), first(srcp), bgo[:m] if bgo is not None else None)
    worst["tap.flow_hourglass"] = C.over_tol(gen.read_tap("flow_hourglass"), ptaps["pixelwise_flow_predictor.hourglass"])
    n, H, Wd = C.geometry(case)
    print(f"{case} ({n} x {H}x{Wd}): worst x tol " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    print(f"{case}: worst {max(worst.values()):.3g} x tol")
    assert max(worst.values()) <= 1.0, worst


def flat(ae, src, drv):
    """every output of FlowAE.forward and of the bg predictor, keyed by name"""
    ae.set_train_input(src, drv)
    ae.forward()
    g = ae.generated
    out = {k: v.clone() for k, v in g.items() if torch.is_tensor(v)}
    for side in ("source_region_params", "driving_region_params"):
        for k in ("shift", "covar", "affine", "heatmap"):
            out[f"{side}.{k}"] = g[side][k].clone()
    out["bg"] = ae.bg_predictor(src, drv)
    return out


def compare_single_frames(ae, src, drv, frames):
    full = flat(ae, src, drv)
    bad = {}
    for i in frames:
        one = flat(ae, src[i:i + 1], drv[i:i + 1])
        for k, v in one.items():
            if not torch.equal(v, full[k][i:i + 1]):
                bad[f"{i}.{k}"] = (v - full[k][i:i + 1]).abs().max().item()
    return bad


@pytest.mark.parametrize("case", ["wide", "sources"])
def test_batch_is_bit_identical_to_single_frames(case):
    """all frames in one call equal each frame run alone, bit for bit, through every stage"""
    src, drv = (t.cuda() for t in C.flowae_inputs(case))
    bad = compare_single_frames(default_flowae(), src, drv, range(src.shape[0]))
    print(f"{case}: batch vs one at a time, max |d| of the outputs that differ:", bad or "none")
    assert not bad


def test_chunks_with_changing_sources():
    """120 frames of 128x256 whose source image changes every 7 frames: the region and bg stages run in calls of 50 frames, so
    source groups straddle the call boundaries.  Frames on both sides of each boundary equal the same frames run alone."""
    from dawn_pytorch_b200.lfg import MOTION_CHUNK
    n, H, Wd = 120, 128, 256
    assert MOTION_CHUNK == 50
    _, drv = M.motion_synth_inputs("lfgmcfg/chunks", n, H, Wd)
    srcs = [M.motion_synth_inputs(f"lfgmcfg/chunks/{g}", 1, H, Wd)[0] for g in range((n + 6) // 7)]
    src = torch.cat([srcs[i // 7] for i in range(n)])
    bad = compare_single_frames(default_flowae(), src.cuda(), drv.cuda(), [0, 49, 50, 51, 99, 100, 119])
    print("120 frames vs one at a time, max |d| of the outputs that differ:", bad or "none")
    assert not bad


def test_geometry_refusals_leave_the_module_usable():
    from dawn_pytorch_b200 import _lib
    ae = default_flowae()
    rp = ae.region_predictor
    x = M.motion_synth_inputs("lfgmcfg/refusal", 2, 128, 256)[1].cuda()
    before = rp(x)["covar"].clone()
    for H, Wd in ((192, 128), (128, 64)):
        with pytest.raises(_lib.DawnError, match="H and W must be multiples of 128"):
            rp(torch.rand(1, 3, H, Wd, device="cuda"))
    h = rp._motion.handle
    with pytest.raises(_lib.DawnError, match=r"frames out of range \[1, 1024\]"):
        _lib.check(_lib.lib.dawn_lfg_motion_set_geometry(h, 1025, 128, 256), "dawn_lfg_motion_set_geometry")
    buf = torch.empty(16, device="cuda")
    with pytest.raises(_lib.DawnError, match=r"n must be in \[1, frames of set_geometry\]"):
        _lib.check(_lib.lib.dawn_lfg_motion_regions(h, _lib.ptr(buf), 1025, _lib.ptr(buf), _lib.ptr(buf), None, _lib.stream()),
                   "dawn_lfg_motion_regions")
    assert torch.equal(rp(x)["covar"], before)


def test_frames_per_call_within_int32_bound():
    """RegionPredictor on 43 frames of 1024x768: 43 x 1024 x 768 x 64 >= 2^31, so the frames run in calls of 42.  Frames 0, 21
    and 42 equal their single-frame runs bit for bit, and frame 0 matches the oracle on this GPU."""
    from dawn_pytorch_b200 import RegionPredictor
    from dawn_pytorch_b200.lfg import _default_model_params, motion_frames_per_call
    n, H, Wd = 43, 1024, 768
    assert motion_frames_per_call(n, H, Wd) == 42
    rp = RegionPredictor(num_regions=10, num_channels=3, estimate_affine=True, **_default_model_params()['region_predictor_params'])
    sd = C.state_dicts("wide")["region_predictor"]
    rp.load_state_dict(sd, strict=True)
    rp = rp.cuda()
    src = M.motion_synth_inputs("lfgmcfg/int32", 1, H, Wd)[0].cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    x = src * 0.7 + torch.rand((n, 3, H, Wd), device="cuda", generator=g) * 0.3
    full = rp(x)
    assert rp._motion.geom[0] == 42
    bad = {}
    for i in (0, 21, 42):
        one = rp(x[i:i + 1])
        for k in ("shift", "covar", "affine", "heatmap"):
            if not torch.equal(one[k], full[k][i:i + 1]):
                bad[f"{i}.{k}"] = (one[k] - full[k][i:i + 1]).abs().max().item()
    with torch.no_grad(), _NoTF32():
        taps = {}
        ref = M.region_predictor(cuda(sd), M.MotionCfg(), x[:1], taps=taps)
    worst = {k: C.over_tol(full[k][:1], ref[k]) for k in ("shift", "covar", "heatmap")}
    eig, gap = M.conditioning(ref["covar"])
    if eig > C.MIN_EIG and gap > C.MIN_GAP:
        worst["affine"] = C.over_tol(full["affine"][:1], ref["affine"])
    rp(x[:1])
    worst["tap.region_predictor"] = C.over_tol(rp.read_tap("region_predictor"), taps["predictor"])
    print(f"43 x 1024x768: frame 0 vs oracle x tol " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()),
          "; single frames vs batch:", bad or "bit-identical")
    assert not bad
    assert max(worst.values()) <= 1.0, worst
