"""LFG motion-estimator cases beyond DAWN's own configuration (tests/golden/lfg_motion_configs.npz and
lfg_motion_configs_report.json, written by oracle/make_golden_lfg_motion_configs.py): the geometry, configuration and seeded
inputs of every case, shared by that script and the CPU and GPU tests.

FlowAE cases run FlowAE.forward (flow_autoenc.py:37-46) on synthetic frames.  Generator cases call Generator.forward
(generator.py:92-130) on constructed region parameters, so that A = A_s inv(A_d) has A[0, 0] < 0 in several regions of every
frame: that is the only place revert_axis_swap acts (pixelwise_flow_predictor.py:76-78).
"""
import hashlib
import json
import math
import os

import numpy as np
import torch

from oracle import lfg_motion_oracle as M
from oracle import weights as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
RTOL, ATOL = 1e-3, 1e-4            # BASELINE.json north_star: rtol=1e-3 / atol=1e-4 fp32
PROBE_N = 1024                     # elements kept of every output larger than FULL_MAX
FULL_MAX = 4096
MIN_EIG, MIN_GAP = 1e-3, 0.05      # covariance conditioning every FlowAE case keeps (oracle/make_golden_lfg_motion.py)

# id -> (frames, H, W, bg_type, input tag, gamma).  The images of M.motion_synth_inputs(tag, ...) are raised to `gamma`: on
# 384x128 frames the plain recipe leaves one region's covariance at a minimum eigenvalue of 9e-4 whatever the tag, and gamma 1.4
# (darker frames) lifts it to 2e-3.  On 512x384 and 640x384 frames some region's covariance stays near-isotropic
# ((s1 - s2) / s1 < 0.04 for every tag and gamma tried), so the large case is 384x640, whose gap is 0.06 at gamma 1.4.
FLOWAE = {
    'wide':     (2, 128, 384, 'affine', 'lfgmcfg/wide', 1.0),       # H < W: deepest hourglass level 1x3
    'tall':     (2, 384, 128, 'affine', 'lfgmcfg/tall', 1.4),       # the same shapes transposed
    'w640':     (1, 128, 640, 'affine', 'lfgmcfg/w640', 1.0),       # deepest level 1x5; mma.sync and wgmma levels in one hourglass
    'r384x640': (1, 384, 640, 'affine', 'lfgmcfg/r384x640', 1.4),   # both sides above 256, neither a power of two
    'bgzero':   (2, 128, 256, 'zero', 'lfgmcfg/bgzero', 1.0),       # BGMotionPredictor(bg_type='zero'): no parameters, identity bg
    'sources':  (4, 128, 128, 'affine', 'lfgmcfg/sources/3', 1.0),    # one source image per frame, A A B A: three decode groups
}
SOURCE_PATTERN = {'sources': 'AABA'}

# id -> (revert_axis_swap, bg kind)
GENERATOR = {
    'revert_on':  (True, 'affine'),
    'revert_off': (False, 'affine'),
    'bg_persp':   (True, 'perspective'),   # bottom row (0.05, -0.03, 1): h_z != 1
    'bg_none':    (True, None),            # bg_params=None: the identity grid
}
GEN_FRAMES, GEN_H, GEN_W = 3, 128, 256
GEN_TAG = 'lfgmcfg/generator'
GEN_NEGATIVE = 4                   # regions per frame whose driving affine is turned by 180 degrees so that A[0, 0] < 0
CASES = tuple(FLOWAE) + tuple(GENERATOR)

FLOWAE_OUTPUTS = ("optical_flow", "occlusion_map", "prediction", "deformed", "bottle_neck_feat")


def over_tol(a, ref):
    a = torch.as_tensor(a).detach().double().cpu()
    ref = torch.as_tensor(np.asarray(ref) if not torch.is_tensor(ref) else ref).detach().double().cpu()
    return ((a - ref).abs() / (ATOL + RTOL * ref.abs())).max().item()


def cfg(case):
    if case in FLOWAE:
        return M.MotionCfg(bg_type=FLOWAE[case][3], revert_axis_swap=True)
    return M.MotionCfg(revert_axis_swap=GENERATOR[case][0])


def geometry(case):
    """(frames, H, W)"""
    return FLOWAE[case][:3] if case in FLOWAE else (GEN_FRAMES, GEN_H, GEN_W)


def schemas(case):
    c = cfg(case)
    return {"region_predictor": M.region_predictor_schema(c), "bg_predictor": M.bg_predictor_schema(c),
            "generator": M.generator_schema(c)}


def schema_digest(schema):
    """SHA-256 of {part: [(name, shape), ...]} in order"""
    return hashlib.sha256(json.dumps({k: [[n, list(s)] for n, s in v] for k, v in schema.items()},
                                     separators=(',', ':'), sort_keys=True).encode()).hexdigest()


def state_dicts(case):
    return {k: M.motion_synth_state_dict(v) for k, v in schemas(case).items()}


def flowae_inputs(case):
    """ref_img (n, 3, H, W) and dri_img (n, 3, H, W) of a FlowAE case"""
    n, H, Wd, _, tag, gamma = FLOWAE[case]
    src, drv = M.motion_synth_inputs(tag, n, H, Wd)
    if gamma != 1.0:
        src, drv = src ** gamma, drv ** gamma
    pattern = SOURCE_PATTERN.get(case)
    if pattern is None:
        return src.expand(n, -1, -1, -1).contiguous(), drv
    other = {c: M.motion_synth_inputs(f"{tag}/{c}", 1, H, Wd)[0] ** gamma for c in sorted(set(pattern) - {'A'})}
    return torch.cat([src if c == 'A' else other[c] for c in pattern]), drv


def _rot(phi):
    c, s = np.cos(phi), np.sin(phi)
    return np.stack([np.stack([c, -s], -1), np.stack([s, c], -1)], -2)


def _region_params(key, n, R):
    """shift in [-0.6, 0.6]^2; covar = rot(phi) diag(l) rot(phi)^T with l in [0.004, 0.04] (positive definite, eigenvalue ratio
    at most 0.8); affine = rot(phi) diag(sqrt(l)), the form of region_predictor.py:107-115's u diag(sqrt(s))"""
    shift = W.symmetric(f"{key}/shift", (n, R, 2), 0.6).astype(np.float64)
    phi = W.symmetric(f"{key}/phi", (n, R), math.pi).astype(np.float64)
    l1 = 0.01 + 0.03 * W.uniform01(f"{key}/l1", n * R).astype(np.float64).reshape(n, R)
    l2 = l1 * (0.25 + 0.55 * W.uniform01(f"{key}/l2", n * R).astype(np.float64).reshape(n, R))
    rot = _rot(phi)
    lam = np.stack([l1, l2], -1)
    covar = rot @ (lam[..., :, None] * np.swapaxes(rot, -1, -2))
    affine = rot * np.sqrt(lam)[..., None, :]
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))   # noqa: E731
    return {"shift": f(shift), "covar": f(covar), "affine": f(affine)}


def generator_inputs(case):
    """source_image (n, 3, H, W), driving_region_params, source_region_params, bg_params (n, 3, 3) or None of a Generator case.
    The inputs are the same in every case; only the bg differs.  In frame i the driving affines of regions (r + i) mod R <
    GEN_NEGATIVE are negated (a 180-degree turn, which leaves the covariance as it is), so that A[0, 0] < 0 there."""
    n, H, Wd, R = GEN_FRAMES, GEN_H, GEN_W, M.MotionCfg().num_regions
    src = W.lfg_synth_inputs(f"{GEN_TAG}/src", 1, H, Wd, 1, 1)[0].expand(n, -1, -1, -1).contiguous()
    sp = _region_params(f"{GEN_TAG}/source", n, R)
    dp = _region_params(f"{GEN_TAG}/driving", n, R)
    a = torch.matmul(sp["affine"].double(), torch.inverse(dp["affine"].double()))[..., 0, 0]
    want_neg = torch.tensor([[(r + i) % R < GEN_NEGATIVE for r in range(R)] for i in range(n)])
    flip = (a < 0) != want_neg
    dp["affine"] = torch.where(flip[..., None, None], -dp["affine"], dp["affine"])
    kind = GENERATOR[case][1]
    if kind is None:
        return src, dp, sp, None
    top = np.array([[1, 0, 0], [0, 1, 0]], dtype=np.float32) + W.symmetric(f"{GEN_TAG}/bg", (n, 2, 3), 0.08)
    bottom = np.tile(np.array([0.05, -0.03, 1.0] if kind == 'perspective' else [0.0, 0.0, 1.0], dtype=np.float32), (n, 1, 1))
    return src, dp, sp, torch.from_numpy(np.concatenate([top, bottom], axis=1))


def composed_affine(drv, src):
    """A = A_s inv(A_d) per frame and region, as pixelwise_flow_predictor.py:76 forms it (before the revert)"""
    return torch.matmul(src["affine"], torch.inverse(drv["affine"].float()))


def probe(case, name, t):
    """the stored elements of output `name`: all of it up to FULL_MAX elements, else PROBE_N fixed ones"""
    flat = torch.as_tensor(t).detach().cpu().reshape(-1)
    if flat.numel() <= FULL_MAX:
        return flat
    return flat[torch.from_numpy(W.probe_indices(f"lfgmcfg/{case}/{name}", flat.numel(), PROBE_N))]


def report(case=None):
    with open(os.path.join(GOLD, "lfg_motion_configs_report.json")) as f:
        r = json.load(f)
    return r if case is None else r[case]


_GOLDEN = None


def golden(case, name):
    global _GOLDEN
    if _GOLDEN is None:
        _GOLDEN = np.load(os.path.join(GOLD, "lfg_motion_configs.npz"))
    return _GOLDEN[f"{case}/{name}"]
