"""UNet configurations other than DAWN's own (tests/golden/configs_report.json, written by oracle/make_golden_configs.py):
constructor keywords, clips, synthetic weights and the matching oracle configuration, shared by the CPU and GPU tests."""
import hashlib
import json
import os

import numpy as np
import torch

from oracle import unet_oracle as O
from oracle import weights as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
TAGS = ("dim128", "mult16_k3", "l3_k5", "l2_w1", "l6", "io", "w120", "narrow")
RTOL, ATOL = 1e-3, 1e-4            # BASELINE.json north_star: rtol=1e-3 / atol=1e-4 fp32
_ORACLE_KEYS = ('dim', 'dim_mults', 'channels', 'cond_aud', 'cond_pose', 'cond_eye', 'out_grid_dim', 'out_conf_dim',
                'init_kernel_size', 'win_width')
_REPORT = None
_GOLDEN = None
_SD = {}


def over_tol(a, ref):
    a, ref = a.detach().float().cpu(), ref.detach().float().cpu()
    return ((a - ref).abs() / (ATOL + RTOL * ref.abs())).max().item()


def report(tag=None):
    global _REPORT
    if _REPORT is None:
        with open(os.path.join(GOLD, "configs_report.json")) as f:
            _REPORT = json.load(f)
    return _REPORT if tag is None else _REPORT[tag]


def golden():
    global _GOLDEN
    if _GOLDEN is None:
        _GOLDEN = np.load(os.path.join(GOLD, "configs.npz"))
    return _GOLDEN


def ctor(tag):
    """constructor keywords of the configuration (tuples restored)"""
    return {k: (tuple(v) if isinstance(v, list) else v) for k, v in report(tag)["ctor"].items()}


def oracle_cfg(tag):
    kw = ctor(tag)
    return O.UnetCfg(**{k: kw[k] for k in _ORACLE_KEYS if k in kw})


def schema(tag):
    """[(name, shape), ...] of the library module's state_dict at the configuration; tests/test_configs_cpu.py checks that it is
    the reference's (report(tag)["schema_digest"])"""
    from dawn_pytorch_b200 import DynamicNfUnet3D
    return [(k, list(v.shape)) for k, v in DynamicNfUnet3D(**ctor(tag)).state_dict().items()]


def schema_digest(sch):
    """SHA-256 of a schema in order, as oracle/make_golden_configs.py computes it for the reference's"""
    return hashlib.sha256(json.dumps([[n, list(s)] for n, s in sch], separators=(",", ":")).encode()).hexdigest()


def synth_sd(tag):
    if tag not in _SD:
        _SD[tag] = W.synth_state_dict(schema(tag))
    return _SD[tag]


def golden_taps(tag):
    """{tap: (shape, abs-mean, 64 probe values)} the reference recorded at every sub-module boundary"""
    g = golden()
    return {str(n): (list(map(int, sh)), float(am), pr) for n, sh, am, pr in
            zip(g[f"taps/{tag}"], g[f"shapes/{tag}"], g[f"absmean/{tag}"], g[f"probes/{tag}"])}


def clip(tag, key=None, amp=1.0, t=None):
    """x (1, channels, F, h, w), t (1,), cond (1, F, cond_dim), x_t (1, 3, F, h, w), fea (1, channels-3, h, w) of the tag's clip
    (key: another seed at the same geometry; amp scales the noisy channels)"""
    rep, kw = report(tag), ctor(tag)
    Fr, h, w = rep["F"], rep["h"], rep["w"]
    x_t, fea, cond = W.synth_inputs(key or tag, Fr, h, w, cond_dim=kw["cond_dim"], fea_ch=kw["channels"] - 3)
    x_t = x_t * amp
    x = torch.cat([x_t, fea.unsqueeze(2).expand(-1, -1, Fr, -1, -1)], dim=1).contiguous()
    return x, torch.full((1,), rep["t"] if t is None else t, dtype=torch.long), cond, x_t, fea


def oracle(tag, x, t, cond, taps=None):
    with torch.no_grad():
        return O.unet_forward(synth_sd(tag), oracle_cfg(tag), x, t, cond, taps=taps)
