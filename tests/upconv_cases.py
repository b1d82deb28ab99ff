"""UNets with the upconv variant (nearest x2 + 3x3 conv in each padding mode) or without spatial linear attention
(tests/golden/upconv_report.json, written by oracle/make_golden_upconv.py): constructor keywords, clips, synthetic weights and
the matching oracle configuration, shared by the CPU and GPU tests."""
import json
import os

import numpy as np
import torch

from oracle import upconv_oracle as UO
from oracle import weights as W
from tests import config_cases as CC

TAGS = ("up_zeros", "up_reflect", "up_replicate", "up_circular", "upconv_nosla", "deconv_nosla", "rect_reflect", "rect_circular",
        "dim128_reflect")
MODES = ("zeros", "reflect", "replicate", "circular")
_ORACLE_KEYS = CC._ORACLE_KEYS + ("use_deconv", "padding_mode", "use_sparse_linear_attn")
over_tol, schema_digest = CC.over_tol, CC.schema_digest
_REPORT = None
_GOLDEN = None
_SD = {}


def report(tag=None):
    global _REPORT
    if _REPORT is None:
        with open(os.path.join(CC.GOLD, "upconv_report.json")) as f:
            _REPORT = json.load(f)
    return _REPORT if tag is None else _REPORT[tag]


def golden():
    global _GOLDEN
    if _GOLDEN is None:
        _GOLDEN = np.load(os.path.join(CC.GOLD, "upconv.npz"))
    return _GOLDEN


def ctor(tag):
    return {k: (tuple(v) if isinstance(v, list) else v) for k, v in report(tag)["ctor"].items()}


def oracle_cfg(tag):
    kw = ctor(tag)
    return UO.UpconvCfg(**{k: kw[k] for k in _ORACLE_KEYS if k in kw})


def schema(tag):
    from dawn_pytorch_b200 import DynamicNfUnet3D
    return [(k, list(v.shape)) for k, v in DynamicNfUnet3D(**ctor(tag)).state_dict().items()]


def synth_sd(tag):
    if tag not in _SD:
        _SD[tag] = W.synth_state_dict(schema(tag))
    return _SD[tag]


def golden_taps(tag):
    g = golden()
    return {str(n): (list(map(int, sh)), float(am), pr) for n, sh, am, pr in
            zip(g[f"taps/{tag}"], g[f"shapes/{tag}"], g[f"absmean/{tag}"], g[f"probes/{tag}"])}


def clip(tag, key=None, amp=1.0, t=None):
    """x (1, channels, F, h, w), t (1,), cond (1, F, cond_dim), x_t (1, 3, F, h, w), fea (1, channels-3, h, w)"""
    rep, kw = report(tag), ctor(tag)
    Fr, h, w = rep["F"], rep["h"], rep["w"]
    x_t, fea, cond = W.synth_inputs(key or tag, Fr, h, w, cond_dim=kw["cond_dim"], fea_ch=kw["channels"] - 3)
    x_t = x_t * amp
    x = torch.cat([x_t, fea.unsqueeze(2).expand(-1, -1, Fr, -1, -1)], dim=1).contiguous()
    return x, torch.full((1,), rep["t"] if t is None else t, dtype=torch.long), cond, x_t, fea


def oracle(tag, x, t, cond, taps=None):
    with torch.no_grad():
        return UO.unet_forward(synth_sd(tag), oracle_cfg(tag), x, t, cond, taps=taps)
