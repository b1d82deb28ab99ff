"""LFG decoder configurations other than DAWN-128's own (tests/golden/lfg_configs_report.json, written by
oracle/make_golden_lfg_configs.py): constructor keywords, inputs, synthetic weights, the matching oracle configuration and the
reference's probes, shared by the CPU and GPU tests."""
import hashlib
import json
import os

import numpy as np
import torch

from oracle import lfg_oracle as L
from oracle import weights as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
TAGS = ("dawn256", "be128", "down1", "down3_mf256", "down4", "res0", "res1", "res32", "noskip", "mf96", "flow_big")
RTOL, ATOL = 1e-3, 1e-4            # BASELINE.json north_star: rtol=1e-3 / atol=1e-4 fp32
PROBE_N = 512
_ORACLE_KEYS = ('num_channels', 'block_expansion', 'max_features', 'num_down_blocks', 'num_bottleneck_blocks', 'skips')
_REPORT = None
_GOLDEN = None


def over_tol(a, ref):
    a, ref = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(ref).detach().double().cpu()
    return ((a - ref).abs() / (ATOL + RTOL * ref.abs())).max().item()


def report(tag=None):
    global _REPORT
    if _REPORT is None:
        with open(os.path.join(GOLD, "lfg_configs_report.json")) as f:
            _REPORT = json.load(f)
    return _REPORT if tag is None else _REPORT[tag]


def golden():
    global _GOLDEN
    if _GOLDEN is None:
        _GOLDEN = np.load(os.path.join(GOLD, "lfg_configs.npz"))
    return _GOLDEN


def ctor(tag):
    return dict(report(tag)["ctor"])


def oracle_cfg(tag):
    kw = ctor(tag)
    return L.LfgCfg(**{k: kw[k] for k in _ORACLE_KEYS})


def schema(tag):
    """[(name, shape), ...] of the library module's state_dict at the configuration"""
    from dawn_pytorch_b200 import LfgGenerator
    return [(k, list(v.shape)) for k, v in LfgGenerator(**ctor(tag)).state_dict().items()]


def schema_digest(sch):
    """SHA-256 of a schema in order, as oracle/make_golden_lfg_configs.py computes it for the reference's"""
    return hashlib.sha256(json.dumps([[n, list(s)] for n, s in sch], separators=(",", ":")).encode()).hexdigest()


def synth_sd(tag):
    return W.lfg_synth_state_dict([(n, tuple(s)) for n, s in L.state_dict_schema(oracle_cfg(tag))], report(tag)["residual_gain"])


def inputs(tag):
    """source (1, 3, H, W), flow (F, h, w, 2), occ (F, 1, h, w) of the configuration"""
    r = report(tag)
    return W.lfg_synth_inputs("lfgcfg/" + tag, r["frames"], r["H"], r["W"], r["h"], r["w"])


def probe_idx(key, numel):
    u = W.uniform01("probe/lfgcfg/" + key, PROBE_N)
    return np.minimum((u.astype(np.float64) * numel).astype(np.int64), numel - 1)


def probes(tag, name, t):
    """the elements of t (the full tensor `name` of configuration `tag`) at the reference's probe positions"""
    flat = torch.as_tensor(t).detach().cpu().reshape(-1)
    return flat[probe_idx(f"{tag}/{name}", flat.numel())].double().numpy()


def ref_probes(tag, name):
    g = golden()
    return g[f"{tag}/{name}"].astype(np.float64), float(g[f"{tag}/{name}.absmean"].reshape(-1)[0])


def oracle(tag, src=None, flow=None, occ=None):
    """oracle outputs {prediction, deformed, fea, bottleneck, up0, ...} of the configuration (its own inputs by default)"""
    if src is None:
        src, flow, occ = inputs(tag)
    taps, sd, cfg = {}, synth_sd(tag), oracle_cfg(tag)
    with torch.no_grad():
        out = L.forward_with_flow(sd, cfg, src, flow, occ, taps=taps)
        out["fea"] = L.compute_fea(sd, cfg, src)
    out.update({k: taps[k] for k in report(tag)["taps"]})
    return out
