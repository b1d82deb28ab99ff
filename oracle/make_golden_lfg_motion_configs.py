"""TEST INFRASTRUCTURE — reference goldens for the LFG motion estimator beyond DAWN's own configuration.

Run in the build container only (needs /root/reference; the GPU box never runs this):
    python oracle/make_golden_lfg_motion_configs.py
Every case of tests/lfg_motion_config_cases.py runs through the unmodified reference modules on the CPU, with the synthetic
weights of oracle/lfg_motion_oracle.py over that case's own schema:
  FlowAE cases     RegionPredictor, BGMotionPredictor and Generator as FlowAE.forward runs them (flow_autoenc.py:37-46), on
                   non-square frames, with bg_type 'zero', and with one source image per frame
  Generator cases  Generator.forward (generator.py:92-130) on constructed region parameters whose A = A_s inv(A_d) has
                   A[0, 0] < 0 in GEN_NEGATIVE regions of every frame, with revert_axis_swap on and off, a perspective bg
                   (bottom row != (0, 0, 1)) and bg_params=None
The oracle is checked against the reference (margin < 0.2 x tol) and the reference outputs are stored in
  tests/golden/lfg_motion_configs.npz          <case>/<name>: small outputs in full, larger ones as PROBE_N fixed elements
  tests/golden/lfg_motion_configs_report.json  per case: geometry, configuration, schema digest, covariance conditioning, the
                                               A[0, 0] signs and the oracle-vs-reference margins in units of the tolerance
Both files depend on the arrays only, so a rerun reproduces them byte for byte.
"""
import json
import os
import sys
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, 'shims'))
sys.path.insert(0, '/root/reference')
warnings.filterwarnings("ignore")

from oracle import lfg_motion_oracle as M                                    # noqa: E402
from oracle.make_golden_configs import save_npz_stable                      # noqa: E402
from oracle.make_golden_lfg_motion import build_reference, check_schema    # noqa: E402
from tests import lfg_motion_config_cases as C                              # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
REGION_KEYS = ("shift", "covar", "affine", "u", "d")


def model_params(cfg):
    import yaml
    with open('/root/reference/config/hdtf256.yaml') as f:
        mp = yaml.safe_load(f)['model_params']
    mp['bg_predictor_params']['bg_type'] = cfg.bg_type
    mp['revert_axis_swap'] = cfg.revert_axis_swap
    return mp


def reference(case):
    cfg = C.cfg(case)
    gen, rp, bgp = build_reference(model_params(cfg))
    sch = C.schemas(case)
    sds = {"region_predictor": check_schema(rp, sch["region_predictor"]), "bg_predictor": check_schema(bgp, sch["bg_predictor"]),
           "generator": check_schema(gen, sch["generator"])}
    return cfg, gen, rp, bgp, sds, sch


def flowae_case(case, arrays):
    cfg, gen, rp, bgp, sds, sch = reference(case)
    src, drv = C.flowae_inputs(case)
    with torch.no_grad():
        s_ref, d_ref = rp(src), rp(drv)                                          # flow_autoenc.py:38-41
        bg_ref = bgp(src, drv)
        g_ref = gen(src, source_region_params=s_ref, driving_region_params=d_ref, bg_params=bg_ref)
        mine = M.flowae_forward(sds["region_predictor"], sds["bg_predictor"], sds["generator"], cfg, src, drv)
    eig, gap = M.conditioning(torch.cat([s_ref["covar"], d_ref["covar"]]))
    m = {}
    for side, a, b in (("source", mine["source_region_params"], s_ref), ("driving", mine["driving_region_params"], d_ref)):
        for k in REGION_KEYS + ("heatmap",):
            m[f"{side}_{k}"] = C.over_tol(a[k], b[k])
            arrays[f"{case}/{side}_{k}"] = C.probe(case, f"{side}_{k}", b[k]).numpy()
    m["bg"] = C.over_tol(mine["bg_params"], bg_ref)
    arrays[f"{case}/bg"] = bg_ref.numpy()
    for k in C.FLOWAE_OUTPUTS:
        m[k] = C.over_tol(mine[k], g_ref[k])
        arrays[f"{case}/{k}"] = C.probe(case, k, g_ref[k]).numpy()
    a00 = C.composed_affine(d_ref, s_ref)[..., 0, 0]
    n, H, Wd = C.geometry(case)
    print(f"[{case}] {n} x {H}x{Wd}, bg_type {cfg.bg_type}: covariance min eigenvalue {eig:.3e} (> {C.MIN_EIG}), "
          f"min (s1 - s2) / s1 {gap:.3f} (> {C.MIN_GAP}); A00 < 0 in {int((a00 < 0).sum())} of {a00.numel()} region-frames; "
          f"|bg - I| max {(bg_ref - torch.eye(3)).abs().max():.3f}; |flow| max {g_ref['optical_flow'].abs().max():.3f}")
    print("   oracle vs reference (x tol): " + ", ".join(f"{k} {v:.3g}" for k, v in m.items()))
    assert eig > C.MIN_EIG and gap > C.MIN_GAP, f"{case}: ill-conditioned covariances: SVD column signs would not be meaningful"
    assert max(m.values()) < 0.2, m
    return dict(kind="flowae", frames=n, H=H, W=Wd, bg_type=cfg.bg_type, revert_axis_swap=cfg.revert_axis_swap,
                input_tag=C.FLOWAE[case][4], input_gamma=C.FLOWAE[case][5], source_pattern=C.SOURCE_PATTERN.get(case), min_eig=eig, min_gap=gap,
                a00_negative=int((a00 < 0).sum()), schema_digest=C.schema_digest(sch),
                schema_entries={k: len(v) for k, v in sch.items()}, oracle_margins=m)


def generator_case(case, arrays):
    cfg, gen, _, _, sds, sch = reference(case)
    src, dp, sp, bg = C.generator_inputs(case)
    with torch.no_grad():
        g_ref = gen(src, driving_region_params=dp, source_region_params=sp, bg_params=bg)
        mine = M.generator_forward(sds["generator"], cfg, src, dp, sp, bg)
    m = {}
    for k in C.FLOWAE_OUTPUTS:
        m[k] = C.over_tol(mine[k], g_ref[k])
        arrays[f"{case}/{k}"] = C.probe(case, k, g_ref[k]).numpy()
    a00 = C.composed_affine(dp, sp)[..., 0, 0]
    neg = [int(v) for v in (a00 < 0).sum(dim=1)]
    eig, gap = M.conditioning(torch.cat([sp["covar"], dp["covar"]]))
    hz = None if bg is None else [float(bg[:, 2, 0].abs().max()), float(bg[:, 2, 1].abs().max())]
    print(f"[{case}] {C.GEN_FRAMES} x {C.GEN_H}x{C.GEN_W}, revert_axis_swap {cfg.revert_axis_swap}, bg {C.GENERATOR[case][1]}: "
          f"A00 < 0 in {neg} of {a00.shape[1]} regions per frame, min |A00| {a00.abs().min():.3f}; covariance min eigenvalue "
          f"{eig:.3e}; |flow| max {g_ref['optical_flow'].abs().max():.3f}")
    print("   oracle vs reference (x tol): " + ", ".join(f"{k} {v:.3g}" for k, v in m.items()))
    assert min(neg) >= 3 and a00.abs().min() > 0.01, "the revert branch must act on several well-separated regions of every frame"
    assert max(m.values()) < 0.2, m
    return g_ref, dict(kind="generator", frames=C.GEN_FRAMES, H=C.GEN_H, W=C.GEN_W, revert_axis_swap=cfg.revert_axis_swap,
                       bg=C.GENERATOR[case][1], bg_bottom_row_absmax=hz, a00_negative_per_frame=neg,
                       a00_min_abs=a00.abs().min().item(), min_eig=eig, min_gap=gap, schema_digest=C.schema_digest(sch),
                       schema_entries={k: len(v) for k, v in sch.items()}, oracle_margins=m)


def main():
    torch.set_num_threads(os.cpu_count())
    arrays, report, flows = {}, {}, {}
    for case in C.FLOWAE:
        report[case] = flowae_case(case, arrays)
    for case in C.GENERATOR:
        g_ref, report[case] = generator_case(case, arrays)
        flows[case] = g_ref["optical_flow"]
    d = C.over_tol(flows["revert_on"], flows["revert_off"])
    print(f"revert_on vs revert_off reference flows differ by {d:.3g} x tol")
    assert d > 100, "revert_axis_swap must change the reference flow by far more than the tolerance"
    report["revert_off"]["flow_vs_revert_on"] = d
    save_npz_stable(os.path.join(GOLD, 'lfg_motion_configs.npz'), arrays)
    with open(os.path.join(GOLD, 'lfg_motion_configs_report.json'), 'w') as f:
        f.write('{\n' + ',\n'.join(f'{json.dumps(k)}: {json.dumps(report[k], sort_keys=True)}' for k in sorted(report)) + '\n}\n')
    print('golden vectors written to', GOLD)


if __name__ == '__main__':
    main()
