"""CPU: the oracle restatement (oracle/unet_oracle.py with O.UnetCfg(...)) against golden vectors of the REAL reference at UNet
configurations other than DAWN's own (oracle/make_golden_configs.py): 128 base channels, 2 to 6 levels, 1024-channel levels on
1x1 images, 3x3 and 5x5 init convs, other input / conditioning / output widths, windows of 1 and 120 frames.  The GPU tests of
these configurations (tests/test_configs_gpu.py) compare the CUDA path with the oracle, so this pins the oracle where the
reference cannot run.  Tolerance as tests/test_oracle_golden.py: half the north-star rtol 1e-3 / atol 1e-4."""
import numpy as np
import pytest
import torch

from oracle import weights as W
from tests import config_cases as CC


def test_report_lists_every_configuration():
    assert tuple(CC.report()) == tuple(sorted(CC.TAGS))
    g = CC.golden()
    assert {f"{k}/{t}" for t in CC.TAGS for k in ("eps", "taps", "shapes", "absmean", "probes")} <= set(g.files)


@pytest.mark.parametrize("tag", CC.TAGS)
def test_oracle_matches_reference_at_config(tag):
    rep, g = CC.report(tag), CC.golden()
    x, t, cond, _, _ = CC.clip(tag)
    taps = {}
    out = CC.oracle(tag, x, t, cond, taps=taps)
    ref = torch.from_numpy(g[f"eps/{tag}"])
    assert out.shape == ref.shape == (1, rep["ctor"]["out_grid_dim"] + rep["ctor"]["out_conf_dim"], rep["F"], rep["h"], rep["w"])
    r = CC.over_tol(out, ref)
    print(f"{tag}: eps {r:.4f} x tol")
    assert r <= 0.5
    gt = CC.golden_taps(tag)
    assert set(taps) == set(gt)
    for name, (shape, absmean, probes) in gt.items():
        flat = taps[name].reshape(-1)
        assert list(taps[name].shape) == shape, name
        idx = W.probe_indices(f"{tag}/{name}", flat.numel(), 64)
        assert CC.over_tol(flat[idx], torch.from_numpy(probes)) <= 0.5, name
        assert abs(float(flat.abs().mean()) - absmean) < 1e-4 * max(1.0, absmean), name


def test_configs_reach_the_shapes_they_are_for():
    """Each configuration really has the geometry it is meant to cover."""
    sh = {t: dict(CC.schema(t)) for t in CC.TAGS}
    assert sh["dim128"]["mid_block1.time_mlp.1.weight"] == [2048, 512]                 # 1024-channel cond block: FiLM n = 2048
    assert sh["mult16_k3"]["mid_block1.time_mlp.1.weight"] == [2048, 256]
    assert sh["mult16_k3"]["init_conv.weight"][-1] == 3 and sh["l3_k5"]["init_conv.weight"][-1] == 5
    assert CC.golden_taps("mult16_k3")["mid_block1"][0][-2:] == [1, 1]                # 16x16 latent, 5 levels
    assert CC.golden_taps("l6")["mid_block1"][0][-2:] == [1, 1]
    assert sh["io"]["init_conv.weight"][1] == 19 and sh["io"]["occlusion_map.1.weight"][0] == 2
    assert sh["io"]["downs.0.0.audio_mlp.1.weight"][1] == 256 and sh["io"]["downs.0.0.pose_mlp.1.weight"][1] == 7
    assert CC.ctor("w120")["win_width"] == 120 and CC.report("w120")["F"] > 121       # |rel| up to 120 and a window that cuts
    assert CC.ctor("l2_w1")["win_width"] == 1
