"""CPU: LFG decoder configurations other than DAWN-128's own (tests/lfg_config_cases.py).  The oracle matches the real
reference's probes at each of them, the module's state_dict schema is the reference's, the library accepts every one, and it
refuses with a message the configurations its kernels cannot run (dawn_lfg_create needs no GPU)."""
import ctypes

import numpy as np
import pytest

from tests import lfg_config_cases as CC


def create(**over):
    from dawn_pytorch_b200 import _lib
    cfg = _lib.DawnLfgCfg(num_channels=3, block_expansion=64, max_features=512, num_down_blocks=2, num_bottleneck_blocks=6, skips=1)
    for k, v in over.items():
        setattr(cfg, k, v)
    h = ctypes.c_void_p()
    rc = _lib.lib.dawn_lfg_create(ctypes.byref(cfg), ctypes.byref(h))
    if rc == 0:
        _lib.lib.dawn_lfg_destroy(h)
    return rc, _lib.lib.dawn_last_error().decode()


def test_configurations_cover_the_issue_list():
    assert set(CC.report()) == set(CC.TAGS)
    kws = {t: CC.ctor(t) for t in CC.TAGS}
    assert {kw["block_expansion"] for kw in kws.values()} == {64, 128}
    assert {kw["num_down_blocks"] for kw in kws.values()} == {1, 2, 3, 4}
    assert {0, 1, 6, 32} <= {kw["num_bottleneck_blocks"] for kw in kws.values()}
    assert {True, False} == {kw["skips"] for kw in kws.values()}


@pytest.mark.parametrize("tag", CC.TAGS)
def test_oracle_matches_reference_probes(tag):
    out = CC.oracle(tag)
    r = CC.report(tag)
    assert out["prediction"].shape == (r["frames"], 3, r["H"], r["W"])
    for name in ("prediction", "deformed", "fea", *r["taps"]):
        ref, absmean = CC.ref_probes(tag, name)
        got = CC.probes(tag, name, out[name])
        if name == "deformed":
            assert np.abs(got - ref).max() <= 1e-5, name
        else:
            assert CC.over_tol(got, ref) <= 0.2, name
        assert abs(float(out[name].double().abs().mean()) - absmean) <= 1e-4 * (1 + absmean), name


@pytest.mark.parametrize("tag", CC.TAGS)
def test_state_dict_schema_equals_reference(tag):
    """the module's state_dict names and shapes, in order, are the reference's decode path at the same configuration"""
    sch, rep = CC.schema(tag), CC.report(tag)
    assert (len(sch), CC.schema_digest(sch)) == (rep["schema_entries"], rep["schema_digest"])


@pytest.mark.parametrize("tag", CC.TAGS)
def test_create_accepts_config(tag):
    from dawn_pytorch_b200 import LfgGenerator
    rc, err = create(**{f: getattr(LfgGenerator(**CC.ctor(tag))._cfg, f) for f in
                        ("num_channels", "block_expansion", "max_features", "num_down_blocks", "num_bottleneck_blocks", "skips")})
    assert rc == 0, err


@pytest.mark.parametrize("kw,msg", [
    (dict(max_features=32), "max_features must be at least block_expansion"),
    (dict(block_expansion=128, max_features=96), "max_features must be at least block_expansion"),
    (dict(max_features=80), "multiple of 32, got 80"),
    (dict(max_features=200), "multiple of 32, got 200"),
    (dict(block_expansion=128, max_features=144, num_down_blocks=1), "multiple of 32, got 144"),
    (dict(block_expansion=96), "block_expansion must be 64 or 128"),
    (dict(num_down_blocks=5), "num_down_blocks"),
    (dict(num_bottleneck_blocks=33), "num_bottleneck_blocks"),
])
def test_create_refuses_unsupported(kw, msg):
    rc, err = create(**kw)
    assert rc == -1 and msg in err, err
