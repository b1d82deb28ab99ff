"""CPU: PBnet's pose / blink generator (dawn_pytorch_b200/pbnet.py) at its boundary.

* the float64 oracle (oracle/pbnet_oracle.py) reproduces every golden output of the reference's generate, at DAWN's shape and at
  the other configurations of oracle/pbnet_oracle.CONFIG_CASES (d_model 32 to 256, 2 to 32 heads, 1 to 4 layers, ff 1 to 2048);
* get_model builds a CVAE whose state_dict keys, order and shapes are the reference's, and strict loading succeeds;
* the relative-position bias table uses the reference's bucket of every j - i up to 2000 frames;
* unsupported architectures, head counts and durations raise, and CPU models refuse to generate;
* include/dawn_pbnet.h and the library's exports agree, and so do the header's kernel-test case struct and its ctypes mirror.
"""
import json
import os
import re

import numpy as np
import pytest
import torch

from oracle import pbnet_oracle as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
RTOL, ATOL = 1e-3, 1e-4


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLD, "pbnet.npz"))


@pytest.fixture(scope="module")
def schema():
    with open(os.path.join(GOLD, "pbnet_schema.json")) as f:
        return {k: [(n, tuple(s)) for n, s in v] for k, v in json.load(f).items()}


@pytest.fixture(scope="module")
def config_golden():
    return np.load(os.path.join(GOLD, "pbnet_configs.npz"))


@pytest.fixture(scope="module")
def config_schema():
    with open(os.path.join(GOLD, "pbnet_configs_schema.json")) as f:
        return {k: [(n, tuple(s)) for n, s in v] for k, v in json.load(f).items()}


@pytest.mark.parametrize("case", list(P.CASES))
def test_oracle_matches_reference_golden(case, golden, schema):
    cfg, lengths = P.CASES[case]
    sd = P.synth_state_dict(schema[case])
    pose, audio, z, lens = P.synth_inputs(case, cfg, lengths)
    out = P.decoder_forward(sd, cfg, pose, audio, z, lens)
    ref = torch.from_numpy(golden[f"{case}/output"]).double()
    assert out.shape == ref.shape
    assert ((out - ref).abs() / (ATOL + RTOL * ref.abs())).max().item() < 0.05


@pytest.mark.parametrize("case", list(P.CONFIG_CASES))
def test_oracle_matches_reference_golden_at_other_configurations(case, config_golden, config_schema):
    cfg, lengths = P.CONFIG_CASES[case]
    sd = P.synth_state_dict(config_schema[case])
    pose, audio, z, lens = P.synth_inputs(case, cfg, lengths)
    out = P.decoder_forward(sd, cfg, pose, audio, z, lens)
    ref = torch.from_numpy(config_golden[f"{case}/output"]).double()
    assert out.shape == ref.shape == (len(lengths), max(lengths), cfg.out_dim)
    assert ((out - ref).abs() / (ATOL + RTOL * ref.abs())).max().item() < 0.05


@pytest.mark.parametrize("case", list(P.CONFIG_CASES))
def test_state_dict_at_other_configurations_equals_reference_and_loads_strictly(case, config_schema):
    from dawn_pytorch_b200.pbnet import get_model
    cfg, _ = P.CONFIG_CASES[case]
    model = get_model(cfg.parameters())
    assert [(k, tuple(v.shape)) for k, v in model.state_dict().items()] == config_schema[case]
    res = model.load_state_dict(P.synth_state_dict(config_schema[case]), strict=True)
    assert not res.missing_keys and not res.unexpected_keys


@pytest.mark.parametrize("case", list(P.CASES))
def test_state_dict_equals_reference_and_loads_strictly(case, schema):
    from dawn_pytorch_b200.pbnet import get_model
    cfg, _ = P.CASES[case]
    model = get_model(cfg.parameters())
    mine = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
    assert mine == schema[case], "same keys, order and shapes as the reference's CVAE"
    res = model.load_state_dict(P.synth_state_dict(schema[case]), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert model.decoder._pbnet.dirty


def test_bias_table_uses_reference_buckets_up_to_2000_frames(golden):
    from dawn_pytorch_b200.unet import _rel_bias_table
    ids = torch.arange(128, dtype=torch.float32)[:, None]              # an embedding whose value is its bucket index
    tab = _rel_bias_table(ids, 1999, num_buckets=128, max_distance=128)[0]
    assert torch.equal(tab.long(), torch.from_numpy(golden["bucket_2000"].astype(np.int64)))
    rel = torch.arange(-1999, 2000)
    assert torch.equal(P.bucket(rel, 128, 128), torch.from_numpy(golden["bucket_2000"].astype(np.int64)))


@pytest.mark.parametrize("bad", [dict(archiname="transformerreemb7"), dict(archiname="transformerreemb8"),
                                 dict(archiname="transformer"), dict(modeltype="cae"), dict(num_heads=64),
                                 dict(pose_latent_dim=48), dict(num_layers=9), dict(num_layers=5),
                                 dict(latent_dim=128)])
def test_unsupported_configurations_raise(bad):
    from dawn_pytorch_b200.pbnet import get_model
    p = {**P.PbCfg().parameters(), **bad}
    with pytest.raises(ValueError):
        get_model(p)


def test_odd_heads_raise():
    from dawn_pytorch_b200.pbnet import get_model
    p = {**P.PbCfg().parameters(), "num_heads": 3}
    with pytest.raises(ValueError, match="num_heads"):
        get_model(p)


def test_bad_durations_and_cpu_model_raise():
    from dawn_pytorch_b200._lib import DawnError
    from dawn_pytorch_b200.pbnet import get_model
    model = get_model(P.PbCfg().parameters())
    pose, audio = torch.zeros(1, 1, 6), torch.zeros(1, 10, 1024)
    for d in (torch.tensor([[10]]), torch.tensor([9]), torch.tensor([11]), torch.tensor([10, 10])):
        with pytest.raises(ValueError):
            model.generate(pose, audio, d)
    with pytest.raises(DawnError, match="no CPU path"):
        model.generate(pose, audio, torch.tensor([10]))
    for call in (lambda: model(None), lambda: model.compute_loss(None), lambda: model.return_latent(None), lambda: model.train()):
        with pytest.raises(NotImplementedError):
            call()


def test_lengths_to_mask_is_static():
    from dawn_pytorch_b200.pbnet import CVAE
    m = CVAE.lengths_to_mask(torch.tensor([3, 1]))
    assert m.tolist() == [[True, True, True], [True, False, False]]


def test_header_declares_exactly_the_exports():
    from dawn_pytorch_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "dawn_pbnet.h")).read()
    declared = set(re.findall(r"\b(dawn_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.PBNET_EXPORTS)
    for sym in declared:
        assert hasattr(_lib.lib, sym)


def test_kernel_case_struct_matches_the_header():
    import ctypes
    from dawn_pytorch_b200 import _lib
    from tests.test_hubert_cpu import _c_struct_fields
    ctype = {ctypes.c_int: "int", ctypes.c_float: "float", ctypes.c_int * 8: "int[8]", ctypes.c_void_p: "pointer"}
    got = [(n, ctype[t]) for n, t in _lib.DawnPbnetKernelCase._fields_]
    want = [(n, "pointer" if t.endswith("*") else t) for n, t in _c_struct_fields("dawn_pbnet.h", "dawn_pbnet_kernel_case")]
    assert got == want
    with open(os.path.join(ROOT, "include", "dawn_pbnet.h")) as f:
        kinds = re.findall(r"DAWN_PBNET_(\w+) = (\d+)", f.read())
    assert [(k, int(v)) for k, v in kinds] == [(k, getattr(_lib, "PBNET_" + k)) for k, _ in kinds] and len(kinds) == 4
