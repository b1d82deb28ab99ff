"""CPU: the HuBERT audio encoder (dawn_pytorch_b200/hubert.py) at its boundary.

* the float64 oracle (oracle/hubert_oracle.py) reproduces every golden output of transformers' HubertModel, and the per-layer
  mean |h| of its boundaries, within 0.1x the north-star tolerance;
* HubertModel accepts the stable-layer-norm family from a HubertConfig, a dict or a config.json, and refuses the rest with a
  message; it refuses attention masks, output_attentions / output_hidden_states, training and CPU tensors;
* its state_dict is transformers' (the committed schema), loads strictly from either weight-norm spelling and from a
  HubertForCTC checkpoint through from_pretrained;
* frame counts equal transformers' _get_feat_extract_output_lengths for 400 to 10^6 samples;
* the segment plan is the generator's loop, and full segments share a forward at most SEGMENTS_PER_CALL at a time;
* the normalisation equals Wav2Vec2FeatureExtractor's and the interpolation scipy's interp1d, bit for bit;
* include/dawn_hubert.h and the library's exports agree, and so do the header's kernel-test case struct and its ctypes mirror,
  field by field in order.
"""
import json
import os
import re

import numpy as np
import pytest
import torch

from oracle import hubert_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
RTOL, ATOL = 1e-3, 1e-4


def over_tol(a, ref):
    a, ref = a.detach().double(), ref.detach().double()
    return ((a - ref).abs() / (ATOL + RTOL * ref.abs())).max().item()


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLD, "hubert.npz"))


@pytest.fixture(scope="module")
def schema():
    with open(os.path.join(GOLD, "hubert_schema.json")) as f:
        return {k: [(n, tuple(s)) for n, s in v] for k, v in json.load(f).items()}


def small(**over):
    return dict(O.SMALL_A, **over)


# ------------------------------------------------------------------------------------------------ oracle against the goldens
@pytest.mark.parametrize("case", list(O.CASES))
def test_oracle_matches_transformers_golden(case, golden, schema):
    cname, kind, lengths = O.CASES[case]
    c = O.CONFIGS[cname]
    sd = O.synth_state_dict(schema[cname])
    step = O.PROBE_STEP.get(case, 1)
    ref = torch.from_numpy(golden[f"{case}/out"])
    if kind == "model":
        out, taps = O.forward(sd, c, O.synth_input_values(case, lengths).double(), boundaries=True)
        am = torch.stack([t.abs().mean(-1) for t in taps])
        assert over_tol(am, torch.from_numpy(golden[f"{case}/absmean"])) <= 0.1
    else:
        out = O.features(lambda v: O.forward(sd, c, v.double()), O.synth_speech(case, lengths[0]))
    assert out[..., ::step].shape == ref.shape
    assert over_tol(out[..., ::step], ref) <= 0.1


def test_schema_is_the_oracles_and_large_has_422_entries(schema):
    assert len(schema["large"]) == 422
    for cname, c in O.CONFIGS.items():
        assert O.schema_of(c) == schema[cname]


# ------------------------------------------------------------------------------------------------ configurations
def test_accepts_config_dict_object_and_json(tmp_path, schema):
    from dawn_pytorch_b200.hubert import HubertModel
    m = HubertModel(small())
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == schema["small_a"]
    path = tmp_path / "config.json"
    path.write_text(json.dumps(small()))
    assert HubertModel(str(path)).config.hidden_size == 256
    assert HubertModel(str(tmp_path)).config.hidden_size == 256
    assert HubertModel(type("Cfg", (), {"to_dict": lambda self: small()})()).config.num_hidden_layers == 2


def test_large_state_dict_is_transformers(schema):
    from dawn_pytorch_b200.hubert import HubertModel
    m = HubertModel(O.LARGE)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == schema["large"]


@pytest.mark.parametrize("over, what", [
    (dict(feat_extract_norm="group"), "feat_extract_norm"),
    (dict(do_stable_layer_norm=False), "do_stable_layer_norm"),
    (dict(hidden_size=320, num_attention_heads=4, num_conv_pos_embedding_groups=5), "64 wide"),
    (dict(conv_dim=[256] * 6 + [200]), "multiples of 64"),
    (dict(intermediate_size=500), "multiples of 64"),
    (dict(num_conv_pos_embedding_groups=16), "hidden_size / 64"),
    (dict(conv_pos_batch_norm=True), "conv_pos_batch_norm"),
    (dict(hidden_act="relu"), "gelu"),
    (dict(conv_kernel=[10, 3, 3, 3, 3, 2]), "differ in length"),
])
def test_refuses_configs_outside_the_family(over, what):
    from dawn_pytorch_b200.hubert import HubertModel
    with pytest.raises(ValueError, match=what):
        HubertModel(small(**over))


def test_refuses_masks_output_flags_training_and_cpu_tensors():
    from dawn_pytorch_b200._lib import DawnError
    from dawn_pytorch_b200.hubert import HubertModel
    m = HubertModel(small())
    x = torch.zeros(1, 4000)
    for kw in (dict(attention_mask=torch.ones(1, 4000, dtype=torch.long)), dict(output_attentions=True),
               dict(output_hidden_states=True)):
        with pytest.raises(NotImplementedError):
            m(x, **kw)
    with pytest.raises(NotImplementedError):
        m.train()
    with pytest.raises(DawnError, match="CUDA"):
        m(x)
    with pytest.raises(ValueError):
        m(torch.zeros(1, 300))                  # shorter than the receptive field


# ------------------------------------------------------------------------------------------------ keys and loading
def _transformers_spelling(sd):
    return dict(sd)


def _hub_spelling(sd):
    from dawn_pytorch_b200.hubert import WEIGHT_NORM_KEYS
    inv = {v: k for k, v in WEIGHT_NORM_KEYS.items()}
    return {inv.get(k, k): v for k, v in sd.items()}


@pytest.mark.parametrize("spell", [_transformers_spelling, _hub_spelling])
def test_strict_load_from_either_weight_norm_spelling(spell, schema):
    from dawn_pytorch_b200.hubert import HubertModel
    sd = O.synth_state_dict(schema["small_a"])
    m = HubertModel(small())
    m.load_state_dict(spell(sd), strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert m._hubert.dirty
    assert m._param_name("encoder.pos_conv_embed.conv.parametrizations.weight.original1") == "encoder.pos_conv_embed.conv.weight_v"
    assert m._param_name("masked_spec_embed") is None


@pytest.mark.parametrize("fmt", ["bin", "safetensors"])
def test_from_pretrained_loads_a_ctc_checkpoint(tmp_path, fmt, schema):
    from dawn_pytorch_b200.hubert import HubertModel
    sd = O.synth_state_dict(schema["small_a"])
    ctc = {"hubert." + k: v for k, v in _hub_spelling(sd).items()}
    ctc["lm_head.weight"], ctc["lm_head.bias"] = torch.zeros(32, 256), torch.zeros(32)
    (tmp_path / "config.json").write_text(json.dumps(dict(small(), architectures=["HubertForCTC"], vocab_size=32)))
    if fmt == "bin":
        torch.save(ctc, tmp_path / "pytorch_model.bin")
    else:
        from safetensors.torch import save_file
        save_file(ctc, str(tmp_path / "model.safetensors"))
    m = HubertModel.from_pretrained(str(tmp_path))
    assert not m.training
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_state_dict_equals_transformers():
    transformers = pytest.importorskip("transformers")
    from dawn_pytorch_b200.hubert import HubertModel
    for c in (O.SMALL_A, O.SMALL_B):
        ref = transformers.HubertModel(transformers.HubertConfig(**c))
        mine = HubertModel(transformers.HubertConfig(**c))
        assert [(k, v.shape) for k, v in ref.state_dict().items()] == [(k, v.shape) for k, v in mine.state_dict().items()]
        mine.load_state_dict(ref.state_dict(), strict=True)


# ------------------------------------------------------------------------------------------------ the audio pipeline
def test_frame_counts_equal_transformers():
    transformers = pytest.importorskip("transformers")
    from dawn_pytorch_b200.hubert import feat_extract_output_length
    ref = transformers.HubertModel(transformers.HubertConfig(**O.SMALL_A))
    lengths = list(range(400, 2000)) + list(range(2000, 10 ** 6 + 1, 997)) + [320080, 320000, 10 ** 6]
    got = [feat_extract_output_length(O.SMALL_A, n) for n in lengths]
    exp = ref._get_feat_extract_output_lengths(torch.tensor(lengths)).tolist()
    assert got == exp
    assert feat_extract_output_length(O.SMALL_A, 320080) == 1000


def _generator_plan(n):
    """unified_video_generator.py:461-489, the sample ranges it passes to the model"""
    kernel, stride = 400, 320
    clip_length = stride * 1000
    num_iter = n // clip_length
    plan = []
    for i in range(num_iter):
        start_idx = 0 if i == 0 else clip_length * i
        end_idx = (clip_length - stride + kernel) if i == 0 else start_idx + (clip_length - stride + kernel)
        plan.append((start_idx, min(end_idx, n)))
    start = clip_length * num_iter if num_iter > 0 else 0
    if n - start >= kernel:
        plan.append((start, n))
    return plan


@pytest.mark.parametrize("n", [399, 400, 16000, 319999, 320000, 320040, 320080, 320399, 320400, 336037, 640000, 640500, 1_000_003])
def test_segment_plan_is_the_generators(n):
    from dawn_pytorch_b200.hubert import SEGMENT, segment_plan
    assert segment_plan(n) == _generator_plan(n)
    assert SEGMENT == 320080


@pytest.mark.parametrize("full, tail", [(0, 0), (0, 1), (1, 1), (4, 0), (5, 1), (9, 1), (66, 1)])
def test_segment_batches_cap_the_full_segments_per_forward(full, tail):
    from dawn_pytorch_b200.hubert import CLIP, SEGMENT, SEGMENTS_PER_CALL, segment_batches, segment_plan
    n = CLIP * full + (SEGMENT - CLIP if full else 0) + 5000 * tail
    plan = segment_plan(n)
    batches = segment_batches(plan)
    assert [s for b in batches for s in b] == plan                                   # every range once, in order
    assert all(len(b) <= SEGMENTS_PER_CALL for b in batches)
    assert all(len(b) == 1 or all(e - a == SEGMENT for a, e in b) for b in batches)   # only full segments share a forward
    n_full = sum(e - a == SEGMENT for a, e in plan)
    assert len(batches) == -(-n_full // SEGMENTS_PER_CALL) + (len(plan) - n_full)


def _speech(n, dtype, channels=None):
    x = O.synth_speech("norm", n).astype(dtype) * dtype(3.0) + dtype(0.01)
    return np.stack([x, -x], 1) if channels else x


@pytest.mark.parametrize("n, dtype, channels", [(16000, np.float64, None), (336037, np.float64, None), (12345, np.float32, None),
                                                (20000, np.float64, 2)])
def test_normalisation_equals_wav2vec2_feature_extractor(n, dtype, channels):
    transformers = pytest.importorskip("transformers")
    from dawn_pytorch_b200.hubert import normalize
    fe = transformers.Wav2Vec2FeatureExtractor(feature_size=1, sampling_rate=16000, padding_value=0.0, do_normalize=True,
                                               return_attention_mask=True)
    speech = _speech(n, dtype, channels)
    mono = speech[:, 0] if channels else speech                  # unified_video_generator.py:451-452
    ref = fe(mono, return_tensors="np", sampling_rate=16000).input_values[0]
    got = normalize(speech)
    assert got.dtype == np.float32 and np.array_equal(got, ref)


@pytest.mark.parametrize("T, num_frames", [(2, 1), (2, 5), (49, 25), (1049, 525), (999, 2000), (64015, 20000)])
def test_interpolation_equals_interp1d(T, num_frames):
    from scipy.interpolate import interp1d
    from dawn_pytorch_b200.hubert import interpolate
    h = torch.from_numpy(O.synth_speech(f"interp{T}", T * 8).reshape(T, 8) * 30)
    ref = interp1d(np.arange(T), h.numpy(), kind="linear", axis=0)(np.linspace(0, T - 1, num_frames)).astype(np.float32)
    got = interpolate(h, num_frames)
    assert got.dtype == torch.float32 and np.array_equal(got.numpy(), ref)


# ------------------------------------------------------------------------------------------------ C-ABI
def test_header_declares_the_bound_exports():
    from dawn_pytorch_b200 import _lib
    with open(os.path.join(ROOT, "include", "dawn_hubert.h")) as f:
        declared = set(re.findall(r"\b(dawn_hubert_\w+)\s*\(", f.read()))
    assert declared == set(_lib.HUBERT_EXPORTS)
    for name in _lib.HUBERT_EXPORTS:
        assert hasattr(_lib.lib, name)


def _c_struct_fields(header, name):
    """(field, ctype) of `typedef struct { ... } name;` in declaration order; arrays as (field, type[n])"""
    with open(os.path.join(ROOT, "include", header)) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    body = re.search(r"typedef struct \{([^{}]*)\}\s*" + name + r"\s*;", text).group(1)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        m = re.match(r"((?:const\s+)?\w+)\s*(\*?)\s*(.*)", decl)
        base, ptr = m.group(1).replace("const ", ""), m.group(2)
        for item in m.group(3).split(","):
            item = item.strip()
            star = ptr or ("*" if item.startswith("*") else "")
            item = item.lstrip("*").strip()
            arr = re.match(r"(\w+)\[(\w+)\]", item)
            fields.append((arr.group(1), f"{base}{star}[{arr.group(2)}]") if arr else (item, base + star))
    return fields


def test_kernel_case_struct_matches_the_header():
    import ctypes
    from dawn_pytorch_b200 import _lib
    ctype = {ctypes.c_int: "int", ctypes.c_float: "float", ctypes.c_void_p: "float*"}
    got = [(n, ctype[t]) for n, t in _lib.DawnHubertKernelCase._fields_]
    assert got == _c_struct_fields("dawn_hubert.h", "dawn_hubert_kernel_case")
    with open(os.path.join(ROOT, "include", "dawn_hubert.h")) as f:
        kinds = re.findall(r"DAWN_HUBERT_(\w+) = (\d+)", f.read())
    assert [(k, int(v)) for k, v in kinds] == [(k, getattr(_lib, "HUBERT_" + k)) for k, _ in kinds]
