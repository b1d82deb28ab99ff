"""CPU: the drop-in boundary — module mirror of the reference state_dict, C-ABI symbols, host-side logic."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CTOR = dict(dim=64, cond_dim=1032, cond_aud=1024, cond_pose=6, cond_eye=2, num_frames=40, channels=275,
            out_grid_dim=2, out_conf_dim=1, dim_mults=(1, 2, 4, 8), use_hubert_audio_cond=True,
            learn_null_cond=False, use_final_activation=False, use_deconv=True, padding_mode="zeros", win_width=40)


def test_library_exports_every_declared_symbol():
    from dawn_pytorch_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "dawn_unet.h")).read()
    declared = set(re.findall(r"\b(dawn_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    for sym in declared:
        assert hasattr(_lib.lib, sym), f"{sym} declared in include/dawn_unet.h but not exported"
    assert declared == set(_lib.EXPORTS)
    assert b"sm_90a" in _lib.lib.dawn_build_info()


def test_state_dict_schema_equals_reference(schema):
    from dawn_pytorch_b200 import DynamicNfUnet3D
    net = DynamicNfUnet3D(**CTOR)
    mine = [(k, list(v.shape)) for k, v in net.state_dict().items()]
    ref = [(k, list(s)) for k, s in schema["entries"]]
    assert len(mine) == len(ref) == 900
    assert dict(mine) == dict(ref)
    assert [k for k, _ in mine] == [k for k, _ in ref], "same registration order as the reference"
    assert net.num_frames == 20 and net.has_cond


def test_load_reference_style_state_dict_and_api_surface(synth_sd):
    from dawn_pytorch_b200 import DynamicNfUnet3D
    net = DynamicNfUnet3D(**CTOR).eval()
    missing = net.load_state_dict(synth_sd, strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    net.update_num_frames(16)
    assert net.num_frames == 16
    for attr in ("forward", "forward_with_cond_scale", "update_num_frames", "null_cond_mask", "has_cond"):
        assert hasattr(net, attr)


def test_cpu_tensors_fail_loudly(synth_sd):
    """No CPU fallback: calling the module with CPU tensors must raise, not silently compute."""
    from dawn_pytorch_b200 import DynamicNfUnet3D
    from dawn_pytorch_b200._lib import DawnError
    net = DynamicNfUnet3D(**CTOR).eval()
    net.update_num_frames(4)
    with pytest.raises(DawnError):
        net.forward_with_cond_scale(torch.zeros(1, 275, 4, 8, 8), torch.zeros(1, dtype=torch.long),
                                    cond=torch.zeros(1, 4, 1032), cond_scale=1.0)


def test_c_abi_argument_checks_without_gpu():
    from dawn_pytorch_b200 import _lib
    lib = _lib.lib
    cfg = _lib.DawnUnetCfg()
    cfg.dim, cfg.n_levels = 64, 4
    for i, m in enumerate((1, 2, 4, 8)):
        cfg.dim_mults[i] = m
    cfg.channels, cfg.cond_aud, cfg.cond_pose, cfg.cond_eye = 275, 1024, 6, 2
    cfg.out_grid_dim, cfg.out_conf_dim, cfg.attn_heads, cfg.attn_dim_head, cfg.resnet_groups = 2, 1, 8, 32, 8
    cfg.init_kernel_size, cfg.win_width = 7, 40
    h = ctypes.c_void_p()
    assert lib.dawn_unet_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    # wrong call order is an error, not a crash
    assert lib.dawn_unet_set_num_frames(h, 16, 32, 32) == -1
    assert b"commit_params" in lib.dawn_last_error()
    lib.dawn_unet_destroy(h)
    cfg.attn_heads = 4
    assert lib.dawn_unet_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
    assert b"attn_heads" in lib.dawn_last_error()


def test_rel_bias_table_matches_oracle(synth_sd):
    from dawn_pytorch_b200.unet import _rel_bias_table, _time_freqs
    from oracle import unet_oracle as O
    w = synth_sd["time_rel_pos_bias.relative_attention_bias.weight"]
    full = O.rel_pos_bias(w, 200, 40)                      # (8, 200, 200) incl. -1e8 mask
    tab = _rel_bias_table(w, 40)                           # (8, 81)
    for i in (0, 57, 199):
        for j in range(max(0, i - 40), min(200, i + 41)):
            assert torch.equal(full[:, i, j], tab[:, j - i + 40])
    assert torch.equal(O.sinusoidal(torch.tensor([500]), 64)[0, :32], torch.sin(500 * _time_freqs(64)))


# ----------------------------------------------------------------------------- LFG flow decoder boundary (include/dawn_lfg.h)
LFG_CTOR = dict(num_channels=3, num_regions=10, block_expansion=64, max_features=512, num_down_blocks=2, num_bottleneck_blocks=6,
                pixelwise_flow_predictor_params={"block_expansion": 64}, skips=True, revert_axis_swap=True)


def test_lfg_library_exports_every_declared_symbol():
    from dawn_pytorch_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "dawn_lfg.h")).read()
    declared = set(re.findall(r"\b(dawn_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.LFG_EXPORTS) | set(_lib.MISC_EXPORTS)
    for sym in declared:
        assert hasattr(_lib.lib, sym), f"{sym} declared in include/dawn_lfg.h but not exported"


def test_lfg_state_dict_schema_equals_reference_decode_path(golden_dir):
    import json
    from dawn_pytorch_b200 import LfgGenerator
    from oracle import weights as W
    with open(os.path.join(golden_dir, "lfg_state_dict_schema.json")) as f:
        sch = json.load(f)
    g = LfgGenerator(**LFG_CTOR)
    mine = [(k, list(v.shape)) for k, v in g.state_dict().items()]
    assert mine == [(k, list(s)) for k, s in sch["entries"]]          # same keys, shapes and registration order (dumped from the reference)
    sd = W.lfg_synth_state_dict([(n, tuple(s)) for n, s in sch["entries"]])
    sd["pixelwise_flow_predictor.hourglass.encoder.down_blocks.0.conv.weight"] = torch.zeros(4)     # training-only entries of the checkpoint
    res = g.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert not g.training
    with pytest.raises(NotImplementedError):
        g.train()


def test_lfg_cpu_tensors_fail_loudly_and_argument_checks():
    from dawn_pytorch_b200 import LfgGenerator, _lib
    g = LfgGenerator(**LFG_CTOR)
    with pytest.raises(_lib.DawnError):
        g.forward_with_flow(torch.rand(1, 3, 64, 64), torch.zeros(2, 16, 16, 2), torch.zeros(2, 1, 16, 16))
    lib = _lib.lib
    cfg = _lib.DawnLfgCfg()
    cfg.num_channels, cfg.block_expansion, cfg.max_features = 3, 64, 512
    cfg.num_down_blocks, cfg.num_bottleneck_blocks, cfg.skips = 2, 6, 1
    h = ctypes.c_void_p()
    assert lib.dawn_lfg_create(ctypes.byref(cfg), ctypes.byref(h)) == 0
    assert lib.dawn_lfg_set_geometry(h, 4, 64, 64, 16, 16) == -1          # wrong call order is an error, not a crash
    assert b"commit_params" in lib.dawn_last_error()
    lib.dawn_lfg_destroy(h)
    cfg.num_channels = 4
    assert lib.dawn_lfg_create(ctypes.byref(cfg), ctypes.byref(h)) == -1


def test_flow_diffusion_wrapper_structure_and_bbox_mask(golden_dir):
    """N3: the consumer wrapper keeps the reference's attribute names / state_dict layout (UVG:527-528 loads `diffusion`),
    and its face-box mask equals the reference's (value from the real `generate_bbox_mask`, oracle/make_golden_e2e.py)."""
    import numpy as np
    from dawn_pytorch_b200 import FlowDiffusion
    m = FlowDiffusion(sampling_timesteps=20, pose_dim=6)
    assert len(m.diffusion.state_dict()) == 912 and len(m.unet.state_dict()) == 900
    assert len(m.generator.state_dict()) == 121 and list(m.face_loc_emb.state_dict()) == ["conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias"]
    m.update_num_frames(123)
    assert m.unet.num_frames == 123 and m.diffusion.num_frames == 123
    g = np.load(os.path.join(golden_dir, "e2e_sample_one_video.npz"))
    bbox = torch.tensor([[20., 44., 16., 50., 64., 64.]]).unsqueeze(-1).repeat(1, 1, 8)
    mask = m.generate_bbox_mask(bbox, size=64)
    assert mask.shape == (1, 1, 64, 64) and float(mask.sum()) == float(g["bbox_mask_sum"])
    assert bbox[0, 0, 0] == 20.0                                  # the caller's tensor is not modified (the reference scales it in place)
    # the shipped configs (config/DAWN_128.yaml: is_train: true) construct with is_train=True and only ever sample (UVG:516, 529):
    # accepted with a warning, the module stays in eval mode, the training entry point raises
    with pytest.warns(UserWarning):
        mt = FlowDiffusion(is_train=True)
    assert not mt.training and not mt.unet.training
    with pytest.raises(NotImplementedError):
        mt(None)


def test_fast_path_checks_shapes_before_touching_the_device():
    """ADVICE r1: the hoisted entry takes raw pointers, so a geometry mismatch must raise instead of reading out of bounds
    (the reference raises a broadcast error at U:925-926)."""
    from dawn_pytorch_b200 import DynamicNfUnet3D
    from dawn_pytorch_b200._lib import DawnError
    from tests.gpu_common import CTOR
    net = DynamicNfUnet3D(**CTOR).eval()
    net.update_num_frames(8)
    with pytest.raises(ValueError):
        net.set_clip_invariants(torch.zeros(271, 8, 8), torch.zeros(8, 1032))         # wrong feature channels
    with pytest.raises(ValueError):
        net.set_clip_invariants(torch.zeros(272, 8, 8), torch.zeros(8, 1031))         # wrong cond width
    with pytest.raises(ValueError):
        net.set_clip_invariants(torch.zeros(272, 8, 8), torch.zeros(9, 1032))         # update_num_frames not called for 9 frames
    with pytest.raises(ValueError):
        net.set_clip_invariants(torch.zeros(1, 272, 8, 8), torch.zeros(8, 1032))      # batched tensor
    with pytest.raises(DawnError):
        net.set_clip_invariants(torch.zeros(272, 8, 8), torch.zeros(8, 1032))         # right shapes, CPU tensors: no CPU path
    with pytest.raises(DawnError):
        net.forward_x3(torch.zeros(3, 8, 8, 8), torch.zeros(1, dtype=torch.long))     # invariants never set
