"""ctypes binding of include/dawn_unet.h, include/dawn_lfg.h, include/dawn_pbnet.h, include/dawn_hubert.h and include/dawn_video.h,
and the lifecycle every module shares
with its native handles.  The product path has no fallback: if the CUDA library is missing or fails to load, importing this
module raises."""
import ctypes
import os

import torch
from torch import nn

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdawn_unet.so")


class DawnUnetCfg(ctypes.Structure):
    _fields_ = [("dim", ctypes.c_int), ("n_levels", ctypes.c_int), ("dim_mults", ctypes.c_int * 8),
                ("channels", ctypes.c_int), ("cond_aud", ctypes.c_int), ("cond_pose", ctypes.c_int),
                ("cond_eye", ctypes.c_int), ("out_grid_dim", ctypes.c_int), ("out_conf_dim", ctypes.c_int),
                ("attn_heads", ctypes.c_int), ("attn_dim_head", ctypes.c_int), ("resnet_groups", ctypes.c_int),
                ("init_kernel_size", ctypes.c_int), ("win_width", ctypes.c_int),
                ("upconv", ctypes.c_int), ("pad_mode", ctypes.c_int), ("no_sla", ctypes.c_int)]


class DawnLfgCfg(ctypes.Structure):
    """include/dawn_lfg.h: dawn_lfg_cfg"""
    _fields_ = [("num_channels", ctypes.c_int), ("block_expansion", ctypes.c_int), ("max_features", ctypes.c_int),
                ("num_down_blocks", ctypes.c_int), ("num_bottleneck_blocks", ctypes.c_int), ("skips", ctypes.c_int)]


PATH_MMA_SYNC, PATH_TC_GEMM, PATH_TC_GEMM_PRESPLIT, PATH_TC_CONV3, PATH_TC_CONV3_TMA = range(5)
EPI_PLAIN, EPI_QKV_TEMPORAL, EPI_QKV_SLA, EPI_QKV_MID, EPI_CA_GATE, EPI_GN_APPLY, EPI_GELU, EPI_LN_BIAS, EPI_LN_BIAS_GELU = range(9)


class DawnContractionCase(ctypes.Structure):
    """include/dawn_unet.h: dawn_contraction_case (pointers are device addresses)"""
    _i, _p = ctypes.c_int, ctypes.c_void_p
    _fields_ = [("path", _i), ("epi", _i),
                ("F", _i), ("IH", _i), ("IW", _i), ("Cin", _i), ("lda", _i),
                ("ntaps", _i), ("dy", _i * 52), ("dx", _i * 52), ("in_stride", _i),
                ("OHs", _i), ("OWs", _i), ("OH", _i), ("OW", _i), ("out_stride", _i), ("oy0", _i), ("ox0", _i),
                ("up2", _i),
                ("perm_pb", _i), ("perm_F", _i), ("perm_in", _i), ("perm_out", _i), ("perm_f_lo", _i), ("perm_f_hi", _i),
                ("P", _i),
                ("N", _i), ("ldb", _i), ("ldo", _i), ("ldr", _i), ("drain", _i), ("ln_inline", _i),
                ("rows_per_batch", _i), ("b_batch_stride", ctypes.c_longlong), ("cpg", _i),
                ("q_post_scale", ctypes.c_float),
                ("A", _p), ("B", _p), ("bias", _p), ("Res", _p), ("Out", _p),
                ("stats", _p), ("rowstats", _p), ("wsum", _p), ("rot", _p),
                ("kq", _p), ("nkq", _p), ("gates", _p),
                ("Y", _p), ("ldy", _i), ("gn_stats", _p), ("gn_w", _p), ("gn_b", _p), ("film", _p), ("gn_count", ctypes.c_double)]


FUSED_TEMPORAL, FUSED_ATTN_TC, FUSED_ATTN_SIMT, FUSED_SLA_CTX, FUSED_SLA_OUT, FUSED_SLA_CTX_UNFUSED, FUSED_CA_WT, \
    FUSED_CA_RSTD, FUSED_GN_HCOND, FUSED_TEMPORAL_MMA_SYNC = range(10)


class DawnFusedCase(ctypes.Structure):
    """include/dawn_unet.h: dawn_fused_case (pointers are device addresses)"""
    _i, _p = ctypes.c_int, ctypes.c_void_p
    _fields_ = [("kernel", _i), ("F", _i), ("P", _i), ("C", _i), ("band", _i), ("q_lo", _i), ("q_hi", _i),
                ("nseq", _i), ("L", _i), ("pb", _i), ("seq_base_stride", ctypes.c_longlong), ("elem_stride", ctypes.c_longlong),
                ("ldx", _i), ("ldr", _i), ("ldo", _i), ("ld", _i), ("ldb", _i), ("ldy", _i), ("ldbT", _i),
                ("x", _p), ("res", _p), ("out", _p), ("gamma", _p), ("w_qkv", _p), ("w_out", _p), ("rot", _p), ("bias", _p),
                ("qkv", _p), ("Bf", _p), ("out_bias", _p), ("kq", _p), ("nkq", _p), ("G", _p), ("gates", _p), ("Wt", _p),
                ("T", _p), ("Y", _p), ("out16h", _p), ("out16l", _p),
                ("gn_stats", _p), ("gn_count", ctypes.c_double), ("cpg", _i), ("gn_w", _p), ("gn_b", _p), ("film", _p)]


KERNEL_ROWSTATS, KERNEL_GN_APPLY, KERNEL_COND_TABLES, KERNEL_TIME_MLP, KERNEL_FILM, KERNEL_ROTARY, KERNEL_SPLIT_ROWS, \
    KERNEL_NCF_TO_NHWC, KERNEL_FRAME_INVARIANCE, KERNEL_FEA_SHIFT, KERNEL_MAP_REDUCE, KERNEL_INIT_CONV_X3, KERNEL_HEADS_OUT, \
    KERNEL_DDIM_STEP, KERNEL_DDPM_STEP, KERNEL_Q_SAMPLE, KERNEL_MOTION_TO_LATENT = range(17)
KERNEL_MAX_DESC = 16


class DawnKernelDesc(ctypes.Structure):
    """include/dawn_unet.h: dawn_kernel_desc (pointers are device addresses)"""
    _i, _p = ctypes.c_int, ctypes.c_void_p
    _fields_ = [("off", _i), ("K", _i), ("co", _i), ("ldbT", _i), ("ca", _i),
                ("mW", _p), ("mB", _p), ("Wkv", _p), ("nkv", _p), ("qs", _p), ("ks", _p), ("Wout", _p), ("gout", _p),
                ("ctx", _p), ("kv", _p), ("kq", _p), ("nkq", _p), ("T", _p), ("G", _p),
                ("W", _p), ("b", _p), ("out", _p), ("n", _i)]


class DawnKernelCase(ctypes.Structure):
    """include/dawn_unet.h: dawn_kernel_case (pointers are device addresses)"""
    _i, _p, _ll = ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong
    _fields_ = [("kernel", _i), ("M", _i), ("C", _i), ("ld", _i), ("ldy", _i), ("ldr", _i), ("ldo", _i),
                ("F", _i), ("H", _i), ("W", _i), ("P", _i), ("clips", _i),
                ("Cpad", _i), ("c0", _i), ("k", _i), ("skip_if", _i), ("cpg", _i), ("t_stride", _i), ("pos0", _i), ("dim", _i),
                ("ng", _i), ("nc", _i), ("cond_ld", _i), ("ndesc", _i),
                ("n", _ll), ("cstride", _ll), ("clip_stride", _ll), ("count", ctypes.c_double), ("eps", ctypes.c_float),
                ("x", _p), ("y", _p), ("res", _p), ("w", _p), ("b", _p), ("w2", _p), ("b2", _p),
                ("map", _p), ("freqs", _p), ("stats", _p), ("t", _p), ("skip_flag", _p),
                ("out", _p), ("out_hi", _p), ("out_lo", _p), ("flag", _p),
                ("desc", DawnKernelDesc * KERNEL_MAX_DESC),
                ("xs", _p), ("e", _p), ("noise", _p), ("scratch", _p), ("tab", _p), ("t_slot", _p), ("num_t", _i),
                ("replicas", _i), ("coef", ctypes.c_float * 5), ("q", ctypes.c_float)]


LFG_MOTION_PACK, LFG_WARP_BLEND, LFG_AFFINE_RELU, LFG_RESIDUAL_BN_RELU, LFG_RELU_AVGPOOL2, LFG_CHW_TO_HWC, LFG_HWC_TO_CHW, \
    LFG_FINAL_CONV = range(8)


class DawnLfgKernelCase(ctypes.Structure):
    """include/dawn_lfg.h: dawn_lfg_kernel_case (pointers are device addresses)"""
    _i, _p = ctypes.c_int, ctypes.c_void_p
    _fields_ = [("kernel", _i), ("F", _i), ("H", _i), ("W", _i), ("h", _i), ("w", _i), ("C", _i), ("Cpad", _i),
                ("layout", _i), ("blend", _i), ("ldx", _i), ("ldp", _i), ("ldo", _i), ("M", ctypes.c_longlong),
                ("x", _p), ("y", _p), ("flow", _p), ("occ", _p), ("motion", _p), ("prev", _p), ("scale", _p), ("shift", _p),
                ("weight", _p), ("bias", _p), ("source", _p), ("out", _p), ("out2", _p)]


class DawnLfgMotionCfg(ctypes.Structure):
    """include/dawn_lfg.h: dawn_lfg_motion_cfg"""
    _i, _f = ctypes.c_int, ctypes.c_float
    _fields_ = [("num_regions", _i), ("num_channels", _i), ("estimate_affine", _i), ("pca_based", _i), ("fast_svd", _i),
                ("rp_block_expansion", _i), ("rp_max_features", _i), ("rp_num_blocks", _i), ("rp_temperature", _f),
                ("rp_scale_factor", _f), ("bg_block_expansion", _i), ("bg_max_features", _i), ("bg_num_blocks", _i),
                ("bg_type", _i), ("pw_block_expansion", _i), ("pw_max_features", _i), ("pw_num_blocks", _i),
                ("pw_scale_factor", _f), ("use_covar_heatmap", _i), ("use_deformed_source", _i),
                ("estimate_occlusion_map", _i), ("revert_axis_swap", _i)]


LFG_BG_ZERO, LFG_BG_AFFINE = 0, 1
LFGM_AA_DOWN, LFGM_REGION_MOMENTS, LFGM_FLOW_INPUT, LFGM_FLOW_COMBINE, LFGM_BG_HEAD = range(5)


class DawnLfgMotionKernelCase(ctypes.Structure):
    """include/dawn_lfg.h: dawn_lfg_motion_kernel_case (pointers are device addresses)"""
    _i, _p = ctypes.c_int, ctypes.c_void_p
    _fields_ = [("kernel", _i), ("N", _i), ("H", _i), ("W", _i), ("h", _i), ("w", _i), ("R", _i), ("ld", _i), ("off", _i),
                ("cw", _i), ("ldl", _i), ("revert", _i), ("temperature", ctypes.c_float),
                ("x", _p), ("weight", _p), ("logits", _p), ("motion", _p), ("source", _p), ("bg", _p), ("fc_w", _p), ("fc_b", _p),
                ("src_shift", _p), ("src_covar", _p), ("src_affine", _p), ("drv_shift", _p), ("drv_covar", _p), ("drv_affine", _p),
                ("out", _p), ("out2", _p), ("out3", _p)]


class DawnPbnetCfg(ctypes.Structure):
    """include/dawn_pbnet.h: dawn_pbnet_cfg"""
    _fields_ = [(n, ctypes.c_int) for n in ("band", "pose_dim", "audio_dim", "latent_dim", "audio_latent_dim", "pose_latent_dim",
                                            "ff_size", "num_layers", "num_heads")]


class DawnPbnetAttentionCase(ctypes.Structure):
    """include/dawn_pbnet.h: dawn_pbnet_attention_case (pointers are device addresses)"""
    _i, _p = ctypes.c_int, ctypes.c_void_p
    _fields_ = [("bs", _i), ("F", _i), ("D", _i), ("H", _i), ("band", _i), ("npairs", _i), ("qscale", ctypes.c_float),
                ("x_q", _p), ("x_kv", _p), ("wq", _p), ("wk", _p), ("wv", _p), ("freqs", _p), ("bias", _p), ("out", _p)]


PBNET_MEMORY, PBNET_PROJ, PBNET_OUT_LN, PBNET_FFN_LN = range(4)


class DawnPbnetKernelCase(ctypes.Structure):
    """include/dawn_pbnet.h: dawn_pbnet_kernel_case (pointers are device addresses)"""
    _fields_ = [(n, ctypes.c_int) for n in ("kernel", "T", "bs", "F", "D", "Lz", "PE", "ldx", "hid", "ngroups", "npairs", "ldr", "ff",
                                            "nout")] + \
               [("flags", ctypes.c_int * 8), ("qscale", ctypes.c_float)] + \
               [(n, ctypes.c_void_p) for n in ("x", "z", "xref", "w", "w2", "b1", "b2", "gamma", "beta", "wf", "bf", "rot", "res",
                                               "mask", "out")]


class DawnHubertCfg(ctypes.Structure):
    """include/dawn_hubert.h: dawn_hubert_cfg"""
    _i = ctypes.c_int
    _fields_ = [("hidden_size", _i), ("num_layers", _i), ("num_heads", _i), ("intermediate_size", _i), ("num_conv", _i),
                ("conv_dim", _i * 8), ("conv_kernel", _i * 8), ("conv_stride", _i * 8), ("conv_bias", _i), ("pos_kernel", _i),
                ("pos_groups", _i), ("layer_norm_eps", ctypes.c_float)]


HUBERT_ATTENTION, HUBERT_CONV0, HUBERT_POS_CONV, HUBERT_ROW_LN, HUBERT_FE_CONV, HUBERT_LN_LINEAR = range(6)


class DawnHubertKernelCase(ctypes.Structure):
    """include/dawn_hubert.h: dawn_hubert_kernel_case (pointers are device addresses)"""
    _i, _p = ctypes.c_int, ctypes.c_void_p
    _fields_ = [("kernel", _i), ("B", _i), ("T", _i), ("L", _i), ("H", _i), ("ld", _i), ("C", _i), ("k", _i), ("s", _i), ("G", _i),
                ("eps", ctypes.c_float), ("q", _p), ("kk", _p), ("v", _p), ("x", _p), ("w", _p), ("bias", _p), ("gamma", _p),
                ("beta", _p), ("g", _p), ("out", _p),
                ("M", _i), ("N", _i), ("ldo", _i), ("gelu", _i), ("parts", _i), ("qscale", ctypes.c_float)]


class DawnError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python dawn_pytorch_b200/build.py` "
            "(nvcc, sm_90a). There is no CPU or PyTorch fallback for the DAWN denoising UNet.")
    lib = ctypes.CDLL(LIB_PATH)
    vp, i64p, fp, cp = ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64), ctypes.c_void_p, ctypes.c_char_p
    lib.dawn_unet_create.argtypes = [ctypes.POINTER(DawnUnetCfg), ctypes.POINTER(vp)]
    lib.dawn_unet_destroy.argtypes = [vp]
    lib.dawn_unet_destroy.restype = None
    lib.dawn_unet_set_param.argtypes = [vp, cp, fp, i64p, ctypes.c_int]
    lib.dawn_unet_commit_params.argtypes = [vp]
    lib.dawn_unet_set_num_frames.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.dawn_unet_set_geometry.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.dawn_unet_set_clip_invariants.argtypes = [vp, fp, fp, vp]
    lib.dawn_unet_forward.argtypes = [vp, fp, vp, fp, fp, vp]
    lib.dawn_unet_forward_x3.argtypes = [vp, fp, vp, fp, vp]
    lib.dawn_unet_forward_host.argtypes = [vp, fp, fp, fp, ctypes.c_int64, fp]
    lib.dawn_unet_set_tap.argtypes = [vp, cp, fp]
    lib.dawn_unet_tap_shape.argtypes = [vp, cp, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int),
                                        ctypes.POINTER(ctypes.c_int)]
    dp = ctypes.POINTER(ctypes.c_double)
    lib.dawn_unet_profile_enable.argtypes = [vp, ctypes.c_int]
    lib.dawn_unet_profile_read.argtypes = [vp, dp, dp, dp, i64p]
    lib.dawn_unet_last_launch_count.argtypes = [vp]
    lib.dawn_unet_last_launch_count.restype = ctypes.c_int64
    lib.dawn_unet_workspace_bytes.argtypes = [vp]
    lib.dawn_unet_workspace_bytes.restype = ctypes.c_int64
    lib.dawn_test_contraction.argtypes = [ctypes.POINTER(DawnContractionCase), vp]
    lib.dawn_test_fused.argtypes = [ctypes.POINTER(DawnFusedCase), vp]
    lib.dawn_test_kernel.argtypes = [ctypes.POINTER(DawnKernelCase), vp]
    lib.dawn_nccl_unique_id.argtypes = [ctypes.c_char_p]
    lib.dawn_unet_init_shard.argtypes = [vp, ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.dawn_unet_shard_ipc_export.argtypes = [vp, ctypes.c_char_p]
    lib.dawn_unet_shard_ipc_import.argtypes = [vp, ctypes.c_char_p]
    lib.dawn_ddim_step.argtypes = [fp, fp, fp, ctypes.c_int64] + [ctypes.c_float] * 6 + [vp, vp]
    lib.dawn_unet_ddim_step.argtypes = [vp, fp, fp, fp, ctypes.c_int64] + [ctypes.c_float] * 6 + [vp, vp]
    lib.dawn_unet_sampler_capture.argtypes = [vp, fp, fp, fp, vp, ctypes.POINTER(ctypes.c_float), ctypes.c_int, ctypes.c_float, vp]
    lib.dawn_unet_sampler_launch.argtypes = [vp, vp]
    lib.dawn_unet_ddim_step_guided.argtypes = [vp, fp, fp, fp, ctypes.c_int64, fp] + [ctypes.c_float] * 6 + [vp, vp]
    lib.dawn_unet_sampler_capture_guided.argtypes = [vp, fp, fp, fp, vp, fp, ctypes.POINTER(ctypes.c_float), ctypes.c_int,
                                                     ctypes.c_float, vp]
    lib.dawn_unet_sampler_launch_guided.argtypes = [vp, vp]
    lib.dawn_ddpm_step.argtypes = [fp, fp, fp, ctypes.c_int64] + [ctypes.c_float] * 6 + [vp, vp]
    lib.dawn_unet_ddpm_step.argtypes = [vp, fp, fp, fp, ctypes.c_int64] + [ctypes.c_float] * 6 + [vp, vp]
    lib.dawn_unet_ddpm_capture.argtypes = [vp, fp, fp, fp, vp, fp, ctypes.c_int, ctypes.c_float, vp]
    lib.dawn_unet_ddpm_launch.argtypes = [vp, vp]
    lib.dawn_q_sample.argtypes = [fp, fp, vp, fp, fp, ctypes.c_int, ctypes.c_int64, ctypes.c_int64, fp, vp]
    lib.dawn_motion_to_latent.argtypes = [fp, fp, ctypes.c_int64] + [ctypes.c_int] * 3 + [vp, fp, fp, fp, ctypes.c_int, fp, vp]
    ip = ctypes.POINTER(ctypes.c_int)
    lib.dawn_lfg_create.argtypes = [ctypes.POINTER(DawnLfgCfg), ctypes.POINTER(vp)]
    lib.dawn_lfg_destroy.argtypes = [vp]
    lib.dawn_lfg_destroy.restype = None
    lib.dawn_lfg_set_param.argtypes = [vp, cp, fp, i64p, ctypes.c_int]
    lib.dawn_lfg_commit_params.argtypes = [vp]
    lib.dawn_lfg_set_geometry.argtypes = [vp] + [ctypes.c_int] * 5
    lib.dawn_lfg_set_source.argtypes = [vp, fp, vp]
    lib.dawn_lfg_get_fea.argtypes = [vp, fp, vp]
    lib.dawn_lfg_decode.argtypes = [vp, fp, fp, fp, fp, vp]
    lib.dawn_lfg_decode_sample.argtypes = [vp, fp, fp, fp, vp]
    lib.dawn_lfg_decode_sample_rgb8.argtypes = [vp, fp, ctypes.POINTER(ctypes.c_double), fp, vp]
    lib.dawn_lfg_read_tap.argtypes = [vp, cp, fp, ip, ip, ip, vp]
    lib.dawn_conv3x3_s2_relu.argtypes = [fp, ctypes.c_int, ctypes.c_int, ctypes.c_int, fp, fp, ctypes.c_int, fp, vp]
    lib.dawn_lfg_last_launch_count.argtypes = [vp]
    lib.dawn_lfg_last_launch_count.restype = ctypes.c_int64
    lib.dawn_lfg_workspace_bytes.argtypes = [vp]
    lib.dawn_lfg_workspace_bytes.restype = ctypes.c_int64
    lib.dawn_lfg_test_kernel.argtypes = [ctypes.POINTER(DawnLfgKernelCase), vp]
    lib.dawn_lfg_motion_create.argtypes = [ctypes.POINTER(DawnLfgMotionCfg), ctypes.POINTER(vp)]
    lib.dawn_lfg_motion_destroy.argtypes = [vp]
    lib.dawn_lfg_motion_destroy.restype = None
    lib.dawn_lfg_motion_set_param.argtypes = [vp, cp, fp, i64p, ctypes.c_int]
    lib.dawn_lfg_motion_commit_params.argtypes = [vp]
    lib.dawn_lfg_motion_set_geometry.argtypes = [vp] + [ctypes.c_int] * 3
    lib.dawn_lfg_motion_regions.argtypes = [vp, fp, ctypes.c_int, fp, fp, fp, vp]
    lib.dawn_lfg_motion_bg.argtypes = [vp, fp, ctypes.c_int, fp, ctypes.c_int, fp, vp]
    lib.dawn_lfg_motion_flow.argtypes = [vp, fp, ctypes.c_int] + [fp] * 9 + [vp]
    lib.dawn_lfg_motion_read_tap.argtypes = [vp, cp, fp, ip, ip, ip, ip, vp]
    lib.dawn_lfg_motion_last_launch_count.argtypes = [vp]
    lib.dawn_lfg_motion_last_launch_count.restype = ctypes.c_int64
    lib.dawn_lfg_motion_workspace_bytes.argtypes = [vp]
    lib.dawn_lfg_motion_workspace_bytes.restype = ctypes.c_int64
    lib.dawn_lfg_motion_test_kernel.argtypes = [ctypes.POINTER(DawnLfgMotionKernelCase), vp]
    lib.dawn_pbnet_create.argtypes = [ctypes.POINTER(DawnPbnetCfg), ctypes.POINTER(vp)]
    lib.dawn_pbnet_destroy.argtypes = [vp]
    lib.dawn_pbnet_destroy.restype = None
    lib.dawn_pbnet_set_param.argtypes = [vp, cp, fp, i64p, ctypes.c_int]
    lib.dawn_pbnet_commit_params.argtypes = [vp]
    lib.dawn_pbnet_generate.argtypes = [vp, fp, fp, fp, fp, ctypes.c_int, ctypes.c_int, fp, vp]
    lib.dawn_pbnet_last_launch_count.argtypes = [vp]
    lib.dawn_pbnet_last_launch_count.restype = ctypes.c_int64
    lib.dawn_pbnet_workspace_bytes.argtypes = [vp]
    lib.dawn_pbnet_workspace_bytes.restype = ctypes.c_int64
    lib.dawn_pbnet_test_attention.argtypes = [ctypes.POINTER(DawnPbnetAttentionCase), vp]
    lib.dawn_pbnet_test_kernel.argtypes = [ctypes.POINTER(DawnPbnetKernelCase), vp]
    lib.dawn_hubert_create.argtypes = [ctypes.POINTER(DawnHubertCfg), ctypes.POINTER(vp)]
    lib.dawn_hubert_destroy.argtypes = [vp]
    lib.dawn_hubert_destroy.restype = None
    lib.dawn_hubert_set_param.argtypes = [vp, cp, fp, i64p, ctypes.c_int]
    lib.dawn_hubert_commit_params.argtypes = [vp]
    lib.dawn_hubert_forward.argtypes = [vp, fp, ctypes.c_int, ctypes.c_int, fp, vp]
    lib.dawn_hubert_output_length.argtypes = [vp, ctypes.c_int]
    lib.dawn_hubert_hidden.argtypes = [vp, fp, ctypes.c_int, ctypes.c_int, ctypes.c_int, fp, vp]
    lib.dawn_hubert_last_launch_count.argtypes = [vp]
    lib.dawn_hubert_last_launch_count.restype = ctypes.c_int64
    lib.dawn_hubert_workspace_bytes.argtypes = [vp]
    lib.dawn_hubert_workspace_bytes.restype = ctypes.c_int64
    lib.dawn_hubert_test_kernel.argtypes = [ctypes.POINTER(DawnHubertKernelCase), vp]
    lib.dawn_portrait_resize.argtypes = [fp, ctypes.c_int, ctypes.c_int, ctypes.c_int, fp, fp, vp]
    lib.dawn_last_error.restype = cp
    lib.dawn_live_bytes.argtypes = []
    lib.dawn_live_bytes.restype = ctypes.c_int64
    lib.dawn_build_info.restype = cp
    return lib


lib = _load()

EXPORTS = ["dawn_unet_create", "dawn_unet_destroy", "dawn_unet_set_param", "dawn_unet_commit_params",
           "dawn_unet_set_num_frames", "dawn_unet_set_geometry", "dawn_nccl_unique_id", "dawn_unet_init_shard", "dawn_unet_shard_ipc_export", "dawn_unet_shard_ipc_import", "dawn_unet_set_clip_invariants", "dawn_unet_forward",
           "dawn_unet_forward_x3", "dawn_unet_forward_host", "dawn_unet_set_tap", "dawn_unet_tap_shape",
           "dawn_unet_profile_enable", "dawn_unet_profile_read", "dawn_unet_last_launch_count", "dawn_unet_workspace_bytes", "dawn_ddim_step", "dawn_unet_ddim_step", "dawn_unet_sampler_capture", "dawn_unet_sampler_launch",
           "dawn_unet_ddim_step_guided", "dawn_unet_sampler_capture_guided", "dawn_unet_sampler_launch_guided",
           "dawn_ddpm_step", "dawn_unet_ddpm_step", "dawn_unet_ddpm_capture", "dawn_unet_ddpm_launch",
           "dawn_q_sample", "dawn_motion_to_latent",
           "dawn_test_contraction", "dawn_test_fused", "dawn_test_kernel", "dawn_last_error", "dawn_live_bytes", "dawn_build_info"]


LFG_EXPORTS = ["dawn_lfg_create", "dawn_lfg_destroy", "dawn_lfg_set_param", "dawn_lfg_commit_params", "dawn_lfg_set_geometry",
               "dawn_lfg_set_source", "dawn_lfg_get_fea", "dawn_lfg_decode", "dawn_lfg_decode_sample",
               "dawn_lfg_decode_sample_rgb8", "dawn_lfg_read_tap",
               "dawn_lfg_last_launch_count", "dawn_lfg_workspace_bytes", "dawn_lfg_test_kernel"]
LFG_MOTION_EXPORTS = ["dawn_lfg_motion_create", "dawn_lfg_motion_destroy", "dawn_lfg_motion_set_param",
                      "dawn_lfg_motion_commit_params", "dawn_lfg_motion_set_geometry", "dawn_lfg_motion_regions", "dawn_lfg_motion_bg",
                      "dawn_lfg_motion_flow", "dawn_lfg_motion_read_tap", "dawn_lfg_motion_last_launch_count",
                      "dawn_lfg_motion_workspace_bytes", "dawn_lfg_motion_test_kernel"]
LFG_EXPORTS += LFG_MOTION_EXPORTS                       # both handles are declared in include/dawn_lfg.h
MISC_EXPORTS = ["dawn_conv3x3_s2_relu"]
PBNET_EXPORTS = ["dawn_pbnet_create", "dawn_pbnet_destroy", "dawn_pbnet_set_param", "dawn_pbnet_commit_params",
                 "dawn_pbnet_generate", "dawn_pbnet_last_launch_count", "dawn_pbnet_workspace_bytes", "dawn_pbnet_test_attention",
                 "dawn_pbnet_test_kernel"]
HUBERT_EXPORTS = ["dawn_hubert_create", "dawn_hubert_destroy", "dawn_hubert_set_param", "dawn_hubert_commit_params",
                  "dawn_hubert_forward", "dawn_hubert_output_length", "dawn_hubert_hidden", "dawn_hubert_last_launch_count", "dawn_hubert_workspace_bytes",
                  "dawn_hubert_test_kernel"]
VIDEO_EXPORTS = ["dawn_portrait_resize"]

PROF_CATS = ["conv3x3", "conv_other", "qkv_proj", "out_proj", "ca_gate", "gn_hcond", "attn_core", "sla_context",
             "gn_apply", "rowstats", "ca_rstd", "misc", "prep", "temporal_fused_l0", "conv3x3_l0", "comm_allreduce", "comm_halo"]
PROF_NCAT = 20


def check(rc, what):
    if rc != 0:
        raise DawnError(f"{what} failed (rc={rc}): {lib.dawn_last_error().decode()}")


def stream():
    """The current torch CUDA stream, as the library's `void* stream` argument."""
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """Device address of tensor t; None -> NULL."""
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def put_param(set_param, handle, name, t):
    """Hands tensor t to a handle's `*_set_param` entry under `name`, as fp32 host values in t's shape."""
    t = t.detach().to(device="cpu", dtype=torch.float32).contiguous()
    shape = (ctypes.c_int64 * max(t.dim(), 1))(*t.shape)
    check(set_param(handle, name.encode(), ctypes.c_void_p(t.data_ptr()), shape, t.dim()), f"{set_param.__name__}({name})")


class _Holder(nn.Module):
    """Container of parameters whose forward is never called."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter holder: the computation runs in the CUDA library")


class _Handle:
    """One native handle (entry points `<api>_*`, api "dawn_unet", "dawn_lfg", "dawn_lfg_motion", "dawn_pbnet" or
    "dawn_hubert") that holds a
    module's parameters.  It is created on the device of the module's inputs and created again after a device change, and the
    module's state_dict is uploaded and committed whenever `dirty`; `commits` counts the commits.  param_name(key) is the library's
    name of a state_dict entry, or None for an entry the handle does not take; extra(module) gives further {name: tensor} entries
    derived from the module.  `geom` is the geometry its user set last: create voids it, and so does a commit unless keeps_geom
    (the library re-applies its geometry on commit)."""

    def __init__(self, api, cfg, what, param_name=lambda key: key, extra=lambda module: {}, keeps_geom=False):
        self.api, self.cfg, self.what, self.param_name, self.extra, self.keeps_geom = api, cfg, what, param_name, extra, keeps_geom
        self.handle, self.device_index, self.dirty, self.geom, self.commits = None, None, True, None, 0

    def _entry(self, name):
        return getattr(lib, f"{self.api}_{name}")

    def _create(self):
        hd = ctypes.c_void_p()
        check(self._entry("create")(ctypes.byref(self.cfg), ctypes.byref(hd)), f"{self.api}_create")
        return hd

    def validate(self):
        """Create refuses what the library cannot run; it needs no GPU."""
        self._entry("destroy")(self._create())

    def destroy(self):
        if self.handle is not None:
            self._entry("destroy")(self.handle)
        self.handle, self.geom = None, None

    def ensure(self, module, device):
        """Readies the handle for a call on `device` with the parameters of `module`; returns the device index."""
        if device.type != "cuda":
            raise DawnError(f"{self.what} runs on CUDA (sm_90a) only; there is no CPU path")
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if self.handle is not None and self.device_index != idx:
            self.destroy()
            self.dirty = True
        with torch.cuda.device(idx):
            if self.handle is None:
                self.handle, self.device_index = self._create(), idx
            if self.dirty:
                for key, t in module.state_dict().items():
                    name = None if key.endswith("num_batches_tracked") else self.param_name(key)
                    if name is not None:
                        put_param(self._entry("set_param"), self.handle, name, t)
                for name, t in self.extra(module).items():
                    put_param(self._entry("set_param"), self.handle, name, t)
                check(self._entry("commit_params")(self.handle), f"{self.api}_commit_params")
                self.dirty, self.commits = False, self.commits + 1
                if not self.keeps_geom:
                    self.geom = None
        return idx

    def last_launch_count(self):
        return int(self._entry("last_launch_count")(self.handle)) if self.handle is not None else 0

    def workspace_bytes(self):
        return int(self._entry("workspace_bytes")(self.handle)) if self.handle is not None else 0


class _NativeModule(nn.Module):
    """Base of the modules whose parameters feed the native handles in `_handles`: load_state_dict and .to() / .cuda() mark every
    handle dirty, and the handles die with the module.  A class with a TRAIN_REFUSAL is inference only: it starts in eval mode and
    its train(True) raises with that message."""
    TRAIN_REFUSAL = None

    def _hold(self, *handles):
        self._handles = list(handles)
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.mark_dirty())
        if self.TRAIN_REFUSAL:
            self.eval()

    def mark_dirty(self):
        """Call after mutating parameters in place; load_state_dict / .to() / .cuda() do it automatically."""
        for h in self._handles:
            h.dirty = True

    def _apply(self, fn, *a, **k):
        for h in self.__dict__.get("_handles", ()):
            h.dirty = True
        return super()._apply(fn, *a, **k)

    def train(self, mode=True):
        if mode and self.TRAIN_REFUSAL:
            raise NotImplementedError(self.TRAIN_REFUSAL)
        return super().train(mode)

    def __del__(self):
        # plain dict access: nn.Module.__getattr__ may already be torn down at interpreter shutdown
        for h in self.__dict__.get("_handles", ()):
            try:
                h.destroy()
            except Exception:
                pass

    def last_launch_count(self):
        """Kernels the last call of the module's first handle enqueued."""
        return self._handles[0].last_launch_count()

    def workspace_bytes(self):
        """Device bytes of the workspace of the module's first handle."""
        return self._handles[0].workspace_bytes()
