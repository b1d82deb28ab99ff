"""Drop-in replacement for transformers' `HubertModel` as DAWN's unified_video_generator.py uses it (line 71 and
`_get_hubert_from_16k_speech`, lines 433-501): `HubertModel.from_pretrained(dir)`, `.eval()`, `model(input_values).last_hidden_state`.

The model is the eval forward of the stable-layer-norm HuBERT (`feat_extract_norm="layer"`, `do_stable_layer_norm=True`: the
hubert-large-ls960-ft configuration), restated from transformers' documented semantics.  Its arithmetic runs in hand-written
sm_90a CUDA behind include/dawn_hubert.h; there is no PyTorch fallback and no dependency on transformers.

`hubert_features(model, speech_16k)` is the generator's whole audio pipeline (lines 229-242 and 450-501): the Wav2Vec2
normalisation, the 20 s segments, the length fix-up and the linear interpolation to 25 fps, in one call.
"""
import ctypes
import json
import os
from types import SimpleNamespace

import numpy as np
import torch
from torch import nn

from . import _lib
from ._lib import DawnHubertCfg, _Handle, _Holder, _NativeModule, check, lib, ptr, stream

HEAD_DIM = 64
MAX_CONV = 8                          # DAWN_HUBERT_MAX_CONV
# HubertConfig's defaults for the fields the model reads
CONFIG_DEFAULTS = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072, hidden_act="gelu",
                       layer_norm_eps=1e-5, feat_extract_norm="group", feat_extract_activation="gelu", conv_dim=(512,) * 7,
                       conv_stride=(5, 2, 2, 2, 2, 2, 2), conv_kernel=(10, 3, 3, 3, 3, 2, 2), conv_bias=False,
                       num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=16, conv_pos_batch_norm=False,
                       do_stable_layer_norm=False, feat_proj_layer_norm=True, mask_time_prob=0.05, mask_feature_prob=0.0,
                       adapter_attn_dim=None)
_POS = "encoder.pos_conv_embed.conv."
# the positional conv's weight norm: the hub checkpoints' spelling -> torch.nn.utils.parametrizations' (current transformers)
WEIGHT_NORM_KEYS = {_POS + "weight_g": _POS + "parametrizations.weight.original0",
                    _POS + "weight_v": _POS + "parametrizations.weight.original1"}

# generator audio pipeline (unified_video_generator.py:460-465): HuBERT's receptive field and hop, 1000-frame segments
KERNEL, STRIDE = 400, 320
CLIP = STRIDE * 1000                  # segment stride, samples
SEGMENT = CLIP - STRIDE + KERNEL      # segment length: 320 080 samples = 1000 frames
# full segments per forward: bounds the handle's workspace at any audio length (hubert-large: about 0.9 GB, most of it the feature
# extractor's 4 x 64 015 x 512 rows), while 4 000 encoder rows per call already fill the GEMMs
SEGMENTS_PER_CALL = 4
SAMPLE_RATE, FPS = 16000, 25


def load_config(config):
    """A transformers HubertConfig, a dict, or the path of a config.json (or of the directory holding it) -> SimpleNamespace
    with HubertConfig's defaults for absent fields."""
    if isinstance(config, (str, os.PathLike)):
        path = os.path.join(config, "config.json") if os.path.isdir(config) else config
        with open(path) as fh:
            config = json.load(fh)
    elif not isinstance(config, dict):
        config = config.to_dict() if hasattr(config, "to_dict") else vars(config)
    cfg = dict(CONFIG_DEFAULTS)
    cfg.update({k: v for k, v in config.items() if k in CONFIG_DEFAULTS})
    return SimpleNamespace(**cfg)


def _check_config(c):
    def need(ok, what):
        if not ok:
            raise ValueError(f"unsupported HuBERT configuration: {what}")
    need(c.feat_extract_norm == "layer", f'feat_extract_norm must be "layer" (got {c.feat_extract_norm!r})')
    need(c.do_stable_layer_norm, "do_stable_layer_norm must be True (the pre-LayerNorm encoder)")
    need(c.hidden_act == "gelu" and c.feat_extract_activation == "gelu", "hidden_act and feat_extract_activation must be gelu")
    need(c.num_attention_heads >= 1 and c.hidden_size == HEAD_DIM * c.num_attention_heads,
         f"heads must be {HEAD_DIM} wide (hidden_size {c.hidden_size}, {c.num_attention_heads} heads)")
    need(all(w % 64 == 0 and w > 0 for w in (c.hidden_size, c.intermediate_size, *c.conv_dim)),
         "hidden_size, intermediate_size and conv_dim must be multiples of 64")
    need(len(c.conv_dim) == len(c.conv_kernel) == len(c.conv_stride), "conv_dim, conv_kernel and conv_stride differ in length")
    need(not c.conv_pos_batch_norm, "conv_pos_batch_norm is not supported (the positional conv is weight-normed)")
    need(c.feat_proj_layer_norm, "feat_proj_layer_norm must be True")
    need(c.adapter_attn_dim is None, "attention adapters are not supported")


def _cfg_struct(c):
    if len(c.conv_dim) > MAX_CONV:
        raise ValueError(f"unsupported HuBERT configuration: at most {MAX_CONV} feature-extractor conv layers")
    ints = lambda v: (ctypes.c_int * MAX_CONV)(*v)  # noqa: E731
    return DawnHubertCfg(hidden_size=c.hidden_size, num_layers=c.num_hidden_layers, num_heads=c.num_attention_heads,
                         intermediate_size=c.intermediate_size, num_conv=len(c.conv_dim), conv_dim=ints(c.conv_dim),
                         conv_kernel=ints(c.conv_kernel), conv_stride=ints(c.conv_stride), conv_bias=int(bool(c.conv_bias)),
                         pos_kernel=c.num_conv_pos_embeddings, pos_groups=c.num_conv_pos_embedding_groups,
                         layer_norm_eps=c.layer_norm_eps)


def feat_extract_output_length(config, length):
    """Frames the feature extractor makes of `length` samples: floor((L - k) / s) + 1 per conv layer"""
    c = config if isinstance(config, SimpleNamespace) else load_config(config)
    for k, s in zip(c.conv_kernel, c.conv_stride):
        length = (length - k) // s + 1
    return length


def _layer(c):
    m = _Holder()
    m.attention = _Holder()
    for name in ("k_proj", "v_proj", "q_proj", "out_proj"):             # transformers' order
        setattr(m.attention, name, nn.Linear(c.hidden_size, c.hidden_size))
    m.layer_norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
    m.feed_forward = _Holder()
    m.feed_forward.intermediate_dense = nn.Linear(c.hidden_size, c.intermediate_size)
    m.feed_forward.output_dense = nn.Linear(c.intermediate_size, c.hidden_size)
    m.final_layer_norm = nn.LayerNorm(c.hidden_size, eps=c.layer_norm_eps)
    return m


class HubertModel(_NativeModule):
    """transformers' HubertModel (stable-layer-norm variant), eval forward on the device.  Same state_dict names and shapes, so a
    strict load_state_dict of a transformers checkpoint works; the positional conv's weight norm loads from either spelling."""
    TRAIN_REFUSAL = "the HuBERT encoder here is inference-only: training (dropout, SpecAugment, LayerDrop) is out of scope"

    def __init__(self, config):
        super().__init__()
        c = load_config(config)
        _check_config(c)
        self.config = c
        D = c.hidden_size
        with torch.device("meta"):
            if c.mask_time_prob > 0.0 or c.mask_feature_prob > 0.0:
                self.masked_spec_embed = nn.Parameter(torch.empty(D))     # SpecAugment: unused in eval
            self.feature_extractor = _Holder()
            layers = []
            for i, (co, k, s) in enumerate(zip(c.conv_dim, c.conv_kernel, c.conv_stride)):
                m = _Holder()
                m.conv = nn.Conv1d(1 if i == 0 else c.conv_dim[i - 1], co, k, stride=s, bias=bool(c.conv_bias))
                m.layer_norm = nn.LayerNorm(co)
                layers.append(m)
            self.feature_extractor.conv_layers = nn.ModuleList(layers)
            self.feature_projection = _Holder()
            self.feature_projection.layer_norm = nn.LayerNorm(c.conv_dim[-1], eps=c.layer_norm_eps)
            self.feature_projection.projection = nn.Linear(c.conv_dim[-1], D)
            self.encoder = _Holder()
            pos = self.encoder.pos_conv_embed = _Holder()
            pos.conv = _Holder()
            pos.conv.bias = nn.Parameter(torch.empty(D))
            pos.conv.parametrizations = _Holder()
            pos.conv.parametrizations.weight = _Holder()
            k, G = c.num_conv_pos_embeddings, c.num_conv_pos_embedding_groups
            pos.conv.parametrizations.weight.original0 = nn.Parameter(torch.empty(1, 1, k))
            pos.conv.parametrizations.weight.original1 = nn.Parameter(torch.empty(D, D // G, k))
            self.encoder.layer_norm = nn.LayerNorm(D, eps=c.layer_norm_eps)
            self.encoder.layers = nn.ModuleList([_layer(c) for _ in range(c.num_hidden_layers)])
        # placeholder values until a checkpoint loads: LayerNorms identity, weight-norm gains 1, everything else 0
        self.to_empty(device="cpu")
        with torch.no_grad():
            for name, p in self.named_parameters():
                p.fill_(1.0 if name.endswith(("layer_norm.weight", "original0")) else 0.0)
        self._hubert = _Handle("dawn_hubert", _cfg_struct(c), "the HuBERT encoder", self._param_name)
        try:
            self._hubert.validate()
        except _lib.DawnError as e:
            raise ValueError(f"unsupported HuBERT configuration: {e}") from None
        self.register_load_state_dict_pre_hook(HubertModel._weight_norm_spelling)
        self._hold(self._hubert)

    @staticmethod
    def _weight_norm_spelling(module, state_dict, prefix, *args):
        for old, new in WEIGHT_NORM_KEYS.items():
            if prefix + old in state_dict:
                state_dict[prefix + new] = state_dict.pop(prefix + old)

    @staticmethod
    def _param_name(key):
        if key == "masked_spec_embed":
            return None
        for old, new in WEIGHT_NORM_KEYS.items():
            if key == new:
                return old
        return key

    @classmethod
    def from_pretrained(cls, path, **kwargs):
        """A checkpoint directory holding config.json and pytorch_model.bin or model.safetensors; a HubertForCTC checkpoint
        (hubert.* entries and an lm_head) loads its HubertModel part."""
        if kwargs:
            raise TypeError(f"from_pretrained takes a local checkpoint directory only (got {sorted(kwargs)})")
        model = cls(os.path.join(path, "config.json"))
        st_path, bin_path = os.path.join(path, "model.safetensors"), os.path.join(path, "pytorch_model.bin")
        if os.path.exists(st_path):
            from safetensors.torch import load_file
            sd = load_file(st_path)
        elif os.path.exists(bin_path):
            sd = torch.load(bin_path, map_location="cpu", weights_only=True)
        else:
            raise FileNotFoundError(f"{path} holds neither model.safetensors nor pytorch_model.bin")
        model.load_state_dict(convert_state_dict(sd), strict=True)
        return model.eval()

    def output_length(self, length):
        return feat_extract_output_length(self.config, length)

    @torch.no_grad()
    def forward(self, input_values, attention_mask=None, mask_time_indices=None, output_attentions=None, output_hidden_states=None,
                return_dict=None):
        """input_values (B, L) fp32 on a CUDA device -> object with .last_hidden_state (B, T, hidden_size)"""
        for name, v in (("attention_mask", attention_mask), ("mask_time_indices", mask_time_indices),
                        ("output_attentions", output_attentions), ("output_hidden_states", output_hidden_states)):
            if v is not None and v is not False:
                raise NotImplementedError(f"HubertModel here does not take {name}: it runs unpadded input in eval mode only")
        if return_dict is False:
            raise NotImplementedError("HubertModel here returns its output object only (return_dict=False is not supported)")
        return HubertOutput(self._run(input_values, None))

    @torch.no_grad()
    def hidden_state(self, input_values, layers):
        """The encoder's hidden state after its first `layers` layers (0: after the positional conv), before the final LayerNorm"""
        if not 0 <= layers <= self.config.num_hidden_layers:
            raise ValueError(f"layers must be 0 to {self.config.num_hidden_layers}")
        return self._run(input_values, layers)

    def _run(self, x, layers):
        if x.dim() != 2 or x.dtype != torch.float32:
            raise ValueError(f"input_values must be (batch, samples) float32, got {tuple(x.shape)} {x.dtype}")
        B, L = x.shape
        T = self.output_length(L)
        if T < 1:
            raise ValueError(f"{L} samples are fewer than the feature extractor's receptive field")
        idx = self._hubert.ensure(self, x.device)
        x = x.contiguous()
        with torch.cuda.device(idx):
            out = torch.empty(B, T, self.config.hidden_size, device=x.device, dtype=torch.float32)
            if layers is None:
                check(lib.dawn_hubert_forward(self._hubert.handle, ptr(x), B, L, ptr(out), stream()), "dawn_hubert_forward")
            else:
                check(lib.dawn_hubert_hidden(self._hubert.handle, ptr(x), B, L, layers, ptr(out), stream()), "dawn_hubert_hidden")
        return out


class HubertOutput(SimpleNamespace):
    """The forward's result: .last_hidden_state, also as item 0 (transformers' BaseModelOutput order)"""

    def __init__(self, last_hidden_state):
        super().__init__(last_hidden_state=last_hidden_state)

    def __getitem__(self, i):
        return (self.last_hidden_state,)[i]


def convert_state_dict(sd):
    """A HubertModel or HubertForCTC state_dict -> this HubertModel's: `hubert.` stripped, lm_head.* dropped, the weight norm in
    either spelling (load_state_dict renames it)."""
    if any(k.startswith("hubert.") for k in sd):
        sd = {k[len("hubert."):]: v for k, v in sd.items() if k.startswith("hubert.")}
    return {k: v for k, v in sd.items() if not k.startswith("lm_head.")}


# ------------------------------------------------------------------------------------------------ the generator's audio pipeline
def normalize(speech):
    """Wav2Vec2FeatureExtractor's zero-mean / unit-variance normalisation of one clip, in numpy float32 as it computes it (a
    (samples, channels) array keeps channel 0, as unified_video_generator.py:451-452 does)"""
    x = np.asarray(speech)
    if x.ndim == 2:
        x = x[:, 0]
    x = x.astype(np.float32)
    return (x - x.mean()) / np.sqrt(x.var() + 1e-7)


def segment_plan(n):
    """(start, end) sample ranges the generator runs through HuBERT for a clip of n samples: segments of SEGMENT samples every
    CLIP samples, then the tail from the last multiple of CLIP if it holds at least KERNEL samples"""
    num_iter = n // CLIP
    plan = [(CLIP * i, min(CLIP * i + SEGMENT, n)) for i in range(num_iter)]
    if n - CLIP * num_iter >= KERNEL:
        plan.append((CLIP * num_iter, n))
    return plan


def segment_batches(plan, per_call=None):
    """The forwards that run `plan`, in order: runs of up to per_call (default SEGMENTS_PER_CALL) full segments as one batch
    each, then each shorter range on its own"""
    per_call = per_call or SEGMENTS_PER_CALL
    batches = []
    for seg in plan:
        full = seg[1] - seg[0] == SEGMENT
        if full and batches and len(batches[-1]) < per_call and batches[-1][0][1] - batches[-1][0][0] == SEGMENT:
            batches[-1].append(seg)
        else:
            batches.append([seg])
    return batches


def interp_weights(T, num_frames):
    """scipy.interpolate.interp1d(arange(T), y, kind="linear")(linspace(0, T - 1, num_frames)) as indices and fp64 weights:
    y_new = w_hi y[hi] + w_lo y[lo]"""
    x = np.arange(T)
    x_new = np.linspace(0, T - 1, num_frames)
    hi = np.searchsorted(x, x_new).clip(1, T - 1).astype(int)
    lo = hi - 1
    x_lo, x_hi = x[lo], x[hi]
    return lo, hi, (x_new - x_lo) / (x_hi - x_lo), (x_hi - x_new) / (x_hi - x_lo)


def interpolate(hidden, num_frames):
    """(T, C) fp32 -> (num_frames, C) fp32, linear interpolation evaluated in fp64 exactly as interp1d does, then rounded"""
    T = hidden.shape[0]
    if T < 2:
        raise ValueError("linear interpolation needs at least 2 HuBERT frames (more than 0.045 s of audio)")
    lo, hi, w_hi, w_lo = interp_weights(T, num_frames)
    dev = hidden.device
    y = hidden.double()
    lo, hi = torch.from_numpy(lo).to(dev), torch.from_numpy(hi).to(dev)
    w_hi, w_lo = torch.from_numpy(w_hi).to(dev)[:, None], torch.from_numpy(w_lo).to(dev)[:, None]
    return (w_hi * y[hi] + w_lo * y[lo]).float()


@torch.no_grad()
def hubert_features(model, speech_16k, num_frames=None):
    """unified_video_generator.py:229-242 and 450-501 in one call: 16 kHz speech (numpy or tensor, (samples,) or (samples,
    channels)) -> (num_frames, hidden_size) fp32 on the model's device, num_frames = int(samples / 16000 * 25) by default.
    Full segments run SEGMENTS_PER_CALL to a batch, so device memory stays bounded for any length."""
    speech = speech_16k.detach().cpu().numpy() if torch.is_tensor(speech_16k) else np.asarray(speech_16k)
    n = speech.shape[0]
    if num_frames is None:
        num_frames = int((n / SAMPLE_RATE) * FPS)
    x = normalize(speech)
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        dev = torch.device("cuda", torch.cuda.current_device())
    parts = []
    for batch in segment_batches(segment_plan(n)):
        xb = torch.from_numpy(np.stack([x[a:b] for a, b in batch])).to(dev)
        parts += list(model(xb).last_hidden_state)
    if not parts:
        raise ValueError(f"{n} samples are fewer than HuBERT's receptive field of {KERNEL}")
    ret = torch.cat(parts, 0)
    expected = (n - (KERNEL - STRIDE)) // STRIDE
    if abs(ret.shape[0] - expected) > 1:
        raise RuntimeError(f"HuBERT made {ret.shape[0]} frames of {n} samples, expected {expected}")
    if ret.shape[0] < expected:
        ret = torch.nn.functional.pad(ret, (0, 0, 0, expected - ret.shape[0]))
    else:
        ret = ret[:expected]
    return interpolate(ret, num_frames)
