"""Drop-in replacement for PBnet's `get_model` (PBnet/src/models/get_model.py:19-34) as unified_video_generator.py uses it to
make the pose and blink sequences: `get_model(params)` -> `CVAE`, strict `load_state_dict` of a reference checkpoint, `.eval()`,
`generate(init_pose, audio, durations, fact=1)["output"]`.

Only the decoder runs at inference (CAE.generate, modeltype/cae.py:112-172).  Its arithmetic runs in hand-written sm_90a CUDA
kernels behind include/dawn_pbnet.h: a banded attention that visits the +-band frames the reference's eval-mode bias leaves
unmasked (200 for transformerreemb5, 100 for transformerreemb6), so a minute of audio costs O(frames x band).  The encoder is a
parameter holder, so that checkpoints load unchanged; training is out of scope.  There is no PyTorch fallback.
"""
import math

import torch
from torch import nn

from . import _lib
from ._lib import DawnPbnetCfg, _Handle, _Holder, _NativeModule, check, lib, ptr, stream
from .unet import _Rotary, _rel_bias_table

MODELTYPES = ("cvae",)
ARCHINAMES = ("transformerreemb5", "transformerreemb6")
BANDS = {"transformerreemb5": 200, "transformerreemb6": 100}   # eval-mode masks of RelativePositionBias (reemb5:119-123, reemb6)
DIM_HEAD = 32                                                  # Attention / Attention_2 of transformerdecoder4.py:190-191


class _PositionalEncoding(_Holder):
    """PositionalEncoding (reemb5:61-78): never applied by the decoder, but its `pe` buffer is in the state_dict"""

    def __init__(self, d_model, max_len=20000):
        super().__init__()
        pe = torch.zeros(max_len, d_model)
        position = torch.arange(0, max_len, dtype=torch.float).unsqueeze(1)
        div_term = torch.exp(torch.arange(0, d_model, 2).float() * (-math.log(10000.0) / d_model))
        pe[:, 0::2] = torch.sin(position * div_term)
        pe[:, 1::2] = torch.cos(position * div_term)
        self.register_buffer('pe', pe.unsqueeze(0).transpose(0, 1))


class _RelativePositionBias(_Holder):
    def __init__(self, heads, num_buckets, max_distance):
        super().__init__()
        self.num_buckets, self.max_distance = num_buckets, max_distance
        self.relative_attention_bias = nn.Embedding(num_buckets, heads)


def _attention(dim, heads, rotary):                                # Attention (transformerdecoder4.py:24-39)
    m = _Holder()
    m.rotary_emb = rotary
    m.to_qkv = nn.Linear(dim, DIM_HEAD * heads * 3, bias=False)
    m.to_out = nn.Linear(DIM_HEAD * heads, dim, bias=False)
    return m


def _cross_attention(dim, heads, rotary):                          # Attention_2 (transformerdecoder4.py:102-119)
    m = _Holder()
    m.rotary_emb = rotary
    m.to_q = nn.Linear(dim, DIM_HEAD * heads, bias=False)
    m.to_k = nn.Linear(dim, DIM_HEAD * heads, bias=False)
    m.to_v = nn.Linear(dim, DIM_HEAD * heads, bias=False)
    m.to_out = nn.Linear(DIM_HEAD * heads, dim, bias=False)
    return m


def _decoder_layer(d_model, heads, d_ff, rotary):                  # DecoderLayer (transformerdecoder4.py:186-199)
    m = _Holder()
    m.self_attn = _attention(d_model, heads, rotary)
    m.multihead_attn = _cross_attention(d_model, heads, rotary)
    m.ffn = _Holder()
    m.ffn.linear1 = nn.Linear(d_model, d_ff)
    m.ffn.linear2 = nn.Linear(d_ff, d_model)
    m.layer_norm1 = nn.LayerNorm(d_model)
    m.layer_norm2 = nn.LayerNorm(d_model)
    m.layer_norm3 = nn.LayerNorm(d_model)
    return m


class Encoder(_Holder):
    """Encoder_TRANSFORMERREEMB5 / 6 (reemb5:146-196): its parameters only.  It runs in training alone, which is out of scope."""

    def __init__(self, modeltype, num_frames, audio_dim=1024, pos_dim=6, eye_dim=2, pose_latent_dim=64, audio_latent_dim=256,
                 ff_size=1024, num_layers=4, num_heads=4, dropout=0.1, ablation=None, activation="gelu", **kargs):
        super().__init__()
        latent = audio_latent_dim + pose_latent_dim * 2
        self.mu_layer = nn.Linear(latent, audio_latent_dim)
        self.sigma_layer = nn.Linear(latent, audio_latent_dim)
        self.poseEmbedding = nn.Linear(pos_dim + eye_dim, pose_latent_dim)
        self.firstposeEmbedding = nn.Linear(pos_dim + eye_dim, pose_latent_dim)
        self.audioEmbedding = nn.Linear(audio_dim, audio_latent_dim)
        self.sequence_pos_encoder = _PositionalEncoding(latent)
        layer = nn.TransformerEncoderLayer(d_model=latent, nhead=num_heads, dim_feedforward=ff_size, dropout=dropout,
                                           activation=activation)
        self.seqTransEncoder = nn.TransformerEncoder(layer, num_layers=num_layers, enable_nested_tensor=False)

    def forward(self, batch):
        raise NotImplementedError("the PBnet encoder runs in training only, which is out of scope: use CVAE.generate")


class Decoder(_NativeModule):
    """Decoder_TRANSFORMERREEMB5 / 6 (reemb5:234-378): same keywords and state_dict; forward(batch) runs on the device."""
    TRAIN_REFUSAL = "the PBnet decoder here is inference-only: training (dropout, the training-mode bias) is out of scope"

    def __init__(self, modeltype, num_frames, audio_dim=1024, pos_dim=6, eye_dim=2, pose_latent_dim=64, audio_latent_dim=256,
                 ff_size=1024, num_layers=4, num_heads=4, dropout=0.1, activation="gelu", ablation=None, num_buckets=32,
                 max_distance=32, band=200, latent_dim=None, **kargs):
        super().__init__()
        self.pos_dim, self.eye_dim = pos_dim, eye_dim
        self.band, self.num_buckets, self.max_distance = band, num_buckets, max_distance
        self.firstposeEmbedding = nn.Linear(pos_dim + eye_dim, pose_latent_dim)
        self.audioEmbedding = nn.Linear(audio_dim, audio_latent_dim)
        self.ztimelinear = nn.Linear(audio_latent_dim * 2 + pose_latent_dim, pose_latent_dim)
        self.init_proj = nn.Linear(pose_latent_dim, pose_latent_dim)
        self.sequence_pos_encoder = _PositionalEncoding(pose_latent_dim)
        self.time_rel_pos_bias_tgt = _RelativePositionBias(num_heads, num_buckets, max_distance)
        self.time_rel_pos_bias_mem = _RelativePositionBias(num_heads, num_buckets, max_distance)
        pre = _Holder()                                                # Residual(PreNorm(LayerNorm gamma, Attention))
        pre.fn = _attention(pose_latent_dim, num_heads, _Rotary(min(32, num_heads)))
        pre.norm = _Holder()
        pre.norm.gamma = nn.Parameter(torch.ones(1, 1, pose_latent_dim))
        self.init_temporal_attn = _Holder()
        self.init_temporal_attn.fn = pre
        shared = _Rotary(min(32, num_heads))                           # one RotaryEmbedding for every layer (decoder4:213)
        self.seqTransDecoder = _Holder()
        self.seqTransDecoder.decoder_layers = nn.ModuleList(
            [_decoder_layer(pose_latent_dim, num_heads, ff_size, shared) for _ in range(num_layers)])
        self.finallayer = nn.Linear(pose_latent_dim, pos_dim + eye_dim)
        cfg = DawnPbnetCfg(band=band, pose_dim=pos_dim + eye_dim, audio_dim=audio_dim,
                           latent_dim=audio_latent_dim if latent_dim is None else latent_dim, audio_latent_dim=audio_latent_dim,
                           pose_latent_dim=pose_latent_dim, ff_size=ff_size, num_layers=num_layers, num_heads=num_heads)
        self._pbnet = _Handle("dawn_pbnet", cfg, "the PBnet decoder", self._param_name, Decoder._bias_tables)
        try:
            self._pbnet.validate()
        except _lib.DawnError as e:
            raise ValueError(f"unsupported PBnet configuration: {e}") from None
        self._hold(self._pbnet)

    @staticmethod
    def _param_name(key):
        """the library takes the decoder's parameters; the positional encoding is unused and the bias tables go as aux.*"""
        return None if key.startswith(("sequence_pos_encoder.", "time_rel_pos_bias_")) else key

    def _bias_tables(self):
        """RelativePositionBias values for j - i in [-band, band], with the reference's bucket function (torch CPU ops)"""
        tab = lambda m: _rel_bias_table(m.relative_attention_bias.weight, self.band, self.num_buckets, self.max_distance)  # noqa: E731
        return {"aux.bias_tgt": tab(self.time_rel_pos_bias_tgt), "aux.bias_mem": tab(self.time_rel_pos_bias_mem)}

    @torch.no_grad()
    def forward(self, batch):
        """reemb5:311-378: batch x (bs, >= 1, pose_dim), z (F, bs, latent_dim), y (bs, F, audio_dim), mask (bs, F) -> output"""
        x, z, y, mask = batch["x"], batch["z"], batch["y"], batch["mask"]
        bs, F = mask.shape
        dev = y.device
        idx = self._pbnet.ensure(self, dev)
        audio = y.contiguous().float()
        zz = z.to(dev).contiguous().float()
        first = x[:, 0, :].to(dev).contiguous().float()
        m8 = mask.to(device=dev, dtype=torch.uint8).contiguous()
        if audio.shape[:2] != (bs, F) or zz.shape[:2] != (F, bs):
            raise ValueError(f"shapes disagree: y {tuple(audio.shape)}, z {tuple(zz.shape)}, mask {tuple(mask.shape)}")
        out = torch.empty((bs, F, self.pos_dim + self.eye_dim), device=dev, dtype=torch.float32)
        with torch.cuda.device(idx):
            check(lib.dawn_pbnet_generate(self._pbnet.handle, ptr(audio), ptr(zz), ptr(first), ptr(m8), bs, F, ptr(out), stream()),
                  "dawn_pbnet_generate")
        batch["output"] = out
        return batch


class CVAE(nn.Module):
    """CAE / CVAE (modeltype/cae.py, cvae.py) for inference: `generate` runs the decoder on the device."""

    def __init__(self, encoder, decoder, device, lambdas, latent_dim, archiname="transformerreemb5", **kwargs):
        super().__init__()
        self.encoder = encoder
        self.decoder = decoder
        self.lambdas = lambdas
        self.latent_dim = latent_dim
        self.device = device
        self.losses = list(self.lambdas) + ["mixed"]
        self.archiname = archiname
        self.eval()

    def train(self, mode=True):
        if mode:
            raise NotImplementedError("PBnet training is out of scope: this CVAE is inference-only")
        return super().train(False)

    def forward(self, batch):
        raise NotImplementedError("CVAE.forward (encoder + reparameterisation) is training-only and out of scope; use generate")

    def compute_loss(self, batch, epoch=0):
        raise NotImplementedError("PBnet training losses are out of scope")

    def return_latent(self, batch, seed=None):
        raise NotImplementedError("CVAE.return_latent runs the encoder, which is training-only and out of scope")

    @staticmethod
    def lengths_to_mask(lengths):
        max_len = max(lengths)
        if isinstance(max_len, torch.Tensor):
            max_len = max_len.item()
        index = torch.arange(max_len, device=lengths.device).expand(len(lengths), max_len)
        return index < lengths.unsqueeze(1)

    def _run_device(self):
        dev = self.decoder.finallayer.weight.device
        if dev.type != "cuda":
            raise _lib.DawnError("the PBnet decoder runs on CUDA (sm_90a) only; there is no CPU path")
        return dev

    @torch.no_grad()
    def generate(self, pose, audio, durations, noise_same_action="random", noise_diff_action="random", fact=1, z=None):
        """cae.py:112-172.  pose (bs, >= 1, pos_dim + eye_dim): frame 0 is the first pose; audio (bs, F, audio_dim); durations (bs,)
        with max(durations) == F.  z (F, bs, latent_dim) is drawn with torch.randn on the device when None, as the reference does.
        Returns the reference's batch dict: x, z, y, mask, lengths, output (bs, F, pos_dim + eye_dim; zero past each length), and
        out_pose / out_eye for transformerreemb5."""
        bs, F = len(audio), audio.shape[1]
        if durations.dim() != 1 or durations.shape[0] != bs:
            raise ValueError(f"durations must be 1-D with one length per clip ({bs}), got shape {tuple(durations.shape)}")
        if int(durations.max()) != F or int(durations.min()) < 1:
            raise ValueError(f"max(durations) must equal audio.shape[1] = {F} and every duration be >= 1, got {durations.tolist()}")
        dev = self._run_device()
        x = pose.to(dev)
        y = audio.to(dev)
        lengths = durations.to(dev)
        mask = self.lengths_to_mask(lengths)
        if z is None:
            z = torch.randn(F, bs, self.latent_dim, device=dev)
        elif tuple(z.shape) != (F, bs, self.latent_dim):
            raise ValueError(f"z must be (F, bs, latent_dim) = {(F, bs, self.latent_dim)}, got {tuple(z.shape)}")
        batch = {"x": x, "z": fact * z.to(dev), "y": y, "mask": mask, "lengths": lengths}
        batch = self.decoder(batch)
        if self.archiname == "transformerreemb5":
            batch["out_pose"] = batch["output"][:, :, :6]
            batch["out_eye"] = batch["output"][:, :, 6:]
        return batch

    def last_launch_count(self):
        """kernels the last generate enqueued"""
        return self.decoder.last_launch_count()

    def workspace_bytes(self):
        return self.decoder.workspace_bytes()


def get_model(parameters):
    """get_model.py:19-34 for the architectures DAWN's inference uses.  parameters: the opt.yaml contents plus device, audio_dim,
    pos_dim and eye_dim (unified_video_generator.py:80-92)."""
    modeltype, archiname = parameters["modeltype"], parameters["archiname"]
    if modeltype not in MODELTYPES:
        raise ValueError(f"modeltype {modeltype!r} is not supported: supported are {list(MODELTYPES)}")
    if archiname not in ARCHINAMES:
        raise ValueError(f"archiname {archiname!r} is not supported: supported are {list(ARCHINAMES)} "
                         "(transformerreemb7 / 8 are listed in the reference's ARCHINAMES but have no source)")
    p = dict(parameters)
    if archiname == "transformerreemb6":
        p["eye_dim"] = 0                                               # reemb6 forces eye_dim = 0 in both halves
    encoder = Encoder(**p)
    decoder = Decoder(band=BANDS[archiname], **p)
    return CVAE(encoder, decoder, **p).to(parameters["device"])
