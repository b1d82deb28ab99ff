"""Drop-in replacement for the decode path of the reference's LFG `Generator` (LFG/modules/generator.py:20-171):
`compute_fea` (source-image features for the diffusion UNet) and `forward_with_flow` (frames from flow + occlusion maps).

Same constructor keywords and the same state_dict keys/shapes for everything the decode path reads
(first / down_blocks / up_blocks / bottleneck / final, incl. the BatchNorm running statistics), so
`generator.load_state_dict(checkpoint['generator'])` (FlowDiffusion.__init__, FD:120) works: the checkpoint's
`pixelwise_flow_predictor.*` entries — used by `forward` during LFG training only — are dropped on load.
The reference decodes frame by frame with batch 1 in a Python loop (FD:375-383); here the source encoder runs once per
clip and all frames are decoded as one batch by hand-written sm_90a CUDA kernels behind include/dawn_lfg.h.
The sub-modules only HOLD parameters; there is no PyTorch fallback.
"""
import ctypes

import torch
from torch import nn

from . import _lib
from ._lib import DawnLfgCfg, check, lib


class _Holder(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter holder: the computation runs in the CUDA library")


def _conv_bn(ci, co, k):                                   # SameBlock2d / DownBlock2d / UpBlock2d (util.py:95-150)
    m = _Holder()
    m.conv = nn.Conv2d(ci, co, kernel_size=k, padding=k // 2)
    m.norm = nn.BatchNorm2d(co, affine=True)
    return m


def _res_block(c):                                          # ResBlock2d (util.py:70-93): same registration order as the reference
    m = _Holder()
    m.conv1 = nn.Conv2d(c, c, kernel_size=3, padding=1)
    m.conv2 = nn.Conv2d(c, c, kernel_size=3, padding=1)
    m.norm1 = nn.BatchNorm2d(c, affine=True)
    m.norm2 = nn.BatchNorm2d(c, affine=True)
    return m


class Generator(nn.Module):
    IGNORED_PREFIX = "pixelwise_flow_predictor."

    def __init__(self, num_channels, num_regions, block_expansion, max_features, num_down_blocks, num_bottleneck_blocks,
                 pixelwise_flow_predictor_params=None, skips=False, revert_axis_swap=True):
        super().__init__()
        self.first = _conv_bn(num_channels, block_expansion, 7)                                   # generator.py:36
        self.down_blocks = nn.ModuleList([
            _conv_bn(min(max_features, block_expansion * 2 ** i), min(max_features, block_expansion * 2 ** (i + 1)), 3)
            for i in range(num_down_blocks)])                                                      # :38-44
        self.up_blocks = nn.ModuleList([
            _conv_bn(min(max_features, block_expansion * 2 ** (num_down_blocks - i)),
                     min(max_features, block_expansion * 2 ** (num_down_blocks - i - 1)), 3)
            for i in range(num_down_blocks)])                                                      # :46-52
        self.bottleneck = nn.Sequential()
        cb = min(max_features, block_expansion * 2 ** num_down_blocks)
        for i in range(num_bottleneck_blocks):
            self.bottleneck.add_module('r' + str(i), _res_block(cb))                               # :54-57
        self.final = nn.Conv2d(block_expansion, num_channels, kernel_size=7, padding=3)            # :59
        self.num_channels, self.skips = num_channels, skips
        self.bottleneck_channels, self.num_down_blocks = cb, num_down_blocks
        cfg = DawnLfgCfg()
        cfg.num_channels, cfg.block_expansion, cfg.max_features = num_channels, block_expansion, max_features
        cfg.num_down_blocks, cfg.num_bottleneck_blocks, cfg.skips = num_down_blocks, num_bottleneck_blocks, int(bool(skips))
        self._cfg = cfg
        self._handle, self._dirty, self._geom, self._device_index, self._src_key = None, True, None, None, None
        self._register_load_state_dict_pre_hook(self._drop_training_only_keys)
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.mark_dirty())
        self.eval()

    # the reference checkpoint's `generator` entry also holds the training-time flow predictor (generator.py:29-34)
    @classmethod
    def _drop_training_only_keys(cls, state_dict, prefix, *args):
        for k in [k for k in state_dict if k.startswith(prefix + cls.IGNORED_PREFIX)]:
            del state_dict[k]

    def mark_dirty(self):
        self._dirty = True

    def _apply(self, fn, *a, **k):
        self._dirty = True
        return super()._apply(fn, *a, **k)

    def train(self, mode=True):
        if mode:
            raise NotImplementedError("this LFG decoder is inference-only (eval-mode BatchNorm, FD:121)")
        return super().train(False)

    def __del__(self):
        h = self.__dict__.get("_handle")
        self.__dict__["_handle"] = None
        if h is not None:
            try:
                lib.dawn_lfg_destroy(h)
            except Exception:
                pass

    @staticmethod
    def _stream():
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def _ensure(self, device, frames, H, W, fh, fw):
        if device.type != "cuda":
            raise _lib.DawnError("the LFG decoder runs on CUDA (sm_90a) only; there is no CPU path")
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if self._handle is not None and self._device_index != idx:
            lib.dawn_lfg_destroy(self._handle)
            self._handle, self._dirty, self._geom = None, True, None
        with torch.cuda.device(idx):
            if self._handle is None:
                hd = ctypes.c_void_p()
                check(lib.dawn_lfg_create(ctypes.byref(self._cfg), ctypes.byref(hd)), "dawn_lfg_create")
                self._handle, self._device_index = hd, idx
            if self._dirty:
                for name, t in self.state_dict().items():
                    if name.endswith("num_batches_tracked"):
                        continue
                    t = t.detach().to(device="cpu", dtype=torch.float32).contiguous()
                    shape = (ctypes.c_int64 * max(t.dim(), 1))(*t.shape)
                    check(lib.dawn_lfg_set_param(self._handle, name.encode(), ctypes.c_void_p(t.data_ptr()), shape, t.dim()),
                          f"dawn_lfg_set_param({name})")
                check(lib.dawn_lfg_commit_params(self._handle), "dawn_lfg_commit_params")
                self._dirty, self._geom, self._src_key = False, None, None
            if self._geom != (frames, H, W, fh, fw):
                check(lib.dawn_lfg_set_geometry(self._handle, frames, H, W, fh, fw), "dawn_lfg_set_geometry")
                self._geom, self._src_key = (frames, H, W, fh, fw), None

    def _set_source(self, source_image):
        src = source_image.reshape(-1, *source_image.shape[-3:])
        if src.shape[0] != 1:
            raise ValueError("one source image per call (the reference decodes with batch 1, FD:375-383)")
        src = src[0].contiguous().float()
        with torch.cuda.device(src.device):
            check(lib.dawn_lfg_set_source(self._handle, ctypes.c_void_p(src.data_ptr()), self._stream()), "dawn_lfg_set_source")
        return src

    # ------------------------------------------------------------------ reference API
    @torch.no_grad()
    def compute_fea(self, source_image):
        """generator.py:132-136.  source_image (b, 3, H, W) -> (b, C_bottleneck, H / 2^n, W / 2^n)."""
        b, _, H, W = source_image.shape
        d = 2 ** self.num_down_blocks
        out = torch.empty((b, self.bottleneck_channels, H // d, W // d), device=source_image.device, dtype=torch.float32)
        g = self._geom
        fh, fw, frames = (g[3], g[4], g[0]) if g is not None and g[1:3] == (H, W) else (H // d, W // d, 1)
        self._ensure(source_image.device, frames, H, W, fh, fw)
        for i in range(b):
            self._set_source(source_image[i:i + 1])
            with torch.cuda.device(source_image.device):
                check(lib.dawn_lfg_get_fea(self._handle, ctypes.c_void_p(out[i].data_ptr()), self._stream()), "dawn_lfg_get_fea")
        return out

    @torch.no_grad()
    def forward_with_flow(self, source_image, optical_flow, occlusion_map, need_deformed=True):
        """generator.py:138-171 for a whole batch of frames: source_image (1, 3, H, W); optical_flow (F, h, w, 2) sampling grid
        in [-1, 1]; occlusion_map (F, 1, h, w).  Returns {"prediction": (F, 3, H, W), "deformed": (F, 3, H, W)}."""
        F_, fh, fw, two = optical_flow.shape
        assert two == 2 and occlusion_map.shape == (F_, 1, fh, fw)
        H, W = source_image.shape[-2:]
        dev = source_image.device
        self._ensure(dev, F_, H, W, fh, fw)
        self._set_source(source_image)
        flow = optical_flow.contiguous().float()
        occ = occlusion_map.contiguous().float()
        pred = torch.empty((F_, 3, H, W), device=dev, dtype=torch.float32)
        deformed = torch.empty_like(pred) if need_deformed else None
        with torch.cuda.device(dev):
            check(lib.dawn_lfg_decode(self._handle, ctypes.c_void_p(flow.data_ptr()), ctypes.c_void_p(occ.data_ptr()),
                                      ctypes.c_void_p(pred.data_ptr()),
                                      ctypes.c_void_p(deformed.data_ptr()) if deformed is not None else None, self._stream()),
                  "dawn_lfg_decode")
        return {"prediction": pred, "deformed": deformed}

    @torch.no_grad()
    def decode_sample(self, source_image, sample, need_deformed=False):
        """The sampler's output straight to frames (sample_one_video, FD:366-383): sample (3, F, h, w) = [grid_x, grid_y, conf],
        occlusion = (conf + 1) / 2.  Returns prediction (F, 3, H, W) [and deformed]."""
        _, F_, fh, fw = sample.shape
        H, W = source_image.shape[-2:]
        dev = source_image.device
        self._ensure(dev, F_, H, W, fh, fw)
        self._set_source(source_image)
        s = sample.contiguous().float()
        pred = torch.empty((F_, 3, H, W), device=dev, dtype=torch.float32)
        deformed = torch.empty_like(pred) if need_deformed else None
        with torch.cuda.device(dev):
            check(lib.dawn_lfg_decode_sample(self._handle, ctypes.c_void_p(s.data_ptr()), ctypes.c_void_p(pred.data_ptr()),
                                             ctypes.c_void_p(deformed.data_ptr()) if deformed is not None else None, self._stream()),
                  "dawn_lfg_decode_sample")
        return (pred, deformed) if need_deformed else pred

    def forward(self, *a, **k):
        raise NotImplementedError("Generator.forward (region-driven training path, generator.py:92-130) is out of scope; "
                                  "use forward_with_flow / compute_fea")

    # ------------------------------------------------------------------ debugging taps
    def read_tap(self, name):
        """(frames, C, Hl, Wl) copy of an internal activation of the last decode: 'bottleneck', 'up0', 'up1'."""
        C, Hl, Wl = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        check(lib.dawn_lfg_read_tap(self._handle, name.encode(), None, ctypes.byref(C), ctypes.byref(Hl), ctypes.byref(Wl), None),
              "dawn_lfg_read_tap")
        frames = self._geom[0]
        t = torch.empty((C.value, frames, Hl.value, Wl.value), device=torch.device("cuda", self._device_index))
        with torch.cuda.device(self._device_index):
            check(lib.dawn_lfg_read_tap(self._handle, name.encode(), ctypes.c_void_p(t.data_ptr()), ctypes.byref(C), ctypes.byref(Hl),
                                        ctypes.byref(Wl), self._stream()), "dawn_lfg_read_tap")
        return t.permute(1, 0, 2, 3).contiguous()

    def last_launch_count(self):
        return int(lib.dawn_lfg_last_launch_count(self._handle)) if self._handle is not None else 0

    def workspace_bytes(self):
        return int(lib.dawn_lfg_workspace_bytes(self._handle)) if self._handle is not None else 0
