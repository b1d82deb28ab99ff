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
from ._lib import DawnLfgCfg, _Handle, _Holder, _NativeModule, check, lib, ptr, stream


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


class Generator(_NativeModule):
    IGNORED_PREFIX = "pixelwise_flow_predictor."
    TRAIN_REFUSAL = "this LFG decoder is inference-only (eval-mode BatchNorm, FD:121)"

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
        self._lfg = _Handle("dawn_lfg", cfg, "the LFG decoder")
        self._register_load_state_dict_pre_hook(self._drop_training_only_keys)
        self._hold(self._lfg)

    @property
    def _cfg(self):
        """the dawn_lfg_cfg the decoder's handle is created with"""
        return self._lfg.cfg

    # the reference checkpoint's `generator` entry also holds the training-time flow predictor (generator.py:29-34)
    @classmethod
    def _drop_training_only_keys(cls, state_dict, prefix, *args):
        for k in [k for k in state_dict if k.startswith(prefix + cls.IGNORED_PREFIX)]:
            del state_dict[k]

    def _ensure(self, device, frames, H, W, fh, fw):
        idx = self._lfg.ensure(self, device)
        if self._lfg.geom != (frames, H, W, fh, fw):
            with torch.cuda.device(idx):
                check(lib.dawn_lfg_set_geometry(self._lfg.handle, frames, H, W, fh, fw), "dawn_lfg_set_geometry")
            self._lfg.geom = (frames, H, W, fh, fw)

    def _set_source(self, source_image):
        src = source_image.reshape(-1, *source_image.shape[-3:])
        if src.shape[0] != 1:
            raise ValueError("one source image per call (the reference decodes with batch 1, FD:375-383)")
        src = src[0].contiguous().float()
        with torch.cuda.device(src.device):
            check(lib.dawn_lfg_set_source(self._lfg.handle, ptr(src), stream()), "dawn_lfg_set_source")
        return src

    # ------------------------------------------------------------------ reference API
    @torch.no_grad()
    def compute_fea(self, source_image):
        """generator.py:132-136.  source_image (b, 3, H, W) -> (b, C_bottleneck, H / 2^n, W / 2^n)."""
        b, _, H, W = source_image.shape
        d = 2 ** self.num_down_blocks
        out = torch.empty((b, self.bottleneck_channels, H // d, W // d), device=source_image.device, dtype=torch.float32)
        g = self._lfg.geom
        fh, fw, frames = (g[3], g[4], g[0]) if g is not None and g[1:3] == (H, W) else (H // d, W // d, 1)
        self._ensure(source_image.device, frames, H, W, fh, fw)
        for i in range(b):
            self._set_source(source_image[i:i + 1])
            with torch.cuda.device(source_image.device):
                check(lib.dawn_lfg_get_fea(self._lfg.handle, ptr(out[i]), stream()), "dawn_lfg_get_fea")
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
            check(lib.dawn_lfg_decode(self._lfg.handle, ptr(flow), ptr(occ), ptr(pred), ptr(deformed), stream()), "dawn_lfg_decode")
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
            check(lib.dawn_lfg_decode_sample(self._lfg.handle, ptr(s), ptr(pred), ptr(deformed), stream()), "dawn_lfg_decode_sample")
        return (pred, deformed) if need_deformed else pred

    @torch.no_grad()
    def decode_sample_rgb8(self, source_image, sample, mean=(0.0, 0.0, 0.0)):
        """decode_sample straight to 8-bit RGB frames (F, H, W, 3) uint8 on the device: each fp32 prediction offset by mean / 255,
        clipped to [0, 1], times 255 and truncated, as unified_video_generator.py:544-548 converts a frame (RGB order)."""
        _, F_, fh, fw = sample.shape
        H, W = source_image.shape[-2:]
        dev = source_image.device
        self._ensure(dev, F_, H, W, fh, fw)
        self._set_source(source_image)
        s = sample.contiguous().float()
        m = (ctypes.c_double * 3)(*[float(v) for v in mean])
        frames = torch.empty((F_, H, W, 3), device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            check(lib.dawn_lfg_decode_sample_rgb8(self._lfg.handle, ptr(s), m, ptr(frames), stream()), "dawn_lfg_decode_sample_rgb8")
        return frames

    def forward(self, *a, **k):
        raise NotImplementedError("Generator.forward (region-driven training path, generator.py:92-130) is out of scope; "
                                  "use forward_with_flow / compute_fea")

    # ------------------------------------------------------------------ debugging taps
    def read_tap(self, name):
        """(frames, C, Hl, Wl) copy of an internal activation of the last decode: 'bottleneck', 'up0', 'up1'."""
        C, Hl, Wl = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        h = self._lfg
        check(lib.dawn_lfg_read_tap(h.handle, name.encode(), None, ctypes.byref(C), ctypes.byref(Hl), ctypes.byref(Wl), None),
              "dawn_lfg_read_tap")
        t = torch.empty((C.value, h.geom[0], Hl.value, Wl.value), device=torch.device("cuda", h.device_index))
        with torch.cuda.device(h.device_index):
            check(lib.dawn_lfg_read_tap(h.handle, name.encode(), ptr(t), ctypes.byref(C), ctypes.byref(Hl), ctypes.byref(Wl), stream()),
                  "dawn_lfg_read_tap")
        return t.permute(1, 0, 2, 3).contiguous()



# ====================================================================================================================================
# Motion estimator of the LFG autoencoder: RegionPredictor, BGMotionPredictor, the Generator's PixelwiseFlowPredictor, and FlowAE
# (LFG/modules/region_predictor.py, bg_motion_predictor.py, pixelwise_flow_predictor.py, flow_autoenc.py) behind the
# dawn_lfg_motion handle of include/dawn_lfg.h.  Same constructor keywords and state_dict keys as the reference modules; the
# sub-modules only hold parameters.  The 2x2 SVD of the region covariances runs on the host, as in the reference
# (region_predictor.py:16-25): one device-to-host copy per RegionPredictor call.
MOTION_CHUNK = 50                    # frames per stage call: bounds the workspace (the full-resolution background encoder) and
                                     # keeps every activation index below 2^31


def _encoder(be, cin, mx, nb):                               # Encoder (util.py:153-169)
    m = _Holder()
    m.down_blocks = nn.ModuleList([_conv_bn(cin if i == 0 else min(mx, be * 2 ** i), min(mx, be * 2 ** (i + 1)), 3)
                                   for i in range(nb)])
    return m


def _hourglass(be, cin, mx, nb):                             # Hourglass (util.py:172-215)
    m = _Holder()
    m.encoder = _encoder(be, cin, mx, nb)
    m.decoder = _Holder()
    m.decoder.up_blocks = nn.ModuleList([_conv_bn((1 if i == nb - 1 else 2) * min(mx, be * 2 ** (i + 1)), min(mx, be * 2 ** i), 3)
                                         for i in reversed(range(nb))])
    m.out_filters = be + cin
    return m


def _anti_alias(channels, scale):
    """AntiAliasInterpolation2d (util.py:217-251): the Gaussian `weight` buffer, built as the reference builds it."""
    m = _Holder()
    sigma = (1 / scale - 1) / 2
    ks = 2 * round(sigma * 4) + 1
    g = torch.exp(-(torch.arange(ks, dtype=torch.float32) - (ks - 1) / 2) ** 2 / (2 * sigma ** 2))
    k = g.view(-1, 1) * g.view(1, -1)
    m.register_buffer('weight', (k / torch.sum(k)).view(1, 1, ks, ks).repeat(channels, 1, 1, 1))
    return m


def _motion_cfg(**kw):
    c = _lib.DawnLfgMotionCfg(num_regions=10, num_channels=3, estimate_affine=1, pca_based=1, fast_svd=0,
                              rp_block_expansion=32, rp_max_features=1024, rp_num_blocks=5, rp_temperature=0.1, rp_scale_factor=0.25,
                              bg_block_expansion=32, bg_max_features=1024, bg_num_blocks=5, bg_type=_lib.LFG_BG_AFFINE,
                              pw_block_expansion=64, pw_max_features=1024, pw_num_blocks=5, pw_scale_factor=0.25,
                              use_covar_heatmap=1, use_deformed_source=1, estimate_occlusion_map=1, revert_axis_swap=1)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _motion_handle(cfg, param_name):
    h = _Handle("dawn_lfg_motion", cfg, "the LFG motion estimator", param_name)
    h.validate()
    return h


def _motion_geometry(h, module, device, n, H, W):
    """Readies the motion handle h of `module` for n frames of (H, W) images; returns the frames per stage call.  The
    workspace only grows: fewer frames of the same size reuse it."""
    idx = h.ensure(module, device)
    frames = min(n, MOTION_CHUNK)
    if h.geom is None or h.geom[1:] != (H, W) or h.geom[0] < frames:
        with torch.cuda.device(idx):
            check(lib.dawn_lfg_motion_set_geometry(h.handle, frames, H, W), "dawn_lfg_motion_set_geometry")
        h.geom = (frames, H, W)
    return h.geom[0]


def _motion_read_tap(h, name):
    """(n, C, Hl, Wl) copy of the last call's 'region_predictor' / 'bg_encoder' / 'flow_hourglass' output (last chunk)."""
    C, n, Hl, Wl = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    args = (ctypes.byref(C), ctypes.byref(n), ctypes.byref(Hl), ctypes.byref(Wl))
    check(lib.dawn_lfg_motion_read_tap(h.handle, name.encode(), None, *args, None), "dawn_lfg_motion_read_tap")
    t = torch.empty((C.value, n.value, Hl.value, Wl.value), device=torch.device("cuda", h.device_index))
    with torch.cuda.device(h.device_index):
        check(lib.dawn_lfg_motion_read_tap(h.handle, name.encode(), ptr(t), *args, stream()), "dawn_lfg_motion_read_tap")
    return t.permute(1, 0, 2, 3).contiguous()


_MOTION_TRAIN_REFUSAL = "the LFG motion estimator is inference-only (eval-mode BatchNorm)"


class RegionPredictor(_NativeModule):
    """region_predictor.py:28-117 with DAWN's region_predictor_params (pca_based, host SVD)."""
    TRAIN_REFUSAL = _MOTION_TRAIN_REFUSAL

    def __init__(self, block_expansion, num_regions, num_channels, max_features, num_blocks, temperature, estimate_affine=False,
                 scale_factor=1, pca_based=False, fast_svd=False, pad=3):
        super().__init__()
        self.predictor = _hourglass(block_expansion, num_channels, max_features, num_blocks)
        self.regions = nn.Conv2d(self.predictor.out_filters, num_regions, kernel_size=(7, 7), padding=pad)
        self.jacobian = None
        self.temperature, self.scale_factor, self.pca_based, self.fast_svd = temperature, scale_factor, pca_based, fast_svd
        if scale_factor != 1:
            self.down = _anti_alias(num_channels, scale_factor)
        if pad != 3:
            raise _lib.DawnError("RegionPredictor: only pad 3 (the 7x7 regions conv's same padding) is supported")
        self._motion = _motion_handle(_motion_cfg(num_regions=num_regions, num_channels=num_channels,
                                                  estimate_affine=int(bool(estimate_affine)), pca_based=int(bool(pca_based)),
                                                  fast_svd=int(bool(fast_svd)), rp_block_expansion=block_expansion,
                                                  rp_max_features=max_features, rp_num_blocks=num_blocks, rp_temperature=temperature,
                                                  rp_scale_factor=scale_factor), lambda key: "region_predictor." + key)
        self._hold(self._motion)

    @torch.no_grad()
    def forward(self, x):
        n, _, H, W = x.shape
        dev = x.device
        chunk = _motion_geometry(self._motion, self, dev, n, H, W)
        R = self.regions.out_channels
        x = x.contiguous().float()
        shift = torch.empty((n, R, 2), device=dev)
        covar = torch.empty((n, R, 2, 2), device=dev)
        heat = torch.empty((n, R, H // 4, W // 4), device=dev)
        with torch.cuda.device(dev):
            st = stream()
            for a in range(0, n, chunk):
                b = min(n, a + chunk)
                check(lib.dawn_lfg_motion_regions(self._motion.handle, ptr(x[a:b]), b - a, ptr(shift[a:b]), ptr(covar[a:b]),
                                                  ptr(heat[a:b]), st), "dawn_lfg_motion_regions")
        u, s, _ = torch.svd(covar.view(-1, 2, 2).cpu())                   # region_predictor.py:16-25, as the reference does
        u, s = u.to(dev), s.to(dev)
        d = torch.diag_embed(s ** 0.5)
        affine = torch.matmul(u, d).view(n, R, 2, 2)
        return {"shift": shift, "covar": covar, "heatmap": heat, "affine": affine, "u": u, "d": d}

    def read_tap(self, name):
        return _motion_read_tap(self._motion, name)


class BGMotionPredictor(_NativeModule):
    """bg_motion_predictor.py:15-57 with bg_type 'affine' (DAWN's) or 'zero'."""
    TRAIN_REFUSAL = _MOTION_TRAIN_REFUSAL

    def __init__(self, block_expansion, num_channels, max_features, num_blocks, bg_type='zero'):
        super().__init__()
        if bg_type not in ('zero', 'affine'):
            raise _lib.DawnError(f"dawn_lfg_motion_create failed: lfg_motion: bg_type must be 'affine' or 'zero', got {bg_type!r}")
        self.bg_type = bg_type
        if bg_type != 'zero':
            self.encoder = _encoder(block_expansion, num_channels * 2, max_features, num_blocks)
            self.fc = nn.Linear(min(max_features, block_expansion * 2 ** num_blocks), 6)
        self._motion = _motion_handle(_motion_cfg(num_channels=num_channels, bg_block_expansion=block_expansion,
                                                  bg_max_features=max_features, bg_num_blocks=num_blocks,
                                                  bg_type=_lib.LFG_BG_AFFINE if bg_type == 'affine' else _lib.LFG_BG_ZERO),
                                      lambda key: "bg_predictor." + key)
        self._hold(self._motion)

    @torch.no_grad()
    def forward(self, source_image, driving_image):
        n, _, H, W = driving_image.shape
        dev = driving_image.device
        if source_image.device != dev:
            raise _lib.DawnError("source and driving images must be on the same device")
        chunk = _motion_geometry(self._motion, self, dev, n, H, W)
        src = source_image.contiguous().float()
        drv = driving_image.contiguous().float()
        shared = src.shape[0] == 1 and n > 1
        out = torch.empty((n, 3, 3), device=dev)
        with torch.cuda.device(dev):
            st = stream()
            for a in range(0, n, chunk):
                b = min(n, a + chunk)
                s = src if shared else src[a:b]
                check(lib.dawn_lfg_motion_bg(self._motion.handle, ptr(s), s.shape[0], ptr(drv[a:b]), b - a, ptr(out[a:b]), st),
                      "dawn_lfg_motion_bg")
        return out

    def read_tap(self, name):
        return _motion_read_tap(self._motion, name)


class _FlowPredictor(_Holder):
    """pixelwise_flow_predictor.py:16-46: parameters only; the computation is MotionGenerator.forward."""

    def __init__(self, block_expansion, num_blocks, max_features, num_regions, num_channels, estimate_occlusion_map=False,
                 scale_factor=1, region_var=0.01, use_covar_heatmap=False, use_deformed_source=True, revert_axis_swap=False):
        super().__init__()
        self.hourglass = _hourglass(block_expansion, (num_regions + 1) * (num_channels * use_deformed_source + 1), max_features,
                                    num_blocks)
        self.mask = nn.Conv2d(self.hourglass.out_filters, num_regions + 1, kernel_size=(7, 7), padding=(3, 3))
        self.occlusion = nn.Conv2d(self.hourglass.out_filters, 1, kernel_size=(7, 7), padding=(3, 3)) if estimate_occlusion_map else None
        if scale_factor != 1:
            self.down = _anti_alias(num_channels, scale_factor)
        self.cfg_kw = dict(pw_block_expansion=block_expansion, pw_num_blocks=num_blocks, pw_max_features=max_features,
                           num_regions=num_regions, num_channels=num_channels, estimate_occlusion_map=int(bool(estimate_occlusion_map)),
                           pw_scale_factor=scale_factor, use_covar_heatmap=int(bool(use_covar_heatmap)),
                           use_deformed_source=int(bool(use_deformed_source)), revert_axis_swap=int(bool(revert_axis_swap)))


class MotionGenerator(Generator):
    """The reference Generator with its pixelwise flow predictor (generator.py:20-130): the state_dict holds all of the
    checkpoint's `generator` entry, and forward(source_image, driving_region_params, source_region_params, bg_params) runs the flow
    predictor on the device, then the decoder of Generator (one decode per distinct source image)."""

    def __init__(self, num_channels, num_regions, block_expansion, max_features, num_down_blocks, num_bottleneck_blocks,
                 pixelwise_flow_predictor_params=None, skips=False, revert_axis_swap=True):
        if pixelwise_flow_predictor_params is None:
            raise _lib.DawnError("MotionGenerator needs pixelwise_flow_predictor_params; use Generator for the decoder alone")
        pw = _FlowPredictor(num_regions=num_regions, num_channels=num_channels, revert_axis_swap=revert_axis_swap,
                            **pixelwise_flow_predictor_params)
        Generator.__init__(self, num_channels, num_regions, block_expansion, max_features, num_down_blocks, num_bottleneck_blocks,
                           None, skips, revert_axis_swap)
        self._modules = {"pixelwise_flow_predictor": pw, **self._modules}    # registered first, as generator.py:29-34 does
        self.num_regions = num_regions
        self._motion = _motion_handle(_motion_cfg(**pw.cfg_kw), lambda key: key if key.startswith(Generator.IGNORED_PREFIX) else None)
        self._handles.append(self._motion)

    # keeps pixelwise_flow_predictor.* (the parent class drops them)
    @classmethod
    def _drop_training_only_keys(cls, state_dict, prefix, *args):
        return None

    @torch.no_grad()
    def flow(self, source_image, driving_region_params, source_region_params, bg_params=None):
        """pixelwise_flow_predictor.py:111-137 for n frames of one source image (1 or n, 3, H, W) -> optical_flow, occlusion_map."""
        drv, srcp = driving_region_params, source_region_params
        n = drv["shift"].shape[0]
        H, W = source_image.shape[-2:]
        dev = source_image.device
        chunk = _motion_geometry(self._motion, self, dev, n, H, W)
        R = self.num_regions
        src = source_image.reshape(-1, 3, H, W)[0].contiguous().float()

        def per_frame(t, shape):
            t = t.float()
            return (t.expand(n, *shape) if t.shape[0] == 1 else t).contiguous()

        ss, sc, sa = per_frame(srcp["shift"], (R, 2)), per_frame(srcp["covar"], (R, 2, 2)), per_frame(srcp["affine"], (R, 2, 2))
        ds, dc, da = per_frame(drv["shift"], (R, 2)), per_frame(drv["covar"], (R, 2, 2)), per_frame(drv["affine"], (R, 2, 2))
        bg = per_frame(bg_params, (3, 3)) if bg_params is not None else None
        flow = torch.empty((n, H // 4, W // 4, 2), device=dev)
        occ = torch.empty((n, 1, H // 4, W // 4), device=dev)
        with torch.cuda.device(dev):
            st = stream()
            for a in range(0, n, chunk):
                b = min(n, a + chunk)
                check(lib.dawn_lfg_motion_flow(self._motion.handle, ptr(src), b - a, ptr(ss[a:b]), ptr(sc[a:b]), ptr(sa[a:b]),
                                               ptr(ds[a:b]), ptr(dc[a:b]), ptr(da[a:b]), ptr(bg[a:b]) if bg is not None else None,
                                               ptr(flow[a:b]), ptr(occ[a:b]), st), "dawn_lfg_motion_flow")
        return {"optical_flow": flow, "occlusion_map": occ}

    @torch.no_grad()
    def forward(self, source_image, driving_region_params, source_region_params, bg_params=None):
        """generator.py:92-130: prediction, deformed, optical_flow, occlusion_map and bottle_neck_feat for a batch of frames.
        Frames that share one source image are decoded together."""
        if source_image.device.type != "cuda":
            raise _lib.DawnError("the LFG motion estimator runs on CUDA (sm_90a) only; there is no CPU path")
        n = source_image.shape[0]
        groups = []                                                     # runs of frames with the same source image
        for i in range(n):
            if groups and torch.equal(source_image[i], source_image[groups[-1][0]]):
                groups[-1].append(i)
            else:
                groups.append([i])
        outs = []
        for g in groups:
            a, b = g[0], g[-1] + 1
            sel = lambda p: {k: v[a:b] for k, v in p.items()}            # noqa: E731
            m = self.flow(source_image[a:a + 1], sel(driving_region_params), sel(source_region_params),
                          bg_params[a:b] if bg_params is not None else None)
            o = self.forward_with_flow(source_image[a:a + 1], m["optical_flow"], m["occlusion_map"])
            fea = self.compute_fea(source_image[a:a + 1])
            outs.append({"prediction": o["prediction"], "deformed": o["deformed"], "optical_flow": m["optical_flow"],
                         "occlusion_map": m["occlusion_map"], "bottle_neck_feat": fea.expand(b - a, -1, -1, -1)})
        out = {k: torch.cat([o[k] for o in outs]) for k in outs[0]}
        out["bottle_neck_feat"] = out["bottle_neck_feat"].contiguous()
        return out

    def read_tap(self, name):
        """'flow_hourglass' reads the flow predictor; every other name the decoder (Generator.read_tap)."""
        return _motion_read_tap(self._motion, name) if name == "flow_hourglass" else super().read_tap(name)


class FlowAE(nn.Module):
    """flow_autoenc.py:15-51: region predictor, background predictor and generator of one LFG checkpoint; forward() reconstructs
    dri_img from ref_img into self.generated.  CUDA tensors only."""

    def __init__(self, is_train=False, config_pth=None):
        super().__init__()
        if is_train:
            raise NotImplementedError("FlowAE training is out of scope: this is the inference path")
        mp = _default_model_params()
        if config_pth is not None:
            import yaml
            with open(config_pth) as f:
                mp = yaml.safe_load(f)['model_params']
        self.generator = MotionGenerator(num_regions=mp['num_regions'], num_channels=mp['num_channels'],
                                         revert_axis_swap=mp['revert_axis_swap'], **mp['generator_params'])
        self.region_predictor = RegionPredictor(num_regions=mp['num_regions'], num_channels=mp['num_channels'],
                                                estimate_affine=mp['estimate_affine'], **mp['region_predictor_params'])
        self.bg_predictor = BGMotionPredictor(num_channels=mp['num_channels'], **mp['bg_predictor_params'])
        self.is_train = is_train
        self.ref_img = self.dri_img = self.generated = None
        self.eval()

    def train(self, mode=True):
        if mode:
            raise NotImplementedError("FlowAE here is inference-only")
        return super().train(False)

    def set_train_input(self, ref_img, dri_img):
        self.ref_img, self.dri_img = ref_img, dri_img

    @torch.no_grad()
    def forward(self):
        for t in (self.ref_img, self.dri_img):
            if t.device.type != "cuda":
                raise _lib.DawnError("FlowAE runs on CUDA (sm_90a) only; there is no CPU path")
        source_region_params = self.region_predictor(self.ref_img)
        self.driving_region_params = self.region_predictor(self.dri_img)
        bg_params = self.bg_predictor(self.ref_img, self.dri_img)
        self.generated = self.generator(self.ref_img, source_region_params=source_region_params,
                                        driving_region_params=self.driving_region_params, bg_params=bg_params)
        self.generated.update({'source_region_params': source_region_params, 'driving_region_params': self.driving_region_params})


def _default_model_params():
    """model_params of config/hdtf256.yaml (== hdtf128.yaml)."""
    return {
        'num_regions': 10, 'num_channels': 3, 'estimate_affine': True, 'revert_axis_swap': True,
        'bg_predictor_params': {'block_expansion': 32, 'max_features': 1024, 'num_blocks': 5, 'bg_type': 'affine'},
        'region_predictor_params': {'temperature': 0.1, 'block_expansion': 32, 'max_features': 1024, 'scale_factor': 0.25,
                                    'num_blocks': 5, 'pca_based': True, 'fast_svd': False},
        'generator_params': {'block_expansion': 64, 'max_features': 512, 'num_down_blocks': 2, 'num_bottleneck_blocks': 6,
                             'skips': True,
                             'pixelwise_flow_predictor_params': {'block_expansion': 64, 'max_features': 1024, 'num_blocks': 5,
                                                                 'scale_factor': 0.25, 'use_deformed_source': True,
                                                                 'use_covar_heatmap': True, 'estimate_occlusion_map': True}},
    }
