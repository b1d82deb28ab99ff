"""TEST INFRASTRUCTURE — torch restatement of the motion estimator of DAWN's LFG autoencoder: the region predictor, the
background motion predictor and the generator's pixelwise flow predictor, plus `Generator.forward` and `FlowAE.forward` on
top of oracle/lfg_oracle.py's decoder.  Only tests/ and tools/ may import this; the product path never does.

Restates, batched over frames:
  LFG/modules/util.py:22-48           region2gaussian                (Gaussian of a region's mean / covariance)
  LFG/modules/util.py:51-67           make_coordinate_grid           ([-1, 1] grid, x first)
  LFG/modules/util.py:153-215         Encoder / Decoder / Hourglass  (DownBlock2d / UpBlock2d stacks, decoder concatenates skips)
  LFG/modules/util.py:217-264         AntiAliasInterpolation2d       (13x13 Gaussian, sigma 1.5, every 4th pixel)
  LFG/modules/region_predictor.py:16-117        RegionPredictor (pca_based, host SVD)
  LFG/modules/bg_motion_predictor.py:15-57      BGMotionPredictor
  LFG/modules/pixelwise_flow_predictor.py:16-137 PixelwiseFlowPredictor
  LFG/modules/generator.py:92-130     Generator.forward
  LFG/modules/flow_autoenc.py:37-46   FlowAE.forward
Pinned against the real reference by oracle/make_golden_lfg_motion.py (golden vectors under tests/golden/lfg_motion_*.npz).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import lfg_oracle as L
from oracle import weights as W


class MotionCfg:
    """model_params of config/hdtf128.yaml == config/hdtf256.yaml: region_predictor_params, bg_predictor_params and
    generator_params.pixelwise_flow_predictor_params."""

    def __init__(self, bg_type='affine', revert_axis_swap=True):
        self.num_regions, self.num_channels = 10, 3
        self.rp = dict(block_expansion=32, max_features=1024, num_blocks=5, temperature=0.1, scale_factor=0.25)
        self.bg = dict(block_expansion=32, max_features=1024, num_blocks=5)
        self.pw = dict(block_expansion=64, max_features=1024, num_blocks=5, scale_factor=0.25)
        self.bg_type, self.revert_axis_swap = bg_type, revert_axis_swap

    @property
    def pw_in(self):                                             # pixelwise_flow_predictor.py:29-30
        return (self.num_regions + 1) * (self.num_channels + 1)


# ----------------------------------------------------------------------------- state_dict schemas
def _enc_features(be, cin, mx, nb):                              # util.py:159-163
    return [(cin if i == 0 else min(mx, be * 2 ** i), min(mx, be * 2 ** (i + 1))) for i in range(nb)]


def _dec_features(be, mx, nb):                                   # util.py:183-186, outermost (first applied) block first
    return [((1 if i == nb - 1 else 2) * min(mx, be * 2 ** (i + 1)), min(mx, be * 2 ** i)) for i in reversed(range(nb))]


def _conv_bn(out, prefix, ci, co, k=3):
    out.append((f"{prefix}.conv.weight", (co, ci, k, k)))
    out.append((f"{prefix}.conv.bias", (co,)))
    out.extend([(f"{prefix}.norm.{n}", (co,)) for n in ("weight", "bias", "running_mean", "running_var")])
    out.append((f"{prefix}.norm.num_batches_tracked", ()))


def _hourglass_schema(out, prefix, be, cin, mx, nb):
    for i, (ci, co) in enumerate(_enc_features(be, cin, mx, nb)):
        _conv_bn(out, f"{prefix}.encoder.down_blocks.{i}", ci, co)
    for j, (ci, co) in enumerate(_dec_features(be, mx, nb)):
        _conv_bn(out, f"{prefix}.decoder.up_blocks.{j}", ci, co)
    return be + cin                                              # util.py:189: out_filters


def region_predictor_schema(cfg=None):
    """RegionPredictor.state_dict() order: predictor (Hourglass), regions, down."""
    cfg = cfg or MotionCfg()
    r = cfg.rp
    out = []
    of = _hourglass_schema(out, "predictor", r["block_expansion"], cfg.num_channels, r["max_features"], r["num_blocks"])
    out += [("regions.weight", (cfg.num_regions, of, 7, 7)), ("regions.bias", (cfg.num_regions,)),
            ("down.weight", (cfg.num_channels, 1, 13, 13))]
    return out


def bg_predictor_schema(cfg=None):
    cfg = cfg or MotionCfg()
    b = cfg.bg
    out = []
    if cfg.bg_type == 'zero':
        return out
    for i, (ci, co) in enumerate(_enc_features(b["block_expansion"], 2 * cfg.num_channels, b["max_features"], b["num_blocks"])):
        _conv_bn(out, f"encoder.down_blocks.{i}", ci, co)
    cf = min(b["max_features"], b["block_expansion"] * 2 ** b["num_blocks"])
    out += [("fc.weight", (6, cf)), ("fc.bias", (6,))]
    return out


def flow_predictor_schema(cfg=None, prefix="pixelwise_flow_predictor"):
    """The generator's pixelwise_flow_predictor.* entries (generator.py:29-34): hourglass, mask, occlusion, down."""
    cfg = cfg or MotionCfg()
    p = cfg.pw
    out = []
    of = _hourglass_schema(out, f"{prefix}.hourglass", p["block_expansion"], cfg.pw_in, p["max_features"], p["num_blocks"])
    out += [(f"{prefix}.mask.weight", (cfg.num_regions + 1, of, 7, 7)), (f"{prefix}.mask.bias", (cfg.num_regions + 1,)),
            (f"{prefix}.occlusion.weight", (1, of, 7, 7)), (f"{prefix}.occlusion.bias", (1,)),
            (f"{prefix}.down.weight", (cfg.num_channels, 1, 13, 13))]
    return out


def generator_schema(cfg=None):
    """The reference Generator's full state_dict order: pixelwise_flow_predictor first (generator.py:29-34), then the decoder."""
    return flow_predictor_schema(cfg) + L.state_dict_schema()


# ----------------------------------------------------------------------------- synthetic weights
def anti_alias_weight(channels=3, scale=0.25):
    """The registered `down.weight` buffer of AntiAliasInterpolation2d (util.py:222-250), fp32 as the reference builds it."""
    sigma = (1 / scale - 1) / 2
    ks = 2 * round(sigma * 4) + 1
    m = torch.arange(ks, dtype=torch.float32)
    g = torch.exp(-(m - (ks - 1) / 2) ** 2 / (2 * sigma ** 2))
    k = g.view(-1, 1) * g.view(1, -1)
    k = k / torch.sum(k)
    return k.view(1, 1, ks, ks).repeat(channels, 1, 1, 1)


def motion_synth_value(name, shape):
    """lfg_synth_value (oracle/weights.py) for convolutions and BatchNorms; the Gaussian buffers keep their own values; the
    background `fc` stays close to its identity initialisation (bg_motion_predictor.py:33-35) with a perturbation that still
    reaches every term of the 3x3 matrix."""
    if name.endswith("down.weight"):
        return anti_alias_weight(shape[0]).numpy()
    if name.endswith("fc.weight"):
        return W.symmetric(name, shape, 0.5 / math.sqrt(shape[1]))
    if name.endswith("fc.bias"):
        return np.array([1, 0, 0, 0, 1, 0], dtype=np.float32) + W.symmetric(name, shape, 0.05)
    return W.lfg_synth_value(name, shape)


def motion_synth_state_dict(schema):
    return {n: torch.from_numpy(np.ascontiguousarray(motion_synth_value(n, s))) for n, s in schema}


def motion_synth_inputs(tag, N, H, Wd):
    """source image (1, 3, H, W) in [0, 1] (lfg_synth_inputs' image) and N driving frames that share 70 % of it, so that the
    regions of source and driving frames are related as in a real clip."""
    src = W.lfg_synth_inputs(tag, 1, H, Wd, 1, 1)[0]
    noise = torch.from_numpy(W.uniform01(f"{tag}/driving", N * 3 * H * Wd).reshape(N, 3, H, Wd))
    drv = src * np.float32(0.7) + noise * np.float32(0.3)
    return src, drv


# ----------------------------------------------------------------------------- primitives
def coordinate_grid(h, w, dtype=torch.float32, device=None):
    """make_coordinate_grid (util.py:51-67): (h, w, 2) with [..., 0] = x = 2 j / (w - 1) - 1, [..., 1] = y."""
    x = 2 * (torch.arange(w, dtype=dtype, device=device) / (w - 1)) - 1
    y = 2 * (torch.arange(h, dtype=dtype, device=device) / (h - 1)) - 1
    return torch.stack([x.view(1, -1).expand(h, w), y.view(-1, 1).expand(h, w)], dim=2)


def anti_alias(x, weight):
    """AntiAliasInterpolation2d.forward (util.py:254-264) at scale 0.25: zero pad 6, depthwise 13x13, every 4th pixel."""
    ka = weight.shape[-1] // 2
    out = F.conv2d(F.pad(x, (ka, ka, ka, ka)), weight, groups=x.shape[1])
    return out[:, :, ::4, ::4]


def encoder(sd, prefix, x, nb):
    """Encoder.forward (util.py:165-169): [x, level 1, ..., level nb]."""
    outs = [x]
    for i in range(nb):
        outs.append(F.avg_pool2d(L.conv_bn_relu(sd, f"{prefix}.down_blocks.{i}", outs[-1], 1), 2))   # util.py:126-131
    return outs


def hourglass(sd, prefix, x, nb, taps=None):
    """Hourglass.forward (util.py:211-215): Decoder (util.py:191-197) over the Encoder's levels, concatenating each skip."""
    outs = encoder(sd, f"{prefix}.encoder", x, nb)
    out = outs.pop()
    for j in range(nb):
        out = L.conv_bn_relu(sd, f"{prefix}.decoder.up_blocks.{j}", F.interpolate(out, scale_factor=2), 1)   # util.py:106-111
        out = torch.cat([out, outs.pop()], dim=1)
    if taps is not None:
        taps[prefix] = out
    return out


def region_moments(heat):
    """region2affine (region_predictor.py:60-75): shift (N, R, 2) and covar (N, R, 2, 2) of (N, R, h, w) heatmaps."""
    grid = coordinate_grid(*heat.shape[2:], dtype=heat.dtype, device=heat.device).view(1, 1, *heat.shape[2:], 2)
    region = heat.unsqueeze(-1)
    mean = (region * grid).sum(dim=(2, 3))
    sub = grid - mean.unsqueeze(-2).unsqueeze(-2)
    covar = (torch.matmul(sub.unsqueeze(-1), sub.unsqueeze(-2)) * region.unsqueeze(-1)).sum(dim=(2, 3))
    return mean, covar


def host_svd(covar):
    """region_predictor.py:16-25 and 107-115: torch.svd on the host, affine = u diag(sqrt(s))."""
    shape = covar.shape
    u, s, _ = torch.svd(covar.reshape(-1, 2, 2).cpu())
    u, s = u.to(covar.device), s.to(covar.device)
    d = torch.diag_embed(s ** 0.5)
    return torch.matmul(u, d).view(*shape), u, d


# ----------------------------------------------------------------------------- the three predictors
def region_predictor(sd, cfg, x, taps=None):
    """RegionPredictor.forward (region_predictor.py:77-117) with pca_based = True, estimate_affine = True."""
    r = cfg.rp
    x = anti_alias(x, sd["down.weight"])
    fm = hourglass(sd, "predictor", x, r["num_blocks"], taps)
    pred = F.conv2d(fm, sd["regions.weight"], sd["regions.bias"], padding=3)
    n, R, h, w = pred.shape
    heat = F.softmax(pred.view(n, R, -1) / r["temperature"], dim=2).view(n, R, h, w)
    shift, covar = region_moments(heat)
    affine, u, d = host_svd(covar)
    return {"shift": shift, "covar": covar, "heatmap": heat, "affine": affine, "u": u, "d": d}


def bg_predictor(sd, cfg, source, driving, taps=None):
    """BGMotionPredictor.forward (bg_motion_predictor.py:42-57), bg_type 'affine' or 'zero'."""
    bs = source.shape[0]
    out = torch.eye(3, dtype=source.dtype, device=source.device).unsqueeze(0).repeat(bs, 1, 1)
    if cfg.bg_type == 'zero':
        return out
    last = encoder(sd, "encoder", torch.cat([source, driving], dim=1), cfg.bg["num_blocks"])[-1]
    if taps is not None:
        taps["encoder"] = last
    pred = F.linear(last.mean(dim=(2, 3)), sd["fc.weight"], sd["fc.bias"])
    out[:, :2, :] = pred.view(bs, 2, 3)
    return out


def region_gaussian(shift, covar, h, w):
    """region2gaussian (util.py:22-48) with a covariance: exp(-0.5 (g - mu)^T covar^-1 (g - mu)), (N, R, h, w)."""
    grid = coordinate_grid(h, w, dtype=shift.dtype, device=shift.device).view(1, 1, h, w, 2)
    sub = grid - shift.view(*shift.shape[:2], 1, 1, 2)
    inv = torch.inverse(covar).view(*shift.shape[:2], 1, 1, 2, 2)
    e = torch.matmul(torch.matmul(sub.unsqueeze(-2), inv), sub.unsqueeze(-1))
    return torch.exp(-0.5 * e.sum(dim=(-1, -2)))


def sparse_motions(cfg, h, w, drv, src, bg):
    """create_sparse_motions (pixelwise_flow_predictor.py:68-97): (N, R + 1, h, w, 2), background grid first."""
    n, R = src["shift"].shape[:2]
    grid = coordinate_grid(h, w, dtype=src["shift"].dtype, device=src["shift"].device).view(1, 1, h, w, 2)
    coord = grid - drv["shift"].view(n, R, 1, 1, 2)
    affine = torch.matmul(src["affine"], torch.inverse(drv["affine"].float()))
    if cfg.revert_axis_swap:
        affine = affine * torch.sign(affine[:, :, 0:1, 0:1])
    coord = torch.matmul(affine.view(n, R, 1, 1, 2, 2), coord.unsqueeze(-1)).squeeze(-1)
    d2s = coord + src["shift"].view(n, R, 1, 1, 2)
    bg_grid = grid.expand(n, 1, h, w, 2)
    if bg is not None:
        hom = torch.cat([bg_grid, torch.ones_like(bg_grid[..., :1])], dim=-1)
        hom = torch.matmul(bg.view(n, 1, 1, 1, 3, 3), hom.unsqueeze(-1)).squeeze(-1)
        bg_grid = hom[..., :2] / hom[..., 2:3]                   # from_homogeneous, util.py:274-275
    return torch.cat([bg_grid, d2s], dim=1)


def flow_predictor(sd, cfg, source, drv, src, bg=None, prefix="pixelwise_flow_predictor", taps=None):
    """PixelwiseFlowPredictor.forward (pixelwise_flow_predictor.py:111-137), use_covar_heatmap / use_deformed_source /
    estimate_occlusion_map all true.  source (N, 3, H, W).  Returns optical_flow (N, h, w, 2), occlusion_map (N, 1, h, w)."""
    x = anti_alias(source, sd[f"{prefix}.down.weight"])
    n, c, h, w = x.shape
    R = cfg.num_regions
    heat = region_gaussian(drv["shift"], drv["covar"], h, w) - region_gaussian(src["shift"], src["covar"], h, w)
    heat = torch.cat([torch.zeros_like(heat[:, :1]), heat], dim=1).unsqueeze(2)              # :63-66
    motion = sparse_motions(cfg, h, w, drv, src, bg)
    rep = x.unsqueeze(1).expand(n, R + 1, c, h, w).reshape(n * (R + 1), c, h, w)
    deformed = F.grid_sample(rep, motion.reshape(n * (R + 1), h, w, 2), mode='bilinear', padding_mode='zeros',
                             align_corners=False).view(n, R + 1, c, h, w)                      # :99-109
    inp = torch.cat([heat, deformed], dim=2).view(n, -1, h, w)
    if taps is not None:
        taps["input"] = inp
    pred = hourglass(sd, f"{prefix}.hourglass", inp, cfg.pw["num_blocks"], taps)
    mask = F.softmax(F.conv2d(pred, sd[f"{prefix}.mask.weight"], sd[f"{prefix}.mask.bias"], padding=3), dim=1)
    flow = (motion.permute(0, 1, 4, 2, 3) * mask.unsqueeze(2)).sum(dim=1).permute(0, 2, 3, 1)
    occ = torch.sigmoid(F.conv2d(pred, sd[f"{prefix}.occlusion.weight"], sd[f"{prefix}.occlusion.bias"], padding=3))
    return {"optical_flow": flow, "occlusion_map": occ}


def decode_sd(gen_sd):
    return {k: v for k, v in gen_sd.items() if not k.startswith("pixelwise_flow_predictor.")}


def generator_forward(gen_sd, cfg, source, drv, src, bg=None, taps=None):
    """Generator.forward (generator.py:92-130): flow predictor, then the decoder of oracle/lfg_oracle.py frame by frame
    against its own source image.  source (N, 3, H, W)."""
    m = flow_predictor(gen_sd, cfg, source, drv, src, bg, taps=taps)
    dsd, lcfg = decode_sd(gen_sd), L.LfgCfg()
    pred, deformed, fea = [], [], []
    for i in range(source.shape[0]):
        o = L.forward_with_flow(dsd, lcfg, source[i:i + 1], m["optical_flow"][i:i + 1], m["occlusion_map"][i:i + 1])
        pred.append(o["prediction"]); deformed.append(o["deformed"])
        fea.append(L.compute_fea(dsd, lcfg, source[i:i + 1]))
    return {"bottle_neck_feat": torch.cat(fea), "deformed": torch.cat(deformed), "optical_flow": m["optical_flow"],
            "occlusion_map": m["occlusion_map"], "prediction": torch.cat(pred)}


def flowae_forward(rp_sd, bg_sd, gen_sd, cfg, ref_img, dri_img):
    """FlowAE.forward (flow_autoenc.py:37-46)."""
    src = region_predictor(rp_sd, cfg, ref_img)
    drv = region_predictor(rp_sd, cfg, dri_img)
    bg = bg_predictor(bg_sd, cfg, ref_img, dri_img)
    out = generator_forward(gen_sd, cfg, ref_img, drv, src, bg)
    out.update({"source_region_params": src, "driving_region_params": drv, "bg_params": bg})
    return out


def conditioning(covar):
    """(min eigenvalue, min (s1 - s2) / s1) over a batch of 2x2 covariances: how well the SVD's column signs are defined."""
    s = torch.linalg.svdvals(covar.reshape(-1, 2, 2).double())
    return s[:, 1].min().item(), ((s[:, 0] - s[:, 1]) / s[:, 0]).min().item()
