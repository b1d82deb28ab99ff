"""TEST INFRASTRUCTURE — CPU oracle for the UNet's upconv variant and for UNets without spatial linear attention.

The reference's Unet3D (U = DM_3/modules/video_flow_diffusion_multiGPU_v0_crema_plus_faceemb_ca_multi_test.py) takes three
constructor options oracle/unet_oracle.py does not restate: `use_deconv=False` with a `padding_mode` (U:165-172),
`use_sparse_linear_attn=False` (U:832-833, 854-855) and `use_final_activation` (U:867-871; forward never applies it, U:956).
This module restates the forward with them, built from oracle/unet_oracle.py's sub-modules, and with every option at its
default it is that file's `unet_forward`.  Pinned to the real reference by oracle/make_golden_upconv.py
(tests/golden/upconv.npz); tests/test_upconv_cpu.py re-checks it against those vectors.  NOT product code.
"""
import torch
import torch.nn.functional as F

from oracle import unet_oracle as O

PADDING_MODES = ('zeros', 'reflect', 'replicate', 'circular')


class UpconvCfg(O.UnetCfg):
    """O.UnetCfg plus the up-path and spatial-linear-attention options, defaulting to DAWN's own network."""

    def __init__(self, use_deconv=True, padding_mode='zeros', use_sparse_linear_attn=True, **kw):
        super().__init__(**kw)
        if padding_mode not in PADDING_MODES:
            raise ValueError(f'padding_mode {padding_mode!r}')
        self.use_deconv, self.padding_mode = use_deconv, padding_mode
        self.sla = use_sparse_linear_attn


def upsample_conv(sd, p, x, padding_mode):
    """U:168-172 Upsample(use_deconv=False): nn.Upsample(scale_factor=(1,2,2), mode='nearest'), then Conv3d (1,3,3) with padding
    (0,1,1) in `padding_mode` (on H and W only).  p = 'ups.K.4'."""
    x = F.interpolate(x, scale_factor=2, mode='nearest')
    w, b = sd[p + '.1.weight'][:, :, 0], sd[p + '.1.bias']
    if padding_mode == 'zeros':
        return F.conv2d(x, w, b, padding=1)
    return F.conv2d(F.pad(x, (1, 1, 1, 1), mode=padding_mode), w, b)


def unet_forward(sd, cfg, x, time, cond, band=None, taps=None):
    """U:892-956 Unet3D.forward for ONE clip, as O.unet_forward (null_cond_prob 0), with cfg's up path and SLA options.
    taps: optional dict of sub-module outputs (NCFHW) at the boundaries oracle/make_golden.py hooks (no '.2' without SLA)."""
    assert x.shape[0] == 1, "oracle handles one clip at a time (batch elements are independent)"
    Fr = x.shape[2]
    c = cond[0]
    xf = x[0].permute(1, 0, 2, 3)

    def tap(name, t):
        if taps is not None:
            taps[name] = t.permute(1, 0, 2, 3).unsqueeze(0).clone()

    bias = O.rel_pos_bias(sd['time_rel_pos_bias.relative_attention_bias.weight'], Fr, cfg.win)
    freqs = sd['init_temporal_attn.fn.fn.fn.rotary_emb.freqs']
    pad = cfg.init_k // 2
    xf = F.conv2d(xf, sd['init_conv.weight'][:, :, 0], sd['init_conv.bias'], padding=pad)      # U:910
    r = xf
    tap('init_conv', xf)
    xf = O.temporal_attention(sd, 'init_temporal_attn.fn', xf, bias, freqs, band=band)         # U:913
    tap('init_temporal_attn', xf)
    te = O.sinusoidal(time, cfg.dim)[0]
    te = F.gelu(te @ sd['time_mlp.1.weight'].t() + sd['time_mlp.1.bias'])
    te = te @ sd['time_mlp.3.weight'].t() + sd['time_mlp.3.bias']                              # U:915

    skips = []
    nres = len(cfg.in_out)
    for L in range(nres):                                                                      # U:934-940
        xf = O.resnet_block(sd, f'downs.{L}.0', xf, cfg, te, c)
        tap(f'downs.{L}.0', xf)
        xf = O.resnet_block(sd, f'downs.{L}.1', xf, cfg, te, c)
        tap(f'downs.{L}.1', xf)
        if cfg.sla:
            xf = O.spatial_linear_attention(sd, f'downs.{L}.2.fn', xf)
            tap(f'downs.{L}.2', xf)
        xf = O.temporal_attention(sd, f'downs.{L}.3.fn', xf, bias, freqs, band=band)
        tap(f'downs.{L}.3', xf)
        skips.append(xf)
        if L < nres - 1:
            xf = F.conv2d(xf, sd[f'downs.{L}.4.weight'][:, :, 0], sd[f'downs.{L}.4.bias'], stride=2, padding=1)   # U:175-176
            tap(f'downs.{L}.4', xf)
    xf = O.resnet_block(sd, 'mid_block1', xf, cfg, te, c)                                      # U:942-945
    tap('mid_block1', xf)
    xf = O.mid_spatial_attention(sd, 'mid_spatial_attn.fn', xf)
    tap('mid_spatial_attn', xf)
    xf = O.temporal_attention(sd, 'mid_temporal_attn.fn', xf, bias, freqs, band=band)
    tap('mid_temporal_attn', xf)
    xf = O.resnet_block(sd, 'mid_block2', xf, cfg, te, c)
    tap('mid_block2', xf)
    for K in range(nres):                                                                      # U:947-953
        xf = torch.cat((xf, skips.pop()), dim=1)
        xf = O.resnet_block(sd, f'ups.{K}.0', xf, cfg, te, c)
        tap(f'ups.{K}.0', xf)
        xf = O.resnet_block(sd, f'ups.{K}.1', xf, cfg, te, c)
        tap(f'ups.{K}.1', xf)
        if cfg.sla:
            xf = O.spatial_linear_attention(sd, f'ups.{K}.2.fn', xf)
            tap(f'ups.{K}.2', xf)
        xf = O.temporal_attention(sd, f'ups.{K}.3.fn', xf, bias, freqs, band=band)
        tap(f'ups.{K}.3', xf)
        if K < nres - 1:
            if cfg.use_deconv:                                                                 # U:165-167
                xf = F.conv_transpose2d(xf, sd[f'ups.{K}.4.weight'][:, :, 0], sd[f'ups.{K}.4.bias'], stride=2, padding=1)
            else:
                xf = upsample_conv(sd, f'ups.{K}.4', xf, cfg.padding_mode)
            tap(f'ups.{K}.4', xf)
    xf = torch.cat((xf, r), dim=1)                                                             # U:955
    outs = []
    for head in ('final_conv', 'occlusion_map'):                                               # U:956 (no final activation)
        hd = O.resnet_block(sd, head + '.0', xf, cfg, None, None)
        tap(head + '.0', hd)
        outs.append(F.conv2d(hd, sd[head + '.1.weight'][:, :, 0], sd[head + '.1.bias']))
    return torch.cat(outs, dim=1).permute(1, 0, 2, 3).unsqueeze(0).contiguous()
