"""CPU: the algebraic rewrites the CUDA paths rely on, checked with plain torch ops (host-side logic, no GPU):
 * nearest-2x upsample + 3x3 conv == four output-parity 2x2 convs over the low-resolution grid with summed taps
   (the summed taps in csrc/contraction.cu::pack_up_nearest, the class convs in csrc/contraction.cu::pack_up / run_up,
   reference UpBlock2d LFG/modules/util.py:106-111);
 * a k x k conv == the sum of k row-convolutions (1 x k) over vertically shifted copies of the input
   (csrc/unet.cu::init_map, the per-clip part of the 7x7 init conv, reference U:776-777);
 * the init conv is linear in its input channels: conv(cat[x_t, fea]) == conv3(x_t) + map(fea)  (SURVEY a2, U:1167, 1177);
 * eval-mode BatchNorm after a conv folds into the conv's weights and bias (csrc/contraction.cu::pack_lfg_conv).
"""
import torch
import torch.nn.functional as F

K_UP_OFF = [[-1, 0], [0, 1]]                       # csrc/contraction.cuh: kUpOff[parity][tap] -> low-resolution offset


def up_in_set(parity, tap, k):                      # csrc/contraction.cuh: up_in_set
    return (k == 0 if tap == 0 else k >= 1) if parity == 0 else (k <= 1 if tap == 0 else k == 2)


def test_upsample_conv_equals_parity_class_convs():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 5, 6, 7, generator=g)
    w = torch.randn(4, 5, 3, 3, generator=g)
    b = torch.randn(4, generator=g)
    ref = F.conv2d(F.interpolate(x, scale_factor=2), w, b, padding=1)
    out = torch.empty_like(ref)
    H, W = x.shape[-2:]
    xp = F.pad(x, (1, 1, 1, 1))
    for py in range(2):
        for px in range(2):
            acc = b.view(1, -1, 1, 1).expand(2, 4, H, W).clone()
            for ty in range(2):
                for tx in range(2):
                    wsum = sum(w[:, :, ky, kx] for ky in range(3) for kx in range(3) if up_in_set(py, ty, ky) and up_in_set(px, tx, kx))
                    dy, dx = K_UP_OFF[py][ty], K_UP_OFF[px][tx]
                    patch = xp[:, :, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W]
                    acc = acc + torch.einsum('oc,bchw->bohw', wsum, patch)
            out[:, :, py::2, px::2] = acc
    assert (out - ref).abs().max().item() < 1e-4


def test_square_conv_equals_sum_of_row_convs_over_shifted_copies():
    g = torch.Generator().manual_seed(1)
    k, pad = 7, 3
    x = torch.randn(1, 6, 12, 10, generator=g)
    w = torch.randn(8, 6, k, k, generator=g)
    b = torch.randn(8, generator=g)
    ref = F.conv2d(x, w, b, padding=pad)
    H = x.shape[2]
    total = b.view(1, -1, 1, 1)
    for ky in range(k):
        shifted = torch.zeros_like(x)                                  # copy ky: the frame shifted by ky - pad rows, zero outside
        lo, hi = max(0, pad - ky), min(H, H + pad - ky)
        shifted[:, :, lo:hi] = x[:, :, lo + ky - pad:hi + ky - pad]
        total = total + F.conv2d(shifted, w[:, :, ky:ky + 1, :], None, padding=(0, pad))
    assert (total - ref).abs().max().item() < 1e-4


def test_init_conv_is_linear_in_the_frame_invariant_channels():
    g = torch.Generator().manual_seed(2)
    Fr, h, w_ = 5, 8, 8
    x_t = torch.randn(1, 3, Fr, h, w_, generator=g)
    fea = torch.relu(torch.randn(1, 9, h, w_, generator=g))
    wt = torch.randn(4, 12, 1, 7, 7, generator=g)
    b = torch.randn(4, generator=g)
    x = torch.cat([x_t, fea.unsqueeze(2).expand(-1, -1, Fr, -1, -1)], dim=1)
    ref = F.conv3d(x, wt, b, padding=(0, 3, 3))
    fmap = F.conv2d(fea, wt[:, 3:, 0], b, padding=3)                   # per clip: (1, 4, h, w), bias included
    live = F.conv3d(x_t, wt[:, :3], None, padding=(0, 3, 3))           # per step: 3 live channels
    assert (live + fmap.unsqueeze(2) - ref).abs().max().item() < 1e-4


def test_batchnorm_after_conv_folds_into_the_conv():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 6, 9, 9, generator=g)
    w, b = torch.randn(5, 6, 3, 3, generator=g), torch.randn(5, generator=g)
    gamma, beta = 1 + 0.2 * torch.randn(5, generator=g), 0.1 * torch.randn(5, generator=g)
    rm, rv = 0.2 * torch.randn(5, generator=g), 1 + 0.3 * torch.rand(5, generator=g)
    ref = F.batch_norm(F.conv2d(x, w, b, padding=1), rm, rv, gamma, beta, False, 0.1, 1e-5)
    s = gamma / torch.sqrt(rv + 1e-5)
    t = beta - rm * s
    out = F.conv2d(x, w * s.view(-1, 1, 1, 1), b * s + t, padding=1)
    assert (out - ref).abs().max().item() < 1e-4


def test_two_key_cross_attention_is_affine_in_one_gate_per_head_with_gram_layernorm():
    """The rewrite behind csrc/kernels.cu::ca_tables_* + ca_fused.cu (reference CrossAttention U:481-559): with exactly two keys
    (null, real) the softmax is one sigmoid gate per head, to_out(o) = u0 + sum_h gate_h * u_h with per-FRAME vectors u, and the
    output LayerNorm's variance is a 9x9 quadratic form in c = [1, gates] over the centred vectors' Gram matrix."""
    from oracle import unet_oracle as O
    g = torch.Generator().manual_seed(4)
    Fr, n, ci, co, H, D = 3, 11, 64, 128, 8, 8
    p = "ca"
    sd = {p + '.norm.g': 1 + 0.2 * torch.randn(ci, generator=g), p + '.to_q.weight': torch.randn(64, ci, generator=g) / 8,
          p + '.to_kv.weight': torch.randn(128, 2 * co, generator=g) / 16, p + '.null_kv': torch.randn(2, D, generator=g),
          p + '.q_scale': 1 + 0.2 * torch.randn(D, generator=g), p + '.k_scale': 1 + 0.2 * torch.randn(D, generator=g),
          p + '.to_out.0.weight': torch.randn(co, 64, generator=g) / 8, p + '.to_out.1.g': 1 + 0.2 * torch.randn(co, generator=g)}
    tok = torch.randn(Fr, n, ci, generator=g)
    ctx = torch.randn(Fr, 2 * co, generator=g)
    ref = O.cross_attention(sd, p, tok, ctx)
    # --- rewritten form
    x = O.token_layernorm(tok, sd[p + '.norm.g'])
    q = (x @ sd[p + '.to_q.weight'].t()).reshape(Fr, n, H, D)
    kv = ctx @ sd[p + '.to_kv.weight'].t()
    k, v = kv[:, :64].reshape(Fr, H, D), kv[:, 64:].reshape(Fr, H, D)
    nk, nv = sd[p + '.null_kv'][0], sd[p + '.null_kv'][1]
    qs, ks = sd[p + '.q_scale'], sd[p + '.k_scale']
    kq = F.normalize(k, dim=-1) * ks * qs                                  # per-frame key with both scales folded  (Fr, H, D)
    nkq = F.normalize(nk, dim=-1) * ks * qs                                # (D,)
    qn = F.normalize(q, dim=-1)
    s_real = 8.0 * torch.einsum('fnhd,fhd->fnh', qn, kq)
    s_null = 8.0 * torch.einsum('fnhd,d->fnh', qn, nkq)
    gate = torch.sigmoid(s_real - s_null)                                  # softmax over {null, real} -> weight of the real key
    Wout = sd[p + '.to_out.0.weight']                                      # (co, 64)
    u0 = Wout @ nv.repeat(H)                                               # (co,)
    uh = torch.einsum('chd,fhd->fhc', Wout.reshape(co, H, D), v - nv)      # (Fr, H, co)
    u = torch.cat([u0.expand(Fr, 1, co), uh], dim=1)                       # (Fr, 9, co)
    uc = u - u.mean(dim=-1, keepdim=True)                                  # centred over channels
    G = torch.einsum('fac,fbc->fab', uc, uc) / co                          # Gram (Fr, 9, 9)
    c = torch.cat([torch.ones(Fr, n, 1), gate], dim=-1)                    # (Fr, n, 9)
    var = torch.einsum('fna,fab,fnb->fn', c, G, c)
    out = torch.einsum('fna,fac->fnc', c, uc) * torch.rsqrt(var + 1e-5).unsqueeze(-1) * sd[p + '.to_out.1.g']
    assert (out - ref).abs().max().item() < 2e-4


def test_layernorm_folds_into_the_following_projection():
    """csrc/unet.cu::pack_linear + the QKV epilogues: W(gamma * (x - mu) * rstd) == rstd * (W' x - mu * rowsum(W')), W' = W diag(gamma)
    (channel LayerNorm without bias, reference U:179-188, 205-213)."""
    g = torch.Generator().manual_seed(5)
    x = torch.randn(37, 64, generator=g) * 3 + 1
    gamma = 1 + 0.2 * torch.randn(64, generator=g)
    Wm = torch.randn(96, 64, generator=g) / 8
    mu = x.mean(-1, keepdim=True)
    rstd = (x.var(-1, unbiased=False, keepdim=True) + 1e-5).rsqrt()
    ref = ((x - mu) * rstd * gamma) @ Wm.t()
    Wp = Wm * gamma
    out = rstd * (x @ Wp.t() - mu * Wp.sum(-1))
    assert (out - ref).abs().max().item() < 1e-4


def test_spatial_linear_attention_context_composes_with_the_out_projection():
    """csrc/sla_fused.cu::sla_merge_kernel: out = to_out(context^T q) == (Wout . blockdiag(context^T)) q + b, one 256 x C matrix
    per frame, so q never needs a separate context product (reference SpatialLinearAttention U:602-627)."""
    from oracle import unet_oracle as O
    g = torch.Generator().manual_seed(6)
    C, H, W_, heads, d = 64, 6, 5, 8, 32
    p = "sla"
    sd = {p + '.norm.gamma': (1 + 0.2 * torch.randn(C, generator=g)).view(1, C, 1, 1, 1),
          p + '.fn.to_qkv.weight': torch.randn(768, C, 1, 1, generator=g) / 8,
          p + '.fn.to_out.weight': torch.randn(C, 256, 1, 1, generator=g) / 16, p + '.fn.to_out.bias': torch.randn(C, generator=g) * 0.05}
    x = torch.randn(2, C, H, W_, generator=g)
    ref = O.spatial_linear_attention(sd, p, x)                             # x + to_out(...)
    xn = O.chan_layernorm(x, sd[p + '.norm.gamma'].view(1, C, 1, 1))
    qkv = F.conv2d(xn, sd[p + '.fn.to_qkv.weight'])
    q, k, v = [t.reshape(2, heads, d, H * W_) for t in qkv.chunk(3, dim=1)]
    q = q.softmax(dim=-2) * d ** -0.5
    k = k.softmax(dim=-1)
    ctx = torch.einsum('bhdn,bhen->bhde', k, v)                            # (b, heads, d, e)
    Wout = sd[p + '.fn.to_out.weight'].view(C, heads, d)                   # columns = (head, e)
    Mf = torch.einsum('che,bhde->bchd', Wout, ctx).reshape(2, C, heads * d)    # per-frame composed matrix (C x 256) acting on q
    out = torch.einsum('bck,bkn->bcn', Mf, q.reshape(2, heads * d, H * W_)) + sd[p + '.fn.to_out.bias'].view(1, C, 1)
    assert (x + out.reshape(2, C, H, W_) - ref).abs().max().item() < 1e-4
