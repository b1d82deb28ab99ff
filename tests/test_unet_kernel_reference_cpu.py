"""CPU: the float64 references of tests/unet_kernel_ref.py, which the per-kernel GPU tests hold the UNet's glue kernels to, against
the oracle functions of oracle/unet_oracle.py, which the goldens pin to the real reference; and dawn_test_kernel's refusals, which
happen before any CUDA call and so need no GPU.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from oracle import unet_oracle as O
from tests import fused_ref as FR
from tests import unet_kernel_ref as R

DT = torch.float64


def rnd(shape, seed, scale=1.0, dtype=DT):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=DT) * scale).to(dtype)


def close(name, a, b, tol):
    err = ((a - b).abs().max() / b.abs().max()).item()
    print(f"  {name}: max |ref - oracle| / max |oracle| = {err:.2e}")
    assert err <= tol, f"{name}: {err:.2e} > {tol:.0e}"


def time_freqs(dim):
    half = dim // 2
    return torch.exp(torch.arange(half) * -(math.log(10000) / (half - 1)))


@pytest.mark.parametrize("dim", [64, 128])
def test_sinusoid_against_oracle(dim):
    t = torch.tensor([0, 1, 47, 999])
    emb, bound = R.sinusoid(t, time_freqs(dim))
    want = O.sinusoidal(t, dim).double()                          # fp32 angle, fp32 sin / cos
    assert ((emb - want).abs() <= 2.0 ** -22 * want.abs() + 2.0 ** -24).all()
    assert (bound > 0).all()


def test_time_mlp_against_oracle():
    dim = 64
    t = torch.tensor([47])
    W1, b1, W2, b2 = rnd((256, dim), 1, 0.125), rnd(256, 2, 0.1), rnd((256, 256), 3, 1 / 16), rnd(256, 4, 0.1)
    got, _ = R.time_mlp(t, time_freqs(dim).double(), W1, b1, W2, b2)
    te = O.sinusoidal(t, dim)[0].double()                          # unet_forward U:915, then every consumer's SiLU (U:366-369)
    te = TF.gelu(te @ W1.t() + b1) @ W2.t() + b2
    close("time mlp", got[0], TF.silu(te), 1e-6)


@pytest.mark.parametrize("F,pos0", [(1, 0), (200, 0), (288, 40)])
def test_rotary_against_oracle(F, pos0):
    freqs = (1.0 / (10000 ** (torch.arange(0, 32, 2).float() / 32)))
    tab, _ = R.rotary_table(freqs, pos0 + F, 0)
    tab = tab[pos0:]
    t = rnd((pos0 + F, 32), 5, dtype=torch.float32)
    want = O.rotary(t, freqs)[pos0:].double()                      # interleaved pairs, position arange(n)
    tt = t[pos0:].double().reshape(F, 16, 2)
    c, s = tab[..., 0], tab[..., 1]
    got = torch.stack((tt[..., 0] * c - tt[..., 1] * s, tt[..., 1] * c + tt[..., 0] * s), -1).reshape(F, 32)
    close("rotary", got, want, 1e-5)
    if pos0:                                                        # the frame-sharded table: rows of the global table
        shard, _ = R.rotary_table(freqs, F, pos0)
        assert torch.equal(shard, tab)


@pytest.mark.parametrize("clips,P,Fc", [(1, 12, 3), (3, 6, 2)])
def test_gn_apply_against_oracle(clips, P, Fc):
    C, cpg = 64, 8
    H, W = 2, P // 2
    frames = rnd((Fc * clips, C, H, W), 7) * (1 + torch.arange(Fc * clips, dtype=DT)[:, None, None, None] % clips) + 3
    y = frames.permute(0, 2, 3, 1).reshape(-1, C)                   # rows (f * clips + b) * P + p
    w, b = 1 + 0.2 * rnd(C, 8), rnd(C, 9)
    st, count = R.gn_stats(y, P, clips, cpg)
    got, _ = R.gn_apply(y, st, count, P, clips, cpg, w, b)
    for cl in range(clips):
        want = TF.silu(O.clip_groupnorm(frames[cl::clips], 8, w, b))   # (F, C, H, W) of clip cl
        close(f"gn clip {cl}", got.reshape(Fc, clips, H, W, C)[:, cl], want.permute(0, 2, 3, 1), 1e-12)


def test_rowstats_against_token_layernorm():
    x = rnd((9, 192), 10) + 50
    g = 1 + 0.2 * rnd(192, 11)
    mu, rstd, _, _ = R.rowstats(x)
    close("layernorm", (x - mu[:, None]) * rstd[:, None] * g, O.token_layernorm(x, g), 1e-12)


@pytest.mark.parametrize("co", [64, 256])
def test_ca_tables_against_oracle(co):
    """kq, nkq, G, T of tests/unet_kernel_ref.py through the cross-attention kernels' references reproduce the oracle"""
    Fr, n, ci = 3, 20, 64
    names = ["pose", "aud", "eye"]
    sd, g3, toq, tabs = {}, [], [], []
    for a, nm in enumerate(names):
        p, s = "ca_" + nm, 11 * a + co
        sd.update({p + ".norm.g": 1 + 0.2 * rnd(ci, s), p + ".to_q.weight": rnd((64, ci), s + 1, ci ** -0.5),
                   p + ".to_kv.weight": rnd((128, 2 * co), s + 2, (2 * co) ** -0.5), p + ".null_kv": rnd((2, 8), s + 3),
                   p + ".q_scale": 1 + 0.3 * rnd(8, s + 4), p + ".k_scale": 1 + 0.3 * rnd(8, s + 5),
                   p + ".to_out.0.weight": rnd((co, 64), s + 6, 0.125), p + ".to_out.1.g": 1 + 0.2 * rnd(co, s + 7)})
        ctx = rnd((Fr, 2 * co), s + 8)
        kv, _ = R.cond_kv(ctx, sd[p + ".to_kv.weight"])
        t = R.ca_tables(kv, sd[p + ".null_kv"], sd[p + ".q_scale"], sd[p + ".k_scale"], sd[p + ".to_out.0.weight"],
                        sd[p + ".to_out.1.g"])
        tabs.append((t, ctx))
        g3.append(sd[p + ".norm.g"]); toq.append(sd[p + ".to_q.weight"])
    tok = rnd((Fr, n, ci), 99)
    kq = torch.stack([t[0][0].reshape(Fr, 64) for t in tabs], 1)
    nkq = torch.stack([t[0][2] for t in tabs], 0)
    G = torch.stack([t[0][4] for t in tabs], 1)
    T = torch.cat([t[0][6] for t in tabs], 1)
    gates, _ = FR.ca_gates(tok, torch.stack(g3), torch.stack(toq), kq, nkq)
    Wt, _ = FR.ca_rstd(gates, G)
    for a, nm in enumerate(names):
        got = Wt[..., 9 * a:9 * (a + 1)] @ T[:, 9 * a:9 * (a + 1)]
        f32 = {k: v.float() for k, v in sd.items() if k.startswith("ca_" + nm)}
        want = O.cross_attention(f32, "ca_" + nm, tok.float(), tabs[a][1].float())
        close(f"cross attention {nm}", got, want.double(), 1e-5)


def test_cond_rows_follow_clip_order():
    """table frame f * clips + b reads cond row b * (F / clips) + f (the clips' frames back to back)"""
    assert R.table_rows(6, 3).tolist() == [0, 2, 4, 1, 3, 5]
    assert R.table_rows(5, 1).tolist() == [0, 1, 2, 3, 4]


@pytest.mark.parametrize("k", [3, 5, 7])
def test_init_conv_linearity(k):
    """the hoisted init conv: the full k x k conv over 275 frame-invariant channels equals map + conv of the 3 noisy channels,
    with the map the sum of the k row convs over fea_shift's copies plus the bias"""
    clips, F, H, W, Co = 2, 2, 5, 7, 16
    w = rnd((Co, 275, k, k), k, 0.05)
    bias = rnd(Co, k + 1)
    xt = rnd((clips, 3, F, H, W), 2)
    fea = rnd((clips, 272, H, W), 3)
    want = torch.stack([TF.conv2d(torch.cat((xt[b].permute(1, 0, 2, 3), fea[b][None].expand(F, 272, H, W)), 1), w, bias,
                                  padding=k // 2) for b in range(clips)], 1)                  # (F, clips, Co, H, W)
    copies = R.fea_shift(fea, k, 272, 0).reshape(k, clips, H, W, 272).permute(0, 1, 4, 2, 3)
    part = torch.stack([TF.conv2d(copies[s], w[:, 3:, s:s + 1, :], padding=(0, k // 2)) for s in range(k)])
    mp = (part.sum(0) + bias[None, :, None, None]).permute(0, 2, 3, 1)                       # (clips, H, W, Co)
    w3 = w[:, :3].permute(2, 3, 1, 0).reshape(k * k * 3, Co)                                 # [(ky k + kx) 3 + c][Co]
    got, bound = R.init_conv_x3(xt, w3, mp, k)
    close("init conv", got, want.permute(0, 1, 3, 4, 2).reshape(F * clips, H * W, Co), 1e-12)
    assert (bound > 0).all()


def test_heads_layout():
    clips, F, HW, C = 3, 2, 5, 8
    hf, ho = rnd((F * clips * HW, C), 1), rnd((F * clips * HW, C), 2)
    Wf, bf, Wo, bo = rnd((2, C), 3), rnd(2, 4), rnd((1, C), 5), rnd(1, 6)
    got, _ = R.heads_out(hf, ho, clips, HW, Wf, bf, Wo, bo)
    for b in range(clips):
        rows = torch.cat([torch.arange((f * clips + b) * HW, (f * clips + b + 1) * HW) for f in range(F)])
        want = torch.cat((hf[rows] @ Wf.t() + bf, ho[rows] @ Wo.t() + bo), 1).t().reshape(3, F, HW)
        assert torch.allclose(got[b], want, rtol=0, atol=1e-12)


def test_split_restatement():
    x = np.concatenate([np.random.default_rng(0).standard_normal(1000).astype(np.float32),
                        np.array([0.0, -0.0, 1e-40, 65504.0, 1 + 2 ** -11], dtype=np.float32)])
    hi, lo = R.split_f16x2_rn(x)
    h, l = hi.view(np.float16).astype(np.float64), lo.view(np.float16).astype(np.float64)
    ok = (np.abs(x) < 60000) & (np.abs(x) >= 2.0 ** -14)             # fp16 normal range
    assert np.all(np.abs(h - x)[ok] <= 2.0 ** -11 * np.abs(x[ok]))
    assert np.all(np.abs(h + l - x)[ok] <= 2.0 ** -22 * np.abs(x[ok]) + 2.0 ** -25)
    assert h[-3] == 0 and l[-3] == 0                                 # far below fp16's range both pieces flush to zero
    assert h[-1] == 1 + 2 ** -10                                     # the tie rounds up on the bit pattern


# ------------------------------------------------------------------------------------------------------------------ refusals
FAKE = 0x10000                                                      # never dereferenced: every case below is refused first


def _run(**kw):
    from dawn_pytorch_b200 import _lib as L
    c = L.DawnKernelCase()
    for k, v in kw.items():
        setattr(c, k, v)
    rc = L.lib.dawn_test_kernel(ctypes.byref(c), None)
    return rc, L.lib.dawn_last_error().decode()


REFUSED = [
    ("rowstats C 2052", dict(kernel=0, x=FAKE, out=FAKE, M=8, C=2052, ld=2052)),
    ("rowstats C % 4", dict(kernel=0, x=FAKE, out=FAKE, M=8, C=66, ld=68)),
    ("rowstats ld % 4", dict(kernel=0, x=FAKE, out=FAKE, M=8, C=64, ld=66)),
    ("gn_apply 7 groups", dict(kernel=1, y=FAKE, stats=FAKE, w=FAKE, b=FAKE, out=FAKE, M=8, P=4, clips=1, C=56, cpg=8, ldy=56,
                               ldo=56, count=1.0)),
    ("gn_apply 17 clips", dict(kernel=1, y=FAKE, stats=FAKE, w=FAKE, b=FAKE, out=FAKE, M=8, P=4, clips=17, C=64, cpg=8, ldy=64,
                               ldo=64, count=1.0)),
    ("cond F % clips", dict(kernel=2, x=FAKE, F=23, clips=2, ndesc=1, cond_ld=1032)),
    ("cond no descriptors", dict(kernel=2, x=FAKE, F=23, clips=1, ndesc=0, cond_ld=1032)),
    ("time_mlp odd dim", dict(kernel=3, t=FAKE, freqs=FAKE, w=FAKE, b=FAKE, w2=FAKE, b2=FAKE, out=FAKE, dim=63, clips=1)),
    ("time_mlp t_stride 2", dict(kernel=3, t=FAKE, freqs=FAKE, w=FAKE, b=FAKE, w2=FAKE, b2=FAKE, out=FAKE, dim=64, clips=1,
                                 t_stride=2)),
    ("ncf Cpad", dict(kernel=7, x=FAKE, out=FAKE, C=275, F=1, P=4, Cpad=277, c0=3, clips=1)),
    ("init conv even k", dict(kernel=11, x=FAKE, w=FAKE, map=FAKE, out=FAKE, F=1, H=4, W=4, clips=1, k=4, C=64, ldo=128,
                              clip_stride=48)),
    ("init conv k 9 Co 128", dict(kernel=11, x=FAKE, w=FAKE, map=FAKE, out=FAKE, F=1, H=4, W=4, clips=1, k=9, C=128, ldo=256,
                                  clip_stride=48)),
    ("heads M % clips", dict(kernel=12, x=FAKE, y=FAKE, w=FAKE, b=FAKE, w2=FAKE, b2=FAKE, out=FAKE, C=64, M=10, P=4, clips=2,
                             ng=2, nc=1)),
    ("unknown kernel", dict(kernel=99)),
]


@pytest.mark.parametrize("name,kw", REFUSED, ids=[r[0] for r in REFUSED])
def test_refusals_without_gpu(name, kw):
    rc, msg = _run(**kw)
    assert rc == -1 and msg.startswith("dawn_test_kernel: "), (rc, msg)


def test_missing_pointer_refused():
    rc, msg = _run(kernel=0, M=8, C=64, ld=64)
    assert rc == -1 and "missing pointer" in msg
