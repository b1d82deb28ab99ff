"""CPU: the UNet's upconv variant (Upsample(use_deconv=False), U:165-172) and UNets without spatial linear attention.

At every configuration of tests/upconv_cases.py the module's state_dict schema is the reference's, the oracle restatement
matches the reference's goldens (oracle/make_golden_upconv.py) and the library accepts the configuration; unknown options are
refused.  The last test checks, in float64, the identity the library's upconv rests on: nearest x2 followed by a 3x3 conv with
a one-pixel pad in any of nn.Conv3d's padding modes is four parity-class 2x2 convs on the low-resolution grid whose taps are
sums of the 3x3 taps, reading the low-resolution grid at zero-outside (zeros), clamped (reflect, replicate) or wrapped
(circular) indices."""
import pytest
import torch
import torch.nn.functional as TF

from oracle import weights as W
from tests import upconv_cases as UC
from tests.test_configs_cpu import create


def test_report_lists_every_case():
    assert tuple(UC.report()) == tuple(sorted(UC.TAGS))
    g = UC.golden()
    assert {f"{k}/{t}" for t in UC.TAGS for k in ("eps", "taps", "shapes", "absmean", "probes")} <= set(g.files)
    modes = {UC.ctor(t)["padding_mode"] for t in UC.TAGS if not UC.ctor(t).get("use_deconv", True)}
    assert modes == set(UC.MODES)


@pytest.mark.parametrize("tag", UC.TAGS)
def test_state_dict_schema_equals_reference(tag):
    sch, rep = UC.schema(tag), UC.report(tag)
    assert (len(sch), UC.schema_digest(sch)) == (rep["schema_entries"], rep["schema_digest"])


@pytest.mark.parametrize("tag", UC.TAGS)
def test_oracle_matches_reference(tag):
    rep, g = UC.report(tag), UC.golden()
    x, t, cond, _, _ = UC.clip(tag)
    taps = {}
    out = UC.oracle(tag, x, t, cond, taps=taps)
    ref = torch.from_numpy(g[f"eps/{tag}"])
    assert out.shape == ref.shape
    r = UC.over_tol(out, ref)
    print(f"{tag}: eps {r:.4f} x tol")
    assert r <= 0.5
    gt = UC.golden_taps(tag)
    assert set(taps) == set(gt)
    for name, (shape, absmean, probes) in gt.items():
        flat = taps[name].reshape(-1)
        assert list(taps[name].shape) == shape, name
        idx = W.probe_indices(f"{tag}/{name}", flat.numel(), 64)
        assert UC.over_tol(flat[idx], torch.from_numpy(probes)) <= 0.5, name
        assert abs(float(flat.abs().mean()) - absmean) < 1e-4 * max(1.0, absmean), name


def test_oracle_defaults_are_the_unet_oracle():
    """oracle/upconv_oracle.py with every option at its default computes oracle/unet_oracle.py's forward, tap for tap"""
    from oracle import unet_oracle as O
    from oracle import upconv_oracle as UO
    from tests import gpu_common as G
    x, t, cond, _, _ = G.clip("upconv_defaults", 3, 8, 8, 321)
    taps_a, taps_b = {}, {}
    with torch.no_grad():
        a = O.unet_forward(G.synth_sd(), O.UnetCfg(), x, t, cond, taps=taps_a)
        b = UO.unet_forward(G.synth_sd(), UO.UpconvCfg(), x, t, cond, taps=taps_b)
    assert torch.equal(a, b) and list(taps_a) == list(taps_b)
    assert all(torch.equal(taps_a[k], taps_b[k]) for k in taps_a)


def test_cases_have_the_structure_they_are_for():
    sh = {t: dict(UC.schema(t)) for t in UC.TAGS}
    assert sh["up_reflect"]["ups.0.4.1.weight"] == [256, 256, 1, 3, 3] and "ups.0.4.weight" not in sh["up_reflect"]
    assert sh["deconv_nosla"]["ups.0.4.weight"] == [256, 256, 1, 4, 4]
    for t in ("upconv_nosla", "deconv_nosla"):
        assert not any(".2.fn." in k and (k.startswith("downs.") or k.startswith("ups.")) for k in sh[t]), t
        assert "mid_spatial_attn.fn.norm.gamma" in sh[t]
    assert UC.golden_taps("rect_reflect")["mid_block1"][0][-2:] == [1, 2]          # deepest level 1 x 2
    assert "ups.0.2" not in UC.golden_taps("upconv_nosla") and "ups.0.2" in UC.golden_taps("up_reflect")


@pytest.mark.parametrize("tag", UC.TAGS)
def test_create_accepts_case(tag):
    from dawn_pytorch_b200 import DynamicNfUnet3D
    cfg = DynamicNfUnet3D(**UC.ctor(tag))._cfg
    kw = UC.ctor(tag)
    assert cfg.upconv == (0 if kw.get("use_deconv", True) else 1)
    assert cfg.no_sla == (0 if kw.get("use_sparse_linear_attn", True) else 1)
    rc, err = create(cfg)
    assert rc == 0, err


@pytest.mark.parametrize("kw,msg", [
    (dict(upconv=2), "upconv must be"),
    (dict(upconv=-1), "upconv must be"),
    (dict(upconv=1, pad_mode=4), "pad_mode must be"),
    (dict(upconv=1, pad_mode=-1), "pad_mode must be"),
    (dict(upconv=0, pad_mode=1), "upconv variant only"),
    (dict(no_sla=2), "no_sla must be"),
])
def test_create_refuses_unknown_values(kw, msg):
    from dawn_pytorch_b200 import DynamicNfUnet3D
    cfg = DynamicNfUnet3D(**UC.ctor("up_zeros"))._cfg
    for k, v in kw.items():
        setattr(cfg, k, v)
    rc, err = create(cfg)
    assert rc == -1 and msg in err, err


def test_constructor_refuses_unknown_padding_and_learned_null_cond():
    from dawn_pytorch_b200 import DynamicNfUnet3D
    kw = UC.ctor("up_zeros")
    with pytest.raises(ValueError, match="padding_mode"):
        DynamicNfUnet3D(**{**kw, "padding_mode": "mirror"})
    with pytest.raises(NotImplementedError, match="learn_null_cond"):
        DynamicNfUnet3D(**{**kw, "learn_null_cond": True})
    for mode, code in zip(UC.MODES, range(4)):
        assert DynamicNfUnet3D(**{**kw, "padding_mode": mode})._cfg.pad_mode == code


# ------------------------------------------------------------------------------------------------ the identity (float64)
OFF = ((-1, 0), (0, 1))                           # [parity][tap] -> low-resolution offset
COVERS = (((0,), (1, 2)), ((0, 1), (2,)))         # [parity][tap] -> 3x3 kernel indices the tap sums


def fold(w):
    """(co, ci, 3, 3) -> {(py, px): (co, ci, 2, 2)} class weights"""
    out = {}
    for py in range(2):
        for px in range(2):
            c = torch.zeros(w.shape[:2] + (2, 2), dtype=w.dtype)
            for ty in range(2):
                for tx in range(2):
                    c[:, :, ty, tx] = sum(w[:, :, ky, kx] for ky in COVERS[py][ty] for kx in COVERS[px][tx])
            out[py, px] = c
    return out


def lowres_index(i, n, mode):
    """low-resolution index read at i in [-1, n], or None (zero)"""
    if 0 <= i < n:
        return i
    if mode == "zeros":
        return None
    if mode == "circular":
        return i % n
    return min(max(i, 0), n - 1)                  # reflect and replicate: clamp


def upconv_by_classes(x, w, b, mode):
    N, _, H, Wd = x.shape
    out = torch.zeros(N, w.shape[0], 2 * H, 2 * Wd, dtype=x.dtype)
    cls = fold(w)
    for (py, px), c in cls.items():
        acc = b.reshape(1, -1, 1, 1).expand(N, -1, H, Wd).clone()
        for ty in range(2):
            rows = [lowres_index(y + OFF[py][ty], H, mode) for y in range(H)]
            for tx in range(2):
                cols = [lowres_index(j + OFF[px][tx], Wd, mode) for j in range(Wd)]
                g = torch.zeros(N, x.shape[1], H, Wd, dtype=x.dtype)
                for y, sy in enumerate(rows):
                    for j, sx in enumerate(cols):
                        if sy is not None and sx is not None:
                            g[:, :, y, j] = x[:, :, sy, sx]
                acc = acc + torch.einsum("oi,nihw->nohw", c[:, :, ty, tx], g)
        out[:, :, py::2, px::2] = acc
    return out


@pytest.mark.parametrize("mode", UC.MODES)
@pytest.mark.parametrize("H,Wd", [(1, 1), (1, 3), (2, 2), (3, 8), (8, 3), (8, 8)])
def test_class_convs_equal_nearest_upsample_then_padded_conv(mode, H, Wd):
    g = torch.Generator().manual_seed(H * 100 + Wd * 7 + UC.MODES.index(mode))
    x = torch.randn(2, 5, H, Wd, generator=g, dtype=torch.float64)
    w = torch.randn(4, 5, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(4, generator=g, dtype=torch.float64)
    u = TF.interpolate(x, scale_factor=2, mode="nearest")
    conv = torch.nn.Conv2d(5, 4, 3, 1, 1, padding_mode=mode).double()
    with torch.no_grad():
        conv.weight.copy_(w)
        conv.bias.copy_(b)
        ref = conv(u)
    got = upconv_by_classes(x, w, b, mode)
    assert (got - ref).abs().max().item() < 1e-12
