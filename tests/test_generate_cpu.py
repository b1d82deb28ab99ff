"""CPU: the talking-head generator's host-side pieces (dawn_pytorch_b200/generate.py).

* a numpy restatement of the fixed-point bilinear resampler dawn_portrait_resize implements equals PIL's Image.resize(BILINEAR)
  bit for bit over a size sweep (down, up, unchanged, one axis, 1 x 1 to 1080 x 1920), and ToTensor / * 255 / / 255 after it
  equals the restatement's fp32 scaling;
* PBnet's initial states and the finishing of its outputs reproduce the golden's dri_pose / dri_blink exactly (golden made by the
  reference's own generate_pose_blink, oracle/make_golden_generate.py), with and without initial states;
* bad inputs raise ValueError naming the reason; from_release names the first missing file of a release tree.
"""
import math
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PREC = 22

# (H0, W0, S): down, up, single pixel, one row, a portrait's odd size, 1080p, unchanged, only the width / height changes
RESIZE_SWEEP = [(1, 1, 64), (1, 300, 64), (83, 97, 64), (1080, 1920, 256), (50, 50, 128), (64, 64, 64), (64, 97, 64),
                (97, 64, 64)]


def axis_coeffs(n_in, n_out):
    """Pillow's bilinear precompute_coeffs + normalize_coeffs_8bpc, written from the algorithm: (xmin, taps, int32 weights)"""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support = 1.0 * fs
    ksize = int(math.ceil(support)) * 2 + 1
    xmin = np.zeros(n_out, np.int64)
    taps = np.zeros(n_out, np.int64)
    k = np.zeros((n_out, ksize), np.int64)
    for i in range(n_out):
        center = (i + 0.5) * scale
        lo = max(int(center - support + 0.5), 0)
        hi = min(int(center + support + 0.5), n_in) - lo
        w = [max(0.0, 1.0 - abs((x + lo - center + 0.5) / fs)) for x in range(hi)]
        ww = sum(w)
        w = [v / ww if ww != 0.0 else v for v in w]
        k[i, :hi] = [int(-0.5 + v * (1 << PREC)) if v < 0 else int(0.5 + v * (1 << PREC)) for v in w]
        xmin[i], taps[i] = lo, hi
    return xmin, taps, k


def _pass(img, n_out, axis):
    """one 8-bit pass along `axis` (1: width, 0: height) of an (H, W, 3) uint8 image"""
    xmin, taps, k = axis_coeffs(img.shape[axis], n_out)
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    acc = np.full((n_out,) + src.shape[1:], 1 << (PREC - 1), np.int64)
    for t in range(k.shape[1]):
        idx = np.minimum(xmin + t, src.shape[0] - 1)
        w = np.where(t < taps, k[:, t], 0)
        acc += src[idx] * w.reshape(-1, *([1] * (src.ndim - 1)))
    return np.moveaxis(np.clip(acc >> PREC, 0, 255).astype(np.uint8), 0, axis)


def resize_reference(img, S):
    """(H0, W0, 3) uint8 -> (S, S, 3) uint8: horizontal then vertical pass, each skipped when its axis keeps its size (a
    horizontal pass over every row equals Pillow's pass over the rows the vertical one reads)"""
    out = img
    if img.shape[1] != S:
        out = _pass(out, S, 1)
    if img.shape[0] != S:
        out = _pass(out, S, 0)
    return out


def source_reference(resized):
    """ToTensor (float(u) / 255), * 255 (UVG:325), / 255. (UVG:372), each rounded to fp32"""
    u = resized.astype(np.float32).transpose(2, 0, 1)
    return ((u / np.float32(255)) * np.float32(255)) / np.float32(255)


def sweep_image(H0, W0):
    rng = np.random.default_rng(H0 * 10007 + W0)
    y, x = np.mgrid[0:H0, 0:W0]
    base = np.stack([x * 255.0 / max(W0, 1), y * 255.0 / max(H0, 1), ((x * 7 + y * 3) % 256).astype(np.float64)], -1)
    return np.clip(base + rng.integers(-60, 61, (H0, W0, 3)), 0, 255).astype(np.uint8)


@pytest.mark.parametrize("H0,W0,S", RESIZE_SWEEP)
def test_fixed_point_resampler_equals_pillow(H0, W0, S):
    from PIL import Image
    from torchvision import transforms
    img = sweep_image(H0, W0)
    ref = np.array(Image.fromarray(img).resize((S, S), Image.BILINEAR))
    mine = resize_reference(img, S)
    assert np.array_equal(mine, ref), f"{int((mine != ref).sum())} of {ref.size} values differ"
    # the source image as UVG:321-325, 372 make it from the PIL image
    t = transforms.Compose([transforms.Resize((S, S)), transforms.ToTensor()])(Image.fromarray(img)) * 255
    assert np.array_equal((t / 255.).numpy(), source_reference(mine))


@pytest.fixture(scope="module")
def golden():
    path = os.path.join(GOLD, "generate.npz")
    return np.load(path)


@pytest.mark.parametrize("case", ["init", "fallback"])
def test_pose_blink_finishing_reproduces_reference(case, golden):
    from dawn_pytorch_b200.generate import finish_pose_blink, pbnet_initial_states
    from oracle.make_golden_generate import INIT_EYE_BBOX, INIT_POSE
    init = case == "init"
    p0, b0 = pbnet_initial_states(np.array(INIT_POSE) if init else None, np.array(INIT_EYE_BBOX) if init else None, "cpu")
    pose, blink = finish_pose_blink(torch.from_numpy(golden[f"{case}/pose_raw"]), torch.from_numpy(golden[f"{case}/blink_raw"]), p0, b0)
    assert pose.dtype == blink.dtype == torch.float32
    assert np.array_equal(pose.numpy(), golden[f"{case}/dri_pose"])
    assert np.array_equal(blink.numpy(), golden[f"{case}/dri_blink"])


def _bare_generator():
    from dawn_pytorch_b200 import TalkingHeadGenerator
    return TalkingHeadGenerator(None, None, None, None, dict(input_size=64, max_n_frames=8, mean=[0, 0, 0], cond_scale=1.0))


@pytest.mark.parametrize("portrait,match", [
    (np.zeros((8, 8, 3), np.float32), "uint8"),
    (np.zeros((8, 8, 4), np.uint8), r"\(H, W, 3\)"),
    (np.zeros((8, 8), np.uint8), r"\(H, W, 3\)"),
])
def test_bad_portrait_raises(portrait, match):
    with pytest.raises(ValueError, match=match):
        _bare_generator()(portrait, np.zeros(16000, np.float32))


def test_short_speech_and_bad_initial_states_raise():
    g, img = _bare_generator(), np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(ValueError, match="receptive field"):
        g(img, np.zeros(399, np.float32))
    with pytest.raises(ValueError, match="no video frame"):
        g(img, np.zeros(500, np.float32))
    with pytest.raises(ValueError, match="init_pose"):
        g(img, np.zeros(16000, np.float32), init_pose=np.zeros((1, 6)), init_eye_bbox=np.zeros((1, 8)))
    with pytest.raises(ValueError, match="init_eye_bbox"):
        g(img, np.zeros(16000, np.float32), init_pose=np.zeros((1, 7)), init_eye_bbox=np.zeros(8))


def test_from_release_names_the_missing_file(tmp_path):
    from dawn_pytorch_b200 import TalkingHeadGenerator
    with pytest.raises(FileNotFoundError, match="DAWN_128.yaml"):
        TalkingHeadGenerator.from_release(str(tmp_path))
    (tmp_path / "config").mkdir()
    (tmp_path / "config" / "DAWN_256.yaml").write_text(
        "input_size: 256\nmax_n_frames: 200\nmean: [0.0, 0.0, 0.0]\nwin_width: 40\nsampling_step: 20\nddim_sampling_eta: 1.0\n"
        "cond_scale: 1.0\nmodel_config:\n  is_train: true\n  pose_dim: 6\n  config_pth: './config/hdtf256.yaml'\n"
        "  ae_pretrained_pth: './pretrain_models/LFG_256_400ep.pth'\n  diffusion_pretrained_pth: './pretrain_models/DAWN_256.pth'\n")
    with pytest.raises(FileNotFoundError, match="hdtf256.yaml"):
        TalkingHeadGenerator.from_release(str(tmp_path), resolution=256)
    (tmp_path / "config" / "hdtf256.yaml").write_text("model_params: {}\n")
    with pytest.raises(FileNotFoundError, match="LFG_256_400ep.pth"):
        TalkingHeadGenerator.from_release(str(tmp_path), resolution=256)
