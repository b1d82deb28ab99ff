"""GPU: the talking-head generator (dawn_pytorch_b200/generate.py) and its two device stages.

* dawn_portrait_resize equals PIL's Image.resize(BILINEAR) bit for bit over the CPU test's size sweep, and its fp32 source equals
  ToTensor / * 255 / / 255 of PIL's result as torch computes them on the host;
* dawn_lfg_decode_sample_rgb8 equals UVG:544-548's numpy conversion of dawn_lfg_decode_sample's fp32 prediction on the same
  handle and sample, exactly, with zero and non-zero mean and values driven past the clip on both sides;
* the whole call against the golden of the reference's own generator methods (oracle/make_golden_generate.py), with and without
  initial states, stage by stage: audio features and drive pose / blink at the north-star tolerance of their modules' tests,
  the source image bit for bit, the sampled grid and conf within 2e-4 as the sample_one_video golden test, the frames within one
  gray level everywhere and equal in at least 99 % of the values;
* use_graph=True and False give frames within one level; two seeded calls, and from_release on a synthetic release tree against
  the modules constructed directly, give the same audio features, pose, blink and source, and frames within one level (the UNet's
  GroupNorm statistics are summed with atomics).
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import lfg_oracle as L
from oracle import make_golden_generate as MG
from oracle import pbnet_oracle as P
from oracle import weights as W
from tests.test_generate_cpu import RESIZE_SWEEP, sweep_image

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RTOL, ATOL = 1e-3, 1e-4


def over_tol(a, ref):
    a, ref = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(ref).detach().double().cpu()
    return ((a - ref).abs() / (ATOL + RTOL * ref.abs())).max().item()


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLD, "generate.npz"))


@pytest.mark.parametrize("H0,W0,S", RESIZE_SWEEP)
def test_portrait_resize_equals_pillow(H0, W0, S):
    from PIL import Image
    from torchvision import transforms
    from dawn_pytorch_b200.generate import portrait_resize
    img = sweep_image(H0, W0)
    ref = np.array(Image.fromarray(img).resize((S, S), Image.BILINEAR))
    source, resized = portrait_resize(torch.from_numpy(img).cuda(), S, with_resized=True)
    assert np.array_equal(resized.cpu().numpy(), ref), f"{int((resized.cpu().numpy() != ref).sum())} values differ"
    t = transforms.Compose([transforms.Resize((S, S)), transforms.ToTensor()])(Image.fromarray(img)) * 255
    assert torch.equal(source.cpu(), t / 255.)


def test_portrait_resize_rejects_bad_sizes():
    from dawn_pytorch_b200._lib import DawnError
    from dawn_pytorch_b200.generate import portrait_resize
    with pytest.raises(DawnError, match="8192"):
        portrait_resize(torch.zeros((8193, 4, 3), dtype=torch.uint8, device="cuda"), 64)
    with pytest.raises(DawnError, match="output side"):
        portrait_resize(torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda"), 0)


@pytest.mark.parametrize("mean", [(0.0, 0.0, 0.0), (17.5, -33.25, 64.0), (-300.0, 0.0, 300.0)])
def test_rgb8_decode_equals_numpy_conversion_of_fp32_decode(mean):
    from dawn_pytorch_b200 import LfgGenerator
    g = LfgGenerator(num_channels=3, num_regions=10, block_expansion=64, max_features=512, num_down_blocks=2, num_bottleneck_blocks=6,
                     skips=True).cuda()
    g.load_state_dict(W.lfg_synth_state_dict(L.state_dict_schema()), strict=True)
    F_, S = 5, 64
    src = torch.from_numpy(W.uniform01("generate_gpu/src", 3 * S * S).reshape(1, 3, S, S)).cuda()
    sample = torch.from_numpy(W.symmetric("generate_gpu/sample", (3, F_, S // 4, S // 4), 1.2)).cuda()
    pred = g.decode_sample(src, sample)
    frames = g.decode_sample_rgb8(src, sample, mean)
    assert frames.dtype == torch.uint8 and frames.shape == (F_, S, S, 3)
    ref = []
    for f in range(F_):                                                # UVG:544-547, in numpy, one frame at a time
        frame = pred[f].permute(1, 2, 0).cpu().numpy().copy()
        frame += np.array(mean) / 255.0
        frame = np.clip(frame, 0, 1)
        ref.append((frame * 255).astype(np.uint8))
    ref = np.stack(ref)
    got = frames.cpu().numpy()
    assert np.array_equal(got, ref), f"{int((got != ref).sum())} values differ"
    if mean[0] < -255:
        assert (got[..., 0] == 0).all() and (got[..., 2] == 255).all()
    if mean[1] < 0:
        assert (got == 0).any()


# ------------------------------------------------------------------------------------------------ the whole call
_MODULES = {}


def modules():
    """the package's modules with the golden's synthetic weights (one set per test session)"""
    if not _MODULES:
        from dawn_pytorch_b200 import HubertModel, get_pbnet_model
        from tests.test_e2e_gpu import build_model
        hub = HubertModel(MG.HUBERT).cuda()
        hub.load_state_dict(MG.hubert_state_dict(), strict=True)

        def pbnet(cfg):
            m = get_pbnet_model(cfg.parameters("cuda:0"))
            m.load_state_dict(P.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()]), strict=True)
            return m.eval()
        _MODULES.update(fd=build_model(MG.STEPS), hubert=hub.eval(), pose=pbnet(MG.PB_POSE), blink=pbnet(MG.PB_BLINK))
    return _MODULES


def generator(case):
    from dawn_pytorch_b200 import TalkingHeadGenerator
    m = modules()
    return TalkingHeadGenerator(m["fd"], m["hubert"], m["pose"], m["blink"], dict(MG.VIDEO_CONFIG, mean=MG.CASES[case]["mean"]))


def run(gen, case, portrait, **kw):
    """the call with the reference's random draws injected, in its order: PBnet pose z, blink z, then the sampler's"""
    init = MG.CASES[case]["init"]
    speech = MG.speech().astype(np.float64)                     # soundfile hands the reference float64 samples
    n_all = int(speech.shape[0] / 16000 * 25)
    return gen(portrait, speech, init_pose=np.array(MG.INIT_POSE) if init else None,
               init_eye_bbox=np.array(MG.INIT_EYE_BBOX) if init else None,
               pose_z=MG.draw(case, 0, (n_all, 1, MG.PB_POSE.latent_dim)).cuda(),
               blink_z=MG.draw(case, 1, (n_all, 1, MG.PB_BLINK.latent_dim)).cuda(),
               noise_fn=lambda k, shape: MG.draw(case, k + 3, shape), **kw)


@pytest.fixture(scope="module")
def portrait_png(tmp_path_factory):
    from PIL import Image
    path = tmp_path_factory.mktemp("generate") / "portrait.png"
    Image.fromarray(MG.portrait()).save(path)
    return str(path)


@pytest.mark.parametrize("case", list(MG.CASES))
def test_whole_call_matches_reference_golden(case, golden, portrait_png):
    out = run(generator(case), case, portrait_png)
    torch.cuda.synchronize()
    g = {k.split("/", 1)[1]: golden[k] for k in golden.files if k.startswith(case + "/")}
    assert out["fps"] == 25 and out["num_frames"] == MG.MAX_FRAMES
    r_audio = over_tol(out["audio_features"], g["audio_features"])
    r_pose, r_blink = over_tol(out["drive_pose"], g["dri_pose"]), over_tol(out["drive_blink"], g["dri_blink"])
    lat = out["latent"].cpu()
    d_grid = (lat[:2].unsqueeze(0) - torch.from_numpy(g["grid"])).abs().max().item()
    d_conf = (((lat[2] + 1) * 0.5)[None, None] - torch.from_numpy(g["conf"])).abs().max().item()
    frames = out["frames"].cpu().numpy().astype(np.int32)
    diff = np.abs(frames - g["frames"].astype(np.int32))
    print(f"{case}: audio {r_audio:.3f} x tol, pose {r_pose:.3f}, blink {r_blink:.3f}, grid max|d| {d_grid:.2e}, conf {d_conf:.2e}, "
          f"frames max|d| {diff.max()} level, equal {np.mean(diff == 0):.4f}")
    assert out["audio_features"].shape == g["audio_features"].shape and r_audio <= 1.0
    assert out["drive_pose"].shape == g["dri_pose"].shape and r_pose <= 1.0
    assert out["drive_blink"].shape == g["dri_blink"].shape and r_blink <= 1.0
    assert torch.equal(out["source"].cpu(), torch.from_numpy(g["source"]))
    assert d_grid < 2e-4 and d_conf < 2e-4
    assert out["frames"].dtype == torch.uint8 and frames.shape == g["frames"].shape
    assert diff.max() <= 1 and np.mean(diff == 0) >= 0.99


def test_graph_and_eager_sampling_give_the_same_frames(portrait_png):
    gen = generator("init")
    a = run(gen, "init", portrait_png, use_graph=True)["frames"].int()
    b = run(gen, "init", portrait_png, use_graph=False)["frames"].int()
    assert (a - b).abs().max().item() <= 1


# The UNet accumulates its GroupNorm statistics with atomics, so two runs of the same clip may differ in the last bits of the
# latent and by one level in a few pixels; the stages before it are deterministic.
def assert_same_clip(a, b):
    for k in ("audio_features", "drive_pose", "drive_blink", "source"):
        assert torch.equal(a[k], b[k]), k
    assert (a["latent"] - b["latent"]).abs().max().item() < 1e-4
    assert (a["frames"].int() - b["frames"].int()).abs().max().item() <= 1


def test_seeded_calls_repeat(portrait_png):
    gen = generator("fallback")
    speech = MG.speech()
    assert_same_clip(gen(portrait_png, speech, seed=11), gen(portrait_png, speech, seed=11))


def test_from_release_gives_the_frames_of_direct_construction(tmp_path, portrait_png):
    import yaml
    from safetensors.torch import save_file
    from dawn_pytorch_b200 import TalkingHeadGenerator
    m = modules()
    root = tmp_path
    (root / "config").mkdir()
    (root / "pretrain_models" / "pbnet_seperate" / "pose").mkdir(parents=True)
    (root / "pretrain_models" / "pbnet_seperate" / "blink").mkdir(parents=True)
    (root / "pretrain_models" / "hubert-large-ls960-ft").mkdir(parents=True)
    vc = dict(MG.VIDEO_CONFIG, mean=MG.CASES["init"]["mean"], random_seed=1234,
              model_config=dict(is_train=True, pose_dim=6, config_pth="./config/hdtf128.yaml",
                                ae_pretrained_pth="./pretrain_models/LFG_128_1000ep.pth",
                                diffusion_pretrained_pth="./pretrain_models/DAWN_128.pth"))
    (root / "config" / "DAWN_128.yaml").write_text(yaml.safe_dump(vc))
    gp = dict(block_expansion=64, max_features=512, num_down_blocks=2, num_bottleneck_blocks=6, skips=True,
              pixelwise_flow_predictor_params=None)
    (root / "config" / "hdtf128.yaml").write_text(yaml.safe_dump(
        {"model_params": dict(num_regions=10, num_channels=3, revert_axis_swap=True, generator_params=gp)}))
    torch.save({"generator": W.lfg_synth_state_dict(L.state_dict_schema())}, root / "pretrain_models" / "LFG_128_1000ep.pth")
    torch.save({"diffusion": {k: v.cpu() for k, v in m["fd"].diffusion.state_dict().items()}}, root / "pretrain_models" / "DAWN_128.pth")
    for name, cfg, ckpt in (("pose", MG.PB_POSE, "checkpoint_40000.pth.tar"), ("blink", MG.PB_BLINK, "checkpoint_95000.pth.tar")):
        d = root / "pretrain_models" / "pbnet_seperate" / name
        opt = {k: v for k, v in cfg.parameters().items() if k not in ("device", "audio_dim", "pos_dim", "eye_dim")}
        (d / "opt.yaml").write_text(yaml.safe_dump(opt))
        torch.save({k: v.cpu() for k, v in m[name].state_dict().items()}, d / ckpt)
    hd = root / "pretrain_models" / "hubert-large-ls960-ft"
    (hd / "config.json").write_text(json.dumps(MG.HUBERT))
    save_file({k: v.contiguous() for k, v in MG.hubert_state_dict().items()}, str(hd / "model.safetensors"))

    rel = TalkingHeadGenerator.from_release(str(root), resolution=128, device="cuda")
    assert rel.video_config["input_size"] == MG.INPUT_SIZE and rel.flow_diffusion.diffusion.sampling_timesteps == MG.STEPS
    # face_loc_emb is not in any release checkpoint (it keeps its default init, as in the reference): give both the same
    m["fd"].face_loc_emb.load_state_dict(rel.flow_diffusion.face_loc_emb.state_dict())
    try:
        a = run(rel, "init", portrait_png)
        b = run(generator("init"), "init", portrait_png)
    finally:
        from oracle.make_golden_e2e import face_sd
        m["fd"].face_loc_emb.load_state_dict(face_sd())
    assert_same_clip(a, b)
