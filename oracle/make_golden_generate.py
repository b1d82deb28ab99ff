"""TEST INFRASTRUCTURE — golden of the whole talking-head generator from the REAL reference `VideoGenerator` methods.

Run in the build container only (needs /root/reference):    python oracle/make_golden_generate.py
Writes tests/golden/generate.npz.  unified_video_generator.py's `process_audio`, `generate_pose_blink` and `generate_final_video`
run UNMODIFIED, on the CPU, on a `VideoGenerator` assembled with __new__ (its __init__ loads 3DDFA, checkpoints and a GPU) from
synthetic weights:
  * transformers' HubertModel with a small stable-layer-norm configuration (hidden size 1024, the width PBnet and the UNet take)
    and a Wav2Vec2FeatureExtractor as `wav2vec2_processor`;
  * the reference PBnet `get_model` for pose and blink with oracle/pbnet_oracle.py's synthetic weights;
  * the reference FlowDiffusion assembled as oracle/make_golden_e2e.py does (3 DDIM steps, 64 x 64);
  * video_config: input_size 64, max_n_frames 8, with 0.5 s of speech (12 frames), so the frame cap is exercised.
The file and codec I/O is replaced in memory: cv2 (cvtColor = channel flip, VideoWriter / imwrite record), soundfile.read (the
test speech), pydub and the 3DDFA imports are stubs; `_convert_wav_to_16k`, `_extract_audio_segment` and `_combine_video_audio`
are no-ops; `Tensor.cuda` is the identity and torch.randn returns oracle.weights.pseudo_normal draws named by call order
(`generate/<case>/randn<i>`: PBnet pose z, blink z, the sampler's start image, one per step but the last).  The portrait is a
97 x 83 PNG, so `Image.open(...).convert("RGB")` and the resize run for real.

Two cases: "init" with init_pose.npy / init_eye_bbox.npy in the cache and a non-zero mean, "fallback" without them (UVG's fallback
branches) and mean 0.  Each stores the HuBERT features, PBnet's raw outputs, dri_pose / dri_blink, the source image the sampler
received (image_tensor / 255.), the sampled grid and conf and the frames the video writer received (flipped back to RGB).
"""
import importlib
import json
import os
import sys
import tempfile
import types
import warnings

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import hubert_oracle as HO    # noqa: E402
from oracle import lfg_oracle as L        # noqa: E402
from oracle import pbnet_oracle as P      # noqa: E402
from oracle import weights as W           # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
TAG = "generate"
IMG_W, IMG_H = 97, 83
INPUT_SIZE, MAX_FRAMES, STEPS = 64, 8, 3
SPEECH_SAMPLES = 8000 + 123                        # int(8123 / 16000 * 25) = 12 frames
# the HuBERT configuration: hubert-large's structure with two layers, 1024 wide as PBnet's and the UNet's audio inputs are
HUBERT = HO.config(num_hidden_layers=2, intermediate_size=1024, conv_dim=[256] * 7, num_conv_pos_embeddings=16)
PB_POSE = P.PbCfg(pos_dim=6, eye_dim=0)            # UVG:81-84's overrides
PB_BLINK = P.PbCfg(pos_dim=0, eye_dim=2)           # UVG:89-92's overrides
INIT_POSE = [[4.0, -6.5, 2.25, 4.6e-04, 58.0, 63.5, 0.0]]
INIT_EYE_BBOX = [[0.27, 0.31, 20.0, 75.0, 12.0, 70.0, 97.0, 83.0]]
CASES = {"init": dict(init=True, mean=[12.0, -7.5, 3.25]), "fallback": dict(init=False, mean=[0.0, 0.0, 0.0])}
VIDEO_CONFIG = dict(input_size=INPUT_SIZE, max_n_frames=MAX_FRAMES, cond_scale=1.0, sampling_step=STEPS, ddim_sampling_eta=1.0,
                    win_width=40)


def portrait():
    """(83, 97, 3) uint8 RGB: a smooth gradient with noise, so the resize has edges and flats to get right"""
    y, x = np.mgrid[0:IMG_H, 0:IMG_W]
    base = np.stack([x * 255.0 / IMG_W, y * 255.0 / IMG_H, (x + y) * 127.0 / (IMG_W + IMG_H)], -1)
    noise = W.uniform01(f"{TAG}/portrait", IMG_H * IMG_W * 3).reshape(IMG_H, IMG_W, 3) * 96.0 - 48.0
    return np.clip(base + noise, 0, 255).astype(np.uint8)


def speech():
    return HO.synth_speech(f"{TAG}/speech", SPEECH_SAMPLES)


def draw(case, i, shape):
    return torch.from_numpy(W.pseudo_normal(f"{TAG}/{case}/randn{i}", tuple(shape)))


def hubert_state_dict():
    return HO.synth_state_dict(HO.schema_of(HUBERT))


def face_sd():
    from oracle.make_golden_e2e import face_sd as f
    return f()


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _install_stubs(record):
    class VideoWriter:
        def __init__(self, *a, **k):
            pass

        def write(self, frame):
            record["writer"].append(np.array(frame))

        def release(self):
            pass

    _stub("cv2", COLOR_RGB2BGR=4, COLOR_RGBA2RGB=1, cvtColor=lambda img, code: np.ascontiguousarray(img[..., ::-1]),
          VideoWriter=VideoWriter, VideoWriter_fourcc=lambda *a: 0, imwrite=lambda path, img: record["imwrite"].append(np.array(img)),
          imread=None)
    _stub("soundfile", read=lambda path: (record["speech"], 16000))
    _stub("pydub", AudioSegment=None)
    _stub("extract_init_states")
    _stub("extract_init_states.FaceBoxes")
    _stub("extract_init_states.FaceBoxes.FaceBoxes_ONNX", FaceBoxes_ONNX=None)
    _stub("extract_init_states.TDDFA_ONNX", TDDFA_ONNX=None)
    _stub("extract_init_states.utils")
    _stub("extract_init_states.utils.pose", get_pose=None)
    _stub("extract_init_states.utils.functions", calculate_eye=None, calculate_bbox=None)


def _flow_diffusion():
    """the reference FlowDiffusion with synthetic weights, assembled as oracle/make_golden_e2e.py does"""
    import yaml
    from oracle.make_golden_e2e import FD_MOD, U_MOD
    FD = importlib.import_module(FD_MOD)
    U = importlib.import_module(U_MOD)
    from LFG.modules.generator import Generator
    with open('/root/reference/config/hdtf128.yaml') as f:
        mp = yaml.safe_load(f)['model_params']
    with open(os.path.join(GOLD, 'state_dict_schema.json')) as f:
        unet_schema = [(n, tuple(s)) for n, s in json.load(f)['entries']]
    fd = FD.FlowDiffusion.__new__(FD.FlowDiffusion)
    nn.Module.__init__(fd)
    fd.use_residual_flow, fd.pose_dim, fd.is_train = False, 6, False
    fd.generator = Generator(num_regions=mp['num_regions'], num_channels=mp['num_channels'], revert_axis_swap=mp['revert_axis_swap'],
                             **mp['generator_params']).eval()
    fd.generator.load_state_dict(W.lfg_synth_state_dict(L.state_dict_schema()), strict=False)
    fd.unet = U.DynamicNfUnet3D(dim=64, cond_dim=1024 + 6 + 2, cond_aud=1024, cond_pose=6, cond_eye=2, num_frames=40, channels=3 + 256 + 16,
                                out_grid_dim=2, out_conf_dim=1, dim_mults=(1, 2, 4, 8), use_hubert_audio_cond=True, learn_null_cond=False,
                                use_final_activation=False, use_deconv=True, padding_mode="zeros", win_width=40)
    fd.unet.load_state_dict(W.synth_state_dict(unet_schema), strict=True)
    fd.diffusion = U.DynamicNfGaussianDiffusion(denoise_fn=fd.unet, num_frames=40, image_size=32, sampling_timesteps=STEPS, timesteps=1000,
                                                loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0)
    fd.face_loc_emb = FD.Face_loc_Encoder()
    fd.face_loc_emb.load_state_dict(face_sd(), strict=True)
    return fd.eval()


def _pbnet(get_model, cfg):
    import contextlib
    import io
    params = dict(cfg.parameters(), device="cpu")
    with contextlib.redirect_stdout(io.StringIO()):
        model = get_model(params).eval()
    model.load_state_dict(P.synth_state_dict([(k, tuple(v.shape)) for k, v in model.state_dict().items()]), strict=True)
    return model


def main():
    import contextlib
    import io
    from PIL import Image
    from transformers import HubertConfig, HubertModel, Wav2Vec2FeatureExtractor
    sys.path.insert(0, os.path.join(HERE, 'shims'))
    sys.path.insert(0, '/root/reference/PBnet')
    sys.path.insert(0, '/root/reference')
    warnings.filterwarnings("ignore")
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    record = {"speech": speech().astype(np.float64), "writer": [], "imwrite": []}
    _install_stubs(record)
    UVG = importlib.import_module("unified_video_generator")
    from src.models.get_model import get_model

    hub = HubertModel(HubertConfig(**HUBERT, attn_implementation="eager")).eval()
    hub.load_state_dict(hubert_state_dict(), strict=True)
    out = {}
    for case, spec in CASES.items():
        tmp = tempfile.mkdtemp()
        cwd = os.getcwd()
        os.chdir(tmp)                                                     # process_audio's temporary file goes to './'
        g = UVG.VideoGenerator.__new__(UVG.VideoGenerator)
        g.audio_path, g.image_path = os.path.join(tmp, "speech.wav"), os.path.join(tmp, "portrait.png")
        g.output_path, g.cache_path = os.path.join(tmp, "out"), os.path.join(tmp, "cache")
        os.makedirs(g.cache_path)
        g.audio_emb_path = os.path.join(g.cache_path, 'target_audio.npy')
        g.device = 'cpu'
        g.wav2vec2_processor = Wav2Vec2FeatureExtractor(feature_size=1, sampling_rate=16000, padding_value=0.0, do_normalize=True,
                                                        return_attention_mask=True)
        g.hubert_model = hub
        g.pose_params = PB_POSE.parameters("cpu")
        g.blink_params = PB_BLINK.parameters("cpu")
        g.max_vals = torch.tensor([90, 90, 90, 1, 720, 1080]).to(torch.float32).reshape(1, 1, 6)      # UVG:95-98
        g.min_vals = torch.tensor([-90, -90, -90, 0, 0, 0]).to(torch.float32).reshape(1, 1, 6)
        g.model_p, g.model_b = _pbnet(get_model, PB_POSE), _pbnet(get_model, PB_BLINK)
        g.video_config = dict(VIDEO_CONFIG, mean=spec["mean"])
        g.video_model = _flow_diffusion()
        g._convert_wav_to_16k = lambda *a: None
        g._extract_audio_segment = lambda *a: None
        g._combine_video_audio = lambda *a: None
        Image.fromarray(portrait()).save(g.image_path)
        if spec["init"]:
            np.save(os.path.join(g.cache_path, 'init_pose.npy'), np.array(INIT_POSE))
            np.save(os.path.join(g.cache_path, 'init_eye_bbox.npy'), np.array(INIT_EYE_BBOX))
        raw, seen = {}, {}

        def wrap_generate(model, key):
            real = model.generate

            def gen(*a, **k):
                with contextlib.redirect_stdout(io.StringIO()):
                    batch = real(*a, **k)
                raw[key] = batch["output"].clone()
                return batch
            model.generate = gen

        wrap_generate(g.model_p, "pose")
        wrap_generate(g.model_b, "blink")
        real_sov = g.video_model.sample_one_video

        def sov(**k):
            seen["source"] = k["sample_img"][0].clone()
            o = real_sov(**k)
            seen.update(grid=o["sample_vid_grid"], conf=o["sample_vid_conf"])
            return o
        g.video_model.sample_one_video = sov
        counter = {"i": 0}

        def injected(*size, **kw):
            shape = size[0] if len(size) == 1 and not isinstance(size[0], int) else size
            t = draw(case, counter["i"], shape)
            counter["i"] += 1
            return t

        real_randn, real_randn_like, real_cuda = torch.randn, torch.randn_like, torch.Tensor.cuda
        torch.randn = injected
        torch.randn_like = lambda t, **kw: injected(tuple(t.shape))
        torch.Tensor.cuda = lambda self, *a, **k: self
        record["writer"].clear()
        try:
            g.process_audio()
            g.generate_pose_blink()
            g.generate_final_video()
        finally:
            torch.randn, torch.randn_like, torch.Tensor.cuda = real_randn, real_randn_like, real_cuda
            os.chdir(cwd)
        assert counter["i"] == 2 + STEPS, counter                      # pose z, blink z, start image, steps but the last
        feats = np.load(g.audio_emb_path)
        frames = np.stack(record["writer"])[..., ::-1]                  # the writer got BGR (UVG:548)
        assert frames.shape == (MAX_FRAMES, INPUT_SIZE, INPUT_SIZE, 3) and feats.shape[0] > MAX_FRAMES, (frames.shape, feats.shape)
        print(f"{case}: features {feats.shape}, frames {frames.shape} mean level {frames.mean():.1f}, "
              f"levels 0 / 255: {(frames == 0).mean():.3f} / {(frames == 255).mean():.3f}")
        out.update({f"{case}/audio_features": feats, f"{case}/pose_raw": raw["pose"].numpy(), f"{case}/blink_raw": raw["blink"].numpy(),
                    f"{case}/dri_pose": np.load(os.path.join(g.cache_path, 'dri_pose.npy')),
                    f"{case}/dri_blink": np.load(os.path.join(g.cache_path, 'dri_blink.npy')),
                    f"{case}/source": seen["source"].numpy(), f"{case}/grid": seen["grid"].numpy(), f"{case}/conf": seen["conf"].numpy(),
                    f"{case}/frames": np.ascontiguousarray(frames), f"{case}/mean": np.array(spec["mean"])})
    np.savez_compressed(os.path.join(GOLD, "generate.npz"), **out)
    print("wrote", os.path.join(GOLD, "generate.npz"), os.path.getsize(os.path.join(GOLD, "generate.npz")), "bytes")


if __name__ == "__main__":
    main()
