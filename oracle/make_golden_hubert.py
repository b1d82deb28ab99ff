"""TEST INFRASTRUCTURE — generate tests/golden/hubert.npz and hubert_schema.json by running the REAL transformers HubertModel.

Run where transformers is installed (5.5 when these goldens were made):    python oracle/make_golden_hubert.py
Builds each case's HubertModel (eager attention, float64, eval), loads the deterministic synthetic weights of
oracle/hubert_oracle.py with a strict load_state_dict, and runs it on the regenerated inputs: the "model" cases call it on input
values; the "features" case runs the generator's own audio steps (Wav2Vec2FeatureExtractor, the 20 s segments, the length
fix-up, scipy's interp1d).  It checks the float64 oracle against every output and stores, per case, the output (channels
[::step] for the large cases, to keep the file near 1 MB) and the mean |h| of every encoder boundary (after the positional conv
and after each layer) per frame.  The inputs are regenerated from their seeds by the tests.
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
warnings.filterwarnings("ignore")

from oracle import hubert_oracle as O   # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def reference_model(c, sd):
    from transformers import HubertConfig, HubertModel
    model = HubertModel(HubertConfig(**c, attn_implementation="eager")).eval().double()
    model.load_state_dict({k: v.double() for k, v in sd.items()}, strict=True)
    return model


def reference_features(model, speech):
    """unified_video_generator.py:226-242 and 450-501, the model in float64"""
    from scipy.interpolate import interp1d
    from transformers import Wav2Vec2FeatureExtractor
    processor = Wav2Vec2FeatureExtractor(feature_size=1, sampling_rate=16000, padding_value=0.0, do_normalize=True,
                                         return_attention_mask=True)
    num_frames = int((speech.shape[0] / 16000) * 25)
    x = processor(speech, return_tensors="pt", sampling_rate=16000).input_values.double()
    kernel, stride = 400, 320
    clip_length = stride * 1000
    num_iter = x.shape[1] // clip_length
    expected_T = (x.shape[1] - (kernel - stride)) // stride
    res = []
    for i in range(num_iter):
        start = clip_length * i
        res.append(model(x[:, start:start + clip_length - stride + kernel]).last_hidden_state[0])
    tail = x[:, clip_length * num_iter:] if num_iter > 0 else x
    if tail.shape[1] >= kernel:
        res.append(model(tail).last_hidden_state[0])
    ret = torch.cat(res, 0)
    assert abs(ret.shape[0] - expected_T) <= 1
    ret = torch.nn.functional.pad(ret, (0, 0, 0, expected_T - ret.shape[0])) if ret.shape[0] < expected_T else ret[:expected_T]
    h = ret.numpy()
    return interp1d(np.arange(h.shape[0]), h, kind="linear", axis=0)(np.linspace(0, h.shape[0] - 1, num_frames)).astype(np.float32)


def boundary_absmeans(model, x):
    taps = []
    hooks = [model.encoder.pos_conv_embed.register_forward_hook(lambda m, i, o: taps.append((i[0] + o).abs().mean(-1)))]
    hooks += [layer.register_forward_hook(lambda m, i, o: taps.append(o[0].abs().mean(-1))) for layer in model.encoder.layers]
    model(x)
    for hk in hooks:
        hk.remove()
    return torch.stack(taps).float().numpy()


def main():
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    out, schema = {}, {}
    with torch.no_grad():
        for cname, c in O.CONFIGS.items():
            sch = O.schema_of(c)
            ref_sch = [(k, tuple(v.shape)) for k, v in reference_model(c, O.synth_state_dict(sch)).state_dict().items()]
            assert ref_sch == sch, f"{cname}: schema_of differs from transformers' state_dict"
            schema[cname] = [[k, list(s)] for k, s in sch]
        for name, (cname, kind, lengths) in O.CASES.items():
            c = O.CONFIGS[cname]
            sch = O.schema_of(c)
            sd = O.synth_state_dict(sch)
            model = reference_model(c, sd)
            step = O.PROBE_STEP.get(name, 1)
            if kind == "model":
                x = O.synth_input_values(name, lengths).double()
                ref = model(x).last_hidden_state
                mine = O.forward(sd, c, x)
                out[f"{name}/absmean"] = boundary_absmeans(model, x)
            else:
                speech = O.synth_speech(name, lengths[0])
                ref = torch.from_numpy(reference_features(model, speech))
                mine = O.features(lambda v: O.forward(sd, c, v.double()), speech)
            r = ((mine.double() - ref.double()).abs() / (1e-4 + 1e-3 * ref.double().abs())).max().item()
            print(f"{name}: out {tuple(ref.shape)}  |ref| max {ref.abs().max().item():.3f}  oracle / tolerance {r:.2e}")
            assert r < 0.01, name
            out[f"{name}/out"] = ref[..., ::step].float().numpy()
    np.savez_compressed(os.path.join(GOLD, "hubert.npz"), **out)
    with open(os.path.join(GOLD, "hubert_schema.json"), "w") as f:
        json.dump(schema, f, indent=0)
    print("wrote", os.path.join(GOLD, "hubert.npz"), os.path.getsize(os.path.join(GOLD, "hubert.npz")), "bytes")


if __name__ == "__main__":
    main()
