"""TEST INFRASTRUCTURE — generate tests/golden/pbnet.npz and pbnet_schema.json by running the REAL reference PBnet.

Run in the build container only (needs /root/reference):    python oracle/make_golden_pbnet.py
Builds each case's model with the unmodified `get_model` (PBnet/src/models/get_model.py; shims for the un-installed
einops_exts / rotary_embedding_torch under oracle/shims), loads the deterministic synthetic weights of oracle/pbnet_oracle.py
with a strict load_state_dict, runs `.eval().generate(...)` on the CPU with an explicit z, checks oracle/pbnet_oracle.py against
it, and stores the outputs (the inputs are regenerated from their seeds by the tests), the reference's relative-position
buckets of every j - i up to F = 2000, and each configuration's state_dict schema.
"""
import contextlib
import io
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, 'shims'))
sys.path.insert(0, '/root/reference/PBnet')
warnings.filterwarnings("ignore")

from oracle import pbnet_oracle as P   # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
BUCKET_F = 2000


def reference_generate(model, pose, audio, lengths, z):
    """CAE.generate (cae.py:112-172) with its torch.randn replaced by the given z"""
    real = torch.randn
    torch.randn = lambda *a, **k: z.clone()
    try:
        with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):      # RelativePositionBias prints 'eval!' per call
            return model.generate(pose, audio, lengths, fact=1)
    finally:
        torch.randn = real


def main():
    from src.models.get_model import get_model
    from src.models.architectures.transformerreemb5 import RelativePositionBias
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    out, schema = {}, {}
    for name, (cfg, lengths) in P.CASES.items():
        with contextlib.redirect_stdout(io.StringIO()):
            model = get_model(cfg.parameters()).eval()
        sch = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
        schema[name] = [[k, list(s)] for k, s in sch]
        sd = P.synth_state_dict(sch)
        model.load_state_dict(sd, strict=True)
        pose, audio, z, lens = P.synth_inputs(name, cfg, lengths)
        batch = reference_generate(model, pose, audio, lens, z)
        ref = batch["output"]
        mine = P.decoder_forward(sd, cfg, pose, audio, z, lens)
        m = ((mine - ref.double()).abs() / (1e-4 + 1e-3 * ref.double().abs())).max().item()
        print(f"{name}: {cfg.archiname} pos {cfg.pos_dim} eye {cfg.eye_dim} lengths {lengths}: output {tuple(ref.shape)}, "
              f"|out| max {ref.abs().max():.3f}; oracle vs reference {m:.3g} x tol")
        assert m < 0.05, m
        out[f"{name}/output"] = ref.numpy()
        if "out_eye" in batch:
            assert torch.equal(batch["out_pose"], ref[:, :, :6]) and torch.equal(batch["out_eye"], ref[:, :, 6:])
    rel = torch.arange(-(BUCKET_F - 1), BUCKET_F)
    out["bucket_2000"] = RelativePositionBias._relative_position_bucket(rel, num_buckets=128, max_distance=128).numpy().astype(np.int16)
    # np.savez (uncompressed) writes no timestamps: the file is byte-reproducible
    np.savez(os.path.join(GOLD, "pbnet.npz"), **out)
    with open(os.path.join(GOLD, "pbnet_schema.json"), "w") as f:
        json.dump(schema, f, indent=0)


if __name__ == "__main__":
    main()
