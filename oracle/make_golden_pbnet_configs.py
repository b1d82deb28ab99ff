"""TEST INFRASTRUCTURE — generate tests/golden/pbnet_configs.npz and pbnet_configs_schema.json by running the REAL reference PBnet
at the configurations of oracle/pbnet_oracle.CONFIG_CASES: d_model 32, 96 and 256, 2 to 32 heads, 1 to 4 layers, ff 1 to 2048,
pose_dim 1 to 32, audio and latent widths other than DAWN's.

Run in the build container only (needs /root/reference):    python oracle/make_golden_pbnet_configs.py
As oracle/make_golden_pbnet.py: the unmodified `get_model` (through the shims under oracle/shims), the deterministic synthetic
weights of oracle/pbnet_oracle.py loaded strictly, `.eval().generate(...)` on the CPU with an explicit z, the float64 oracle
checked against it, and the outputs (inputs are regenerated from their seeds) and state_dict schemas stored.  np.savez writes
no timestamps: re-running gives a byte-identical file.
"""
import contextlib
import io
import json
import os

import numpy as np
import torch

from make_golden_pbnet import GOLD, reference_generate   # noqa: E402  (puts the repository, shims and reference on sys.path)
from oracle import pbnet_oracle as P   # noqa: E402


def main():
    from src.models.get_model import get_model
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    out, schema = {}, {}
    for name, (cfg, lengths) in P.CONFIG_CASES.items():
        with contextlib.redirect_stdout(io.StringIO()):
            model = get_model(cfg.parameters()).eval()
        sch = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
        schema[name] = [[k, list(s)] for k, s in sch]
        sd = P.synth_state_dict(sch)
        model.load_state_dict(sd, strict=True)
        pose, audio, z, lens = P.synth_inputs(name, cfg, lengths)
        ref = reference_generate(model, pose, audio, lens, z)["output"]
        mine = P.decoder_forward(sd, cfg, pose, audio, z, lens)
        m = ((mine - ref.double()).abs() / (1e-4 + 1e-3 * ref.double().abs())).max().item()
        print(f"{name}: {cfg.archiname} d_model {cfg.pose_latent_dim} heads {cfg.num_heads} layers {cfg.num_layers} ff {cfg.ff_size} "
              f"audio {cfg.audio_dim} latent {cfg.latent_dim} out {cfg.out_dim} lengths {lengths}: |out| max {ref.abs().max():.3f}; "
              f"oracle vs reference {m:.3g} x tol")
        assert m < 0.05, m
        out[f"{name}/output"] = ref.numpy()
    np.savez(os.path.join(GOLD, "pbnet_configs.npz"), **out)
    with open(os.path.join(GOLD, "pbnet_configs_schema.json"), "w") as f:
        json.dump(schema, f, indent=0)


if __name__ == "__main__":
    main()
