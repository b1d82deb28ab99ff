"""TEST INFRASTRUCTURE — reference goldens for UNet configurations other than DAWN's own.

Run in the build container only (needs /root/reference; the GPU box never runs this):
    python oracle/make_golden_configs.py
For every row of CONFIGS it builds the unmodified reference DynamicNfUnet3D (with the shims of oracle/shims) with the
constructor keywords of make_golden.CTOR overridden by the row, loads oracle.weights.synth_state_dict over THAT
configuration's own state_dict schema, runs one seeded clip (W.synth_inputs(tag, ...), not stored: it regenerates
exactly) and records
  tests/golden/configs.npz           eps/<tag> (the reference's output), and one row per sub-module boundary (the
                                     forward hooks of make_golden.py) of taps/<tag> (names), shapes/<tag>, absmean/<tag>
                                     and probes/<tag> (64 fixed elements)
  tests/golden/configs_report.json   per tag: ctor keywords, clip, the SHA-256 of the reference's state_dict schema
                                     (schema_digest) and the oracle (oracle/unet_oracle.py with O.UnetCfg(...)) vs
                                     reference margins
The npz is written with fixed zip timestamps, so a rerun reproduces it byte for byte.

The reference accepts every row as listed (cond_pose=7 included: it is the reference's own default), so none had to be
replaced by a nearby configuration.
"""
import hashlib
import importlib
import io
import json
import os
import sys
import time
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import make_golden as MG      # noqa: E402  (puts the shims and the reference on sys.path)
from oracle import unet_oracle as O       # noqa: E402
from oracle import weights as W           # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')

# tag -> (ctor keywords that differ from make_golden.CTOR, (F, h, w, t))
CONFIGS = {
    'dim128':    (dict(dim=128), (8, 16, 16, 500)),
    'mult16_k3': (dict(dim_mults=(1, 2, 4, 8, 16), init_kernel_size=3), (9, 16, 16, 952)),
    'l3_k5':     (dict(dim_mults=(1, 2, 4), init_kernel_size=5), (12, 12, 20, 47)),
    'l2_w1':     (dict(dim_mults=(1, 2), win_width=1), (23, 8, 8, 300)),
    'l6':        (dict(dim_mults=(1, 1, 2, 2, 4, 4)), (5, 32, 32, 999)),
    'io':        (dict(channels=19, cond_aud=256, cond_pose=7, cond_dim=265, out_conf_dim=2), (10, 16, 16, 640)),
    'w120':      (dict(win_width=120), (130, 8, 8, 523)),
    'narrow':    (dict(dim_mults=(2, 1, 2)), (6, 16, 16, 200)),            # a level narrower than the one above it
}
ORACLE_KEYS = ('dim', 'dim_mults', 'channels', 'cond_aud', 'cond_pose', 'cond_eye', 'out_grid_dim', 'out_conf_dim',
               'init_kernel_size', 'win_width')


def ctor(tag):
    return {**MG.CTOR, **CONFIGS[tag][0]}


def oracle_cfg(kw):
    """O.UnetCfg of a constructor-keyword dict."""
    return O.UnetCfg(**{k: kw[k] for k in ORACLE_KEYS if k in kw})


def clip(tag, kw):
    """x (1, channels, F, h, w), t (1,), cond (1, F, cond_dim) of the tag's clip (tests/config_cases.py builds the same)."""
    Fr, h, w, t = CONFIGS[tag][1]
    x_t, fea, cond = W.synth_inputs(tag, Fr, h, w, cond_dim=kw['cond_dim'], fea_ch=kw['channels'] - 3)
    return MG.build_x(x_t, fea), torch.full((1,), t, dtype=torch.long), cond


def schema_digest(schema):
    """SHA-256 of a state_dict schema [(name, shape), ...] in order (tests/config_cases.py computes the same)."""
    return hashlib.sha256(json.dumps([[n, list(sh)] for n, sh in schema], separators=(',', ':')).encode()).hexdigest()


def over_tol(a, ref):
    return ((a - ref).abs() / (1e-4 + 1e-3 * ref.abs())).max().item()


def save_npz_stable(path, arrays):
    """np.savez_compressed with a fixed member order and timestamp: the file depends on the arrays only."""
    with zipfile.ZipFile(path, 'w', compression=zipfile.ZIP_DEFLATED) as zf:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main():
    torch.set_num_threads(os.cpu_count())
    U = importlib.import_module(MG.U_MOD)
    arrays, report = {}, {}
    for tag, (_, (Fr, h, w, t)) in CONFIGS.items():
        kw = ctor(tag)
        net = U.DynamicNfUnet3D(**kw).eval()
        schema = [(k, list(v.shape)) for k, v in net.state_dict().items()]
        sd = W.synth_state_dict(schema)
        net.load_state_dict(sd, strict=True)
        cfg = oracle_cfg(kw)
        x, tt, cond = clip(tag, kw)
        net.update_num_frames(Fr)
        taps_ref, taps_or = {}, {}
        hs = MG.hook_taps(net, taps_ref)
        t0 = time.time()
        with torch.no_grad():
            ref = net.forward_with_cond_scale(x, tt, cond=cond, cond_scale=1.0)
        t_ref = time.time() - t0
        for hdl in hs:
            hdl.remove()
        with torch.no_grad():
            ora = O.unet_forward(sd, cfg, x, tt, cond, taps=taps_or)
        assert set(taps_or) == set(taps_ref), set(taps_or) ^ set(taps_ref)
        r_eps = over_tol(ora, ref)
        margins, probes, absmean = {}, [], []
        for name, tr in taps_ref.items():
            to = taps_or[name]
            assert to.shape == tr.shape, (tag, name, to.shape, tr.shape)
            margins[name] = over_tol(to, tr)
            flat = tr.reshape(-1)
            probes.append(flat[MG.probe_idx(f'{tag}/{name}', flat.numel())].numpy())
            absmean.append(float(flat.abs().mean()))
        arrays[f'taps/{tag}'] = np.array(list(taps_ref))
        arrays[f'shapes/{tag}'] = np.array([list(tr.shape) for tr in taps_ref.values()], dtype=np.int64)
        arrays[f'absmean/{tag}'] = np.array(absmean, dtype=np.float64)
        arrays[f'probes/{tag}'] = np.stack(probes)
        worst = max(margins, key=margins.get)
        print(f'[{tag}] F={Fr} {h}x{w} t={t}: ref {t_ref:.2f}s |eps|max {ref.abs().max():.3f}  oracle/ref x tol: '
              f'eps {r_eps:.4f}, worst tap {margins[worst]:.4f} ({worst})')
        for name, m in margins.items():
            print(f'    {name:24s} {m:.4f}')
        assert r_eps < 0.2 and margins[worst] < 0.2, 'oracle restatement disagrees with the reference'
        arrays[f'eps/{tag}'] = ref.numpy()
        report[tag] = dict(ctor={k: (list(v) if isinstance(v, tuple) else v) for k, v in kw.items()},
                           F=Fr, h=h, w=w, t=t, schema_digest=schema_digest(schema), schema_entries=len(schema),
                           oracle_eps_over_tol=r_eps, oracle_worst_tap=[worst, margins[worst]])
    save_npz_stable(os.path.join(GOLD, 'configs.npz'), arrays)
    with open(os.path.join(GOLD, 'configs_report.json'), 'w') as f:
        f.write('{\n' + ',\n'.join(f'{json.dumps(k)}: {json.dumps(report[k], sort_keys=True)}' for k in sorted(report)) + '\n}\n')
    print('golden vectors written to', GOLD)


if __name__ == '__main__':
    main()
