"""TEST INFRASTRUCTURE — reference goldens for the UNet's upconv variant and for UNets without spatial linear attention.

Run in the build container only (needs /root/reference; the GPU box never runs this):
    python oracle/make_golden_upconv.py
For every row of CASES it builds the unmodified reference DynamicNfUnet3D (with the shims of oracle/shims) with the
constructor keywords of make_golden.CTOR overridden by the row, loads oracle.weights.synth_state_dict over that
configuration's own state_dict schema, runs one seeded clip (W.synth_inputs(tag, ...), not stored: it regenerates exactly)
and records, in the layout of oracle/make_golden_configs.py,
  tests/golden/upconv.npz           eps/<tag> (the reference's output), and one row per sub-module boundary of taps/<tag>
                                    (names), shapes/<tag>, absmean/<tag> and probes/<tag> (64 fixed elements)
  tests/golden/upconv_report.json   per tag: ctor keywords, clip, the SHA-256 of the reference's state_dict schema and the
                                    oracle (oracle/upconv_oracle.py) vs reference margins
Both files are byte-reproducible.

The rows: nearest x2 + 3x3 conv (use_deconv=False, U:165-172) in each of nn.Conv3d's four padding modes at DAWN's own
configuration; DAWN's "upconv" checkpoint (use_deconv=False, padding_mode='reflect', the training script's `upconv` postfix)
without spatial linear attention; the ConvTranspose without spatial linear attention (and use_final_activation=True, which the
reference's forward never applies); a non-square latent whose deepest level is 1 x 2 (reflect needs pad < size: 1 < 2 on the
upsampled grid); and 128 base channels.
"""
import importlib
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import make_golden as MG             # noqa: E402  (puts the shims and the reference on sys.path)
from oracle import make_golden_configs as MGC    # noqa: E402  (save_npz_stable, schema_digest, over_tol)
from oracle import upconv_oracle as UO           # noqa: E402
from oracle import weights as W                  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
UP = dict(use_deconv=False)

# tag -> (ctor keywords that differ from make_golden.CTOR, (F, h, w, t))
CASES = {
    'up_zeros':       (dict(UP, padding_mode='zeros'), (6, 16, 16, 500)),
    'up_reflect':     (dict(UP, padding_mode='reflect'), (6, 16, 16, 731)),
    'up_replicate':   (dict(UP, padding_mode='replicate'), (6, 16, 16, 88)),
    'up_circular':    (dict(UP, padding_mode='circular'), (6, 16, 16, 952)),
    'upconv_nosla':   (dict(UP, padding_mode='reflect', use_sparse_linear_attn=False), (7, 16, 16, 300)),
    'deconv_nosla':   (dict(use_sparse_linear_attn=False, use_final_activation=True), (5, 16, 16, 640)),
    'rect_reflect':   (dict(UP, padding_mode='reflect'), (5, 8, 16, 410)),
    'rect_circular':  (dict(UP, padding_mode='circular'), (5, 8, 16, 17)),
    'dim128_reflect': (dict(UP, dim=128, padding_mode='reflect'), (4, 16, 16, 999)),
}
ORACLE_KEYS = MGC.ORACLE_KEYS + ('use_deconv', 'padding_mode', 'use_sparse_linear_attn')


def ctor(tag):
    return {**MG.CTOR, **CASES[tag][0]}


def oracle_cfg(kw):
    return UO.UpconvCfg(**{k: kw[k] for k in ORACLE_KEYS if k in kw})


def main():
    torch.set_num_threads(os.cpu_count())
    U = importlib.import_module(MG.U_MOD)
    arrays, report = {}, {}
    for tag, (_, (Fr, h, w, t)) in CASES.items():
        kw = ctor(tag)
        net = U.DynamicNfUnet3D(**kw).eval()
        schema = [(k, list(v.shape)) for k, v in net.state_dict().items()]
        sd = W.synth_state_dict(schema)
        net.load_state_dict(sd, strict=True)
        x_t, fea, cond = W.synth_inputs(tag, Fr, h, w, cond_dim=kw['cond_dim'], fea_ch=kw['channels'] - 3)
        x, tt = MG.build_x(x_t, fea), torch.full((1,), t, dtype=torch.long)
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
            ora = UO.unet_forward(sd, oracle_cfg(kw), x, tt, cond, taps=taps_or)
        assert set(taps_or) == set(taps_ref), set(taps_or) ^ set(taps_ref)
        r_eps = MGC.over_tol(ora, ref)
        margins, probes, absmean = {}, [], []
        for name, tr in taps_ref.items():
            to = taps_or[name]
            assert to.shape == tr.shape, (tag, name, to.shape, tr.shape)
            margins[name] = MGC.over_tol(to, tr)
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
        assert r_eps < 0.2 and margins[worst] < 0.2, 'oracle restatement disagrees with the reference'
        arrays[f'eps/{tag}'] = ref.numpy()
        report[tag] = dict(ctor={k: (list(v) if isinstance(v, tuple) else v) for k, v in kw.items()},
                           F=Fr, h=h, w=w, t=t, schema_digest=MGC.schema_digest(schema), schema_entries=len(schema),
                           oracle_eps_over_tol=r_eps, oracle_worst_tap=[worst, margins[worst]])
    MGC.save_npz_stable(os.path.join(GOLD, 'upconv.npz'), arrays)
    with open(os.path.join(GOLD, 'upconv_report.json'), 'w') as f:
        f.write('{\n' + ',\n'.join(f'{json.dumps(k)}: {json.dumps(report[k], sort_keys=True)}' for k in sorted(report)) + '\n}\n')
    print('golden vectors written to', GOLD)


if __name__ == '__main__':
    main()
