"""TEST INFRASTRUCTURE — reference goldens for LFG decoder configurations other than DAWN-128's own.

Run in the build container only (needs /root/reference; the GPU box never runs this):
    python oracle/make_golden_lfg_configs.py
For every row of CONFIGS it builds the unmodified reference `Generator` with config/hdtf256.yaml's constructor keywords
overridden by the row, loads oracle.weights.lfg_synth_state_dict over THAT configuration's decode-path schema, runs
`forward_with_flow` frame by frame as `sample_one_video` does (FD:375-383) and `compute_fea` on seeded inputs
(W.lfg_synth_inputs('lfgcfg/<tag>', ...): not stored, they regenerate exactly), and records
  tests/golden/lfg_configs.npz          <tag>/<name>: PROBE_N fixed elements and <tag>/<name>.absmean of prediction,
                                        deformed, fea and of the outputs of `bottleneck` and every `up_blocks.i` (forward hooks)
  tests/golden/lfg_configs_report.json  per tag: ctor keywords, geometry, the SHA-256 of the reference's decode-path state_dict
                                        schema (schema_digest) and the oracle (oracle/lfg_oracle.py, LfgCfg(...)) vs reference
                                        margins in units of rtol 1e-3 / atol 1e-4 (deformed: max |d|)
Both files depend on the arrays only (fixed zip member order and timestamps), so a rerun reproduces them byte for byte.
"""
import hashlib
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
sys.path.insert(0, '/root/reference')
warnings.filterwarnings("ignore")

from oracle import lfg_oracle as L                        # noqa: E402
from oracle import weights as W                           # noqa: E402
from oracle.make_golden_configs import save_npz_stable    # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
PROBE_N = 512
# tag -> (generator_params that differ from config/hdtf256.yaml's, (frames, H, W, flow h, flow w)[, residual_gain of
# W.lfg_synth_state_dict])
CONFIGS = {
    'dawn256':     (dict(), (2, 256, 256, 64, 64)),                              # the benchmark's geometry: flow == bottleneck
    'be128':       (dict(block_expansion=128), (2, 64, 64, 16, 16)),
    'down1':       (dict(num_down_blocks=1), (2, 64, 64, 16, 16)),
    'down3_mf256': (dict(num_down_blocks=3, max_features=256), (2, 64, 64, 16, 16)),   # two equal-width top levels
    'down4':       (dict(num_down_blocks=4), (2, 128, 128, 32, 32)),
    'res0':        (dict(num_bottleneck_blocks=0), (2, 64, 64, 16, 16)),
    'res1':        (dict(num_bottleneck_blocks=1), (2, 64, 64, 16, 16)),
    # the longest conv stack accepted: 66 convs.  At gain 1 the bottleneck reaches 5e4 and the fp32 reference itself (batched vs
    # per frame) differs by 40x the tolerance after the up blocks' BatchNorm, so the stack is scaled to stay O(1).
    'res32':       (dict(num_bottleneck_blocks=32), (2, 32, 32, 8, 8), 0.25),
    'noskip':      (dict(skips=False), (2, 64, 64, 16, 16)),
    'mf96':        (dict(max_features=96), (2, 64, 64, 16, 16)),                 # widths 64, 96, 96: no halo-conv path
    'flow_big':    (dict(), (2, 80, 112, 36, 44)),                               # flow > bottleneck (20x28), ratio 2.22 / 2.55
}
ORACLE_KEYS = ('num_channels', 'block_expansion', 'max_features', 'num_down_blocks', 'num_bottleneck_blocks', 'skips')


def base_ctor():
    import yaml
    with open('/root/reference/config/hdtf256.yaml') as f:
        mp = yaml.safe_load(f)['model_params']
    return dict(num_regions=mp['num_regions'], num_channels=mp['num_channels'], revert_axis_swap=mp['revert_axis_swap'],
                **mp['generator_params'])                                        # FD:116-121


def schema_digest(schema):
    """SHA-256 of a state_dict schema [(name, shape), ...] in order (tests/lfg_config_cases.py computes the same)."""
    return hashlib.sha256(json.dumps([[n, list(sh)] for n, sh in schema], separators=(',', ':')).encode()).hexdigest()


def probe_idx(key, numel):
    u = W.uniform01('probe/lfgcfg/' + key, PROBE_N)
    return np.minimum((u.astype(np.float64) * numel).astype(np.int64), numel - 1)


def over_tol(a, ref):
    return ((a - ref).abs() / (1e-4 + 1e-3 * ref.abs())).max().item()


def main():
    torch.set_num_threads(os.cpu_count())
    from LFG.modules.generator import Generator
    base = base_ctor()
    arrays, report = {}, {}
    for tag, (over, (nf, H, Wd, h, w), *gain) in CONFIGS.items():
        kw, gain = {**base, **over}, (gain or [1.0])[0]
        gen = Generator(**kw).eval()
        schema = [(k, list(v.shape)) for k, v in gen.state_dict().items() if not k.startswith('pixelwise_flow_predictor.')]
        cfg = L.LfgCfg(**{k: kw[k] for k in ORACLE_KEYS})
        assert schema == [(n, list(s)) for n, s in L.state_dict_schema(cfg)], f'{tag}: oracle schema differs from the reference'
        sd = W.lfg_synth_state_dict(schema, gain)
        missing, unexpected = gen.load_state_dict(sd, strict=False)
        assert not unexpected and all(k.startswith('pixelwise_flow_predictor.') for k in missing)
        src, flow, occ = W.lfg_synth_inputs('lfgcfg/' + tag, nf, H, Wd, h, w)
        hooked = {}
        mods = {'bottleneck': gen.bottleneck, **{f'up{i}': gen.up_blocks[i] for i in range(len(gen.up_blocks))}}
        hs = [m.register_forward_hook(lambda _m, _i, o, name=name: hooked.setdefault(name, []).append(o)) for name, m in mods.items()]
        preds, defs = [], []
        with torch.no_grad():
            fea_ref = gen.compute_fea(src)
            for i in range(nf):                                                  # FD:375-383: batch 1 per frame
                o = gen.forward_with_flow(source_image=src, optical_flow=flow[i:i + 1], occlusion_map=occ[i:i + 1])
                preds.append(o['prediction']); defs.append(o['deformed'])
        for hd in hs:
            hd.remove()
        ref = {'prediction': torch.cat(preds), 'deformed': torch.cat(defs), 'fea': fea_ref,
               **{name: torch.cat(v) for name, v in hooked.items()}}
        taps = {}
        with torch.no_grad():
            mine = L.forward_with_flow(sd, cfg, src, flow, occ, taps=taps)
            mine['fea'] = L.compute_fea(sd, cfg, src)
        mine.update({k: taps[k] for k in mods})
        margins = {}
        for name, r in ref.items():
            assert mine[name].shape == r.shape, (tag, name, mine[name].shape, r.shape)
            margins[name] = ((mine[name] - r).abs().max().item() if name == 'deformed' else over_tol(mine[name], r))
            flat = r.reshape(-1)
            arrays[f'{tag}/{name}'] = flat[probe_idx(f'{tag}/{name}', flat.numel())].numpy()
            arrays[f'{tag}/{name}.absmean'] = np.float64(flat.double().abs().mean())
        worst = max((k for k in margins if k != 'deformed'), key=margins.get)
        print(f'[{tag}] {nf} x {H}x{Wd} from {h}x{w}: oracle vs reference x tol: worst {margins[worst]:.4f} ({worst}), '
              f'deformed max|d| {margins["deformed"]:.1e}; |bottleneck| max {ref["bottleneck"].abs().max():.1f}, '
              f'prediction in [{ref["prediction"].min():.3f}, {ref["prediction"].max():.3f}]')
        assert margins[worst] < 0.2 and margins['deformed'] < 1e-5, 'oracle restatement disagrees with the reference'
        report[tag] = dict(ctor=kw, residual_gain=gain, frames=nf, H=H, W=Wd, h=h, w=w, schema_digest=schema_digest(schema),
                           schema_entries=len(schema), taps=list(mods), oracle_margins=margins)
    save_npz_stable(os.path.join(GOLD, 'lfg_configs.npz'), arrays)
    with open(os.path.join(GOLD, 'lfg_configs_report.json'), 'w') as f:
        f.write('{\n' + ',\n'.join(f'{json.dumps(k)}: {json.dumps(report[k], sort_keys=True)}' for k in sorted(report)) + '\n}\n')
    print('golden vectors written to', GOLD)


if __name__ == '__main__':
    main()
