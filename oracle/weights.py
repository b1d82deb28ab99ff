"""TEST INFRASTRUCTURE — deterministic synthetic weights for the DAWN denoising UNet.

No released checkpoint is reachable offline (SURVEY.md §8c), so parity runs on synthetic
weights.  They must be bit-identical in this container (where the real reference generates
the golden vectors) and on the GPU box (where /root/reference does not exist), therefore
they come from integer arithmetic only (splitmix64 -> 24-bit mantissa uniform), not from
torch/numpy RNG streams whose vectorised paths may differ between CPUs.

Value ranges follow what PyTorch's default initialisers give the reference modules
(kaiming_uniform(a=sqrt(5)) == U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for Conv/Linear weights,
reference file ...ca_multi_test.py:229,505-512,662-663), but norm gains / biases / scales are
perturbed away from their trivial defaults (1 / 0) so that every term of the forward pass is
exercised by the parity tests.
"""
import math
import numpy as np

_MASK = np.uint64(0xFFFFFFFFFFFFFFFF)


def _fnv1a64(s: str) -> int:
    h = 0xcbf29ce484222325
    for ch in s.encode():
        h ^= ch
        h = (h * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h


def _splitmix64(x: np.ndarray) -> np.ndarray:
    with np.errstate(over='ignore'):
        z = (x + np.uint64(0x9E3779B97F4A7C15)) & _MASK
        z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & _MASK
        z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & _MASK
        return z ^ (z >> np.uint64(31))


def uniform01(key: str, n: int) -> np.ndarray:
    """n floats in [0,1) with 24 random bits each; exact on every platform."""
    base = np.uint64(_fnv1a64(key))
    with np.errstate(over='ignore'):
        idx = (np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + base) & _MASK
    bits = _splitmix64(idx) >> np.uint64(40)
    return (bits.astype(np.float64) * (1.0 / 16777216.0)).astype(np.float32)


def symmetric(key: str, shape, bound: float) -> np.ndarray:
    n = int(np.prod(shape)) if len(shape) else 1
    u = uniform01(key, n)
    return ((u * np.float32(2.0) - np.float32(1.0)) * np.float32(bound)).reshape(shape)


def pseudo_normal(key: str, shape) -> np.ndarray:
    """Approximately N(0,1): sum of 4 uniforms, centred and scaled. Exact everywhere (adds only)."""
    n = int(np.prod(shape))
    acc = np.zeros(n, dtype=np.float32)
    for j in range(4):
        acc += uniform01(f"{key}#{j}", n)
    return ((acc - np.float32(2.0)) * np.float32(math.sqrt(3.0))).reshape(shape)


def synth_value(name: str, shape) -> np.ndarray:
    shape = tuple(int(s) for s in shape)
    leaf = name.split('.')[-1]
    if name.endswith('rotary_emb.freqs'):
        d = shape[0] * 2
        # rotary-embedding-torch 0.3.5: 1/theta^(arange(0,dim,2)/dim), fp32 arithmetic
        import torch
        return (1. / (10000 ** (torch.arange(0, d, 2)[:(d // 2)].float() / d))).numpy()
    if leaf in ('g', 'gamma') or (leaf == 'weight' and '.norm.' in name and len(shape) == 1):
        return np.float32(1.0) + symmetric(name, shape, 0.2)
    if leaf in ('q_scale', 'k_scale'):
        return np.float32(1.0) + symmetric(name, shape, 0.2)
    if leaf == 'null_kv' or 'relative_attention_bias' in name:
        return symmetric(name, shape, 1.7)
    if leaf == 'bias':
        if '.norm.' in name:
            return symmetric(name, shape, 0.1)
        return symmetric(name, shape, 0.05)
    if leaf == 'weight' and len(shape) >= 2:
        fan_in = int(np.prod(shape[1:]))
        return symmetric(name, shape, 1.0 / math.sqrt(fan_in))
    raise ValueError(f"no synthetic rule for {name} {shape}")


def synth_state_dict(schema):
    """schema: iterable of (name, shape). Returns {name: torch.float32 tensor}."""
    import torch
    return {n: torch.from_numpy(np.ascontiguousarray(synth_value(n, s))).float() for n, s in schema}


def probe_indices(name: str, numel: int, n: int) -> np.ndarray:
    """n fixed element indices into a flat tensor of `numel` elements (golden probes; exact on every platform)."""
    u = uniform01('probe/' + name, n)
    return np.minimum((u.astype(np.float64) * numel).astype(np.int64), numel - 1)


def synth_inputs(tag: str, F: int, h: int, w: int, cond_dim: int = 1032, fea_ch: int = 272):
    """Synthetic clip: x_t ~ N(0,1) (3,F,h,w); fea >= 0 (post-ReLU features, LFG/modules/util.py:127-132,
    FD:45-50) (fea_ch,h,w); cond ~ N(0,1) (F,cond_dim).  Returned as torch tensors with batch dim."""
    import torch
    x_t = torch.from_numpy(pseudo_normal(f"{tag}/x_t", (1, 3, F, h, w)))
    fea = torch.from_numpy(np.maximum(pseudo_normal(f"{tag}/fea", (1, fea_ch, h, w)), 0))
    cond = torch.from_numpy(pseudo_normal(f"{tag}/cond", (1, F, cond_dim)))
    return x_t, fea, cond


# ----------------------------------------------------------------------------- LFG flow decoder (oracle/lfg_oracle.py)
def lfg_synth_value(name: str, shape) -> np.ndarray:
    """Synthetic Generator weights (LFG/modules/generator.py): He-uniform convs so that 14 conv + ReLU layers keep O(1)
    activations, BatchNorm affine terms and running statistics away from their trivial values (running_var stays positive)."""
    shape = tuple(int(s) for s in shape)
    leaf = name.split('.')[-1]
    if leaf == 'num_batches_tracked':
        return np.zeros((), dtype=np.int64)
    if leaf == 'running_mean':
        return symmetric(name, shape, 0.2)
    if leaf == 'running_var':
        return np.float32(1.0) + symmetric(name, shape, 0.3)
    if '.norm' in name and leaf == 'weight':
        return np.float32(1.0) + symmetric(name, shape, 0.2)
    if '.norm' in name and leaf == 'bias':
        return symmetric(name, shape, 0.1)
    if leaf == 'bias':
        return symmetric(name, shape, 0.05)
    if leaf == 'weight' and len(shape) == 4:
        fan_in = int(np.prod(shape[1:]))
        gain = 1.0 if name.startswith('final') else math.sqrt(2.0)
        return symmetric(name, shape, gain * math.sqrt(3.0 / fan_in))
    raise ValueError(f"no synthetic LFG rule for {name} {shape}")


def lfg_synth_state_dict(schema, residual_gain=1.0):
    """residual_gain scales every ResBlock's second conv (weight and bias): with the He-uniform rule each block grows the
    bottleneck activations by about 1.4x, so a long stack needs a smaller residual branch to stay O(1), as a trained one does."""
    import torch
    sd = {n: torch.from_numpy(np.ascontiguousarray(lfg_synth_value(n, s))) for n, s in schema}
    if residual_gain != 1.0:
        for n in sd:
            if n.startswith('bottleneck.') and '.conv2.' in n:
                sd[n] = sd[n] * np.float32(residual_gain)
    return sd


def lfg_synth_inputs(tag: str, F: int, H: int, W: int, h: int, w: int):
    """source image in [0, 1] (1, 3, H, W); sampling grid = identity + smooth-ish random offsets, some of it outside [-1, 1]
    (zero padding is exercised); occlusion map in [0, 1] (F, 1, h, w) — what sample_one_video feeds forward_with_flow (FD:372-383)."""
    import torch
    src = torch.from_numpy(uniform01(f"{tag}/src", 3 * H * W).reshape(1, 3, H, W))
    ys = (np.arange(h, dtype=np.float32) + np.float32(0.5)) / np.float32(h) * np.float32(2) - np.float32(1)
    xs = (np.arange(w, dtype=np.float32) + np.float32(0.5)) / np.float32(w) * np.float32(2) - np.float32(1)
    gx, gy = np.meshgrid(xs, ys)
    ident = np.stack([gx, gy], axis=-1)[None].astype(np.float32)
    flow = ident + symmetric(f"{tag}/flow", (F, h, w, 2), 0.35)
    occ = uniform01(f"{tag}/occ", F * h * w).reshape(F, 1, h, w)
    return src, torch.from_numpy(flow.astype(np.float32)), torch.from_numpy(occ)
