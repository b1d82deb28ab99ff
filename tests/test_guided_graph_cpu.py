"""CPU: host-side control flow of the graph-captured classifier-free-guided `ddim_sample` (no GPU): one guided capture, then one
guided launch per batch (or per clip when two clips per pass is all a pass takes), invariants of 2b clips laid out as
[fea; fea] / [cond; 0], the plain graph's noise draws, one capture for every cond_scale, and the cases that stay eager."""
import unittest.mock as um

import pytest
import torch

from tests import gpu_common as G


class _FakeLib:
    def __init__(self, calls):
        self.calls = calls

    def __getattr__(self, name):
        def f(*a):
            self.calls.append(name)
            return 0
        return f


def _sampler(steps=3):
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion, DynamicNfUnet3D
    net = DynamicNfUnet3D(**G.CTOR).eval()
    D = DynamicNfGaussianDiffusion(denoise_fn=net, num_frames=40, image_size=32, sampling_timesteps=steps, timesteps=1000, loss_type='l2',
                                   use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0)
    D.update_num_frames(4)
    net.graph_generation = lambda: 7
    net._handle = None
    return D, net


def _run(D, net, b, cond_scale, fea=None, cond=None):
    import dawn_pytorch_b200.diffusion as dd
    calls, draws, inv = [], [], []

    def invariants(f, c):
        inv.append((f.clone(), c.clone()))
        calls.append(("invariants", f.shape[0]))
    net.set_clip_invariants = invariants
    stream = type("S", (), {"cuda_stream": 0})()

    def noise(k, shp):
        draws.append((k, tuple(shp)))
        return torch.zeros(shp)
    fea = torch.rand(b, 272, 8, 8) if fea is None else fea
    cond = torch.randn(b, 4, 1032) if cond is None else cond
    with um.patch.object(dd, "lib", _FakeLib(calls)), um.patch("torch.cuda.current_stream", lambda: stream), \
            um.patch("torch.cuda.synchronize", lambda *a: None):
        D.ddim_sample(fea, (b, 3, 4, 8, 8), cond=cond, cond_scale=cond_scale, noise_fn=noise, use_graph=True)
    return calls, draws, inv


@pytest.mark.parametrize("b", [1, 2])
def test_one_capture_then_one_launch_per_batch(b):
    D, net = _sampler()
    fea, cond = torch.rand(b, 272, 8, 8), torch.randn(b, 4, 1032)
    calls, draws, inv = _run(D, net, b, 2.0, fea, cond)
    assert calls == [("invariants", 2 * b), "dawn_unet_sampler_capture_guided", ("invariants", 2 * b),
                     "dawn_unet_sampler_launch_guided"]
    f2, c2 = inv[-1]
    assert torch.equal(f2, torch.cat([fea, fea])) and torch.equal(c2, torch.cat([cond, torch.zeros_like(cond)]))
    assert float(D._guided_graph["scale"][0]) == 2.0
    # the plain graph draws the same noise: start image, then one draw per step but the last
    _, plain_draws = _plain(b)
    assert draws == plain_draws
    # a different scale replays the cached capture
    calls, _, _ = _run(D, net, b, 3.0)
    assert calls == [("invariants", 2 * b), "dawn_unet_sampler_launch_guided"]
    assert D._guided_captures == 1 and float(D._guided_graph["scale"][0]) == 3.0


def _plain(b, clips_per_pass=None):
    import dawn_pytorch_b200.diffusion as dd
    D, net = _sampler()
    if clips_per_pass is not None:
        net.clips_per_pass = clips_per_pass
    calls, draws = [], []
    net.set_clip_invariants = lambda f, c: calls.append("invariants")
    stream = type("S", (), {"cuda_stream": 0})()

    def noise(k, shp):
        draws.append((k, tuple(shp)))
        return torch.zeros(shp)
    with um.patch.object(dd, "lib", _FakeLib(calls)), um.patch("torch.cuda.current_stream", lambda: stream), \
            um.patch("torch.cuda.synchronize", lambda *a: None):
        D.ddim_sample(torch.rand(b, 272, 8, 8), (b, 3, 4, 8, 8), cond=torch.randn(b, 4, 1032), cond_scale=1.0, noise_fn=noise,
                      use_graph=True)
    assert "dawn_unet_sampler_launch" in calls
    return calls, draws


def test_one_launch_per_clip_when_a_pass_takes_two_clips():
    D, net = _sampler()
    net.clips_per_pass = lambda b, F, h, w: min(b, 2)
    fea, cond = torch.rand(3, 272, 8, 8), torch.randn(3, 4, 1032)
    calls, draws, inv = _run(D, net, 3, 2.0, fea, cond)
    assert calls == [("invariants", 2), "dawn_unet_sampler_capture_guided"] + [("invariants", 2), "dawn_unet_sampler_launch_guided"] * 3
    for i in range(3):
        f2, c2 = inv[1 + i]
        assert torch.equal(f2, fea[[i, i]]) and torch.equal(c2, torch.stack([cond[i], torch.zeros_like(cond[i])]))
    # per clip, as the plain graph loops clips: the start image of the batch, then (ch, F, h, w) per step and clip
    assert draws == [(-1, (3, 3, 4, 8, 8))] + [(k, (3, 4, 8, 8)) for _ in range(3) for k in range(2)]


def test_per_clip_launches_keep_the_batch_draws_of_a_batched_sampler():
    """b = 3 clips fit one pass but 6 do not: the eager and cond_scale = 1 samplers step the batch together and draw
    (b, ch, F, h, w) per step, so the per-clip guided launches take their noise from the same draws, clip i's slice."""
    cpp = lambda b, F, h, w: b if b <= 3 else 2                  # noqa: E731
    D, net = _sampler()
    net.clips_per_pass = cpp
    import dawn_pytorch_b200.diffusion as dd
    calls, seen, slabs = [], {}, []

    class Lib(_FakeLib):                                          # keeps the noise slab each launch reads
        def dawn_unet_sampler_launch_guided(self, *a):
            slabs.append(D._guided_graph["noise"].clone())
            return 0
    net.set_clip_invariants = lambda f, c: calls.append(("invariants", f.shape[0]))
    stream = type("S", (), {"cuda_stream": 0})()
    gen = torch.Generator().manual_seed(0)

    def noise(k, shp):
        seen[k] = torch.randn(shp, generator=gen)
        return seen[k]
    with um.patch.object(dd, "lib", Lib(calls)), um.patch("torch.cuda.current_stream", lambda: stream), \
            um.patch("torch.cuda.synchronize", lambda *a: None):
        D.ddim_sample(torch.rand(3, 272, 8, 8), (3, 3, 4, 8, 8), cond=torch.randn(3, 4, 1032), cond_scale=2.0, noise_fn=noise,
                      use_graph=True)
    assert sorted(seen) == [-1, 0, 1] and all(tuple(seen[k].shape) == (3, 3, 4, 8, 8) for k in seen)
    _, plain_draws = _plain(3, cpp)
    assert plain_draws == [(k, (3, 3, 4, 8, 8)) for k in (-1, 0, 1)]
    assert len(slabs) == 3                                        # one launch per clip, clip i's slice of every step's draw
    for i in range(3):
        for k in range(2):
            assert torch.equal(slabs[i][k, 0], seen[k][i])


def test_cond_scale_one_keeps_the_plain_graph():
    D, net = _sampler()
    calls, _, _ = _run(D, net, 1, 1.0)
    assert "dawn_unet_sampler_capture" in calls and "dawn_unet_sampler_capture_guided" not in calls


def test_sharded_and_too_large_stay_eager():
    D, net = _sampler()
    net._shard = (0, 2, (4, 8, 8))
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        _run(D, net, 1, 2.0)
    D, net = _sampler()
    net.clips_per_pass = lambda b, F, h, w: 1
    with pytest.raises(NotImplementedError, match="do not fit one pass"):
        _run(D, net, 1, 2.0)


def test_entries_are_exported_and_reject_bad_arguments_without_a_gpu():
    import ctypes
    from dawn_pytorch_b200 import _lib
    lib = _lib.lib
    for sym in ("dawn_unet_ddim_step_guided", "dawn_unet_sampler_capture_guided", "dawn_unet_sampler_launch_guided"):
        assert sym in _lib.EXPORTS and hasattr(lib, sym)
    f = ctypes.c_float
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.dawn_unet_ddim_step_guided(None, p, p, p, 16, p, *[f(1.0)] * 6, p, None) == -1
    assert b"null handle" in lib.dawn_last_error()
    assert lib.dawn_unet_sampler_launch_guided(None, None) == -1
    from dawn_pytorch_b200 import DynamicNfUnet3D
    net = DynamicNfUnet3D(**G.CTOR)
    h = ctypes.c_void_p()
    assert lib.dawn_unet_create(ctypes.byref(net._cfg), ctypes.byref(h)) == 0
    try:
        assert lib.dawn_unet_ddim_step_guided(h, p, p, p, 16, p, *[f(1.0)] * 6, p, None) == -1      # B = 1: no pair
        assert b"even clip count" in lib.dawn_last_error()
        assert lib.dawn_unet_sampler_capture_guided(h, p, p, p, p, p, ctypes.cast(buf, ctypes.POINTER(ctypes.c_float)), 3,
                                                    f(0.9), p) == -1
        assert b"set_clip_invariants" in lib.dawn_last_error()
        assert lib.dawn_unet_sampler_launch_guided(h, None) == -1
        assert b"sampler_capture_guided must precede" in lib.dawn_last_error()
    finally:
        lib.dawn_unet_destroy(h)
