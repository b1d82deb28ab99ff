"""CPU: host-side control flow of a batched `ddim_sample` (no GPU).  On an unsharded UNet b clips step together: one set of
invariants, one forward and one update per step, noise drawn as (b, ch, F, h, w) like the reference's randn_like over the batch;
passes are sized by `clips_per_pass`."""
import unittest.mock as um

import torch

from tests import gpu_common as G


class _FakeLib:
    def __init__(self, calls):
        self.calls = calls

    def __getattr__(self, name):
        def f(*a):
            self.calls.append((name, int(a[4])) if name == "dawn_unet_ddim_step" else name)
            return 0
        return f


def _sampler(steps):
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion, DynamicNfUnet3D
    net = DynamicNfUnet3D(**G.CTOR).eval()
    D = DynamicNfGaussianDiffusion(denoise_fn=net, num_frames=40, image_size=32, sampling_timesteps=steps, timesteps=1000, loss_type='l2',
                                   use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0)
    return D, net


def test_native_call_sequence_of_a_batch():
    import dawn_pytorch_b200.diffusion as dd
    D, net = _sampler(3)
    D.update_num_frames(4)
    calls, draws = [], []
    net.set_clip_invariants = lambda f, c: calls.append(("invariants", tuple(f.shape), tuple(c.shape), bool(c.abs().sum() > 0)))
    net.forward_x3 = lambda x, t, e: calls.append(("forward_x3", tuple(x.shape), tuple(t.tolist()), tuple(e.shape)))
    net._handle = None
    stream = type("S", (), {"cuda_stream": 0})()

    def noise(k, shp):
        draws.append((k, tuple(shp)))
        return torch.zeros(shp)
    shape, n = (2, 3, 4, 8, 8), 2 * 3 * 4 * 8 * 8
    with um.patch.object(dd, "lib", _FakeLib(calls)), um.patch("torch.cuda.current_stream", lambda: stream):
        D.ddim_sample(torch.rand(2, 272, 8, 8), shape, cond=torch.randn(2, 4, 1032), cond_scale=1.0, noise_fn=noise)
        plain = list(calls)
        calls.clear()
        D.ddim_sample(torch.rand(2, 272, 8, 8), shape, cond=torch.randn(2, 4, 1032), cond_scale=2.0, noise_fn=noise)
        guided = list(calls)
    ts = [t for t, _ in D.ddim_schedule()]
    inv = lambda real: ("invariants", (2, 272, 8, 8), (2, 4, 1032), real)             # noqa: E731
    fwd = lambda t: ("forward_x3", shape, (t, t), shape)                                # noqa: E731
    assert plain == [inv(True)] + [c for t in ts for c in (fwd(t), ("dawn_unet_ddim_step", n))]
    assert guided == [c for t in ts for c in (inv(True), fwd(t), inv(False), fwd(t), ("dawn_unet_ddim_step", n))]
    # start image and every step but the last (which adds no noise, U:1201) draw the whole batch at once
    assert draws[:3] == [(-1, shape), (0, shape), (1, shape)]


def test_clips_per_pass():
    from dawn_pytorch_b200 import unet as U
    _, net = _sampler(3)
    assert net.clips_per_pass(1, 200, 64, 64) == 1
    assert net.clips_per_pass(4, 200, 64, 64) == 2                 # the pass cap holds two 200-frame 64x64 clips
    assert net.clips_per_pass(5, 200, 64, 64) == 2                 # three passes of two
    assert net.clips_per_pass(3, 400, 64, 64) == 1                 # a clip above half the cap runs alone
    assert net.clips_per_pass(12, 200, 32, 32) == 6                # ten per pass at most: two passes of six
    assert net.clips_per_pass(8, 16, 32, 32) == 8
    assert net.clips_per_pass(40, 16, 32, 32) == 14                # 3 equal passes of at most MAX_CLIPS clips
    assert U.MAX_CLIPS == 16
    net._shard = (0, 2, (16, 32, 32))
    assert net.clips_per_pass(8, 16, 32, 32) == 1                  # a frame-sharded handle runs one clip at a time
