"""CPU: sampling from a real clip without a GPU — the golden's self-consistency (tests/golden/resample.npz against torch's fp32
q_sample and the pinned oracle), the argument checks of q_sample, ddim_sample_from, p_sample_loop_from, interpolate,
motion_to_latent and resample_video, the native call sequence of the suffix samplers with a stub UNet, and the refusals that
stay in place (training entry points, the guided ancestral graph, guided graphs on frame-sharded UNets, learn_null_cond)."""
import ctypes
import os
import unittest.mock as um

import numpy as np
import pytest
import torch

from tests import gpu_common as G


def _gold():
    return np.load(os.path.join(G.ROOT, "tests", "golden", "resample.npz"))


class _FakeLib:
    def __init__(self, calls):
        self.calls = calls

    def __getattr__(self, name):
        def f(*a):
            self.calls.append(name)
            return 0
        return f


def _sampler(steps=20, timesteps=1000):
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion, DynamicNfUnet3D
    net = DynamicNfUnet3D(**G.CTOR).eval()
    D = DynamicNfGaussianDiffusion(denoise_fn=net, num_frames=40, image_size=32, sampling_timesteps=steps, timesteps=timesteps,
                                   loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0)
    D.update_num_frames(4)
    return D, net


def _stub(net, calls):
    net.set_clip_invariants = lambda f, c: calls.append(("invariants", bool(c.abs().sum() > 0)))
    net.forward_x3 = lambda x, t, e: calls.append(("forward_x3", int(t[0])))
    net.graph_generation = lambda: 7
    net._handle = None


def _run(D, fn, *a, **kw):
    import dawn_pytorch_b200.diffusion as dd
    calls, draws = [], []
    _stub(D.denoise_fn, calls)
    stream = type("S", (), {"cuda_stream": 0})()

    def noise(k, shp):
        draws.append(k)
        return torch.zeros(shp)
    with um.patch.object(dd, "lib", _FakeLib(calls)), um.patch("torch.cuda.current_stream", lambda: stream), \
            um.patch("torch.cuda.synchronize", lambda *a: None):
        out = getattr(D, fn)(*a, noise_fn=noise, **kw)
    return calls, draws, out


FEA, COND, SHAPE = torch.rand(1, 272, 8, 8), torch.randn(1, 4, 1032), (1, 3, 4, 8, 8)


def test_golden_self_consistency():
    """The stored q_sample rows are torch's fp32 q_sample of the stored inputs bit for bit, per-clip t included; the suffix is
    the end of the 20-step schedule and the stored trajectories are finite."""
    from oracle import unet_oracle as O
    from oracle import weights as W
    from oracle.make_golden_resample import x0_latent
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion
    g = _gold()
    D = DynamicNfGaussianDiffusion(denoise_fn=None, num_frames=40, image_size=32, sampling_timesteps=20, timesteps=1000)
    shape = tuple(int(v) for v in g["q_shape"])
    x0 = x0_latent(shape)
    z = torch.from_numpy(W.pseudo_normal("resample/q_noise", shape))
    for row, tt in enumerate(g["q_t"].tolist()):
        a = D.sqrt_alphas_cumprod[tt].view(-1, 1, 1, 1, 1)
        b = D.sqrt_one_minus_alphas_cumprod[tt].view(-1, 1, 1, 1, 1)
        assert torch.equal(a * x0 + b * z, torch.from_numpy(g["q_out"][row])), tt
    assert sorted({int(v) for v in g["q_t"][:, 0]}) == [0, 1, 500, 998, 999]
    start = int(g["ddim_start"])
    assert [tuple(p) for p in g["ddim_pairs"].tolist()] == O.ddim_time_pairs()[start:] == D.ddim_schedule()[start:]
    assert g["ddim_out"].shape == (len(g["ddim_pairs"]), 1, 3, 23, 16, 16) and np.isfinite(g["ddim_out"]).all()
    assert g["anc_out"].shape == (1, 3, 23, 16, 16) and np.isfinite(g["anc_out"]).all()
    b, f, hw = (int(v) for v in g["motion"])
    lat = g["motion_latent"]
    assert lat.shape == (b, 3, f, hw // 4, hw // 4)
    assert (lat[:, 2] >= -1).all() and (lat[:, 2] <= 1).all()           # occlusion * 2 - 1 of a sigmoid


def test_argument_checks():
    D, _ = _sampler()
    x = torch.zeros(SHAPE)
    with pytest.raises(ValueError, match="outside"):
        D.q_sample(x, torch.tensor([1000]))
    with pytest.raises(ValueError, match="outside"):
        D.q_sample(x, torch.tensor([-1]))
    with pytest.raises(ValueError, match="t must be"):
        D.q_sample(torch.zeros((2,) + SHAPE[1:]), torch.tensor([1, 2, 3]))
    with pytest.raises(ValueError, match="t must be"):
        D.q_sample(x, torch.tensor([0.5]))
    with pytest.raises(ValueError, match="noise"):
        D.q_sample(x, 3, noise=torch.zeros(1, 3, 4, 8, 7))
    with pytest.raises(ValueError, match="start"):
        D.ddim_sample_from(x, 20, FEA, cond=COND)
    with pytest.raises(ValueError, match="start"):
        D.ddim_sample_from(x, -1, FEA, cond=COND)
    with pytest.raises(ValueError, match="does not match|do not match"):
        D.ddim_sample_from(torch.zeros(1, 3, 4, 8, 6), 0, FEA, cond=COND)
    with pytest.raises(ValueError, match="x_t"):
        D.ddim_sample_from(torch.zeros(3, 4, 8, 8), 0, FEA, cond=COND)
    with pytest.raises(ValueError, match="outside"):
        D.p_sample_loop_from(x, 1001, FEA, cond=COND)
    with pytest.raises(ValueError, match="one timestep"):
        D.p_sample_loop_from(torch.zeros((2,) + SHAPE[1:]), torch.tensor([3, 4]), FEA.repeat(2, 1, 1, 1), cond=COND.repeat(2, 1, 1))
    with pytest.raises(ValueError, match="differ"):
        D.interpolate(x, torch.zeros(1, 3, 4, 8, 6), FEA, cond=COND)
    with pytest.raises(ValueError, match="motion_to_latent"):
        D.motion_to_latent(torch.zeros(6, 8, 8, 2), torch.zeros(6, 1, 8, 8), 4)
    with pytest.raises(ValueError, match="motion_to_latent"):
        D.motion_to_latent(torch.zeros(4, 8, 8, 3), torch.zeros(4, 1, 8, 8), 4)


def test_ddim_sample_from_call_sequence():
    """start = k issues exactly ns - k forwards and updates at the suffix's timesteps; the guided form one pass per step
    (conditioned and null forwards, one update); the draws are numbered as in the whole schedule."""
    D, _ = _sampler()
    pairs = D.ddim_schedule()
    ns = len(pairs)
    for k in (0, 10, ns - 1):
        calls, draws, _ = _run(D, "ddim_sample_from", torch.zeros(SHAPE), k, FEA, cond=COND)
        ts = [t for t, _ in pairs[k:]]
        assert calls == [("invariants", True)] + [c for t in ts for c in (("forward_x3", t), "dawn_unet_ddim_step")]
        assert draws == list(range(k, ns - 1))                            # no start draw; the last step adds no noise
        calls, draws, _ = _run(D, "ddim_sample_from", torch.zeros(SHAPE), k, FEA, cond=COND, cond_scale=2.0)
        assert calls == [c for t in ts for c in (("invariants", True), ("forward_x3", t), ("invariants", False), ("forward_x3", t),
                                                 "dawn_unet_ddim_step")]
    # the graph paths capture the suffix as their own key
    calls, draws, _ = _run(D, "ddim_sample_from", torch.zeros(SHAPE), 15, FEA, cond=COND, use_graph=True)
    assert calls == [("invariants", True), "dawn_unet_sampler_capture", ("invariants", True), "dawn_unet_sampler_launch"]
    assert D._graph["key"][3] == tuple(pairs[15:]) and D._graph["t"].tolist() == [t for t, _ in pairs[15:]]
    assert draws == list(range(15, ns - 1))
    calls, _, _ = _run(D, "ddim_sample_from", torch.zeros(SHAPE), 15, FEA, cond=COND, use_graph=True, cond_scale=3.0)
    assert "dawn_unet_sampler_capture_guided" in calls and calls[-1] == "dawn_unet_sampler_launch_guided"
    assert D._guided_graph["key"][3] == tuple(pairs[15:])


def test_ddim_sample_from_start_zero_is_ddim_sample():
    """start = 0 from the start image ddim_sample draws runs the same calls on the same values."""
    D, _ = _sampler()
    x = torch.randn(SHAPE)
    a_calls, a_draws, _ = _run(D, "ddim_sample", FEA, SHAPE, cond=COND)
    b_calls, b_draws, out = _run(D, "ddim_sample_from", x, 0, FEA, cond=COND)
    assert a_calls == b_calls and a_draws[1:] == b_draws and a_draws[0] == -1
    assert torch.equal(out, x) and out.data_ptr() != x.data_ptr()          # stub updates: the caller's x_t is copied, not modified


def test_p_sample_loop_from_call_sequence():
    D, _ = _sampler(steps=None, timesteps=6)
    for t in (0, 1, 4, 6):
        calls, draws, _ = _run(D, "p_sample_loop_from", torch.zeros(SHAPE), t, FEA, cond=COND)
        steps = list(reversed(range(t)))
        assert calls == ([("invariants", True)] if t else []) + [c for i in steps for c in (("forward_x3", i), "dawn_unet_ddpm_step")]
        assert draws == list(range(t))
        calls, _, _ = _run(D, "p_sample_loop_from", torch.zeros(SHAPE), t, FEA, cond=COND, cond_scale=2.0)
        assert calls == [c for i in steps for c in (("invariants", True), ("forward_x3", i), ("invariants", False), ("forward_x3", i),
                                                    "dawn_unet_ddpm_step")]
    # the step graph of p_sample_loop, replayed t times from a slot set to t - 1, without a capture of its own
    calls, draws, _ = _run(D, "p_sample_loop", FEA, SHAPE, cond=COND, use_graph=True)
    assert calls.count("dawn_unet_ddpm_capture") == 1 and calls.count("dawn_unet_ddpm_launch") == 6
    calls, draws, _ = _run(D, "p_sample_loop_from", torch.zeros(SHAPE), 4, FEA, cond=COND, use_graph=True)
    assert calls == [("invariants", True)] + ["dawn_unet_ddpm_launch"] * 4 and draws == [0, 1, 2, 3]
    assert D._ddpm_graph["t"].tolist() == [3]


def test_interpolate_call_sequence():
    import dawn_pytorch_b200.diffusion as dd
    D, _ = _sampler(steps=None, timesteps=6)
    qs = []
    with um.patch.object(dd.GaussianDiffusion, "q_sample", lambda self, x, t, noise=None: qs.append((t.tolist(), noise)) or x):
        calls, draws, _ = _run(D, "interpolate", torch.zeros(SHAPE), torch.zeros(SHAPE), FEA, cond=COND, t=3, lam=0.25)
    assert [t for t, _ in qs] == [[3], [3]] and draws == [-2, -1, 0, 1, 2]
    assert calls == [("invariants", True)] + [c for i in (2, 1, 0) for c in (("forward_x3", i), "dawn_unet_ddpm_step")]


def test_refusals_stay_in_place():
    from dawn_pytorch_b200 import DynamicNfUnet3D, FlowDiffusion
    D, net = _sampler(steps=None, timesteps=6)
    with pytest.raises(NotImplementedError):
        D(torch.zeros(SHAPE))
    assert not hasattr(D, "p_losses")                                   # the training loss is not part of this sampler
    with pytest.raises(NotImplementedError):
        FlowDiffusion(sampling_timesteps=20, pose_dim=6)(None)
    with pytest.raises(NotImplementedError, match="classifier-free"):
        _run(D, "p_sample_loop", FEA, SHAPE, cond=COND, cond_scale=2.0, use_graph=True)
    with pytest.raises(NotImplementedError, match="classifier-free"):
        _run(D, "p_sample_loop_from", torch.zeros(SHAPE), 3, FEA, cond=COND, cond_scale=2.0, use_graph=True)
    Dd, net = _sampler()
    net._shard = (0, 2, (4, 8, 8))
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        _run(Dd, "ddim_sample", FEA, SHAPE, cond=COND, cond_scale=2.0, use_graph=True)
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        _run(Dd, "ddim_sample_from", torch.zeros(SHAPE), 5, FEA, cond=COND, cond_scale=2.0, use_graph=True)
    with pytest.raises(NotImplementedError, match="learn_null_cond"):
        DynamicNfUnet3D(**{**G.CTOR, "learn_null_cond": True})


def test_flow_diffusion_resample_api():
    """motion is an argument, so the state_dict is unchanged; bad motion / shapes / start raise before any device work."""
    from dawn_pytorch_b200 import FlowDiffusion
    m = FlowDiffusion(sampling_timesteps=20, pose_dim=6)
    assert len(m.diffusion.state_dict()) == 912 and not any("region_predictor" in k for k in m.state_dict())
    with pytest.raises(TypeError, match="FlowAE"):
        m.real_video_latent(torch.zeros(1, 3, 2, 64, 64), torch.zeros(1, 3, 64, 64), object())
    with pytest.raises(ValueError, match="real_vid"):
        m.real_video_latent(torch.zeros(1, 3, 2, 64, 64), torch.zeros(1, 3, 32, 32), (None, None, None))
    m._conditioning = lambda *a: (torch.zeros(1, 272, 8, 8), torch.zeros(1, 4, 1032))
    m.update_num_frames(4)
    args = (torch.zeros(1, 3, 32, 32), torch.zeros(SHAPE), None, None, None, None, 1.0)
    with pytest.raises(ValueError, match="start"):
        m.resample_video(*args, 20)
    with pytest.raises(ValueError, match="x0"):
        m.resample_video(args[0], torch.zeros(1, 3, 5, 8, 8), *args[2:], 3)


def test_entries_are_exported_and_reject_bad_arguments_without_a_gpu():
    from dawn_pytorch_b200 import _lib
    lib = _lib.lib
    for sym in ("dawn_q_sample", "dawn_motion_to_latent"):
        assert sym in _lib.EXPORTS and hasattr(lib, sym)
    p = ctypes.c_void_p(16)
    assert lib.dawn_q_sample(None, p, p, p, p, 1000, 1, 10, p, None) == -1
    assert lib.dawn_q_sample(p, p, p, p, p, 1000, 0, 10, p, None) == -1
    assert lib.dawn_q_sample(p, p, p, p, p, 0, 1, 10, p, None) == -1
    assert b"dawn_q_sample" in lib.dawn_last_error()
    assert lib.dawn_motion_to_latent(p, p, 1, 0, 8, 8, None, None, None, None, 0, p, None) == -1
    assert lib.dawn_motion_to_latent(p, p, 1, 2, 8, 8, p, None, p, p, 1000, p, None) == -1     # t without noise
    assert lib.dawn_motion_to_latent(ctypes.c_void_p(20), p, 1, 2, 8, 8, None, None, None, None, 0, p, None) == -1
    assert b"aligned" in lib.dawn_last_error()
    case = _lib.DawnKernelCase()
    case.kernel = _lib.KERNEL_Q_SAMPLE
    assert lib.dawn_test_kernel(ctypes.byref(case), None) == -1
    case.kernel = _lib.KERNEL_MOTION_TO_LATENT
    assert lib.dawn_test_kernel(ctypes.byref(case), None) == -1
