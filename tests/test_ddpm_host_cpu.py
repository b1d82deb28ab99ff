"""CPU: host side of the ancestral (DDPM) sampler (no GPU): which loop `sample()` picks, which native calls one clip makes
(eager with and without guidance, and the step graph), the host coefficients against the reference's buffers, the exported
entries and their argument checks."""
import ctypes
import os
import unittest.mock as um

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as DO
from tests import gpu_common as G


class _FakeLib:
    """Records native calls by name; dawn_unet_ddpm_step also records its five coefficients."""

    def __init__(self, calls):
        self.calls = calls

    def __getattr__(self, name):
        def f(*a):
            if name == "dawn_unet_ddpm_step":
                self.calls.append((name, tuple(round(float(v), 7) for v in a[5:10])))
            else:
                self.calls.append(name)
            return 0
        return f


def _sampler(timesteps=1000, sampling_timesteps=None):
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion, DynamicNfUnet3D
    net = DynamicNfUnet3D(**G.CTOR).eval()
    D = DynamicNfGaussianDiffusion(denoise_fn=net, num_frames=40, image_size=32, sampling_timesteps=sampling_timesteps,
                                   timesteps=timesteps, loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1,
                                   ddim_sampling_eta=1.0)
    return D, net


@pytest.mark.parametrize("sampling_timesteps,ancestral", [(None, True), (1000, True), (1200, True), (20, False), (999, False)])
def test_sample_dispatches_like_the_reference(sampling_timesteps, ancestral):
    """U:1022-1024, 1150: p_sample_loop unless sampling_timesteps < timesteps."""
    D, _ = _sampler(sampling_timesteps=sampling_timesteps)
    assert D.is_ddim_sampling is not ancestral
    seen = []
    D.p_sample_loop = lambda fea, shape, cond=None, cond_scale=1.: seen.append(("p_sample_loop", fea.shape, shape, cond_scale))
    D.ddim_sample = lambda fea, shape, cond=None, cond_scale=1.: seen.append(("ddim_sample", fea.shape, shape, cond_scale))
    D.update_num_frames(5)
    D.sample(torch.rand(1, 256, 8, 8), torch.rand(1, 16, 8, 8), cond=torch.randn(1, 5, 1032), cond_scale=2.0)
    assert seen == [("p_sample_loop" if ancestral else "ddim_sample", (1, 272, 8, 8), (1, 3, 5, 8, 8), 2.0)]


def _run(D, net, **kw):
    import dawn_pytorch_b200.diffusion as dd
    calls, draws = [], []
    net.set_clip_invariants = lambda f, c: calls.append(("invariants", bool(c.abs().sum() > 0)))
    net.forward_x3 = lambda x, t, e: calls.append(("forward_x3", int(t)))
    net._handle = None
    stream = type("S", (), {"cuda_stream": 0})()

    def noise(k, shp):
        draws.append(k)
        return torch.zeros(shp)
    with um.patch.object(dd, "lib", _FakeLib(calls)), um.patch("torch.cuda.current_stream", lambda: stream), \
            um.patch("torch.cuda.synchronize", lambda *a: None):
        D.p_sample_loop(torch.rand(1, 272, 8, 8), (1, 3, 4, 8, 8), cond=torch.randn(1, 4, 1032), noise_fn=noise, **kw)
    return calls, draws


def test_native_call_sequence_of_one_clip():
    D, net = _sampler(timesteps=4)
    D.update_num_frames(4)
    ts = [3, 2, 1, 0]                                                  # reversed(range(num_timesteps)), U:1130
    step = {t: ("dawn_unet_ddpm_step", tuple(round(v, 7) for v in D.ddpm_coefficients(t))) for t in ts}
    plain, draws = _run(D, net, cond_scale=1.0)
    assert plain == [("invariants", True)] + [c for t in ts for c in (("forward_x3", t), step[t])]
    assert draws == [-1, 0, 1, 2, 3]                                   # start image + one draw per step, t = 0 included (U:1118)
    guided, draws = _run(D, net, cond_scale=2.0)
    per_step = lambda t: [("invariants", True), ("forward_x3", t), ("invariants", False), ("forward_x3", t), step[t]]   # noqa: E731
    assert guided == [c for t in ts for c in per_step(t)]              # cond, then the all-zero null cond (U:879-890, 920)
    assert draws == [-1, 0, 1, 2, 3]
    assert step[0][1][4] == 0.0 and all(step[t][1][4] > 0 for t in ts[:-1])     # no noise at t = 0 (U:1120)
    with pytest.raises(NotImplementedError):
        _run(D, net, cond_scale=2.0, use_graph=True)


def test_step_graph_call_sequence_and_reuse():
    """use_graph: one capture (one step), then num_timesteps replays per clip; a second clip replays the cached graph."""
    D, net = _sampler(timesteps=4)
    D.update_num_frames(4)
    net.graph_generation = lambda: 7
    first, draws = _run(D, net, use_graph=True)
    assert first == [("invariants", True), "dawn_unet_ddpm_capture", ("invariants", True)] + ["dawn_unet_ddpm_launch"] * 4
    assert draws == [-1, 0, 1, 2, 3]
    second, _ = _run(D, net, use_graph=True)
    assert second == [("invariants", True)] + ["dawn_unet_ddpm_launch"] * 4
    g = D._ddpm_graph
    assert g["t"].tolist() == [3] and torch.equal(g["coef"], D.ddpm_table())     # the slot is reset to T-1 per clip


def test_host_coefficients_equal_the_reference_buffers():
    """ddpm_table rows == the reference's own fp32 buffers (dumped by oracle/make_golden_ddpm.py) and == the oracle's
    restatement; sigma = [t > 0] * exp(0.5 * posterior_log_variance_clipped[t]) in fp32 (U:1118-1121)."""
    g = np.load(os.path.join(G.ROOT, "tests", "golden", "ddpm_odd.npz"))
    for T, ref in ((1000, g["buf1000"]), (6, g["buf6"])):
        D, _ = _sampler(timesteps=T)
        tab = D.ddpm_table()
        assert tab.shape == (T, 5) and tab.dtype == torch.float32
        assert torch.equal(tab[:, :4].T.contiguous(), torch.from_numpy(ref[:4]))
        lv = torch.from_numpy(ref[4])
        sigma = torch.stack([(0.5 * lv[t:t + 1]).exp()[0] if t > 0 else torch.zeros(()) for t in range(T)])
        assert torch.equal(tab[:, 4], sigma)
        B = DO.ddpm_buffers(T)
        for j, name in enumerate(("sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_mean_coef1",
                                  "posterior_mean_coef2", "posterior_log_variance_clipped")):
            assert torch.equal(B[name], torch.from_numpy(ref[j])), name
        assert D.ddpm_coefficients(T - 1) == tuple(float(v) for v in tab[T - 1])
    assert abs(float(g["buf1000"][0, 999]) - 64166.3125) < 1e-3          # the x0 amplification at t = 999


def test_p_sample_checks_its_arguments():
    D, _ = _sampler()
    D.update_num_frames(4)
    x, fea, cond = torch.zeros(1, 3, 4, 8, 8), torch.zeros(1, 272, 8, 8), torch.zeros(1, 4, 1032)
    with pytest.raises(ValueError):
        D.p_sample(x, 1000, fea, cond=cond)                            # t outside the schedule
    with pytest.raises(ValueError):
        D.p_sample(torch.zeros(2, 3, 4, 8, 8), torch.tensor([5, 6]), torch.zeros(2, 272, 8, 8), cond=torch.zeros(2, 4, 1032))
    with pytest.raises(ValueError):
        D.p_sample(x, 5, torch.zeros(1, 272, 4, 4), cond=cond)         # fea does not match the sample
    with pytest.raises(ValueError):
        D.p_sample_loop(fea, (1, 3, 5, 8, 8), cond=cond)               # cond frames do not match


def test_entries_are_exported_and_reject_bad_arguments_without_a_gpu():
    from dawn_pytorch_b200 import _lib
    lib = _lib.lib
    for sym in ("dawn_ddpm_step", "dawn_unet_ddpm_step", "dawn_unet_ddpm_capture", "dawn_unet_ddpm_launch"):
        assert sym in _lib.EXPORTS and hasattr(lib, sym)
    f = ctypes.c_float
    assert lib.dawn_ddpm_step(None, None, None, 16, *[f(1.0)] * 6, None, None) == -1
    assert b"dawn_ddpm_step" in lib.dawn_last_error()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.dawn_ddpm_step(p, p, None, 0, *[f(1.0)] * 6, p, None) == -1         # n = 0
    assert lib.dawn_unet_ddpm_step(None, p, p, None, 16, *[f(1.0)] * 6, p, None) == -1
    assert b"null handle" in lib.dawn_last_error()
    assert lib.dawn_unet_ddpm_capture(None, p, p, p, p, p, 10, f(0.9), p) == -1
    assert lib.dawn_unet_ddpm_launch(None, None) == -1
    from dawn_pytorch_b200 import DynamicNfUnet3D
    net = DynamicNfUnet3D(**G.CTOR)
    h = ctypes.c_void_p()
    assert lib.dawn_unet_create(ctypes.byref(net._cfg), ctypes.byref(h)) == 0
    try:
        assert lib.dawn_unet_ddpm_capture(h, p, p, p, p, p, 10, f(0.9), p) == -1          # wrong call order is an error
        assert b"set_clip_invariants" in lib.dawn_last_error()
        assert lib.dawn_unet_ddpm_capture(h, p, p, p, p, p, 0, f(0.9), p) == -1           # empty schedule
        assert lib.dawn_unet_ddpm_launch(h, None) == -1
        assert b"ddpm_capture must precede" in lib.dawn_last_error()
    finally:
        lib.dawn_unet_destroy(h)
