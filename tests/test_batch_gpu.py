"""-m gpu: a batch of B clips in one UNet pass (dawn_unet_set_geometry).  Every clip of a batched pass must equal its own
single-clip run: per-clip GroupNorm statistics, FiLM tables, init-conv maps, cross-attention tables and output layout."""
import ctypes

import pytest
import torch

from dawn_pytorch_b200 import _lib
from oracle import unet_oracle as O
from tests import gpu_common as G

pytestmark = pytest.mark.gpu


def clips(case, B, F, h, w, t0):
    """B different clips of one shape: own inputs, own timestep, amplitude growing with the clip index."""
    xs, ts, cs = [], [], []
    for i in range(B):
        x, _, cond, _, _ = G.clip(f"{case}/batch{i}", F, h, w, t0)
        x[:, :3] *= 1.0 + i
        xs.append(x); cs.append(cond)
        ts.append((t0 + 131 * i) % 1000)
    return torch.cat(xs), torch.tensor(ts, dtype=torch.long), torch.cat(cs)


def forward(net, x, t, cond):
    net.update_num_frames(x.shape[2])
    with torch.no_grad():
        out = net.forward(x.cuda(), t.cuda(), cond=cond.cuda())
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("case", ["odd", "band", "cfg1"])
@pytest.mark.parametrize("B", [2, 3, 4])
def test_each_clip_matches_its_own_run(case, B):
    F, h, w, t0 = G.CASES[case]
    net = G.cuda_net()
    x, t, cond = clips(case, B, F, h, w, t0)
    yb = forward(net, x, t, cond)
    assert net.clip_count() == B
    worst, dmax = 0.0, 0.0
    for i in range(B):
        yi = forward(net, x[i:i + 1], t[i:i + 1], cond[i:i + 1])
        worst = max(worst, G.over_tol(yb[i:i + 1], yi))
        dmax = max(dmax, (yb[i:i + 1] - yi).abs().max().item())
    print(f"{case} B={B}: batched vs per-clip max|d| = {dmax:.3e} ({worst:.4f} x tol)")
    assert worst <= 0.05


@pytest.mark.parametrize("case,B", [("cfg1", 4), ("odd", 3)])
def test_one_pass_not_a_loop(case, B):
    """The batch runs as one pass.  On cfg1 every contraction keeps its kernel path, so the launch count is the single-clip
    one.  On odd the 2x2 level has 23 x 4 = 92 rows per clip, under the 128-row minimum of the wgmma GEMM, and 3 x 92 rows
    above it, so those layers change kernel path; a pass over B clips then launches exactly what one clip of B x F frames
    (the same rows at every level) launches."""
    F, h, w, t0 = G.CASES[case]
    net = G.cuda_net()
    x, t, cond = clips(case, B, F, h, w, t0)
    forward(net, x[:1], t[:1], cond[:1])
    n1 = net.last_launch_count()
    xl, tl, cl = G.clip(f"{case}/long", B * F, h, w, t0)[:3]
    forward(net, xl, tl, cl)
    n_long = net.last_launch_count()
    forward(net, x, t, cond)
    nb = net.last_launch_count()
    print(f"{case}: {n1} launches for one clip, {n_long} for one clip of {B * F} frames, {nb} for {B} clips")
    assert nb == n_long
    if case == "cfg1":
        assert nb == n1


def test_more_clips_than_one_pass_takes():
    """b = 17 > MAX_CLIPS: two equal passes of 9 clips (the second filled up with a copy of its last clip); every clip equals
    its own single-clip run."""
    F, h, w, t0 = 8, 8, 8, 500
    net = G.cuda_net()
    b = 17
    x, t, cond = clips("many", b, F, h, w, t0)
    assert net.clips_per_pass(b, F, h, w) == 9
    y = forward(net, x, t, cond)
    assert net.clip_count() == 9
    for i in (0, 8, 9, 16):
        assert G.over_tol(y[i:i + 1], forward(net, x[i:i + 1], t[i:i + 1], cond[i:i + 1])) <= 0.05


@pytest.mark.parametrize("cond_scale", [1.0, 2.0])
def test_batched_ddim_sample_equals_per_clip_sampling(cond_scale):
    """ddim_sample over b = 2 clips steps both together (one forward and one update per step, per-clip quantile) and gives
    what sampling each clip alone gives with the same noise; the second clip starts at 3x the amplitude of the first."""
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion
    F, h, w, _ = G.CASES["odd"]
    net = G.cuda_net()
    D = DynamicNfGaussianDiffusion(denoise_fn=net, num_frames=F, image_size=h, sampling_timesteps=3, timesteps=1000, loss_type='l2',
                                   use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0).cuda()
    per = [G.clip(f"odd/sample{i}", F, h, w, 47) for i in range(2)]
    fea = torch.cat([p[4] for p in per]).cuda()
    cond = torch.cat([p[2] for p in per]).cuda()
    g = torch.Generator().manual_seed(1)
    noise = {k: torch.randn(2, 3, F, h, w, generator=g) for k in range(-1, 3)}
    noise[-1][1] *= 3.0
    yb = D.ddim_sample(fea, (2, 3, F, h, w), cond=cond, cond_scale=cond_scale, noise_fn=lambda k, s: noise[k].clone()).cpu()
    assert net.clip_count() == 2
    for i in range(2):
        yi = D.ddim_sample(fea[i:i + 1], (1, 3, F, h, w), cond=cond[i:i + 1], cond_scale=cond_scale,
                           noise_fn=lambda k, s: noise[k][i].reshape(s).clone()).cpu()
        r = G.over_tol(yb[i:i + 1], yi)
        print(f"cond_scale {cond_scale}, clip {i}: batched vs alone {r:.4f} x tol")
        assert r <= 0.05


def test_batched_invariants_and_forward_x3():
    F, h, w, t0 = G.CASES["odd"]
    net = G.cuda_net()
    B = 3
    net.update_num_frames(F)
    per = [G.clip(f"odd/x3batch{i}", F, h, w, t0) for i in range(B)]
    x_t = torch.cat([p[3] for p in per]).cuda()
    fea = torch.cat([p[4] for p in per]).cuda()
    cond = torch.cat([p[2] for p in per]).cuda()
    t = torch.tensor([47, 500, 952], dtype=torch.long, device="cuda")
    with torch.no_grad():
        net.set_clip_invariants(fea, cond)
        yb = net.forward_x3(x_t.contiguous(), t).cpu()
        ref = [None] * B
        for i in range(B):
            net.set_clip_invariants(fea[i], cond[i])
            ref[i] = net.forward_x3(x_t[i].contiguous(), t[i:i + 1]).cpu()
    assert yb.shape == (B, 3, F, h, w)
    for i in range(B):
        assert G.over_tol(yb[i:i + 1], ref[i][None]) <= 0.05


def test_batched_forward_matches_oracle_with_per_clip_init_path():
    """Clip 0 has frame-invariant features (hoisted init conv), clip 1 frame-varying ones (full conv): the general entry
    picks the path per clip on the device, and both clips match the oracle."""
    F, h, w = 8, 8, 8
    net = G.cuda_net()
    x0, _, c0, _, _ = G.clip("batch/inv", F, h, w, 500)
    x1, _, c1, _, _ = G.clip("batch/var", F, h, w, 500)
    x1[:, 3:] = torch.relu(x1[:, 3:] + torch.linspace(-0.5, 0.5, F).view(1, 1, F, 1, 1))
    t = torch.tensor([500, 123], dtype=torch.long)
    y = forward(net, torch.cat([x0, x1]), t, torch.cat([c0, c1]))
    with torch.no_grad():
        r0 = O.unet_forward(G.synth_sd(), O.UnetCfg(), x0, t[:1], c0)
        r1 = O.unet_forward(G.synth_sd(), O.UnetCfg(), x1, t[1:], c1)
    e0, e1 = G.over_tol(y[0:1], r0), G.over_tol(y[1:2], r1)
    print(f"invariant clip {e0:.3f} x tol, varying clip {e1:.3f} x tol")
    assert e0 <= 1.0 and e1 <= 1.0
    # the invariant clip took the hoisted path, exactly as it does alone
    assert G.over_tol(y[0:1], forward(net, x0, t[:1], c0)) <= 0.05


def test_geometry_round_trip_reproduces_single_clip_golden():
    F, h, w, t0 = G.CASES["odd"]
    net = G.cuda_net()
    x, t, cond = clips("odd", 2, F, h, w, t0)
    forward(net, x, t, cond)
    gen = net.graph_generation()
    xo, to, co, _, _ = G.clip("odd")
    y = forward(net, xo, to, co)
    assert net.clip_count() == 1 and net.graph_generation() != gen
    assert G.over_tol(y, torch.from_numpy(G.golden("odd")["eps"])) <= 1.0


def test_batched_ddim_update_uses_each_clips_quantile():
    """dawn_unet_ddim_step on B clips back to back equals dawn_ddim_step on each clip alone; the clips' amplitudes differ 3x,
    so one shared quantile would give another answer."""
    F, h, w, t0 = G.CASES["odd"]
    net = G.cuda_net()
    x, t, cond = clips("odd", 2, F, h, w, t0)
    forward(net, x, t, cond)
    lib = _lib.lib
    n1 = 3 * F * h * w
    g = torch.Generator().manual_seed(0)
    xt = torch.randn(2, 3, F, h, w, generator=g)
    xt[1] *= 3.0
    eps = torch.randn(2, 3, F, h, w, generator=g).cuda()
    noise = torch.randn(2, 3, F, h, w, generator=g).cuda()
    scratch = torch.empty(2 * n1 + 512, dtype=torch.int32, device="cuda")
    coef = [1.3, 0.4, 0.9, 0.2, 0.1, 0.9]
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    fp = lambda a: ctypes.c_void_p(a.data_ptr())
    xb = xt.clone().cuda()
    _lib.check(lib.dawn_unet_ddim_step(net._handle, fp(xb), fp(eps), fp(noise), 2 * n1, *coef, fp(scratch), st), "ddim_step")
    xs = xt.clone().cuda()
    for i in range(2):
        _lib.check(lib.dawn_ddim_step(fp(xs[i]), fp(eps[i]), fp(noise[i]), n1, *coef, fp(scratch), st), "ddim_step")
    torch.cuda.synchronize()
    assert torch.equal(xb, xs)
    # a single quantile over both clips differs
    xj = xt.clone().cuda()
    _lib.check(lib.dawn_ddim_step(fp(xj), fp(eps), fp(noise), 2 * n1, *coef, fp(scratch), st), "ddim_step")
    torch.cuda.synchronize()
    assert (xj - xb).abs().max().item() > 1e-3


def test_refusals_on_a_batched_geometry():
    """Frame sharding, the host-buffer entry and debugging taps run one clip: the library refuses them on a B > 1 geometry
    (the module switches its handle back to one clip before it uses them).  The other order, set_geometry(B > 1) on a handle
    already sharded over several ranks, needs an NCCL communicator of two or more ranks; the module never asks for it
    (`clips_per_pass` is 1 on a sharded handle)."""
    F, h, w, t0 = G.CASES["band"]
    net = G.cuda_net()
    x, t, cond = clips("band", 2, F, h, w, t0)
    y0 = forward(net, x, t, cond)
    assert net.clip_count() == 2 and torch.isfinite(y0).all()
    lib = _lib.lib
    rc = lib.dawn_unet_init_shard(net._handle, b"\0" * 128, 2, 0, 2 * F)
    assert rc == -1 and b"one clip" in lib.dawn_last_error()
    _, _, c1, x_t, fea = G.clip("band")
    out = torch.empty(3, F, h, w)
    rc = lib.dawn_unet_forward_host(net._handle, ctypes.c_void_p(x_t.data_ptr()), ctypes.c_void_p(fea.data_ptr()),
                                    ctypes.c_void_p(c1.data_ptr()), 952, ctypes.c_void_p(out.data_ptr()))
    assert rc == -1 and b"one clip" in lib.dawn_last_error()
    buf = torch.empty(64 * F * h * w, device="cuda")
    rc = lib.dawn_unet_set_tap(net._handle, b"downs.0.0", ctypes.c_void_p(buf.data_ptr()))
    assert rc == -1 and b"B = 1" in lib.dawn_last_error()
    # nothing changed: the batch still runs and gives the same result
    y1 = forward(net, x, t, cond)
    assert torch.equal(y0, y1)
