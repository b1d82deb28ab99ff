"""GPU: the sampler's update kernels (csrc/sampler.cu: x0_abs_kernel, ddim_update_kernel, ddpm_x0_abs_kernel, ddpm_update_kernel,
threshold_kernel and the radix select between them) and the per-clip / per-pair dispatch of csrc/unet.cu (update_clips,
dawn_unet_ddim_step_guided), bit for bit against the reference's own fp32 arithmetic.

The reference is tests/sampler_ref.py: the lines of U:1181-1205 (DDIM), U:1072-1121 (DDPM) and U:879-890 (guided eps) as fp32
torch ops on the CPU, equal to oracle.unet_oracle.ddim_step / oracle.ddpm_oracle.ddpm_step where those apply
(tests/test_sampler_ref_cpu.py).  Coefficients are the five floats DynamicNfGaussianDiffusion.ddim_coefficients and ddpm_table
hand the kernels.

Error model: none.  Every element equals the reference's bit for bit, the sign of zero included (the last DDIM step adds the
reference's sigma * 0., which turns -0 into +0); where the reference gives NaN the kernel gives NaN (payloads are not compared).
The threshold s is held to torch.quantile + clamp_(min=1): where the kernel's s differs from it, s must be within 1 ulp of the
float64 lerp of the exact order statistics (exact where the lerp weight is 0), and the reference is then evaluated at the
kernel's s.  Every case prints how many elements differ and whether s equalled torch.quantile.

Every x buffer has sentinel guards on both sides and the select scratch one past its keys; all must keep the sentinel.

`dawn_test_kernel` (DAWN_KERNEL_DDIM_STEP / DDPM_STEP) reaches two paths the public entries cannot on one GPU: the frame-sharded
select, through a reducer that stands for W ranks holding the same keys (sums are W times the own value, the min is the own
value, n_global = W n), and the ancestral step's device table read at *t_slot.

Coverage: path x variant -> test.
  path                       variant                                                          test
  ddim update + select       the 20-step schedule as a chain; eta 1, 0; q 0.9, 0, -1;          test_ddim_chain
                             noise / none
  ddim update + select       first, middle, last step of the 250-, 500-, 999-step schedules;   test_ddim_step
                             n 1, 255, 257, 303 104, 303 105 (148 * 8 * 256 + 1), 2 457 600;
                             eta 1, 0; q 0.9, 0, -1; noise / none
  guided pair update         dawn_unet_ddim_step_guided, b = 1, 2, 3 pairs, each its own       test_guided
                             quantile; scale 0, 1, 2, 7.5; both slots written
  update_clips               dawn_unet_ddim_step / dawn_unet_ddpm_step, B = 1, 2, 3, 16 clips   test_batched
                             of their own data, amplitude and noise
  ddpm update + select       t = 999, 998, 500, 1, 0; q 0.9, 0, -1                             test_ddpm_step
  ddpm device table          rows at t = 999, 998, 500, 1, 0 and slots -1, num_t + 5           test_ddpm_table
  frame-sharded select       W = 2, 3 (ties; the count_le >= lo + 2 and min_gt paths),          test_replicas
                             W = 1000 (n_global 2 457 600 000, lo above 2^31); DDIM, DDPM
  non-finite                 NaN, +inf, -inf in x or eps under q 0.9, 0, -1; inf - inf in the   test_nonfinite,
                             lerp; s = +inf; NaN through the sharded select                     test_nonfinite_threshold
"""
import ctypes

import numpy as np
import pytest
import torch

from tests import sampler_ref as S

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = 1234.5
GUARD = 64
SENT_WORD = 0x5A5A5A5A
NAN = float("nan")
INF = float("inf")


def _lib():
    from dawn_pytorch_b200 import _lib
    return _lib


def p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


_DIFF = {}


def diffusion(eta=1.0):
    """a sampler without a network: only its schedule buffers and coefficient functions are used"""
    if eta not in _DIFF:
        from dawn_pytorch_b200 import DynamicNfGaussianDiffusion
        _DIFF[eta] = DynamicNfGaussianDiffusion(denoise_fn=None, num_frames=40, image_size=32, sampling_timesteps=20,
                                                timesteps=1000, loss_type='l2', use_dynamic_thres=True, ddim_sampling_eta=eta)
    return _DIFF[eta]


def ddim_pairs(steps):
    D = diffusion()
    D.sampling_timesteps = steps
    return D.ddim_schedule()


class Guarded:
    """n floats (x, in place) between sentinel guards, and a select scratch of n + 512 words with a guard after it"""

    def __init__(self, x):
        x = x.reshape(-1).float()
        self.n = x.numel()
        self.buf = torch.full((GUARD + self.n + GUARD,), SENT, device=DEV)
        self.buf[GUARD:GUARD + self.n] = x.to(DEV)
        self.x = self.buf[GUARD:GUARD + self.n]
        self.scratch = torch.full((self.n + 512 + GUARD,), SENT_WORD, dtype=torch.int32, device=DEV)

    def out(self):
        torch.cuda.synchronize()
        assert torch.all(self.buf[:GUARD] == SENT) and torch.all(self.buf[GUARD + self.n:] == SENT), "store outside x"
        assert torch.all(self.scratch[self.n + 512:] == SENT_WORD), "store past the select scratch"
        return self.x.cpu()

    def words(self):
        return self.scratch[:265].cpu()


def kernel_s(words):
    return words[263:264].view(torch.float32).item()


def same_bits(name, out, ref, s_note=""):
    """asserts out == ref bit for bit (both NaN counts as equal); prints the count of differing elements"""
    out, ref = out.reshape(-1).float(), ref.reshape(-1).float()
    on, rn = torch.isnan(out), torch.isnan(ref)
    diff = (on != rn) | (~on & ~rn & (out.view(torch.int32) != ref.view(torch.int32)))
    nd = int(diff.sum())
    fin = diff & ~on & ~rn
    worst = (out[fin].double() - ref[fin].double()).abs().max().item() if bool(fin.any()) else 0.0
    print(f"  {name}: {nd} of {out.numel()} elements differ from the reference (worst |d| {worst:.3g}, "
          f"{int(rn.sum())} NaN){s_note}")
    assert nd == 0, f"{name}: {nd} elements differ (worst |d| {worst:.3g})"


def resolve_s(x0, q, s_k=None, replicas=1):
    """the s to evaluate the reference at: torch.quantile's, or the kernel's s_k where that differs and is within 1 ulp of the
    float64 lerp of the exact order statistics.  Returns (s, note)."""
    a = x0.reshape(-1).abs()
    want, lo, hi, w = S.order_stat_s(a.numpy(), q, replicas)
    s_t = S.quantile_s(a.repeat(replicas), q).item() if a.numel() * replicas <= 16_000_000 else None
    if s_t is not None:
        assert (np.isnan(s_t) and np.isnan(want)) or s_t == want or abs(s_t - want) <= np.spacing(np.float32(want)), (s_t, want)
    if s_k is None:
        return (s_t if s_t is not None else np.float32(want)), ""
    if np.isnan(want):
        assert np.isnan(s_k), f"s {s_k!r}: the reference gives NaN"
        return NAN, " s NaN as torch's"
    if s_t is not None and s_k == s_t:
        return s_t, " s == torch.quantile"
    if w == 0 or np.isinf(want):
        assert s_k == np.float32(want), f"s {s_k!r} != {want!r} (lerp weight 0)"
    else:
        assert abs(s_k - want) <= np.spacing(np.float32(want)), f"s {s_k!r} more than 1 ulp from {want!r}"
    return s_k, f" s {s_k!r} != torch.quantile {s_t!r}, within 1 ulp of the float64 lerp"


def sampled(t, n, seed, amp=1.5):
    """x_t = sqrt(ab) x0 + sqrt(1 - ab) e as in sampling, so ca x - cb e cancels as there; and a noise draw"""
    g = torch.Generator().manual_seed(seed)
    acp = diffusion().alphas_cumprod[t].double()
    x0, e, z = (torch.randn(n, generator=g, dtype=torch.float64) for _ in range(3))
    return (acp.sqrt() * amp * x0 + (1 - acp).sqrt() * e).float(), e.float(), z.float()


def eps_for(x, t, seed, amp=1.5):
    """an eps that makes x0 = ca x - cb eps about amp N(0, 1), as a trained UNet's would"""
    g = torch.Generator().manual_seed(seed)
    acp = diffusion().alphas_cumprod[t].double()
    x0 = torch.randn(x.numel(), generator=g, dtype=torch.float64) * amp
    return ((x.double() - acp.sqrt() * x0) / (1 - acp).sqrt()).float()


def x0_of(x, e, coef):
    return S._f(coef[0]) * x - S._f(coef[1]) * e


def plain_step(ddpm, g, e, z, coef, q):
    L = _lib()
    fn = L.lib.dawn_ddpm_step if ddpm else L.lib.dawn_ddim_step
    rc = fn(p(g.x), p(e), p(z), g.n, *coef, q, p(g.scratch), None)
    assert rc == 0, L.lib.dawn_last_error().decode()


def entry_step(ddpm, g, e, z, coef, q, replicas=0, tab=None, t_slot=None, num_t=0):
    L = _lib()
    c = L.DawnKernelCase()
    c.kernel = L.KERNEL_DDPM_STEP if ddpm else L.KERNEL_DDIM_STEP
    c.xs, c.e, c.noise, c.scratch = g.x.data_ptr(), e.data_ptr(), z.data_ptr() if z is not None else None, g.scratch.data_ptr()
    c.n, c.replicas, c.q = g.n, replicas, q
    c.coef[:] = [float(v) for v in coef]
    if tab is not None:
        c.tab, c.t_slot, c.num_t = tab.data_ptr(), t_slot.data_ptr(), num_t
    torch.cuda.synchronize()
    rc = L.lib.dawn_test_kernel(ctypes.byref(c), None)
    assert rc == 0, L.lib.dawn_last_error().decode()


def check_step(name, ddpm, x, e, z, coef, q, step=plain_step, replicas=0, **kw):
    """one update of x (CPU fp32) on the device against the reference; returns the kernel's x"""
    g = Guarded(x)
    ed, zd = e.reshape(-1).to(DEV), None if z is None else z.reshape(-1).to(DEV)
    if replicas:
        kw["replicas"] = replicas
    step(ddpm, g, ed, zd, coef, q, **kw)
    out = g.out()
    s, note = None, ""
    if q > 0:
        s, note = resolve_s(x0_of(x.reshape(-1), e.reshape(-1), coef), q, kernel_s(g.words()), max(replicas, 1))
    ref = (S.ddpm_step if ddpm else S.ddim_step)(x.reshape(-1), e.reshape(-1), None if z is None else z.reshape(-1), coef, q, s)
    same_bits(name, out, ref, note)
    return out


# ================================================================================================================= DDIM
@pytest.mark.parametrize("with_noise", [True, False], ids=["noise", "no_noise"])
@pytest.mark.parametrize("q", [0.9, 0.0, -1.0])
@pytest.mark.parametrize("eta", [1.0, 0.0])
def test_ddim_chain(eta, q, with_noise):
    """every step of the 20-step schedule, each fed the kernel's previous x (the last step adds no noise, U:1201)"""
    D = diffusion(eta)
    pairs = ddim_pairs(20)
    n = 303105
    x, _, _ = sampled(pairs[0][0], n, 11)
    for k, (t, tn) in enumerate(pairs):
        e = eps_for(x, t, 100 + k)
        z = torch.randn(n, generator=torch.Generator().manual_seed(200 + k)) if with_noise and tn > 0 else None
        x = check_step(f"ddim 20 steps, step {k} t={t}->{tn} eta {eta} q {q}", False, x, e, z, D.ddim_coefficients(t, tn), q)


SIZES = [1, 255, 257, 303104, 303105, 2457600]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("which", ["first", "middle", "last"])
@pytest.mark.parametrize("steps", [250, 500, 999])
def test_ddim_step(steps, which, n):
    pairs = ddim_pairs(steps)
    k = {"first": 0, "middle": len(pairs) // 2, "last": len(pairs) - 1}[which]
    t, tn = pairs[k]
    x, e, z = sampled(t, n, steps * 7 + k)
    for eta in (1.0, 0.0):
        coef = diffusion(eta).ddim_coefficients(t, tn)
        for q in (0.9, 0.0, -1.0):
            for zz in ((z, None) if tn > 0 else (None,)):
                check_step(f"ddim {steps} steps t={t}->{tn} n {n} eta {eta} q {q} noise {zz is not None}", False, x, e, zz,
                           coef, q)


# ================================================================================================================= handles
_NET = {}


def handle(B, F, h, w):
    """a small UNet handle of this module's own with B clips of (3, F, h, w); only its clip geometry is used"""
    if "net" not in _NET:
        from dawn_pytorch_b200 import DynamicNfUnet3D
        from tests import gpu_common as G
        _NET["net"] = DynamicNfUnet3D(**dict(G.CTOR, dim_mults=(1, 2), win_width=1)).eval()
    net = _NET["net"]
    net._ensure(torch.device(DEV), F, h, w, B)
    return net._handle


@pytest.mark.parametrize("scale", [0.0, 1.0, 2.0, 7.5])
@pytest.mark.parametrize("b", [1, 2, 3])
def test_guided(b, scale):
    """dawn_unet_ddim_step_guided on a handle of 2b clips: pair i = (clip i, clip b + i), eps = null + (cond - null) * scale in
    three fp32 ops, one quantile per pair, the new x in both slots"""
    L = _lib()
    F, h, w = 8, 16, 16
    nc = 3 * F * h * w
    hd = handle(2 * b, F, h, w)
    pairs = ddim_pairs(20)
    for (t, tn) in (pairs[0], pairs[-1]):
        coef = diffusion().ddim_coefficients(t, tn)
        gen = torch.Generator().manual_seed(b * 100 + int(scale * 10) + t)
        amp = [1.0, 3.0, 0.5]                                 # one quantile shared by the pairs would show
        x = torch.cat([sampled(t, nc, 1000 * i + t, amp[i])[0] for i in range(b)])
        ec = torch.cat([eps_for(x[i * nc:(i + 1) * nc], t, 50 + i, amp[i]) for i in range(b)])
        en = ec + 0.1 * torch.randn(b * nc, generator=gen)
        z = torch.randn(b * nc, generator=gen) if tn > 0 else None
        for q in (0.9, 0.0, -1.0):
            g = Guarded(torch.cat([x, x]))
            eps, zd = torch.cat([ec, en]).to(DEV), None if z is None else z.to(DEV)      # held until the kernels ran
            sc = torch.tensor([scale], device=DEV)
            rc = L.lib.dawn_unet_ddim_step_guided(hd, p(g.x), p(eps), p(zd), nc, p(sc), *coef, q, p(g.scratch), None)
            assert rc == 0, L.lib.dawn_last_error().decode()
            out = g.out()
            assert torch.equal(out[:b * nc].view(torch.int32), out[b * nc:].view(torch.int32)), "the null slots differ"
            for i in range(b):
                sl = slice(i * nc, (i + 1) * nc)
                e = S.guided_eps(ec[sl], en[sl], scale)
                s, note = (resolve_s(x0_of(x[sl], e, coef), q, single_s(False, x[sl], e, coef, q)) if q > 0 else (None, ""))
                ref = S.ddim_step(x[sl], e, None if z is None else z[sl], coef, q, s)
                same_bits(f"guided b {b} pair {i} scale {scale} t={t}->{tn} q {q}", out[sl], ref, note)


def single_s(ddpm, x, e, coef, q):
    """the kernel's s of one clip, from the single-clip entry (a handle's clips share one scratch, so only the last one's s is
    left in it)"""
    g = Guarded(x)
    plain_step(ddpm, g, e.reshape(-1).to(DEV), None, coef, q)
    g.out()
    return kernel_s(g.words())


@pytest.mark.parametrize("ddpm", [False, True], ids=["ddim", "ddpm"])
@pytest.mark.parametrize("B", [1, 2, 3, 16])
def test_batched(B, ddpm):
    """the handle entries on B clips back to back: each clip its own data, amplitude, quantile and noise"""
    L = _lib()
    F, h, w = (23, 16, 16) if B <= 3 else (5, 8, 8)
    nc = 3 * F * h * w
    hd = handle(B, F, h, w)
    t, tn = (500, 450)
    coef = diffusion().ddpm_coefficients(t) if ddpm else diffusion().ddim_coefficients(t, tn)
    amps = [1.5 * (0.5 + (i * 7 % 5)) for i in range(B)]
    parts = [sampled(t, nc, 300 * B + i, amps[i]) for i in range(B)]
    x = torch.cat([v[0] for v in parts])
    e = torch.cat([eps_for(parts[i][0], t, 17 * i + B, amps[i]) for i in range(B)])
    z = torch.cat([v[2] for v in parts])
    fn = L.lib.dawn_unet_ddpm_step if ddpm else L.lib.dawn_unet_ddim_step
    ed = e.to(DEV)
    for q in (0.9, 0.0, -1.0):
        for zz in (z, None):
            g = Guarded(x)
            zd = None if zz is None else zz.to(DEV)                   # held until the kernels ran
            rc = fn(hd, p(g.x), p(ed), p(zd), B * nc, *coef, q, p(g.scratch), None)
            assert rc == 0, L.lib.dawn_last_error().decode()
            out = g.out()
            for i in range(B):
                sl = slice(i * nc, (i + 1) * nc)
                s, note = (resolve_s(x0_of(x[sl], e[sl], coef), q, single_s(ddpm, x[sl], e[sl], coef, q)) if q > 0 else (None, ""))
                ref = (S.ddpm_step if ddpm else S.ddim_step)(x[sl], e[sl], None if zz is None else zz[sl], coef, q, s)
                same_bits(f"{'ddpm' if ddpm else 'ddim'} B {B} clip {i} q {q} noise {zz is not None}", out[sl], ref, note)


# ================================================================================================================= DDPM
T_DDPM = [999, 998, 500, 1, 0]


@pytest.mark.parametrize("q", [0.9, 0.0, -1.0])
@pytest.mark.parametrize("t", T_DDPM)
def test_ddpm_step(t, q):
    n = 3 * 23 * 16 * 16
    x, e, z = sampled(t, n, 31 * t + 5)
    coef = diffusion().ddpm_coefficients(t)
    for zz in (z, None):
        check_step(f"ddpm t={t} q {q} noise {zz is not None}", True, x, e, zz, coef, q)


@pytest.mark.parametrize("slot", T_DDPM + [-1, 1005])
def test_ddpm_table(slot):
    """the step graph's coefficients: row clamp(*t_slot, 0, num_t - 1) of the device table; the by-value set is NaN here"""
    tab = diffusion().ddpm_table()
    row = min(max(slot, 0), tab.shape[0] - 1)
    n = 3 * 23 * 16 * 16
    x, e, z = sampled(row, n, 41 * row + 3)
    tab_d, slot_d = tab.contiguous().to(DEV), torch.tensor([slot], dtype=torch.int64, device=DEV)
    for q in (0.9, 0.0, -1.0):
        check_step(f"ddpm table slot {slot} (row {row}) q {q}", True, x, e, z, tuple(tab[row].tolist()), q,
                   step=lambda d, g, ed, zd, coef, q: entry_step(d, g, ed, zd, [NAN] * 5, q, tab=tab_d, t_slot=slot_d,
                                                                 num_t=tab.shape[0]))
        assert slot_d.item() == slot, "the slot is read, not advanced"


# ================================================================================================================= sharded select
def replica_case(name):
    g = torch.Generator().manual_seed(len(name))
    if name == "w2_ties":             # five values: lo and hi inside one run of equal keys
        return 2, torch.tensor([1.5, 2.0, 3.0, 7.0, 9.0])[torch.randint(0, 5, (10007,), generator=g)] * torch.sign(
            torch.randn(10007, generator=g)), 0.9
    if name == "w2_count_le":         # 2 * 1001 keys: lo = 1800, hi = 1801 are both copies of local key 900 (count_le >= lo + 2)
        return 2, torch.randn(1001, generator=g) * 3, 0.9
    if name == "w3_min_gt":           # 3 * 1000 keys: lo = 2699 is a copy of local key 899, hi = 2700 of key 900 (the min_gt path)
        return 3, torch.randn(1000, generator=g) * 3, 0.9
    if name == "w3_below_one":
        return 3, torch.rand(4099, generator=g) * 1.8 - 0.9, 0.9
    if name == "w1000":               # n_global = 2 457 600 000: lo above 2^31, every histogram bin times 1000
        return 1000, torch.randn(2457600, generator=g) * 3, 0.9
    if name == "w1000_q_half":
        return 1000, torch.randn(2457600, generator=g) * 3, 0.5
    raise KeyError(name)


@pytest.mark.parametrize("ddpm", [False, True], ids=["ddim", "ddpm"])
@pytest.mark.parametrize("name", ["w2_ties", "w2_count_le", "w3_min_gt", "w3_below_one", "w1000", "w1000_q_half"])
def test_replicas(name, ddpm):
    """the frame-sharded select on W ranks that hold the same keys: its statistics are those of W copies, and the update of the
    local values is the reference's at that s.  x = keys, eps = 0 and unit coefficients make the keys |x|; then a real step"""
    W, keys, q = replica_case(name)
    n = keys.numel()
    unit = (1.0, 0.0, 1.0, 0.0, 0.0)
    g = Guarded(keys)
    entry_step(ddpm, g, torch.zeros(n, device=DEV), None, unit, q, replicas=W)
    out, words = g.out(), g.words()
    loc = np.sort(keys.abs().numpy().astype(np.float64))
    _, lo, hi, w = S.order_stat_s(loc, q, W)
    vlo = words[0:1].view(torch.float32).item()
    assert vlo == loc[lo // W], f"order statistic {lo}: {vlo!r} != {loc[lo // W]!r}"
    count_le = int(words[260].item() & 0xFFFFFFFF) | (int(words[261].item() & 0xFFFFFFFF) << 32)
    assert count_le == W * int(np.sum(loc <= vlo)), "count of keys <= v[lo] over the W ranks"
    above = loc[loc > vlo]
    min_gt = int(words[262].item()) & 0xFFFFFFFF
    assert min_gt == (int(np.float32(above.min()).view(np.uint32)) if above.size else 0xFFFFFFFF), "min key above v[lo]"
    assert int(words[264].item()) == 0, "a NaN was flagged"
    s, note = resolve_s(keys, q, kernel_s(words), W)
    print(f"  {name}: n {n} x {W}: lo {lo} hi {hi} w {w:.4g} count_le {count_le}")
    same_bits(f"replicas {name} select", out, (S.ddpm_step if ddpm else S.ddim_step)(keys, torch.zeros(n), None, unit, q, s), note)
    # a real update at t = 500 on the same path
    t = 500
    x, e, z = sampled(t, n, W + n)
    coef = diffusion().ddpm_coefficients(t) if ddpm else diffusion().ddim_coefficients(t, 450)
    check_step(f"replicas {name} step", ddpm, x, e, z, coef, q, step=entry_step, replicas=W)


# ================================================================================================================= non-finite
@pytest.mark.parametrize("ddpm", [False, True], ids=["ddim", "ddpm"])
@pytest.mark.parametrize("q", [0.9, 0.0, -1.0])
@pytest.mark.parametrize("where", ["x", "eps"])
@pytest.mark.parametrize("value", [NAN, INF, -INF], ids=["nan", "inf", "-inf"])
def test_nonfinite(value, where, q, ddpm):
    """one non-finite x or eps element: torch.quantile makes s NaN for a NaN key, so the whole clip goes NaN under q > 0; the
    static clamp and no clip keep the element's own NaN / inf arithmetic"""
    t = 500
    n = 257
    x, e, z = sampled(t, n, 77)
    (x if where == "x" else e)[100] = value
    coef = diffusion().ddpm_coefficients(t) if ddpm else diffusion().ddim_coefficients(t, 450)
    check_step(f"{'ddpm' if ddpm else 'ddim'} {value} in {where} q {q}", ddpm, x, e, z, coef, q)


THRESHOLD_CASES = {
    "inf_minus_inf_n5": ([0.5, 3.0, INF, 2.0, 1.5], 0.9),                # lerp(3, inf, 0.6) = inf - inf = NaN
    "inf_minus_inf_n1001": ([1.0 + i / 1000 for i in range(900)] + [INF] * 101, 0.9),
    "inf_pair_w0": ([1.0, INF, INF], 1.0),                               # inf + 0 * (inf - inf) = NaN
    "s_inf": ([1.0 + i for i in range(10)] + [INF], 0.92),             # vlo + w * inf = inf: finite x0 / inf = 0, inf / inf = NaN
    "nan_above_lo": ([1.0 + i for i in range(999)] + [NAN], 0.5),       # lo far below the NaN key
}


@pytest.mark.parametrize("replicas", [0, 3], ids=["unsharded", "w3"])
@pytest.mark.parametrize("ddpm", [False, True], ids=["ddim", "ddpm"])
@pytest.mark.parametrize("name", list(THRESHOLD_CASES))
def test_nonfinite_threshold(name, ddpm, replicas):
    """x = keys (signs alternate), eps = 0, unit coefficients: s and clamp(x, -s, s) / s as torch gives them, NaN included"""
    vals, q = THRESHOLD_CASES[name]
    keys = torch.tensor(vals) * torch.tensor([1.0, -1.0]).repeat(len(vals))[:len(vals)]
    unit = (1.0, 0.0, 1.0, 0.0, 0.0)
    out = check_step(f"{name} {'ddpm' if ddpm else 'ddim'} W {replicas}", ddpm, keys, torch.zeros_like(keys), None, unit, q,
                     step=entry_step, replicas=replicas)
    s_t = S.quantile_s(keys.abs().repeat(max(replicas, 1)), q).item()
    assert bool(torch.isnan(out).all()) == bool(np.isnan(s_t)), f"s = {s_t}: the clip is NaN exactly when torch's s is"
