"""Every attention kernel's softmax read back one probability per output element, each checked against fp64.

The readout. q and k are the same in every head, so every head computes the same logits, and V is a block identity: V[j, c] = 1
if c == j, else 0 (c = h * D + d, head_dim D = 128 or 72). Head h's output row is then exactly the softmax probabilities of keys
[h * D, (h + 1) * D), and with heads >= ceil(Lk / D) one call returns the whole softmax row of every query: out[:, :Lk] = P and
out[:, Lk:] = 0. Each read-back probability is compared with the fp64 softmax p64 of the same bf16 q and k. bf16 keeps fp32's
exponent range, so the tiny probabilities of early tiles keep their relative precision: a wrong rescale factor, a wrong scale, a
mis-masked key or a wrong V layout is a per-element relative error of its own, not averaged away over thousands of keys as it is
in a random-V output.

The logits (`logit_operands`): x = q k^T * scale * log2(e) = A_i B_j + C_j + noise, with A uniform in [-8, 8], B in [-1, 1],
C a random level, a rising or a falling ramp over the keys (the running max moves on every tile, or never after the first), and
a noise term of every q / k column (every column of both 64-column TMA boxes takes part). The log2 spread covers every fractional
part, so every branch-free path of the exponential (MUFU and the FMA-pipe cubic alike) is exercised, and p >= 2^-60 everywhere,
so nothing is flushed. q = 0 (`kind="uniform"`) makes every logit 0: every probability is exactly 1 / Lk (the coverage oracle).

The bounds, from each kernel's rounding chain (csrc/attn_wgmma.cu, csrc/opensora_kernels.cu):
  * attn_kernel (64- and 128-key tiles), attn_combine_kernel, attn_varlen_d72_kernel: e = 2^(x - m_t) in fp32 against the running
    max m_t of the tile (ex2.approx / exp2f, relative error < 2^-21; the FMA-pipe cubic of MC_ATTN_EMU < 8.8e-5), rounded to bf16
    for the PV product (<= 2^-8 relative), scaled by the later tiles' rescale factors (fp32, < 2^-21 each), divided by the fp32
    row sum l of the UNROUNDED e (relative error <= the largest e error plus the fp32 summation's, < 1e-4 at 4095 keys), and the
    output rounded to bf16 (<= 2^-8). The split-KV form adds fp32 steps only (partials normalised by their own l, merged with
    fp32 weights). So |out - p64| <= (2^-7 + 2e-4 + 2 * 8.8e-5 [MC_ATTN_EMU > 0 only]) * p64.
  * attn_temporal_d72_kernel: P stays fp32 (exp2f, fp32 dot products over 72 columns, fp32 accumulation), so only the output's
    bf16 rounding applies: |out - p64| <= (2^-8 + 1e-4) * p64, half a bf16 ulp plus the fp32 chain.
  * The mean signed relative error over all read-back probabilities must stay below BIAS_BOUND = 5e-4. Round-to-nearest has
    zero mean (the standard deviation of that mean is ~1e-5 over a test here, 6e-5 for the 1440 probabilities of T = 2);
    truncating P to bf16 biases it by about -2.8e-3, and a cubic or a scale that is off shifts it too.
  * Coverage (q = 0): exp2(0) is exactly 1 on the MUFU and on the cubic (constant term 1, f = 0), every rescale factor is 1 and
    l counts the keys exactly, so every read-back element is bf16(1 / Lk); the split-KV merge may move it by one ulp. A dropped,
    doubly counted or unmasked key moves l by a whole unit.

`test_readout_checkers_catch_each_modelled_mutant` (CPU) runs a torch model of these chains through the same checkers: the
faithful model passes, and truncated P, a 1 % cubic, a 0.3 % scale error, a dropped tile and an unmasked pad tile each fail. The
GPU tests print the worst relative error and the bias they observed next to the bounds (`pytest -s`).

Only the CPU test runs without a GPU; this module imports without initialising CUDA.
"""
import math

import pytest
import torch

DEV = "cuda"
BF = torch.bfloat16
LOG2E = 1.4426950408889634
EMU_ERR = 8.8e-5           # documented maximum relative error of ptx::ex2_emul
ATTN_REL = 2.0 ** -7 + 2e-4  # two bf16 roundings (P, output) + the fp32 chain, see the module docstring
TEMPORAL_REL = 2.0 ** -8 + 1e-4  # the output's bf16 rounding + the fp32 chain
BIAS_BOUND = 5e-4
P_FLOOR = 2.0 ** -60


def _ops():
    from magcache_b200 import ops
    return ops


def attn_bound(emu):
    return ATTN_REL + (2 * EMU_ERR if emu else 0.0)


# ------------------------------------------------------------------------------------------- operands and references
def logit_operands(nq, nk, D, scale, kind, g, batch=(), device=DEV):
    """Single-head bf16 q [*batch, nq, D], k [*batch, nk, D] whose scaled log2 logits are A_i B_j + C_j + noise (module
    docstring); kind in {"random", "rise", "fall", "uniform"} ("uniform": q = 0)."""
    kap = scale * LOG2E

    def r(*s):
        return torch.rand(*batch, *s, generator=g, device=device, dtype=torch.float64)

    q = torch.randn(*batch, nq, D, generator=g, device=device, dtype=torch.float64)
    k = torch.randn(*batch, nk, D, generator=g, device=device, dtype=torch.float64) * (0.5 / math.sqrt(D) / kap)
    if kind == "uniform":
        q.zero_()
    else:
        j = torch.linspace(0.0, 1.0, nk, device=device, dtype=torch.float64)
        C = {"random": lambda: 16 * r(nk), "rise": lambda: 20 * j + 2 * r(nk), "fall": lambda: 20 * (1 - j) + 2 * r(nk)}[kind]()
        q[..., 0] = 16 * r(nq) - 8
        q[..., D - 1] = 1.0
        k[..., 0] = (2 * r(nk) - 1) / kap
        k[..., D - 1] = C / kap
    return q.to(BF), k.to(BF)


def probs64(q, k, scale):
    """fp64 softmax(q k^T * scale) of the bf16 operands."""
    p = torch.softmax((q.double() @ k.double().transpose(-1, -2)) * scale, -1)
    assert float(p.min()) >= P_FLOOR, "logit spread too wide: a probability would flush"
    return p


def logits32(q, k, scale):
    """The logits as the kernels hold them: fp32, in the scaled log2 domain."""
    return ((q.double() @ k.double().transpose(-1, -2)) * (scale * LOG2E)).float()


# ------------------------------------------------------------------------------------------- checkers
class Readout:
    """One kernel's read-back probabilities over a test: every launch must hold |got - p64| <= rel_bound * p64 per element
    (`check`); `finish` asserts the mean signed relative error over all of them (a mean over a launch of a few rows means
    little) and prints the observed margins."""

    def __init__(self, label, rel_bound):
        self.label, self.rel_bound = label, rel_bound
        self.worst, self.sum, self.n = 0.0, 0.0, 0

    def check(self, got, p64, what):
        rel = (got.double() - p64) / p64
        assert bool(torch.isfinite(rel).all()), (what, "non-finite readout")
        worst = float(rel.abs().max())
        self.worst, self.sum, self.n = max(self.worst, worst), self.sum + float(rel.sum()), self.n + rel.numel()
        assert worst <= self.rel_bound, (what, f"worst relative error {worst:.3e} > {self.rel_bound:.3e}")

    def finish(self):
        bias = self.sum / max(self.n, 1)
        print(f"\nreadout {self.label}: {self.n} probabilities, worst relative error {self.worst:.3e} (bound {self.rel_bound:.3e}), "
              f"mean signed relative error {bias:+.2e} (bound {BIAS_BOUND:.1e})")
        assert abs(bias) <= BIAS_BOUND, (self.label, f"mean signed relative error {bias:.3e} beyond {BIAS_BOUND:.1e}")


def check_coverage(got, n_keys, what):
    """Every element within one bf16 ulp of bf16(1 / n_keys)."""
    want = torch.tensor(1.0 / n_keys, dtype=torch.float64).to(BF).double().item()
    ulp = 2.0 ** (math.floor(math.log2(1.0 / n_keys)) - 7)
    err = float((got.double() - want).abs().max())
    assert err <= ulp, (what, f"|got - bf16(1/{n_keys})| = {err:.3e} > one ulp {ulp:.3e}")


# ------------------------------------------------------------------------------------------- CPU models of the rounding chains
def _bf16_rn(x):
    return x.to(BF).float()


def _bf16_trunc(x):
    return (x.view(torch.int32) & -65536).view(torch.float32)


def _fma32(a, b, c):
    return (a.double() * b.double() + c.double()).float()


_CUBIC = (0.077119089663028717041015625, 0.227564394474029541015625, 0.695146143436431884765625)


def _ex2_cubic(x, c3=_CUBIC[0]):
    """ptx::ex2_emul: x = floor(x) + f, a cubic for 2^f, floor(x) added into the exponent."""
    x = x.clamp_min(-126.0)
    n = torch.floor(x)
    f = x - n
    p = _fma32(torch.full_like(f, c3), f, torch.full_like(f, _CUBIC[1]))
    p = _fma32(p, f, torch.full_like(f, _CUBIC[2]))
    p = _fma32(p, f, torch.ones_like(f))
    return torch.ldexp(p, n.to(torch.int32)).float()


def _ex2(x):
    return torch.exp2(x.double()).float()


def model_attn(x, tile, emu_mask=0, rot=0, splits=1, p_round=_bf16_rn, c3=_CUBIC[0], drop_tile=None, unmask_pad=False):
    """attn_kernel + attn_combine_kernel on the readout (V = identity), in torch fp32: x [n, Lk] scaled log2 logits; KV tiles
    of `tile` keys in the order rot, rot + 1, ... (mod the tile count), cut into `splits` contiguous runs; per tile the running
    max, fp32 rescale of l and O, e = 2^(x - m) (the cubic where column group (c % tile) / 8 has its bit in emu_mask), l += e,
    O += p_round(e); out = bf16(O / l), or the split partials O_s / l_s merged with weights l_s 2^(m_s - max m). The mutants:
    p_round, c3, drop_tile (skipped), unmask_pad (the ragged tile's zero-filled keys enter l with logit 0)."""
    n, Lk = x.shape
    total = -(-Lk // tile)
    order = [(rot + j) % total for j in range(total)]
    per = -(-total // splits)
    parts = []
    for s0 in range(0, total, per):
        m = torch.full((n, 1), -math.inf)
        l = torch.zeros(n, 1)
        o = torch.zeros(n, Lk)
        for t in order[s0:s0 + per]:
            if t == drop_tile:
                continue
            c0, c1 = t * tile, min(t * tile + tile, Lk)
            xt = x[:, c0:c1]
            if unmask_pad and c1 - c0 < tile:
                xt = torch.cat([xt, torch.zeros(n, tile - (c1 - c0))], 1)
            m_new = torch.maximum(m, xt.max(1, keepdim=True).values)
            f = _ex2(m - m_new)
            l, o = l * f, o * f
            arg = xt - m_new
            emul = torch.tensor([(emu_mask >> ((c // 8) & 7)) & 1 for c in range(xt.shape[1])], dtype=torch.bool)
            e = torch.where(emul, _ex2_cubic(arg, c3), _ex2(arg))
            l = l + e.sum(1, keepdim=True)
            o[:, c0:c1] += p_round(e[:, :c1 - c0])
            m = m_new
        parts.append((o, m, l))
    if len(parts) == 1:
        o, _, l = parts[0]
        return _bf16_rn(o * (1.0 / l))
    mmax = torch.stack([mm for _, mm, _ in parts]).max(0).values
    acc, wsum = torch.zeros(n, Lk), torch.zeros(n, 1)
    for o, mm, l in parts:
        w = l * _ex2(mm - mmax)
        acc, wsum = acc + w * (o * (1.0 / l)), wsum + w
    return _bf16_rn(acc * (1.0 / wsum))


def model_temporal(x, out_round=_bf16_rn):
    """attn_temporal_d72_kernel on the readout: fp32 online softmax, fp32 accumulation, out = out_round(acc / l)."""
    m = x.max(-1, keepdim=True).values
    e = _ex2(x - m)
    return out_round(e * (1.0 / e.sum(-1, keepdim=True)))


def readout_passes(got, p64, rel_bound):
    r = Readout("model", rel_bound)
    try:
        r.check(got, p64, "model")
        r.finish()
    except AssertionError:
        return False
    return True


def coverage_passes(got, n_keys):
    try:
        check_coverage(got, n_keys, "model")
    except AssertionError:
        return False
    return True


def test_readout_checkers_catch_each_modelled_mutant():
    """The checkers bite (CPU): the faithful models of attn_kernel (both tile widths, a quarter and three eighths of the
    exponentials on the cubic, 3- and 5-way splits in rotated order) and of the temporal kernel pass the readout and the
    coverage oracle; P truncated to bf16, a cubic whose leading coefficient is 0.02 too large (~1 % as f -> 1), a scale 0.3 %
    off and a dropped tile each fail the readout (the temporal kernel: a scale 0.3 % off, a truncated output); an unmasked pad
    tile and a dropped tile each fail the coverage oracle."""
    g = torch.Generator().manual_seed(0)
    Lq, Lk, scale = 64, 1300, 0.3  # 11 tiles of 128 keys (21 of 64), the last holding 20
    q, k = logit_operands(Lq, Lk, 128, scale, "random", g, device="cpu")
    p64, x = probs64(q, k, scale), logits32(q, k, scale)
    qu, ku = logit_operands(Lq, Lk, 128, scale, "uniform", g, device="cpu")
    xu = logits32(qu, ku, scale)
    assert bool((xu == 0).all())

    faithful = [dict(tile=64), dict(tile=128), dict(tile=128, emu_mask=0x88), dict(tile=128, emu_mask=0x92, rot=4, splits=3),
                dict(tile=64, rot=7, splits=5)]
    for kw in faithful:
        assert readout_passes(model_attn(x, **kw), p64, attn_bound(kw.get("emu_mask", 0))), kw
        assert coverage_passes(model_attn(xu, **kw), Lk), kw
    readout_mutants = [dict(tile=128, p_round=_bf16_trunc), dict(tile=64, p_round=_bf16_trunc, rot=7, splits=5),
                       dict(tile=128, emu_mask=0x92, c3=_CUBIC[0] + 0.02), dict(tile=128, emu_mask=0x88, c3=_CUBIC[0] + 0.02, rot=4, splits=3),
                       dict(tile=128, drop_tile=3), dict(tile=64, drop_tile=20)]
    for kw in readout_mutants:
        assert not readout_passes(model_attn(x, **kw), p64, attn_bound(kw.get("emu_mask", 0))), kw
    for kw in (dict(tile=128), dict(tile=64, rot=7, splits=5)):
        assert not readout_passes(model_attn(x * 1.003, **kw), p64, attn_bound(0)), ("scale", kw)
    for kw in (dict(tile=128, unmask_pad=True), dict(tile=128, unmask_pad=True, rot=4, splits=3), dict(tile=64, unmask_pad=True),
               dict(tile=128, drop_tile=0), dict(tile=128, drop_tile=10, rot=4, splits=3)):
        assert not coverage_passes(model_attn(xu, **kw), Lk), kw
    # the temporal kernel's chain: 15 sequences of T = 31 frames
    qt, kt = logit_operands(31, 31, 72, scale, "random", g, batch=(15,), device="cpu")
    pt, xt = probs64(qt, kt, scale), logits32(qt, kt, scale)
    assert readout_passes(model_temporal(xt), pt, TEMPORAL_REL)
    assert not readout_passes(model_temporal(xt * 1.003), pt, TEMPORAL_REL)
    assert not readout_passes(model_temporal(xt, out_round=_bf16_trunc), pt, TEMPORAL_REL)


# ------------------------------------------------------------------------------------------- head_dim 128: attn_kernel
def _attn_readout(Lq, Lk, scale, kind, g, ro, first_key_row=0, flags=None, heads=None):
    """One mc_attn_fwd_ex launch on the readout operands (K / V views with NaN rows after Lk, a NaN-filled output): checks the
    readout into `ro` (or coverage when kind == "uniform") and that the columns past Lk are exactly 0; returns the output."""
    ops = _ops()
    H = heads or -(-Lk // 128)
    W = H * 128
    q1, k1 = logit_operands(Lq, Lk, 128, scale, kind, g)
    q = q1.repeat(1, H)
    k = torch.full((Lk + 128, W), float("nan"), dtype=BF, device=DEV)[:Lk]
    k.copy_(k1.repeat(1, H))
    v = torch.full((Lk + 128, W), float("nan"), dtype=BF, device=DEV)[:Lk]
    v.zero_()
    idx = torch.arange(Lk, device=DEV)
    v[idx, idx] = 1.0
    out = torch.full((Lq, W), float("nan"), dtype=BF, device=DEV)
    fl = {}
    if flags is not None:
        fl = dict(seg_flags=flags[0], seg_epoch=flags[1], seg_rows=flags[2])
    ops.attention(q, k, v, H, scale=scale, out=out, first_key_row=first_key_row, **fl)
    what = (ro.label, Lq, Lk, H, scale, kind, first_key_row, flags[2] if flags else None)
    assert bool((out[:, Lk:] == 0).all()), (what, "a column past Lk is not 0")
    if kind == "uniform":
        check_coverage(out[:, :Lk], Lk, what)
    else:
        ro.check(out[:, :Lk], probs64(q1, k1, scale), what)
    return out


_SCALES = (1.0 / math.sqrt(128), 0.3)


@pytest.mark.gpu
def test_readout_short_kernel(monkeypatch):
    """The 64-key kernel (MC_ATTN_KERNEL unset, Lk < 1024, no split): Lk in {1, 63, 64, 65, 511, 1023} x Lq in {1, 127, 300},
    both scales, random logits and q = 0; rising and falling ramps at 511 and 1023 keys."""
    monkeypatch.delenv("MC_ATTN_KERNEL", raising=False)
    monkeypatch.setenv("MC_ATTN_SPLITS", "1")
    g = torch.Generator(device=DEV).manual_seed(64)
    ro = Readout("attn_kernel<64>", attn_bound(0))
    for Lk in (1, 63, 64, 65, 511, 1023):
        for Lq in (1, 127, 300):
            for scale in _SCALES:
                for kind in ("random", "uniform"):
                    _attn_readout(Lq, Lk, scale, kind, g, ro)
        if Lk >= 511:
            for kind in ("rise", "fall"):
                _attn_readout(127, Lk, 0.3, kind, g, ro)
    ro.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("emu", [0, 2, 3, 4])
def test_readout_long_kernel(emu, monkeypatch):
    """The 128-key kernel forced (MC_ATTN_KERNEL=2) for each MC_ATTN_EMU fraction: Lk in {128, 1025, 1500, 4095} x Lq in
    {1, 127, 300}, random logits and q = 0, rising and falling ramps; and chosen by default at Lk 1025."""
    monkeypatch.setenv("MC_ATTN_SPLITS", "1")
    monkeypatch.setenv("MC_ATTN_EMU", str(emu))
    monkeypatch.setenv("MC_ATTN_KERNEL", "2")
    g = torch.Generator(device=DEV).manual_seed(128 + emu)
    ro = Readout(f"attn_kernel<128> MC_ATTN_EMU={emu}", attn_bound(emu))
    for i, Lk in enumerate((128, 1025, 1500, 4095)):
        for Lq in (1, 127, 300):
            _attn_readout(Lq, Lk, _SCALES[(i + Lq) % 2], "random", g, ro)
            _attn_readout(Lq, Lk, 0.3, "uniform", g, ro)
        for kind in ("rise", "fall"):
            _attn_readout(300, Lk, 0.3, kind, g, ro)
    monkeypatch.delenv("MC_ATTN_KERNEL")
    _attn_readout(127, 1025, 0.3, "random", g, ro)
    _attn_readout(127, 1025, 0.3, "uniform", g, ro)
    ro.finish()


@pytest.mark.gpu
def test_readout_split_kv(monkeypatch):
    """Split-KV partials + attn_combine_kernel: the default plan at Lq 128 x 32 heads (a partial wave, split 4 ways over
    Lk 4095 on 132 SMs) and at Lq 100 x 12 heads, and MC_ATTN_SPLITS in {2, 3, 5} on ragged Lk for both tile widths; three
    eighths of the exponentials on the cubic once."""
    import ctypes

    from magcache_b200 import _lib
    g = torch.Generator(device=DEV).manual_seed(5)
    ro = Readout("attn_kernel + attn_combine_kernel", attn_bound(0))
    monkeypatch.delenv("MC_ATTN_KERNEL", raising=False)
    monkeypatch.delenv("MC_ATTN_SPLITS", raising=False)
    monkeypatch.delenv("MC_ATTN_EMU", raising=False)
    for Lq, Lk, H in ((128, 4095, 32), (100, 1500, 12)):
        need = ctypes.c_int64(0)
        _lib.check(_lib.lib.mc_attn_workspace_bytes(Lq, Lk, H, ctypes.byref(need)))
        assert need.value > 0, ("the default plan no longer splits this shape", Lq, Lk, H)
    for kind in ("random", "rise", "fall", "uniform"):
        _attn_readout(128, 4095, 0.3, kind, g, ro)
    _attn_readout(100, 1500, 1.0 / math.sqrt(128), "random", g, ro, heads=12)
    _attn_readout(100, 1500, 0.3, "uniform", g, ro, heads=12)
    for splits in (2, 3, 5):
        monkeypatch.setenv("MC_ATTN_SPLITS", str(splits))
        for Lk in (1023, 1025, 1500):
            for Lq in (1, 300):
                for kind in ("random", "uniform"):
                    _attn_readout(Lq, Lk, 0.3, kind, g, ro)
            _attn_readout(127, Lk, 0.3, "rise", g, ro)
    ro.finish()
    monkeypatch.setenv("MC_ATTN_SPLITS", "3")
    monkeypatch.setenv("MC_ATTN_EMU", "3")
    ro = Readout("attn_kernel + attn_combine_kernel MC_ATTN_EMU=3", attn_bound(3))
    for kind in ("random", "fall", "uniform"):
        _attn_readout(300, 1500, 0.3, kind, g, ro)
    ro.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [1, 3, 5])
def test_readout_rotated_order(splits, monkeypatch):
    """The rotated key order of token-sharded runs (`first_key_row` in {1, 127, 128, 129, Lk - 1}) on ragged Lk 1025 / 1500,
    unsplit and with forced splits: the ragged tile lands mid-order and inside a later split."""
    monkeypatch.delenv("MC_ATTN_KERNEL", raising=False)
    monkeypatch.delenv("MC_ATTN_EMU", raising=False)
    monkeypatch.setenv("MC_ATTN_SPLITS", str(splits))
    g = torch.Generator(device=DEV).manual_seed(splits)
    ro = Readout(f"attn_kernel<128> rotated, MC_ATTN_SPLITS={splits}", attn_bound(0))
    for Lk in (1025, 1500):
        for first in (1, 127, 128, 129, Lk - 1):
            for kind in ("random", "uniform"):
                _attn_readout(127, Lk, 0.3, kind, g, ro, first_key_row=first)
        _attn_readout(300, Lk, 0.3, "rise", g, ro, first_key_row=700)
    ro.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [1, 3])
def test_readout_flag_gated_order(splits, monkeypatch):
    """The flag-gated order (`seg_flags`, `seg_epoch`, `seg_rows`) on one GPU, every flag already at the epoch (the whole flag
    buffer, margins included, so no read can wait): bit-equal to the same call without flags (MC_ATTN_KERNEL=2, same
    `first_key_row`), and the readout / coverage oracles hold. seg_rows 300 / 500 are not multiples of the 128-key tile."""
    monkeypatch.setenv("MC_ATTN_KERNEL", "2")
    monkeypatch.delenv("MC_ATTN_EMU", raising=False)
    monkeypatch.setenv("MC_ATTN_SPLITS", str(splits))
    ro = Readout(f"attn_kernel<128> flag-gated, MC_ATTN_SPLITS={splits}", attn_bound(0))
    epoch = 7
    for Lk in (1025, 1500):
        for seg_rows in (300, 500):
            n_seg = -(-Lk // seg_rows)
            fbuf = torch.full((n_seg + 128,), epoch, dtype=torch.int32, device=DEV)  # 64 flags of margin either side
            flags = (fbuf[64:64 + n_seg], torch.full((1,), epoch, dtype=torch.int32, device=DEV), seg_rows)
            for first in (0, 129, Lk - 1):
                for kind in ("random", "uniform"):
                    seed = Lk + seg_rows + first + splits
                    a = _attn_readout(127, Lk, 0.3, kind, torch.Generator(device=DEV).manual_seed(seed), ro, first_key_row=first, flags=flags)
                    b = _attn_readout(127, Lk, 0.3, kind, torch.Generator(device=DEV).manual_seed(seed), ro, first_key_row=first)
                    assert torch.equal(a, b), (Lk, seg_rows, first, kind, "flag-gated result differs from the ungated one")
            assert bool((fbuf == epoch).all())
    ro.finish()


# ------------------------------------------------------------------------------------------- head_dim 72: Open-Sora kernels
@pytest.mark.gpu
def test_readout_varlen_d72():
    """`mc_attn_varlen_d72`: segments of 1 / 63 / 64 / 65 / 130 / 1000 keys with 1 / 63 / 127 / 300 query rows in one launch at
    scattered query and key offsets (14 heads read a 1000-key segment back), random, rising, falling and q = 0 segments; both
    scales. Rows between the segments stay NaN, the columns past each segment's keys exactly 0."""
    ops = _ops()
    H, D = 14, 72
    W = H * D
    ro = Readout("attn_varlen_d72", attn_bound(0))
    spec = [(1, 1, "random"), (63, 63, "random"), (127, 64, "random"), (300, 65, "random"), (63, 130, "random"),
            (300, 1000, "random"), (127, 1000, "rise"), (63, 1000, "fall"), (127, 130, "rise"), (1, 1000, "random"),
            (1, 1, "uniform"), (63, 63, "uniform"), (127, 64, "uniform"), (300, 65, "uniform"), (63, 130, "uniform"),
            (127, 1000, "uniform")]
    for i, scale in enumerate((1.0 / math.sqrt(D), 0.3)):
        g = torch.Generator(device=DEV).manual_seed(72 + i)
        segs, qs, ks = [], 3, 0
        for ql, kl, kind in spec:
            segs.append((qs, ql, ks, kl, kind))
            qs, ks = qs + ql + 5, ks + kl + 7  # 5 unassigned query rows and 7 NaN key rows between segments
        Lq, Lk = qs, ks
        q = torch.full((Lq, W), float("nan"), dtype=BF, device=DEV)
        k = torch.full((Lk + 64, W), float("nan"), dtype=BF, device=DEV)[:Lk]
        v = torch.full((Lk + 64, W), float("nan"), dtype=BF, device=DEV)[:Lk]
        refs = []
        for s0, ql, k0, kl, kind in segs:
            q1, k1 = logit_operands(ql, kl, D, scale, kind, g)
            q[s0:s0 + ql] = q1.repeat(1, H)
            k[k0:k0 + kl] = k1.repeat(1, H)
            v[k0:k0 + kl] = 0.0
            idx = torch.arange(kl, device=DEV)
            v[k0 + idx, idx] = 1.0
            refs.append(None if kind == "uniform" else probs64(q1, k1, scale))
        segs_dev = torch.tensor([s[:4] for s in segs], dtype=torch.int32, device=DEV)
        out = torch.full((Lq, W), float("nan"), dtype=BF, device=DEV)
        ops.attention_varlen_d72(q, k, v, H, segs_dev, max(s[1] for s in segs), scale=scale, out=out)
        assigned = torch.zeros(Lq, dtype=torch.bool, device=DEV)
        for (s0, ql, k0, kl, kind), p64 in zip(segs, refs):
            assigned[s0:s0 + ql] = True
            o, what = out[s0:s0 + ql], (ro.label, ql, kl, kind, scale)
            assert bool((o[:, kl:] == 0).all()), (what, "a column past the segment's keys is not 0")
            if p64 is None:
                check_coverage(o[:, :kl], kl, what)
            else:
                ro.check(o[:, :kl], p64, what)
        assert bool(out[~assigned].isnan().all()), "a store landed on a row that belongs to no segment"
    ro.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 2, 15, 31, 32])
def test_readout_temporal_d72(T):
    """`mc_attn_temporal_d72`: V = I in each head's first T columns (V[b, t, s, h, d] = [d == t]), so each (b, s, h) returns its
    T x T probability matrix in out[..., :T] and 0 after it. Heads differ here (every head reads its own sequence back).
    (B, S) in {(1, 1), (2, 7), (3, 5)}, 3 heads, both scales, random / rising / falling logits and q = 0. P stays fp32 in
    this kernel: within half a bf16 ulp (plus the fp32 chain) everywhere, and q = 0 gives bf16(1 / T) exactly."""
    ops = _ops()
    H, D = 3, 72
    ro = Readout(f"attn_temporal_d72 T={T}", TEMPORAL_REL)
    g = torch.Generator(device=DEV).manual_seed(T)
    for B, S in ((1, 1), (2, 7), (3, 5)):
        for scale, kind in ((1.0 / math.sqrt(D), "random"), (0.3, "random"), (0.3, "rise"), (0.3, "fall"), (0.3, "uniform")):
            qs, ks = logit_operands(T, T, D, scale, kind, g, batch=(B, S, H))  # [B, S, H, T, D]
            rows = lambda t: t.permute(0, 3, 1, 2, 4).reshape(B * T * S, H * D).contiguous()  # noqa: E731  (b, t, s) rows
            vs = torch.zeros(B, S, H, T, D, dtype=BF, device=DEV)
            vs[..., torch.arange(T), torch.arange(T)] = 1.0
            out = torch.full((B * T * S, H * D), float("nan"), dtype=BF, device=DEV)
            ops.attention_temporal_d72(rows(qs), rows(ks), rows(vs), H, B, T, S, scale=scale, out=out)
            o = out.reshape(B, T, S, H, D).permute(0, 2, 3, 1, 4)  # [B, S, H, T(query), D]
            what = (ro.label, B, S, scale, kind)
            assert bool((o[..., T:] == 0).all()), (what, "a column past T is not 0")
            if kind == "uniform":
                want = torch.tensor(1.0 / T).to(BF).item()
                assert bool((o[..., :T] == want).all()), (what, "q = 0 is not bf16(1/T) exactly")
            else:
                ro.check(o[..., :T], probs64(qs, ks, scale), what)
    ro.finish()
