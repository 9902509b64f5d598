"""Every GEMM epilogue read back over every finite bf16 input, each output held to the rounding chain include/magcache_b200.h
states for it.

The readout. A[m, k] = a when k == m mod K and 0 otherwise, so every accumulator is one product plus zeros:
acc[m, n] = a * B[n, m mod K], exactly (two bf16 significands make at most 16 bits, and the zeros add nothing). B holds the
sweep, all 65 280 finite bf16 bit patterns (`bf16_sweep`), laid over B's (n, k) positions in order from a starting offset that
moves on by the number of positions after every launch, so each launch reads the next stretch of the table. Every geometry
launches until every sweep value has reached at least one output element, and the test asserts that it has. Two passes:
  * plain: a = 1, no bias. Each epilogue, and each activation, sees every bf16 value itself. (-0 reads back as +0: zeros are
    compared by value.)
  * scaled: a = 255/256 (bf16 0x3F7F, eight significant bits) and a random bf16-valued bias. acc = a * x is exact in fp32 but is
    not a bf16 value, and bf16(acc + bias) is a real rounding, so a bias added after acc is rounded shows, and so does an
    activation applied to the unrounded acc + bias. a < 1 keeps every acc finite.

Geometries, each at MC_GEMM_BN = 128 and 256 (M x N x K):
  * 256 x 1024 x 64, even ldo: every 16 x 32 patch takes the branch-free interior path of `epilogue_patch`;
  * 200 x 333 x 64: ragged rows (200 is not a multiple of 16), the edge path's pair stores and its single-column tail (N odd);
  * 256 x 1023 x 64 with an odd ldo: the scalar `__float2bfloat16_rn` stores (bf16 outputs only);
  * 256 x 1024 x 72: rows 64..71 select B columns of the second K block, which TMA zero-fills past K;
  * 1024 x 256 x 1000: 16 K blocks; a dropped or doubled block changes the readout.
A and B carry NaN past K, bias and gate carry NaN on both sides, and every output is a fenced window (`fenced` / `check_fence`
of test_kernel_bounds_gpu).

Criteria. The expected output is the header's chain in eager torch on the same device, one rounding per op (`epilogue_model`).
  * MC_EPI_BIAS_BF16 bf16(acc + b[n]), MC_EPI_ROWBIAS_BF16 bf16(acc + b[m]), MC_EPI_BIAS_F32 acc + b[n],
    MC_EPI_BIAS_GATE_RESID old + float(bf16(acc + b)) * g (fp32 stream, fp32 gate) and MC_EPI_BIAS_GATE_RESID_BF16
    bf16(old + bf16(g * bf16(acc + b))) (bf16 stream, bf16-valued gate): bit-equal.
  * GELU (tanh), GELU (erf) and SiLU of x = bf16(acc + b). torch evaluates these in fp32 with accurate library tanhf / erff /
    expf, so no one bit pattern is the right one. The output must be the bf16 rounding of some real within eps of f64, torch's
    formula evaluated in fp64: RN(f64 - eps) <= got <= RN(f64 + eps). `rn_bf16` rounds fp64 to bf16 exactly (ties to even), not
    through fp32, so no allowance for double rounding is needed. eps is what an accurate fp32 evaluation of the formula can be
    off by: unit roundoff 2^-24 per operation and per fp32 constant, tanhf / erff / expf within 2 ulps (CUDA's stated bound).
      - GELU tanh, 0.5 x (1 + tanh(u)), u = beta (x + kappa x^3). x^3 is exact for a bf16 x. kappa's rounding, kappa x^3, the sum
        of two terms of one sign, beta's rounding and the last product leave u within 5 |u| 2^-24, and |tanh'| <= 1 carries that
        into t. tanhf adds 2^-23, 1 + t 2^-24, 0.5 x is exact and the last product adds 2^-24 |out| <= 2^-24 |x|. Altogether
        |x| (1 + |u|) 2.5 * 2^-24 <= eps = |x| (1 + |u|) 2^-21.
      - GELU erf, 0.5 x (1 + erf(x / sqrt 2)). The argument's two roundings move erf by at most
        (2 / sqrt pi) exp(-x^2 / 2) |x| 2^-23.5 < 2^-24; erff adds 2^-23 and 1 + erf 2^-23; times |x| / 2, plus 2^-24 |x| for the
        last product: 1.75 * 2^-23 |x| <= eps = |x| 2^-21.
      - SiLU, x / (1 + exp(-x)). expf's 2^-22, the sum's and the quotient's 2^-24 each: 1.5 * 2^-22 |f64| <= eps = |f64| 2^-20.
        Where x < -ln(FLT_MAX) = -88.72, fp32's exp(-x) is +inf and the formula returns -0 for a value of magnitude below
        2.7e-37, so there eps also covers |f64|.
    torch CUDA's own F.gelu(x, approximate="tanh"), F.gelu(x) and F.silu(x) must meet the same criterion over the sweep
    (`test_torch_activations_meet_the_readout_criterion`). Beside it, every output is compared with torch CUDA's activation of
    the same bf16 x: a difference is allowed only in the last bit (one bf16 ulp); the GPU tests print how many differ.

`test_readout_checkers_reject_each_modelled_mutant` (CPU) runs torch models of the chains through the same checkers over the
sweep: the faithful models pass, and each modelled defect fails. The same test shows that three of those defects (tanh off by
2^-11, a truncating store, an activation of the unrounded pre-activation) pass the bounds against fp64 that the rest of the
suite applies to random operands.

Only the CPU test runs without a GPU; this module imports without initialising CUDA.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from test_kernel_bounds_gpu import check_fence, fenced, gemm_fp64_bounds_ok
from test_kernels_gpu import bf16_ulp_close

DEV = "cuda"
BF, F32 = torch.bfloat16, torch.float32
SWEEP_SIZE = 65280            # finite bf16 bit patterns: 2^16 minus the 256 with an all-ones exponent
SCALED_A = 255.0 / 256.0      # bf16 0x3F7F
BETA, KAPPA = math.sqrt(2.0 / math.pi), 0.044715
EXP_OVERFLOW_X = -math.log(torch.finfo(torch.float32).max)  # fp32 exp(-x) is +inf below this x

EPIS = ["MC_EPI_BIAS_BF16", "MC_EPI_BIAS_GELU_BF16", "MC_EPI_BIAS_GATE_RESID", "MC_EPI_ROWBIAS_BF16", "MC_EPI_BIAS_F32",
        "MC_EPI_BIAS_GELU_ERF_BF16", "MC_EPI_BIAS_GATE_RESID_BF16", "MC_EPI_BIAS_SILU_BF16"]
F32_OUT = ("MC_EPI_BIAS_GATE_RESID", "MC_EPI_BIAS_F32")
ACT = {"MC_EPI_BIAS_GELU_BF16": "gelu_tanh", "MC_EPI_BIAS_GELU_ERF_BF16": "gelu_erf", "MC_EPI_BIAS_SILU_BF16": "silu"}
# (name, M, N, K, odd ldo)
GEOMETRIES = [("interior", 256, 1024, 64, False), ("ragged", 200, 333, 64, False), ("odd_ldo", 256, 1023, 64, True),
              ("k72", 256, 1024, 72, False), ("k1000", 1024, 256, 1000, False)]
# (name, a, bias?, offset of the sweep table)
PASSES = [("plain", 1.0, False, 0), ("scaled", SCALED_A, True, 4099)]


def _ops():
    from magcache_b200 import ops
    return ops


def _lib():
    from magcache_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------- bf16 helpers
def bf16_sweep(device):
    """All finite bf16 values, in bit-pattern order (both zeros included)."""
    bits = torch.arange(-32768, 32768, dtype=torch.int32)
    finite = (bits & 0x7F80) != 0x7F80
    out = bits[finite].to(torch.int16).view(BF).to(device)
    assert out.numel() == SWEEP_SIZE
    return out


def rn_bf16(v):
    """fp64 -> the nearest bf16 value, ties to even, computed exactly in fp64 (bf16: 8 significant bits, fp32's exponent range,
    subnormal spacing 2^-133). Magnitudes past the largest bf16 come out as the next power of two, which compares correctly."""
    _, e = torch.frexp(v)  # |v| in [2^(e-1), 2^e)
    q = torch.exp2((torch.clamp(e - 1, min=-126) - 7).to(torch.float64))
    return torch.round(v / q) * q


def bf16_ordinal(t):
    """bf16 -> int32 that orders like the value and steps by one per representable value (+0 and -0 both 0)."""
    b = t.view(torch.int16).to(torch.int32)
    return torch.where(b < 0, -(b & 0x7FFF), b)


def truncate_bf16(x32):
    """fp32 -> bf16 by dropping the low 16 bits (a truncating store: the mutant the round-to-nearest stores are tested against)."""
    return (x32.contiguous().view(torch.int32) & -65536).view(F32).to(BF)


# ------------------------------------------------------------------------------------------- the chains and their criteria
def act32(kind, x, t_scale=None):
    """torch's fp32 formula for an activation, one rounding per op, as torch's kernels write it. `t_scale` multiplies tanh's
    result (the mutant with a tanh off by 2^-11 relative)."""
    if kind == "gelu_tanh":
        inner = BETA * (x + KAPPA * (x * x * x))
        t = torch.tanh(inner)
        if t_scale is not None:
            t = t * t_scale
        return 0.5 * x * (1.0 + t)
    if kind == "gelu_erf":
        return x * 0.5 * (1.0 + torch.erf(x * (1.0 / math.sqrt(2.0))))
    return x / (1.0 + torch.exp(-x))


def act_f64_eps(kind, x):
    """(f64, eps): torch's formula for the activation of the bf16 values x, evaluated in fp64, and the distance from it an
    accurate fp32 evaluation may land (module docstring)."""
    x = x.double()
    if kind == "gelu_tanh":
        u = BETA * (x + KAPPA * x ** 3)
        return 0.5 * x * (1.0 + torch.tanh(u)), x.abs() * (1.0 + u.abs()) * 2.0 ** -21
    if kind == "gelu_erf":
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0))), x.abs() * 2.0 ** -21
    f = x / (1.0 + torch.exp(-x))
    return f, f.abs() * 2.0 ** -20 + torch.where(x < EXP_OVERFLOW_X, f.abs(), torch.zeros_like(f))


def act_ok(kind, x, got):
    """Elementwise: is `got` (bf16) the bf16 rounding of a real within eps of the fp64 activation of the bf16 input x?
    Returns (ok, f64)."""
    f64, eps = act_f64_eps(kind, x)
    g = got.double()
    return (rn_bf16(f64 - eps) <= g) & (g <= rn_bf16(f64 + eps)), f64


def epilogue_model(epi, acc32, bias=None, old=None, gate=None, mutant=None):
    """The header's chain for `epi` in eager torch, one rounding per op, from the fp32 accumulator (bias / gate already shaped to
    broadcast against it). For the activation epilogues it returns x = bf16(acc + bias) and the bf16 output. `mutant` swaps in
    one modelled defect: "truncate" (truncating bf16 store), "bias_after_round" (bf16(bf16(acc) + bias)), "unrounded_act" (the
    activation of the fp32 acc + bias), "tanh_hi" / "tanh_lo" (tanh off by +-2^-11 relative), "fused_gate" (old + y * g in one
    rounding), "no_inner_round" (bf16(old + g * y) without rounding g * y)."""
    store = truncate_bf16 if mutant == "truncate" else (lambda v: v.to(BF))
    if bias is None:
        pre = acc32 + 0.0
    elif mutant == "bias_after_round":
        pre = acc32.to(BF).float() + bias
    else:
        pre = acc32 + bias
    if epi in ("MC_EPI_BIAS_BF16", "MC_EPI_ROWBIAS_BF16"):
        return store(pre)
    if epi == "MC_EPI_BIAS_F32":
        return pre
    y = pre.to(BF).float()
    if epi == "MC_EPI_BIAS_GATE_RESID":
        if mutant == "fused_gate":
            return (old.double() + y.double() * gate.double()).float()
        return old + y * gate
    if epi == "MC_EPI_BIAS_GATE_RESID_BF16":
        gy = gate * y
        if mutant != "no_inner_round":
            gy = gy.to(BF).float()
        return store(old.float() + gy)
    t_scale = {"tanh_hi": 1.0 + 2.0 ** -11, "tanh_lo": 1.0 - 2.0 ** -11}.get(mutant)
    x = pre if mutant == "unrounded_act" else y
    return y.to(BF), store(act32(ACT[epi], x, t_scale))


def epilogue_ok(epi, got, acc32, bias=None, old=None, gate=None):
    """Elementwise verdict of this module's criterion on an epilogue's output `got` (module docstring); returns (ok, x, f64),
    x / f64 None for the bit-equal epilogues."""
    if epi in ACT:
        x, _ = epilogue_model(epi, acc32, bias)
        ok, f64 = act_ok(ACT[epi], x, got)
        return ok, x, f64
    want = epilogue_model(epi, acc32, bias, old, gate)
    return got.float() == want.float(), None, None  # by value: -0 == +0 (no NaN can arise)


# ------------------------------------------------------------------------------------------- one launch
def _launch(epi, M, N, K, odd_ldo, a_val, b_vals, bias, gate, old):
    """mc_gemm_bf16 on the readout operands: A[m, m mod K] = a_val, B = b_vals [N, K], all views with NaN past K; the output a
    fenced window (odd pitch when asked), holding `old` before the call for the in-place epilogues."""
    ops, L = _ops(), _lib()
    a, _ = fenced((M, K), BF, (0, 1, 8, 8))
    a.zero_()
    rows = torch.arange(M, device=DEV)
    a[rows, rows % K] = a_val
    b, _ = fenced((N, K), BF, (0, 1, 8, 8))
    b.copy_(b_vals)
    odt = F32 if epi in F32_OUT else BF
    if odd_ldo:
        out, obuf = fenced((M, N), odt, (8, 1, 8, 8), fill="fence", pitch=8 + N + 8 + 1 - (N % 2))  # 8 rows: aligned start
        assert out.stride(0) % 2 == 1
    else:
        out, obuf = fenced((M, N), odt, (1, 1, 8, 8), fill="fence")
        assert out.stride(0) % 2 == 0
    if old is not None:
        out.copy_(old)
    ops.gemm(a, b, bias, getattr(L, epi), out=out, gate=gate)
    check_fence(out, obuf)
    return out.clone()


def _side_vector(n, g, scale, bf16_valued):
    """A fenced fp32 [n] input with NaN on both sides (bias or gate)."""
    v, _ = fenced((n,), F32, (0, 0, 4, 4))
    r = torch.randn(n, device=DEV, generator=g) * scale
    v.copy_(r.to(BF).float() if bf16_valued else r)
    return v


class TorchAgreement:
    """Compares outputs with torch CUDA's activation of the same bf16 x, in bf16 ulps (signed: got above torch is positive):
    each may differ in the last bit only. Keeps the count that differ, above and below, and the worst difference with its x;
    likewise the worst distance from RN(f64), for the report."""

    TORCH = {"gelu_tanh": lambda x: F.gelu(x, approximate="tanh"), "gelu_erf": F.gelu, "silu": F.silu}

    def __init__(self, label):
        self.label, self.n, self.above, self.below = label, 0, 0, 0
        self.worst = {"torch": (0, None), "RN(f64)": (0, None)}
        self.far = []  # (x, signed ulps) of the outputs more than one ulp from torch

    def _worst(self, key, d, x):
        i = int(d.abs().flatten().argmax())
        if abs(int(d.flatten()[i])) > abs(self.worst[key][0]):
            self.worst[key] = (int(d.flatten()[i]), float(x.flatten()[i]))

    def add(self, kind, x, got, f64, what):
        d = bf16_ordinal(got) - bf16_ordinal(self.TORCH[kind](x))
        self.n, self.above, self.below = self.n + d.numel(), self.above + int((d > 0).sum()), self.below + int((d < 0).sum())
        self._worst("torch", d, x)
        self._worst("RN(f64)", bf16_ordinal(got) - bf16_ordinal(rn_bf16(f64).float().to(BF)), x)
        far = d.abs() > 1
        self.far += list(zip(x[far].float().tolist(), d[far].tolist()))
        assert not bool(far.any()), (what, f"{int(far.sum())} outputs more than one bf16 ulp from torch's {kind}")

    def report(self):
        (wt, xt), (wf, xf) = self.worst["torch"], self.worst["RN(f64)"]
        print(f"\n{self.label}: {self.above + self.below} of {self.n} outputs differ from torch's bits ({self.above} above, "
              f"{self.below} below); worst {wt:+d} ulp from torch at x = {xt}, worst {wf:+d} ulp from RN(f64) at x = {xf}")
        if self.far:
            xs = [x for x, _ in self.far]
            print(f"  {len(self.far)} more than one ulp from torch ({sum(e > 0 for _, e in self.far)} above, "
                  f"{sum(e < 0 for _, e in self.far)} below), x in [{min(xs)}, {max(xs)}]; (x, ulps) by x: {sorted(set(self.far))[:40]}")


def _explain(epi, ok, got, acc32, x, f64, what):
    """Assertion message for the first elements that fail the criterion."""
    bad = (~ok).nonzero()
    head = bad[:4].tolist()
    parts = []
    for idx in head:
        i = tuple(idx)
        s = f"acc={float(acc32[i])!r} got={float(got[i])!r}"
        if x is not None:
            s += f" x={float(x[i])!r} f64={float(f64[i])!r}"
        parts.append(s)
    return f"{what}: {bad.shape[0]} outputs fail; first at {head}: " + "; ".join(parts)


# ------------------------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("epi", EPIS)
def test_gemm_epilogue_readout(epi, bn, monkeypatch):
    """One epilogue, one tile width, every geometry and both passes: every finite bf16 value through the epilogue, each output
    bit-equal to the header's chain or (activations) the rounding of a value within eps of fp64, and within one ulp of torch."""
    monkeypatch.setenv("MC_GEMM_BN", str(bn))
    sweep = bf16_sweep(DEV)
    g = torch.Generator(device=DEV).manual_seed(EPIS.index(epi) * 2 + bn)
    agree = TorchAgreement(f"{epi} BN={bn}") if epi in ACT else None
    try:
        _readout_all_geometries(epi, bn, sweep, g, agree)
    finally:
        if agree is not None:
            agree.report()


def _readout_all_geometries(epi, bn, sweep, g, agree):
    rowbias = epi == "MC_EPI_ROWBIAS_BF16"
    for geo, M, N, K, odd_ldo in GEOMETRIES:
        if odd_ldo and epi in F32_OUT:
            continue
        assert M >= K  # every B column is selected by some row
        for pas, a_val, with_bias, offset in PASSES:
            covered = torch.zeros(SWEEP_SIZE, dtype=torch.bool, device=DEV)
            per_launch = N * K
            for launch in range(-(-SWEEP_SIZE // per_launch)):
                what = (epi, bn, geo, pas, launch)
                table = (torch.arange(per_launch, device=DEV) + offset + launch * per_launch) % SWEEP_SIZE
                b_vals = sweep[table].view(N, K)
                bias = _side_vector(M if rowbias else N, g, 2.0, True) if with_bias else None
                gate = old = None
                if epi == "MC_EPI_BIAS_GATE_RESID":
                    gate = _side_vector(N, g, 0.5, False)
                    old = torch.randn(M, N, device=DEV, generator=g)
                elif epi == "MC_EPI_BIAS_GATE_RESID_BF16":
                    gate = _side_vector(N, g, 0.5, True)
                    old = torch.randn(M, N, device=DEV, generator=g).to(BF)
                got = _launch(epi, M, N, K, odd_ldo, a_val, b_vals, bias, gate, old)
                cols = torch.arange(M, device=DEV) % K
                covered[table.view(N, K)[:, cols]] = True
                acc32 = b_vals[:, cols].t().float() * a_val  # exact: a_val has 8 significant bits, and a_val <= 1
                bias_b = None if bias is None else (bias[:, None] if rowbias else bias[None, :])
                gate_b = None if gate is None else gate[None, :]
                ok, x, f64 = epilogue_ok(epi, got, acc32, bias_b, old, gate_b)
                if agree is not None:
                    agree.add(ACT[epi], x, got, f64, what)
                assert bool(ok.all()), _explain(epi, ok, got, acc32, x, f64, what)
            assert bool(covered.all()), (epi, bn, geo, pas, f"{int((~covered).sum())} sweep values never reached an output")


@pytest.mark.gpu
def test_silu_kernel_readout():
    """`mc_silu_bf16` (its own kernel, the same formula as the SiLU epilogue) over every finite bf16 value, NaN around the
    input, a fenced output: the SiLU criterion, and within one ulp of torch's F.silu."""
    ops = _ops()
    sweep = bf16_sweep(DEV)
    x, _ = fenced((SWEEP_SIZE,), BF, (0, 0, 8, 8))
    x.copy_(sweep)
    y, ybuf = fenced((SWEEP_SIZE,), BF, (0, 0, 8, 8), fill="fence")
    ops.silu(x, out=y)
    check_fence(y, ybuf)
    ok, f64 = act_ok("silu", sweep, y)
    assert bool(ok.all()), _explain("silu", ok, y, sweep.float(), sweep, f64, "mc_silu_bf16")
    agree = TorchAgreement("mc_silu_bf16")
    agree.add("silu", sweep, y, f64, "mc_silu_bf16")
    agree.report()


@pytest.mark.gpu
def test_torch_activations_meet_the_readout_criterion():
    """The criterion is one that torch CUDA's own activations meet: F.gelu (tanh and erf) and F.silu of every finite bf16 value,
    and of the scaled pass's rounded pre-activations, are within eps of fp64."""
    sweep = bf16_sweep(DEV)
    g = torch.Generator(device=DEV).manual_seed(7)
    bias = (torch.randn(SWEEP_SIZE, device=DEV, generator=g) * 2.0).to(BF).float()
    scaled = (sweep.float() * SCALED_A + bias).to(BF)
    for x in (sweep, scaled):
        for kind, fn in TorchAgreement.TORCH.items():
            got = fn(x)
            ok, f64 = act_ok(kind, x, got)
            assert bool(ok.all()), _explain(kind, ok, got, x.float(), x, f64, f"torch {kind}")


# ------------------------------------------------------------------------------------------- the checkers themselves (CPU)
def _passes_cpu(g):
    """The two passes' inputs as 1-D CPU vectors over the sweep: (name, acc32, bias, old fp32, gate fp32, old bf16,
    bf16-valued gate)."""
    sweep = bf16_sweep("cpu")
    n = SWEEP_SIZE
    side = dict(old32=torch.randn(n, generator=g), gate32=torch.randn(n, generator=g) * 0.5,
                old16=torch.randn(n, generator=g).to(BF), gate16=(torch.randn(n, generator=g) * 0.5).to(BF).float())
    bias = (torch.randn(n, generator=g) * 2.0).to(BF).float()
    return [("plain", sweep.float(), None, side), ("scaled", sweep.float() * SCALED_A, bias, side)]


def _model_ok(epi, acc32, bias, side, mutant=None):
    """Run the model of `epi` (with `mutant`) through this module's checker; True when every output passes."""
    old, gate = {"MC_EPI_BIAS_GATE_RESID": (side["old32"], side["gate32"]),
                 "MC_EPI_BIAS_GATE_RESID_BF16": (side["old16"], side["gate16"])}.get(epi, (None, None))
    out = epilogue_model(epi, acc32, bias, old, gate, mutant)
    if epi in ACT:
        out = out[1]
    ok, _, _ = epilogue_ok(epi, out, acc32, bias, old, gate)
    return bool(ok.all())


MUTANTS = [("tanh_hi", ["MC_EPI_BIAS_GELU_BF16"]), ("tanh_lo", ["MC_EPI_BIAS_GELU_BF16"]),
           ("truncate", ["MC_EPI_BIAS_BF16", "MC_EPI_ROWBIAS_BF16", "MC_EPI_BIAS_GELU_BF16", "MC_EPI_BIAS_GATE_RESID_BF16"]),
           ("bias_after_round", ["MC_EPI_BIAS_BF16", "MC_EPI_BIAS_F32", "MC_EPI_BIAS_GELU_BF16", "MC_EPI_BIAS_SILU_BF16"]),
           ("unrounded_act", ["MC_EPI_BIAS_GELU_BF16", "MC_EPI_BIAS_GELU_ERF_BF16", "MC_EPI_BIAS_SILU_BF16"]),
           ("fused_gate", ["MC_EPI_BIAS_GATE_RESID"]), ("no_inner_round", ["MC_EPI_BIAS_GATE_RESID_BF16"])]


def test_readout_checkers_reject_each_modelled_mutant():
    """CPU: the faithful models of every chain pass the checkers over both passes of the sweep, and each modelled defect fails
    on at least one pass. Three kinds of defect (tanh off by 2^-11, a truncating store, the activation of the unrounded
    pre-activation) pass the fp64 bounds of test_kernel_bounds_gpu and test_kernels_gpu on random operands like theirs: the gap
    this module closes. The bias added after rounding acc does not: those bounds catch it where acc and bias nearly cancel."""
    g = torch.Generator().manual_seed(0)
    passes = _passes_cpu(g)
    for name, acc32, bias, side in passes:
        for epi in EPIS:
            assert _model_ok(epi, acc32, bias, side), (name, epi, "the faithful model fails its own checker")
    for mutant, epis in MUTANTS:
        for epi in epis:
            assert not all(_model_ok(epi, acc32, bias, side, mutant) for _, acc32, bias, side in passes), (mutant, epi)

    # the defects against the fp64 bounds on random operands (test_kernel_bounds_gpu._gemm_case: a ~ N(0, 1), b ~ N(0, 1 / K),
    # a bf16-valued bias ~ N(0, 1)), with an fp32 accumulator as the kernel's
    M, N, K = 256, 256, 64
    a = torch.randn(M, K, generator=g).to(BF).double()
    b = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(BF).double()
    bias = torch.randn(N, generator=g).to(BF).float()
    acc64 = a @ b.t()
    acc32, pre64 = acc64.float(), acc64 + bias.double()
    for mutant, epis in MUTANTS:
        for epi in epis:
            if epi not in ("MC_EPI_BIAS_BF16", "MC_EPI_BIAS_GELU_BF16", "MC_EPI_BIAS_GELU_ERF_BF16", "MC_EPI_BIAS_SILU_BF16"):
                continue
            out = epilogue_model(epi, acc32, bias[None, :], mutant=mutant)
            got = (out[1] if epi in ACT else out).double()
            ok = bool(gemm_fp64_bounds_ok(epi, got, pre64).all())
            if epi == "MC_EPI_BIAS_BF16":
                assert ok == (bf16_ulp_close(got.to(BF), pre64.float())[0] == 0), (mutant, epi)
            # rounding acc before the bias costs up to half an ulp of acc, which is many ulps of acc + bias where the two
            # nearly cancel: random operands meet such elements (about 5 % here), so the fp64 bounds already catch that one
            assert ok == (mutant != "bias_after_round"), (mutant, epi, "the fp64 bounds " + ("miss it" if ok else "catch it"))
