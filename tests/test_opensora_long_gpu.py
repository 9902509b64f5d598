"""Open-Sora 1.2 videos of 8 s and longer (T = 60, 120, 240 latent frames) on the H100.

* `mc_attn_temporal_d72` past 32 frames (attn_temporal_mma_d72_kernel: the varlen kernel's tensor-core tile with strided rows)
  against fp64 SDPA, with NaN-poisoned input margins and fenced outputs, and bit-identical on a second launch;
* its softmax read back one probability per output element (the readout of test_attention_readout_gpu.py, V the identity along
  the frame axis over ceil(T / 72) passes), against the varlen chain's bound, and the coverage oracle at q = 0;
* the engine against the restatement (tests/opensora_ref.py) at hidden 1152 over MagCache miss / hit calls and a TeaCache miss,
  one spatial + temporal block pair at 480p x 8 s against fp64, and the full-size model over a 30-call 480p x 8 s video;
* the MLP's fc1 (GELU epilogue) -> fc2 (gated bf16 residual epilogue) over an `ff` buffer of more than 2^31 elements, the size
  the engine allocates at 720p x 16 s and 480p x 32 s."""
import contextlib
import copy
import io
import math

import pytest
import torch
import torch.nn.functional as F

import magcache_b200 as mc
from magcache_b200 import _lib as L
from magcache_b200 import ops

import opensora_ref as R
import opensora_tea_ref as TR
from test_attention_readout_gpu import ATTN_REL, Readout, check_coverage, logit_operands, probs64
from test_kernel_bounds_gpu import check_fence, fenced, gemm_fp64_bounds_ok
from test_opensora_gpu import _run_pair

pytestmark = pytest.mark.gpu
dev = "cuda"
BF = torch.bfloat16


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _seq(t, B, T, S, H):
    """B (T S) C rows -> [B*S, H, T, 72]: the reference's `(B S) T C` view per head."""
    return t.reshape(B, T, S, H, 72).permute(0, 2, 3, 1, 4).reshape(B * S, H, T, 72)


# ------------------------------------------------------------------------------------------- the kernel against fp64
@pytest.mark.parametrize("T", [33, 48, 63, 64, 65, 120, 128, 129, 240])
def test_temporal_long_fenced(T):
    """heads 1 / 16, S 1 / 7, B 1 / 2: q / k / v column views with NaN on both sides and a NaN row after the last, fenced output.
    Overall within twice bf16 SDPA's error of fp64; elementwise within P's bf16 rounding (2^-9 sum_j p_j |v_j|) and the output's
    (2^-9 |o|), each doubled for the fp32 chain; a second launch gives the same bits."""
    scale = 1.0 / math.sqrt(72)
    g = torch.Generator(device=dev).manual_seed(T)
    for heads in (1, 16):
        for S in (1, 7):
            for B in (1, 2):
                rows, W = B * T * S, heads * 72
                qkv = []
                for _ in range(3):
                    t, _ = fenced((rows, W), BF, (0, 1, 8, 8))
                    t.copy_(1.5 * torch.randn(rows, W, device=dev, generator=g))
                    qkv.append(t)
                q, k, v = qkv
                out, obuf = fenced((rows, W), BF, (1, 1, 8, 8), fill="fence")
                ops.attention_temporal_d72(q, k, v, heads, B, T, S, scale=scale, out=out)
                check_fence(out, obuf)
                what = (T, heads, S, B)
                assert bool(torch.isfinite(out.float()).all()), what
                sq, sk, sv = (_seq(x, B, T, S, heads) for x in (q, k, v))
                p64 = torch.softmax((sq.double() @ sk.double().transpose(-1, -2)) * scale, -1)
                r64 = p64 @ sv.double()
                err = (_seq(out, B, T, S, heads).double() - r64).abs()
                bound = (p64 @ sv.double().abs()) * 2.0 ** -8 + r64.abs() * 2.0 ** -8 + 1e-6
                assert bool((err <= bound).all()), (what, float((err / bound).max()))
                e_sdpa = rel(F.scaled_dot_product_attention(sq, sk, sv, scale=scale), r64)
                assert rel(_seq(out, B, T, S, heads), r64) <= 2 * e_sdpa + 1e-6, what
                first = out.clone()
                ops.attention_temporal_d72(q, k, v, heads, B, T, S, scale=scale, out=out)
                assert torch.equal(out.view(torch.int16), first.view(torch.int16)), (what, "a second launch differs")


# ------------------------------------------------------------------------------------------- the softmax readout
@pytest.mark.parametrize("T", [33, 64, 65, 120, 129, 240])
def test_readout_temporal_long(T):
    """V is the identity along the frame axis in pass p: V[b, t, s, h, d] = [d == t - 72 p], so out[..., d] of pass p is the
    probability of key 72 p + d. Every probability within the varlen chain's (2^-7 + 2e-4) p64 (P rounded to bf16 for PV, the
    output rounded to bf16), the mean signed relative error within 5e-4; q = 0 gives bf16(1 / T) within one ulp."""
    H, D = 3, 72
    ro = Readout(f"attn_temporal_mma_d72 T={T}", ATTN_REL)
    g = torch.Generator(device=dev).manual_seed(1000 + T)
    passes = -(-T // D)
    for B, S in ((1, 1), (2, 7)):
        for scale, kind in ((1.0 / math.sqrt(D), "random"), (0.3, "random"), (0.3, "rise"), (0.3, "fall"), (0.3, "uniform")):
            qs, ks = logit_operands(T, T, D, scale, kind, g, batch=(B, S, H))  # [B, S, H, T, D]
            rows = lambda t: t.permute(0, 3, 1, 2, 4).reshape(B * T * S, H * D).contiguous()  # noqa: E731  (b, t, s) rows
            p64 = None if kind == "uniform" else probs64(qs, ks, scale)
            for p in range(passes):
                n = min(D, T - D * p)
                vs = torch.zeros(B, S, H, T, D, dtype=BF, device=dev)
                vs[..., D * p + torch.arange(n, device=dev), torch.arange(n, device=dev)] = 1.0
                out = torch.full((B * T * S, H * D), float("nan"), dtype=BF, device=dev)
                ops.attention_temporal_d72(rows(qs), rows(ks), rows(vs), H, B, T, S, scale=scale, out=out)
                o = out.reshape(B, T, S, H, D).permute(0, 2, 3, 1, 4)  # [B, S, H, T(query), D]
                what = (ro.label, B, S, scale, kind, p)
                assert bool((o[..., n:] == 0).all()), (what, "a column past the pass's keys is not 0")
                if p64 is None:
                    check_coverage(o[..., :n], T, what)
                else:
                    ro.check(o[..., :n], p64[..., D * p:D * p + n], what)
    ro.finish()


# ------------------------------------------------------------------------------------------- the engine
_WIDE2 = dict(R.CONFIGS["wide"], depth=2)


@pytest.mark.parametrize("T", [60, 120])
def test_forward_long_video_miss_hit(T):
    """hidden 1152, 2 block pairs, 8 x 12 latents (S = 24), B = 2: MagCache miss / hit calls against the restatement."""
    skips = _run_pair(_WIDE2, 2, T, 8, 12, (20, 13), calls=5)
    assert True in skips and False in skips, skips


@pytest.mark.parametrize("T", [60, 120])
def test_teacache_long_video(T):
    """`teacache_opensora_forward` at T > 32: the forced first call and a distance call, per the project's criterion."""
    cfg, B, H, W = _WIDE2, 2, 8, 12
    base = R.STDiT3(**cfg).init_synthetic(0)
    models = []
    for name, dtype in (("RefTeaL", BF), ("RefTeaL64", torch.float64)):
        m = copy.deepcopy(base).to(dev, dtype)
        m.__class__ = type(name, (R.STDiT3,), {})
        TR.install_teacache(m.__class__, 0.1)
        models.append(m)
    ref, ref64 = models
    ref64.decisions_from = ref
    ours = copy.deepcopy(base).to(dev, BF)
    ours.__class__ = type("OursTeaL", (R.STDiT3,), {})
    mc.init_teacache_opensora(ours, rel_l1_thresh=0.1)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 4, T, H, W, generator=g).to(dev)
    d = torch.randn(B, 4, T, H, W, generator=g).to(dev)
    y = torch.randn(B, 1, cfg["model_max_length"], cfg["caption_channels"], generator=g).to(dev)
    mask = torch.ones(B, cfg["model_max_length"], dtype=torch.long, device=dev)
    kw = dict(mask=mask, fps=torch.tensor([24.0], device=dev), height=torch.tensor([8.0 * H], device=dev), width=torch.tensor([8.0 * W], device=dev))
    ts = [torch.full((B,), 1000.0, device=dev), torch.full((B,), 966.5, device=dev)]
    all_ts = [1000, 966, 933]
    forced = []
    with torch.no_grad():
        for i in range(2):
            lat = x + 0.004 * i * d
            r = ref(lat, ts[i], all_ts, y, **kw)
            r64 = ref64(lat.double(), ts[i].to(BF).double(), all_ts, y.double(), **kw)
            o = ours(lat, ts[i], all_ts, y, **kw)
            forced.append(ref.last_forced)
            e_ref = rel(r, r64)
            assert rel(o, r) <= 2 * e_ref + 1e-3 and rel(o, r64) <= 1.5 * e_ref + 1e-3, (i, rel(o, r), rel(o, r64), e_ref)
            assert float(ours.accumulated_rel_l1_distance) == float(ref.accumulated_rel_l1_distance), i
    assert forced == [True, False], forced


@contextlib.contextmanager
def _batched_fp64_sdpa(max_bytes=4 << 30):
    """fp64 SDPA (torch's math path materialises [N, H, Lq, Lk]) over slices of the leading dimension; the result is the same,
    the peak memory of the 480p x 8 s spatial attention (120 frames x 16 heads x 1590^2 in fp64) is not."""
    sdpa = F.scaled_dot_product_attention

    def sliced(q, k, v, *a, **kw):
        if q.dtype != torch.float64 or q.dim() != 4:
            return sdpa(q, k, v, *a, **kw)
        per = q.shape[1] * q.shape[2] * k.shape[2] * 8 * 3
        n = max(1, max_bytes // per)
        return torch.cat([sdpa(q[i:i + n], k[i:i + n], v[i:i + n], *a, **kw) for i in range(0, q.shape[0], n)])

    F.scaled_dot_product_attention = sliced
    try:
        yield
    finally:
        F.scaled_dot_product_attention = sdpa


def test_block_pair_480p_8s():
    """One spatial + temporal block pair at 60 x 106 latents (S = 1590), T = 60, B = 2 (190 800 rows) at full width against fp64."""
    cfg = dict(R.CONFIGS["wide"], caption_channels=4096, model_max_length=300)
    with _batched_fp64_sdpa():
        _run_pair(cfg, 2, 60, 60, 106, (300, 300), calls=1, check_attrs=False)


def test_full_model_video_480p_8s():
    """`magcache_opensora_forward` on the full-size STDiT3-XL/2 (random weights) over one 30-call video at 480p 9:16 x 8 s (T = 60,
    60 x 106 latents, B = 2, 300 caption tokens) under the slow preset: every output finite, the hits where the preset's schedule
    has them, and the call counter back at 0 after the video."""
    model = R.STDiT3(**R.CONFIGS["full"]).init_synthetic(0).to(dev, BF).eval()
    model.__class__ = type("OursFull", (R.STDiT3,), {})
    mc.init_magcache_opensora(model, thresh=0.12, K=3, skip_time=6)
    B, T, H, W, L_ = 2, 60, 60, 106, 300
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(B, 4, T, H, W, device=dev, generator=g)
    y = torch.randn(B, 1, L_, 4096, device=dev, generator=g)
    kw = dict(mask=torch.ones(B, L_, dtype=torch.long, device=dev), fps=torch.tensor([24.0], device=dev),
              height=torch.tensor([480.0], device=dev), width=torch.tensor([854.0], device=dev))
    hits = []
    with torch.no_grad():
        for i in range(30):
            with contextlib.redirect_stdout(io.StringIO()) as log:  # a hit prints its "skip time" line (:312)
                out = model(x, torch.full((B,), 1000.0 * (1 - i / 30), device=dev), None, y, **kw)
            hits.append(int(log.getvalue().startswith("skip time")))
            assert out.shape == (B, 8, T, H, W) and bool(torch.isfinite(out).all()), i
    assert hits == [int(v) for v in mc.PRESETS["opensora-slow-E012K3"].schedule()], hits
    assert model.t == 0


# ------------------------------------------------------------------------------------------- more than 2^31 elements
def test_mlp_over_2_31_elements():
    """fc1 (MC_EPI_BIAS_GELU_BF16) over M = 480 000 rows into ff [M, 4608] (2.21e9 elements), then fc2
    (MC_EPI_BIAS_GATE_RESID_BF16) per sample, as the engine launches them, in place on x. Rows at the start, the middle, across
    element 2^31 of ff and at the end checked against fp64 (`gemm_fp64_bounds_ok`)."""
    D, Dff, M = 1152, 4608, 480_000
    assert M * Dff > 2 ** 31
    g = torch.Generator(device=dev).manual_seed(31)
    h = torch.randn(M, D, device=dev, generator=g, dtype=BF)
    w1 = (torch.randn(Dff, D, device=dev, generator=g) / math.sqrt(D)).to(BF)
    b1 = torch.randn(Dff, device=dev, generator=g).to(BF).float()
    w2 = (torch.randn(D, Dff, device=dev, generator=g) / math.sqrt(Dff)).to(BF)
    b2 = torch.randn(D, device=dev, generator=g).to(BF).float()
    gates = [0.5 * torch.randn(D, device=dev, generator=g) for _ in range(2)]
    x = torch.randn(M, D, device=dev, generator=g, dtype=BF)
    edge = 2 ** 31 // Dff
    sample = torch.cat([torch.arange(0, 64), torch.arange(M // 2 - 32, M // 2 + 32), torch.arange(edge - 32, edge + 32),
                        torch.arange(M - 64, M)]).to(dev)
    x_old = x[sample].double()
    ff = torch.empty(M, Dff, device=dev, dtype=BF)
    ops.gemm(h, w1, b1, L.MC_EPI_BIAS_GELU_BF16, out=ff)
    half = M // 2
    for b in range(2):
        ops.gemm(ff[b * half:(b + 1) * half], w2, b2, L.MC_EPI_BIAS_GATE_RESID_BF16, out=x[b * half:(b + 1) * half], gate=gates[b])
    torch.cuda.synchronize()
    pre1 = h[sample].double() @ w1.double().T + b1.double()
    ok1 = gemm_fp64_bounds_ok("MC_EPI_BIAS_GELU_BF16", ff[sample].double(), pre1)
    assert bool(ok1.all()), ("fc1", sample[~ok1.all(1)][:8].tolist())
    pre2 = ff[sample].double() @ w2.double().T + b2.double()
    gate = torch.where((sample < half)[:, None], gates[0].double(), gates[1].double())
    ok2 = gemm_fp64_bounds_ok("MC_EPI_BIAS_GATE_RESID_BF16", x[sample].double(), pre2, x_old, gate)
    assert bool(ok2.all()), ("fc2", sample[~ok2.all(1)][:8].tolist())
