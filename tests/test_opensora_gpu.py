"""Open-Sora (STDiT3) on the H100: the head_dim-72 kernels against fp64 torch, the LN + t2i_modulate mode bit-equal to its
emulation, and the patched forward against the restatement of eval/magcache/experiments/opensora.py:229-373 (tests/opensora_ref.py)
through a miss / hit loop, at a reduced size, at the real width and for one block pair at the 480p shape."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

import magcache_b200 as mc
from magcache_b200 import ops

import opensora_emu
import opensora_ref as R

pytestmark = pytest.mark.gpu
dev = "cuda"


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _sdpa_err(q, k, v, ref64):
    """torch SDPA's own bf16 error against fp64 on the same operands: the yardstick of the attention kernels."""
    return rel(F.scaled_dot_product_attention(q, k, v), ref64)


def _heads(t, H):
    return t.view(t.shape[0], H, 72).transpose(0, 1)


@pytest.mark.parametrize("kind", ["spatial", "cross"])
def test_varlen_attention_d72(kind):
    torch.manual_seed(0)
    H = 16
    if kind == "spatial":
        qlens = [1590, 1590, 77, 200]
        klens = qlens
    else:
        qlens = [3000, 2500]
        klens = [300, 173]
    Lq, Lk = sum(qlens), sum(klens)
    q = torch.randn(Lq, 3 * H * 72, device=dev).bfloat16()[:, : H * 72]  # a column slice with a row stride, like q of q|k|v
    k = torch.randn(Lk, H * 72, device=dev).bfloat16()
    v = torch.randn(Lk, H * 72, device=dev).bfloat16()
    segs, qs, ks = [], 0, 0
    for ql, kl in zip(qlens, klens):
        segs.append((qs, ql, qs if kind == "spatial" else ks, kl))
        qs, ks = qs + ql, ks + kl
    out = ops.attention_varlen_d72(q, k, v, H, torch.tensor(segs, dtype=torch.int32, device=dev), max(qlens))
    for qs, ql, ks, kl in segs:
        qh, kh, vh = _heads(q[qs:qs + ql], H), _heads(k[ks:ks + kl], H), _heads(v[ks:ks + kl], H)
        r64 = F.scaled_dot_product_attention(qh.double(), kh.double(), vh.double())
        e_sdpa = _sdpa_err(qh, kh, vh, r64)
        e = rel(_heads(out[qs:qs + ql], H), r64)
        assert e <= 2 * e_sdpa + 1e-6, (kind, ql, kl, e, e_sdpa)


@pytest.mark.parametrize("T,S", [(15, 1590), (7, 333), (32, 40)])
def test_temporal_attention_d72(T, S):
    torch.manual_seed(1)
    B, H = 2, 16
    q, k, v = (torch.randn(B * T * S, H * 72, device=dev).bfloat16() for _ in range(3))
    out = ops.attention_temporal_d72(q, k, v, H, B, T, S)
    seq = lambda t: t.view(B, T, S, H, 72).permute(0, 2, 3, 1, 4).reshape(B * S, H, T, 72)  # noqa: E731
    r64 = F.scaled_dot_product_attention(seq(q).double(), seq(k).double(), seq(v).double())
    e_sdpa = _sdpa_err(seq(q), seq(k), seq(v), r64)
    assert rel(seq(out), r64) <= 2 * e_sdpa + 1e-6


@pytest.mark.parametrize("rope", [False, True])
def test_rmsnorm72_rope(rope):
    torch.manual_seed(2)
    B, T, S, H = 2, 5, 37, 16
    x = torch.randn(B * T * S, 3 * H * 72, device=dev).bfloat16()
    w = (1 + 0.2 * torch.randn(72, device=dev)).bfloat16()
    norm = R.LlamaRMSNorm(72).to(dev).bfloat16().requires_grad_(False)
    norm.weight.copy_(w)
    q = x[:, : H * 72].view(B, T, S, H, 72).permute(0, 2, 3, 1, 4).reshape(B * S, H, T, 72)  # the reference's (B S) H T D view
    ref = norm(q)
    if rope:
        ref = R.RotaryEmbedding(72).rotate_queries_or_keys(ref)
    cs = mc.opensora.rope_table(T, 72, dev) if rope else None
    got = ops.rmsnorm_head72_rope_(x[:, : H * 72], w.float(), H, cs, pos_div=S)
    got = got.view(B, T, S, H, 72).permute(0, 2, 3, 1, 4).reshape(B * S, H, T, 72)
    ulp = (ref.float().abs().clamp_min(1e-30).log2().floor() - 7).exp2()
    err = ((got.float() - ref.float()).abs() / ulp)
    assert float(err.max()) <= 2.0
    assert float((err > 0).float().mean()) < 0.01


def test_ln_t2i_modulate_matches_emulation():
    """Every step after the LayerNorm statistics is a correctly rounded bf16 op in both; the statistics are fp32 sums in a different
    order, so LN(x) * (1 + scale) may land on the other side of a bf16 rounding boundary: at most an ulp of that product (which the
    final add can cancel down to a small result), rarely."""
    torch.manual_seed(3)
    x = (3 * torch.randn(4099, 1152, device=dev) + 0.5).bfloat16()
    em = (torch.randn(6, 1152, device=dev) * 0.5).bfloat16().float()
    got = ops.ln_t2i_modulate(x, em, 4, 3)
    want = opensora_emu.ln_t2i_modulate(x.cpu(), em.cpu(), 4, 3)
    g, w_ = got.cpu().float(), want.float()
    mag = torch.maximum(w_.abs(), (w_ - em[3].cpu()).abs())  # |result| and |LN(x) * (1 + scale)|
    ulp = (mag.clamp_min(1e-30).log2().floor() - 7).exp2()
    diff = (g - w_).abs() / ulp
    assert float(diff.max()) <= 2.0 and float((diff > 0).float().mean()) < 1e-3, (float(diff.max()), float((diff > 0).float().mean()))


def _run_pair(cfg, B, T, H, W, y_lens, calls, thresh=0.5, K=3, skip_time=2, L=None, cy=None, check_attrs=True):
    base = R.STDiT3(**cfg).init_synthetic(0)
    ref = copy.deepcopy(base).to(dev, torch.bfloat16)
    ref.__class__ = type("RefOS", (R.STDiT3,), {})
    R.install_magcache(ref.__class__, thresh=thresh, K=K, skip_time=skip_time)
    ref64 = copy.deepcopy(base).to(dev, torch.float64)
    ref64.__class__ = type("Ref64", (R.STDiT3,), {})
    R.install_magcache(ref64.__class__, thresh=thresh, K=K, skip_time=skip_time)
    ours = copy.deepcopy(base).to(dev, torch.bfloat16)
    ours.__class__ = type("OursOS", (R.STDiT3,), {})
    mc.init_magcache_opensora(ours, thresh=thresh, K=K, skip_time=skip_time)
    g = torch.Generator().manual_seed(0)
    L = L or cfg["model_max_length"]
    x = torch.randn(B, 4, T, H, W, generator=g).to(dev)
    y = torch.randn(B, 1, L, cfg["caption_channels"], generator=g).to(dev)
    mask = torch.zeros(B, L, dtype=torch.long, device=dev)
    for b, n in enumerate(y_lens):
        mask[b, :n] = 1
    kw = dict(mask=mask, fps=torch.tensor([24.0], device=dev), height=torch.tensor([8.0 * H], device=dev), width=torch.tensor([8.0 * W], device=dev))
    skips = []
    with torch.no_grad():
        for i in range(calls):
            ts = torch.tensor([1000.0 - 33.0 * i, 990.0 - 29.0 * i][:B], device=dev)  # distinct per sample
            r = ref(x, ts, None, y, **kw)
            # the fp64 yardstick gets the timestep as the bf16 models see it (`timestep.to(dtype)`, :246)
            r64 = ref64(x.double(), ts.to(torch.bfloat16).double(), None, y.double(), **kw)
            o = ours(x, ts, None, y, **kw)
            skips.append(bool(ref.last_skip))
            e_ref = rel(r, r64)
            assert rel(o, r) <= 2 * e_ref + 1e-3 and rel(o, r64) <= 1.5 * e_ref + 1e-3, (i, rel(o, r), rel(o, r64), e_ref)
            if check_attrs:
                for a in ("t", "accumulated_sim", "accumulated_err", "accumulated_steps", "skip_steps"):
                    assert getattr(ours, a) == getattr(ref, a), (i, a)
    return skips


def test_forward_reduced_size_miss_hit():
    skips = _run_pair(R.CONFIGS["tiny"], 2, 5, 16, 22, (12, 9), calls=8)
    assert True in skips and False in skips


def test_forward_real_width_miss_hit():
    skips = _run_pair(R.CONFIGS["wide"], 2, 3, 20, 36, (20, 20), calls=5)
    assert True in skips and False in skips


def test_block_pair_full_480p_shape():
    """One spatial + temporal block pair at 60x106 latents, T = 15, B = 2 (47 700 rows, S = 1590) against fp64."""
    cfg = dict(R.CONFIGS["wide"], caption_channels=4096, model_max_length=300)
    _run_pair(cfg, 2, 15, 60, 106, (300, 300), calls=1, check_attrs=False)
