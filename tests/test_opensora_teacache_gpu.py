"""Open-Sora's TeaCache comparator on the H100: the fused LN + t2i_modulate + input-distance kernel (`mc_ln_t2i_modulate_rel_l1`)
against `mc_ln_modulate` mode 2 and fp64 sums, with fenced outputs, and `teacache_opensora_forward` over a 30-call video against the
restatement of eval/magcache/experiments/opensora.py:34-227 (tests/opensora_tea_ref.py): decisions equal, `rel` within two bf16 ulps,\noutputs per the project's criterion, and a TeaCache miss bit-equal to the MagCache engine's miss."""
import copy

import pytest
import torch

import magcache_b200 as mc
from magcache_b200 import ops
from magcache_b200.controller import opensora_rel_l1

import opensora_ref as R
import opensora_tea_ref as TR
from test_kernel_bounds_gpu import _rb, check_fence, fenced

pytestmark = pytest.mark.gpu
dev = "cuda"


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("cols", [144, 1152])
@pytest.mark.parametrize("rows", [1, 5, 1029, 47700])
def test_fused_distance_kernel(rows, cols):
    """rows 1 and 5 leave most warps of the grid idle, 1029 is not a multiple of 8, 47 700 is one 480p sample pair's rows."""
    g = torch.Generator(device=dev).manual_seed(rows + cols)
    x, _ = fenced((rows, cols), torch.bfloat16, (1, 1, 0, 0), pitch=cols)
    x.copy_((3 * torch.randn(rows, cols, device=dev, generator=g) + 0.5).bfloat16())
    prev, _ = fenced((rows, cols), torch.bfloat16, (1, 1, 0, 0), pitch=cols)
    prev.copy_(torch.randn(rows, cols, device=dev, generator=g).bfloat16())
    em = (0.5 * torch.randn(6, cols, device=dev, generator=g)).bfloat16().float()
    out, obuf = fenced((rows, cols), torch.bfloat16, (2, 2, 0, 0), fill="fence", pitch=cols)
    partials = ops.rel_l1_partials(dev)
    sums = torch.zeros(2, dtype=torch.float64, device=dev)
    ops.ln_t2i_modulate_rel_l1(x, em, 1, 0, prev, out, partials, sums)
    check_fence(out, obuf)
    want = ops.ln_t2i_modulate(x, em, 1, 0)
    assert torch.equal(out.view(torch.int16), want.view(torch.int16))
    d64 = _rb(out.double() - prev.double()).abs().sum()
    p64 = prev.double().abs().sum()
    got = sums.cpu()
    assert abs(float(got[0]) - float(d64)) <= 1e-6 * float(d64) and abs(float(got[1]) - float(p64)) <= 1e-6 * float(p64), (got, d64, p64)
    again = torch.zeros(2, dtype=torch.float64, device=dev)
    out2 = torch.empty_like(want)
    ops.ln_t2i_modulate_rel_l1(x, em, 1, 0, prev, out2, partials, again)
    assert torch.equal(again.view(torch.int64), sums.view(torch.int64)) and torch.equal(out2.view(torch.int16), want.view(torch.int16))
    # per-sample launches add into one pair of sums
    if rows >= 2:
        h = rows // 2
        both = torch.zeros(2, dtype=torch.float64, device=dev)
        out3 = torch.empty_like(want)
        ops.ln_t2i_modulate_rel_l1(x[:h].contiguous(), em, 1, 0, prev[:h].contiguous(), out3[:h], partials, both)
        ops.ln_t2i_modulate_rel_l1(x[h:].contiguous(), em, 1, 0, prev[h:].contiguous(), out3[h:], partials, both)
        assert torch.allclose(both, sums, rtol=1e-9, atol=0)


def _run(cfg, B, T, H, W, calls, thresh, L=None):
    base = R.STDiT3(**cfg).init_synthetic(0)
    with torch.no_grad():
        for n, p in base.named_parameters():
            if n.startswith("t_block."):
                p.mul_(0.05)
    ref = copy.deepcopy(base).to(dev, torch.bfloat16)
    ref.__class__ = type("RefTea", (R.STDiT3,), {})
    TR.install_teacache(ref.__class__, thresh)
    ref64 = copy.deepcopy(base).to(dev, torch.float64)
    ref64.__class__ = type("RefTea64", (R.STDiT3,), {})
    TR.install_teacache(ref64.__class__, thresh)
    ref64.decisions_from = ref
    ours = copy.deepcopy(base).to(dev, torch.bfloat16)
    ours.__class__ = type("OursTea", (R.STDiT3,), {})
    mc.init_teacache_opensora(ours, rel_l1_thresh=thresh)
    mag = copy.deepcopy(base).to(dev, torch.bfloat16)
    mag.__class__ = type("OursMag", (R.STDiT3,), {})
    mc.init_magcache_opensora(mag, thresh=0.0, K=0, skip_time=100)  # every call a miss
    g = torch.Generator().manual_seed(0)
    L = L or cfg["model_max_length"]
    x = torch.randn(B, 4, T, H, W, generator=g).to(dev)
    d = torch.randn(B, 4, T, H, W, generator=g).to(dev)
    y = torch.randn(B, 1, L, cfg["caption_channels"], generator=g).to(dev)
    mask = torch.ones(B, L, dtype=torch.long, device=dev)
    kw = dict(mask=mask, fps=torch.tensor([24.0], device=dev), height=torch.tensor([8.0 * H], device=dev), width=torch.tensor([8.0 * W], device=dev))
    ts = [torch.full((B,), (1.0 - i / calls) * 1000.0, device=dev) for i in range(calls)]  # the sampler's linear schedule, one t per pair
    all_ts = [int(t[0].to(torch.bfloat16).item()) for t in ts]
    calcs = []
    with torch.no_grad():
        for i in range(calls):
            lat = x + 0.004 * i * d
            r = ref(lat, ts[i], all_ts, y, **kw)
            r64 = ref64(lat.double(), ts[i].to(torch.bfloat16).double(), all_ts, y.double(), **kw)
            res_before = ours.previous_residual
            o = ours(lat, ts[i], all_ts, y, **kw)
            assert (ours.previous_residual is not res_before) == ref.last_calc, i  # a compute stores a new residual view
            calcs.append(ref.last_calc)
            e_ref = rel(r, r64)
            assert rel(o, r) <= 2 * e_ref + 1e-3 and rel(o, r64) <= 1.5 * e_ref + 1e-3, (i, rel(o, r), rel(o, r64), e_ref)
            eng = ours._mc_opensora_engine
            if ref.last_rel is not None:
                # `rel` is the quotient of two means that are each rounded to bf16, over inputs whose LN statistics are fp32 sums in
                # another order than torch's: each mean can land one bf16 step away, so the quotient can differ by up to two ulps
                ulp = 2.0 ** (torch.tensor(ref.last_rel).abs().log2().floor().item() - 7)
                sums = eng.tea_sums.tolist()
                assert abs(opensora_rel_l1(sums[0], sums[1], eng.R * eng.w.dim) - ref.last_rel) <= 2 * ulp, i
            if ref.last_calc:  # the TeaCache miss is the MagCache engine's miss, bit for bit
                m = mag(lat, ts[i], all_ts, y, **kw)
                assert torch.equal(o, m), i
    assert True in calcs and False in calcs, calcs
    return calcs


def test_forward_reduced_size_video():
    _run(R.CONFIGS["tiny"], 2, 5, 16, 22, 30, 0.2)


def test_forward_real_width_video():
    _run(R.CONFIGS["wide"], 2, 3, 20, 36, 30, 0.1)
