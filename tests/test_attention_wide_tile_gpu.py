"""attn_kernel<176>, the 176-key KV tile that long key sequences and the rotated / flag-gated key order run on, read back and
bounded like the other widths: the softmax readout against fp64 (test_attention_readout_gpu's oracles and bounds: P is still
rounded to bf16 against the running max of its own tile, only the tiles are wider), and the fenced edge shapes of
test_kernel_bounds_gpu around one and two 176-key tiles. MC_ATTN_KERNEL=3 forces the width onto short key ranges."""
import math

import pytest
import torch

from test_attention_readout_gpu import (DEV, Readout, _attn_readout, _bf16_trunc, attn_bound, coverage_passes, logit_operands, logits32,  # noqa: E402
                                         model_attn, probs64, readout_passes)
from test_kernel_bounds_gpu import _attn_check  # noqa: E402

_SCALES = (1.0 / math.sqrt(128), 0.3)


def test_readout_model_of_the_176_key_tile():
    """CPU: the torch model of the rounding chain at 176-key tiles (unsplit, and 3-way split in rotated order) passes the
    readout and coverage oracles; P truncated to bf16, a dropped tile and an unmasked pad tile fail them."""
    g = torch.Generator().manual_seed(176)
    Lq, Lk, scale = 64, 1300, 0.3  # 8 tiles of 176 keys, the last holding 68
    q, k = logit_operands(Lq, Lk, 128, scale, "random", g, device="cpu")
    p64, x = probs64(q, k, scale), logits32(q, k, scale)
    qu, ku = logit_operands(Lq, Lk, 128, scale, "uniform", g, device="cpu")
    xu = logits32(qu, ku, scale)
    for kw in (dict(tile=176), dict(tile=176, rot=3, splits=3)):
        assert readout_passes(model_attn(x, **kw), p64, attn_bound(0)), kw
        assert coverage_passes(model_attn(xu, **kw), Lk), kw
    for kw in (dict(tile=176, p_round=_bf16_trunc), dict(tile=176, drop_tile=2, rot=3, splits=3)):
        assert not readout_passes(model_attn(x, **kw), p64, attn_bound(0)), kw
    for kw in (dict(tile=176, unmask_pad=True), dict(tile=176, unmask_pad=True, rot=3, splits=3)):
        assert not coverage_passes(model_attn(xu, **kw), Lk), kw


@pytest.mark.gpu
def test_readout_wide_kernel(monkeypatch):
    """MC_ATTN_KERNEL=3, unsplit: Lk in {176, 177, 352, 1025, 1500, 4095} x Lq in {1, 127, 300}, random logits and q = 0,
    rising and falling ramps; and the default choice at Lk 1025 (176-key tiles)."""
    monkeypatch.setenv("MC_ATTN_SPLITS", "1")
    monkeypatch.setenv("MC_ATTN_KERNEL", "3")
    g = torch.Generator(device=DEV).manual_seed(176)
    ro = Readout("attn_kernel<176>", attn_bound(0))
    for i, Lk in enumerate((176, 177, 352, 1025, 1500, 4095)):
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
@pytest.mark.parametrize("splits", [0, 3, 5])
def test_readout_wide_kernel_split_and_rotated(splits, monkeypatch):
    """Split-KV partials (the default plan at Lq 128 x 32 heads, Lk 4095: 24 tiles split 4 ways; forced 3 / 5 ways) and the
    rotated key order (`first_key_row` in {1, 175, 176, 177, Lk - 1}) on 176-key tiles, ragged Lk 1025 / 1500."""
    monkeypatch.delenv("MC_ATTN_KERNEL", raising=False)
    monkeypatch.delenv("MC_ATTN_EMU", raising=False)
    g = torch.Generator(device=DEV).manual_seed(17600 + splits)
    ro = Readout(f"attn_kernel<176> + attn_combine_kernel, splits {splits}", attn_bound(0))
    if splits:
        monkeypatch.setenv("MC_ATTN_SPLITS", str(splits))
    else:
        monkeypatch.delenv("MC_ATTN_SPLITS", raising=False)
        for kind in ("random", "rise", "fall", "uniform"):
            _attn_readout(128, 4095, 0.3, kind, g, ro)
    for Lk in (1025, 1500):
        for first in (1, 175, 176, 177, Lk - 1):
            for kind in ("random", "uniform"):
                _attn_readout(127, Lk, 0.3, kind, g, ro, first_key_row=first)
        _attn_readout(300, Lk, 0.3, "rise", g, ro, first_key_row=700)
    ro.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [1, 3])
def test_readout_wide_kernel_flag_gated(splits, monkeypatch):
    """The flag-gated order on 176-key tiles, every flag already at the epoch: bit-equal to the same call without flags (same
    `first_key_row`); seg_rows 300 / 500 are not multiples of 176."""
    monkeypatch.setenv("MC_ATTN_KERNEL", "3")
    monkeypatch.delenv("MC_ATTN_EMU", raising=False)
    monkeypatch.setenv("MC_ATTN_SPLITS", str(splits))
    ro = Readout(f"attn_kernel<176> flag-gated, MC_ATTN_SPLITS={splits}", attn_bound(0))
    epoch = 7
    for Lk in (1025, 1500):
        for seg_rows in (300, 500):
            n_seg = -(-Lk // seg_rows)
            fbuf = torch.full((n_seg + 128,), epoch, dtype=torch.int32, device=DEV)
            flags = (fbuf[64:64 + n_seg], torch.full((1,), epoch, dtype=torch.int32, device=DEV), seg_rows)
            for first in (0, 177, Lk - 1):
                for kind in ("random", "uniform"):
                    seed = Lk + seg_rows + first + splits
                    a = _attn_readout(127, Lk, 0.3, kind, torch.Generator(device=DEV).manual_seed(seed), ro, first_key_row=first, flags=flags)
                    b = _attn_readout(127, Lk, 0.3, kind, torch.Generator(device=DEV).manual_seed(seed), ro, first_key_row=first)
                    assert torch.equal(a, b), (Lk, seg_rows, first, kind, "flag-gated result differs from the ungated one")
            assert bool((fbuf == epoch).all())
    ro.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [1, 24])
def test_attention_wide_kernel_ragged_fenced(heads, monkeypatch):
    """MC_ATTN_KERNEL=3 at Lk in {1, 24, 175, 176, 177, 352, 353} x Lq in {1, 65, 128, 300}, K / V as views with NaN rows after
    Lk, the output a fenced window; Lk = 1 is exact, and a 40-logit peak in the last full tile and in the ragged tile must
    return that key's V row. Each result bit-reproducible."""
    monkeypatch.setenv("MC_ATTN_KERNEL", "3")
    monkeypatch.setenv("MC_ATTN_SPLITS", "1")
    g = torch.Generator(device=DEV).manual_seed(1760 + heads)
    for scale in (0.05, 0.3):
        for Lk in (1, 24, 175, 176, 177, 352, 353):
            for Lq in (1, 65, 128, 300):
                _attn_check(Lq, Lk, heads, scale, g)
        for Lk, peak in ((176, 175), (176, 88), (177, 176), (353, 352), (353, 351), (352, 176), (24, 23)):
            _attn_check(65, Lk, heads, scale, g, peak=peak)
    monkeypatch.setenv("MC_ATTN_SPLITS", "3")
    a = _attn_check(300, 1500, heads, 0.3, torch.Generator(device=DEV).manual_seed(1))
    b = _attn_check(300, 1500, heads, 0.3, torch.Generator(device=DEV).manual_seed(1))
    assert torch.equal(a, b)
