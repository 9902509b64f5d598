"""Open-Sora (STDiT3) engine orchestration on CPU: `magcache_opensora_forward` + `OpenSoraEngine` through the kernel emulation
(tests/emu_ops.py + tests/opensora_emu.py) against the restatement of eval/magcache/experiments/opensora.py:229-373 in
tests/opensora_ref.py — weight reading by the reference's names, B (T S) row order, per-sample modulation and gates, spatial /
temporal / varlen cross-attention segments, RoPE by frame, final layer and unpatchify, hit / miss and the controller attributes."""
import copy

import pytest
import torch

from magcache_b200 import opensora as os_mod
from magcache_b200 import patch as patch_mod

import magcache_b200 as mc
import opensora_emu
import opensora_ref as R


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(os_mod, "ops", opensora_emu.namespace())
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def _inputs(B, T, H, W, y_lens, L=12, cy=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, T, H, W, generator=g)
    y = torch.randn(B, 1, L, cy, generator=g)
    mask = torch.zeros(B, L, dtype=torch.long)
    for b, n in enumerate(y_lens):
        mask[b, :n] = 1
    return x, y, mask


def _pair(thresh=0.5, K=3, skip_time=2):
    base = R.STDiT3(**R.CONFIGS["tiny"]).init_synthetic(0)
    ref = copy.deepcopy(base).to(torch.bfloat16)
    ref.__class__ = type("RefOS", (R.STDiT3,), {})
    R.install_magcache(ref.__class__, thresh=thresh, K=K, skip_time=skip_time)
    ref64 = copy.deepcopy(base).double()
    ref64.__class__ = type("Ref64", (R.STDiT3,), {})
    R.install_magcache(ref64.__class__, thresh=thresh, K=K, skip_time=skip_time)
    ours = copy.deepcopy(base).to(torch.bfloat16)
    ours.__class__ = type("OursOS", (R.STDiT3,), {})
    patch_mod.init_magcache_opensora(ours, thresh=thresh, K=K, skip_time=skip_time)
    return ref, ref64, ours


ATTRS = ("t", "accumulated_sim", "accumulated_err", "accumulated_steps", "skip_steps")


@pytest.mark.parametrize("B,T,H,W,y_lens", [(2, 3, 6, 10, (12, 12)), (2, 3, 6, 10, (12, 7)), (1, 4, 4, 6, (9,)), (2, 5, 12, 24, (5, 12))],
                         ids=["B2-equal", "B2-unequal", "B1-evenT", "B2-S72-oddT"])
def test_engine_matches_oracle_over_miss_hit(emulated, B, T, H, W, y_lens):
    ref, ref64, ours = _pair()
    x, y, mask = _inputs(B, T, H, W, y_lens)
    kw = dict(mask=mask, fps=torch.tensor([24.0]), height=torch.tensor([8.0 * H]), width=torch.tensor([8.0 * W]))
    skips = []
    with torch.no_grad():
        for i in range(6):
            ts = torch.tensor([1000.0 - 37.0 * i, 990.0 - 29.0 * i][:B])  # distinct per sample: per-sample modulation and gates
            r = ref(x, ts, None, y, **kw)
            # the fp64 yardstick gets the timestep as the bf16 models see it (`timestep.to(dtype)`, :246)
            r64 = ref64(x.double(), ts.to(torch.bfloat16).double(), None, y.double(), **kw)
            o = ours(x, ts, None, y, **kw)
            skips.append(bool(ref.last_skip))
            assert bool(ref64.last_skip) == skips[-1]
            assert o.shape == r.shape and o.dtype == torch.float32
            e_ref = rel_l2(r, r64)
            assert rel_l2(o, r64) <= 1.5 * e_ref + 1e-3, (i, rel_l2(o, r64), e_ref)
            assert rel_l2(o, r) <= 2 * e_ref + 1e-3, (i, rel_l2(o, r), e_ref)
            for a in ATTRS:
                assert getattr(ours, a) == getattr(ref, a), (i, a)
            assert ours.residual_cache.shape == (B, T * (H // 2) * (W // 2), R.CONFIGS["tiny"]["hidden_size"], 1)
    assert True in skips and False in skips, skips


def test_replaced_residual_cache_is_read_at_last_index(emulated):
    ref, _, ours = _pair(thresh=10.0, K=5, skip_time=1)
    B, T, H, W = 2, 2, 4, 6
    x, y, mask = _inputs(B, T, H, W, (12, 12))
    kw = dict(mask=mask, fps=torch.tensor([24.0]), height=torch.tensor([32.0]), width=torch.tensor([48.0]))
    with torch.no_grad():
        ts = torch.full((B,), 900.0)
        ours(x, ts, None, y, **kw)
        ref(x, ts, None, y, **kw)
        fifo = torch.randn(*ours.residual_cache.shape[:-1], 3).to(torch.bfloat16)
        ours.residual_cache = fifo.clone()
        ref.residual_cache = fifo.clone()
        o = ours(x, ts, None, y, **kw)
        r = ref(x, ts, None, y, **kw)
    assert ref.last_skip
    assert rel_l2(o, r) < 2e-2


def test_invalidate_engine_repacks_changed_weights(emulated):
    """After a weight change and `invalidate_engine`, the next forward runs on the new weights (the engine holds a packed copy)."""
    ref, ref64, ours = _pair()
    B, T, H, W = 2, 3, 6, 10
    x, y, mask = _inputs(B, T, H, W, (12, 7))
    kw = dict(mask=mask, fps=torch.tensor([24.0]), height=torch.tensor([8.0 * H]), width=torch.tensor([8.0 * W]))
    ts = torch.tensor([1000.0, 990.0])

    def run():
        return ref(x, ts, None, y, **kw), ref64(x.double(), ts.to(torch.bfloat16).double(), None, y.double(), **kw), ours(x, ts, None, y, **kw)

    with torch.no_grad():
        run()
        for m in (ref, ref64, ours):
            for p in m.final_layer.parameters():
                p.mul_(2.0)
        mc.invalidate_engine(ours)
        r, r64, o = run()
    assert not ref.last_skip
    e_ref = rel_l2(r, r64)
    assert rel_l2(o, r64) <= 1.5 * e_ref + 1e-3, (rel_l2(o, r64), e_ref)


def test_token_shard_rejected(emulated):
    """The Open-Sora engine has no token-sharded path: a shard over more than one rank raises instead of having every rank compute
    the whole video, and `enable_token_shard` after the first forward raises like for the other engines."""
    _, _, ours = _pair()
    x, y, mask = _inputs(1, 2, 4, 6, (9,))
    kw = dict(mask=mask, fps=torch.tensor([24.0]), height=torch.tensor([32.0]), width=torch.tensor([48.0]))
    mc.enable_token_shard(ours, 0, 2)
    with pytest.raises(NotImplementedError, match="token sharding"), torch.no_grad():
        ours(x, torch.tensor([900.0]), None, y, **kw)
    _, _, ours = _pair()
    with torch.no_grad():
        ours(x, torch.tensor([900.0]), None, y, **kw)
    with pytest.raises(RuntimeError, match="before the first forward"):
        mc.enable_token_shard(ours, 0, 2)


def test_unsupported_inputs_raise():
    class M:
        parallel_manager = None
    x = torch.zeros(1, 4, 1, 4, 4)
    with pytest.raises(NotImplementedError, match="x_mask"):
        patch_mod.magcache_opensora_forward(M(), x, None, None, None, x_mask=torch.ones(1, 1, dtype=torch.bool))
    for sp, cp in ((2, 1), (1, 2)):
        m = M()
        m.parallel_manager = type("PM", (), dict(sp_size=sp, cp_size=cp))()
        with pytest.raises(NotImplementedError, match="parallelism"):
            patch_mod.magcache_opensora_forward(m, x, None, None, None)


def test_weights_reject_other_head_dims():
    m = R.STDiT3(hidden_size=128, depth=1, num_heads=2, caption_channels=16, model_max_length=4)
    with pytest.raises(NotImplementedError, match="head_dim"):
        os_mod.OpenSoraWeights.from_module(m, "cpu")
