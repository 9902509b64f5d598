"""Token-sharded FLUX / Kontext / HunyuanVideo engines at image token counts that do not divide by the world size (the pad rule:
rank r owns image rows [r ceil(N/P), min((r+1) ceil(N/P), N)), the last rank fewer) against the single-engine run, over gloo at
world 2, 3 and 4 with the kernels emulated on CPU (tests/emu_ops.py and the ControlNet / LoRA / IP-Adapter / FP8 emulations built
on it). Also: the collective exchange's gathered key rows are exactly [all token rows | tail rows] with and without a pad, and a
count that leaves a rank without rows is refused on every rank."""
import copy
import os
import sys
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROWS_1 = {3: 7, 4: 10}  # image tokens that leave the last rank a single row: 3 + 3 + 1, 3 + 3 + 3 + 1


def _flux_model(fr):
    return fr.FluxTransformer2DModel(in_channels=64, num_layers=2, num_single_layers=2, num_attention_heads=2, joint_attention_dim=96,
                                     pooled_projection_dim=48).init_synthetic(0)


def _flux_inputs(fr, hw, ref_hw=None, n_txt=19, seed=3):
    """FLUX latent tokens (h x w); Kontext: the reference image's tokens behind them, first id coordinate 1."""
    g = torch.Generator().manual_seed(seed)
    img_ids, txt_ids = fr.make_ids(hw[0], hw[1], n_txt)
    if ref_hw is not None:
        ref_ids, _ = fr.make_ids(ref_hw[0], ref_hw[1], 0)
        ref_ids[:, 0] = 1
        img_ids = torch.cat([img_ids, ref_ids])
    hs = torch.randn(1, img_ids.shape[0], 64, generator=g).bfloat16()
    enc, pooled = torch.randn(1, n_txt, 96, generator=g).bfloat16(), torch.randn(1, 48, generator=g).bfloat16()
    return hs, enc, pooled, img_ids, txt_ids


def _hunyuan_model(hr):
    return hr.HYVideoDiffusionTransformer(hidden_size=256, heads_num=2, mm_double_blocks_depth=2, mm_single_blocks_depth=2, text_states_dim=96,
                                          text_states_dim_2=48).init_synthetic(0)


def _hunyuan_inputs(hr, grid, seed=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, 16, grid[0], 2 * grid[1], 2 * grid[2], generator=g).bfloat16()
    txt, pooled = torch.randn(1, 16, 96, generator=g).bfloat16(), torch.randn(1, 48, generator=g).bfloat16()
    mask = torch.zeros(1, 16, dtype=torch.long)
    mask[0, :11] = 1
    cos, sin = hr.rope_cos_sin(grid)
    return x, txt, mask, pooled, cos, sin


def _cases(world):
    """(name, family, shape, extra): every shape here has a pad at this world size."""
    one = ROWS_1.get(world)
    cases = [("flux", "flux", (7, 5), None), ("kontext", "flux", ((5, 5), (2, 5)), None), ("hunyuan", "hunyuan", (1, 5, 7), None)]
    if one is not None:
        cases += [("flux_one_row", "flux", (1, one), None), ("hunyuan_one_row", "hunyuan", (1, 1, one), None)]
    if world == 2:
        cases += [("controlnet", "flux", (7, 5), "controlnet"), ("ip_adapter", "flux", ((5, 5), (2, 5)), "ip_adapter"),
                  ("lora", "flux", (7, 5), "lora"), ("fp8", "hunyuan", (1, 5, 7), "fp8")]
    return cases


def _worker(rank, world, initfile, results):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import flux_ip_adapter_ref as ipr
    import flux_lora_ref as lr
    import hunyuan_fp8_ref as f8

    import magcache_b200 as mc
    from magcache_b200 import mmdit
    from magcache_b200 import patch as patch_mod
    from oracle import flux_ref as fr
    from oracle import hunyuan_ref as hr
    torch.set_num_threads(2)  # P ranks share the machine's cores
    dist.init_process_group("gloo", init_method=f"file://{initfile}", rank=rank, world_size=world)
    try:
        emu = ipr.emu  # emu_ops + the ControlNet addend, the LoRA tail and the IP-Adapter attention
        emu.dequant_fp8_bf16 = f8.emu_dequant_fp8_bf16
        mmdit.ops = emu
        patch_mod.ops = emu
        torch.Tensor.is_cuda = property(lambda self: True)
        out = {}
        for name, family, shape, extra in _cases(world):
            if family == "flux":
                hw, ref_hw = (shape if isinstance(shape[0], tuple) else (shape, None))
                model = _flux_model(fr)
                kw = {}
                if extra == "lora":
                    lr.inject_lora(model, "all", ("a", "b"), rank=12, seed=5)
                    kw = dict(joint_attention_kwargs={"scale": 0.7})
                elif extra == "ip_adapter":
                    model = ipr.load_ip_adapter(model, 2, [16, 4], seed=5)
                    kw = dict(joint_attention_kwargs={"ip_adapter_image_embeds": ipr.make_embeds(2, 2)})
                hs, enc, pooled, img_ids, txt_ids = _flux_inputs(fr, hw, ref_hw)
                n_img = img_ids.shape[0]

                def call(m, i, hs=hs, enc=enc, pooled=pooled, img_ids=img_ids, txt_ids=txt_ids, kw=kw, n_img=n_img, extra=extra):
                    if extra == "controlnet":
                        g = torch.Generator().manual_seed(1000 + i)
                        kw = dict(controlnet_block_samples=[(0.2 * torch.randn(1, n_img, 256, generator=g)).bfloat16() for _ in range(2)],
                                  controlnet_single_block_samples=[(0.2 * torch.randn(1, n_img, 256, generator=g)).bfloat16()])
                    return m(hs * (1 - 0.05 * i), enc, pooled, torch.tensor([1.0 - i / 6]), img_ids, txt_ids, torch.tensor([3.5]),
                             return_dict=False, **kw)[0]

                def install(m):
                    mc.init_magcache_flux(m, 6, thresh=10.0, K=2, retention_ratio=0.34)  # miss miss hit hit miss miss
                install_cal, eng_attr = mc.init_magcache_flux_calibration, "_mc_flux_engine"
            else:
                model = _hunyuan_model(hr)
                if extra == "fp8":
                    model = f8.to_fp8_checkpoint(model)
                x, txt, mask, pooled, cos, sin = _hunyuan_inputs(hr, shape)
                n_img = shape[0] * shape[1] * shape[2]

                def call(m, i, x=x, txt=txt, mask=mask, pooled=pooled, cos=cos, sin=sin):
                    return m(x * (1 - 0.05 * i), torch.tensor([900.0 - 100 * i]), txt, mask, pooled, cos, sin, torch.tensor([6000.0]),
                             return_dict=False)

                def install(m):
                    mc.init_magcache_hunyuan(m, 6, thresh=10.0, K=2, retention_ratio=0.34, mag_ratios=[1.0] * 6)
                install_cal, eng_attr = mc.init_magcache_hunyuan_calibration, "_mc_hunyuan_engine"
            outs = {}
            for which in ("single", "sharded"):
                m = copy.deepcopy(model)
                m.__class__ = type(f"M_{name}_{which}", (m.__class__,), {})
                install(m)
                if which == "sharded":
                    mc.enable_token_shard(m, rank, world)
                with torch.no_grad():
                    outs[which] = ([call(m, i).clone() for i in range(6)], getattr(m, eng_attr))
            eng = outs["sharded"][1]
            sh = eng.shard
            errs = [float((a.float() - b.float()).abs().max() / b.float().abs().max()) for a, b in zip(outs["sharded"][0], outs["single"][0])]
            full_res = outs["single"][1].res
            res_err = float((eng.res.float() - full_res[sh.start:sh.stop].float()).abs().max() / full_res.float().abs().max())
            same_shape = all(a.shape == b.shape for a, b in zip(outs["sharded"][0], outs["single"][0]))
            cal = None
            if extra is None:  # the calibration twin on a padded shard: the statistics' partial sums add over the ranks' own rows
                cal = {}
                for which in ("single", "sharded"):
                    m = copy.deepcopy(model)
                    m.__class__ = type(f"C_{name}_{which}", (m.__class__,), {})
                    install_cal(m, 5)
                    type(m).calibration_dir = None
                    if which == "sharded":
                        mc.enable_token_shard(m, rank, world)
                    with torch.no_grad():
                        for i in range(4):
                            call(m, i)
                    cal[which] = [list(getattr(m, k)) for k in ("norm_ratio", "norm_std", "cos_dis")]
                    ceng = getattr(m, eng_attr)
                    cal[which + "_n_img"] = ceng.n_img
            out[name] = dict(errs=errs, res_err=res_err, n_img=n_img, n_loc=eng.n_img, n_tot=eng.n_img_total, start=sh.start, pad=sh.pad,
                             s_keys=eng.S_keys, n_txt=eng.n_txt, same_shape=same_shape, cal=cal)
        results[rank] = out
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_padded_shard_equals_single(world):
    """Every rank's output over a miss, miss, hit, hit, miss, miss schedule, its residual-cache rows and the calibration lists
    against one engine's, at the existing sharded tests' bounds; ControlNet, IP-Adapter, LoRA and FP8 on a padded shard at world 2."""
    with tempfile.TemporaryDirectory() as d:
        results = mp.get_context("spawn").Manager().dict()
        mp.spawn(_worker, args=(world, os.path.join(d, "init"), results), nprocs=world, join=True)
        assert set(results.keys()) == set(range(world))
        names = [c[0] for c in _cases(world)]
        for name in names:
            per_rank = [results[r][name] for r in range(world)]
            n = per_rank[0]["n_img"]
            slots = -(-n // world)
            assert per_rank[0]["pad"] > 0, (name, world, "not a padded shape")
            # ownership follows TokenShard: consecutive ranges of ceil(N/P) rows, the last rank's cut at N
            assert [o["start"] for o in per_rank] == [r * slots for r in range(world)], name
            assert [o["n_loc"] for o in per_rank] == [min(slots, n - r * slots) for r in range(world)], name
            assert sum(o["n_loc"] for o in per_rank) == n
            if name.endswith("one_row"):
                assert per_rank[-1]["n_loc"] == 1
            for r, o in enumerate(per_rank):
                what = (name, world, r)
                assert o["n_tot"] == n and o["s_keys"] == n + o["n_txt"], what   # no pad row among the keys
                assert o["same_shape"], what
                assert len(o["errs"]) == 6 and max(o["errs"]) < 1.2e-2, (what, o["errs"])
                assert o["res_err"] < 3e-2, (what, o["res_err"])
                cal = o["cal"]
                if cal is not None:
                    assert cal["sharded_n_img"] == o["n_loc"] and cal["single_n_img"] == n, what  # the twin really ran sharded
                    assert all(len(v) == 3 for v in cal["single"]) and all(len(v) == 3 for v in cal["sharded"]), (what, cal)
                    for a, b in zip(sum(cal["sharded"], []), sum(cal["single"], [])):
                        assert abs(a - b) <= 2e-2 * abs(b) + 2e-3, (what, cal)


# ------------------------------------------------------------------------------------------- exchange layout
def _exchange_worker(rank, world, initfile, results):
    from magcache_b200.shard import CollectiveExchange, TokenShard
    dist.init_process_group("gloo", init_method=f"file://{initfile}", rank=rank, world_size=world)
    try:
        out = []
        width, extra = 16, 5
        for n in (4 * world, 4 * world - 1, 3 * world + 1):  # pad 0, 1 and P - 1 (the last rank owns 5 - P rows)
            sh = TokenShard(rank, world, n)
            g = torch.Generator().manual_seed(n)
            rows = torch.randn(n, width, generator=g).bfloat16()
            xch = CollectiveExchange(sh, width, (1,), "cpu", extra_rows=extra)
            for rep in range(3):
                tail = torch.randn(extra, width, generator=g).bfloat16()  # replicated: every rank draws the same
                xch.own_rows(rep % 2).copy_(sh.rows(rows) * (rep + 1))
                xch.tail_rows(rep % 2).copy_(tail)
                xch.begin(rep % 2)
                kv, kw = xch.keys_values(rep % 2)
                ok = kw == {} and torch.equal(kv, torch.cat([rows * (rep + 1), tail]))
                out.append((n, sh.pad, rep, ok))
            xch.join()
        results[rank] = out
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_collective_exchange_keys_are_token_rows_then_tail(world):
    """The gathered key rows equal cat(all token rows, tail rows) bit for bit, for pad 0 and pad > 0, over repeated exchanges."""
    with tempfile.TemporaryDirectory() as d:
        results = mp.get_context("spawn").Manager().dict()
        mp.spawn(_exchange_worker, args=(world, os.path.join(d, "init"), results), nprocs=world, join=True)
        for r in range(world):
            got = results[r]
            assert {p for _, p, _, _ in got} == {0, 1, world - 1} and all(ok for *_, ok in got), got


def test_pad_zero_collective_layout_is_unchanged():
    """Without a pad the tail rows are written straight into the gathered buffer behind the token rows, as before the pad rule."""
    from magcache_b200.shard import CollectiveExchange, TokenShard
    xch = CollectiveExchange(TokenShard(1, 2, 12), 16, (1,), "cpu", extra_rows=5)
    tail = xch.tail_rows(0)
    assert xch._tail is None and tail.data_ptr() == xch.kv_all[12:].data_ptr() and tail.shape == (5, 16)
    xch = CollectiveExchange(TokenShard(1, 2, 11), 16, (1,), "cpu", extra_rows=5)
    assert xch.tail_rows(0).data_ptr() != xch.kv_all.data_ptr() and xch.kv_all.shape == (12 + 5, 16)


# ------------------------------------------------------------------------------------------- refusal
@pytest.mark.parametrize("family", ["flux", "hunyuan"])
def test_rank_without_rows_is_refused_on_every_rank(family, monkeypatch):
    """9 image tokens over 4 ranks (3 + 3 + 3 + 0): the first forward raises ValueError on every rank, before any exchange."""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import emu_ops

    import magcache_b200 as mc
    from magcache_b200 import mmdit
    from magcache_b200 import patch as patch_mod
    from oracle import flux_ref as fr
    from oracle import hunyuan_ref as hr
    monkeypatch.setattr(mmdit, "ops", emu_ops)
    monkeypatch.setattr(patch_mod, "ops", emu_ops)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    for rank in (0, 3):
        if family == "flux":
            m = copy.deepcopy(_flux_model(fr))
            m.__class__ = type(f"R{rank}", (m.__class__,), {})
            mc.init_magcache_flux(m, 6)
            mc.enable_token_shard(m, rank, 4)
            hs, enc, pooled, img_ids, txt_ids = _flux_inputs(fr, (3, 3))
            with torch.no_grad(), pytest.raises(ValueError, match="without tokens"):
                m(hs, enc, pooled, torch.tensor([1.0]), img_ids, txt_ids, torch.tensor([3.5]), return_dict=False)
        else:
            m = copy.deepcopy(_hunyuan_model(hr))
            m.__class__ = type(f"R{rank}", (m.__class__,), {})
            mc.init_magcache_hunyuan(m, 6, mag_ratios=[1.0] * 6)
            mc.enable_token_shard(m, rank, 4)
            x, txt, mask, pooled, cos, sin = _hunyuan_inputs(hr, (1, 3, 3))
            with torch.no_grad(), pytest.raises(ValueError, match="without tokens"):
                m(x, torch.tensor([900.0]), txt, mask, pooled, cos, sin, torch.tensor([6000.0]), return_dict=False)
