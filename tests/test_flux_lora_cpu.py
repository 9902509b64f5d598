"""FLUX / Kontext with unmerged LoRA adapters on the MMDiT engine, on CPU: `magcache_flux_forward` / `magcache_flux_calibration` on a
model whose Linears carry PEFT-layout LoRA layers, the engine driven through the kernel emulation with the tailed GEMM
(tests/flux_lora_ref.py) against the oracle running the reference's scale / unscale statements (MagCache4FLUX/magcache_flux.py:274-287,
:437-439). The tailed GEMM itself: test_flux_lora_gpu.py."""
import copy
import os
import sys
import tempfile

import pytest
import torch
import torch.multiprocessing as mp
from torch import nn

import magcache_b200 as mc
from magcache_b200 import lora as lora_mod
from magcache_b200 import mmdit as flux_mod
from magcache_b200 import patch as patch_mod
from oracle import flux_ref as fr

import flux_controlnet_ref as cref
import flux_lora_ref as lref

T0, GD = torch.tensor([0.25]), torch.tensor([1.0])  # t * 1000 and g * 1000 are exact in bf16: the fp64 run sees the same inputs


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(flux_mod, "ops", lref.emu)
    monkeypatch.setattr(patch_mod, "ops", lref.emu)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def _model(num_layers=2, num_single_layers=3, seed=0):
    return fr.FluxTransformer2DModel(in_channels=64, num_layers=num_layers, num_single_layers=num_single_layers, num_attention_heads=2,
                                     joint_attention_dim=96, pooled_projection_dim=48).init_synthetic(seed)


def _inputs(seed=0, hw=(8, 6), n_txt=19):
    g = torch.Generator().manual_seed(seed)
    n_img = hw[0] * hw[1]
    hs = torch.randn(1, n_img, 64, generator=g).bfloat16()
    enc = torch.randn(1, n_txt, 96, generator=g).bfloat16()
    pooled = torch.randn(1, 48, generator=g).bfloat16()
    img_ids, txt_ids = fr.make_ids(hw[0], hw[1], n_txt)
    return hs, enc, pooled, img_ids, txt_ids


def _as(cls_name, model):
    m = copy.deepcopy(model)
    m.__class__ = type(cls_name, (m.__class__,), {})
    return m


def _ref(model, name, calibration=False, steps=28, **kw):
    """A copy of `model` running the oracle's forward (or calibration twin) inside the reference's LoRA statements."""
    m = _as(name, model)
    if calibration:
        type(m).forward = lref.reference_lora(fr.magcache_calibration)
        type(m).cnt, type(m).num_steps = 0, steps
        type(m).norm_ratio, type(m).norm_std, type(m).cos_dis, type(m).previous_residual = [], [], [], None
    else:
        fr.install_magcache(type(m), mc.tables()[kw.pop("table", "flux_dev")], steps, **kw)
        type(m).forward = lref.reference_lora(fr.magcache_forward)
    return m


def _ours(model, name, steps=28, **kw):
    m = _as(name, model)
    mc.init_magcache_flux(m, steps, **kw)
    return m


def _lora_model(targets="all", rank=8, adapters=("a",), seed=0, blocks=None, **kw):
    model = _model()
    lref.inject_lora(model, targets, adapters, rank=rank, seed=seed + 7, names=lref.target_names(model, targets, blocks), **kw)
    return model


def _run(m, inp, t=T0, **kw):
    hs, enc, pooled, img_ids, txt_ids = inp
    with torch.no_grad():
        return m(hs, enc, pooled, t, img_ids, txt_ids, GD, return_dict=False, **kw)[0]


def _exact(model, inp, **kw):
    m64 = _ref(copy.deepcopy(model).double(), "Ref64")
    hs, enc, pooled, img_ids, txt_ids = inp
    with torch.no_grad(), fr.exact():
        return m64(hs.double(), enc.double(), pooled.double(), T0.double(), img_ids, txt_ids, GD.double(), return_dict=False, **kw)[0]


def _check(model, inp, tag, base=None, **kw):
    ref_m, ours = _ref(model, "RefL"), _ours(model, "OurL")
    ref, out, exact = _run(ref_m, inp, **kw), _run(ours, inp, **kw), _exact(model, inp, **kw)
    e_ours, e_ref, e_vs = rel_l2(out, exact), rel_l2(ref, exact), rel_l2(out, ref)
    print(f"[flux lora {tag}] ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e} | ours vs oracle {e_vs:.3e}")
    assert e_ours <= 1.5 * e_ref + 1e-3
    assert e_vs <= 2.0 * e_ref + 1e-3
    assert lref.scaling_state(ours) == lref.scaling_state(ref_m)
    if base is not None:
        assert rel_l2(base, exact) > 3 * e_ours, "the adapters changed the output well beyond the rounding noise"
    return out


def test_adapters_without_kwargs_run_and_match_the_oracle(emulated):
    """`joint_attention_kwargs=None`, as diffusers' pipelines pass it: the adapters are applied, not the base model alone."""
    model, inp = _lora_model(), _inputs()
    base = _run(_ours(_model(), "OurBase"), inp)
    _check(model, inp, "kwargs None", base=base)


@pytest.mark.parametrize("targets,rank", [(t, 12) for t in ("attn", "blocks", "ada", "all")] + [("all", r) for r in (4, 16, 72)])
def test_targets_and_ranks(emulated, targets, rank):
    _check(_lora_model(targets, rank), _inputs(), f"{targets} r{rank}", base=_run(_ours(_model(), "OurBase"), _inputs()))


@pytest.mark.parametrize("scale", [1.0, 0.6, 0.0, -1.0])
def test_two_adapters_weights_and_scales(emulated, scale):
    model = _lora_model("all", 8, adapters=("a", "b"))
    lref.set_adapters(model, ["a", "b"], [0.7, -0.4])
    _check(model, _inputs(), f"two adapters scale {scale}", joint_attention_kwargs={"scale": scale})


def test_some_blocks_only_with_controlnet(emulated):
    model = _lora_model("ada", 16, blocks=lambda n: n.startswith(("transformer_blocks.1.", "single_transformer_blocks.0.")))
    samples = [(0.3 * torch.randn(1, 48, 256, generator=torch.Generator().manual_seed(5))).bfloat16()]
    ours_kw = dict(controlnet_block_samples=samples, controlnet_single_block_samples=samples * 2)
    ref_m, ours = _ref(model, "RefCL"), _ours(model, "OurCL")
    inp = _inputs()
    with cref.controlnet_blocks(ref_m, samples, samples * 2, 19):
        ref = _run(ref_m, inp)
    out = _run(ours, inp, **ours_kw)
    assert rel_l2(out, ref) <= 2e-2
    plain = _run(_ours(model, "OurCL2"), inp)  # same adapters, no samples
    assert rel_l2(out, plain) > 10 * rel_l2(out, ref)


def test_scaling_state_follows_the_reference_call_for_call(emulated):
    """scale_lora_layers / unscale_lora_layers on every call: repeated non-unit scales (ulp drift included) and scale 0's reset of
    `set_adapters` weights leave every layer's `scaling` where the reference leaves it."""
    model = _lora_model("blocks", 8, adapters=("a", "b"))
    lref.set_adapters(model, ["a", "b"], [0.3, 1.7])
    ref_m, ours = _ref(model, "RefS", thresh=10.0, K=2, retention_ratio=0.2), _ours(model, "OurS", thresh=10.0, K=2, retention_ratio=0.2)
    inp = _inputs()
    for i, scale in enumerate([0.7, 0.7, 1.0 / 3, 1.0 / 3, 1.0 / 3, 1.0, 0.0, 0.9, 0.0]):
        jak = {"scale": scale}
        a, b = _run(ref_m, inp, t=torch.tensor([1 - i / 10]), joint_attention_kwargs=jak), _run(ours, inp, t=torch.tensor([1 - i / 10]), joint_attention_kwargs=jak)
        assert lref.scaling_state(ours) == lref.scaling_state(ref_m), (i, scale)
        assert rel_l2(b, a) <= 0.05, (i, scale)
        assert jak == {"scale": scale}  # the caller's dict is not consumed
    assert lref.scaling_state(ours)[0]["a"] == 1.0  # the reset at scale 0 dropped the set_adapters weight


def test_adapter_changes_take_effect_on_the_next_call(emulated):
    model, inp = _model(), _inputs()
    ours, ref_m = _ours(model, "OurD", thresh=-1.0), _ref(model, "RefD", thresh=-1.0)  # every call a miss
    both = (ours, ref_m)

    def step(tag):
        a, b = _run(ref_m, inp), _run(ours, inp)
        assert rel_l2(b, a) <= 2e-2, tag
        return b

    base = step("none")
    for m in both:  # load
        lref.inject_lora(m, "all", ("a",), rank=8, seed=3)
    loaded = step("loaded")
    assert rel_l2(loaded, base) > 0.05
    for m in both:  # a second adapter, then re-weighted
        lref.inject_lora(m, "attn", ("b",), rank=16, seed=4)
    two = step("two")
    for m in both:
        lref.set_adapters(m, ["a", "b"], [0.5, 2.0])
    rew = step("reweighted")
    assert rel_l2(rew, two) > 1e-2
    for m in both:  # disabled
        for lay in lref.lora_layers(m):
            lay.disable_adapters = True
    assert torch.equal(step("disabled"), base)
    for m in both:  # enabled, then b deleted
        for lay in lref.lora_layers(m):
            lay.disable_adapters = False
            if "b" in lay.lora_A:
                del lay.lora_A["b"], lay.lora_B["b"]
                lay._active = [x for x in lay._active if x != "b"]
    step("deleted")
    for m in both:  # merged: the update is in the base weights now and must not be added a second time
        for lay in lref.lora_layers(m):
            lay.merge()
    merged = step("merged")
    assert rel_l2(merged, base) > 0.05
    for m in both:
        for lay in lref.lora_layers(m):
            lay.unmerge()
    step("unmerged")


def test_fused_then_unloaded_adapters_repack_the_base_weights(emulated):
    """`fuse_lora()` then `unload_lora_weights()` after the engine has run the adapters: the merge wrote into base weights the
    engine partly aliases and partly copied (q|k, the AdaLayerNorm table), and the LoRA layers are gone; the next forward must
    repack and equal an engine built fresh from the fused module."""
    model, inp = _lora_model("all", 16), _inputs()
    ours, twin = _ours(model, "OurF", thresh=-1.0), _ours(model, "OurF2", thresh=-1.0)
    before = _run(ours, inp)
    for m in (ours, twin):  # the same fuse and unload on both; `twin` builds its engine only afterwards
        for lay in lref.lora_layers(m):
            lay.merge()
        lref.unload_lora(m)
    got = _run(ours, inp)
    assert torch.equal(got, _run(twin, inp))
    assert ours._mc_flux_engine.lora is None
    assert rel_l2(got, before) <= 2e-2  # the fused model computes what the adapters did


def test_fuse_and_unload_between_forwards_with_invalidate_engine(emulated):
    """Adapters loaded, fused and unloaded between two forwards leave nothing on the module that tells a merge happened; the
    documented `invalidate_engine` makes the next forward equal a fresh engine's."""
    model, inp = _model(), _inputs()
    ours, twin = _ours(model, "OurFI", thresh=-1.0), _ours(model, "OurFI2", thresh=-1.0)
    base = _run(ours, inp)
    for m in (ours, twin):
        for lay in lref.inject_lora(m, "all", ("a",), rank=16, seed=3):
            lay.merge()
        lref.unload_lora(m)
    mc.invalidate_engine(ours)
    got = _run(ours, inp)
    assert torch.equal(got, _run(twin, inp))
    assert rel_l2(got, base) > 0.05


@pytest.mark.parametrize("bad", ["dora", "controlnet_sample"])
def test_a_refused_call_leaves_scaling_unscaled(emulated, bad):
    """The engine refuses an input after `scale_lora_layers` ran: `unscale_lora_layers` still runs, so each layer's `scaling`
    ends where a completed call leaves it, not multiplied by the scale."""
    model = _lora_model("attn", 8, adapters=("a", "b"))
    lref.set_adapters(model, ["a", "b"], [0.3, 1.7])
    ours = _ours(model, "OurRef")
    kw = dict(joint_attention_kwargs={"scale": 0.6})
    if bad == "dora":
        lref.lora_layers(ours)[-1].use_dora["b"] = True
    else:
        kw["controlnet_block_samples"] = [torch.zeros(1, 47, 256, dtype=torch.bfloat16)]
    want = copy.deepcopy(model)  # where the reference's scale then unscale leaves `scaling` (a multiply and a divide: ulp drift)
    lref.scale_lora_layers(want, 0.6)
    lref.unscale_lora_layers(want, 0.6)
    with pytest.raises(NotImplementedError):
        _run(ours, _inputs(), **kw)
    assert lref.scaling_state(ours) == lref.scaling_state(want)


@pytest.mark.parametrize("bad", ["dora", "lora_bias", "dropout", "time_text_embed", "ip_adapter", "scale_without_adapters"])
def test_unsupported_adapters_raise(emulated, bad):
    model = _lora_model("attn", 8, dropout=0.1 if bad == "dropout" else 0.0)
    lay = lref.lora_layers(model)[0]
    kw = {}
    if bad == "dora":
        lay.use_dora["a"] = True
    elif bad == "lora_bias":
        lay.lora_B["a"] = nn.Linear(8, lay.base_layer.out_features, bias=True).bfloat16()
    elif bad == "dropout":
        model.train()
    elif bad == "time_text_embed":
        lref.inject_lora(model, "attn", ("a",), names=["time_text_embed.timestep_embedder.linear_1"])
    elif bad == "ip_adapter":
        kw = dict(joint_attention_kwargs={"scale": 1.0, "ip_adapter_image_embeds": [torch.zeros(1)]})
    elif bad == "scale_without_adapters":
        model, kw = _model(), dict(joint_attention_kwargs={"scale": 0.5})
    ours = _ours(model, "OurBad")
    with pytest.raises(NotImplementedError) as e:
        _run(ours, _inputs(), **kw)
    want = {"dora": "DoRA", "lora_bias": "lora_bias", "dropout": "dropout", "time_text_embed": "time_text_embed.timestep_embedder.linear_1",
            "ip_adapter": "ip_adapter_image_embeds", "scale_without_adapters": "no LoRA layer"}[bad]
    assert want in str(e.value)


def test_hunyuan_with_a_lora_layer_raises():
    from oracle import hunyuan_ref as hr
    model = hr.HYVideoDiffusionTransformer(hidden_size=256, heads_num=2, mm_double_blocks_depth=1, mm_single_blocks_depth=1,
                                           text_states_dim=64, text_states_dim_2=32)
    blk = model.double_blocks[0]
    blk.img_attn_proj = lref.LoraLinear(blk.img_attn_proj)
    with pytest.raises(NotImplementedError, match="double_blocks.0.img_attn_proj"):
        flux_mod.HunyuanWeights.from_module(model, torch.device("cpu"))


@pytest.mark.parametrize("preset", ["flux_dev", "flux_kontext"])
def test_twelve_step_loops_keep_the_references_skip_mask(emulated, preset):
    thresh, K, retention = (0.24, 5, 0.1) if preset == "flux_dev" else (0.05, 4, 0.2)
    model = _lora_model("all", 16, adapters=("a", "b"), seed=1)
    hs, enc, pooled, img_ids, txt_ids = _inputs(1)
    steps = 12
    ref_m = _ref(model, "RefLoop", steps=steps, thresh=thresh, K=K, retention_ratio=retention, table=preset)
    ours = _ours(model, "OurLoop", steps=steps, thresh=thresh, K=K, retention_ratio=retention, table=preset)
    skips, ours_skips = [], []
    for i in range(steps):
        t = torch.tensor([1.0 - i / steps])
        x = hs * (1.0 - 0.03 * i)
        jak = {"scale": 0.8}
        a = _run(ref_m, (x, enc, pooled, img_ids, txt_ids), t=t, joint_attention_kwargs=jak)
        skips.append(bool(ref_m.last_skip))
        b = _run(ours, (x, enc, pooled, img_ids, txt_ids), t=t, joint_attention_kwargs=jak)
        assert rel_l2(b, a) <= 0.15, (i, rel_l2(b, a))
        for attr in ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"):
            assert float(getattr(ours, attr)) == float(getattr(ref_m, attr)), (i, attr)
        assert lref.scaling_state(ours) == lref.scaling_state(ref_m)
    assert 0 < sum(skips) < steps, skips


def test_calibration_twin(emulated, capsys):
    model = _lora_model("all", 8, seed=2)
    hs, enc, pooled, img_ids, txt_ids = _inputs(2)
    steps = 4
    ref_m = _ref(model, "RefCal", calibration=True, steps=steps)
    ours = _as("OurCal", model)
    mc.init_magcache_flux_calibration(ours, steps)
    for i in range(steps):
        t = torch.tensor([1.0 - i / steps])
        x = hs * (1.0 - 0.1 * i)
        a = _run(ref_m, (x, enc, pooled, img_ids, txt_ids), t=t, joint_attention_kwargs={"scale": 0.5})
        if i < steps - 1:
            stats_ref = [list(ref_m.norm_ratio), list(ref_m.norm_std), list(ref_m.cos_dis)]
        b = _run(ours, (x, enc, pooled, img_ids, txt_ids), t=t, joint_attention_kwargs={"scale": 0.5})
        if i < steps - 1:
            stats_ours = [list(ours.norm_ratio), list(ours.norm_std), list(ours.cos_dis)]
        assert rel_l2(b, a) <= 0.15
        assert lref.scaling_state(ours) == lref.scaling_state(ref_m)
    assert all(len(v) == steps - 2 for v in stats_ref + stats_ours)
    for r, o in zip(stats_ref, stats_ours):
        for a, b in zip(o, r):
            assert abs(a - b) <= 2e-2 * abs(b) + 2e-3, (stats_ours, stats_ref)
    assert ours.cnt == 0 and "norm ratio" in capsys.readouterr().out


def test_per_call_check_cost_at_flux_dev_module_count():
    """Host cost of `FluxLoraScan.scan` on an unchanged module with FLUX.1-dev's 19 + 38 blocks: printed, and bounded loosely."""
    import time
    model = fr.FluxTransformer2DModel(in_channels=64, num_layers=19, num_single_layers=38, num_attention_heads=1, joint_attention_dim=32,
                                      pooled_projection_dim=16)
    for tag in ("no adapters", "rank-16 adapters on every covered target"):
        if tag != "no adapters":
            lref.inject_lora(model, "all", ("a",), rank=16)
        scan = lora_mod.FluxLoraScan(model)
        scan.scan()
        n = 50
        t0 = time.perf_counter()
        for _ in range(n):
            *_, changed = scan.scan()
        us = (time.perf_counter() - t0) / n * 1e6
        assert not changed
        print(f"[flux lora per-call check] {tag}: {us:.0f} us per call ({len(scan.positions)} positions)")
        assert us < 50000


def _shard_worker(rank, world, initfile, results):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch.distributed as dist
    import flux_lora_ref as lr
    dist.init_process_group("gloo", init_method=f"file://{initfile}", rank=rank, world_size=world)
    try:
        flux_mod.ops = lr.emu
        patch_mod.ops = lr.emu
        torch.Tensor.is_cuda = property(lambda self: True)
        model = _model(2, 2)
        lr.inject_lora(model, "all", ("a", "b"), rank=12, seed=5)
        hs, enc, pooled, img_ids, txt_ids = _inputs(3)
        outs = {}
        for name in ("single", "sharded"):
            m = _as("S_" + name, model)
            mc.init_magcache_flux(m, 6, thresh=10.0, K=2, retention_ratio=0.34)  # miss miss hit hit miss miss
            if name == "sharded":
                mc.enable_token_shard(m, rank, world)
            got = []
            with torch.no_grad():
                for i in range(6):
                    got.append(m(hs * (1 - 0.05 * i), enc, pooled, torch.tensor([1.0 - i / 6]), img_ids, txt_ids, torch.tensor([3.5]),
                                 return_dict=False, joint_attention_kwargs={"scale": 0.7})[0].clone())
            outs[name] = got
        eng = m._mc_flux_engine
        errs = [float((a.float() - b.float()).abs().max() / b.float().abs().max()) for a, b in zip(outs["sharded"], outs["single"])]
        results[rank] = (errs, eng.n_img, eng.n_img_total)
    finally:
        dist.destroy_process_group()


def test_lora_sharded_equals_single_world2():
    """Token-sharded (image rows split over 2 ranks, gloo): q and k launch separately on row blocks of the packed weights and
    their tails, and the single block's K|V GEMMs read row blocks of the down-projected input."""
    with tempfile.TemporaryDirectory() as d:
        results = mp.get_context("spawn").Manager().dict()
        mp.spawn(_shard_worker, args=(2, os.path.join(d, "init"), results), nprocs=2, join=True)
        assert set(results.keys()) == {0, 1}
        for r in (0, 1):
            errs, n_loc, n_tot = results[r]
            assert n_loc * 2 == n_tot == 48
            assert len(errs) == 6 and max(errs) < 1.2e-2, errs
