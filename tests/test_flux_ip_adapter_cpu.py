"""FLUX / Kontext with IP-Adapter image prompts on the MMDiT engine, on CPU: `magcache_flux_forward` / `magcache_flux_calibration`
on a model with IP-Adapter processors and an image projection (tests/flux_ip_adapter_ref.py), the engine driven through the kernel
emulation against the oracle running the reference's ip-adapter statements (MagCache4FLUX/magcache_flux.py:321-324, :108-111).
The kernel itself: test_flux_ip_adapter_gpu.py."""
import copy
import os
import sys
import tempfile

import pytest
import torch
import torch.multiprocessing as mp

import magcache_b200 as mc
from magcache_b200 import mmdit as flux_mod
from magcache_b200 import patch as patch_mod
from oracle import flux_ref as fr

import flux_controlnet_ref as cref
import flux_ip_adapter_ref as ipr
import flux_lora_ref as lref

T0, GD = torch.tensor([0.25]), torch.tensor([1.0])


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(flux_mod, "ops", ipr.emu)
    monkeypatch.setattr(patch_mod, "ops", ipr.emu)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def _model(num_layers=2, num_single_layers=3, seed=0):
    return fr.FluxTransformer2DModel(in_channels=64, num_layers=num_layers, num_single_layers=num_single_layers, num_attention_heads=2,
                                     joint_attention_dim=96, pooled_projection_dim=48).init_synthetic(seed)


def _ip_model(n_adapters=1, T=16, seed=0, **kw):
    return ipr.load_ip_adapter(_model(seed=seed), n_adapters, T, seed=seed + 3, **kw)


def _inputs(seed=0, hw=(8, 6), n_txt=19, kontext=False):
    g = torch.Generator().manual_seed(seed)
    img_ids, txt_ids = fr.make_ids(hw[0], hw[1], n_txt)
    if kontext:  # the reference image's tokens behind the latent's, first id coordinate 1
        ref_ids, _ = fr.make_ids(4, hw[1], 0)
        ref_ids[:, 0] = 1
        img_ids = torch.cat([img_ids, ref_ids])
    hs = torch.randn(1, img_ids.shape[0], 64, generator=g).bfloat16()
    enc = torch.randn(1, n_txt, 96, generator=g).bfloat16()
    pooled = torch.randn(1, 48, generator=g).bfloat16()
    return hs, enc, pooled, img_ids, txt_ids


def _as(cls_name, model):
    m = copy.deepcopy(model)
    m.__class__ = type(cls_name, (m.__class__,), {})
    return m


def _ref(model, name, calibration=False, steps=28, **kw):
    m = _as(name, model)
    if calibration:
        type(m).forward = ipr.reference_ip(lref.reference_lora(fr.magcache_calibration))
        type(m).cnt, type(m).num_steps = 0, steps
        type(m).norm_ratio, type(m).norm_std, type(m).cos_dis, type(m).previous_residual = [], [], [], None
    else:
        fr.install_magcache(type(m), mc.tables()[kw.pop("table", "flux_dev")], steps, **kw)
        type(m).forward = ipr.reference_ip(lref.reference_lora(fr.magcache_forward))
    return m


def _ours(model, name, steps=28, **kw):
    m = _as(name, model)
    mc.init_magcache_flux(m, steps, **kw)
    return m


def _run(m, inp, t=T0, **kw):
    hs, enc, pooled, img_ids, txt_ids = inp
    with torch.no_grad():
        return m(hs, enc, pooled, t, img_ids, txt_ids, GD, return_dict=False, **kw)[0]


def _exact(model, inp, **kw):
    m64 = _ref(copy.deepcopy(model).double(), "Ref64")
    hs, enc, pooled, img_ids, txt_ids = inp
    with torch.no_grad(), fr.exact():
        return m64(hs.double(), enc.double(), pooled.double(), T0.double(), img_ids, txt_ids, GD.double(), return_dict=False, **kw)[0]


def _jak(embeds, **kw):
    return dict(joint_attention_kwargs=dict(ip_adapter_image_embeds=embeds, **kw))


def _check(model, inp, embeds, tag, **kw):
    ref_m, ours = _ref(model, "RefI"), _ours(model, "OurI")
    ref, out, exact = _run(ref_m, inp, **_jak(embeds), **kw), _run(ours, inp, **_jak(embeds), **kw), _exact(model, inp, **_jak(embeds), **kw)
    e_ours, e_ref, e_vs = rel_l2(out, exact), rel_l2(ref, exact), rel_l2(out, ref)
    print(f"[flux ip-adapter {tag}] ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e} | ours vs oracle {e_vs:.3e}")
    assert e_ours <= 1.5 * e_ref + 1e-3
    assert e_vs <= 2.0 * e_ref + 1e-3
    return out, exact


@pytest.mark.parametrize("n_adapters,T,n_images,scale", [(1, 16, 1, 1.0), (1, 4, 2, -0.5), (3, 4, 1, 1.0), (3, 16, 2, 0.6), (1, 16, 1, 0.0)])
def test_forward_matches_the_oracle(emulated, n_adapters, T, n_images, scale):
    model = _ip_model(n_adapters, T)
    ipr.set_ip_adapter_scale(model, scale)
    out, exact = _check(model, _inputs(), ipr.make_embeds(n_adapters, n_images), f"A{n_adapters} T{T} n{n_images} s{scale}")
    base = _exact(_model(), _inputs())  # the same transformer without the adapter
    if scale == 0.0:
        assert torch.equal(out, _run(_ours(_model(), "OurBase0"), _inputs()))  # scale 0 adds +0: bit-equal to no adapter
    else:
        assert rel_l2(base, exact) > 0.02, "the image prompt changed the output well beyond the rounding noise"


def test_per_block_and_per_adapter_scales(emulated):
    model = _ip_model(3, [4, 16, 4], blocks=(0, 1))
    ipr.set_ip_adapter_scale(model, [[1.0, -0.5, 0.25], [0.0, 2.0, 1.0]])
    _check(model, _inputs(), ipr.make_embeds(3, 2), "per-block scales")


def test_some_blocks_only(emulated):
    _check(_ip_model(1, 16, blocks=(1,)), _inputs(), ipr.make_embeds(1, 1), "block 1 only")


def test_kontext_shaped_inputs(emulated):
    _check(_ip_model(1, 16), _inputs(kontext=True), ipr.make_embeds(1, 1), "kontext rows")


def test_with_controlnet_and_lora(emulated):
    model = _ip_model(2, [16, 4])
    lref.inject_lora(model, "all", ("a",), rank=8, seed=9)
    inp = _inputs()
    g = torch.Generator().manual_seed(5)
    samples = [(0.3 * torch.randn(1, 48, 256, generator=g)).bfloat16() for _ in range(2)]
    ctrl = dict(controlnet_block_samples=samples, controlnet_single_block_samples=samples)
    embeds = ipr.make_embeds(2, 1)
    ref_m, ours = _ref(model, "RefCLI"), _ours(model, "OurCLI")
    with cref.controlnet_blocks(ref_m, samples, samples, 19):
        ref = _run(ref_m, inp, **_jak(embeds, scale=0.7))
    out = _run(ours, inp, **_jak(embeds, scale=0.7), **ctrl)
    assert rel_l2(out, ref) <= 2e-2
    no_ip = _ours(model, "OurCL")
    ipr.set_ip_adapter_scale(no_ip, 0.0)  # adds +0: the image prompt off
    no_ip = _run(no_ip, inp, **_jak(embeds, scale=0.7), **ctrl)
    assert rel_l2(out, no_ip) > 10 * rel_l2(out, ref)
    assert lref.scaling_state(ours) == lref.scaling_state(ref_m)


@pytest.mark.parametrize("preset", ["flux_dev", "flux_kontext"])
def test_twelve_step_loops_keep_the_references_skip_mask_and_hits_ignore_the_embeds(emulated, preset):
    thresh, K, retention = (0.24, 5, 0.1) if preset == "flux_dev" else (0.05, 4, 0.2)
    model = _ip_model(1, 16, seed=1)
    hs, enc, pooled, img_ids, txt_ids = _inputs(1, kontext=preset == "flux_kontext")
    steps = 12
    kw = dict(steps=steps, thresh=thresh, K=K, retention_ratio=retention, table=preset)
    ref_m, ours, ours2 = _ref(model, "RefLoop", **kw), _ours(model, "OurLoop", **kw), _ours(model, "OurLoop2", **kw)
    embeds, other = ipr.make_embeds(1, 1), ipr.make_embeds(1, 2, seed=7)
    skips = []
    for i in range(steps):
        t = torch.tensor([1.0 - i / steps])
        inp = (hs * (1.0 - 0.03 * i), enc, pooled, img_ids, txt_ids)
        a = _run(ref_m, inp, t=t, **_jak(embeds))
        skips.append(bool(ref_m.last_skip))
        b = _run(ours, inp, t=t, **_jak(embeds))
        c = _run(ours2, inp, t=t, **_jak(other if skips[-1] else embeds))  # other embeds on the hit steps only
        assert rel_l2(b, a) <= 0.15, (i, rel_l2(b, a))
        assert torch.equal(b, c), i
        for attr in ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"):
            assert float(getattr(ours, attr)) == float(getattr(ref_m, attr)), (i, attr)
    assert 0 < sum(skips) < steps, skips


def test_calibration_twin(emulated, capsys):
    model = _ip_model(2, 4, seed=2)
    hs, enc, pooled, img_ids, txt_ids = _inputs(2)
    steps = 4
    ref_m = _ref(model, "RefCal", calibration=True, steps=steps)
    ours = _as("OurCal", model)
    mc.init_magcache_flux_calibration(ours, steps)
    embeds = ipr.make_embeds(2, 1)
    for i in range(steps):
        t = torch.tensor([1.0 - i / steps])
        x = (hs * (1.0 - 0.1 * i), enc, pooled, img_ids, txt_ids)
        a = _run(ref_m, x, t=t, **_jak(embeds))
        if i < steps - 1:
            stats_ref = [list(ref_m.norm_ratio), list(ref_m.norm_std), list(ref_m.cos_dis)]
        b = _run(ours, x, t=t, **_jak(embeds))
        if i < steps - 1:
            stats_ours = [list(ours.norm_ratio), list(ours.norm_std), list(ours.cos_dis)]
        assert rel_l2(b, a) <= 0.15
    assert all(len(v) == steps - 2 for v in stats_ref + stats_ours)
    for r, o in zip(stats_ref, stats_ours):
        for x, y in zip(o, r):
            assert abs(x - y) <= 2e-2 * abs(y) + 2e-3, (stats_ours, stats_ref)
    assert ours.cnt == 0 and "norm ratio" in capsys.readouterr().out


def test_scale_change_and_unload_take_effect_on_the_next_call_bit_equal_to_a_fresh_engine(emulated):
    """Processors, scales and weights are read at every call: after `set_ip_adapter_scale`, a new adapter, or `unload_ip_adapter`,
    the next forward equals the same forward on a model whose engine is built only then."""
    model, inp = _ip_model(1, 16), _inputs()
    embeds = ipr.make_embeds(1, 1)
    ours = _ours(model, "OurS", thresh=-1.0)  # every call a miss
    first = _run(ours, inp, **_jak(embeds))

    def fresh(m, **kw):  # a copy of the module as it is now, without the engine and controllers cached on it
        saved = {k: m.__dict__.pop(k) for k in ("_mc_flux_engine", "_mc_ctrls") if k in m.__dict__}
        try:
            twin = _ours(m, "OurFresh", thresh=-1.0)
        finally:
            m.__dict__.update(saved)
        return _run(twin, inp, **kw)

    ipr.set_ip_adapter_scale(ours, 0.3)
    got = _run(ours, inp, **_jak(embeds))
    assert torch.equal(got, fresh(ours, **_jak(embeds))) and not torch.equal(got, first)
    ipr.unload_ip_adapter(ours)
    got = _run(ours, inp)
    assert torch.equal(got, fresh(ours)) and torch.equal(got, _run(_ours(_model(), "OurPlain", thresh=-1.0), inp))
    ipr.load_ip_adapter(ours, 3, 4, seed=11)
    embeds3 = ipr.make_embeds(3, 2)
    got = _run(ours, inp, **_jak(embeds3))
    assert torch.equal(got, fresh(ours, **_jak(embeds3)))


def _bad_case(bad):
    model, embeds, kw = _ip_model(2, 4), ipr.make_embeds(2, 1), {}
    if bad == "single_block_processor":
        model.single_transformer_blocks[1].attn.processor = ipr.FluxIPAdapterAttnProcessor(256, 64, [4, 4])
    elif bad == "unknown_processor":
        model.transformer_blocks[0].attn._modules.pop("processor")
        model.transformer_blocks[0].attn.processor = type("AttnProcessor2_0", (), {})()
    elif bad == "lora_to_k_ip":
        lref.inject_lora(model, "attn", ("a",), names=["transformer_blocks.1.attn.processor.to_k_ip.1"])
    elif bad == "lora_to_v_ip":
        lref.inject_lora(model, "attn", ("a",), names=["transformer_blocks.0.attn.processor.to_v_ip.0"])
    elif bad == "lora_encoder_hid_proj":
        lref.inject_lora(model, "attn", ("a",), names=["encoder_hid_proj.image_projection_layers.0.image_embeds"])
    elif bad == "count":
        embeds = embeds[:1]
    elif bad == "not_a_list":
        embeds = embeds[0]
    elif bad == "shape":
        embeds[1] = embeds[1][:, :, :16]
    elif bad == "batch":
        embeds[0] = torch.cat([embeds[0], embeds[0]])
    elif bad == "dtype":
        embeds[0] = embeds[0].float()
    elif bad == "device":
        embeds[0] = embeds[0].to("meta")
    elif bad == "no_embeds":
        embeds = None
    elif bad == "too_many_keys":
        model, embeds = _ip_model(1, 16), ipr.make_embeds(1, 25)  # 400 image-prompt tokens
    elif bad == "other_key":
        kw = {"ip_adapter_masks": [None]}
    return model, None if embeds is None else dict(ip_adapter_image_embeds=embeds, **kw)


@pytest.mark.parametrize("bad", ["single_block_processor", "unknown_processor", "lora_to_k_ip", "lora_to_v_ip", "lora_encoder_hid_proj",
                                 "count", "not_a_list", "shape", "batch", "dtype", "device", "no_embeds", "too_many_keys", "other_key"])
def test_refusals(emulated, bad):
    model, jak = _bad_case(bad)
    ours = _ours(model, "OurBad")
    with pytest.raises(NotImplementedError) as e:
        _run(ours, _inputs(), joint_attention_kwargs=jak)
    want = {"single_block_processor": "single_transformer_blocks.1.attn", "unknown_processor": "AttnProcessor2_0",
            "lora_to_k_ip": "to_k_ip.1", "lora_to_v_ip": "to_v_ip.0", "lora_encoder_hid_proj": "encoder_hid_proj",
            "count": "list of 2", "not_a_list": "list of 2", "shape": "[1]", "batch": "[0]", "dtype": "[0]", "device": "[0]",
            "no_embeds": "no ip_adapter_image_embeds", "too_many_keys": "400", "other_key": "ip_adapter_masks"}[bad]
    assert want in str(e.value), str(e.value)


def test_embeds_on_a_model_without_ip_adapter_raise(emulated):
    with pytest.raises(NotImplementedError, match="ip_adapter_image_embeds"):
        _run(_ours(_model(), "OurNoIP"), _inputs(), **_jak(ipr.make_embeds(1, 1)))


def _shard_worker(rank, world, initfile, results):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch.distributed as dist
    import flux_ip_adapter_ref as ip_ref
    dist.init_process_group("gloo", init_method=f"file://{initfile}", rank=rank, world_size=world)
    try:
        flux_mod.ops = ip_ref.emu
        patch_mod.ops = ip_ref.emu
        torch.Tensor.is_cuda = property(lambda self: True)
        model = ip_ref.load_ip_adapter(_model(2, 2), 2, [16, 4], seed=5)
        embeds = ip_ref.make_embeds(2, 2)
        hs, enc, pooled, img_ids, txt_ids = _inputs(3)
        outs, first_ip = {}, {}
        attend = ip_ref.emu.ip_attention

        def recording(*a, **kw):
            out = attend(*a, **kw)
            first_ip.setdefault(name, out.clone())
            return out

        ip_ref.emu.ip_attention = recording
        for name in ("single", "sharded"):
            m = _as("S_" + name, model)
            mc.init_magcache_flux(m, 6, thresh=10.0, K=2, retention_ratio=0.34)  # miss miss hit hit miss miss
            if name == "sharded":
                mc.enable_token_shard(m, rank, world)
            got = []
            with torch.no_grad():
                for i in range(6):
                    got.append(m(hs * (1 - 0.05 * i), enc, pooled, torch.tensor([1.0 - i / 6]), img_ids, txt_ids, torch.tensor([3.5]),
                                 return_dict=False, joint_attention_kwargs={"ip_adapter_image_embeds": embeds})[0].clone())
            outs[name] = got
        eng = m._mc_flux_engine
        errs = [float((a.float() - b.float()).abs().max() / b.float().abs().max()) for a, b in zip(outs["sharded"], outs["single"])]
        ip_equal = torch.equal(first_ip["sharded"], first_ip["single"][eng.shard.start:eng.shard.stop])
        results[rank] = (errs, ip_equal, eng.n_img, eng.n_img_total)
    finally:
        dist.destroy_process_group()


def test_ip_adapter_sharded_equals_single_world2():
    """Token-sharded (image rows split over 2 gloo ranks): every rank projects the replicated embeds and attends its own image rows.
    The first block's image-prompt attention (whose inputs are row-local) is bit-equal to one rank's rows of it; the outputs
    match one rank's within the sharded engine's tolerance (its joint attention orders the keys differently)."""
    with tempfile.TemporaryDirectory() as d:
        results = mp.get_context("spawn").Manager().dict()
        mp.spawn(_shard_worker, args=(2, os.path.join(d, "init"), results), nprocs=2, join=True)
        assert set(results.keys()) == {0, 1}
        for r in (0, 1):
            errs, ip_equal, n_loc, n_tot = results[r]
            assert n_loc * 2 == n_tot == 48
            assert ip_equal
            assert len(errs) == 6 and max(errs) < 1.2e-2, errs
