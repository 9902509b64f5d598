"""Qwen-Image / Qwen-Image-Edit with unmerged LoRA adapters on the H100 kernels: the patched forward and its calibration twin
against tests/qwen_image_ref.py's model running the reference's LoRA statements (tests/test_qwen_image_lora_cpu.py's oracle) in
bf16 and fp64 — reduced size on CPU oracles, one block at full width with rank-64 adapters on every covered target on GPU
oracles — zero updates bit-equal to no adapters, and the full 60-block model's memory with rank-64 adapters everywhere."""
import contextlib
import copy
import gc
import io

import pytest
import torch

import magcache_b200 as mc
import qwen_image_ref as qr
import flux_lora_ref as lref
from test_qwen_image_lora_cpu import reference_lora, target_names

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def rel_l2(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30))


def _own_class(m, name):
    m.__class__ = type(name, (m.__class__,), {})
    return m


def _calls(shapes, steps, n_cond, n_uncond, dims, dev, seed=0):
    out = []
    for s in range(steps):
        for b, n in enumerate((n_cond, n_uncond)):
            kw = qr.call_inputs(seed + 10 * s + b, shapes, n, in_channels=dims[0], joint_dim=dims[1], t=1.0 - 0.9 * s / steps)
            out.append({k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in kw.items()})
    return out


def _run(model, calls, scale=None, f64=False):
    extra = {} if scale is None else {"attention_kwargs": {"scale": scale}}
    with torch.no_grad(), (qr.exact() if f64 else contextlib.nullcontext()):
        return [model(**{k: (v.double() if f64 and torch.is_tensor(v) and v.is_floating_point() else v) for k, v in kw.items()},
                      **extra, return_dict=False)[0] for kw in calls]


def _check(ours, ref, ref64):
    for i, (o, r, r64) in enumerate(zip(ours, ref, ref64)):
        e = rel_l2(r, r64)
        assert rel_l2(o, r) <= 2 * e + 1e-3 and rel_l2(o, r64) <= 1.5 * e + 1e-3, (i, rel_l2(o, r), rel_l2(o, r64), e)


def _install(model, name, steps, thresh, K, retention, ours, calibration=False):
    m = _own_class(model, name)
    if calibration:
        (mc.init_magcache_qwen_image_calibration if ours else qr.init_magcache_calibration)(m, steps)
    elif ours:
        mc.init_magcache_qwen_image(m, "qwen_image", steps, thresh, K, retention)
    else:
        qr.init_magcache(m, list(mc.tables()["qwen_image"][2:]), steps, thresh, K, retention)
    if not ours:
        type(m).forward = reference_lora(qr.magcache_calibration if calibration else qr.magcache_forward)
    return m


def _with_lora(model, rank, adapters=("a",), seed=7, **kw):
    lref.inject_lora(model, None, adapters, rank=rank, seed=seed, names=target_names(model, "all"), **kw)
    return model


@pytest.mark.parametrize("shapes", [[(1, 16, 12)], [(1, 12, 10), (1, 9, 14)]], ids=["t2i", "edit"])
@pytest.mark.parametrize("mode", ["forward", "calibration"])
def test_reduced_size_loop_matches_oracle(shapes, mode):
    """2 blocks, 2 heads x 128, two weighted rank-12 / rank-40 adapters on every covered target, scale 0.7, 37-token cond and
    6-token uncond text, 10 steps (hits in the forward): GPU engine against the bf16 and fp64 oracle on CPU, `scaling` equal."""
    model = qr.tiny_model(11)
    lref.inject_lora(model, None, ("a",), rank=12, seed=3, names=target_names(model, "all"))
    lref.inject_lora(model, None, ("b",), rank=40, seed=4, names=target_names(model, "all"))
    lref.set_adapters(model, ["a", "b"], [0.9, -0.6])
    steps, dims = 10, (16, 96)
    cal = mode == "calibration"
    ref = _install(copy.deepcopy(model), "RefL", steps, 0.5, 2, 0.2, False, cal)
    ref64 = _install(copy.deepcopy(model).double(), "RefL64", steps, 0.5, 2, 0.2, False, cal)
    ours = _install(copy.deepcopy(model).to(DEV), "OursL", steps, 0.5, 2, 0.2, True, cal)
    calls = _calls(shapes, steps, 37, 6, dims, "cpu")
    with contextlib.redirect_stdout(io.StringIO()):
        r, r64 = _run(ref, calls, 0.7), _run(ref64, calls, 0.7, f64=True)
        o = _run(ours, [{k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in kw.items()} for kw in calls], 0.7)
    _check(o, r, r64)
    assert lref.scaling_state(ours) == lref.scaling_state(ref)
    assert ours._mc_qwen_engine.lora is not None
    if not cal:
        assert int(ours.cnt) == int(ref.cnt) and ours.accumulated_steps == ref.accumulated_steps


def test_zero_updates_equal_no_adapters():
    """All-zero lora_B, and scale 0 on rank-16 adapters, on every covered target: the tail adds exact zeros to the fp32
    accumulator, so every output (misses and hits of both branches) is bit-equal to the model without adapters."""
    model = qr.tiny_model(13)
    calls = _calls([(1, 16, 12)], 6, 37, 6, (16, 96), DEV)
    plain = _run(_install(copy.deepcopy(model).to(DEV), "Plain", 6, 0.5, 2, 0.2, True), calls)
    zero_b = _install(_with_lora(copy.deepcopy(model), 16, zero_b=True).to(DEV), "ZeroB", 6, 0.5, 2, 0.2, True)
    scale0 = _install(_with_lora(copy.deepcopy(model), 16).to(DEV), "Scale0", 6, 0.5, 2, 0.2, True)
    for name, outs in (("zero lora_B", _run(zero_b, calls)), ("scale 0", _run(scale0, calls, 0.0))):
        assert all(torch.equal(a, b) for a, b in zip(outs, plain)), name
    assert zero_b._mc_qwen_engine.lora is not None and scale0._mc_qwen_engine.lora is not None


def _full_width_layer(seed=0):
    with torch.device("meta"):
        m = qr.QwenImageTransformer2DModel(num_layers=1).to(torch.bfloat16)
    return m.to_empty(device=DEV).init_synthetic(seed)


@pytest.mark.parametrize("shapes", [[(1, 83, 83)], [(1, 58, 104)], [(1, 64, 64), (1, 64, 64)]],
                         ids=["1328x1328", "1664x928", "edit_1024x1024"])
def test_full_width_layer_miss_miss_hit_hit(shapes):
    """One block at full width (3072 wide, 24 heads, 3584-wide text) with a rank-64 adapter on every covered target, scale 0.8:
    cond (200 text tokens) miss, uncond (6) miss, cond hit, uncond hit through the patched forward, against the oracle on the
    GPU in bf16 and fp64. The allocator reserves nothing new after the first two calls."""
    model = _with_lora(_full_width_layer(), 64).to(DEV)
    calls = _calls(shapes, 2, 200, 6, (64, 3584), DEV)
    ref = _install(copy.deepcopy(model), "RefLW", 2, 10.0, 2, 0.5, False)
    r = _run(ref, calls, 0.8)
    del ref
    ref64 = _install(copy.deepcopy(model).double(), "RefLW64", 2, 10.0, 2, 0.5, False)
    r64 = [x.cpu() for x in _run(ref64, calls, 0.8, f64=True)]
    del ref64
    torch.cuda.empty_cache()
    ours = _install(model, "OursLW", 2, 10.0, 2, 0.5, True)
    o = []
    with torch.no_grad():
        for i, kw in enumerate(calls):
            o.append(ours(**kw, attention_kwargs={"scale": 0.8}, return_dict=False)[0].cpu())
            if i == 1:
                torch.cuda.synchronize()
                segs = torch.cuda.memory_stats()["segment.all.allocated"]
    torch.cuda.synchronize()
    assert torch.cuda.memory_stats()["segment.all.allocated"] == segs
    _check(o, r, r64)
    plain = _install(copy.deepcopy(_full_width_layer()), "PlainLW", 2, 10.0, 2, 0.5, True)
    assert rel_l2(_run(plain, calls[:1])[0], o[0]) > 10 * rel_l2(o[0], r64[0]), "the adapters changed the output beyond the noise"


def test_full_depth_memory_with_rank64_adapters_everywhere(capsys):
    """The 60-block model (weights allocated in place on the device) with a rank-64 adapter on every covered target: one miss
    and one hit at 1328^2. Printed: the module's base and adapter weights, and the peak beyond them (the engine's packed A / T,
    its copies, workspaces and activations)."""
    gc.collect()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    with torch.device("meta"):
        m = qr.QwenImageTransformer2DModel().to(torch.bfloat16)
    m = m.to_empty(device=DEV).init_synthetic(0)
    params = sum(p.numel() * p.element_size() for p in m.parameters())
    m = _own_class(_with_lora(m, 64).to(DEV), "FullL")
    lora_params = sum(p.numel() * p.element_size() for p in m.parameters()) - params
    mc.init_magcache_qwen_image(m, "qwen_image", 2, 10.0, 2, 0.5)
    calls = _calls([(1, 83, 83)], 2, 200, 6, (64, 3584), DEV)[:3]  # cond miss, uncond miss, cond hit
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        outs = [m(**kw, return_dict=False)[0] for kw in calls]
    torch.cuda.synchronize()
    assert all(bool(torch.isfinite(o.float()).all()) for o in outs) and not torch.equal(outs[0], outs[2])
    eng = m._mc_qwen_engine
    packed = sum(v[1].numel() * v[1].element_size() for v in eng.lora._cache.values())
    extra = torch.cuda.max_memory_allocated() - base - params - lora_params
    with capsys.disabled():
        print(f"\nqwen-image full depth 1328^2, rank-64 adapters on every covered target: module weights {params / 1e9:.2f} GB + "
              f"adapters {lora_params / 1e9:.2f} GB, peak beyond them {extra / 1e9:.2f} GB (packed A / T {packed / 1e9:.2f} GB)")
    del m, eng, outs
    gc.collect()
    torch.cuda.empty_cache()
    assert packed < 2 * lora_params + 1e8
    assert extra - packed < 5e9
    assert torch.cuda.memory_allocated() - base < 1e8, "the model and its engine are freed with the last reference to them"
