"""Qwen-Image / Qwen-Image-Edit on the H100 kernels: the patched forward and its calibration twin against the restatement
(tests/qwen_image_ref.py) in bf16 and fp64 — reduced size on CPU oracles, one layer at full width (3072 wide, 24 heads, 3584-wide
text) at the pipelines' shapes on GPU oracles — later generations against a fresh engine, the allocator after the first two calls,
and the full 60-block model's memory beside its own weights."""
import contextlib
import copy
import io

import pytest
import torch

import magcache_b200 as mc
import qwen_image_ref as qr

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


def _run(model, calls, f64=False):
    with torch.no_grad(), (qr.exact() if f64 else contextlib.nullcontext()):
        return [model(**{k: (v.double() if f64 and torch.is_tensor(v) and v.is_floating_point() else v) for k, v in kw.items()},
                      return_dict=False)[0] for kw in calls]


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
    return m


@pytest.mark.parametrize("shapes", [[(1, 16, 12)], [(1, 12, 10), (1, 9, 14)]], ids=["t2i", "edit"])
@pytest.mark.parametrize("mode", ["forward", "calibration"])
def test_reduced_size_loop_matches_oracle(shapes, mode):
    """2 blocks, 2 heads x 128, 37-token cond and 6-token uncond text, 10 steps (hits in the forward): GPU engine against the
    bf16 and fp64 restatement on CPU."""
    model = qr.tiny_model(11)
    steps, dims = 10, (16, 96)
    cal = mode == "calibration"
    ref = _install(copy.deepcopy(model), "Ref", steps, 0.5, 2, 0.2, False, cal)
    ref64 = _install(copy.deepcopy(model).double(), "Ref64", steps, 0.5, 2, 0.2, False, cal)
    ours = _install(copy.deepcopy(model).to(DEV), "Ours", steps, 0.5, 2, 0.2, True, cal)
    calls = _calls(shapes, steps, 37, 6, dims, "cpu")
    with contextlib.redirect_stdout(io.StringIO()):
        r, r64 = _run(ref, calls), _run(ref64, calls, f64=True)
        o = _run(ours, [{k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in kw.items()} for kw in calls])
    _check(o, r, r64)
    if not cal:
        assert ours._mc_qwen_engine is not None and int(ours.cnt) == int(ref.cnt)


def _full_width_layer(seed=0):
    with torch.device("meta"):
        m = qr.QwenImageTransformer2DModel(num_layers=1).to(torch.bfloat16)
    return m.to_empty(device=DEV).init_synthetic(seed)


@pytest.mark.parametrize("shapes", [[(1, 83, 83)], [(1, 58, 104)], [(1, 64, 64), (1, 64, 64)]],
                         ids=["1328x1328", "1664x928", "edit_1024x1024"])
def test_full_width_layer_miss_miss_hit_hit(shapes):
    """One block at full width through the patched forward: cond (200 text tokens) miss, uncond (6) miss, cond hit, uncond hit,
    against the restatement on the GPU in bf16 and fp64. The allocator reserves nothing new after the first two calls."""
    model = _full_width_layer()
    calls = _calls(shapes, 2, 200, 6, (64, 3584), DEV)
    ref = _install(copy.deepcopy(model), "RefW", 2, 10.0, 2, 0.5, False)
    r = _run(ref, calls)
    del ref
    ref64 = _install(copy.deepcopy(model).double(), "RefW64", 2, 10.0, 2, 0.5, False)
    r64 = [x.cpu() for x in _run(ref64, calls, f64=True)]
    del ref64
    torch.cuda.empty_cache()
    ours = _install(model, "OursW", 2, 10.0, 2, 0.5, True)
    o = []
    with torch.no_grad():
        for i, kw in enumerate(calls):
            o.append(ours(**kw, return_dict=False)[0].cpu())  # (a caller's held outputs are the caller's allocations)
            if i == 1:
                torch.cuda.synchronize()
                segs = torch.cuda.memory_stats()["segment.all.allocated"]
                spaces = {k: {n: id(v) for n, v in ws.items()} for k, ws in ours._mc_qwen_engine._spaces.items()}
    torch.cuda.synchronize()
    assert torch.cuda.memory_stats()["segment.all.allocated"] == segs
    assert {k: {n: id(v) for n, v in ws.items()} for k, ws in ours._mc_qwen_engine._spaces.items()} == spaces
    _check(o, r, r64)


def test_later_generations_equal_a_fresh_engine():
    """Three generations on one model (other text lengths, the transposed grid, then Edit shapes) against each on a fresh model
    that starts from the accumulators the previous generation left (the reference's wrap resets only the counter)."""
    model = qr.tiny_model(12).to(DEV)
    steps, dims = 8, (16, 96)
    gens = [_calls([(1, 16, 12)], steps, 37, 6, dims, DEV), _calls([(1, 12, 16)], steps, 20, 5, dims, DEV, seed=100),
            _calls([(1, 12, 8), (1, 8, 12)], steps, 37, 6, dims, DEV, seed=200)]
    a = _install(copy.deepcopy(model), "SessA", steps, 0.5, 2, 0.2, True)
    for i, g in enumerate(gens):
        fresh = _install(copy.deepcopy(model), f"SessF{i}", steps, 0.5, 2, 0.2, True)
        for n in ("accumulated_err", "accumulated_steps", "accumulated_ratio"):
            setattr(type(fresh), n, list(getattr(a, n)))
        o_a, o_f = _run(a, g), _run(fresh, g)
        assert all(torch.equal(x, y) for x, y in zip(o_a, o_f)), i
        assert all(torch.equal(x, y) for x, y in zip(a.residual_cache, fresh.residual_cache)), i


def test_full_depth_memory_beside_the_modules_weights(capsys):
    """The 60-block, 20 B-parameter model (weights allocated in place on the device): one miss and one hit at 1328^2. The
    engine reads the module's weights in place, so the peak minus the module's own weights is its copies (under 5 GB) plus
    activations."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.device("meta"):
        m = qr.QwenImageTransformer2DModel().to(torch.bfloat16)
    m = _own_class(m.to_empty(device=DEV).init_synthetic(0), "Full")
    params = sum(p.numel() * p.element_size() for p in m.parameters())
    mc.init_magcache_qwen_image(m, "qwen_image", 2, 10.0, 2, 0.5)
    calls = _calls([(1, 83, 83)], 2, 200, 6, (64, 3584), DEV)[:3]  # cond miss, uncond miss, cond hit
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        outs = [m(**kw, return_dict=False)[0] for kw in calls]
    torch.cuda.synchronize()
    assert all(bool(torch.isfinite(o.float()).all()) for o in outs) and not torch.equal(outs[0], outs[2])
    eng = m._mc_qwen_engine
    ws = sum(t.numel() * t.element_size() for sp in eng._spaces.values() for t in sp.values() if torch.is_tensor(t))
    ws += sum(t.numel() * t.element_size() for t in eng.res + [eng.spare])
    own = sum(t.numel() * t.element_size() for b in eng.w.double for t in b.values() if torch.is_tensor(t) and t.dtype == torch.float32)
    own += eng.w.ada_b.numel() * 4
    extra = torch.cuda.max_memory_allocated() - base - params
    with capsys.disabled():
        print(f"\nqwen-image full depth 1328^2: module weights {params / 1e9:.2f} GB, peak beyond them {extra / 1e9:.2f} GB "
              f"(engine copies {own / 1e6:.1f} MB, workspace + slots {ws / 1e9:.2f} GB)")
    assert own < 5e9
    assert extra - ws < 5e9
