"""Qwen-Image / Qwen-Image-Edit with unmerged LoRA adapters on the MMDiT engine, on CPU: `magcache_qwen_image_forward` /
`magcache_qwen_image_calibration` on a model whose Linears carry PEFT-layout LoRA layers (tests/flux_lora_ref.py's `LoraLinear`,
injected by path), the engine driven through the kernel emulation with the tailed GEMM against tests/qwen_image_ref.py's model
running the reference's LoRA statements (MagCache4QwenImage/magcache_generate.py:185-192 and :249-250; calibration :106-113 and
:168-169; the Edit script has the same lines). The tailed GEMM itself: tests/test_flux_lora_gpu.py; the H100 run:
tests/test_qwen_image_lora_gpu.py."""
import contextlib
import copy
import io

import pytest
import torch
from torch import nn

import magcache_b200 as mc
import qwen_image_ref as qr
import flux_lora_ref as lref
from magcache_b200 import lora as lora_mod
from magcache_b200 import mmdit
from magcache_b200 import patch as patch_mod

T2I = [(1, 3, 4)]
EDIT = [(1, 3, 4), (1, 2, 3)]

# the covered targets, diffusers names: per block, then top level
ATTN = lref.ATTN
MLP = ("img_mlp.net.0.proj", "img_mlp.net.2", "txt_mlp.net.0.proj", "txt_mlp.net.2")
MOD = ("img_mod.1", "txt_mod.1")
TOP = ("img_in", "txt_in", "norm_out.linear", "proj_out")
SETS = {"attn": ATTN, "blocks": ATTN + MLP, "mod": MOD, "block_all": ATTN + MLP + MOD, "top": TOP, "all": ATTN + MLP + MOD + TOP}


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(mmdit, "ops", lref.emu)
    monkeypatch.setattr(patch_mod, "ops", lref.emu)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def target_names(model, which, blocks=None):
    """Module paths of the set `which` (a key of SETS); `blocks`: None or the block indices that get adapters."""
    out = []
    for i in range(len(model.transformer_blocks)):
        if blocks is None or i in blocks:
            out += [f"transformer_blocks.{i}.{t}" for t in SETS[which] if t not in TOP]
    return out + [t for t in SETS[which] if t in TOP]


def reference_lora(inner):
    """The oracle's forward (or calibration twin) inside the reference's statements: copy `attention_kwargs`, pop "scale",
    `scale_lora_layers`, the function, `unscale_lora_layers`."""

    def forward(self, *args, attention_kwargs=None, **kw):
        if attention_kwargs is not None:
            attention_kwargs = attention_kwargs.copy()
            lora_scale = attention_kwargs.pop("scale", 1.0)
        else:
            lora_scale = 1.0
        lref.scale_lora_layers(self, lora_scale)
        out = inner(self, *args, attention_kwargs=attention_kwargs, **kw)
        lref.unscale_lora_layers(self, lora_scale)
        return out

    return forward


def _as(model, name):
    m = copy.deepcopy(model)
    m.__class__ = type(name, (m.__class__,), {})
    return m


def _lora_model(which="all", rank=8, adapters=("a",), seed=0, blocks=None, model_seed=0, **kw):
    model = qr.tiny_model(model_seed)
    lref.inject_lora(model, None, adapters, rank=rank, seed=seed + 7, names=target_names(model, which, blocks), **kw)
    return model


def _models(model, steps=10, thresh=0.06, K=2, calibration=False):
    """(oracle, fp64 oracle, ours), each its own copy of `model` with its own class."""
    mr = list(mc.tables()["qwen_image"][2:])
    out = []
    for name in ("RefQL", "RefQL64"):
        m = _as(model, name)
        if calibration:
            qr.init_magcache_calibration(m, steps)
        else:
            qr.init_magcache(m, mr, steps, thresh, K)
        type(m).forward = reference_lora(qr.magcache_calibration if calibration else qr.magcache_forward)
        out.append(m)
    ours = _as(model, "OurQL")
    if calibration:
        mc.init_magcache_qwen_image_calibration(ours, steps)
    else:
        mc.init_magcache_qwen_image(ours, mr, steps, thresh, K)
    out[1].double()
    return out[0], out[1], ours


def _schedule(shapes, steps, n_cond=7, n_uncond=3, seed=0):
    calls = []
    for s in range(steps):
        t = 1.0 - s / steps * 0.9
        for b, n in enumerate((n_cond, n_uncond)):
            calls.append(qr.call_inputs(seed + 10 * s + b, shapes, n, t=t))
    return calls


def _call(m, kw, **extra):
    with torch.no_grad():
        return m(**kw, **extra, return_dict=False)[0]


def _call64(m, kw, **extra):
    kw = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in kw.items()}
    with qr.exact(), torch.no_grad():
        return m(**kw, **extra, return_dict=False)[0]


def _ok(o, r, r64):
    """The project's rule: rel-L2 to the bf16 oracle <= 2 e_ref + 1e-3 and to fp64 <= 1.5 e_ref + 1e-3, e_ref the bf16 oracle's own
    distance to fp64."""
    e_ref = rel_l2(r, r64)
    return rel_l2(o, r) <= 2 * e_ref + 1e-3 and rel_l2(o, r64) <= 1.5 * e_ref + 1e-3, (rel_l2(o, r), rel_l2(o, r64), e_ref)


def _loop(model, calls, scales, **kw):
    """Every call through the oracle, the fp64 oracle and ours with `attention_kwargs={"scale": s}` (None for 1.0 given as None);
    after each call `scaling` of every layer bit-equal to the oracle's, and the hit/miss decisions equal."""
    ref, ref64, ours = _models(model, **kw)
    bad, skips = [], []
    for i, (c, s) in enumerate(zip(calls, scales)):
        extra = {} if s is None else {"attention_kwargs": {"scale": s}}
        r, r64, o = _call(ref, c, **extra), _call64(ref64, c, **extra), _call(ours, c, **extra)
        skips.append(ref.last_skip)
        ok, errs = _ok(o, r, r64)
        if not ok:
            bad.append((i, errs))
        assert lref.scaling_state(ours) == lref.scaling_state(ref), i
        if s is not None:
            assert extra == {"attention_kwargs": {"scale": s}}  # the caller's dict is not consumed
    for n in ("accumulated_err", "accumulated_steps", "accumulated_ratio"):
        assert getattr(ours, n) == getattr(ref, n), n
    return bad, skips, ours


# ----------------------------------------------------------------------------------------------- against the oracles
@pytest.mark.parametrize("shapes", [T2I, EDIT], ids=["t2i", "edit"])
def test_loop_with_hits_both_branches(emulated, shapes):
    """Twelve steps (cond and uncond calls, own text lengths) with hits, adapters on every covered target, a non-unit scale."""
    steps = 12
    model = _lora_model("all", 8, adapters=("a", "b"), seed=1)
    lref.set_adapters(model, ["a", "b"], [0.8, -0.5])
    calls = _schedule(shapes, steps)
    bad, skips, ours = _loop(model, calls, [0.7] * len(calls), steps=steps, thresh=0.5)
    assert not bad, bad
    assert any(skips[4:]) and not all(skips[4:]), skips
    assert ours._mc_qwen_engine.lora is not None


def test_adapters_without_kwargs_change_the_output(emulated):
    """`attention_kwargs=None`, as the pipelines pass it: the adapters are applied, not the base model alone."""
    model = _lora_model("all", 16)
    calls = _schedule(T2I, 1)
    bad, _, ours = _loop(model, calls, [None] * 2)
    assert not bad, bad
    _, _, plain = _models(qr.tiny_model(0))
    for c in calls:
        assert rel_l2(_call(plain, c), _call(ours, c)) > 0.05


@pytest.mark.parametrize("which,rank", [(w, 12) for w in ("attn", "blocks", "mod", "top")] + [("all", r) for r in (4, 16, 72)])
def test_targets_and_ranks(emulated, which, rank):
    model = _lora_model(which, rank)
    calls = _schedule(EDIT, 1)
    bad, _, ours = _loop(model, calls, [0.9, 0.9])
    assert not bad, bad
    _, _, plain = _models(qr.tiny_model(0))
    assert rel_l2(_call(plain, calls[0]), _call(ours, calls[0])) > 1e-2


def test_some_blocks_only(emulated):
    model = _lora_model("block_all", 16, blocks=(1,))
    bad, _, _ = _loop(model, _schedule(T2I, 1), [None, None])
    assert not bad, bad


@pytest.mark.parametrize("scale", [1.0, 0.6, 0.0, -1.0])
def test_two_weighted_adapters_and_scales(emulated, scale):
    model = _lora_model("all", 8, adapters=("a", "b"))
    lref.set_adapters(model, ["a", "b"], [0.7, -0.4])
    calls = _schedule(T2I, 2)
    bad, _, _ = _loop(model, calls, [scale] * len(calls), thresh=-1.0)
    assert not bad, bad


def test_scaling_state_follows_the_reference_call_for_call(emulated):
    """Repeated non-unit scales (ulp drift included), scale 0's reset of `set_adapters` weights, hits and misses: every layer's
    `scaling` where the reference leaves it after each call."""
    model = _lora_model("all", 8, adapters=("a", "b"))
    lref.set_adapters(model, ["a", "b"], [0.3, 1.7])
    scales = [0.7, 0.7, 1.0 / 3, 1.0 / 3, 1.0 / 3, 1.0, 0.0, 0.9, 0.0, 0.9, 1.0 / 3, 1.0 / 3]
    bad, skips, ours = _loop(model, _schedule(T2I, 6), scales, steps=6, thresh=10.0, K=3)
    assert not bad, bad
    assert any(skips) and not all(skips)
    assert lref.scaling_state(ours)[0]["a"] == 1.0  # the reset at scale 0 dropped the set_adapters weight


def test_zero_lora_b_and_scale_zero_equal_no_adapters(emulated):
    """All-zero lora_B, and scale 0 on a rank-16 adapter: the update is an exact zero added in fp32, so the output equals the same
    model with no adapters."""
    calls = _schedule(EDIT, 2)
    _, _, plain = _models(qr.tiny_model(0), thresh=-1.0)
    _, _, zero_b = _models(_lora_model("all", 16, zero_b=True), thresh=-1.0)
    _, _, scale0 = _models(_lora_model("all", 16), thresh=-1.0)
    for c in calls:
        p = _call(plain, c)
        assert torch.equal(_call(zero_b, c), p)
        assert torch.equal(_call(scale0, c, attention_kwargs={"scale": 0.0}), p)


# ----------------------------------------------------------------------------------------------- adapters changing between calls
def test_adapter_changes_take_effect_on_the_next_call(emulated):
    model = qr.tiny_model(0)
    ref, _, ours = _models(model, thresh=-1.0)  # every call a miss
    both = (ref, ours)
    c = _schedule(T2I, 1)[0]

    def step(tag):
        a, b = _call(ref, c), _call(ours, c)
        assert rel_l2(b, a) <= 2e-2, tag
        return b

    base = step("none")
    for m in both:
        lref.inject_lora(m, None, ("a",), rank=8, seed=3, names=target_names(m, "all"))
    loaded = step("loaded")
    assert rel_l2(loaded, base) > 0.05
    for m in both:
        lref.inject_lora(m, None, ("b",), rank=16, seed=4, names=target_names(m, "attn"))
    two = step("two")
    for m in both:
        lref.set_adapters(m, ["a", "b"], [0.5, 2.0])
    assert rel_l2(step("reweighted"), two) > 1e-2
    for m in both:
        for lay in lref.lora_layers(m):
            lay.disable_adapters = True
    assert torch.equal(step("disabled"), base)
    for m in both:
        for lay in lref.lora_layers(m):
            lay.disable_adapters = False
            if "b" in lay.lora_A:
                del lay.lora_A["b"], lay.lora_B["b"]
                lay._active = [x for x in lay._active if x != "b"]
    step("deleted")
    for m in both:
        for lay in lref.lora_layers(m):
            lay.merge()
    assert rel_l2(step("merged"), base) > 0.05
    for m in both:
        for lay in lref.lora_layers(m):
            lay.unmerge()
    step("unmerged")
    for m in both:
        lref.unload_lora(m)
    assert ours._mc_qwen_engine.lora is not None
    step("removed")
    assert ours._mc_qwen_engine.lora is None


def test_fused_then_unloaded_adapters_equal_a_fresh_engine(emulated):
    """`fuse_lora()` then `unload_lora_weights()` after the engine ran the adapters: the next forward equals an engine built
    fresh from the fused module, and computes what the adapters did."""
    model = _lora_model("all", 16)
    c = _schedule(EDIT, 1)[0]
    _, _, ours = _models(model, thresh=-1.0)
    _, _, twin = _models(model, thresh=-1.0)
    before = _call(ours, c)
    for m in (ours, twin):
        for lay in lref.lora_layers(m):
            lay.merge()
        lref.unload_lora(m)
    got = _call(ours, c)
    assert torch.equal(got, _call(twin, c))
    assert ours._mc_qwen_engine.lora is None
    assert rel_l2(got, before) <= 2e-2


def test_rescale_repacks_only_t(emulated):
    """A new scale rebuilds T; the A stacks (copies of lora_A) are kept."""
    model = _lora_model("all", 8)
    _, _, ours = _models(model, thresh=-1.0)
    c = _schedule(T2I, 1)[0]
    _call(ours, c, attention_kwargs={"scale": 0.5})
    pack = ours._mc_qwen_engine.lora
    a0 = {k: v[1] for k, v in pack._cache.items() if k[-1] in ("h", "ada", "x") and len(k) <= 3}
    t0 = pack.double[0]["qk_w"][0].t
    _call(ours, c, attention_kwargs={"scale": 0.25})
    pack2 = ours._mc_qwen_engine.lora
    assert pack2 is not pack and a0 and all(pack2._cache[k][1] is v for k, v in a0.items())
    assert pack2.double[0]["qk_w"][0].t is not t0


# ----------------------------------------------------------------------------------------------- calibration twin
def test_calibration_twin(emulated):
    steps = 4
    model = _lora_model("all", 8, seed=2)
    ref, ref64, ours = _models(model, steps, calibration=True)
    calls = _schedule(EDIT, steps)
    b1, b2 = io.StringIO(), io.StringIO()
    for i, c in enumerate(calls):
        extra = {"attention_kwargs": {"scale": 0.5}}
        with contextlib.redirect_stdout(b1):
            r = _call(ref, c, **extra)
        with contextlib.redirect_stdout(io.StringIO()):
            r64 = _call64(ref64, c, **extra)
        with contextlib.redirect_stdout(b2):
            o = _call(ours, c, **extra)
        ok, errs = _ok(o, r, r64)
        assert ok, (i, errs)
        assert lref.scaling_state(ours) == lref.scaling_state(ref)
    assert len(ours.norm_ratio) == len(ref.norm_ratio) == 2 * steps - 2
    for n in ("norm_ratio", "norm_std", "cos_dis"):
        for a, b in zip(getattr(ours, n), getattr(ref, n)):
            assert abs(a - b) <= 3e-2 * abs(b) + 3e-2, n
    assert [x.split(":")[0] for x in b1.getvalue().splitlines()] == [x.split(":")[0] for x in b2.getvalue().splitlines()]


# ----------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("bad", ["dora", "lora_bias", "dropout", "time_text_embed", "stub", "other_key", "scale_without_adapters"])
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
        lref.inject_lora(model, None, ("a",), names=["time_text_embed.timestep_embedder.linear_2"])
    elif bad == "stub":  # the recognised attributes, without the rest of PEFT's surface
        class Stub(nn.Module):
            def __init__(self, base):
                super().__init__()
                self.base_layer, self.lora_A, self.lora_B, self.scaling = base, nn.ModuleDict(), nn.ModuleDict(), {}

        blk = model.transformer_blocks[1]
        blk.img_mlp.net[2] = Stub(blk.img_mlp.net[2])
    elif bad == "other_key":
        kw = dict(attention_kwargs={"scale": 0.5, "other": 1})
    elif bad == "scale_without_adapters":
        model, kw = qr.tiny_model(0), dict(attention_kwargs={"scale": 0.5})
    _, _, ours = _models(model)
    with pytest.raises(NotImplementedError) as e:
        _call(ours, _schedule(T2I, 1)[0], **kw)
    want = {"dora": "DoRA", "lora_bias": "lora_bias", "dropout": "dropout", "time_text_embed": "time_text_embed.timestep_embedder.linear_2",
            "stub": "transformer_blocks.1.img_mlp.net.2", "other_key": "other", "scale_without_adapters": "no LoRA layer"}[bad]
    assert want in str(e.value)


@pytest.mark.parametrize("calibration", [False, True], ids=["forward", "calibration"])
def test_a_refused_call_leaves_scaling_unscaled(emulated, calibration):
    """The engine refuses an input after `scale_lora_layers` ran: `unscale_lora_layers` still runs."""
    model = _lora_model("attn", 8, adapters=("a", "b"))
    lref.set_adapters(model, ["a", "b"], [0.3, 1.7])
    _, _, ours = _models(model, calibration=calibration)
    lref.lora_layers(ours)[-1].use_dora["b"] = True
    want = copy.deepcopy(model)
    lref.scale_lora_layers(want, 0.6)
    lref.unscale_lora_layers(want, 0.6)
    with pytest.raises(NotImplementedError):
        _call(ours, _schedule(T2I, 1)[0], attention_kwargs={"scale": 0.6})
    assert lref.scaling_state(ours) == lref.scaling_state(want)


def test_token_shard_still_refused_with_adapters(emulated):
    _, _, ours = _models(_lora_model("all", 8))
    mc.enable_token_shard(ours, 0, 2)
    with pytest.raises(NotImplementedError, match="token-sharded"):
        _call(ours, _schedule(T2I, 1)[0])


def test_base_weights_read_in_place_with_adapters():
    """With LoRA layers on every covered target the engine still reads each base weight in place; fp32 adapter weights are
    accepted (LoraPack converts them) while an fp32 base weight is refused."""
    model = _lora_model("all", 8)
    for lay in lref.lora_layers(model)[:3]:
        lay.lora_A["a"].float()
    w = mmdit.QwenImageWeights.from_module(model, torch.device("cpu"))
    params = {p.data_ptr() for p in model.parameters()}
    mats = [w.img_w, w.txt_w, w.out_w] + [wt for _, wt in w.ada_parts]
    for b in w.double:
        mats += list(b["qk_w"]) + list(b["cqk_w"]) + [b[k] for k in ("v_w", "o_w", "ff1_w", "ff2_w", "cv_w", "co_w", "cff1_w", "cff2_w")]
    assert all(t.data_ptr() in params for t in mats)
    assert w.double[0]["qk_w"][0].data_ptr() == model.transformer_blocks[0].attn.to_q.base_layer.weight.data_ptr()
    model.transformer_blocks[0].attn.to_v.base_layer.float()
    with pytest.raises(NotImplementedError, match="to_v.base_layer.weight"):
        mmdit.QwenImageWeights.from_module(model, torch.device("cpu"))


# ----------------------------------------------------------------------------------------------- what a call launches
def _launches(monkeypatch, ours, calls):
    """Per call of `calls`: the GEMMs launched, as (weight data pointer, whether it carries a tail)."""
    log, out = [], []
    real = lref.emu.gemm
    monkeypatch.setattr(lref.emu, "gemm", lambda a, b, *x, **k: (log.append((b.data_ptr(), k.get("tail") is not None)), real(a, b, *x, **k))[1])
    for c in calls:
        log.clear()
        _call(ours, c)
        out.append(list(log))
    monkeypatch.setattr(lref.emu, "gemm", real)
    return out


def test_launch_plan(emulated, monkeypatch):
    """A hit with adapters only on block Linears issues the launches of a hit without adapters (it reads no block adapter or
    modulation weight); a miss with adapters on every covered target adds exactly one down-projection per distinct adapted GEMM
    input (8 per block, the block and final-layer modulation groups, img_in, txt_in, proj_out) and tails every adapted GEMM; a hit
    with adapters everywhere adds only those of img_in, norm_out.linear and proj_out."""
    steps = 8
    calls = _schedule(T2I, steps)
    model = qr.tiny_model(0)
    runs = {}
    for tag, which in (("none", None), ("blocks", "block_all"), ("all", "all")):
        m = copy.deepcopy(model)
        if which is not None:
            lref.inject_lora(m, None, ("a",), rank=8, seed=3, names=target_names(m, which))
        _, _, ours = _models(m, steps, thresh=0.5)
        runs[tag] = (_launches(monkeypatch, ours, calls), ours._mc_qwen_engine)
    n_blocks = len(model.transformer_blocks)
    (none, e_none), (blocks, e_blocks), (alls, e_all) = runs["none"], runs["blocks"], runs["all"]
    hits = [i for i, log in enumerate(none) if len(log) == 5]
    assert hits and len(hits) < len(calls), [len(x) for x in none]
    for i in hits:
        for log, eng in ((none[i], e_none), (blocks[i], e_blocks)):
            w = eng.w
            assert log == [(t.data_ptr(), False) for t in (w.img_w, w.t_mlp[0], w.t_mlp[2], w.ada_parts[-1][1], w.out_w)]
        w0, groups = e_all.w, e_all.lora.groups
        assert [p for p, _ in alls[i]] == [groups["x"].A.data_ptr(), w0.img_w.data_ptr(), w0.t_mlp[0].data_ptr(), w0.t_mlp[2].data_ptr(),
                                               groups["ada_out"].A.data_ptr(), w0.ada_parts[-1][1].data_ptr(),
                                               groups["head"].A.data_ptr(), w0.out_w.data_ptr()]
        assert [t for _, t in alls[i]] == [False, True, False, False, False, True, False, True]
    miss = [i for i in range(len(calls)) if i not in hits]
    for i in miss:
        extra = len(alls[i]) - len(none[i])
        assert extra == 8 * n_blocks + 5, extra
        assert sum(t for _, t in alls[i]) == len(target_names(model, "all"))
        a_ptrs = {g.A.data_ptr() for g in e_all.lora.groups.values()} | {g.A.data_ptr() for b in e_all.lora.double for g in b["lora"].values()}
        assert sum(p in a_ptrs for p, _ in alls[i]) == extra
        assert len(blocks[i]) - len(none[i]) == 8 * n_blocks + 1  # the blocks' groups and the block modulation group


def test_cfg_calls_share_one_pack_with_their_own_u(emulated):
    """True CFG: the cond and uncond calls of a step (own text lengths, own workspaces) read one pack; each workspace keeps its
    own U buffers, allocated on its first call with adapters only."""
    model = _lora_model("all", 8)
    _, _, ours = _models(model, thresh=-1.0)
    calls = _schedule(T2I, 3)
    _call(ours, calls[0]), _call(ours, calls[1])
    eng = ours._mc_qwen_engine
    pack = eng.lora
    us = {k: {n: v.data_ptr() for n, v in ws["_lora_u"].items()} for k, ws in eng._spaces.items()}
    assert len(us) == 2 and all(us.values())
    assert {n[1] for n in us[(12, 3)] if n[0] == "ch"} == {3} and {n[1] for n in us[(12, 7)] if n[0] == "ch"} == {7}
    for c in calls[2:]:
        _call(ours, c)
    assert eng.lora is pack
    assert {k: {n: v.data_ptr() for n, v in ws["_lora_u"].items()} for k, ws in eng._spaces.items()} == us


def test_per_call_check_cost_at_qwen_image_module_count():
    """Host cost of `LoraScan.scan` on an unchanged module with Qwen-Image's 60 blocks: printed, and bounded loosely."""
    import time
    model = qr.QwenImageTransformer2DModel(in_channels=16, out_channels=4, num_layers=60, num_attention_heads=1, joint_attention_dim=32)
    for tag in ("no adapters", "rank-16 adapters on every covered target"):
        if tag != "no adapters":
            lref.inject_lora(model, None, ("a",), rank=16, names=target_names(model, "all"))
        scan = lora_mod.LoraScan(model, lora_mod.QWEN)
        scan.scan()
        n = 20
        t0 = time.perf_counter()
        for _ in range(n):
            *_, changed = scan.scan()
        us = (time.perf_counter() - t0) / n * 1e6
        assert not changed
        print(f"[qwen lora per-call check] {tag}: {us:.0f} us per call ({len(scan.positions)} positions)")
        assert us < 100000
