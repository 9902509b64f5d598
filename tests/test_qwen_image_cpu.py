"""Qwen-Image / Qwen-Image-Edit on the MMDiT engine, orchestration on CPU: `magcache_qwen_image_forward` / `_calibration` and
`QwenImageEngine` driven through tests/emu_ops.py (torch emulation of the kernels' documented arithmetic) against the restatement
in tests/qwen_image_ref.py, which tests/golden/qwen_image.{json,npz} pins to the reference's own statements. Weight reading, RoPE
positions, the two CFG branches with their own text lengths and residual slots, hits that read only the final layer, the
calibration twin, refusals, and later generations against a fresh engine. The kernels themselves: tests/test_qwen_image_gpu.py."""
import contextlib
import copy
import io
import json
import os

import numpy as np
import pytest
import torch

import emu_ops
import magcache_b200 as mc
import qwen_image_ref as qr
from magcache_b200 import mmdit
from magcache_b200 import patch as patch_mod

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
T2I = [(1, 3, 4)]
EDIT = [(1, 3, 4), (1, 2, 3)]


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(mmdit, "ops", emu_ops)
    monkeypatch.setattr(patch_mod, "ops", emu_ops)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))  # the forward insists on CUDA tensors


def _own_class(m, name):
    m.__class__ = type(name, (m.__class__,), {})
    return m


def _schedule(shapes, steps, n_cond=7, n_uncond=3, seed=0):
    """The cond / uncond calls of `steps` steps: per step two calls with their own text (lengths differ) and the step's timestep."""
    calls = []
    for s in range(steps):
        t = 1.0 - s / steps * 0.9
        for b, n in enumerate((n_cond, n_uncond)):
            kw = qr.call_inputs(seed + 10 * s + b, shapes, n, t=t)
            calls.append(kw)
    return calls


def _run(model, calls):
    with torch.no_grad():
        return [model(**kw, return_dict=False)[0] for kw in calls]


def _run64(model, calls):
    m64 = copy.deepcopy(model).double()
    with qr.exact(), torch.no_grad():
        return [m64(**{k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in kw.items()},
                    return_dict=False)[0] for kw in calls]


def _models(model, steps, thresh=0.06, K=2, table="qwen_image"):
    mr = list(mc.tables()[table][2:])
    ref = _own_class(copy.deepcopy(model), "RefQwen")
    qr.init_magcache(ref, mr, steps, thresh, K)
    ref64 = _own_class(copy.deepcopy(model), "RefQwen64")
    qr.init_magcache(ref64, mr, steps, thresh, K)
    ours = _own_class(copy.deepcopy(model), "OurQwen")
    mc.init_magcache_qwen_image(ours, mr, steps, thresh, K)
    return ref, ref64, ours


def _parity(ours, ref, ref64):
    """The project's rule per output: rel-L2 to the bf16 oracle <= 2 e_ref + 1e-3 and to fp64 <= 1.5 e_ref + 1e-3, with e_ref the
    bf16 oracle's own distance to fp64."""
    bad = []
    for i, (o, r, r64) in enumerate(zip(ours, ref, ref64)):
        e_ref = rel_l2(r, r64)
        if not (rel_l2(o, r) <= 2 * e_ref + 1e-3 and rel_l2(o, r64) <= 1.5 * e_ref + 1e-3):
            bad.append((i, rel_l2(o, r), rel_l2(o, r64), e_ref))
    return bad


def _loop(shapes, steps=12, thresh=0.5, K=2, seed=0):
    model = qr.tiny_model(seed)
    ref, ref64, ours = _models(model, steps, thresh, K)
    calls = _schedule(shapes, steps, seed=seed)
    r = []
    with torch.no_grad():
        for kw in calls:
            r.append(ref(**kw, return_dict=False)[0])
            ref.__dict__.setdefault("skips", []).append(ref.last_skip)
    o = _run(ours, calls)
    r64 = _run64(ref64, calls)
    return ref, ours, r, r64, o


# ----------------------------------------------------------------------------------------------- the fixture
def _golden():
    with open(os.path.join(GOLDEN, "qwen_image.json")) as f:
        meta = json.load(f)
    return meta, np.load(os.path.join(GOLDEN, "qwen_image.npz"))


def _attrs(m, names):
    out = {}
    for n in names:
        v = getattr(m, n)
        if torch.is_tensor(v):
            v = ["tensor", int(v)]
        elif isinstance(v, list) and n in ("norm_ratio", "norm_std", "cos_dis"):  # appended to only: the length per call, the
            v = ["len", len(v)]                                                   # whole lists at the end of each generation
        elif isinstance(v, list) and not any(torch.is_tensor(x) or x is None for x in v):
            v = [float(x) for x in v]
        elif isinstance(v, list):
            v = [None if x is None else "tensor" for x in v]
        else:
            v = ["int", int(v)] if isinstance(v, int) else float(v)
        out[n] = v
    return out


@pytest.mark.parametrize("run", ["t2i_forward", "edit_forward", "t2i_calibration", "edit_calibration"])
def test_restatement_reproduces_reference_fixture(run):
    """The fixture holds the reference's own functions run on the restated model: bf16 outputs and attributes bit-equal."""
    meta, arrs = _golden()
    spec = meta["runs"][run]
    model = _own_class(qr.tiny_model(meta["seed"]), "Pinned")
    if spec["mode"] == "forward":
        qr.init_magcache(model, list(mc.tables()[spec["table"]][2:]), meta["steps"], spec["thresh"], spec["K"])
    else:
        qr.init_magcache_calibration(model, meta["steps"])
    calls = _schedule([tuple(s) for s in spec["shapes"]], meta["steps"], meta["n_cond"], meta["n_uncond"], meta["seed"])
    buf = io.StringIO()
    with torch.no_grad(), contextlib.redirect_stdout(buf):
        for _ in range(meta["generations"]):
            for i, kw in enumerate(calls):
                out = model(**kw, return_dict=False)[0]
                k = f"{run}_{i}" if _ == 0 else f"{run}_g1_{i}"
                if k in arrs.files:
                    assert torch.equal(out.view(torch.int16), torch.from_numpy(arrs[k])), k
                want = spec["attrs"][_][i]
                assert _attrs(model, list(want)) == want, (k, _attrs(model, list(want)), want)
            for n, v in (spec["lists"][_].items() if spec["mode"] == "calibration" else ()):
                assert getattr(model, n) == v, n
    assert buf.getvalue() == spec["stdout"]


# ----------------------------------------------------------------------------------------------- engine against the restatement
@pytest.mark.parametrize("shapes", [T2I, EDIT], ids=["t2i", "edit"])
def test_single_calls_match_oracle(emulated, shapes):
    model = qr.tiny_model(1)
    ref, ref64, ours = _models(model, 10)
    calls = _schedule(shapes, 1)
    assert not _parity(_run(ours, calls), _run(ref, calls), _run64(ref64, calls))


@pytest.mark.parametrize("shapes", [T2I, EDIT], ids=["t2i", "edit"])
def test_loop_with_hits_matches_oracle(emulated, shapes):
    ref, ours, r, r64, o = _loop(shapes)
    assert any(ref.skips) and not all(ref.skips[4:]), ref.skips
    assert not _parity(o, r, r64)
    for n in ("accumulated_err", "accumulated_steps", "accumulated_ratio"):
        assert getattr(ours, n) == getattr(ref, n), n
    assert int(ours.cnt) == int(ref.cnt) and type(ours.cnt) is type(ref.cnt)


def test_hit_reads_only_the_final_layer(emulated, monkeypatch):
    """A hit runs img_in, the time MLP, the final layer's modulation rows, the add, LN+modulate and proj_out: no block
    modulation weight, no txt_norm / txt_in."""
    model = qr.tiny_model(2)
    _, _, ours = _models(model, 12, thresh=0.5)
    calls = _schedule(T2I, 12)
    read = []
    real = emu_ops.gemm
    monkeypatch.setattr(emu_ops, "gemm", lambda a, b, *x, **k: (read.append(b.data_ptr()), real(a, b, *x, **k))[1])
    norms = []
    monkeypatch.setattr(emu_ops, "rmsnorm_rope_", lambda x, *a, **k: norms.append(x.shape))
    eng = None
    with torch.no_grad():
        for kw in calls:
            read.clear()
            norms.clear()
            ours(**kw)
            eng = ours._mc_qwen_engine
            if eng.res_valid[0] and len(read) == 5:  # a hit: img_in, linear_1, linear_2, norm_out.linear, proj_out
                break
        else:
            pytest.fail("no hit in the schedule")
    w = eng.w
    assert read == [p.data_ptr() for p in (w.img_w, w.t_mlp[0], w.t_mlp[2], w.ada_parts[-1][1], w.out_w)]
    assert norms == []


# ----------------------------------------------------------------------------------------------- calibration twin
def test_calibration_twin(emulated):
    steps = 6
    model = qr.tiny_model(3)
    ref = _own_class(copy.deepcopy(model), "RefCal")
    qr.init_magcache_calibration(ref, steps)
    ref64 = _own_class(copy.deepcopy(model), "RefCal64")
    qr.init_magcache_calibration(ref64, steps)
    ours = _own_class(copy.deepcopy(model), "OurCal")
    mc.init_magcache_qwen_image_calibration(ours, steps)
    calls = _schedule(EDIT, steps) * 2  # two images: the wrap keeps the lists
    b1, b2 = io.StringIO(), io.StringIO()
    with contextlib.redirect_stdout(b1):
        r = _run(ref, calls)
    with contextlib.redirect_stdout(b2):
        o = _run(ours, calls)
    with contextlib.redirect_stdout(io.StringIO()):
        r64 = _run64(ref64, calls)
    assert not _parity(o, r, r64)
    assert len(ours.norm_ratio) == len(ref.norm_ratio) == 2 * (2 * steps - 2)
    for n in ("norm_ratio", "norm_std", "cos_dis"):  # fp32/fp64 statistics against upstream's bf16 tensor ops
        assert np.allclose(getattr(ours, n), getattr(ref, n), atol=3e-2, rtol=3e-2), n
    lr, lo = b1.getvalue().splitlines(), b2.getvalue().splitlines()
    assert len(lr) == len(lo) and [x.split(":")[0] for x in lr] == [x.split(":")[0] for x in lo]
    assert lo[0].startswith("Step 2: norm_ratio=") and "\nCalibration Results:" in b2.getvalue()
    assert ours.cnt == 0 and isinstance(ours.cnt, int)


# ----------------------------------------------------------------------------------------------- refusals
def _installed(**kw):
    m = _own_class(qr.tiny_model(4, **kw), "Refuse")
    mc.init_magcache_qwen_image(m, list(mc.tables()["qwen_image"][2:]), 10)
    return m


@pytest.mark.parametrize("change,exc", [
    (dict(hidden_states=torch.zeros(2, 12, 16, dtype=torch.bfloat16)), NotImplementedError),
    (dict(encoder_hidden_states_mask=torch.tensor([[1, 1, 1, 1, 1, 1, 0]])), NotImplementedError),
    (dict(guidance=torch.tensor([1.0])), NotImplementedError),
    (dict(attention_kwargs={"scale": 0.5}), NotImplementedError),
    (dict(attention_kwargs={"other": 1}), NotImplementedError),
    (dict(txt_seq_lens=[6]), ValueError),
    (dict(img_shapes=[(1, 3, 5)]), ValueError),
])
def test_call_refusals(emulated, change, exc):
    m = _installed()
    kw = {**qr.call_inputs(0, T2I, 7), **change}
    with pytest.raises(exc), torch.no_grad():
        m(**kw)


def test_accepted_masks_and_scale(emulated):
    m = _installed()
    with torch.no_grad():
        m(**{**qr.call_inputs(0, T2I, 7), "encoder_hidden_states_mask": None, "attention_kwargs": {"scale": 1.0}})
        m(**qr.call_inputs(1, T2I, 3))


def test_token_shard_refused(emulated):
    m = mc.enable_token_shard(_installed(), 0, 2)
    with pytest.raises(NotImplementedError), torch.no_grad():
        m(**qr.call_inputs(0, T2I, 7))


@pytest.mark.parametrize("kw", [dict(attention_head_dim=64), dict(axes_dims_rope=(8, 28, 28)), dict(guidance_embeds=True)])
def test_model_refusals(emulated, kw):
    if "axes_dims_rope" in kw:
        m = _installed()
        m.config.axes_dims_rope = kw["axes_dims_rope"]
    else:
        m = _installed(**kw)
    with pytest.raises(NotImplementedError), torch.no_grad():
        m(**qr.call_inputs(0, T2I, 7, in_channels=16))


def test_fp32_parameter_and_lora_refused(emulated):
    m = _installed()
    m.proj_out.float()
    with pytest.raises(NotImplementedError), torch.no_grad():
        m(**qr.call_inputs(0, T2I, 7))
    m = _installed()

    class LoraLinear(torch.nn.Module):
        def __init__(self, base):
            super().__init__()
            self.base_layer, self.lora_A, self.lora_B, self.scaling = base, torch.nn.ModuleDict(), torch.nn.ModuleDict(), {}

    m.transformer_blocks[0].attn.to_q = LoraLinear(m.transformer_blocks[0].attn.to_q)
    with pytest.raises(NotImplementedError), torch.no_grad():
        m(**qr.call_inputs(0, T2I, 7))


def test_weights_are_the_modules_own(emulated):
    """No block matrix is copied: every weight the engine reads is the module parameter's storage."""
    m = qr.tiny_model(5)
    w = mmdit.QwenImageWeights.from_module(m, torch.device("cpu"))
    params = {p.data_ptr() for p in m.parameters()}
    mats = [w.img_w, w.txt_w, w.out_w, w.t_mlp[0], w.t_mlp[2]] + [wt for _, wt in w.ada_parts]
    for b in w.double:
        mats += list(b["qk_w"]) + list(b["cqk_w"]) + [b[k] for k in ("v_w", "o_w", "ff1_w", "ff2_w", "cv_w", "co_w", "cff1_w", "cff2_w")]
    assert all(t.data_ptr() in params for t in mats)
    assert len(w.ada_parts) == 2 * len(m.transformer_blocks) + 1 and w.single == []


# ----------------------------------------------------------------------------------------------- sessions
def test_later_generations_equal_a_fresh_engine(emulated):
    """Two generations on one model (the second with other text lengths and the transposed grid) against the second on a fresh
    model: every output and the residual slots bit-equal. The reference's wrap resets only the counter, so the fresh model starts
    from the accumulators the first generation left."""
    steps = 8
    model = qr.tiny_model(6)
    mr = list(mc.tables()["qwen_image"][2:])
    a = _own_class(copy.deepcopy(model), "SessA")
    mc.init_magcache_qwen_image(a, mr, steps, 0.5)
    fresh = _own_class(copy.deepcopy(model), "SessB")
    mc.init_magcache_qwen_image(fresh, mr, steps, 0.5)
    g1 = _schedule([(1, 3, 4)], steps, 7, 3, seed=0)
    g2 = _schedule([(1, 4, 3)], steps, 5, 2, seed=100)
    _run(a, g1)
    allocs = dict(a._mc_qwen_engine._spaces)
    for n in ("accumulated_err", "accumulated_steps", "accumulated_ratio"):
        setattr(type(fresh), n, list(getattr(a, n)))
    o_a, o_f = _run(a, g2), _run(fresh, g2)
    assert all(torch.equal(x, y) for x, y in zip(o_a, o_f))
    assert all(torch.equal(x, y) for x, y in zip(a.residual_cache, fresh.residual_cache))
    assert a.accumulated_err == fresh.accumulated_err and int(a.cnt) == int(fresh.cnt)
    assert len(a._mc_qwen_engine._spaces) == 2 and not set(allocs) & set(a._mc_qwen_engine._spaces)


def test_later_calls_allocate_no_workspace(emulated):
    model = _own_class(qr.tiny_model(7), "Alloc")
    mc.init_magcache_qwen_image(model, list(mc.tables()["qwen_image"][2:]), 6, 0.5)
    calls = _schedule(EDIT, 6)
    _run(model, calls[:2])
    eng = model._mc_qwen_engine
    before = {k: {n: id(v) for n, v in ws.items()} for k, ws in eng._spaces.items()}
    slots = [t.data_ptr() for t in eng.res]
    _run(model, calls[2:])
    assert {k: {n: id(v) for n, v in ws.items()} for k, ws in eng._spaces.items()} == before
    assert [t.data_ptr() for t in eng.res] == slots


# ----------------------------------------------------------------------------------------------- modelled defects
def _uncentred(shapes, n_txt):
    p = _real_positions(shapes, n_txt)
    n = n_txt
    for f, h, w in shapes:
        k = f * h * w
        p[n:n + k, 1] += h - h // 2
        n += k
    return p


def _text_at_zero(shapes, n_txt):
    p = _real_positions(shapes, n_txt)
    p[:n_txt] = p[:n_txt] - p[0, 0]
    return p


def _edit_frame_zero(shapes, n_txt):
    p = _real_positions(shapes, n_txt)
    p[n_txt + sum(f * h * w for f, h, w in shapes[:1]):, 0] -= 1
    return p


_real_positions = mmdit.qwen_rope_positions


def _rope_matches_oracle(shapes, n_txt):
    img_shapes = [tuple(shapes[0])] if len(shapes) == 1 else [list(shapes)]
    vid, txt = qr.QwenEmbedRope()(img_shapes, [n_txt])
    ref = torch.cat([txt, vid], dim=0)
    ref = torch.stack([ref.real, ref.imag], dim=-1).reshape(len(ref), 128)
    ours = mmdit.qwen_rope_table(mmdit.qwen_img_shapes(img_shapes), n_txt, "cpu")
    ulp = torch.abs(torch.nextafter(ref, torch.full_like(ref, 2.0)) - ref)
    return ours.shape == ref.shape and bool(((ours - ref).abs() <= ulp).all())


@pytest.mark.parametrize("shapes,n_txt", [(T2I, 7), (EDIT, 3), ([(1, 5, 2)], 4), ([(1, 83, 83)], 200), ([(1, 64, 64), (1, 64, 64)], 6)])
def test_rope_table_within_one_ulp(shapes, n_txt):
    assert _rope_matches_oracle(shapes, n_txt)


@pytest.mark.parametrize("defect", [_uncentred, _text_at_zero, _edit_frame_zero])
def test_rope_defects_are_caught(monkeypatch, defect):
    monkeypatch.setattr(mmdit, "qwen_rope_positions", defect)
    assert not _rope_matches_oracle(EDIT, 3)


def test_hit_reading_the_other_slot_is_caught(emulated, monkeypatch):
    real = mmdit.QwenImageEngine.forward
    monkeypatch.setattr(mmdit.QwenImageEngine, "forward", lambda self, kind, slot: real(self, kind, 1 - slot if kind == "hit" else slot))
    ref, ours, r, r64, o = _loop(T2I)
    assert _parity(o, r, r64)


def test_timestep_rounded_before_the_sinusoid_is_caught(emulated, monkeypatch):
    real = mmdit.QwenImageEngine.stage_inputs

    def staged(self, *a):
        real(self, *a)
        self.s_t.copy_((self.s_t.to(torch.bfloat16)).double())  # bf16(bf16(t) * 1000): FLUX's staging

    monkeypatch.setattr(mmdit.QwenImageEngine, "stage_inputs", staged)
    model = qr.tiny_model(9)
    ref, ref64, ours = _models(model, 10)
    calls = [qr.call_inputs(0, T2I, 7, t=0.7373)]
    assert _parity(_run(ours, calls), _run(ref, calls), _run64(ref64, calls))
