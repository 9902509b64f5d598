"""Open-Sora's TeaCache comparator (`teacache_forward`, eval/magcache/experiments/opensora.py:34-227) without a GPU: the restatement
(tests/opensora_tea_ref.py) against the fixture made by executing the reference's own code (tests/golden/make_opensora_teacache_golden.py),
the C decision entry `mc_tea_opensora_decide` against the restatement, the host's bf16 `rel` against torch, and the engine's
`teacache_opensora_forward` through the kernel emulation against the restatement over miss, hit, forced and plain calls."""
import copy
import ctypes
import json
import os

import numpy as np
import pytest
import torch
from hypothesis import given, settings
from hypothesis import strategies as hs

import magcache_b200 as mc
from magcache_b200 import _lib as L
from magcache_b200 import opensora as os_mod
from magcache_b200 import patch as patch_mod
from magcache_b200.controller import OpenSoraTeaController, opensora_rel_l1

import opensora_ref as R
import opensora_tea_ref as TR

GOLD = os.path.join(os.path.dirname(__file__), "golden")
DOC = json.load(open(os.path.join(GOLD, "opensora_teacache.json")))
ARR = np.load(os.path.join(GOLD, "opensora_teacache.npz"))


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _fixture_model(dtype, thresh):
    m = R.STDiT3(**DOC["config"]).init_synthetic(DOC["seed"])
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.startswith("t_block."):
                p.mul_(DOC["t_block_scale"])
    m = m.to(dtype).eval()
    m.__class__ = type(f"TeaOracle_{dtype}_{thresh}", (R.STDiT3,), {})
    TR.install_teacache(m.__class__, thresh)
    return m


@pytest.mark.parametrize("key", sorted(DOC["runs"]))
def test_restatement_matches_reference_execution(key):
    run = DOC["runs"][key]
    dtype = torch.float32 if run["dtype"] == "fp32" else torch.bfloat16
    m = _fixture_model(dtype, run["thresh"])
    latents, y, kw = TR.video_inputs(DOC)
    gold = ARR[key]
    with torch.no_grad():
        for j, rec in enumerate(run["records"]):
            i = j % DOC["calls"]
            out = m(latents(j), TR.timestep_tensor(run, i), run["all_timesteps"], y, **kw)
            assert (m.last_forced, m.last_calc) == (rec["forced"], rec["calc"]), (key, j)
            assert m.last_rel == rec["rel"], (key, j, m.last_rel, rec["rel"])
            assert float(m.accumulated_rel_l1_distance) == rec["acc"], (key, j)
            if run["dtype"] == "fp32":
                assert rel_l2(out, torch.from_numpy(gold[j])) <= 1e-6, (key, j)
            else:
                want = torch.from_numpy(gold[j]).view(torch.bfloat16).float()
                assert torch.equal(out, want), (key, j)


def test_fixture_covers_forced_hit_and_miss():
    for key, run in DOC["runs"].items():
        recs = run["records"]
        assert recs[0]["forced"] and recs[DOC["calls"]]["forced"], key  # first call of each video
        assert any(not r["calc"] for r in recs) and any(r["calc"] and not r["forced"] for r in recs), key
    last = {k: r["records"][DOC["calls"] - 1]["forced"] for k, r in DOC["runs"].items() if r["dtype"] == "bf16"}
    assert True in last.values() and False in last.values(), last  # one schedule ends on a whole bf16 timestep, one does not


# ---- the C decision ---------------------------------------------------------------------------------------------------------
class _State:
    def __init__(self, thresh, acc=0):
        self.rel_l1_thresh, self.accumulated_rel_l1_distance = thresh, acc


def _py_rule(forced, rel, acc, thresh):
    """:96-107 literally (np.poly1d in float64)."""
    if forced:
        return True, 0
    acc += np.poly1d(TR.COEFFICIENTS)(rel)
    if acc < thresh:
        return False, acc
    return True, 0


@pytest.mark.parametrize("key", sorted(DOC["runs"]))
def test_c_decision_replays_the_fixture(key):
    run = DOC["runs"][key]
    ctrl, st = OpenSoraTeaController(), _State(run["thresh"])
    for j, rec in enumerate(run["records"]):
        calc = ctrl.decide(st, rec["forced"], rec["rel"])
        assert (calc, st.accumulated_rel_l1_distance) == (rec["calc"], rec["acc"]), (key, j)


@settings(max_examples=400, deadline=None)
@given(forced=hs.booleans(), thresh=hs.sampled_from([0.1, 0.2]), rel=hs.floats(0.0, 0.2), nudge=hs.integers(-3, 3),
       acc0=hs.floats(0.0, 0.3))
def test_c_decision_fuzz_around_threshold(forced, thresh, rel, nudge, acc0):
    """Accumulated sums placed within a few ulps of the threshold after the polynomial is added, and the forced cases."""
    rel = TR.opensora_rel_bf16(rel)
    y = float(np.poly1d(TR.COEFFICIENTS)(rel))
    acc = float(np.nextafter(thresh - y, np.inf if nudge > 0 else -np.inf)) if nudge else thresh - y
    for _ in range(abs(nudge) - 1):
        acc = float(np.nextafter(acc, np.inf if nudge > 0 else -np.inf))
    for a in (acc, acc0):
        st = _State(thresh, a)
        calc = OpenSoraTeaController().decide(st, forced, rel)
        want_calc, want_acc = _py_rule(forced, rel, a, thresh)
        assert calc == want_calc and st.accumulated_rel_l1_distance == float(want_acc), (forced, rel, a)


def test_c_decision_rejects_bad_arguments():
    calc, acc = ctypes.c_int32(), ctypes.c_double()
    coef = (ctypes.c_double * 1)(1.0)
    assert L.lib.mc_tea_opensora_decide(0, 0.1, 0.0, 0.1, coef, 0, ctypes.byref(calc), ctypes.byref(acc)) == L.MC_ERR_INVALID
    assert L.lib.mc_tea_opensora_decide(0, 0.1, 0.0, 0.1, coef, 1, None, ctypes.byref(acc)) == L.MC_ERR_INVALID


@pytest.mark.parametrize("seed", range(6))
def test_host_rel_matches_torch_bf16_expression(seed):
    """`opensora_rel_l1` from fp64 sums of the bf16-rounded terms equals torch's bf16 `((cur - prev).abs().mean() / prev.abs().mean())`."""
    g = torch.Generator().manual_seed(seed)
    prev = (torch.randn(2, 96, 144, generator=g) * 2).bfloat16()
    cur = (prev.float() + 0.02 * (seed + 1) * torch.randn(2, 96, 144, generator=g)).bfloat16()
    want = ((cur - prev).abs().mean() / prev.abs().mean()).item()
    d = (cur - prev).abs().double().sum().item()
    p = prev.abs().double().sum().item()
    assert opensora_rel_l1(d, p, cur.numel()) == want


# ---- the engine through the kernel emulation ----------------------------------------------------------------------------------
@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(os_mod, "ops", TR.namespace())
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def _trio(thresh, enable=True):
    base = R.STDiT3(**R.CONFIGS["tiny"]).init_synthetic(0)
    with torch.no_grad():
        for n, p in base.named_parameters():
            if n.startswith("t_block."):
                p.mul_(0.05)
    out = []
    for name, dtype in (("RefTea", torch.bfloat16), ("RefTea64", torch.float64)):
        m = copy.deepcopy(base).to(dtype)
        m.__class__ = type(name, (R.STDiT3,), {})
        TR.install_teacache(m.__class__, thresh, enable)
        out.append(m)
    out[1].decisions_from = out[0]
    ours = copy.deepcopy(base).to(torch.bfloat16)
    ours.__class__ = type("OursTea", (R.STDiT3,), {})
    mc.init_teacache_opensora(ours, rel_l1_thresh=thresh)
    ours.__class__.enable_teacache = enable
    return out[0], out[1], ours


def _inputs(B, T, H, W, L=12, cy=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, T, H, W, generator=g)
    d = torch.randn(B, 4, T, H, W, generator=g)
    y = torch.randn(B, 1, L, cy, generator=g)
    mask = torch.ones(B, L, dtype=torch.long)
    mask[-1, L // 2:] = 0
    kw = dict(mask=mask, fps=torch.tensor([24.0]), height=torch.tensor([8.0 * H]), width=torch.tensor([8.0 * W]))
    return (lambda i: x + 0.004 * i * d), y, kw


def _steps(n, B):
    # one timestep per sample pair, like the sampler; whole-number first / last so both are forced
    ts = [torch.tensor([1000.0 - 30.0 * i, 990.0 - 30.0 * i][:B]) for i in range(n)]
    return ts, [int(t[0].to(torch.bfloat16).item()) for t in ts]


def _check_call(i, o, r, r64, ref, ours):
    e_ref = rel_l2(r, r64)
    assert rel_l2(o, r64) <= 1.5 * e_ref + 1e-3, (i, rel_l2(o, r64), e_ref)
    assert rel_l2(o, r) <= 2 * e_ref + 1e-3, (i, rel_l2(o, r), e_ref)
    assert float(ours.accumulated_rel_l1_distance) == float(ref.accumulated_rel_l1_distance), i


@pytest.mark.parametrize("thresh", [0.1, 0.2])
@pytest.mark.parametrize("B,T,H,W", [(2, 3, 6, 10), (1, 2, 4, 6)], ids=["B2", "B1"])
def test_engine_matches_restatement(emulated, thresh, B, T, H, W):
    ref, ref64, ours = _trio(thresh)
    latents, y, kw = _inputs(B, T, H, W)
    ts, all_ts = _steps(12, B)
    calcs, forced = [], []
    with torch.no_grad():
        for i in range(12):
            r = ref(latents(i), ts[i], all_ts, y, **kw)
            # the fp64 yardstick gets the timestep as the bf16 models see it (`timestep.to(dtype)`, :51)
            r64 = ref64(latents(i).double(), ts[i].to(torch.bfloat16).double(), all_ts, y.double(), **kw)
            o = ours(latents(i), ts[i], all_ts, y, **kw)
            calcs.append(ref.last_calc)
            forced.append(ref.last_forced)
            _check_call(i, o, r, r64, ref, ours)
            assert ours.previous_modulated_input.shape == ref.previous_modulated_input.shape
            assert torch.equal(ours.previous_modulated_input.float(), ref.previous_modulated_input.float()) or \
                rel_l2(ours.previous_modulated_input, ref.previous_modulated_input) < 1e-2
            assert ours.previous_residual.shape == ref.previous_residual.shape
    assert forced[0] and forced[-1] and not all(forced)
    assert True in calcs and False in calcs, calcs


def test_plain_forward_keeps_no_residual(emulated):
    ref, ref64, ours = _trio(0.1, enable=False)
    latents, y, kw = _inputs(2, 2, 4, 6)
    ts, all_ts = _steps(3, 2)
    with torch.no_grad():
        for i in range(3):
            r = ref(latents(i), ts[i], all_ts, y, **kw)
            r64 = ref64(latents(i).double(), ts[i].to(torch.bfloat16).double(), all_ts, y.double(), **kw)
            o = ours(latents(i), ts[i], all_ts, y, **kw)
            e_ref = rel_l2(r, r64)
            assert rel_l2(o, r64) <= 1.5 * e_ref + 1e-3 and rel_l2(o, r) <= 2 * e_ref + 1e-3
    assert ours.previous_residual is None and ours.previous_modulated_input is None


def test_replaced_attributes_are_honoured(emulated):
    ref, _, ours = _trio(10.0)  # every non-forced call hits
    latents, y, kw = _inputs(2, 2, 4, 6)
    ts, all_ts = _steps(6, 2)
    with torch.no_grad():
        for m in (ref, ours):
            m(latents(0), ts[0], all_ts, y, **kw)
        g = torch.Generator().manual_seed(7)
        res = (0.3 * torch.randn(*ref.previous_residual.shape, generator=g)).bfloat16()
        mi = (ref.previous_modulated_input.float() * 1.05).bfloat16()
        for m in (ref, ours):
            m.previous_residual, m.previous_modulated_input = res.clone(), mi.clone()
        r = ref(latents(1), ts[1], all_ts, y, **kw)
        o = ours(latents(1), ts[1], all_ts, y, **kw)
    assert not ref.last_calc
    assert float(ours.accumulated_rel_l1_distance) == float(ref.accumulated_rel_l1_distance)
    assert rel_l2(o, r) < 2e-2


def test_distance_without_previous_input_raises(emulated):
    _, _, ours = _trio(0.1)
    latents, y, kw = _inputs(1, 2, 4, 6)
    with pytest.raises(TypeError, match="previous_modulated_input"), torch.no_grad():
        ours(latents(0), torch.tensor([500.0]), [1000, 33], y, **kw)


def test_unsupported_inputs_raise():
    class M:
        parallel_manager = None
        enable_teacache = True
    x = torch.zeros(1, 4, 1, 4, 4)
    with pytest.raises(NotImplementedError, match="x_mask"):
        mc.teacache_opensora_forward(M(), x, None, None, None, x_mask=torch.ones(1, 1, dtype=torch.bool))
    for sp, cp in ((2, 1), (1, 2)):
        m = M()
        m.parallel_manager = type("PM", (), dict(sp_size=sp, cp_size=cp))()
        with pytest.raises(NotImplementedError, match="parallelism"):
            mc.teacache_opensora_forward(m, x, None, None, None)
    with pytest.raises(RuntimeError, match="CUDA"):
        mc.teacache_opensora_forward(M(), x, None, None, None)


def test_init_installs_the_reference_attributes():
    class Model:
        pass
    m = mc.init_teacache_opensora(Model(), rel_l1_thresh=0.2)
    cls = type(m)
    assert (cls.enable_teacache, cls.rel_l1_thresh, cls.accumulated_rel_l1_distance) == (True, 0.2, 0)
    assert cls.previous_modulated_input is None and cls.previous_residual is None
    assert cls.forward is patch_mod.teacache_opensora_forward
