"""Open-Sora's RFLOW sampler (`magcache_b200.sampler.OpenSoraRFlowSampler`) without a GPU: its host arithmetic and its unfused path
against the fixture made by executing the reference's own `RFLOW.sample` (tests/golden/make_opensora_rflow_golden.py), its refusals,
and the fused step (`OpenSoraEngine.arm_step` -> `mc_opensora_head` step mode, emulated below by the op chain it replaces) against the
engine's plain forward followed by the reference's statements, over whole 30-call videos under MagCache and TeaCache."""
import copy
import json
import os

import numpy as np
import pytest
import torch

import magcache_b200 as mc
from magcache_b200 import _lib as L
from magcache_b200 import opensora as os_mod
from magcache_b200 import patch as patch_mod
from magcache_b200.sampler import OpenSoraRFlowSampler

import opensora_ref as R
import opensora_rflow_stub as S
import opensora_tea_ref as TR

GOLD = os.path.join(os.path.dirname(__file__), "golden")
DOC = json.load(open(os.path.join(GOLD, "opensora_rflow.json")))
ARR = np.load(os.path.join(GOLD, "opensora_rflow.npz"))


# ---- host arithmetic and the unfused path against the reference's execution ----------------------------------------------------
@pytest.mark.parametrize("name", sorted(S.CASES))
def test_host_schedule_matches_reference(name):
    rec = DOC["cases"][name]
    z, model_args, _ = S.case_inputs(name)
    smp = OpenSoraRFlowSampler(**S.scheduler_kwargs(name))
    ts = smp.timesteps(z.shape[0], model_args)
    assert [str(t.dtype) for t in ts] == [rec["timestep_dtype"]] * S.STEPS
    assert [t.tolist() for t in ts] == rec["timesteps"]
    dts = [smp.dt(ts, i) for i in range(S.STEPS)]
    assert [str(d.dtype) for d in dts] == [rec["dt_dtype"]] * S.STEPS
    assert [d.tolist() for d in dts] == rec["dt"]


@pytest.mark.parametrize("name", sorted(S.CASES))
def test_unfused_sampling_matches_reference(name):
    rec = DOC["cases"][name]
    z, model_args, y_null = S.case_inputs(name)
    B = z.shape[0]
    model = S.StubSTDiT3()
    with torch.no_grad():
        out = OpenSoraRFlowSampler(**S.scheduler_kwargs(name)).sample(model, z, model_args, y_null, "cpu", progress=False)
    assert len(model.calls) == S.STEPS
    assert all(c[2] == rec["all_timesteps"] for c in model.calls)
    assert [c[1][:B].tolist() for c in model.calls] == rec["timesteps"]
    zs = [c[0][:B].float() for c in model.calls] + [out]
    assert str(out.dtype) == rec["out_dtype"]
    for i, (got, want) in enumerate(zip(zs, ARR[name])):
        assert torch.equal(got.float(), torch.from_numpy(want)), (name, i)


def test_fixture_records_the_reference_refusing_two_prompts():
    for name, (_, _, _, _, _, B) in S.CASES.items():
        err = DOC["cases"][name]["reference_error"]
        assert (err is not None) == (B > 1) and (err is None or "cannot be converted to Scalar" in err), name


def test_mask_is_refused():
    z, model_args, y_null = S.case_inputs("480p_51_cfg7_B1")
    with pytest.raises(NotImplementedError, match="image / video conditioning"):
        OpenSoraRFlowSampler().sample(S.StubSTDiT3(), z, model_args, y_null, "cpu", mask=torch.ones(1, 2))


def test_token_sharded_engine_is_refused():
    m = copy.deepcopy(R.STDiT3(**R.CONFIGS["tiny"]).init_synthetic(0)).to(torch.bfloat16)
    m.__class__ = type("ShardedOS", (R.STDiT3,), {})
    patch_mod.init_magcache_opensora(m)
    mc.enable_token_shard(m, 0, 2)
    z, model_args, y_null = S.case_inputs("480p_51_cfg7_B1")
    with pytest.raises(NotImplementedError, match="token-sharded"):
        OpenSoraRFlowSampler().sample(m, z, model_args, y_null, "cpu", progress=False)


# ---- the fused step through the kernel emulation --------------------------------------------------------------------------------
def _emulated_namespace():
    ns = TR.namespace()

    def opensora_head(x, mod, w, bias, grid, crop, res=None, step=None, out=None, eps=1e-6, tag=None):
        """The op chain mc_opensora_head replaces: hit add, per-sample LN + t2i_modulate, the 32-wide GEMM, unpatchify + crop;
        step mode: the reference's statements (scheduling_rflow_open_sora.py:244-251) on that prediction."""
        T, H, W = grid
        Tx, Hx, Wx = crop
        N = T * H * W
        B, D = x.shape[0] // N, x.shape[1]
        if res is not None:
            x = ns.cache_hit_add(x, res)
        h = torch.cat([ns.ln_t2i_modulate(x[b * N:(b + 1) * N], mod[b], 1, 0) for b in range(B)])
        o = ns.gemm(h, w, bias, L.MC_EPI_BIAS_BF16)
        pred = o.view(B, T, H, W, 1, 2, 2, 8).permute(0, 7, 1, 4, 2, 5, 3, 6).reshape(B, 8, T, 2 * H, 2 * W)[:, :, :Tx, :Hx, :Wx].float()
        if step is None:
            return pred
        z, g, dt = step
        pred_cond, pred_uncond = pred.chunk(2, dim=1)[0].chunk(2, dim=0)
        v_pred = pred_uncond + g * (pred_cond - pred_uncond)
        out.copy_(z + v_pred * dt[:, None, None, None, None])
        return out

    ns.opensora_head = opensora_head
    return ns


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(os_mod, "ops", _emulated_namespace())
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


class _Unfused:
    """Hides the installed forward from the sampler: its unfused path runs the engine's forward, then the reference's statements."""

    def __init__(self, m):
        self.m, self.x_embedder = m, m.x_embedder

    def __call__(self, *a, **k):
        return self.m(*a, **k)


PRESETS = {"magcache_slow": ("magcache", 0.12, 3), "magcache_fast": ("magcache", 0.24, 5), "teacache_0.1": ("teacache", 0.1, None)}


def _model(kind, thresh, K, tag):
    base = R.STDiT3(**R.CONFIGS["tiny"]).init_synthetic(0)
    if kind == "teacache":
        with torch.no_grad():
            for n, p in base.named_parameters():
                if n.startswith("t_block."):
                    p.mul_(0.05)  # keeps the modulated input's step-to-step change in TeaCache's working range
    m = base.to(torch.bfloat16)
    m.__class__ = type(f"OursOS_{kind}_{tag}", (R.STDiT3,), {})
    if kind == "magcache":
        patch_mod.init_magcache_opensora(m, thresh=thresh, K=K)
    else:
        patch_mod.init_teacache_opensora(m, rel_l1_thresh=thresh)
    return m


def _video(seed=0, T=3, Hx=5, Wx=9, L_cap=12, cy=64):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(1, 4, T, Hx, Wx, generator=g).to(torch.bfloat16)
    y = torch.randn(1, 1, L_cap, cy, generator=g)
    y_null = torch.randn(1, 1, L_cap, cy, generator=g)
    bf = dict(dtype=torch.bfloat16)
    args = dict(y=y, mask=torch.ones(1, L_cap, dtype=torch.long), fps=torch.tensor([24], **bf), height=torch.tensor([480], **bf),
                width=torch.tensor([854], **bf), num_frames=torch.tensor([51], **bf))
    return z, args, y_null


def _run(model, wrap, record):
    z, args, y_null = _video()
    calls = []
    hook = model.register_forward_hook(lambda mod, a, out: calls.append((a[0][:1].float().clone(), {k: copy.deepcopy(getattr(mod, k, None))
                                                                                                      for k in record})))
    try:
        with torch.no_grad():
            out = OpenSoraRFlowSampler().sample(_Unfused(model) if wrap else model, z, args, y_null, "cpu", progress=False)
    finally:
        hook.remove()
    return calls, out


@pytest.mark.parametrize("preset", sorted(PRESETS))
def test_fused_step_matches_engine_plus_reference_statements(emulated, preset):
    kind, thresh, K = PRESETS[preset]
    record = (("t", "accumulated_sim", "accumulated_err", "accumulated_steps", "skip_steps") if kind == "magcache"
              else ("accumulated_rel_l1_distance",))
    fused_calls, fused = _run(_model(kind, thresh, K, "fused"), False, record)
    plain_calls, plain = _run(_model(kind, thresh, K, "plain"), True, record)
    assert len(fused_calls) == len(plain_calls) == 30
    for i, ((zf, af), (zp, ap)) in enumerate(zip(fused_calls, plain_calls)):
        assert torch.equal(zf, zp), (preset, i)  # the latent entering step i
        assert af == ap, (preset, i)             # the controller's attributes after the call
    assert torch.equal(fused, plain) and fused.dtype == torch.float32
    if kind == "magcache":  # the run covers both branches
        skips = [a["skip_steps"] for _, a in fused_calls]
        assert max(skips) > 0 and skips[0] == 0, skips
    else:  # a hit leaves the accumulated distance non-zero
        assert any(a["accumulated_rel_l1_distance"] > 0 for _, a in fused_calls)
