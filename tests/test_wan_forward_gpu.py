"""End-to-end parity of the H100 path (called exactly as the reference calls it: `model.forward = magcache_forward` + class
attributes) against the CPU oracle restatement of MagCache4Wan2.1/magcache_generate.py:198-312 on identical synthetic latents,
timesteps, text embeddings and weights.

Tolerances. The skip mask / controller state: bit-exact. Tensors: both implementations run bf16 GEMMs with fp32 accumulation
but sum in different orders (MKL/oneDNN vs wgmma), so individual bf16 roundings flip by one ulp and the difference grows
with depth; an element-wise rtol 1e-3 is not meaningful for a bf16 pipeline. We therefore check (a) relative L2 error of our
output against the oracle <= 2e-2, and (b) the north-star criterion in the only form that is well defined: our error against
an fp64 evaluation of the same network is no larger than 1.5x the bf16 oracle's own error against it (+1e-4 absolute).
"""
import copy
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def build(cfg_name, seed=0):
    from oracle import wan_ref
    model = wan_ref.WanModel(**wan_ref.CONFIGS[cfg_name], text_dim=512, text_len=64).init_synthetic(seed)
    return wan_ref, model


def make_inputs(seed, grid=(3, 16, 24), text_dim=512, L=37):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(16, *grid, generator=g)
    ctx = torch.randn(L, text_dim, generator=g)
    ctx_null = torch.randn(L - 5, text_dim, generator=g)
    return lat, ctx, ctx_null


def install_ref(wan_ref, model, steps, **kw):
    cls = type("RefWan", (model.__class__,), {})  # private subclass: class-level state does not leak between tests
    model.__class__ = cls
    from magcache_b200 import tables
    wan_ref.install_magcache(cls, tables()["wan2.1_t2v_1.3b"], steps, **kw)
    return model


def install_ours(model_gpu, steps, **kw):
    import magcache_b200 as mc
    cls = type("OurWan", (model_gpu.__class__,), {})
    model_gpu.__class__ = cls
    mc.init_magcache(model_gpu, steps, table="wan2.1_t2v_1.3b", **kw)
    return model_gpu


@pytest.mark.parametrize("cfg_name", ["tiny", "small"])
def test_single_forward_vs_oracle_and_fp64(cfg_name):
    wan_ref, model = build(cfg_name)
    lat, ctx, _ = make_inputs(1)
    n_tok = lat.shape[1] * (lat.shape[2] // 2) * (lat.shape[3] // 2)
    t = torch.tensor([731.0])
    ref_model = install_ref(wan_ref, copy.deepcopy(model), 10)
    with torch.no_grad():
        ref = ref_model([lat], t=t, context=[ctx], seq_len=n_tok)[0]
        # fp64 evaluation of the same network (no bf16 rounding anywhere)
        m64 = install_ref(wan_ref, copy.deepcopy(model).double(), 10)
        with wan_ref.exact_fp64():
            exact = m64([lat.double()], t=t, context=[ctx.double()], seq_len=n_tok)[0]
    ours_model = install_ours(copy.deepcopy(model).to(DEV), 10)
    out = ours_model([lat.to(DEV)], t=t.to(DEV), context=[ctx.to(DEV)], seq_len=n_tok)[0].cpu()
    assert out.shape == ref.shape == (16, *lat.shape[1:]) and out.dtype == torch.float32
    e_ours, e_ref, e_vs = rel_l2(out, exact), rel_l2(ref, exact), rel_l2(out, ref)
    print(f"[{cfg_name}] rel-L2: ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e} | ours vs oracle {e_vs:.3e}")
    assert e_vs <= 2e-2
    assert e_ours <= 1.5 * e_ref + 1e-4


def test_seq_len_padding_is_accepted():
    """seq_len > token count (upstream rounds it up to the sequence-parallel size, magcache_generate.py:242-246): same output as the
    oracle run WITH the padded rows; our residual cache keeps token-count rows."""
    wan_ref, model = build("tiny")
    lat, ctx, _ = make_inputs(4)
    n_tok = lat.shape[1] * (lat.shape[2] // 2) * (lat.shape[3] // 2)
    t = torch.tensor([512.0])
    ref_model = install_ref(wan_ref, copy.deepcopy(model), 10)
    ours_model = install_ours(copy.deepcopy(model).to(DEV), 10)
    with torch.no_grad():
        ref = ref_model([lat], t=t, context=[ctx], seq_len=n_tok + 7)[0]
    out = ours_model([lat.to(DEV)], t=t.to(DEV), context=[ctx.to(DEV)], seq_len=n_tok + 7)[0].cpu()
    assert rel_l2(out, ref) <= 2e-2
    assert ref_model.residual_cache[0].shape[1] == n_tok + 7 and ours_model.residual_cache[0].shape[1] == n_tok
    assert rel_l2(ours_model.residual_cache[0].cpu()[0], ref_model.residual_cache[0][0, :n_tok]) <= 3e-2
    with pytest.raises(AssertionError):  # :242
        ours_model([lat.to(DEV)], t=t.to(DEV), context=[ctx.to(DEV)], seq_len=n_tok - 1)


def test_i2v_forward_vs_oracle_and_fp64():
    """The same patched forward on an i2v model (magcache_generate.py:226-227, :233-234, :264-266; installed at :989-1018 with
    the 480P / 720P tables): `y` concatenated under the latent channels (in_dim 36), CLIP tokens through `img_emb`
    (LayerNorm - Linear - GELU(erf) - Linear - LayerNorm) and the image cross-attention branch summed with the text one.
    miss, miss, then the hit path on both CFG slots, against the oracle; first call also against the fp64 evaluation."""
    from oracle import wan_ref
    import magcache_b200 as mc
    model = wan_ref.WanModel(dim=256, ffn_dim=512, num_heads=2, num_layers=2, in_dim=36, text_dim=512, text_len=64, model_type="i2v",
                             clip_dim=192).init_synthetic(3)
    g = torch.Generator().manual_seed(5)
    lat = torch.randn(16, 3, 16, 24, generator=g)
    y = torch.randn(20, 3, 16, 24, generator=g)
    ctx, ctx_null = torch.randn(37, 512, generator=g), torch.randn(30, 512, generator=g)
    clip = torch.randn(1, 257, 192, generator=g)
    n_tok = 3 * 8 * 12
    t = torch.tensor([640.0])
    steps = 4
    table = mc.tables()["wan2.1_i2v_480p"]

    def ref_install(m):
        cls = type("RefWanI2V", (m.__class__,), {})
        m.__class__ = cls
        wan_ref.install_magcache(cls, table, steps, thresh=10.0, K=3, retention_ratio=0.25)  # eligible from call 2: hit, hit
        return m

    ref_model = ref_install(copy.deepcopy(model))
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("OurWanI2V", (ours.__class__,), {})
    mc.init_magcache(ours, steps, thresh=10.0, K=3, retention_ratio=0.25, mag_ratios=table)
    with torch.no_grad():
        m64 = ref_install(copy.deepcopy(model).double())
        with wan_ref.exact_fp64():
            exact = m64([lat.double()], t=t, context=[ctx.double()], seq_len=n_tok, clip_fea=clip.double(), y=[y.double()])[0]
        for i, c in enumerate((ctx, ctx_null, ctx, ctx_null)):
            ref = ref_model([lat], t=t, context=[c], seq_len=n_tok, clip_fea=clip, y=[y])[0]
            out = ours([lat.to(DEV)], t=t.to(DEV), context=[c.to(DEV)], seq_len=n_tok, clip_fea=clip.to(DEV), y=[y.to(DEV)])[0].cpu()
            assert out.shape == ref.shape == (16, 3, 16, 24)
            assert bool(ref_model.last_skip) == (i >= 2)
            assert rel_l2(out, ref) <= 2e-2, (i, rel_l2(out, ref))
            if i == 0:
                e_ours, e_ref = rel_l2(out, exact), rel_l2(ref, exact)
                print(f"[i2v] rel-L2: ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e}")
                assert e_ours <= 1.5 * e_ref + 1e-4
            assert ours.cnt == ref_model.cnt and ours.accumulated_err == ref_model.accumulated_err
    with pytest.raises(AssertionError):  # :226-227
        ours([lat.to(DEV)], t=t.to(DEV), context=[ctx.to(DEV)], seq_len=n_tok)


def test_vace_forward_vs_oracle_and_fp64():
    """`magcache_vace_forward` (magcache_generate.py:439-560, installed at :1126-1150): control video -> vace_patch_embedding ->
    control blocks (before_proj mixing with the main input, after_proj hints) -> every second main block adds its hint.
    miss, miss, hit, hit against the oracle, the first call also against fp64; then a non-default vace_context_scale."""
    from oracle import wan_ref
    import magcache_b200 as mc
    model = wan_ref.WanModel(dim=256, ffn_dim=512, num_heads=2, num_layers=4, text_dim=512, text_len=64, model_type="vace",
                             vace_in_dim=24).init_synthetic(7)
    g = torch.Generator().manual_seed(6)
    lat, vc = torch.randn(16, 3, 16, 24, generator=g), torch.randn(24, 3, 16, 24, generator=g)
    ctx, ctx_null = torch.randn(37, 512, generator=g), torch.randn(30, 512, generator=g)
    n_tok, t, steps = 3 * 8 * 12, torch.tensor([777.0]), 4
    table = mc.tables()["wan2.1_vace_1.3b"]

    def ref_install(m):
        cls = type("RefWanVace", (m.__class__,), {})
        m.__class__ = cls
        wan_ref.install_magcache(cls, table, steps, thresh=10.0, K=3, retention_ratio=0.25, vace=True)
        return m

    ref_model = ref_install(copy.deepcopy(model))
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("OurWanVace", (ours.__class__,), {})
    mc.init_magcache(ours, steps, thresh=10.0, K=3, retention_ratio=0.25, mag_ratios=table)
    assert type(ours).forward is mc.magcache_vace_forward
    with torch.no_grad():
        m64 = ref_install(copy.deepcopy(model).double())
        with wan_ref.exact_fp64():
            exact = m64([lat.double()], t=t, vace_context=[vc.double()], context=[ctx.double()], seq_len=n_tok)[0]
        for i, c in enumerate((ctx, ctx_null, ctx, ctx_null)):
            ref = ref_model([lat], t=t, vace_context=[vc], context=[c], seq_len=n_tok)[0]
            out = ours([lat.to(DEV)], t=t.to(DEV), vace_context=[vc.to(DEV)], context=[c.to(DEV)], seq_len=n_tok)[0].cpu()
            assert bool(ref_model.last_skip) == (i >= 2)
            assert rel_l2(out, ref) <= 2e-2, (i, rel_l2(out, ref))
            if i == 0:
                e_ours, e_ref = rel_l2(out, exact), rel_l2(ref, exact)
                print(f"[vace] rel-L2: ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e}")
                assert e_ours <= 1.5 * e_ref + 1e-4
            assert ours.cnt == ref_model.cnt and ours.accumulated_err == ref_model.accumulated_err
        # the control branch matters, and a scaled hint follows the oracle too
        mc.reset_magcache(ours)
        ref_model.cnt = 0
        ref_s = ref_model([lat], t=t, vace_context=[vc], context=[ctx], seq_len=n_tok, vace_context_scale=0.5)[0]
        out_s = ours([lat.to(DEV)], t=t.to(DEV), vace_context=[vc.to(DEV)], context=[ctx.to(DEV)], seq_len=n_tok, vace_context_scale=0.5)[0].cpu()
        assert rel_l2(out_s, ref_s) <= 2e-2
        assert rel_l2(out_s, ref) > 1e-2  # != the scale-1 result
    with pytest.raises(TypeError):
        mc.magcache_forward(ours, [lat.to(DEV)], t.to(DEV), [ctx.to(DEV)], n_tok)  # a VACE model without its control video


def test_teacache_comparator_loop_vs_oracle():
    """`teacache_forward` (eval/magcache/experiments/Wan2.1_EVAL/wan_teacache.py:457-590) on the same engine: 8 steps x cond/uncond,
    the timestep embedding drifting as in a real schedule; same compute/skip decisions as the oracle on every call (the distance is
    measured on each side's own embedding), same accumulators to 1e-4, outputs and cached residuals within the usual tolerance."""
    import magcache_b200 as mc
    wan_ref, model = build("tiny")
    steps = 8
    coef = [0.02, 0.04, 0.0]  # rescale polynomial sized for this random-weight model (rel. L1 between steps ~0.9): mixes hits and misses
    ref_model = copy.deepcopy(model)
    ref_model.__class__ = type("RefTea", (ref_model.__class__,), {})
    wan_ref.install_teacache(type(ref_model), steps, 0.08, coef)
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("OurTea", (ours.__class__,), {})
    mc.init_teacache(ours, steps, teacache_thresh=0.08, coefficients=coef)
    assert type(ours).ret_steps == 2 and type(ours).cutoff_steps == 2 * steps - 2
    lat, ctx, ctx_null = make_inputs(3)
    n_tok = lat.shape[1] * (lat.shape[2] // 2) * (lat.shape[3] // 2)
    sig = wan_ref.flow_sigmas(steps)
    skips = []
    with torch.no_grad():
        for i in range(steps):
            t = torch.tensor([float(sig[i] * 1000)])
            for c in (ctx, ctx_null):
                ref = ref_model([lat], t=t, context=[c], seq_len=n_tok)[0]
                out = ours([lat.to(DEV)], t=t.to(DEV), context=[c.to(DEV)], seq_len=n_tok)[0].cpu()
                skips.append(int(ref_model.last_skip))
                assert rel_l2(out, ref) <= 2e-2, (i, rel_l2(out, ref))
                assert ours.cnt == ref_model.cnt
                for sfx in ("even", "odd"):
                    a, b = getattr(ours, "accumulated_rel_l1_distance_" + sfx), getattr(ref_model, "accumulated_rel_l1_distance_" + sfx)
                    assert abs(a - b) <= 1e-4 * max(1.0, abs(b)), (i, sfx, a, b)
                    ro, rr = getattr(ours, "previous_residual_" + sfx), getattr(ref_model, "previous_residual_" + sfx)
                    assert (ro is None) == (rr is None)
                    if rr is not None:
                        assert rel_l2(ro.cpu(), rr) <= 3e-2
    assert 0 < sum(skips) < len(skips) - 4, skips  # the run exercised both branches beyond the forced first / last steps
    print("teacache skips:", "".join(map(str, skips)))


def test_magcache_loop_mask_cache_and_outputs():
    """20 forward calls (10 steps x cond/uncond) through the patched forward on both sides, same inputs every call.
    Checks: identical skip decisions (bit-exact), controller attributes, residual-cache contents, per-call outputs."""
    wan_ref, model = build("tiny")
    steps = 10
    kw = dict(thresh=0.12, K=2, retention_ratio=0.2)
    ref_model = install_ref(wan_ref, copy.deepcopy(model), steps, **kw)
    ours_model = install_ours(copy.deepcopy(model).to(DEV), steps, **kw)
    assert np.array_equal(type(ref_model).mag_ratios, type(ours_model).mag_ratios)
    lat, ctx, ctx_null = make_inputs(2)
    n_tok = lat.shape[1] * (lat.shape[2] // 2) * (lat.shape[3] // 2)
    sig = wan_ref.flow_sigmas(steps)
    skips_ref, skips_ours = [], []
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():
        for i in range(steps):
            t = torch.tensor([float(sig[i] * 1000)])
            x = lat + 0.1 * i * torch.randn(lat.shape, generator=g)  # a new latent every step, identical on both sides
            for c in (ctx, ctx_null):
                cnt_before = ours_model.cnt
                ref = ref_model([x], t=t, context=[c], seq_len=n_tok)[0]
                out = ours_model([x.to(DEV)], t=t.to(DEV), context=[c.to(DEV)], seq_len=n_tok)[0].cpu()
                skips_ref.append(int(ref_model.last_skip))
                slot = cnt_before % 2
                r_ours = ours_model.residual_cache[slot]
                r_ref = ref_model.residual_cache[slot]
                assert r_ours.shape == r_ref.shape and r_ours.dtype == torch.float32
                assert rel_l2(r_ours.cpu(), r_ref) <= 3e-2, (i, rel_l2(r_ours.cpu(), r_ref))
                assert rel_l2(out, ref) <= 2e-2, (i, rel_l2(out, ref))
                for attr in ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"):
                    assert getattr(ours_model, attr) == getattr(ref_model, attr), attr  # float64 state, bit-exact
    from magcache_b200.controller import make_ctrl_config, schedule_mask
    from magcache_b200.config import MagCacheConfig
    cfg = MagCacheConfig("wan2.1", sample_steps=steps, table="wan2.1_t2v_1.3b", **{"thresh": 0.12, "K": 2, "retention_ratio": 0.2})
    mask = schedule_mask(make_ctrl_config(cfg.num_steps, cfg.thresh, cfg.K, cfg.retention_ratio, cfg.resolved_ratios(), **cfg.ctrl_kwargs()), 2 * steps)
    assert mask.tolist() == skips_ref and sum(skips_ref) > 0
    assert ours_model.cnt == 0  # wrapped around after num_steps calls


def test_fused_denoise_step_equals_two_calls_plus_cfg_step():
    """SURVEY §8f-1 as written: `FlowEulerSampler.denoise` (cond call, then the unconditional call whose head epilogue applies the
    CFG combine and the Euler update, `mc_head_unpatchify_step`) against the two patched-forward calls + `mc_cfg_step`, over a
    schedule with hits and misses: same hit / miss sequence, latents bit-equal every step, latent updated in place."""
    import magcache_b200 as mc
    from magcache_b200 import ops
    wan_ref, model = build("tiny")
    steps, guide = 10, 5.0
    kw = dict(thresh=0.12, K=2, retention_ratio=0.2)
    a_model = install_ours(copy.deepcopy(model).to(DEV), steps, **kw)
    b_model = install_ours(copy.deepcopy(model).to(DEV), steps, **kw)
    lat, ctx, ctx_null = (v.to(DEV) for v in make_inputs(4))
    n_tok = lat.shape[1] * (lat.shape[2] // 2) * (lat.shape[3] // 2)
    sig = mc.sampling_sigmas(steps, 5.0)
    sa, sb = mc.FlowEulerSampler(sig), mc.FlowEulerSampler(sig)
    xa, xb = lat.clone(), lat.clone()
    launches = []
    with torch.no_grad():
        for i in range(steps):
            t = torch.tensor([sa.timestep], dtype=torch.float32, device=DEV)
            cond = a_model([xa], t=t, context=[ctx], seq_len=n_tok)[0]
            uncond = a_model([xa], t=t, context=[ctx_null], seq_len=n_tok)[0]
            xa = sa.step(cond, uncond, guide, xa)
            n0 = ops.LAUNCHES
            out = sb.denoise(b_model, xb, t, ctx, ctx_null, n_tok, guide)
            launches.append(ops.LAUNCHES - n0)
            assert out.data_ptr() == xb.data_ptr()
            assert torch.equal(xa, xb), i
            for attr in ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"):
                assert getattr(a_model, attr) == getattr(b_model, attr), attr
    assert min(launches) < 40 < max(launches)  # steps where both calls hit the cache: two prologues + two head launches


def test_eval_variant_loop_vs_oracle():
    """`magcache_eval_forward` (eval/magcache/experiments/Wan2.1_EVAL/wan_magcache.py:682-817, the code behind the paper's Wan2.1
    rows) for one whole 50-step video: identical hit/miss sequence (62 of 100 skipped at 0.12 / K4), float64 accumulators bit-equal,
    outputs and the `[2, B, N, D, 1]` residual tensor within the usual tolerance of the oracle's rolled FIFO."""
    import magcache_b200 as mc
    wan_ref, model = build("tiny")
    steps = 50
    ref_model = copy.deepcopy(model)
    ref_model.__class__ = type("RefEval", (ref_model.__class__,), {})
    wan_ref.install_magcache_eval(type(ref_model), mc.tables()["wan2.1_eval"], steps, 0.12, 4)
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("OurEval", (ours.__class__,), {})
    mc.init_magcache_eval(ours, steps, thresh=0.12, K=4)
    lat, ctx, ctx_null = make_inputs(8, grid=(2, 8, 12))
    n_tok = lat.shape[1] * (lat.shape[2] // 2) * (lat.shape[3] // 2)
    sig = wan_ref.flow_sigmas(steps)
    skips = 0
    with torch.no_grad():
        for i in range(steps):
            t = torch.tensor([float(sig[i] * 1000)])
            for c in (ctx, ctx_null):
                t_before = ours.t
                ref = ref_model([lat], t=t, context=[c], seq_len=n_tok)[0]
                out = ours([lat.to(DEV)], t=t.to(DEV), context=[c.to(DEV)], seq_len=n_tok)[0].cpu()
                skips += int(ref_model.last_skip)
                assert rel_l2(out, ref) <= 2e-2, (i, rel_l2(out, ref))
                assert ours.t == ref_model.t and ours.skip_steps == ref_model.skip_steps
                for attr in ("accumulated_sim", "accumulated_err", "accumulated_steps"):
                    assert [float(v) for v in getattr(ours, attr)] == [float(v) for v in getattr(ref_model, attr)], (i, attr)
                if t_before >= 10:
                    slot = t_before % 2
                    assert tuple(ours.residual_cache.shape) == tuple(ref_model.residual_cache.shape) == (2, 1, n_tok, 256, 1)
                    assert rel_l2(ours.residual_cache[slot][..., -1].cpu(), ref_model.residual_cache[slot][..., -1]) <= 3e-2
                else:
                    assert ours.residual_cache is None and ref_model.residual_cache is None
    assert skips == 62 and ours.t == 0


def test_cuda_graph_replay_equals_eager_with_split_attention(monkeypatch):
    """Graph mode (default for token-sharded runs, `MC_GRAPHS=1` here) on one GPU: eager warm-up, capture, replay — bit-equal to
    the eager engine over miss, miss, hit, hit, miss, miss on a 1024-token grid, where the small attention grid takes the split-KV
    path (its scratch is allocated in the eager call, never during capture)."""
    import magcache_b200 as mc
    dims = mc.WanDims(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128, text_len=32)
    g = torch.Generator().manual_seed(11)
    lat = torch.randn(16, 4, 32, 32, generator=g).to(DEV)
    ctxs = [torch.randn(20, 128, generator=g).to(DEV), torch.randn(17, 128, generator=g).to(DEV)]
    n_tok = 4 * 16 * 16
    outs = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("MC_GRAPHS", mode)
        model = mc.WanModelHandle(mc.WanWeights.random(dims, torch.device(DEV), seed=4))
        assert model._mc_engine.use_graphs == (mode == "1")
        mc.init_magcache(model, 3, thresh=10.0, K=1, retention_ratio=0.34, mag_ratios=[1.0] * 6)  # miss miss | hit hit | miss miss
        res = []
        for video in range(2):
            for i in range(6):
                t = torch.tensor([900.0 - 100.0 * (i // 2)], device=DEV)
                res.append(model([lat * (1.0 + 0.05 * i)], t=t, context=[ctxs[i % 2]], seq_len=n_tok)[0].clone())
        outs[mode] = res
        if mode == "1":
            assert all(isinstance(v, tuple) for v in model._mc_engine._graphs.values()) and len(model._mc_engine._graphs) == 4
    for a, b in zip(outs["0"], outs["1"]):
        assert torch.equal(a, b)


def test_calibration_matches_oracle(tmp_path):
    wan_ref, model = build("tiny")
    steps = 3
    ref_model = copy.deepcopy(model)
    ref_cls = type("RefCal", (ref_model.__class__,), {})
    ref_model.__class__ = ref_cls
    wan_ref.install_magcache(ref_cls, None, steps, calibration=True)
    import magcache_b200 as mc
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("OurCal", (ours.__class__,), {})
    mc.init_magcache_calibration(ours, steps)
    type(ours).calibration_dir = str(tmp_path)  # where the end-of-video dump goes (reference: the working directory, :191-193)
    lat, ctx, ctx_null = make_inputs(3)
    n_tok = lat.shape[1] * (lat.shape[2] // 2) * (lat.shape[3] // 2)
    sig = wan_ref.flow_sigmas(steps)
    with torch.no_grad():
        for i in range(steps):
            t = torch.tensor([float(sig[i] * 1000)])
            x = lat * (1 - 0.2 * i)
            for c in (ctx, ctx_null):
                ref_model([x], t=t, context=[c], seq_len=n_tok)
                ours([x.to(DEV)], t=t.to(DEV), context=[c.to(DEV)], seq_len=n_tok)
    assert len(ours.norm_ratio) == len(ref_model.norm_ratio) == 2 * steps - 2
    # the statistics are functions of two bf16-pipeline residuals: agreement to ~1e-2 relative is the noise floor
    for a, b in zip(ours.norm_ratio, ref_model.norm_ratio):
        assert abs(a - b) <= 2e-2 * abs(b), (ours.norm_ratio, ref_model.norm_ratio)
    for a, b in zip(ours.cos_dis, ref_model.cos_dis):
        assert abs(a - b) <= 2e-2 + 0.2 * abs(b), (ours.cos_dis, ref_model.cos_dis)
    # the dump is the reference's (`save_json("wan2_1_mag_ratio", self.norm_ratio)`) and feeds straight back as a table
    import json
    with open(tmp_path / "wan2_1_mag_ratio.json") as f:
        assert json.load(f) == ours.norm_ratio
    assert (tmp_path / "wan2_1_mag_std.json").exists() and (tmp_path / "wan2_1_cos_dis.json").exists()
    mc.init_magcache(ours, steps, thresh=0.12, K=2, retention_ratio=0.34, mag_ratios=str(tmp_path / "wan2_1_mag_ratio.json"))
    assert type(ours).mag_ratios.tolist() == [1.0, 1.0] + ours.norm_ratio and type(ours).forward is mc.magcache_forward


def test_scalar_family_branch_flux_and_hunyuan():
    """BASELINE config 1 plumbing (FLUX, scalar controller with the step-11 veto) and the Hunyuan variant: controller + K1/K2
    kernels around a stand-in block stack, checked call by call against the oracle controller and torch arithmetic."""
    import types as _t
    from magcache_b200 import PRESETS, magcache_branch
    from oracle.controller_ref import ControllerRef
    for preset, fam, attr in [("flux-E024K5R01", "flux", "previous_residual"), ("hunyuan-720p-E024K6R02", "hunyuan", "residual_cache")]:
        cfg = PRESETS[preset]
        ratios = cfg.resolved_ratios()
        cls = type("Fake", (), {})
        m = cls()
        cls.cnt, cls.num_steps, cls.magcache_thresh, cls.K, cls.retention_ratio = 0, cfg.num_steps, cfg.thresh, cfg.K, cfg.retention_ratio
        cls.accumulated_ratio, cls.accumulated_err, cls.accumulated_steps, cls.mag_ratios = 1, 0, 0, ratios
        setattr(cls, attr, None)
        ref_ctl = ControllerRef(fam, ratios, cfg.num_steps, cfg.thresh, cfg.K, cfg.retention_ratio)
        g = torch.Generator(device=DEV).manual_seed(0)
        cache_ref = None
        for i in range(cfg.num_steps + 3):
            h = torch.randn(1, 4096, 3072 if fam == "flux" else 256, device=DEV, generator=g).bfloat16()
            blocks = lambda z: (z.float() * 1.01 + 0.003 * (i + 1)).bfloat16()  # noqa: E731
            out = magcache_branch(m, h, blocks, fam, attr)
            skip = ref_ctl.step()
            if skip:
                exp = h + cache_ref
            else:
                exp = blocks(h)
                cache_ref = exp - h
            assert torch.equal(out, exp), (preset, i)
            assert torch.equal(getattr(m, attr), cache_ref)
            assert m.cnt == ref_ctl.cnt


def test_branch_other_adapters_follow_their_preset_schedule():
    """FramePack (ratio veto, cnt >= 1, scalar cache), Qwen-Image and Wan2.2 T2V-A14B (per-CFG-branch cache list, expert
    window read from `split_step`): the branch taken on every call is the one `MagCacheConfig.schedule()` predicts — itself
    pinned to the reference's statements by tests/test_paper_eval_adapters.py and tests/test_extra_adapters.py — and the K1/K2
    arithmetic equals torch's."""
    from magcache_b200 import PRESETS, magcache_branch
    for preset, attr in [("framepack-E010K3R02", "previous_residual"), ("qwen-image-E006K2R02", "residual_cache"),
                         ("wan2.2-t2v-a14b-E006K2R04", "residual_cache")]:
        cfg = PRESETS[preset]
        per_branch = cfg.branches == 2
        n_calls = cfg.num_steps + 5
        want = cfg.schedule(n_calls)
        cls = type("Fake", (), {})
        m = cls()
        cls.cnt, cls.num_steps, cls.magcache_thresh, cls.K, cls.retention_ratio = 0, cfg.num_steps, cfg.thresh, cfg.K, cfg.retention_ratio
        cls.mag_ratios = cfg.resolved_ratios()
        if per_branch:
            cls.accumulated_ratio, cls.accumulated_err, cls.accumulated_steps = [1.0, 1.0], [0.0, 0.0], [0, 0]
            setattr(cls, attr, [None, None])
            cls.split_step = None if cfg.high_noise_steps is None else 2 * cfg.high_noise_steps
        else:
            cls.accumulated_ratio, cls.accumulated_err, cls.accumulated_steps = 1.0, 0, 0
            setattr(cls, attr, None)
        g = torch.Generator(device=DEV).manual_seed(1)
        cache_ref = [None, None]
        ran = []
        for i in range(n_calls):
            slot = (m.cnt % 2) if per_branch else 0
            h = torch.randn(1, 1024, 384, device=DEV, generator=g).bfloat16()

            def blocks(z, i=i):
                ran.append(i)
                return (z.float() * 0.99 - 0.002 * (i + 1)).bfloat16()

            before = len(ran)
            out = magcache_branch(m, h, blocks, cfg.family, attr)
            skipped = len(ran) == before
            assert skipped == bool(want[i]), (preset, i)
            if skipped:
                exp = h + cache_ref[slot]
            else:
                exp = (h.float() * 0.99 - 0.002 * (i + 1)).bfloat16()
                cache_ref[slot] = exp - h
            assert torch.equal(out, exp), (preset, i)
            cur = getattr(m, attr)[slot] if per_branch else getattr(m, attr)
            assert torch.equal(cur, cache_ref[slot])
        assert int(m.cnt) == n_calls % cfg.num_steps


def test_wan14b_shaped_blocks_vs_oracle():
    """BASELINE configs[4] shapes (dim 5120, 40 heads, ffn 13824) at reduced depth / token count: exercises the wide-row
    LayerNorm / RMSNorm paths (cols > 2048), 40-head attention and the N = 13824 GEMM tiling against the oracle."""
    from oracle import wan_ref
    model = wan_ref.WanModel(dim=5120, ffn_dim=13824, num_heads=40, num_layers=1, text_dim=256, text_len=32).init_synthetic(1)
    lat, ctx, _ = make_inputs(4, grid=(2, 8, 12), text_dim=256, L=19)
    n_tok = lat.shape[1] * (lat.shape[2] // 2) * (lat.shape[3] // 2)
    t = torch.tensor([333.0])
    ref_model = install_ref(wan_ref, copy.deepcopy(model), 10)
    with torch.no_grad():
        ref = ref_model([lat], t=t, context=[ctx], seq_len=n_tok)[0]
    ours_model = install_ours(copy.deepcopy(model).to(DEV), 10)
    out = ours_model([lat.to(DEV)], t=t.to(DEV), context=[ctx.to(DEV)], seq_len=n_tok)[0].cpu()
    e = rel_l2(out, ref)
    print("14B-shaped rel-L2 vs oracle", e)
    assert e <= 2e-2


def test_ti2v_per_token_timesteps_vs_oracle_and_fp64():
    """Wan2.2 TI2V-5B's forward (MagCache4Wan2.2/magcache_generate.py:209-336) at test size on the kernels: 48 latent channels in and out
    (three 16-channel head launches per row range), `t` [1, seq_len] with the first-frame tokens at t = 0 (row ranges [0, 384) and
    [384, 1152) — neither a multiple of the 128-row tiles' grid), seq_len > token count, `split_step` None. miss, miss, then hits on
    both CFG slots against the oracle; the first call also against the fp64 evaluation of the same network."""
    from oracle import wan_ref
    import magcache_b200 as mc
    model = wan_ref.WanModel(dim=256, ffn_dim=512, num_heads=2, num_layers=2, in_dim=48, out_dim=48, text_dim=512, text_len=64).init_synthetic(6)
    g = torch.Generator().manual_seed(9)
    grid = (3, 16, 24)
    lat = torch.randn(48, 3, 32, 48, generator=g)
    ctx, ctx_null = torch.randn(37, 512, generator=g), torch.randn(30, 512, generator=g)
    n_tok = grid[0] * grid[1] * grid[2]
    seq_len = n_tok + 24
    ratios = mc.tables()["wan2.2_ti2v_5b_a"][2:].tolist()

    def timesteps(v):
        t = torch.full((1, seq_len), float(v))
        t[0, :grid[1] * grid[2]] = 0.0
        return t

    RefCls, Ref64, OurCls = (type(n, (wan_ref.WanModel,), {}) for n in ("RefTI2V", "Ref64TI2V", "OurTI2V"))
    ref, m64, our = copy.deepcopy(model), copy.deepcopy(model).double(), copy.deepcopy(model).to(DEV)
    ref.__class__, m64.__class__, our.__class__ = RefCls, Ref64, OurCls
    kw = dict(thresh=10.0, K=3, retention_ratio=0.25)  # 4 steps = 8 calls: miss, miss, then hits
    wan_ref.install_magcache_wan22(RefCls, ratios, 4, **kw)
    wan_ref.install_magcache_wan22(Ref64, ratios, 4, **kw)
    mc.init_magcache_wan22(our, ratios, 4, **kw)
    kinds = []
    with torch.no_grad():
        for call in range(6):
            t = timesteps(900.0 - 100.0 * (call // 2))
            c = ctx if call % 2 == 0 else ctx_null
            a = ref([lat], t=t, context=[c], seq_len=seq_len)[0]
            b = our([lat.to(DEV)], t=t.to(DEV), context=[c.to(DEV)], seq_len=seq_len)[0].cpu()
            kinds.append(int(ref.last_skip))
            assert b.shape == a.shape == (48, 3, 32, 48) and b.dtype == torch.float32
            e_vs = rel_l2(b, a)
            print(f"[ti2v call {call} {'hit' if kinds[-1] else 'miss'}] rel-L2 ours vs oracle {e_vs:.3e}")
            assert e_vs <= 2e-2
            assert rel_l2(OurCls.residual_cache[call % 2].cpu()[0], RefCls.residual_cache[call % 2][0, :n_tok]) <= 3e-2
            if call == 0:
                with wan_ref.exact_fp64():
                    exact = m64([lat.double()], t=t.double(), context=[c.double()], seq_len=seq_len)[0]
                e_ours, e_ref = rel_l2(b, exact), rel_l2(a, exact)
                print(f"[ti2v] rel-L2: ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e}")
                assert e_ours <= 1.5 * e_ref + 1e-4
                eng = our._mc_engine
                assert eng.t_values == 2 and eng.runs == [(0, 384, 0), (384, n_tok, 1)] and len(eng.head_groups) == 3
    assert kinds == [0, 0, 1, 1, 1, 1]
