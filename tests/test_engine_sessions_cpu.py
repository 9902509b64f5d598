"""Sessions on the emulated engines (tests/emu_ops.py, tests/opensora_emu.py): several generations on one patched model, one input
changed between them, every step bit-equal to a fresh model's (tests/session_harness.py). The cached inputs — FLUX / Kontext ids,
the HunyuanVideo text mask and RoPE cos / sin — arrive in place, in a recycled block and as new tensors: an engine that keys its
tables on a tensor's address returns the previous generation's positions or text length in the first two cases."""
import copy
import os

import pytest
import torch

import magcache_b200 as mc
from magcache_b200 import mmdit as mmdit_mod
from magcache_b200 import opensora as os_mod
from magcache_b200 import patch as patch_mod
from magcache_b200 import wan as wan_mod
from oracle import flux_ref as fr
from oracle import hunyuan_ref as hr
from oracle import wan_ref

import emu_ops
import flux_controlnet_ref as cref
import hunyuan_fp8_ref as f8
import opensora_emu
import opensora_ref as R
import opensora_sp_cases as SP
import opensora_tea_ref as TR
from session_harness import MODES, Session, deliver, generation, record_hits  # noqa: F401  (record_hits: fixture)


@pytest.fixture()
def emulated(monkeypatch, record_hits):  # noqa: F811
    monkeypatch.setattr(emu_ops, "dequant_fp8_bf16", f8.emu_dequant_fp8_bf16, raising=False)
    for mod in (mmdit_mod, wan_mod, patch_mod):
        monkeypatch.setattr(mod, "ops", emu_ops)
    monkeypatch.setattr(os_mod, "ops", opensora_emu.namespace())
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def _has_hits_and_misses(recs):
    kinds = [h for r in recs for h in r["hit"]]
    assert True in kinds and False in kinds, kinds


# ---------------------------------------------------------------------------------------------------------------------- FLUX / Kontext
FLUX_STATE = ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps", "norm_ratio", "norm_std", "cos_dis")
FLUX_STEPS = 8
FLUX_KW = dict(thresh=0.24, K=5, retention_ratio=0.2)
D_FLUX = 256


def _flux_base():
    return fr.FluxTransformer2DModel(in_channels=64, num_layers=2, num_single_layers=3, num_attention_heads=2, joint_attention_dim=96,
                                     pooled_projection_dim=48, guidance_embeds=True).init_synthetic(4)


def _patched(base, install):
    def fresh():
        m = copy.deepcopy(base)
        m.__class__ = type("Session" + type(base).__name__, (type(base),), {})
        install(m)
        return m
    return fresh


def _flux_session(install=None):
    install = install or (lambda m: mc.init_magcache_flux(m, FLUX_STEPS, **FLUX_KW))
    return Session(_patched(_flux_base(), install), lambda m: m.previous_residual, FLUX_STATE)


def _flux_inputs(hw=(8, 6), n_txt=19, seed=0):
    g = torch.Generator().manual_seed(seed)
    img_ids, txt_ids = fr.make_ids(hw[0], hw[1], n_txt)
    return {"hs": torch.randn(1, hw[0] * hw[1], 64, generator=g).bfloat16(), "enc": torch.randn(1, n_txt, 96, generator=g).bfloat16(),
            "pooled": torch.randn(1, 48, generator=g).bfloat16(), "img_ids": img_ids, "txt_ids": txt_ids,
            "guidance": torch.tensor([3.5]), "cn": None}


def _flux_calls(steps=FLUX_STEPS):
    def make(inp):
        def call(i):
            def fn(m):
                cn = inp["cn"] or (None, None)
                return m(inp["hs"] * (1.0 - 0.03 * i), inp["enc"], inp["pooled"], torch.tensor([1.0 - i / steps]), inp["img_ids"],
                         inp["txt_ids"], inp["guidance"], controlnet_block_samples=cn[0], controlnet_single_block_samples=cn[1],
                         return_dict=False)[0]
            return fn
        return [call(i) for i in range(steps)]
    return make


@pytest.mark.parametrize("mode", MODES)
def test_flux_transposed_aspect_ratio(emulated, mode):
    """8x6 then 6x8 latent tokens (FLUX 1024x768 then 768x1024 at test size): the same 48 image tokens at other positions."""
    s = _flux_session()
    inp = _flux_inputs((8, 6))
    _has_hits_and_misses(s.run(_flux_calls(), inp))
    for hw in ((6, 8), (8, 6)):
        deliver(inp, "img_ids", fr.make_ids(hw[0], hw[1], 19)[0], mode)
        s.run(_flux_calls(), inp)


@pytest.mark.parametrize("mode", MODES)
def test_flux_transposed_aspect_ratio_under_inference_mode(emulated, mode):
    """Inference tensors (servers run under `torch.inference_mode()`) have no version counter, and an in-place write to one inside
    inference mode leaves no trace on it: the engine compares their content."""
    with torch.inference_mode():
        s = _flux_session()
        inp = _flux_inputs((8, 6))
        assert inp["img_ids"].is_inference()
        s.run(_flux_calls(), inp)
        for hw in ((6, 8), (8, 6)):
            deliver(inp, "img_ids", fr.make_ids(hw[0], hw[1], 19)[0], mode)
            s.run(_flux_calls(), inp)


def test_flux_text_length_and_guidance(emulated):
    s = _flux_session()
    s.run(_flux_calls(), _flux_inputs(n_txt=19))
    s.run(_flux_calls(), _flux_inputs(n_txt=24, seed=1))   # a new workspace for the text rows
    inp = _flux_inputs(n_txt=19)
    s.run(_flux_calls(), inp)
    inp["guidance"].fill_(5.0)
    s.run(_flux_calls(), inp)


def test_flux_controlnet_on_off_on(emulated, monkeypatch):
    monkeypatch.setattr(mmdit_mod, "ops", cref.emu)  # the emulation with the ControlNet GEMM epilogue
    monkeypatch.setattr(patch_mod, "ops", cref.emu)
    s = _flux_session()
    inp = _flux_inputs()
    g = torch.Generator().manual_seed(7)
    samples = ([(0.1 * torch.randn(1, 48, D_FLUX, generator=g)).bfloat16() for _ in range(2)],
               [(0.1 * torch.randn(1, 48, D_FLUX, generator=g)).bfloat16() for _ in range(2)])
    for cn in (samples, None, samples):
        inp["cn"] = cn
        s.run(_flux_calls(), inp)


def test_flux_calibration_then_inference(emulated, capsys):
    s = _flux_session(install=lambda m: mc.init_magcache_flux_calibration(m, FLUX_STEPS))
    inp = _flux_inputs()
    s.run(_flux_calls(), inp)
    s.run(_flux_calls(), inp, before=lambda m: mc.init_magcache_flux(m, FLUX_STEPS, **FLUX_KW))
    capsys.readouterr()


def test_flux_num_inference_steps_between_sessions(emulated):
    s = _flux_session()
    inp = _flux_inputs()
    s.run(_flux_calls(), inp)
    _has_hits_and_misses(s.run(_flux_calls(12), inp, before=lambda m: mc.init_magcache_flux(m, 12, **FLUX_KW)))
    s.run(_flux_calls(), inp, before=lambda m: mc.init_magcache_flux(m, FLUX_STEPS, **FLUX_KW))


def _kontext_ids(ref_hw):
    """Kontext's joint image ids: the 8x6 output latent (first id 0), then the reference image's tokens (first id 1)."""
    out = fr.make_ids(8, 6, 19)[0]
    ref = fr.make_ids(ref_hw[0], ref_hw[1], 0)[0]
    ref[:, 0] = 1
    return torch.cat([out, ref])


@pytest.mark.parametrize("mode", MODES)
def test_kontext_reference_image_of_transposed_aspect_ratio(emulated, mode):
    s = _flux_session(install=lambda m: mc.init_magcache_flux(m, FLUX_STEPS, thresh=0.05, K=4, retention_ratio=0.2, table="flux_kontext"))
    g = torch.Generator().manual_seed(3)
    inp = _flux_inputs()
    inp["hs"], inp["img_ids"] = torch.randn(1, 96, 64, generator=g).bfloat16(), _kontext_ids((4, 12))
    s.run(_flux_calls(), inp)
    for ref_hw in ((12, 4), (4, 12)):
        deliver(inp, "img_ids", _kontext_ids(ref_hw), mode)
        s.run(_flux_calls(), inp)


# ---------------------------------------------------------------------------------------------------------------------- HunyuanVideo
HY_STATE = ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps")
HY_STEPS = 10


def _hy_session(fp8):
    base = hr.HYVideoDiffusionTransformer(hidden_size=256, heads_num=2, mm_double_blocks_depth=2, mm_single_blocks_depth=3, text_states_dim=96,
                                          text_states_dim_2=48, guidance_embed=True).init_synthetic(5)
    if fp8:
        base = f8.to_fp8_checkpoint(base)
    install = lambda m: mc.init_magcache_hunyuan(m, HY_STEPS, thresh=0.24, K=6, retention_ratio=0.2)  # noqa: E731
    return Session(_patched(base, install), lambda m: m.residual_cache, HY_STATE)


def _hy_inputs(grid=(2, 4, 6), valid=11, seed=0):
    g = torch.Generator().manual_seed(seed)
    mask = torch.zeros(1, 16, dtype=torch.long)
    mask[0, :valid] = 1
    cos, sin = hr.rope_cos_sin(grid)
    return {"x": torch.randn(1, 16, grid[0], 2 * grid[1], 2 * grid[2], generator=g).bfloat16(),
            "txt": torch.randn(1, 16, 96, generator=g).bfloat16(), "mask": mask, "pooled": torch.randn(1, 48, generator=g).bfloat16(),
            "cos": cos, "sin": sin}


def _hy_calls(inp):
    def call(i):
        return lambda m: m(inp["x"] * (1.0 - 0.03 * i), torch.tensor([1000.0 - 90.0 * i]), inp["txt"], inp["mask"], inp["pooled"],
                           inp["cos"], inp["sin"], torch.tensor([6000.0]), return_dict=False)
    return [call(i) for i in range(HY_STEPS)]


def _mask(valid):
    m = torch.zeros(1, 16, dtype=torch.long)
    m[0, :valid] = 1
    return m


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("mode", MODES)
def test_hunyuan_valid_text_tokens(emulated, fp8, mode):
    """The mask is [1, 16] every time; 11, then 7, then 11 valid tokens."""
    s = _hy_session(fp8)
    inp = _hy_inputs(valid=11)
    _has_hits_and_misses(s.run(_hy_calls, inp))
    for valid in (7, 11):
        deliver(inp, "mask", _mask(valid), mode)
        s.run(_hy_calls, inp)


@pytest.mark.parametrize("mode", MODES)
def test_hunyuan_text_tokens_and_resolution_under_inference_mode(emulated, mode):
    with torch.inference_mode():
        s = _hy_session(False)
        inp = _hy_inputs((2, 4, 6), valid=11)
        assert inp["mask"].is_inference() and inp["cos"].is_inference()
        s.run(_hy_calls, inp)
        deliver(inp, "mask", _mask(7), mode)
        s.run(_hy_calls, inp)
        new = _hy_inputs((2, 6, 4), valid=7)
        inp["x"] = new["x"]
        deliver(inp, "cos", new["cos"], mode)
        deliver(inp, "sin", new["sin"], mode)
        s.run(_hy_calls, inp)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("mode", MODES)
def test_hunyuan_transposed_resolution(emulated, fp8, mode):
    """A 4x6 then a 6x4 token grid (720x1280 then 1280x720 at test size): the RoPE cos / sin keep their shape, not their values."""
    s = _hy_session(fp8)
    inp = _hy_inputs((2, 4, 6))
    s.run(_hy_calls, inp)
    for grid in ((2, 6, 4), (2, 4, 6)):
        new = _hy_inputs(grid)
        inp["x"] = new["x"]
        deliver(inp, "cos", new["cos"], mode)
        deliver(inp, "sin", new["sin"], mode)
        s.run(_hy_calls, inp)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_hunyuan_frame_count(emulated, fp8):
    s = _hy_session(fp8)
    for grid in ((2, 4, 6), (3, 4, 6), (2, 4, 6)):
        s.run(_hy_calls, _hy_inputs(grid))


def test_hunyuan_rope_dropped_then_restored(emulated):
    """A call without cos / sin drops the table; the next call with the same cos / sin tensors must build it again."""
    s = _hy_session(False)
    inp = _hy_inputs()
    s.run(_hy_calls, inp)
    cos, sin = inp["cos"], inp["sin"]
    inp["cos"] = inp["sin"] = None
    s.run(_hy_calls, inp)
    inp["cos"], inp["sin"] = cos, sin
    s.run(_hy_calls, inp)


def test_write_torch_does_not_see_needs_invalidate_engine(emulated):
    """A write through `.data` does not bump `_version`, so the engine keeps the table it built: INTEGRATION.md documents that
    such writes need `invalidate_engine`, after which the session is bit-equal to a fresh model again."""
    s = _flux_session()
    inp = _flux_inputs((8, 6))
    first = s.run(_flux_calls(), inp)
    inp["img_ids"].data.copy_(fr.make_ids(6, 8, 19)[0])
    stale = generation(s.model, _flux_calls()(inp), s.residual, s.state)
    assert torch.equal(stale[0]["out"], first[0]["out"])  # the 8x6 positions, not the 6x8 ones the ids now hold
    mc.invalidate_engine(s.model)
    s.run(_flux_calls(), inp)


# ---------------------------------------------------------------------------------------------------------------------- Wan
WAN_STATE = ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps")


def _wan_session(install, **over):
    kw = dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128, text_len=32)
    kw.update(over)
    base = wan_ref.WanModel(**kw).init_synthetic(6)

    def inst(m):
        install(m)
        object.__setattr__(m, "_mc_engine", mc.WanEngine(mc.WanWeights.from_module(m, torch.device("cpu"))))
    # the residual slot this call wrote (the other CFG branch's slot still holds the previous generation's until its first call)
    return Session(_patched(base, inst), lambda m: m.residual_cache[(int(m.cnt) - 1) % 2], WAN_STATE)


def _wan_calls(lat, steps, t_of=lambda t, n: torch.tensor([t])):
    g = torch.Generator().manual_seed(9)
    ctxs = [torch.randn(9, 128, generator=g), torch.randn(7, 128, generator=g)]
    n_tok = lat.shape[1] * (lat.shape[2] // 2) * (lat.shape[3] // 2)

    def make(_):
        def call(c):
            return lambda m: m([lat * (1.0 - 0.03 * (c // 2))], t=t_of(950.0 - 90.0 * (c // 2), n_tok), context=[ctxs[c % 2]],
                               seq_len=n_tok)[0]
        return [call(c) for c in range(2 * steps)]
    return make


def test_wan_two_resolutions(emulated):
    """8x12 -> 12x8 (same tokens, other grid) -> 8x8 (a new workspace) -> 8x12 latents on one Wan2.1 engine."""
    s = _wan_session(lambda m: mc.init_magcache(m, 5, mag_ratios=mc.tables()["wan2.1_t2v_1.3b"], thresh=0.12, K=2, retention_ratio=0.2))
    g = torch.Generator().manual_seed(2)
    for hw in ((8, 12), (12, 8), (8, 8), (8, 12)):
        recs = s.run(_wan_calls(torch.randn(16, 2, *hw, generator=g), 5), None)
    _has_hits_and_misses(recs)


def test_ti2v_timestep_ranges(emulated):
    """TI2V-5B with per-token timesteps: first frame clean, then the first two frames, then a uniform t — each generation with its
    own row ranges (which key the engine's captured graphs)."""
    s = _wan_session(lambda m: mc.init_magcache_wan22(m, mc.tables()["wan2.2_ti2v_5b_a"][2:].tolist(), 5, thresh=0.12, K=2,
                                                      retention_ratio=0.2), in_dim=48, out_dim=48)
    lat = torch.randn(48, 3, 8, 8, generator=torch.Generator().manual_seed(4))

    def ranges(clean):
        def t_of(t, n):
            tt = torch.full((1, n), t)
            tt[0, :clean] = 0.0
            return tt
        return t_of
    for clean in (16, 32, 0, 16):
        s.run(_wan_calls(lat, 5, ranges(clean)), None)
        assert s.model._mc_engine.runs == ([(0, clean, 0), (clean, 48, 1)] if clean else None)


# ---------------------------------------------------------------------------------------------------------------------- Open-Sora
OS_STEPS = 30  # the evaluation forward's generation length (eval/magcache/experiments/opensora.py:349-354)
OS_STATE = ("t", "accumulated_sim", "accumulated_err", "accumulated_steps", "skip_steps")


def _os_session():
    base = R.STDiT3(**R.CONFIGS["tiny"]).init_synthetic(0).to(torch.bfloat16)
    return Session(_patched(base, lambda m: patch_mod.init_magcache_opensora(m, thresh=0.5, K=3, skip_time=2)),
                   lambda m: m.residual_cache, OS_STATE)


def _os_calls(T=3, H=6, W=10, y_len=12, fps=24.0, dev="cpu"):
    g = torch.Generator().manual_seed(T * 100 + H * 10 + W)
    x, y = torch.randn(1, 4, T, H, W, generator=g).to(dev), torch.randn(1, 1, 12, 64, generator=g).to(dev)
    mask = torch.zeros(1, 12, dtype=torch.long)
    mask[0, :y_len] = 1
    mask = mask.to(dev)
    kw = dict(mask=mask, fps=torch.tensor([fps]), height=torch.tensor([8.0 * H]), width=torch.tensor([8.0 * W]))

    def make(_):
        return [lambda m, i=i: m(x, torch.tensor([1000.0 - 33.0 * i]), None, y, **kw) for i in range(OS_STEPS)]
    return make


def test_opensora_resolution_frames_caption_fps(emulated):
    s = _os_session()
    _has_hits_and_misses(s.run(_os_calls(), None))
    for kw in (dict(H=10, W=6), dict(T=4), dict(y_len=7), dict(fps=12.0), {}):
        s.run(_os_calls(**kw), None)


class _Experts:
    """The Wan2.2 A14B pair as one session model: two instances of one class that share the counter, the accumulators and the
    residual-cache list (class attributes), one engine each. The decisions of both land in one list."""

    def __init__(self, models):
        self.models, self._session_hits = models, []
        for m in models:
            m.__dict__["_session_hits"] = self._session_hits

    def __getattr__(self, name):
        return getattr(self.models[0], name)


def _wan22_session(high):
    kw = dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128, text_len=32)
    protos = [wan_ref.WanModel(**kw).init_synthetic(seed) for seed in (1, 2)]
    ratios = mc.tables()["wan2.2_t2v_a14b"][2:].tolist()

    def fresh():
        cls = type("SessionW22", (wan_ref.WanModel,), {})
        models = []
        for p in protos:
            m = copy.deepcopy(p)
            m.__class__ = cls
            object.__setattr__(m, "_mc_engine", mc.WanEngine(mc.WanWeights.from_module(m, torch.device("cpu"))))
            models.append(m)
        mc.init_magcache_wan22(models[0], ratios, 12, thresh=0.12, K=2, retention_ratio=0.2, split_steps=high)
        return _Experts(models)
    return Session(fresh, lambda m: m.residual_cache[(int(m.cnt) - 1) % 2], WAN_STATE)


def _wan22_calls(lat, high, steps=12):
    g = torch.Generator().manual_seed(9)
    ctxs = [torch.randn(9, 128, generator=g), torch.randn(7, 128, generator=g)]
    n_tok = lat.shape[1] * (lat.shape[2] // 2) * (lat.shape[3] // 2)

    def make(_):
        def call(c):
            e = 0 if c < 2 * high else 1  # the high-noise expert first, then the low-noise one
            return lambda p: p.models[e]([lat * (1.0 - 0.03 * (c // 2))], t=torch.tensor([950.0 - 90.0 * (c // 2)]),
                                         context=[ctxs[c % 2]], seq_len=n_tok)[0]
        return [call(c) for c in range(2 * steps)]
    return make


def _reset_experts(pair):
    for m in pair.models:
        mc.reset_magcache(m)


def test_wan22_expert_switch_across_sessions(emulated):
    """Two generations through the expert switch, then one at another resolution, with `reset_magcache` on both experts between
    them: the low-noise expert's engine takes over the residual slots of the high-noise one's, every step bit-equal to a fresh
    pair. (Without the reset a later generation is not a fresh one in the reference either: at the wrap the low-noise expert
    rebinds fresh accumulators on itself, magcache_generate.py:330-334, and the high-noise one keeps the class-level lists.)"""
    s = _wan22_session(high=5)  # int(split_step * R) = 2: both cache slots are filled before the first eligible call
    g = torch.Generator().manual_seed(5)
    lat = torch.randn(16, 2, 8, 8, generator=g)
    for x in (lat, lat, torch.randn(16, 2, 8, 12, generator=g)):
        recs = s.run(_wan22_calls(x, 5), None, before=_reset_experts)
        _has_hits_and_misses(recs)
        # one counter for both experts, also after a reset
        cls = type(s.model.models[0])
        assert torch.is_tensor(cls.cnt) and not any("cnt" in m.__dict__ for m in s.model.models)


# ---------------------------------------------------------------------------------------------------------------------- Open-Sora TeaCache
def _tea_session(thresh):
    base = R.STDiT3(**R.CONFIGS["tiny"]).init_synthetic(0)
    with torch.no_grad():
        for n, p in base.named_parameters():
            if n.startswith("t_block."):
                p.mul_(0.05)  # keeps the modulated input's step-to-step change in TeaCache's working range
    base = base.to(torch.bfloat16)
    return Session(_patched(base, lambda m: mc.init_teacache_opensora(m, rel_l1_thresh=thresh)), lambda m: m.previous_residual,
                   ("accumulated_rel_l1_distance", "previous_modulated_input"))


def _tea_calls(T, H, W, dev="cpu", n=6):
    g = torch.Generator().manual_seed(T * 100 + H * 10 + W)
    x, d = torch.randn(1, 4, T, H, W, generator=g).to(dev), torch.randn(1, 4, T, H, W, generator=g).to(dev)
    y = torch.randn(1, 1, 12, 64, generator=g).to(dev)
    kw = dict(mask=torch.ones(1, 12, dtype=torch.long, device=dev), fps=torch.tensor([24.0], device=dev),
              height=torch.tensor([8.0 * H], device=dev), width=torch.tensor([8.0 * W], device=dev))
    ts = [torch.tensor([1000.0 - 30.0 * i], device=dev) for i in range(n)]
    all_ts = [int(t[0].to(torch.bfloat16).item()) for t in ts]  # the first and the last call are forced

    def make(_):
        return [lambda m, i=i: m(x + 0.004 * i * d, ts[i], all_ts, y, **kw) for i in range(n)]
    return make


def test_opensora_teacache_across_sessions(emulated, monkeypatch):
    """Two generations at one resolution, then one at another: `previous_modulated_input` still holds the previous generation's
    (`mi_prev`), which the first, forced call of a generation never reads."""
    monkeypatch.setattr(os_mod, "ops", TR.namespace())
    s = _tea_session(10.0)
    for shape in ((2, 4, 6), (2, 4, 6), (2, 6, 10)):
        recs = s.run(_tea_calls(*shape), None)
        _has_hits_and_misses(recs)


def _sp_worker(rank, world, initfile):
    import torch.distributed as dist
    from test_opensora_sp_cpu import namespace
    dist.init_process_group("gloo", init_method=f"file://{initfile}", rank=rank, world_size=world)
    torch.set_num_threads(max(1, (os.cpu_count() or 1) // world))
    try:
        os_mod.ops = namespace()
        torch.Tensor.is_cuda = property(lambda self: True)

        def fresh():
            m = SP.build("teacache", thresh=10.0)[0]
            SP.enable(m, rank, world)
            return m
        model = fresh()
        # the crops 12x14 -> 14x12 -> 11x13 (the first one's padded 6x7 patch grid under another crop) -> 12x14
        for T, Hx, Wx in ((7, 12, 14), (7, 14, 12), (7, 11, 13), (7, 12, 14)):
            got = SP.calls(model, "teacache", 6, 2, T, Hx, Wx, "cpu")
            want = SP.calls(fresh(), "teacache", 6, 2, T, Hx, Wx, "cpu")
            assert len(got) == len(want)
            for i, ((o, a, r), (o1, a1, r1)) in enumerate(zip(got, want)):
                assert torch.equal(o, o1) and a == a1, (rank, (T, Hx, Wx), i)
                assert (r is None) == (r1 is None) and (r is None or torch.equal(r, r1)), (rank, (T, Hx, Wx), i)
            assert any(a["accumulated_rel_l1_distance"] > 0 for _, a, _ in got)  # hits
    finally:
        dist.destroy_process_group()


def test_opensora_sequence_parallel_crops_across_sessions():
    """Open-Sora under VideoSys's sequence parallelism (two gloo ranks): TeaCache generations at several crops on one sharded
    model, each bit-equal on every rank to a fresh sharded model's."""
    import tempfile

    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_sp_worker, args=(2, os.path.join(d, "init")), nprocs=2, join=True)
