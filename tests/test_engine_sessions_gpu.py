"""Sessions on the H100 kernels: the sessions of tests/test_engine_sessions_cpu.py with the reduced-size models on cuda, every step of
every later generation bit-equal to a fresh model's (tests/session_harness.py). The cached inputs live on the device here, so the
"recycled" delivery goes through PyTorch's caching allocator, which hands a freed block to the next tensor of its size."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import magcache_b200 as mc  # noqa: E402
import test_engine_sessions_cpu as C  # noqa: E402  (the models, inputs and calls of the emulated sessions)
from oracle import wan_ref  # noqa: E402
from session_harness import MODES, Session, deliver, record_hits  # noqa: E402, F401  (record_hits: fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("record_hits")]
DEV = "cuda"


def _dev(inp):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in inp.items()}


def _on_dev(fresh):
    return lambda: fresh().to(DEV)


# ---------------------------------------------------------------------------------------------------------------------- FLUX / Kontext
def _flux_session(install=None):
    install = install or (lambda m: mc.init_magcache_flux(m, C.FLUX_STEPS, **C.FLUX_KW))
    return Session(_on_dev(C._patched(C._flux_base(), install)), lambda m: m.previous_residual, C.FLUX_STATE)


@pytest.mark.parametrize("mode", MODES)
def test_flux_transposed_aspect_ratio(mode):
    s = _flux_session()
    inp = _dev(C._flux_inputs((8, 6)))
    C._has_hits_and_misses(s.run(C._flux_calls(), inp))
    for hw in ((6, 8), (8, 6)):
        deliver(inp, "img_ids", C.fr.make_ids(hw[0], hw[1], 19)[0].to(DEV), mode)
        s.run(C._flux_calls(), inp)


def test_flux_text_length_guidance_and_controlnet():
    s = _flux_session()
    s.run(C._flux_calls(), _dev(C._flux_inputs(n_txt=19)))
    s.run(C._flux_calls(), _dev(C._flux_inputs(n_txt=24, seed=1)))
    inp = _dev(C._flux_inputs(n_txt=19))
    inp["guidance"].fill_(5.0)
    s.run(C._flux_calls(), inp)
    g = torch.Generator(device=DEV).manual_seed(7)
    samples = tuple([(0.1 * torch.randn(1, 48, C.D_FLUX, device=DEV, generator=g)).bfloat16() for _ in range(2)] for _ in range(2))
    for cn in (samples, None, samples):
        inp["cn"] = cn
        s.run(C._flux_calls(), inp)


def test_flux_calibration_then_inference_then_other_step_count(capsys):
    s = _flux_session(install=lambda m: mc.init_magcache_flux_calibration(m, C.FLUX_STEPS))
    inp = _dev(C._flux_inputs())
    s.run(C._flux_calls(), inp)
    s.run(C._flux_calls(), inp, before=lambda m: mc.init_magcache_flux(m, C.FLUX_STEPS, **C.FLUX_KW))
    C._has_hits_and_misses(s.run(C._flux_calls(12), inp, before=lambda m: mc.init_magcache_flux(m, 12, **C.FLUX_KW)))
    capsys.readouterr()


@pytest.mark.parametrize("mode", MODES)
def test_kontext_reference_image_of_transposed_aspect_ratio(mode):
    s = _flux_session(install=lambda m: mc.init_magcache_flux(m, C.FLUX_STEPS, thresh=0.05, K=4, retention_ratio=0.2, table="flux_kontext"))
    inp = C._flux_inputs()
    inp["hs"], inp["img_ids"] = torch.randn(1, 96, 64, generator=torch.Generator().manual_seed(3)).bfloat16(), C._kontext_ids((4, 12))
    inp = _dev(inp)
    s.run(C._flux_calls(), inp)
    for ref_hw in ((12, 4), (4, 12)):
        deliver(inp, "img_ids", C._kontext_ids(ref_hw).to(DEV), mode)
        s.run(C._flux_calls(), inp)


# ---------------------------------------------------------------------------------------------------------------------- HunyuanVideo
def _hy_session(fp8):
    s = C._hy_session(fp8)
    return Session(_on_dev(s.fresh), s.residual, s.state)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("mode", MODES)
def test_hunyuan_valid_text_tokens(fp8, mode):
    s = _hy_session(fp8)
    inp = _dev(C._hy_inputs(valid=11))
    C._has_hits_and_misses(s.run(C._hy_calls, inp))
    for valid in (7, 11):
        deliver(inp, "mask", C._mask(valid).to(DEV), mode)
        s.run(C._hy_calls, inp)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("mode", MODES)
def test_hunyuan_transposed_resolution(fp8, mode):
    s = _hy_session(fp8)
    inp = _dev(C._hy_inputs((2, 4, 6)))
    s.run(C._hy_calls, inp)
    for grid in ((2, 6, 4), (2, 4, 6)):
        new = _dev(C._hy_inputs(grid))
        inp["x"] = new["x"]
        deliver(inp, "cos", new["cos"], mode)
        deliver(inp, "sin", new["sin"], mode)
        s.run(C._hy_calls, inp)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_hunyuan_frame_count(fp8):
    s = _hy_session(fp8)
    for grid in ((2, 4, 6), (3, 4, 6), (2, 4, 6)):
        s.run(C._hy_calls, _dev(C._hy_inputs(grid)))


# ---------------------------------------------------------------------------------------------------------------------- Wan
def _wan_session(install, native=False, graphs=False, **over):
    kw = dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128, text_len=32)
    kw.update(over)
    base = wan_ref.WanModel(**kw).init_synthetic(6)

    def fresh():
        m = C._patched(base, install)().to(DEV)
        eng = mc.WanEngine(mc.WanWeights.from_module(m, torch.device(DEV)), native=native)
        eng.use_graphs = graphs
        object.__setattr__(m, "_mc_engine", eng)
        return m
    return Session(fresh, lambda m: m.residual_cache[(int(m.cnt) - 1) % 2], C.WAN_STATE)


@pytest.mark.parametrize("native,graphs", [(False, False), (False, True), (True, False)], ids=["python", "graphs", "native"])
def test_wan_two_resolutions(native, graphs):
    """A new workspace (and on the native engine a new `mc_dit_bind`) per token count; 8x12 and 12x8 share one."""
    s = _wan_session(lambda m: mc.init_magcache(m, 5, mag_ratios=mc.tables()["wan2.1_t2v_1.3b"], thresh=0.12, K=2, retention_ratio=0.2),
                     native=native, graphs=graphs)
    g = torch.Generator().manual_seed(2)
    for hw in ((8, 12), (12, 8), (8, 8), (8, 12)):
        recs = s.run(C._wan_calls(torch.randn(16, 2, *hw, generator=g).to(DEV), 5), None)
    C._has_hits_and_misses(recs)
    if native:
        assert s.model._mc_engine._nat is not None, "the native engine must really have gone through mc_dit_forward"


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_ti2v_timestep_ranges(graphs):
    """Per-token timesteps with other row ranges each generation: a captured forward bakes the ranges in and must be dropped."""
    s = _wan_session(lambda m: mc.init_magcache_wan22(m, mc.tables()["wan2.2_ti2v_5b_a"][2:].tolist(), 5, thresh=0.12, K=2,
                                                      retention_ratio=0.2), graphs=graphs, in_dim=48, out_dim=48)
    lat = torch.randn(48, 3, 8, 8, generator=torch.Generator().manual_seed(4)).to(DEV)

    def ranges(clean):
        def t_of(t, n):
            tt = torch.full((1, n), t)
            tt[0, :clean] = 0.0
            return tt
        return t_of
    for clean in (16, 32, 0, 16):
        s.run(C._wan_calls(lat, 5, ranges(clean)), None)


# ---------------------------------------------------------------------------------------------------------------------- Open-Sora
def test_opensora_resolution_frames_caption_fps():
    s = C._os_session()
    s = Session(_on_dev(s.fresh), s.residual, s.state)
    C._has_hits_and_misses(s.run(C._os_calls(dev=DEV), None))
    for kw in (dict(H=10, W=6), dict(T=4), dict(y_len=7), dict(fps=12.0), {}):
        s.run(C._os_calls(dev=DEV, **kw), None)


# ---------------------------------------------------------------------------------------------------------------------- inference mode
@pytest.mark.parametrize("mode", MODES)
def test_flux_and_hunyuan_under_inference_mode(mode):
    """Inference tensors have no version counter; an in-place write to one inside inference mode must still reach the tables."""
    with torch.inference_mode():
        s = _flux_session()
        inp = _dev(C._flux_inputs((8, 6)))
        assert inp["img_ids"].is_inference()
        s.run(C._flux_calls(), inp)
        deliver(inp, "img_ids", C.fr.make_ids(6, 8, 19)[0].to(DEV), mode)
        s.run(C._flux_calls(), inp)
        s = _hy_session(False)
        inp = _dev(C._hy_inputs((2, 4, 6), valid=11))
        s.run(C._hy_calls, inp)
        deliver(inp, "mask", C._mask(7).to(DEV), mode)
        s.run(C._hy_calls, inp)
        new = _dev(C._hy_inputs((2, 6, 4), valid=7))
        inp["x"] = new["x"]
        deliver(inp, "cos", new["cos"], mode)
        deliver(inp, "sin", new["sin"], mode)
        s.run(C._hy_calls, inp)


# ---------------------------------------------------------------------------------------------------------------------- Wan2.2, TeaCache
def test_wan22_expert_switch_across_sessions():
    s = C._wan22_session(high=5)
    fresh = s.fresh

    def fresh_dev():
        pair = fresh()
        for m in pair.models:
            m.to(DEV)
            object.__setattr__(m, "_mc_engine", mc.WanEngine(mc.WanWeights.from_module(m, torch.device(DEV))))
        return pair
    s = Session(fresh_dev, s.residual, s.state)
    g = torch.Generator().manual_seed(5)
    lat = torch.randn(16, 2, 8, 8, generator=g).to(DEV)
    for x in (lat, lat, torch.randn(16, 2, 8, 12, generator=g).to(DEV)):
        C._has_hits_and_misses(s.run(C._wan22_calls(x, 5), None, before=C._reset_experts))


def test_opensora_teacache_across_sessions():
    s = C._tea_session(10.0)
    s = Session(_on_dev(s.fresh), s.residual, s.state)
    for shape in ((2, 4, 6), (2, 4, 6), (2, 6, 10)):
        C._has_hits_and_misses(s.run(C._tea_calls(*shape, dev=DEV), None))
