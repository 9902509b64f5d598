"""`FlowDPMSolverSampler` (DPM-Solver++ 2M on the flow parameterisation, magcache_b200/sampler.py) on CPU: the host's float64
scalars against the tensor-form restatement in tests/dpm_solver_ref.py, the first-order step against Euler, the convergence order
on an ODE with a closed-form solution, the recycled x0-prediction buffers, and the caller loop over the Wan engine with emulated
kernels (tests/emu_ops.py): Wan2.1 t2v and a Wan2.2 A14B expert pair, the fused step (`denoise`: the update in the unconditional
call's head, `mc_head_unpatchify_step_hist`) bit-equal to the two calls + `mc_cfg_step`, the hit / miss sequence the controller's,
the latents held to the oracle. The emulation checks the plumbing; tests/test_dpm_solver_gpu.py checks the kernel."""
import copy
import math

import pytest
import torch

import magcache_b200 as mc
from magcache_b200 import _lib as L
from magcache_b200 import patch as patch_mod
from magcache_b200 import sampler as S
from magcache_b200 import wan as wan_mod
from oracle import sampler_ref, wan_ref

import dpm_solver_ref as R
import emu_ops

_EMU_HEAD = emu_ops.head_unpatchify


def cfg_step_any(cond, uncond, guide_scale, x, coef_v, coef_x=1.0, hist=(), coef_h=(), sigma=0.0, out=None, x0_out=None):
    """mc_cfg_step's chain in the dtype of x (float64 here: the host arithmetic without the kernel's fp32 rounding)."""
    f = lambda a: torch.tensor(a, dtype=x.dtype)  # noqa: E731
    v = uncond + f(guide_scale) * (cond - uncond)
    acc = f(coef_x) * x + f(coef_v) * v
    for h, c in zip(hist, coef_h):
        acc = acc + f(c) * h
    if x0_out is not None:
        x0_out.copy_(x - f(sigma) * v)
    if out is None:
        return acc
    out.copy_(acc)
    return out


def model_v(x, sigma, branch):
    """A smooth, non-linear stand-in for the two DiT forwards (flow prediction), as in test_sampler_cpu.py."""
    c = 0.7 if branch == 0 else -0.2
    return torch.tanh(1.3 * x + c) * (0.5 + float(sigma)) - 0.8 * x * float(sigma)


@pytest.fixture()
def f64_kernel(monkeypatch):
    monkeypatch.setattr(S.ops, "cfg_step", cfg_step_any)


# ------------------------------------------------------------------------------------------- host arithmetic
@pytest.mark.parametrize("order", [1, 2])
def test_first_order_steps_are_euler(f64_kernel, order):
    """alpha_t (e^-h - 1) = sigma_t / sigma_s - 1, so every first-order step is x + (sigma_t - sigma_s) v (to 1e-12 relative in
    float64), from sigma 1 (lambda = -inf) on; the last step (sigma_t = 0, lambda = +inf) returns the x0-prediction x - sigma_s v
    exactly."""
    torch.manual_seed(0)
    sig = S.sampling_sigmas(20, 5.0)
    assert sig[0] == 1.0 and sig[-1] == 0.0
    smp = S.FlowDPMSolverSampler(sig, order=order)
    x = torch.randn(4, 33, dtype=torch.float64)
    n_first = 0
    for i in range(20):
        c, u = model_v(x, sig[i], 0), model_v(x, sig[i], 1)
        v = u + 5.0 * (c - u)
        first = smp.step_order() == 1
        want = x - sig[i] * v if i == 19 else x + (sig[i + 1] - sig[i]) * v
        x_in = x.clone()
        y = smp.step(c, u, 5.0, x)
        assert y is x
        if i == 19:
            assert torch.equal(y, want)
            assert torch.equal(smp._m[0], x_in - sig[i] * v)
        if first:
            n_first += 1
            assert float((y - want).abs().max()) <= 1e-12 * float(want.abs().max()), i
    assert n_first == (20 if order == 1 else 2)


@pytest.mark.parametrize("steps", [10, 20, 40, 50])
@pytest.mark.parametrize("shift", [3.0, 5.0, 8.0, 16.0])
def test_coefficients_equal_the_restatement(steps, shift):
    """cx, cv, ch of every step against DPMppRef's update read out on unit inputs, and the order schedule 1, 2, ..., 2, 1."""
    sig = S.sampling_sigmas(steps, shift)
    smp = S.FlowDPMSolverSampler(sig)
    want, orders = R.ref_coeffs(torch.tensor(sig, dtype=torch.float64))
    assert orders == [1] + [2] * (steps - 2) + [1]
    assert [smp.step_order(i) for i in range(steps)] == orders
    for i in range(steps):
        got = smp.coeffs(i)
        for a, b in zip(got, want[i]):
            assert math.isfinite(a) and abs(a - b) <= 1e-12 * max(1.0, abs(b)), (i, got, want[i])
    # the second step after sigma 1: r0 = +inf, the history term has no weight
    assert smp.coeffs(1)[2] == 0.0
    assert smp.coeffs(steps - 1) == (1.0, -sig[steps - 1], 0.0)


def test_trajectory_follows_the_restatement(monkeypatch):
    """fp32 kernel emulation (emu_ops.cfg_step) against DPMppRef in float64 on a non-linear model, with a guide scale."""
    monkeypatch.setattr(S.ops, "cfg_step", emu_ops.cfg_step)
    torch.manual_seed(3)
    sig = S.sampling_sigmas(25, 5.0)
    smp, ref = S.FlowDPMSolverSampler(sig), R.DPMppRef(torch.tensor(sig, dtype=torch.float64))
    x = torch.randn(3, 41)
    xr = x.double()
    for i in range(25):
        assert smp.timestep == 1000.0 * sig[i]
        x = smp.step(model_v(x, sig[i], 0), model_v(x, sig[i], 1), 5.0, x)
        xr = ref.step(sampler_ref.cfg(model_v(xr, sig[i], 0), model_v(xr, sig[i], 1), 5.0), xr)
        assert smp.step_order(i) == ref.this_order
        err = float((x.double() - xr).abs().max()) / max(1.0, float(xr.abs().max()))
        assert err < 2e-5, (i, err)


def test_second_order_convergence(f64_kernel):
    """dx/dsigma = k x + c has the closed form x(sigma) = (x0 + c/k) e^{k (sigma - sigma0)} - c/k, and its data prediction
    x - sigma v varies with sigma (were it constant, every order would be exact). Over 0.95 -> 0.05 the global error of the 2M
    solver falls ~4x per doubling of the step count, Euler's (and the first-order solver's) ~2x."""
    k, c = -2.0, 0.3  # measured ratios: 2M 4.35 / 4.20 / 4.09, Euler 1.89 / 1.94 / 1.97
    torch.manual_seed(4)
    x0 = torch.randn(16, dtype=torch.float64)

    def run(order, n):
        sig = torch.linspace(0.95, 0.05, n + 1, dtype=torch.float64).tolist()
        smp = S.FlowDPMSolverSampler(sig, order=order) if order else S.FlowEulerSampler(sig)
        x = x0.clone()
        for i in range(n):
            v = k * x + c
            x = smp.step(v, v, 1.0, x)
        exact = (x0 + c / k) * math.exp(k * (sig[-1] - sig[0])) - c / k
        return float((x - exact).abs().max())

    for order, lo, hi in ((2, 3.5, 4.6), (1, 1.7, 2.3), (0, 1.7, 2.3)):
        err = [run(order, n) for n in (16, 32, 64, 128)]
        ratios = [a / b for a, b in zip(err, err[1:])]
        assert all(lo < r < hi for r in ratios), (order, err, ratios)
    assert run(2, 32) < 0.1 * run(0, 32)


def test_history_buffers_are_recycled(f64_kernel):
    """Two buffers for the whole schedule: step i reads the previous x0-prediction (zeros, with weight 0, on the first step)
    and writes its own into the other one."""
    sig = S.sampling_sigmas(8, 5.0)
    smp = S.FlowDPMSolverSampler(sig)
    x = torch.randn(2, 9, dtype=torch.float64)
    ptrs = None
    for i in range(8):
        c, u = model_v(x, sig[i], 0), model_v(x, sig[i], 1)
        v = u + 2.0 * (c - u)
        m0 = x - sig[i] * v
        if i == 0:
            assert smp._m is None
        smp.step(c, u, 2.0, x)
        got = {b.data_ptr() for b in smp._m}
        ptrs = ptrs or got
        assert got == ptrs and len(got) == 2
        assert torch.equal(smp._m[0], m0)
    assert smp.i == 8


# ------------------------------------------------------------------------------------------- the caller loop, emulated kernels
def _head_with_hist(*args, step_hist=None, **kw):
    """mc_head_unpatchify_step_hist as the op chain it replaces: the head's unconditional prediction, then cfg_step with the one
    history term and the x0 output (the same fp32 emulation the unfused path runs)."""
    if step_hist is None:
        return _EMU_HEAD(*args, **kw)
    _head_with_hist.calls += 1
    cond, x_lat, g, cx, cv = kw.pop("step")
    out = kw.pop("out")
    hist, ch, sig, x0_out = step_hist
    y = _EMU_HEAD(*args, **kw)
    emu_ops.LAUNCHES -= 1  # one launch in all
    return emu_ops.cfg_step(cond, y, g, x_lat, cv, coef_x=cx, hist=[hist], coef_h=[ch], sigma=sig, out=out, x0_out=x0_out)


@pytest.fixture()
def emulated(monkeypatch):
    for mod in (wan_mod, patch_mod, S):
        monkeypatch.setattr(mod, "ops", emu_ops)
    monkeypatch.setattr(emu_ops, "head_unpatchify", _head_with_hist)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    _head_with_hist.calls = 0


def _wan21_models(steps, table, n_ours):
    model = wan_ref.WanModel(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128, text_len=32).init_synthetic(4)
    ref = copy.deepcopy(model)
    ref.__class__ = type("Ref", (ref.__class__,), {})
    wan_ref.install_magcache(type(ref), table, steps, thresh=0.12, K=2, retention_ratio=0.2)
    ours = []
    for _ in range(n_ours):
        o = copy.deepcopy(model)
        o.__class__ = type("Ours", (o.__class__,), {})
        mc.init_magcache(o, steps, thresh=0.12, K=2, retention_ratio=0.2, mag_ratios=table)
        object.__setattr__(o, "_mc_engine", mc.WanEngine(mc.WanWeights.from_module(o, torch.device("cpu"))))
        ours.append(o)
    return ref, ours


def test_wan21_loop_fused_equals_unfused_and_follows_the_oracle(emulated):
    steps, guide = 10, 5.0
    table = mc.tables()["wan2.1_t2v_1.3b"]
    ref, (a_model, b_model) = _wan21_models(steps, table, 2)
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(16, 2, 8, 8, generator=g)
    ctx, ctx_null = torch.randn(9, 128, generator=g), torch.randn(7, 128, generator=g)
    sig = mc.sampling_sigmas(steps, 5.0)
    sa, sb = mc.FlowDPMSolverSampler(sig), mc.FlowDPMSolverSampler(sig)
    sr = R.DPMppRef(torch.tensor(sig, dtype=torch.float64))
    xa, xb, xr = lat.clone(), lat.clone(), lat.clone()
    kinds = []
    with torch.no_grad():
        for i in range(steps):
            t = torch.tensor([sa.timestep], dtype=torch.float32)
            cond = a_model([xa], t=t, context=[ctx], seq_len=32)[0]
            uncond = a_model([xa], t=t, context=[ctx_null], seq_len=32)[0]
            xa = sa.step(cond, uncond, guide, xa)
            out = sb.denoise(b_model, xb, t, ctx, ctx_null, 32, guide)
            assert out.data_ptr() == xb.data_ptr()  # in place
            assert torch.equal(xa, xb) and torch.equal(sa._m[0], sb._m[0]), i
            assert a_model.cnt == b_model.cnt and a_model.accumulated_err == b_model.accumulated_err
            c_r = ref([xr], t=t, context=[ctx], seq_len=32)[0]
            kinds.append(int(ref.last_skip))
            u_r = ref([xr], t=t, context=[ctx_null], seq_len=32)[0]
            kinds.append(int(ref.last_skip))
            xr = sr.step(sampler_ref.cfg(c_r, u_r, guide), xr).float()
            assert b_model.cnt == ref.cnt and b_model.accumulated_err == ref.accumulated_err
            rel = float((xb.double() - xr.double()).norm() / xr.double().norm())
            assert rel < 3e-2, (i, rel)
    assert _head_with_hist.calls == steps  # every step's update ran in the unconditional call's head
    assert b_model._mc_engine._step is None
    want = mc.MagCacheConfig("wan2.1", 0.12, 2, 0.2, steps, table="wan2.1_t2v_1.3b").schedule().tolist()
    assert kinds == want and 0 < sum(want) < 2 * steps
    assert bool(torch.isfinite(xb).all())


def test_wan22_expert_pair_loop_fused_equals_unfused_and_follows_the_oracle(emulated):
    """Wan2.2 A14B: the high-noise expert for the first `high` steps, the low-noise one afterwards, one counter and one residual
    list for both (MagCache4Wan2.2/magcache_generate.py:209-362); the sampler keeps its history across the switch."""
    kw = dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128, text_len=32)
    steps, high, guide = 12, 5, 4.0
    protos = [wan_ref.WanModel(**kw).init_synthetic(seed) for seed in (1, 2)]
    ratios = mc.tables()["wan2.2_t2v_a14b"][2:].tolist()
    RefCls = type("RefW22", (wan_ref.WanModel,), {})
    classes = [type("OurW22a", (wan_ref.WanModel,), {}), type("OurW22b", (wan_ref.WanModel,), {})]
    refs, ours = [], [[], []]
    for p in protos:
        r = copy.deepcopy(p)
        r.__class__ = RefCls
        refs.append(r)
        for side, cls in enumerate(classes):
            o = copy.deepcopy(p)
            o.__class__ = cls
            object.__setattr__(o, "_mc_engine", mc.WanEngine(mc.WanWeights.from_module(o, torch.device("cpu"))))
            ours[side].append(o)
    wan_ref.install_magcache_wan22(RefCls, ratios, steps, thresh=0.12, K=2, retention_ratio=0.2, split_steps=high, mode="t2v")
    for side in (0, 1):
        mc.init_magcache_wan22(ours[side][0], ratios, steps, thresh=0.12, K=2, retention_ratio=0.2, split_steps=high, mode="t2v")
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(16, 2, 8, 8, generator=g)
    ctx, ctx_null = torch.randn(9, 128, generator=g), torch.randn(7, 128, generator=g)
    sig = mc.sampling_sigmas(steps, 12.0)
    sa, sb = mc.FlowDPMSolverSampler(sig), mc.FlowDPMSolverSampler(sig)
    sr = R.DPMppRef(torch.tensor(sig, dtype=torch.float64))
    xa, xb, xr = lat.clone(), lat.clone(), lat.clone()
    kinds = []
    with torch.no_grad():
        for i in range(steps):
            e = 0 if i < high else 1
            t = torch.tensor([sa.timestep], dtype=torch.float32)
            ma, mb = ours[0][e], ours[1][e]
            cond = ma([xa], t=t, context=[ctx], seq_len=32)[0]
            uncond = ma([xa], t=t, context=[ctx_null], seq_len=32)[0]
            xa = sa.step(cond, uncond, guide, xa)
            sb.denoise(mb, xb, t, ctx, ctx_null, 32, guide)
            assert torch.equal(xa, xb), i
            c_r = refs[e]([xr], t=t, context=[ctx], seq_len=32)[0]
            kinds.append(int(refs[e].last_skip))
            u_r = refs[e]([xr], t=t, context=[ctx_null], seq_len=32)[0]
            kinds.append(int(refs[e].last_skip))
            xr = sr.step(sampler_ref.cfg(c_r, u_r, guide), xr).float()
            for cls in classes:
                assert cls.accumulated_err == RefCls.accumulated_err and cls.accumulated_steps == RefCls.accumulated_steps
            rel = float((xb.double() - xr.double()).norm() / xr.double().norm())
            assert rel < 3e-2, (i, rel)
    assert _head_with_hist.calls == steps
    want = mc.MagCacheConfig("wan2.2-t2v", 0.12, 2, 0.2, steps, mag_ratios=classes[1].mag_ratios, high_noise_steps=high).schedule().tolist()
    assert kinds == want and 0 < sum(want) < 2 * steps
    assert any(kinds[2 * high:]), "the low-noise expert must reach hits"
    assert bool(torch.isfinite(xb).all())


# ------------------------------------------------------------------------------------------- plumbing and argument checks
def test_x0_out_needs_a_history_term(emulated):
    _, (m,) = _wan21_models(4, mc.tables()["wan2.1_t2v_1.3b"], 1)
    x = torch.zeros(16, 2, 8, 8)
    with pytest.raises(ValueError):
        m._mc_engine.arm_step(x, x, 5.0, 1.0, -0.1, out=x, x0_out=torch.zeros_like(x))
    assert m._mc_engine._step is None
    with pytest.raises(ValueError):
        S.cfg_denoise_step(m, x, torch.tensor([999.0]), torch.zeros(9, 128), torch.zeros(7, 128), 32, 5.0, -0.1, x0_out=torch.zeros_like(x))


def test_solver_order_refused():
    with pytest.raises(NotImplementedError):
        S.FlowDPMSolverSampler(S.sampling_sigmas(10, 5.0), order=3)


def _head_step_hist_args(**over):
    """mc_head_unpatchify_step_hist's arguments with plausible (never dereferenced) device addresses; every case below fails an
    argument check, which runs before any device work."""
    a = dict(x=0x10000, x_dtype=L.MC_F32, r=None, rows=32760, row_offset=0, cols=1536, F=21, Hp=30, Wp=52, C_out=16, eps=1e-6,
             outs=[0x20000], prepared=0x30000, prepared_bytes=1 << 20, flags=0, cond=0x40000, x_latent=0x20000, g=5.0, cx=1.0,
             cv=-0.1, hist=0x50000, ch=0.3, sigma=0.9, x0_out=0x60000)
    a.update(over)
    return a


def _call(a):
    import ctypes
    outs = (ctypes.c_void_p * len(a["outs"]))(*a["outs"])
    return L.lib.mc_head_unpatchify_step_hist(a["x"], a["x_dtype"], a["r"], a["rows"], a["row_offset"], a["cols"], a["F"], a["Hp"], a["Wp"],
                                              a["C_out"], a["eps"], outs, len(a["outs"]), a["prepared"], a["prepared_bytes"], a["flags"],
                                              a["cond"], a["x_latent"], a["g"], a["cx"], a["cv"], a["hist"], a["ch"], a["sigma"], a["x0_out"], None)


@pytest.mark.parametrize("case,over,msg", [
    ("null hist", dict(hist=None), "null cond / latent / hist"),
    ("null cond", dict(cond=None), "null cond / latent / hist"),
    ("null latent", dict(x_latent=None), "null cond / latent / hist"),
    ("misaligned hist", dict(hist=0x50004), "8-byte aligned"),
    ("misaligned x0_out", dict(x0_out=0x60004), "8-byte aligned"),
    ("misaligned cond", dict(cond=0x40004), "8-byte aligned"),
    ("hist is out", dict(hist=0x20000), "hist aliases out[0]"),
    ("hist is a peer out", dict(outs=[0x20000, 0x70000], hist=0x70000), "hist aliases out[1]"),
    ("hist is x0_out", dict(hist=0x60000), "hist aliases x0_out"),
    ("x0_out is out", dict(x0_out=0x20000, x_latent=0x80000), "x0_out aliases out[0]"),
    ("x0_out is the latent", dict(x0_out=0x80000, x_latent=0x80000), "x0_out may not alias the latent"),
    ("x0_out is cond", dict(x0_out=0x40000), "x0_out may not alias the latent"),
    ("cond is out", dict(cond=0x20000), "cond aliases out[0]"),
    ("no outs", dict(outs=[]), "n_out=0"),
    ("null x", dict(x=None), "null pointer"),
])
def test_step_hist_argument_checks(case, over, msg):
    """Each refusal of mc_head_unpatchify_step_hist returns MC_ERR_INVALID with its message, before any device work (so on CPU)."""
    assert _call(_head_step_hist_args(**over)) == L.MC_ERR_INVALID, case
    assert msg in L.lib.mc_last_error().decode(), (case, L.lib.mc_last_error().decode())
