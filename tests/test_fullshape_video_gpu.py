"""The benchmarked video held to fp64 at full depth: Wan2.1-T2V-1.3B at 832x480x81 (latent 16 x 21 x 60 x 104, 32 760 tokens),
all 30 blocks, through the denoising step bench.py times, with hits and misses.

Wan-1.3B is the one benchmarked model whose whole network fits on an H100 in fp64 (about 11 GB of weights; FLUX, HunyuanVideo
and Wan-14B would need 96-112 GB, so their full-shape tests run one block). So here the computation the bench reports is held
to an fp64 evaluation of the same network at its real depth and shape, across steps whose timestep changes on every call.

Window. Steps 8 to 25 of the 50-step schedule (36 calls), where the bench's warm-up and attribution passes run. Every controller
is restarted at step 8 the way bench.py's `set_step` does (fresh accumulators, cnt = 16; `test_restart_at_step_8_is_the_walked_state`
holds that this is the state a video walked from step 0 has there). Under E012K4R02 the window then misses at steps 8, 9, 14,
19 and 24 on both CFG slots and hits in runs of four in between: 10 computed forwards per side. The walked skip sequence equals
`schedule_mask(...)[16:52]` on every side, and the controller state is bit-equal after every call.

Sides, each walking its own latent from bench.py's inputs (its latent, its two 512 x 4096 text contexts, its fp32 sigmas,
guidance 5):
* ours: `mc.cfg_denoise_step` called as bench.py calls it: the cond forward, then the unconditional forward whose head epilogue
  applies the CFG combine and the Euler update in place on the latent (`arm_step` + `mc_head_unpatchify_step`);
* the bf16 oracle and the fp64 oracle: the caller loop of wan_magcache.py:296-310 with Euler (cond call, uncond call,
  v = u + g (c - u), x <- x + dt v), in fp32 and in fp64. They run on the GPU with `_oracle_on_gpu`'s query-chunked attention,
  one after the other, before ours (module fixture).

Compared after every step, at DESIGN §5's rule: the cond prediction (the fused step never writes the unconditional one), the
latent increment x_{i+1} - x_i = dt v, the displacement x_{i+1} - x_8 (drift that builds up over steps), and after a miss both
slots' residual caches. Not the raw latent: |dt| is 0.005-0.011 here, so |dt v| is about 1 % of |x| and an error in v would
sit below the rule's 1e-3 floor.

A hit must use the current step's time embedding for the head's modulation together with the residual stored at the slot's last
miss; a hit that reused the last miss's head preparation would give the same result at a fixed t, which is all the one-layer
full-shape tests use. `test_modelled_defects_fail_the_rule` shows that the rule fails, within the window, on a bf16-oracle
trajectory carrying one such defect, against the references of the main run."""
import contextlib
import copy
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_fullshape_workloads_gpu import _need_device_memory, _oracle_on_gpu, _report, rule_fraction  # noqa: E402

import bench  # noqa: E402  (the workload: shape, preset, table, warm-up step)

DEV = "cuda"
GUIDE, SHIFT = 5.0, 5.0  # bench.py's guidance and sigma shift
FIRST, LAST = bench.WARM_START_STEP, 25
STEPS = range(FIRST, LAST + 1)
ATTRS = ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps")


def bench_sigmas():
    """bench.py's schedule by its own fp32 statements: sigmas (terminal 0 included), t_i = 1000 sigma_i as fp32 [1] tensors,
    dt_i = sigma_{i+1} - sigma_i."""
    n = bench.SAMPLE_STEPS
    s = torch.linspace(1.0, 1.0 / n, n)
    sig = torch.cat([SHIFT * s / (1 + (SHIFT - 1) * s), torch.zeros(1)])
    return sig, [sig[i:i + 1] * 1000.0 for i in range(n)], [float(sig[i + 1] - sig[i]) for i in range(n)]


def bench_config():
    import magcache_b200 as mc
    return mc.MagCacheConfig("wan2.1", sample_steps=bench.SAMPLE_STEPS, table=bench.TABLE, **bench.PRESET)


def video_mask():
    """The skip schedule of one whole video (one entry per call) from the C controller."""
    from magcache_b200.controller import make_ctrl_config, schedule_mask
    cfg = bench_config()
    return schedule_mask(make_ctrl_config(cfg.num_steps, cfg.thresh, cfg.K, cfg.retention_ratio, cfg.resolved_ratios(), **cfg.ctrl_kwargs()),
                         cfg.num_steps).tolist()


def _state(m):
    return [np.asarray(getattr(m, a), dtype=np.float64).tolist() for a in ATTRS]


# ------------------------------------------------------------------------------------------- CPU
def test_bench_sigmas_are_the_sampling_sigmas():
    """The fp32 schedule the bench builds is `mc.sampling_sigmas(50, 5.0)` to fp32 rounding (within 2 ulps), terminal 0 exact."""
    import magcache_b200 as mc
    sig, _, _ = bench_sigmas()
    want = torch.tensor(mc.sampling_sigmas(bench.SAMPLE_STEPS, SHIFT), dtype=torch.float64)
    assert sig.shape == want.shape and float(sig[-1]) == 0.0 == float(want[-1])
    assert bool(((sig.double() - want).abs() <= 2.0 ** -22 * want).all()), (sig.double() - want).abs().max()


def test_restart_at_step_8_is_the_walked_state():
    """bench.py's `set_step(8)` (and the GPU test here) restart a controller with fresh accumulators and cnt = 16, on the claim
    that this is the state a video walked from call 0 has at call 16 (steps 0-9 lie in the retention window). Held on the oracle
    controller and on ours (the C controller behind the patched forward's attributes) with bench.py's preset and table: the
    walked and the restarted state are equal, both walk on to `schedule_mask[16:52]`, and that window misses at steps 8, 9, 14,
    19 and 24 on both slots."""
    import magcache_b200 as mc
    from magcache_b200.config import FAMILIES
    from magcache_b200.controller import AttrController
    from oracle.controller_ref import ControllerRef
    cfg = bench_config()
    start, calls = 2 * FIRST, 2 * len(STEPS)
    window = video_mask()[start:start + calls]
    assert [FIRST + c // 2 for c, hit in enumerate(window) if not hit] == [8, 8, 9, 9, 14, 14, 19, 19, 24, 24]

    args = ("wan2.1", cfg.resolved_ratios(), cfg.num_steps, cfg.thresh, cfg.K, cfg.retention_ratio)
    walked, restarted = ControllerRef(*args), ControllerRef(*args)
    assert walked.mask(start) == [0] * start
    restarted._reset()
    restarted.cnt = start
    for c in (walked, restarted):
        assert (c.cnt, c.ratio, c.err, c.steps) == (start, [1.0, 1.0], [0.0, 0.0], [0, 0])
        assert c.mask(calls) == window

    ctrl = AttrController(FAMILIES["wan2.1"])

    def patched():
        o = type("CtrlOnly", (), {})()
        return mc.init_magcache(o, bench.SAMPLE_STEPS, table=bench.TABLE, **bench.PRESET)

    def walk(o, n):
        out = []
        for _ in range(n):
            out.append(int(ctrl.decide(o)))
            ctrl.advance(o)
        return out

    ours_walked, ours_restarted = patched(), patched()
    assert walk(ours_walked, start) == [0] * start
    mc.reset_magcache(ours_restarted)
    ours_restarted.cnt = start  # bench.py's set_step
    assert _state(ours_walked) == _state(ours_restarted) == [start, [1.0, 1.0], [0.0, 0.0], [0, 0]]
    assert walk(ours_walked, calls) == walk(ours_restarted, calls) == window
    assert _state(ours_walked) == _state(ours_restarted)


# ------------------------------------------------------------------------------------------- GPU: the three trajectories
def _inputs():
    """bench.py's inputs: its latent (seed 0) and its cond / null text contexts (seeds 1, 2, bf16), on the device; its t and dt."""
    lat = torch.randn(*bench.LATENT, generator=torch.Generator().manual_seed(0)).to(DEV)
    ctx = torch.randn(bench.TEXT_LEN, bench.TEXT_DIM, generator=torch.Generator().manual_seed(1)).bfloat16().to(DEV)
    ctx_null = torch.randn(bench.TEXT_LEN, bench.TEXT_DIM, generator=torch.Generator().manual_seed(2)).bfloat16().to(DEV)
    _, ts, dts = bench_sigmas()
    return lat, ctx, ctx_null, [t.to(DEV) for t in ts], dts


def _as_oracle(m, name):
    """`m` (in place) as an oracle model of its own class, restarted at step 8: installed fresh (`install_magcache` with the
    resolved table), then cnt = 16 — what `reset_magcache` + `cnt = 16` leave on ours."""
    from oracle import wan_ref
    m.__class__ = type(name, (wan_ref.WanModel,), {})
    m.__dict__.pop("cnt", None)
    cfg = bench_config()
    wan_ref.install_magcache(type(m), cfg.resolved_ratios(), bench.SAMPLE_STEPS, **bench.PRESET)
    m.cnt = 2 * FIRST
    return m


def _record(step, skips, states, cond, x_prev, x, x_first, res):
    return dict(step=step, skips=skips, states=states, cond=cond, inc=x - x_prev, disp=x - x_first, res=res)


def _oracle_walk(m, inputs, exact=False, dt_ahead=0):
    """The caller loop over the window on an oracle model, one record per step. `exact`: the fp64 evaluation (latent and
    update in fp64); `dt_ahead` = 1 is defect (c), the Euler update with the next step's dt."""
    from oracle import wan_ref
    lat, ctx, ctx_null, ts, dts = inputs
    dt_type = torch.float64 if exact else torch.float32
    precision = wan_ref.exact_fp64 if exact else contextlib.nullcontext
    x = x_first = lat.to(dt_type)
    for i in STEPS:
        t = ts[i].to(dt_type)
        preds, skips, states = [], [], []
        for c in (ctx, ctx_null):
            with torch.no_grad(), precision():
                preds.append(m([x], t=t, context=[c.to(dt_type) if exact else c], seq_len=bench.N_TOK)[0])
            skips.append(int(m.last_skip))
            states.append(_state(m))
        cond, uncond = preds
        x_next = x + dts[i + dt_ahead] * (uncond + GUIDE * (cond - uncond))
        res = {s: m.residual_cache[s][0] for s in (0, 1) if not skips[s]}
        yield _record(i, skips, states, cond, x, x_next, x_first, res)
        x = x_next


def _compare(rec, ref, ex):
    """DESIGN §5's rule on every compared quantity of one step: {quantity: (e_ref, fraction of the bound)}."""
    pairs = [(q, rec[q], ref[q], ex[q]) for q in ("cond", "inc", "disp")]
    assert rec["res"].keys() == ref["res"].keys() == ex["res"].keys(), rec["step"]
    pairs += [(f"res{s}", rec["res"][s], ref["res"][s], ex["res"][s]) for s in sorted(ref["res"])]
    out = {}
    for q, a, b, c in pairs:
        e_ref, _, _, frac = rule_fraction(a, b, c)
        out[q] = (e_ref, frac)
    return out


def _line(step, skips, fr):
    kinds = "/".join("hit" if s else "miss" for s in skips)
    return f"  step {step:2d} {kinds:9s} " + "  ".join(f"{q} {e:.2e} ({f:.2f})" for q, (e, f) in fr.items())


@pytest.fixture(scope="module")
def refs():
    """The model (seeded synthetic weights, on the device) and the two reference trajectories over the window: the fp64 oracle
    (run first, its model dropped after), then the bf16 oracle on the model itself."""
    from oracle import wan_ref
    _need_device_memory(40)
    t0 = time.time()
    model = wan_ref.WanModel(dim=bench.D, ffn_dim=bench.FFN, num_heads=bench.HEADS, num_layers=bench.LAYERS, text_dim=bench.TEXT_DIM,
                             text_len=bench.TEXT_LEN).init_synthetic(0).to(DEV)
    inputs = _inputs()
    with pytest.MonkeyPatch.context() as mp:
        _oracle_on_gpu(mp)
        m64 = _as_oracle(copy.deepcopy(model).double(), "VideoRef64")
        t1 = time.time()
        ex = list(_oracle_walk(m64, inputs, exact=True))
        del m64
        torch.cuda.empty_cache()
        _report("fp64 oracle, 36 calls", t1)
        t1 = time.time()
        ref = list(_oracle_walk(_as_oracle(model, "VideoRef"), inputs))
        _report("bf16 oracle, 36 calls", t1)
    return dict(model=model, inputs=inputs, ex=ex, ref=ref, t0=t0)


@pytest.mark.gpu
def test_bench_video_steps_8_to_25_vs_fp64(refs, monkeypatch):
    """Ours through `cfg_denoise_step` as bench.py calls it, over steps 8-25, against both references at DESIGN §5's rule."""
    import magcache_b200 as mc
    from magcache_b200.patch import _engine
    from oracle import wan_ref
    lat, ctx, ctx_null, ts, dts = refs["inputs"]
    ours = copy.deepcopy(refs["model"])
    ours.__class__ = type("VideoOurs", (wan_ref.WanModel,), {})
    mc.init_magcache(ours, bench.SAMPLE_STEPS, table=bench.TABLE, **bench.PRESET)
    mc.reset_magcache(ours)  # bench.py's set_step(8)
    ours.cnt = 2 * FIRST

    eng = _engine(ours)  # the engine the first forward would build; its two entry points recorded
    kinds, armed = [], []
    engine_forward, engine_arm = eng.forward, eng.arm_step

    def forward_kind(kind, slot):
        kinds.append(kind)
        return engine_forward(kind, slot)

    def arm_step(cond, x_latent, *a, out=None):
        armed.append((x_latent.data_ptr(), None if out is None else out.data_ptr()))
        return engine_arm(cond, x_latent, *a, out=out)

    monkeypatch.setattr(eng, "forward", forward_kind)
    monkeypatch.setattr(eng, "arm_step", arm_step)
    mask = video_mask()
    t1 = time.time()
    x = lat.clone()
    x_first = x.clone()
    worst = {}
    print()
    for n, i in enumerate(STEPS):
        preds, states = [], []

        def forward(xx, tt, cc):
            out = ours([xx], t=tt, context=[cc], seq_len=bench.N_TOK)[0]
            preds.append(out)
            states.append(_state(ours))
            return out

        x_prev = x.clone()
        with torch.no_grad():
            out = mc.cfg_denoise_step(ours, x, ts[i], ctx, ctx_null, bench.N_TOK, GUIDE, dts[i], forward=forward)
        # the fused form: the engine armed with this latent as the output, which the unconditional call returned, updated in place
        assert len(armed) == n + 1 and armed[-1] == (x.data_ptr(), x.data_ptr()), (i, armed)
        assert out.data_ptr() == x.data_ptr() and len(preds) == 2
        skips = [int(k == "hit") for k in kinds[-2:]]
        rec = _record(i, skips, states, preds[0], x_prev, x, x_first,
                      {s: ours.residual_cache[s][0] for s in (0, 1) if not skips[s]})
        ref, ex = refs["ref"][n], refs["ex"][n]
        assert ref["step"] == ex["step"] == i
        assert rec["skips"] == ref["skips"] == ex["skips"] == mask[2 * i:2 * i + 2], (i, rec["skips"], ref["skips"], ex["skips"])
        assert rec["states"] == ref["states"] == ex["states"], (i, rec["states"], ref["states"], ex["states"])
        fr = _compare(rec, ref, ex)
        print(_line(i, skips, fr))
        for q, (e_ref, f) in fr.items():
            lo, hi, w = worst.get(q, (e_ref, e_ref, 0.0))
            worst[q] = (min(lo, e_ref), max(hi, e_ref), max(w, f))
        assert all(f <= 1.0 for _, f in fr.values()), (i, fr)
    assert len(kinds) == 2 * len(STEPS) and kinds.count("miss") == 10, kinds
    assert bool(torch.isfinite(x).all())
    for q, (lo, hi, w) in worst.items():
        print(f"  {q}: e_ref {lo:.2e}-{hi:.2e}, worst fraction of the bound {w:.2f}")
    _report("ours, 36 calls", t1)
    _report("module so far", refs["t0"])
    del ours, eng
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------- teeth
@pytest.mark.gpu
def test_modelled_defects_fail_the_rule(refs, monkeypatch):
    """The bf16 oracle's trajectory re-run with one modelled defect, checked against the faithful bf16 and the fp64 records of
    the main run, fails DESIGN §5's rule within the window for each of:
      (a) on a hit, the head gets the t of the slot's last miss;
      (b) on a hit, the residual comes from the other CFG slot;
      (c) the Euler update uses the next step's dt;
      (d) a miss runs 29 of the 30 blocks (the last block passes its input through).
    Each run stops at its first failing step."""
    from oracle import wan_ref
    _oracle_on_gpu(monkeypatch)
    mask = video_mask()
    model, inputs = refs["model"], refs["inputs"]

    def last_miss_t(m, mp):
        base, last = type(m).forward, {}

        def forward(self, x, t, context, seq_len):
            slot = self.cnt % 2
            if mask[self.cnt]:
                t = last[slot]  # a hit's t feeds only the head (e0 feeds the blocks, which a hit skips)
            else:
                last[slot] = t
            return base(self, x, t, context, seq_len)
        mp.setattr(type(m), "forward", forward)

    def other_slot(m, mp):
        base = type(m).forward

        def forward(self, *a, **kw):
            if not mask[self.cnt]:
                return base(self, *a, **kw)
            self.residual_cache.reverse()  # the hit reads (and stores back) the other slot's residual
            try:
                return base(self, *a, **kw)
            finally:
                self.residual_cache.reverse()
        mp.setattr(type(m), "forward", forward)

    def depth_29(m, mp):
        mp.setattr(m.blocks[-1], "forward", lambda x, **kw: x)

    defects = [("a: hit head with the last miss's t", last_miss_t, 0), ("b: hit reads the other slot's residual", other_slot, 0),
               ("c: Euler update with the next step's dt", None, 1), ("d: miss runs 29 of 30 blocks", depth_29, 0)]
    print()
    for name, patch, dt_ahead in defects:
        t1 = time.time()
        failed = None
        with monkeypatch.context() as mp:
            m = _as_oracle(model, "VideoDefect")
            if patch is not None:
                patch(m, mp)
            for n, rec in enumerate(_oracle_walk(m, inputs, dt_ahead=dt_ahead)):
                fr = _compare(rec, refs["ref"][n], refs["ex"][n])
                q, (e_ref, f) = max(fr.items(), key=lambda kv: kv[1][1])
                if f > 1.0:
                    failed = (rec["step"], q, e_ref, f)
                    print(f"  [{name}] fails at step {rec['step']} on {q}: {f:.1f}x the bound (e_ref {e_ref:.2e}), {time.time() - t1:.0f} s")
                    break
        assert failed is not None, f"defect ({name}) passes the rule over the whole window"
