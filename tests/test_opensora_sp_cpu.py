"""Open-Sora sequence parallelism (`enable_sequence_parallel`, VideoSys DSP) without a GPU: the frame / position partition against
VideoSys's `split_sequence` pad rule, the interface's refusals, and world-2 / world-4 gloo runs of the engine through the kernel
emulation with the collective switch (`shard.CollectiveSwitch`). Every rank's output must be bit-equal to the unsharded engine's on
the same inputs — MagCache, TeaCache at two thresholds, the plain forward and the RFlow sampler's fused step — its residual rows
the unsharded engine's rows of its frames, and the controller attributes the same on every rank."""
import json
import math
import os
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import magcache_b200 as mc
from magcache_b200 import opensora as os_mod
from magcache_b200 import shard

import opensora_emu
import opensora_ref as R
import opensora_sp_cases as C
import opensora_tea_ref as TR

BF, F32 = torch.bfloat16, torch.float32


GOLD = os.path.join(os.path.dirname(__file__), "golden")
DOC = json.load(open(os.path.join(GOLD, "opensora_sp.json")))


# ---- partition ------------------------------------------------------------------------------------------------------------------
def _split_sequence_ranges(n, world):
    """videosys/core/comm.py: `set_pad` pads the axis to a multiple of P, `split_sequence` takes chunk r of P equal chunks; the real
    (unpadded) indices of each chunk."""
    pad = (world - n % world) % world
    idx = torch.arange(n + pad)
    return [[int(i) for i in c if i < n] for c in idx.chunk(world)]


# (T, S, P): the fixture's shapes, the latent lengths of Open-Sora's 2 s ... 32 s videos at 480p, and a position count P does not divide
@pytest.mark.parametrize("T,S,P", [(7, 42, 2), (7, 42, 4), (35, 42, 2), (15, 1800, 2), (15, 1800, 4), (15, 1800, 8), (30, 1800, 8),
                                   (60, 1800, 8), (120, 1800, 8), (240, 1800, 8), (51, 43, 4)])
def test_partition_is_split_sequence(T, S, P):
    frames, positions = shard.frame_position_shards(P, T, S)
    for shards, n in ((frames, T), (positions, S)):
        assert [list(range(s.start, s.stop)) for s in shards] == _split_sequence_ranges(n, P)
        assert all(s.n_slots == -(-n // P) for s in shards)


@pytest.mark.parametrize("key", sorted(DOC["runs"]))
def test_partition_is_the_references_recorded_split(key):
    """Each rank's frame range after the reference's own `set_pad` + `split_sequence` (tests/golden/make_opensora_sp_golden.py)."""
    run = DOC["runs"][key]
    frames, _ = shard.frame_position_shards(run["world"], run["T"], (DOC["Hx"] // 2) * (DOC["Wx"] // 2))
    assert [r["split"] for r in run["ranks"]] == [[f.start, f.stop] for f in frames]


@pytest.mark.parametrize("key", sorted(DOC["runs"]))
def test_reference_dsp_equals_its_sp1_run(key):
    """The premise of holding the engine bit-equal to its one-GPU run, from the reference's own DSP code: in fp32 every rank's output
    equals the sp = 1 output exactly (the fixture records 0.0, within the 1e-6 asked) and the controller attributes are the sp = 1
    run's on every rank (TeaCache's distance to 1e-6 relative). In bf16 the reference's torch-CPU ops round differently on a rank's smaller tensors: outputs move by up to
    0.06 (recorded), and the attributes still agree on every rank."""
    run = DOC["runs"][key]
    for r in run["ranks"]:
        assert r["attrs"] == run["ranks"][0]["attrs"], key
        if key.endswith("fp32"):
            assert r["bit_equal_sp1"] and r["max_abs_diff_sp1"] <= 1e-6, key
            # TeaCache's accumulated distance is an fp32 torch mean over all rows, summed in an order that follows the thread count
            # of the process: within 1e-6 relative of the sp = 1 run's, with the same decisions (the outputs above are the same bits)
            for a, a1 in zip(r["attrs"], run["sp1_attrs"]):
                assert all(abs(a[k] - a1[k]) <= 1e-6 * abs(a1[k]) for k in a1), key
        else:
            assert r["max_abs_diff_sp1"] <= 0.0625, key


@pytest.mark.parametrize("T,P", [(5, 4), (1, 2), (9, 8)])
def test_partition_without_a_frame_raises(T, P):
    with pytest.raises(ValueError, match=rf"T = {T} latent frames on P = {P} ranks"):
        shard.frame_position_shards(P, T, 42)


# ---- interface ------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(os_mod, "ops", namespace())
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def test_enable_sequence_parallel_refusals(emulated):
    class NotOpenSora(torch.nn.Module):
        def forward(self, x):
            return x
    with pytest.raises(RuntimeError, match="Open-Sora forward"):
        mc.enable_sequence_parallel(NotOpenSora(), 0, 2)
    m, _ = C.build("magcache")
    with pytest.raises(ValueError, match="rank 2 outside"):
        mc.enable_sequence_parallel(m, 2, 2)
    C.calls(m, "magcache", 1, 2, 3, 8, 8, "cpu")
    with pytest.raises(RuntimeError, match="before the first forward"):
        mc.enable_sequence_parallel(m, 0, 2)


def test_world_one_is_the_unsharded_engine(emulated):
    sp, one = C.build("magcache")
    mc.enable_sequence_parallel(sp, 0, 1)
    got, want = C.calls(sp, "magcache", 4, 2, 3, 8, 8, "cpu"), C.calls(one, "magcache", 4, 2, 3, 8, 8, "cpu")
    assert sp._mc_opensora_engine.sp is None and sp._mc_opensora_engine.switch is None
    C.compare(got, want, 3, 0, 3, "world 1")


# ---- kernel emulation -----------------------------------------------------------------------------------------------------------
def attention_temporal_d72(q, k, v, heads, B, T, S, scale=None, out=None, tag=None):
    """`ops.attention_temporal_d72`: T <= 32 the fp32-P kernel (opensora_emu's model), past 32 frames the tensor-core kernel's chain
    (fp32 scores, e = 2^(x - max), O = sum bf16(e) v, l = sum e, bf16(O / l)). Every value is formed in fp64 and rounded to fp32, so
    that a sequence's result depends only on its own rows, as the kernel's does. In fp32, torch's CPU kernels do not give that: its
    vectorised exp2 and its scalar loop for the elements left over differ in the last bit, and which elements are left over depends on
    how the tensor is split among threads — that is, on how many sequences the call holds (a rank's S_r against S). That once moved one
    bf16 output of a sharded TeaCache run at T = 35 against the unsharded one."""
    if T <= 32:
        return opensora_emu.attention_temporal_d72(q, k, v, heads, B, T, S, scale, out, tag)
    scale = 1.0 / math.sqrt(72) if scale is None else scale
    seq = lambda t: t.to(F32).view(B, T, S, heads, 72).permute(0, 2, 3, 1, 4)  # noqa: E731
    x = (seq(q).double() @ seq(k).double().transpose(-1, -2)).float() * (scale * 1.4426950408889634)
    e = torch.exp2((x - x.max(-1, keepdim=True).values).double()).float()
    o = (e.to(BF).double() @ seq(v).double()).float() / e.double().sum(-1, keepdim=True).float()
    out.copy_(o.permute(0, 3, 1, 2, 4).reshape(B * T * S, heads * 72).to(BF))
    return out


def namespace():
    ns = TR.namespace()
    ns.attention_temporal_d72 = attention_temporal_d72

    def opensora_head(x, mod, w, bias, grid, crop, res=None, step=None, out=None, eps=1e-6, tag=None):
        """The op chain `mc_opensora_head` replaces (as tests/test_opensora_sampler_cpu.py states it)."""
        T, H, W = grid
        Tx, Hx, Wx = crop
        N = T * H * W
        B, D = x.shape[0] // N, x.shape[1]
        if res is not None:
            x = ns.cache_hit_add(x, res)
        h = torch.cat([ns.ln_t2i_modulate(x[b * N:(b + 1) * N], mod[b], 1, 0) for b in range(B)])
        o = ns.gemm(h, w, bias, 0)
        pred = o.view(B, T, H, W, 1, 2, 2, 8).permute(0, 7, 1, 4, 2, 5, 3, 6).reshape(B, 8, T, 2 * H, 2 * W)[:, :, :Tx, :Hx, :Wx].float()
        if step is None:
            return pred
        z, g, dt = step
        pred_cond, pred_uncond = pred.chunk(2, dim=1)[0].chunk(2, dim=0)
        out.copy_(z + (pred_uncond + g * (pred_cond - pred_uncond)) * dt[:, None, None, None, None])
        return out

    def opensora_head_frames(x, mod, w, bias, grid, crop, t0, out, res=None, step=None, eps=1e-6, tag=None):
        """`mc_opensora_head_frames`: the window [t0, t0 + T) of the full-size `out` (and of z)."""
        T, H, W = grid
        _, Hx, Wx = crop
        if step is None:
            out[:, :, t0:t0 + T] = opensora_head(x, mod, w, bias, grid, (T, Hx, Wx), res=res)
            return out
        z, g, dt = step
        zw = z[:, :, t0:t0 + T].contiguous()
        out[:, :, t0:t0 + T] = opensora_head(x, mod, w, bias, grid, (T, Hx, Wx), res=res, step=(zw, g, dt), out=torch.empty_like(zw))
        return out

    ns.opensora_head = opensora_head
    ns.opensora_head_frames = opensora_head_frames
    return ns


# ---- world-2 / world-4 runs -----------------------------------------------------------------------------------------------------
def _oracle_check(T, Hx, Wx, outs):
    """The project's criterion for the sharded outputs against the reference restatement (bf16 and fp64), as
    tests/test_opensora_engine_emulated_cpu.py applies it to the unsharded engine."""
    base = R.STDiT3(**R.CONFIGS["tiny"]).init_synthetic(0)
    refs = []
    for dt in (torch.bfloat16, torch.float64):
        m = base.to(dt) if dt == torch.bfloat16 else R.STDiT3(**R.CONFIGS["tiny"]).init_synthetic(0).double()
        m.__class__ = type(f"SPRef_{dt}", (R.STDiT3,), {})
        R.install_magcache(m.__class__, thresh=0.5, K=3, skip_time=2)
        refs.append(m)
    lat, y, kw = C.video(2, T, Hx, Wx)
    ts, _ = C.timesteps(len(outs), 2, "cpu")
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())  # noqa: E731
    with torch.no_grad():
        for i, o in enumerate(outs):
            r = refs[0](lat(i), ts[i], None, y, **kw)
            r64 = refs[1](lat(i).double(), ts[i].to(torch.bfloat16).double(), None, y.double(), **kw)
            e_ref = rel(r, r64)
            assert rel(o, r64) <= 1.5 * e_ref + 1e-3 and rel(o, r) <= 2 * e_ref + 1e-3, (i, rel(o, r64), rel(o, r), e_ref)


def _worker(rank, world, initfile, shapes):
    dist.init_process_group("gloo", init_method=f"file://{initfile}", rank=rank, world_size=world)
    torch.set_num_threads(max(1, (os.cpu_count() or 1) // world))  # the ranks share the machine's cores
    try:
        os_mod.ops = namespace()
        torch.Tensor.is_cuda = property(lambda self: True)
        B = 2
        for T, Hx, Wx in shapes:
            S = (-(-Hx // 2)) * (-(-Wx // 2))
            fr = shard.frame_position_shards(world, T, S)[0][rank]
            for kind, thresh, n in (("magcache", None, 10), ("teacache", 0.1, 10), ("teacache", 10.0, 6), ("plain", None, 2)):
                sp, one = C.build(kind, thresh=thresh)
                C.enable(sp, rank, world)
                got = C.calls(sp, kind, n, B, T, Hx, Wx, "cpu")
                want = C.calls(one, kind, n, B, T, Hx, Wx, "cpu")
                C.compare(got, want, T, fr.start, fr.stop, (world, T, kind, thresh))
                eng = sp._mc_opensora_engine
                assert (eng.t0, eng.T_loc) == (fr.start, fr.n_local) and not eng.switch.p2p
                if kind == "magcache":
                    assert any(a["skip_steps"] > 0 for _, a, _ in got) and got[0][1]["skip_steps"] == 0
                    if rank == 0 and T < 32:
                        _oracle_check(T, Hx, Wx, [o for o, _, _ in got])
                if kind == "teacache" and thresh > 1:
                    assert any(a["accumulated_rel_l1_distance"] > 0 for _, a, _ in got)  # hits
            sp, one = C.build("magcache")
            C.enable(sp, rank, world)
            seen, out = C.sample(sp, T, Hx, Wx, "cpu")
            seen1, out1 = C.sample(one, T, Hx, Wx, "cpu")
            assert len(seen) == 30 and all(torch.equal(a, b) for a, b in zip(seen, seen1)) and torch.equal(out, out1), (world, T, "sampler")
            assert sp.skip_steps == one.skip_steps
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,shapes", [(2, [(7, 12, 14), (35, 11, 13)]), (4, [(7, 12, 14)])], ids=["world2", "world4"])
def test_sequence_parallel_runs_are_bit_equal_to_one_engine(world, shapes):
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(world, os.path.join(d, "init"), shapes), nprocs=world, join=True)
