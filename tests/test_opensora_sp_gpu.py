"""Open-Sora sequence parallelism on the H100: the head's frame-window entry point (`mc_opensora_head_frames`) and the 2-D peer push
(`mc_p2p_push2d`) on one device, then world-2 runs of the patched forwards, the RFlow sampler and the engine at the full 480p x 51-frame
shape, every rank's output bit-equal to the unsharded engine's. With one GPU both ranks share it (the P2P form then moves data within
the device through the same IPC windows); the collective form (MC_SHARD_P2P=0, NCCL) needs two."""
import ctypes
import os
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _head_inputs(B, T, H, W, D=1152, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    x = torch.randn(B * T * H * W, D, device=dev, generator=g).bfloat16()
    res = (0.1 * torch.randn(B * T * H * W, D, device=dev, generator=g)).bfloat16()
    mod = (0.2 * torch.randn(B, 2, D, device=dev, generator=g)).bfloat16().float()
    w = (torch.randn(32, D, device=dev, generator=g) / D ** 0.5).bfloat16()
    bias = (0.02 * torch.randn(32, device=dev, generator=g)).bfloat16().float()
    return x, res, mod, w, bias


@pytest.mark.parametrize("mode", ["plain", "hit", "step"])
@pytest.mark.parametrize("T,H,W,Hx,Wx,P", [(7, 6, 7, 12, 14, 2), (15, 30, 53, 60, 106, 2), (35, 6, 7, 11, 13, 4)])
def test_head_frame_window_writes_exactly_its_frames(mode, T, H, W, Hx, Wx, P):
    from magcache_b200 import ops, shard
    B = 2
    x, res, mod, w, bias = _head_inputs(B, T, H, W)
    S = H * W
    step = None
    if mode == "step":
        z = torch.randn(B // 2, 4, T, Hx, Wx, device="cuda")
        dt = torch.tensor([0.031], device="cuda")
        step = (z, 7.0, dt)
    r = res if mode == "hit" else None
    full = ops.opensora_head(x, mod, w, bias, (T, H, W), (T, Hx, Wx), res=r, step=step)
    for fr in shard.frame_position_shards(P, T, S)[0]:
        rows = [slice(b * T * S + fr.start * S, b * T * S + fr.stop * S) for b in range(B)]
        xl = torch.cat([x[s] for s in rows])
        rl = torch.cat([res[s] for s in rows]) if r is not None else None
        out = torch.full(full.shape, float("nan"), device="cuda")
        ops.opensora_head_frames(xl, mod, w, bias, (fr.n_local, H, W), (T, Hx, Wx), fr.start, out, res=rl, step=step)
        torch.cuda.synchronize()
        assert torch.equal(out[:, :, fr.start:fr.stop], full[:, :, fr.start:fr.stop]), (mode, fr.rank)
        assert out[:, :, :fr.start].isnan().all() and out[:, :, fr.stop:].isnan().all(), (mode, fr.rank)


def _push(copies, flags, epoch):
    from magcache_b200 import _lib
    arr = (_lib.Copy2D * max(len(copies), 1))(*[_lib.Copy2D(*c) for c in copies])
    flg = (ctypes.c_void_p * max(len(flags), 1))(*flags)
    return _lib.lib.mc_p2p_push2d(arr, len(copies), flg, len(flags), epoch, torch.cuda.current_stream().cuda_stream)


def test_push2d_places_every_block_and_publishes_its_flag():
    from magcache_b200 import _lib
    fence = 4096
    src = torch.arange(2 * 5 * 96, dtype=torch.int32, device="cuda").view(2, 5, 96)   # 2 samples, 5 runs, pitch 96 words
    dst = torch.full((fence + 2 * 5 * 40 + fence,), -7, dtype=torch.int32, device="cuda")
    body = dst[fence:fence + 2 * 5 * 40].view(2, 5, 40)
    epoch = torch.tensor([41], dtype=torch.int32, device="cuda")
    flag = torch.zeros(64, dtype=torch.int32, device="cuda")
    copies = [(body[b].data_ptr(), 40 * 4, src[b, :, 30:].data_ptr(), 96 * 4, 40 * 4, 5) for b in range(2)]
    assert _push(copies, [flag[3:4].data_ptr()], epoch.data_ptr()) == 0
    torch.cuda.synchronize()
    assert torch.equal(body, src[:, :, 30:70])
    assert (dst[:fence] == -7).all() and (dst[fence + 400:] == -7).all()
    assert flag[3].item() == 41 and (flag[:3] == 0).all() and (flag[4:] == 0).all()
    good = copies[0]
    for bad in [(good[0], good[1], good[2], good[3], -4, 5), (good[0], 39 * 4, good[2], good[3], 40 * 4, 5), (None, 160, good[2], 384, 160, 5)]:
        before = body.clone()
        assert _push([bad], [], epoch.data_ptr()) == _lib.MC_ERR_INVALID
        torch.cuda.synchronize()
        assert torch.equal(body, before)
    assert _push([good], [None], epoch.data_ptr()) == _lib.MC_ERR_INVALID
    assert _push([good], [flag.data_ptr()], None) == _lib.MC_ERR_INVALID


# ---- world-2 runs ---------------------------------------------------------------------------------------------------------------
def _full_engine_case(rank, world, dev, group):
    """The full STDiT3 (random weights) at 480p x 51 frames (T = 15 latent frames, 60 x 106, B = 2): one miss and one hit."""
    from magcache_b200 import opensora as os_mod
    w = os_mod.random_opensora_weights(dev)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 4, 15, 60, 106, generator=g).to(dev)
    y = torch.randn(2, 1, 300, 4096, generator=g).to(dev)
    mask = torch.ones(2, 300, dtype=torch.long, device=dev)
    mask[:, 200:] = 0
    args = (torch.tensor([700.0, 700.0], device=dev), y, mask, torch.tensor([24.0], device=dev), torch.tensor([480.0], device=dev),
            torch.tensor([854.0], device=dev))
    one = os_mod.OpenSoraEngine(w)
    outs1 = []
    for kind in ("miss", "hit"):
        one.stage_inputs(x, *args)
        outs1.append(one.forward(kind))
    torch.cuda.synchronize(dev)
    del one
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    sp = os_mod.OpenSoraEngine(w, sp_world=world, sp_rank=rank, sp_group=group)
    for kind, o1 in zip(("miss", "hit"), outs1):
        sp.stage_inputs(x, *args)
        o = sp.forward(kind)
        assert torch.equal(o, o1), ("full shape", kind, float((o - o1).abs().max()))
    print(f"rank {rank}: full-shape peak memory {torch.cuda.max_memory_allocated(dev) / 2**30:.2f} GiB", flush=True)
    sp.switch.close()


def _worker(rank, world, initfile, p2p):
    import opensora_ref as R
    import opensora_sp_cases as C
    from magcache_b200 import shard
    os.environ["MC_SHARD_P2P"] = "1" if p2p else "0"
    ngpu = torch.cuda.device_count()
    dev = torch.device("cuda", rank % ngpu)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo" if p2p else "nccl", init_method=f"file://{initfile}", rank=rank, world_size=world,
                            **({} if p2p else dict(device_id=dev)))
    try:
        B = 2
        for cfg, (T, Hx, Wx) in (("tiny", (7, 12, 14)), ("tiny", (15, 12, 14)), ("tiny", (35, 11, 13)), ("wide", (15, 11, 13))):
            S = (-(-Hx // 2)) * (-(-Wx // 2))
            fr = shard.frame_position_shards(world, T, S)[0][rank]
            cy = R.CONFIGS[cfg]["caption_channels"]
            for kind, thresh, n in (("magcache", None, 10), ("teacache", 0.1, 10), ("teacache", 10.0, 6), ("plain", None, 2)):
                sp, one = C.build(kind, cfg=cfg, thresh=thresh, device=dev)
                C.enable(sp, rank, world)
                got = C.calls(sp, kind, n, B, T, Hx, Wx, dev, cy=cy)
                want = C.calls(one, kind, n, B, T, Hx, Wx, dev, cy=cy)
                C.compare(got, want, T, fr.start, fr.stop, (cfg, T, kind, thresh, p2p))
                assert sp._mc_opensora_engine.switch.p2p == p2p
                sp._mc_opensora_engine.switch.close()
            if cfg == "tiny":
                sp, one = C.build("magcache", cfg=cfg, device=dev)
                C.enable(sp, rank, world)
                seen, out = C.sample(sp, T, Hx, Wx, dev)
                seen1, out1 = C.sample(one, T, Hx, Wx, dev)
                assert torch.equal(out, out1) and all(torch.equal(a, b) for a, b in zip(seen, seen1)), (T, "sampler", p2p)
                sp._mc_opensora_engine.switch.close()
        if p2p:
            _full_engine_case(rank, world, dev, None)
        torch.cuda.synchronize(dev)
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("p2p", [True, False], ids=["p2p", "collective"])
def test_world2_bit_equal_to_one_engine(p2p):
    if not p2p and torch.cuda.device_count() < 2:
        pytest.skip("the NCCL form needs two GPUs")
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_worker, args=(2, os.path.join(d, "init"), p2p), nprocs=2, join=True)
