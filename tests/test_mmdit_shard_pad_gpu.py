"""The pad rule of the token-sharded MMDiT engines on the H100: image token counts N that do not divide by the world size P, so the
last rank owns fewer rows and its key segment is short, with the replicated text rows written locally right behind row N.

* One GPU: `mc_attn_fwd_ex` with seg_rows = ceil(N/P), a short last segment, a text tail, each rank's `first_key_row` and every
  flag published before the launch (no tile can wait), against the unsegmented `mc_attn_fwd` on the same keys and fp64, into
  fenced outputs.
* The peer-to-peer exchange's gathered key rows, with its ranks as processes sharing whatever GPUs there are (gloo carries only the
  IPC handles; nothing on the device waits for a peer): exactly [all image rows | text rows], and every flag a key tile can
  touch is one a rank publishes or one that is permanently set.
* Two GPUs (skipped below): FLUX at 45 x 91 latent tokens and HunyuanVideo at a 720 x 720 bucket's grid (33 x 45 x 45), reduced
  depth and full width, over the peer-to-peer and the NCCL exchange, each rank against the single-GPU engine."""
import math
import os
import sys
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_bounds_gpu import _attn64, _randn, check_fence, fenced  # noqa: E402

DEV = "cuda"
BF = torch.bfloat16


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


# ------------------------------------------------------------------------------------------- kernel, one GPU
@pytest.mark.parametrize("N,P,n_txt", [(4095, 2, 512), (4095, 8, 512), (1001, 4, 77), (405, 2, 11), (10, 4, 24)])
def test_flag_gated_short_last_segment_then_tail(N, P, n_txt, monkeypatch):
    """Keys [N image rows | n_txt text rows]: segments of ceil(N/P) rows, the last one short, then the tail, whose first rows
    fall in segment P - 1. The flag table (with margins) is at the epoch before the launch. For every rank's first_key_row: the
    flag-gated result is bit-equal to the same rotated order without flags, and it and the unsegmented kernel both meet the fp64
    bounds of test_kernel_bounds_gpu.py; no store leaves the output view."""
    from magcache_b200 import ops
    heads, scale, Lq = 2, 1.0 / math.sqrt(128), 300
    W, Lk = heads * 128, N + n_txt
    seg = -(-N // P)
    assert N - (P - 1) * seg < seg  # a short last segment
    n_flags = -(-Lk // seg)          # every segment index a key tile can touch
    epoch = 5
    fbuf = torch.full((n_flags + 128,), epoch, dtype=torch.int32, device=DEV)  # 64 published flags of margin either side
    flags = dict(seg_flags=fbuf[64:64 + n_flags], seg_epoch=torch.full((1,), epoch, dtype=torch.int32, device=DEV), seg_rows=seg)
    g = torch.Generator(device=DEV).manual_seed(N + P)
    q, _ = fenced((Lq, W), BF, (0, 0, 8, 8))
    k, _ = fenced((Lk, W), BF, (0, 128, 8, 8))
    v, _ = fenced((Lk, W), BF, (0, 128, 8, 8))
    q.copy_(_randn((Lq, W), g))
    k.copy_(_randn((Lk, W), g))
    v.copy_(_randn((Lk, W), g))
    want = _attn64(q, k, v, heads, scale)

    def run(**kw):
        out, obuf = fenced((Lq, W), BF, (1, 1, 8, 8), fill="fence")
        ops.attention(q, k, v, heads, scale=scale, out=out, **kw)
        check_fence(out, obuf)
        err = (out.double() - want).abs()
        assert bool(torch.isfinite(out.float()).all()) and float(err.max()) < 2e-2 and float(err.mean()) < 2e-3, (kw.keys(), float(err.max()))
        return out

    plain = run()
    for r in range(P):
        got = run(first_key_row=r * seg, **flags)
        assert float((got.float() - plain.float()).abs().max()) < 2e-2, r
        monkeypatch.setenv("MC_ATTN_KERNEL", "3")  # the ungated rotated order on the same 176-key tiles
        assert torch.equal(got, run(first_key_row=r * seg)), (N, P, r, "flag-gated result differs from the ungated one")
        monkeypatch.delenv("MC_ATTN_KERNEL")
    torch.cuda.synchronize()
    assert bool((fbuf == epoch).all())


# ------------------------------------------------------------------------------------------- P2P exchange layout
def _p2p_worker(rank, world, initfile, results):
    import torch.distributed as dist

    from magcache_b200.shard import P2PExchange, TokenShard
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=f"file://{initfile}", rank=rank, world_size=world)
    try:
        out = []
        width = 64
        for extra, n in [(e, n) for e in (37, 0) for n in (8 * world, 8 * world - 1, 7 * world + 1)]:  # pad 0, 1 and P - 1; no tail (Wan)
            sh = TokenShard(rank, world, n)
            g = torch.Generator().manual_seed(n)
            rows = torch.randn(n, width, generator=g).bfloat16().to(dev)
            xch = P2PExchange(sh, width, (1,), dev, extra_rows=extra)
            flags = xch.window[:xch.FLAG_BYTES].view(torch.int32)
            for rep in range(4):
                i = rep % 2
                tail = torch.randn(extra, width, generator=g).bfloat16().to(dev)  # replicated: every rank draws the same
                xch.own_rows(i).copy_(sh.rows(rows) * (rep + 1))
                xch.tail_rows(i).copy_(tail)
                xch.begin(i)
                torch.cuda.synchronize(dev)
                dist.barrier()  # every peer's pushes into this rank's buffer have completed
                kv, kw = xch.keys_values(i)
                assert kv.shape == (n + extra, width)
                ok = torch.equal(kv, torch.cat([rows * (rep + 1), tail])) and kw["seg_rows"] == sh.n_slots and kw["first_key_row"] == sh.start
                ep = int(xch.epochs[0])
                segs = sorted({r // sh.n_slots for r in range(n + extra)})
                fl = flags[64 * i:64 * i + 64].tolist()
                covered = all((fl[s] == ep) if s < world else (fl[s] == 0x7FFFFFFF) for s in segs)
                out.append((n, sh.pad, rep, ok, covered))
                dist.barrier()  # nobody writes the next round's rows into a buffer a peer is still reading
            xch.join()
            torch.cuda.synchronize(dev)
            dist.barrier()
            xch.close()
            dist.barrier()
        results[rank] = out
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_p2p_exchange_keys_are_image_rows_then_text(world):
    """Each rank pushes only its valid rows, so the last rank's pad slots [N, n_padded) of a peer's buffer keep the peer's own text
    rows: gathered keys == cat(all image rows, text rows) bit for bit, for pad 0 and pad > 0, over both buffers twice; and with no
    tail rows (the Wan engines' exchange)."""
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        results = mp.get_context("spawn").Manager().dict()
        mp.spawn(_p2p_worker, args=(world, os.path.join(d, "init"), results), nprocs=world, join=True)
        for r in range(world):
            got = results[r]
            assert {p for _, p, *_ in got} == {0, 1, world - 1}, got
            assert all(ok for *_, ok, _ in got), ("gathered rows", got)
            assert all(cov for *_, cov in got), ("flag coverage", got)


# ------------------------------------------------------------------------------------------- engines, two GPUs
def _engine_worker(rank, world, initfile, results, family):
    import copy

    import torch.distributed as dist

    import magcache_b200 as mc
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", init_method=f"file://{initfile}", rank=rank, world_size=world, device_id=dev)
    try:
        g = torch.Generator().manual_seed(3)
        if family == "flux":  # 720 x 1456: 45 x 91 = 4095 latent tokens, full width, one double and one single block
            from oracle import flux_ref as fr
            model = fr.FluxTransformer2DModel(num_layers=1, num_single_layers=1).init_synthetic(0)
            hs, enc, pooled = (torch.randn(1, 4095, 64, generator=g).bfloat16().to(dev), torch.randn(1, 512, 4096, generator=g).bfloat16().to(dev),
                               torch.randn(1, 768, generator=g).bfloat16().to(dev))
            img_ids, txt_ids = (t.to(dev) for t in fr.make_ids(45, 91, 512))

            def call(m, i):
                return m(hs * (1 - 0.05 * i), enc, pooled, torch.tensor([1.0 - i / 6], device=dev), img_ids, txt_ids, torch.tensor([3.5], device=dev),
                         return_dict=False)[0]

            def install(m):
                mc.init_magcache_flux(m, 6, thresh=10.0, K=2, retention_ratio=0.34)  # miss miss hit hit miss miss
            eng_attr, n_img = "_mc_flux_engine", 4095
        else:  # 720 x 720, 129 frames: 33 x 45 x 45 = 66 825 latent tokens, full width, one double and one single block
            from oracle import hunyuan_ref as hr
            model = hr.HYVideoDiffusionTransformer(mm_double_blocks_depth=1, mm_single_blocks_depth=1).init_synthetic(0)
            grid = (33, 45, 45)
            x = torch.randn(1, 16, grid[0], 2 * grid[1], 2 * grid[2], generator=g).bfloat16().to(dev)
            txt, pooled = torch.randn(1, 256, 4096, generator=g).bfloat16().to(dev), torch.randn(1, 768, generator=g).bfloat16().to(dev)
            mask = torch.zeros(1, 256, dtype=torch.long, device=dev)
            mask[0, :97] = 1
            cos, sin = (t.to(dev) for t in hr.rope_cos_sin(grid))

            def call(m, i):
                return m(x * (1 - 0.05 * i), torch.tensor([900.0 - 100 * i], device=dev), txt, mask, pooled, cos, sin, torch.tensor([6000.0], device=dev),
                         return_dict=False)

            def install(m):
                mc.init_magcache_hunyuan(m, 6, thresh=10.0, K=2, retention_ratio=0.34, mag_ratios=[1.0] * 6)
            eng_attr, n_img = "_mc_hunyuan_engine", 66825
        res = {}
        single = None
        for mode in ("single", "p2p", "collective"):
            os.environ["MC_SHARD_P2P"] = "0" if mode == "collective" else "1"
            m = copy.deepcopy(model).to(dev)
            m.__class__ = type("M_" + mode, (m.__class__,), {})
            install(m)
            if mode != "single":
                mc.enable_token_shard(m, rank, world)
            with torch.no_grad():
                seq = [call(m, i).clone() for i in range(6)]
            eng = getattr(m, eng_attr)
            torch.cuda.synchronize()
            dist.barrier()
            if mode == "single":
                single = (seq, eng.res.clone())
                continue
            sh = eng.shard
            errs = [rel_l2(a, b) for a, b in zip(seq, single[0])]
            res[mode] = (errs, rel_l2(eng.res, single[1][sh.start:sh.stop]), eng.n_img, eng.n_img_total, sh.pad, type(eng.xch).__name__)
            del m, eng
        results[rank] = (res, n_img)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("family", ["flux", "hunyuan"])
def test_padded_mmdit_engine_matches_single_gpu(family):
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        results = mp.Manager().dict()
        mp.spawn(_engine_worker, args=(2, os.path.join(d, "init"), results, family), nprocs=2, join=True)
        assert set(results.keys()) == {0, 1}
        for r in (0, 1):
            res, n_img = results[r]
            assert res["p2p"][5] == "P2PExchange" and res["collective"][5] == "CollectiveExchange"
            for mode, (errs, res_err, n_loc, n_tot, pad, _) in res.items():
                assert pad == 1 and n_tot == n_img and n_loc == (n_img + 1) // 2 - r, (mode, r, n_loc)
                # the bounds of test_shard_gpu.py::test_sharded_mmdit_engine_matches_single_gpu
                assert len(errs) == 6 and max(errs) < 2e-2, (mode, errs)
                assert res_err < 3e-2, (mode, res_err)
