"""FLUX IP-Adapter image prompts on the H100: `mc_ip_attn` read out against fp64 with poisoned input margins and fenced outputs, the
patched forward against the oracle (tests/flux_ip_adapter_ref.py) and fp64 at reduced depth and at the FLUX.1-dev 1024^2 shape
with an XLabs-shaped adapter (768 -> 16 x 4096), and a two-GPU token-sharded run against one GPU."""
import copy
import math
import os
import tempfile
import time

import pytest
import torch

from test_kernel_bounds_gpu import check_fence, fenced

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF = torch.bfloat16


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


# ------------------------------------------------------------------------------------------- kernel readout
def _readout_case(rows, heads, ldq_twice, n_keys, scales, seed):
    """q in the q half of a q|k buffer (the k half NaN) or alone, NaN rows past the end; K random, V rows unit vectors so that
    key j of adapter a writes its probability to column off_a + j of every head (off_a: the keys of the adapters before a)."""
    from magcache_b200 import ops
    g = torch.Generator().manual_seed(seed)
    D = heads * 128
    N = sum(n_keys)
    assert N <= 128
    qv, qbuf = fenced((rows, D), BF, margin=(0, 5, 0, D if ldq_twice else 0))
    qv.copy_(torch.randn(rows, D, generator=g).to(BF))
    kv, kvbuf = fenced((N, 2 * D), BF, margin=(0, 3, 0, 8))
    kv[:, :D] = torch.randn(N, D, generator=g).to(BF)
    v = torch.zeros(N, heads, 128)
    v[torch.arange(N), :, torch.arange(N)] = 1.0
    kv[:, D:] = v.reshape(N, D).to(BF)
    w = (1.0 + 0.2 * torch.randn(128, generator=g)).to(BF).float().to(DEV)
    out, obuf = fenced((rows, D), BF, margin=(2, 2, 8, 8), fill="fence")
    q_before = qbuf.clone()
    ops.ip_attention(qv, w, heads, kv, n_keys, scales, out=out)
    torch.cuda.synchronize()
    check_fence(out, obuf)
    assert torch.equal(qbuf.view(torch.int16), q_before.view(torch.int16)), "q is read only"
    qn = qv.clone()
    ops.rmsnorm_head_rope_(qn, w, heads)  # the header's qn: the same per-head RMSNorm code
    return qn.double().cpu(), kv[:, :D].double().cpu(), out.cpu()


@pytest.mark.parametrize("rows,heads,ldq_twice,n_keys", [(4096, 24, True, (16,)), (333, 24, False, (4, 16, 32)), (65, 3, True, (32, 4)),
                                                          (1, 3, False, (16,)), (130, 24, True, (4,)), (77, 3, True, (16, 16, 16))])
def test_ip_attention_readout_is_p_within_the_header_bound(rows, heads, ldq_twice, n_keys):
    """Each output of a key is that key's probability: |out - p| <= 1.01 * 2^-7 * p + 2^-24 against fp64 from qn, for scales that
    are powers of two (the scale product is exact); every column no key writes is +0."""
    scales = [(1.0, -0.5, 2.0)[a % 3] for a in range(len(n_keys))]
    qn, k, out = _readout_case(rows, heads, ldq_twice, list(n_keys), scales, seed=rows + heads)
    D, off = heads * 128, 0
    o = out.double().view(rows, heads, 128)
    covered = torch.zeros(128, dtype=torch.bool)
    for n, sc in zip(n_keys, scales):
        kh = k[off:off + n].view(n, heads, 128)
        s = torch.einsum("rhd,nhd->rhn", qn.view(rows, heads, 128), kh) / math.sqrt(128)
        p = torch.softmax(s, -1)
        got = o[:, :, off:off + n] / sc
        bound = 1.01 * 2.0 ** -7 * p + 2.0 ** -24
        err = (got - p).abs()
        assert bool((err <= bound).all()), f"adapter keys [{off}, {off + n}): worst {float((err / bound).max()):.3f} of the bound"
        covered[off:off + n] = True
        off += n
    rest = out.view(rows, heads, 128)[:, :, ~covered]
    assert bool((rest.view(torch.int16) == 0).all()), "columns no key writes must be +0"


def test_ip_attention_scale_zero_is_plus_zero():
    rows, heads = 200, 24
    _, _, out = _readout_case(rows, heads, True, [16, 4], [0.0, 0.0], seed=3)
    assert bool((out.view(torch.int16) == 0).all())
    _, _, out = _readout_case(rows, heads, True, [16], [-0.0], seed=4)
    assert bool((out.view(torch.int16) == 0).all())


def test_ip_attention_matches_the_emulation_chain():
    """Random V at the FLUX shape with three adapters and mixed scales: the kernel against the chain in torch fp32 (P unrounded) within
    a few bf16 ulps of each adapter's output."""
    import flux_ip_adapter_ref as ipr
    from magcache_b200 import ops
    g = torch.Generator().manual_seed(8)
    heads, rows, n_keys, scales = 24, 1000, [16, 4, 32], [0.7, -1.3, 0.25]
    D = heads * 128
    q = torch.randn(rows, 2 * D, generator=g).to(BF)
    kv = torch.randn(sum(n_keys), 2 * D, generator=g).to(BF)
    w = (1.0 + 0.2 * torch.randn(128, generator=g)).to(BF).float()
    got = ops.ip_attention(q.to(DEV)[:, :D], w.to(DEV), heads, kv.to(DEV), n_keys, scales).cpu()
    want = ipr.ip_attention(q[:, :D], w, heads, kv, n_keys, scales)
    d = (got.float() - want.float()).abs()
    assert float(d.max()) <= 4 * 2.0 ** -8 * float(want.float().abs().max()), float(d.max())
    assert rel_l2(got, want) < 4e-3


def test_ip_attention_limits():
    from magcache_b200 import _lib as L
    from magcache_b200 import ops
    heads, D = 3, 384
    q = torch.zeros(16, D, dtype=BF, device=DEV)
    w = torch.ones(128, device=DEV)
    kv = torch.zeros(400, 2 * D, dtype=BF, device=DEV)
    with pytest.raises(NotImplementedError):
        ops.ip_attention(q, w, heads, kv, [385, 15], [1.0, 1.0])
    with pytest.raises(NotImplementedError):
        ops.ip_attention(q, w, heads, kv[:9], [1] * 9, [1.0] * 9)
    ops.ip_attention(q, w, heads, kv[:384], [384], [1.0])  # the largest staging that fits
    import ctypes
    p = lambda t: t.data_ptr()  # noqa: E731
    for n_keys in ([385], [369, 1], [0]):
        nk, sc = (ctypes.c_int32 * len(n_keys))(*n_keys), (ctypes.c_float * len(n_keys))(*([1.0] * len(n_keys)))
        rc = L.lib.mc_ip_attn(p(q), D, 16, heads, p(w), 1e-6, p(kv), 2 * D, nk, sc, len(n_keys), p(q), D, None)
        assert rc == L.MC_ERR_INVALID, n_keys
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------- forwards
def _flux(num_layers=2, num_single_layers=3, heads=2, seed=0, text_dim=96, pooled=48):
    from oracle import flux_ref as fr
    return fr.FluxTransformer2DModel(in_channels=64, num_layers=num_layers, num_single_layers=num_single_layers, num_attention_heads=heads,
                                     joint_attention_dim=text_dim, pooled_projection_dim=pooled).init_synthetic(seed)


def _as(name, model, dtype=None):
    m = copy.deepcopy(model).to(DEV)
    if dtype is not None:
        m = m.to(dtype)
    m.__class__ = type(name, (m.__class__,), {})
    return m


class _WithEmbeds:
    """A FLUX model called with return_dict=False and the call's image-prompt embeds, its first output returned."""

    def __init__(self, m, embeds):
        object.__setattr__(self, "_m", m)
        object.__setattr__(self, "embeds", embeds)

    def __call__(self, *a):
        return self._m(*a, return_dict=False, joint_attention_kwargs={"ip_adapter_image_embeds": self.embeds})[0]

    def __getattr__(self, name):
        return getattr(self._m, name)


def _three(model, steps, table, **kw):
    """(ours, bf16 oracle, fp64 oracle) on the device, the oracles running the reference's ip-adapter statements."""
    import flux_ip_adapter_ref as ipr
    import magcache_b200 as mc
    from oracle import flux_ref as fr
    ours = _as("OurIPG", model)
    mc.init_magcache_flux(ours, steps, mag_ratios=table, **kw)
    ref_m, m64 = _as("RefIPG", model), _as("RefIPG64", model, torch.float64)
    for m in (ref_m, m64):
        fr.install_magcache(type(m), table, steps, **kw)
        type(m).forward = ipr.reference_ip(fr.magcache_forward)
    return ours, ref_m, m64


def test_flux_ip_adapter_forward_loop(monkeypatch):
    """12 steps at reduced depth (3 double, 3 single blocks, D = 256), 256 image and 77 text tokens, two adapters (16 and 2 x 4
    image-prompt tokens) at per-block scales: DESIGN §5's rule against the bf16 oracle and fp64 on every output and residual."""
    import flux_ip_adapter_ref as ipr
    import magcache_b200 as mc
    from oracle import flux_ref as fr
    from test_fullshape_workloads_gpu import _forward_loop, _oracle_on_gpu
    _oracle_on_gpu(monkeypatch)
    n_txt, hw, steps = 77, (16, 16), 12
    model = ipr.load_ip_adapter(_flux(3, 3, seed=5), 2, [16, 4], seed=6)
    ipr.set_ip_adapter_scale(model, [[1.0, 0.5], [0.8, -0.6], [1.2, 1.0]])
    g = torch.Generator().manual_seed(5)
    hs = torch.randn(1, hw[0] * hw[1], 64, generator=g).bfloat16().to(DEV)
    enc = torch.randn(1, n_txt, 96, generator=g).bfloat16().to(DEV)
    pooled = torch.randn(1, 48, generator=g).bfloat16().to(DEV)
    img_ids, txt_ids = (t.to(DEV) for t in fr.make_ids(*hw, n_txt))
    embeds = [e.to(DEV) for e in ipr.make_embeds(2, 1)]
    embeds[1] = torch.cat([embeds[1], -embeds[1]], 1)  # two images for the second adapter
    ours, ref_m, m64 = _three(model, steps, mc.tables()["flux_dev"], thresh=0.24, K=5, retention_ratio=0.1)
    w = [_WithEmbeds(m, embeds) for m in (ours, ref_m, m64)]
    calls = []
    for i in range(steps):
        t, gd = torch.tensor([1.0 - i / steps], device=DEV), torch.tensor([4.0], device=DEV)
        x = hs * (1.0 - 0.03 * i)
        calls.append(((x, enc, pooled, t, img_ids, txt_ids, gd),) * 2 +
                     ((x.double(), enc.double(), pooled.double(), t.double(), img_ids, txt_ids, gd.double()),))
    skips = _forward_loop("flux ip-adapter", calls, *w, fr.exact, lambda m: m.previous_residual,
                          ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"))
    assert 0 < sum(skips) < steps, skips


def test_flux_1024_ip_adapter_one_layer_forward(monkeypatch):
    """FLUX.1-dev at 1024 x 1024 (4096 image tokens, 512 text tokens), one double and one single block at 3072 / 24 heads, with an
    XLabs-shaped adapter (768-wide embeds -> 16 tokens of 4096): miss, miss, hit against the bf16 oracle and fp64."""
    import flux_ip_adapter_ref as ipr
    from oracle import flux_ref as fr
    from test_fullshape_workloads_gpu import FLUX, _forward_loop, _need_device_memory, _oracle_on_gpu, _report
    _need_device_memory(40)
    _oracle_on_gpu(monkeypatch)
    t0 = time.time()
    fl = FLUX
    model = ipr.load_ip_adapter(_flux(1, 1, fl["heads"], seed=21, text_dim=fl["text_dim"], pooled=fl["pooled"]), 1, 16, emb_dim=768,
                                C=4096, seed=22)
    g = torch.Generator().manual_seed(21)
    hs = torch.randn(1, fl["n_img"], 64, generator=g).bfloat16().to(DEV)
    enc = torch.randn(1, fl["n_txt"], fl["text_dim"], generator=g).bfloat16().to(DEV)
    pooled = torch.randn(1, fl["pooled"], generator=g).bfloat16().to(DEV)
    img_ids, txt_ids = (t.to(DEV) for t in fr.make_ids(fl["h_tok"], fl["w_tok"], fl["n_txt"]))
    gd = torch.tensor([4.0], device=DEV)
    steps, table = 5, [1.0] + [0.98] * 4
    ours, ref_m, m64 = _three(model, steps, table, thresh=10.0, K=3, retention_ratio=0.4)
    del model
    embeds = [e.to(DEV) for e in ipr.make_embeds(1, 1, emb_dim=768, seed=23)]
    w = [_WithEmbeds(m, embeds) for m in (ours, ref_m, m64)]
    calls = []
    for tv in (1.0, 0.5, 0.25):
        t = torch.tensor([tv], device=DEV)
        a = (hs, enc, pooled, t, img_ids, txt_ids, gd)
        calls.append((a, a, (hs.double(), enc.double(), pooled.double(), t.double(), img_ids, txt_ids, gd.double())))
    skips = _forward_loop("flux 1024 ip-adapter", calls, *w, fr.exact, lambda m: m.previous_residual,
                          ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"))
    assert skips == [0, 0, 1], skips
    _report("flux 1024 ip-adapter forward", t0)


# ------------------------------------------------------------------------------------------- two GPUs
def _shard_worker(rank, world, initfile, results):
    import torch.distributed as dist

    import flux_ip_adapter_ref as ipr
    import magcache_b200 as mc
    from oracle import flux_ref as fr
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", init_method=f"file://{initfile}", rank=rank, world_size=world, device_id=dev)
    try:
        g = torch.Generator().manual_seed(3)
        model = ipr.load_ip_adapter(_flux(2, 2), 2, [16, 4], seed=4)
        embeds = [e.to(dev) for e in ipr.make_embeds(2, 2)]
        hs, enc, pooled = (torch.randn(1, 1152, 64, generator=g).bfloat16().to(dev), torch.randn(1, 24, 96, generator=g).bfloat16().to(dev),
                           torch.randn(1, 48, generator=g).bfloat16().to(dev))
        img_ids, txt_ids = (t.to(dev) for t in fr.make_ids(32, 36, 24))
        outs = {}
        for name in ("single", "sharded"):
            m = copy.deepcopy(model).to(dev)
            m.__class__ = type("M_" + name, (m.__class__,), {})
            mc.init_magcache_flux(m, 6, thresh=10.0, K=2, retention_ratio=0.34)  # miss miss hit hit miss miss
            if name == "sharded":
                mc.enable_token_shard(m, rank, world)
            got = []
            with torch.no_grad():
                for i in range(6):
                    got.append(m(hs * (1 - 0.05 * i), enc, pooled, torch.tensor([1.0 - i / 6], device=dev), img_ids, txt_ids,
                                 torch.tensor([3.5], device=dev), return_dict=False,
                                 joint_attention_kwargs={"ip_adapter_image_embeds": embeds})[0].clone())
            outs[name] = (got, m._mc_flux_engine)
        eng = outs["sharded"][1]
        errs = [rel_l2(a, b) for a, b in zip(outs["sharded"][0], outs["single"][0])]
        res_err = rel_l2(eng.res, outs["single"][1].res[eng.shard.start:eng.shard.stop])
        results[rank] = (errs, res_err, eng.n_img, eng.n_img_total)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_flux_ip_adapter_sharded_matches_single_gpu():
    """Token-sharded over two GPUs (each rank projects the replicated embeds and attends its own image rows, no exchange) against
    one GPU, at the sharded FLUX engine's bound without an adapter (its joint attention orders the keys differently)."""
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        results = mp.Manager().dict()
        mp.spawn(_shard_worker, args=(2, os.path.join(d, "init"), results), nprocs=2, join=True)
        assert set(results.keys()) == {0, 1}
        for r in (0, 1):
            errs, res_err, n_loc, n_tot = results[r]
            assert n_loc * 2 == n_tot == 1152
            assert len(errs) == 6 and max(errs) < 2e-2, errs
            assert res_err < 3e-2, res_err
