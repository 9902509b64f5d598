"""Unmerged LoRA adapters on the H100 kernels.

- The tailed GEMM (`mc_gemm_bf16_lora`, `ops.gemm(tail=(U, T))`) for epilogues 0, 1, 6 and 8 at both tile widths, on the
  geometries of test_gemm_epilogue_readout_gpu.py, R in {8, 16, 72, 136}, with NaN-poisoned margins around every operand and fenced
  outputs (test_kernel_bounds_gpu.py): each output is bit-equal to one untailed launch over [A | 0 | U | 0] and [B | 0 | T | 0]
  (each segment zero-padded to a multiple of 64 columns, the k-blocks the tailed launch walks), and with T = 0 value-equal to the
  plain launch (the extra zero products can only turn a -0 accumulator into +0).
- `magcache_flux_forward` with adapters against the oracle running the reference's scale / unscale statements
  (tests/flux_lora_ref.py) and fp64: a 12-step loop at reduced depth, the FLUX.1-dev 1024^2 shape with one double and one single
  block and rank-64 adapters on every covered target, zero lora_B (PEFT's initial state) value-equal to no adapters, and two GPUs
  token-sharded against one."""
import copy
import os
import sys
import tempfile
import time

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gemm_epilogue_readout_gpu import GEOMETRIES  # noqa: E402
from test_kernel_bounds_gpu import BF, check_fence, fenced  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPIS = ("MC_EPI_BIAS_BF16", "MC_EPI_BIAS_GELU_BF16", "MC_EPI_BIAS_GATE_RESID_BF16", "MC_EPI_BIAS_GATE_RESID_ADD_BF16")


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _bits(t):
    return t.contiguous().view(torch.int16)


def _pad64(k):
    return -(-k // 64) * 64


def _operand(rows, cols, g, scale=1.0):
    """A [rows, cols] bf16 view in a NaN buffer (8 rows before, 1 after, 8 columns each side)."""
    v, _ = fenced((rows, cols), BF, (8, 1, 8, 8))
    v.copy_((scale * torch.randn(rows, cols, device=DEV, generator=g)).to(BF))
    return v


# ------------------------------------------------------------------------------------------- tailed GEMM readout
def _gemm(epi, a, b, bias, gate, old, add, odd_ldo, tail=None):
    from magcache_b200 import _lib as L
    from magcache_b200 import ops
    M, N = a.shape[0], b.shape[0]
    if odd_ldo:
        out, obuf = fenced((M, N), BF, (8, 1, 8, 8), fill="fence", pitch=8 + N + 8 + 1 - (N % 2))
    else:
        out, obuf = fenced((M, N), BF, (1, 1, 8, 8), fill="fence")
    e = getattr(L, epi)
    if e in (L.MC_EPI_BIAS_GATE_RESID_BF16, L.MC_EPI_BIAS_GATE_RESID_ADD_BF16):
        out.copy_(old)
    kw = dict(addend=add, addend_row0=7) if e == L.MC_EPI_BIAS_GATE_RESID_ADD_BF16 else {}
    e = L.MC_EPI_BIAS_GATE_RESID_BF16 if kw else e
    ops.gemm(a, b, bias, e, out=out, gate=gate if e == L.MC_EPI_BIAS_GATE_RESID_BF16 else None, tail=tail, **kw)
    check_fence(out, obuf)
    return out.clone()


def _padded(x, u):
    """[x | 0 | u | 0], each segment zero-padded to a multiple of 64 columns (no NaN margins: the untailed launch reads only K)."""
    rows, K = x.shape
    R = u.shape[1]
    y = torch.zeros(rows, _pad64(K) + _pad64(R), dtype=BF, device=DEV)
    y[:, :K] = x
    y[:, _pad64(K):_pad64(K) + R] = u
    return y


@pytest.mark.parametrize("bn", [128, 256])
def test_tailed_gemm_readout(bn, monkeypatch):
    monkeypatch.setenv("MC_GEMM_BN", str(bn))
    g = torch.Generator(device=DEV).manual_seed(900 + bn)
    for geo, M, N, K, odd_ldo in GEOMETRIES:
        for R in (8, 16, 72, 136):
            a, b = _operand(M, K, g), _operand(N, K, g, 0.1)
            u, t = _operand(M, R, g), _operand(N, R, g, 0.1)
            bias = (torch.randn(N, device=DEV, generator=g)).to(BF).float()
            gate = (0.5 * torch.randn(N, device=DEV, generator=g)).to(BF).float()
            old = torch.randn(M, N, device=DEV, generator=g)
            old[torch.rand(M, N, device=DEV, generator=g) < 0.125] = -0.0
            old = old.to(BF)
            add, _ = fenced((M - 7, N), BF, (8, 1, 8, 8))
            add.copy_(torch.randn(M - 7, N, device=DEV, generator=g).to(BF))
            zero_t = _operand(N, R, g)
            zero_t.zero_()
            for epi in EPIS:
                what = (bn, geo, R, epi)
                got = _gemm(epi, a, b, bias, gate, old, add, odd_ldo, tail=(u, t))
                want = _gemm(epi, _padded(a, u), _padded(b, t), bias, gate, old, add, odd_ldo)
                bad = _bits(got) != _bits(want)
                assert not bool(bad.any()), (what, int(bad.sum()), bad.nonzero()[0].tolist())
                assert not bool(got.isnan().any()), what
                z = _gemm(epi, a, b, bias, gate, old, add, odd_ldo, tail=(u, zero_t))
                plain = _gemm(epi, a, b, bias, gate, old, add, odd_ldo)
                assert bool((z == plain).all()), what


def test_tailed_gemm_argument_checks():
    import ctypes

    from magcache_b200 import _lib as L
    a, b = torch.zeros(32, 64, dtype=BF, device=DEV), torch.zeros(32, 64, dtype=BF, device=DEV)
    out, add = torch.zeros(32, 32, dtype=BF, device=DEV), torch.zeros(32, 32, dtype=BF, device=DEV)
    u, t = torch.zeros(32, 24, dtype=BF, device=DEV), torch.zeros(32, 24, dtype=BF, device=DEV)
    p = lambda x: ctypes.c_void_p(x.data_ptr())  # noqa: E731
    E0, E8 = L.MC_EPI_BIAS_BF16, L.MC_EPI_BIAS_GATE_RESID_ADD_BF16

    def call(epi=E0, add_p=None, ld_add=0, row0=0, U=p(u), ldu=24, T=p(t), ldt=24, R=16):
        return L.lib.mc_gemm_bf16_lora(p(a), 64, p(b), 64, 32, 32, 64, None, epi, p(out), 32, None, add_p, ld_add, row0, U, ldu, T, ldt, R, None)

    assert call() == L.MC_OK and call(E8, p(add), 32, 0) == L.MC_OK
    torch.cuda.synchronize()
    bad = [dict(R=0), dict(R=12), dict(R=32), dict(ldu=20), dict(ldt=12), dict(U=None), dict(T=None),
           dict(U=ctypes.c_void_p(u.data_ptr() + 2)), dict(epi=E8), dict(epi=E8, add_p=p(add), ld_add=31), dict(add_p=p(add), ld_add=32),
           dict(epi=L.MC_EPI_BIAS_F32)]
    for kw in bad:
        assert call(**kw) == L.MC_ERR_INVALID, kw


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


class _WithScale:
    """A FLUX model called with return_dict=False and `joint_attention_kwargs={"scale": scale}`, its first output returned."""

    def __init__(self, m, scale):
        object.__setattr__(self, "_m", m)
        object.__setattr__(self, "_scale", scale)

    def __call__(self, *a):
        return self._m(*a, return_dict=False, joint_attention_kwargs={"scale": self._scale})[0]

    def __getattr__(self, name):
        return getattr(self._m, name)


def _models(model, steps, table, **kw):
    """(ours, bf16 oracle, fp64 oracle); the oracles run the reference's LoRA statements around their forward."""
    import flux_lora_ref as lref

    import magcache_b200 as mc
    from oracle import flux_ref as fr
    ours = _as("OurLG", model)
    mc.init_magcache_flux(ours, steps, mag_ratios=table, **kw)
    ref_m, m64 = _as("RefLG", model), _as("RefLG64", model, torch.float64)
    for m in (ref_m, m64):
        fr.install_magcache(type(m), table, steps, **kw)
        type(m).forward = lref.reference_lora(fr.magcache_forward)
    return ours, ref_m, m64


def test_flux_lora_forward_loop(monkeypatch):
    """12 steps at reduced depth (3 double, 3 single blocks, D = 256), 256 image and 77 text tokens, two rank-12 / rank-72 adapters
    on every covered target at scale 0.8: DESIGN §5's rule against the bf16 oracle and fp64, the controller attributes and every
    layer's `scaling` equal to the oracle's."""
    import flux_lora_ref as lref

    import magcache_b200 as mc
    from oracle import flux_ref as fr
    from test_fullshape_workloads_gpu import _forward_loop, _oracle_on_gpu
    _oracle_on_gpu(monkeypatch)
    n_txt, hw, steps = 77, (16, 16), 12
    model = _flux(3, 3, seed=5)
    lref.inject_lora(model, "all", ("a",), rank=12, seed=6)
    lref.inject_lora(model, "blocks", ("b",), rank=72, seed=7)
    lref.set_adapters(model, ["a", "b"], [1.0, 0.5])
    g = torch.Generator().manual_seed(5)
    hs = torch.randn(1, hw[0] * hw[1], 64, generator=g).bfloat16().to(DEV)
    enc = torch.randn(1, n_txt, 96, generator=g).bfloat16().to(DEV)
    pooled = torch.randn(1, 48, generator=g).bfloat16().to(DEV)
    img_ids, txt_ids = (t.to(DEV) for t in fr.make_ids(*hw, n_txt))
    ms = _models(model, steps, mc.tables()["flux_dev"])
    w = [_WithScale(m, 0.8) for m in ms]
    calls = []
    for i in range(steps):
        t, gd = torch.tensor([1.0 - i / steps], device=DEV), torch.tensor([4.0], device=DEV)
        x = hs * (1.0 - 0.03 * i)
        calls.append(((x, enc, pooled, t, img_ids, txt_ids, gd), (x, enc, pooled, t, img_ids, txt_ids, gd),
                      (x.double(), enc.double(), pooled.double(), t.double(), img_ids, txt_ids, gd.double())))
    skips = _forward_loop("flux lora", calls, *w, fr.exact, lambda m: m.previous_residual,
                          ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"),
                          check=lambda *a: (lref.scaling_state(ms[0]) == lref.scaling_state(ms[1])) or pytest.fail("scaling"))
    assert 0 < sum(skips) < steps, skips


def test_flux_zero_lora_b_equals_no_adapters():
    import flux_lora_ref as lref

    import magcache_b200 as mc
    from oracle import flux_ref as fr
    n_txt, hw = 77, (16, 16)
    model = _flux(2, 3, seed=6)
    g = torch.Generator().manual_seed(6)
    hs = torch.randn(1, hw[0] * hw[1], 64, generator=g).bfloat16().to(DEV)
    enc = torch.randn(1, n_txt, 96, generator=g).bfloat16().to(DEV)
    pooled = torch.randn(1, 48, generator=g).bfloat16().to(DEV)
    img_ids, txt_ids = (t.to(DEV) for t in fr.make_ids(*hw, n_txt))
    a = _as("OurZL0", model)
    adapted = copy.deepcopy(model)
    lref.inject_lora(adapted, "all", ("a",), rank=16, zero_b=True)
    b = _as("OurZL1", adapted)
    mc.init_magcache_flux(a, 28)
    mc.init_magcache_flux(b, 28)
    with torch.no_grad():
        for i in range(3):
            t, gd = torch.tensor([1.0 - i / 28], device=DEV), torch.tensor([3.5], device=DEV)
            x = a(hs, enc, pooled, t, img_ids, txt_ids, gd, return_dict=False)[0]
            y = b(hs, enc, pooled, t, img_ids, txt_ids, gd, return_dict=False)[0]
            assert bool((x == y).all()), i
            assert bool((a.previous_residual == b.previous_residual).all()), i
    assert b._mc_flux_engine.lora is not None  # the zero adapters did run, as tails


def test_flux_1024_lora_one_layer_forward(monkeypatch):
    """FLUX.1-dev at 1024 x 1024 (4096 image tokens, 512 text tokens of width 4096), one double and one single block at 3072 /
    24 heads, rank-64 adapters on every covered target: miss, miss, hit against the bf16 oracle and fp64."""
    import flux_lora_ref as lref

    from oracle import flux_ref as fr
    from test_fullshape_workloads_gpu import FLUX, _forward_loop, _need_device_memory, _oracle_on_gpu, _report
    _need_device_memory(40)
    _oracle_on_gpu(monkeypatch)
    t0 = time.time()
    fl = FLUX
    model = _flux(1, 1, fl["heads"], seed=21, text_dim=fl["text_dim"], pooled=fl["pooled"])
    lref.inject_lora(model, "all", ("a",), rank=64, seed=22)
    g = torch.Generator().manual_seed(21)
    hs = torch.randn(1, fl["n_img"], 64, generator=g).bfloat16().to(DEV)
    enc = torch.randn(1, fl["n_txt"], fl["text_dim"], generator=g).bfloat16().to(DEV)
    pooled = torch.randn(1, fl["pooled"], generator=g).bfloat16().to(DEV)
    img_ids, txt_ids = (t.to(DEV) for t in fr.make_ids(fl["h_tok"], fl["w_tok"], fl["n_txt"]))
    gd = torch.tensor([4.0], device=DEV)
    steps, table = 5, [1.0] + [0.98] * 4
    ms = _models(model, steps, table, thresh=10.0, K=3, retention_ratio=0.4)
    del model
    w = [_WithScale(m, 1.0) for m in ms]
    calls = []
    for tv in (1.0, 0.5, 0.25):
        t = torch.tensor([tv], device=DEV)
        a = (hs, enc, pooled, t, img_ids, txt_ids, gd)
        calls.append((a, a, (hs.double(), enc.double(), pooled.double(), t.double(), img_ids, txt_ids, gd.double())))
    skips = _forward_loop("flux 1024 lora", calls, *w, fr.exact, lambda m: m.previous_residual,
                          ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"))
    assert skips == [0, 0, 1], skips
    _report("flux 1024 lora forward", t0)


# ------------------------------------------------------------------------------------------- two GPUs
def _shard_worker(rank, world, initfile, results):
    import torch.distributed as dist

    import flux_lora_ref as lref
    import magcache_b200 as mc
    from oracle import flux_ref as fr
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", init_method=f"file://{initfile}", rank=rank, world_size=world, device_id=dev)
    try:
        g = torch.Generator().manual_seed(3)
        model = _flux(2, 2)
        lref.inject_lora(model, "all", ("a", "b"), rank=16, seed=4)
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
                                 torch.tensor([3.5], device=dev), return_dict=False, joint_attention_kwargs={"scale": 0.7})[0].clone())
            outs[name] = (got, m._mc_flux_engine)
        eng = outs["sharded"][1]
        errs = [rel_l2(a, b) for a, b in zip(outs["sharded"][0], outs["single"][0])]
        res_err = rel_l2(eng.res, outs["single"][1].res[eng.shard.start:eng.shard.stop])
        results[rank] = (errs, res_err, eng.n_img, eng.n_img_total)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_flux_lora_sharded_matches_single_gpu():
    """Token-sharded over two GPUs with adapters against one GPU, at test_shard_gpu.py's bound for the sharded FLUX engine."""
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
