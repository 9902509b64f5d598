"""FLUX ControlNet residuals on the H100 kernels.

- Epilogue 8 (MC_EPI_BIAS_GATE_RESID_ADD_BF16, `mc_gemm_bf16_add`) read out over every finite bf16 value through B, on the
  geometries of test_gemm_epilogue_readout_gpu.py (ragged rows / columns, odd ldo, K tails), with NaN-poisoned operand margins and
  fenced outputs (test_kernel_bounds_gpu.py). The addend lies in a NaN-poisoned buffer: rows before its first row, columns past
  N and, with an odd ld_add, the padding column. Each output is bit-equal to the header's chain in eager torch, and the rows below
  add_row0 are bit-equal to an epilogue-6 launch on the same inputs (no addend read, no 0 added: -0 stays -0).
- `magcache_flux_forward` with samples against the oracle running the reference's ControlNet statements (tests/flux_controlnet_ref.py)
  and fp64, at reduced depth and at the FLUX.1-dev 1024^2 shape with one double and one single block (the chunked-attention oracle of
  test_fullshape_workloads_gpu.py); zero samples leave the output unchanged; two GPUs token-sharded against one."""
import copy
import os
import sys
import tempfile
import time

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gemm_epilogue_readout_gpu import GEOMETRIES, SCALED_A, SWEEP_SIZE, _launch, _side_vector, bf16_sweep, epilogue_model  # noqa: E402
from test_kernel_bounds_gpu import BF, check_fence, fenced  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPI6 = "MC_EPI_BIAS_GATE_RESID_BF16"


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------- epilogue 8 readout
def _addend(rows, N, g, odd_ld, unaligned):
    """A [rows, N] bf16 addend inside a NaN buffer (8 rows before it, columns past N, the odd pitch's padding column); with
    `unaligned` the view starts one element (2 bytes) past a 16-byte boundary, after a NaN column. Values: normal, 1 in 8 set to -0."""
    shift = 1 if unaligned else 0
    pitch = None
    if odd_ld:
        pitch = 8 + N + shift + 8 + 1 - ((N + shift) % 2)
    v, buf = fenced((rows, N + shift), BF, (8, 1, 8, 8), pitch=pitch)
    v = v[:, shift:]
    r = torch.randn(rows, N, device=DEV, generator=g)
    r[torch.rand(rows, N, device=DEV, generator=g) < 0.125] = -0.0
    v.copy_(r.to(BF))
    assert (v.stride(0) % 2 == 1) == odd_ld and (v.data_ptr() % 4 != 0) == unaligned
    return v


def _launch8(M, N, K, odd_ldo, a_val, b_vals, bias, gate, old, add, row0):
    """`_launch` of the readout module with the addend: epilogue 8 through ops.gemm(addend=...)."""
    from magcache_b200 import _lib as L
    from magcache_b200 import ops
    a, _ = fenced((M, K), BF, (0, 1, 8, 8))
    a.zero_()
    rows = torch.arange(M, device=DEV)
    a[rows, rows % K] = a_val
    b, _ = fenced((N, K), BF, (0, 1, 8, 8))
    b.copy_(b_vals)
    if odd_ldo:
        out, obuf = fenced((M, N), BF, (8, 1, 8, 8), fill="fence", pitch=8 + N + 8 + 1 - (N % 2))
    else:
        out, obuf = fenced((M, N), BF, (1, 1, 8, 8), fill="fence")
    out.copy_(old)
    ops.gemm(a, b, bias, L.MC_EPI_BIAS_GATE_RESID_BF16, out=out, gate=gate, addend=add, addend_row0=row0)
    check_fence(out, obuf)
    return out.clone()


@pytest.mark.parametrize("bn", [128, 256])
def test_epilogue8_readout(bn, monkeypatch):
    monkeypatch.setenv("MC_GEMM_BN", str(bn))
    sweep = bf16_sweep(DEV)
    g = torch.Generator(device=DEV).manual_seed(800 + bn)
    for geo, M, N, K, odd_ldo in GEOMETRIES:
        for row0 in (0, 7, 16, M - 1):
            for odd_ld, unaligned in ((False, False), (True, False), (False, True)):
                per_launch = N * K
                offset = 4099 + 17 * row0
                for launch in range(-(-SWEEP_SIZE // per_launch)):
                    what = (bn, geo, row0, odd_ld, unaligned, launch)
                    table = (torch.arange(per_launch, device=DEV) + offset + launch * per_launch) % SWEEP_SIZE
                    b_vals = sweep[table].view(N, K)
                    bias = _side_vector(N, g, 2.0, True)
                    gate = _side_vector(N, g, 0.5, True)
                    old = torch.randn(M, N, device=DEV, generator=g)
                    old[torch.rand(M, N, device=DEV, generator=g) < 0.125] = -0.0
                    old = old.to(BF)
                    add = _addend(M - row0, N, g, odd_ld, unaligned)
                    got = _launch8(M, N, K, odd_ldo, SCALED_A, b_vals, bias, gate, old, add, row0)
                    x6 = _launch(EPI6, M, N, K, odd_ldo, SCALED_A, b_vals, bias, gate, old)
                    cols = torch.arange(M, device=DEV) % K
                    acc32 = b_vals[:, cols].t().float() * SCALED_A  # exact, as in the readout module
                    x1 = epilogue_model(EPI6, acc32, bias[None, :], old, gate[None, :])
                    want = x1.clone()
                    want[row0:] = (x1[row0:].float() + add.float()).to(BF)
                    bad = _bits(got) != _bits(want)
                    assert not bool(bad.any()), (what, int(bad.sum()), bad.nonzero()[0].tolist())
                    assert torch.equal(_bits(got[:row0]), _bits(x6[:row0])), what
                    assert not bool(got.isnan().any()), what  # the sweep's largest values overflow to inf; NaN only from poison


def test_epilogue8_argument_checks():
    import ctypes

    from magcache_b200 import _lib as L
    a = torch.zeros(32, 64, dtype=BF, device=DEV)
    b = torch.zeros(32, 64, dtype=BF, device=DEV)
    out = torch.zeros(32, 32, dtype=BF, device=DEV)
    add = torch.zeros(32, 32, dtype=BF, device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    ok = L.lib.mc_gemm_bf16_add(p(a), 64, p(b), 64, 32, 32, 64, None, p(out), 32, None, p(add), 32, 0, None)
    torch.cuda.synchronize()
    assert ok == L.MC_OK
    for add_ptr, ld_add, row0 in ((None, 32, 0), (p(add), 31, 0), (p(add), 32, 32), (p(add), 32, -1)):
        assert L.lib.mc_gemm_bf16_add(p(a), 64, p(b), 64, 32, 32, 64, None, p(out), 32, None, add_ptr, ld_add, row0, None) == L.MC_ERR_INVALID
    # mc_gemm_bf16 keeps epilogue 8 to mc_gemm_bf16_add
    assert L.lib.mc_gemm_bf16(p(a), 64, p(b), 64, 32, 32, 64, None, L.MC_EPI_BIAS_GATE_RESID_ADD_BF16, p(out), 32, None, None) == L.MC_ERR_INVALID


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


def _samples(n, n_img, D, seed, scale, dev=DEV):
    if n is None:
        return None
    g = torch.Generator().manual_seed(seed)
    return [(scale * torch.randn(1, n_img, D, generator=g)).bfloat16().to(dev) for _ in range(n)]


class _WithSamples:
    """A FLUX model called with return_dict=False and the call's ControlNet samples, its first output returned; for the oracle the
    samples go through the reference's statements around its blocks. Attributes read through."""

    def __init__(self, m, oracle, n_txt, repeat=False):
        object.__setattr__(self, "_m", m)
        object.__setattr__(self, "_cfg", (oracle, n_txt, repeat))
        object.__setattr__(self, "samples", (None, None))

    def __call__(self, *a):
        import flux_controlnet_ref as cref
        oracle, n_txt, repeat = self._cfg
        bs, ss = self.samples
        if oracle:
            dt = next(self._m.parameters()).dtype
            cast = (lambda v: None if v is None else [x.to(dt) for x in v])
            with cref.controlnet_blocks(self._m, cast(bs), cast(ss), n_txt, repeat):
                return self._m(*a, return_dict=False)[0]
        return self._m(*a, return_dict=False, controlnet_block_samples=bs, controlnet_single_block_samples=ss,
                       controlnet_blocks_repeat=repeat)[0]

    def __getattr__(self, name):
        return getattr(self._m, name)


@pytest.mark.parametrize("repeat", [False, True])
def test_flux_controlnet_forward_loop(repeat, monkeypatch):
    """12 steps at reduced depth (3 double, 3 single blocks, D = 256), 256 image and 77 text tokens (n_txt not a multiple of 16:
    add_row0 inside a 16-row patch of the single blocks' `out` GEMM), fresh samples every step: DESIGN §5's rule against the bf16
    oracle and fp64 on every output and residual, the controller attributes equal."""
    import magcache_b200 as mc
    from oracle import flux_ref as fr
    from test_fullshape_workloads_gpu import _forward_loop, _oracle_on_gpu
    _oracle_on_gpu(monkeypatch)  # the oracle's host-built tensors (timestep sinusoid, RoPE) placed on the device
    n_txt, hw, steps = 77, (16, 16), 12
    model = _flux(3, 3, seed=5)
    g = torch.Generator().manual_seed(5)
    hs = torch.randn(1, hw[0] * hw[1], 64, generator=g).bfloat16().to(DEV)
    enc = torch.randn(1, n_txt, 96, generator=g).bfloat16().to(DEV)
    pooled = torch.randn(1, 48, generator=g).bfloat16().to(DEV)
    img_ids, txt_ids = (t.to(DEV) for t in fr.make_ids(*hw, n_txt))
    ours = _as("OurCNG", model)
    mc.init_magcache_flux(ours, steps)
    ref_m, m64 = _as("RefCNG", model), _as("RefCNG64", model, torch.float64)
    fr.install_magcache(type(ref_m), mc.tables()["flux_dev"], steps)
    fr.install_magcache(type(m64), mc.tables()["flux_dev"], steps)
    w = [_WithSamples(m, oracle, n_txt, repeat) for m, oracle in ((ours, False), (ref_m, True), (m64, True))]
    calls = []
    for i in range(steps):
        t, gd = torch.tensor([1.0 - i / steps], device=DEV), torch.tensor([4.0], device=DEV)
        x = hs * (1.0 - 0.03 * i)
        calls.append(((x, enc, pooled, t, img_ids, txt_ids, gd), (x, enc, pooled, t, img_ids, txt_ids, gd),
                      (x.double(), enc.double(), pooled.double(), t.double(), img_ids, txt_ids, gd.double())))

    class _Calls:  # fresh samples for each call, set on all three models before it runs
        def __iter__(self):
            for i, c in enumerate(calls):
                s = (_samples(2, hw[0] * hw[1], 256, 100 + i, 0.1), _samples(2, hw[0] * hw[1], 256, 200 + i, 0.1))
                for m in w:
                    object.__setattr__(m, "samples", s)
                yield c

    skips = _forward_loop("flux controlnet", _Calls(), *w, fr.exact, lambda m: m.previous_residual,
                          ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"))
    assert 0 < sum(skips) < steps, skips


def test_flux_zero_samples_equal_no_samples():
    import magcache_b200 as mc
    from oracle import flux_ref as fr
    n_txt, hw = 77, (16, 16)
    model = _flux(2, 3, seed=6)
    g = torch.Generator().manual_seed(6)
    hs = torch.randn(1, hw[0] * hw[1], 64, generator=g).bfloat16().to(DEV)
    enc = torch.randn(1, n_txt, 96, generator=g).bfloat16().to(DEV)
    pooled = torch.randn(1, 48, generator=g).bfloat16().to(DEV)
    img_ids, txt_ids = (t.to(DEV) for t in fr.make_ids(*hw, n_txt))
    zeros = [torch.zeros(1, hw[0] * hw[1], 256, dtype=BF, device=DEV)]
    a, b = _as("OurZ0", model), _as("OurZ1", model)
    mc.init_magcache_flux(a, 28)
    mc.init_magcache_flux(b, 28)
    with torch.no_grad():
        for i in range(3):
            t, gd = torch.tensor([1.0 - i / 28], device=DEV), torch.tensor([3.5], device=DEV)
            x = a(hs, enc, pooled, t, img_ids, txt_ids, gd, return_dict=False)[0]
            y = b(hs, enc, pooled, t, img_ids, txt_ids, gd, return_dict=False, controlnet_block_samples=zeros * 2,
                  controlnet_single_block_samples=zeros)[0]
            assert torch.equal(x, y), i
            assert torch.equal(a.previous_residual, b.previous_residual), i


def test_flux_1024_controlnet_one_layer_forward(monkeypatch):
    """FLUX.1-dev at 1024 x 1024 (4096 image tokens, 512 text tokens of width 4096), one double and one single block at 3072 /
    24 heads, a ControlNet sample after each: miss, miss, hit, with the samples of test_fullshape_workloads_gpu.py's FLUX test's
    exact timesteps and guidance."""
    import magcache_b200 as mc
    from oracle import flux_ref as fr
    from test_fullshape_workloads_gpu import FLUX, _forward_loop, _need_device_memory, _oracle_on_gpu, _report
    _need_device_memory(40)
    _oracle_on_gpu(monkeypatch)
    t0 = time.time()
    fl = FLUX
    model = _flux(1, 1, fl["heads"], seed=21, text_dim=fl["text_dim"], pooled=fl["pooled"])
    g = torch.Generator().manual_seed(21)
    hs = torch.randn(1, fl["n_img"], 64, generator=g).bfloat16().to(DEV)
    enc = torch.randn(1, fl["n_txt"], fl["text_dim"], generator=g).bfloat16().to(DEV)
    pooled = torch.randn(1, fl["pooled"], generator=g).bfloat16().to(DEV)
    img_ids, txt_ids = (t.to(DEV) for t in fr.make_ids(fl["h_tok"], fl["w_tok"], fl["n_txt"]))
    gd = torch.tensor([4.0], device=DEV)
    steps, table = 5, [1.0] + [0.98] * 4
    kw = dict(thresh=10.0, K=3, retention_ratio=0.4)
    ours = _as("OurCNFull", model)
    mc.init_magcache_flux(ours, steps, mag_ratios=table, **kw)
    ref_m = _as("RefCNFull", model)
    fr.install_magcache(type(ref_m), table, steps, **kw)
    m64 = _as("RefCNFull64", model, torch.float64)
    fr.install_magcache(type(m64), table, steps, **kw)
    del model
    samples = (_samples(1, fl["n_img"], fl["hidden"], 22, 0.1), _samples(1, fl["n_img"], fl["hidden"], 23, 0.1))
    w = [_WithSamples(m, oracle, fl["n_txt"]) for m, oracle in ((ours, False), (ref_m, True), (m64, True))]
    for m in w:
        object.__setattr__(m, "samples", samples)
    calls = []
    for tv in (1.0, 0.5, 0.25):
        t = torch.tensor([tv], device=DEV)
        a = (hs, enc, pooled, t, img_ids, txt_ids, gd)
        calls.append((a, a, (hs.double(), enc.double(), pooled.double(), t.double(), img_ids, txt_ids, gd.double())))
    skips = _forward_loop("flux 1024 controlnet", calls, *w, fr.exact, lambda m: m.previous_residual,
                          ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"))
    assert skips == [0, 0, 1], skips
    _report("flux 1024 controlnet forward", t0)


# ------------------------------------------------------------------------------------------- two GPUs
def _shard_worker(rank, world, initfile, results):
    import torch.distributed as dist

    import magcache_b200 as mc
    from oracle import flux_ref as fr
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", init_method=f"file://{initfile}", rank=rank, world_size=world, device_id=dev)
    try:
        g = torch.Generator().manual_seed(3)
        model = _flux(2, 2)
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
                    bs, ss = _samples(2, 1152, 256, 300 + i, 0.2, dev), _samples(1, 1152, 256, 400 + i, 0.2, dev)
                    got.append(m(hs * (1 - 0.05 * i), enc, pooled, torch.tensor([1.0 - i / 6], device=dev), img_ids, txt_ids,
                                 torch.tensor([3.5], device=dev), return_dict=False, controlnet_block_samples=bs,
                                 controlnet_single_block_samples=ss)[0].clone())
            outs[name] = (got, m._mc_flux_engine)
        eng = outs["sharded"][1]
        errs = [rel_l2(a, b) for a, b in zip(outs["sharded"][0], outs["single"][0])]
        res_err = rel_l2(eng.res, outs["single"][1].res[eng.shard.start:eng.shard.stop])
        results[rank] = (errs, res_err, eng.n_img, eng.n_img_total)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_flux_controlnet_sharded_matches_single_gpu():
    """Token-sharded over two GPUs with samples (each rank adds its own rows of every sample, a view) against one GPU, at
    test_shard_gpu.py's bound for the sharded FLUX engine without samples: the sharded attention's key order differs from the
    single engine's, so the two are not bit-equal with or without samples."""
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
