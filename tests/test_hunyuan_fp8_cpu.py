"""HunyuanVideo FP8-weight checkpoints on the MMDiT engine, on CPU through the kernel emulation (tests/emu_ops.py plus the emulated
`dequant_fp8_bf16` of tests/hunyuan_fp8_ref.py): the oracle converts upstream's set of Linears, `HunyuanWeights.from_module` keeps
the block weights in FP8, and the engine on an FP8 module is bit-equal to the engine on the dequantised bf16 module."""
import copy
import os
import sys
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import emu_ops  # noqa: E402
import hunyuan_fp8_ref as f8  # noqa: E402
import magcache_b200 as mc  # noqa: E402
from magcache_b200 import mmdit as mmdit_mod  # noqa: E402
from magcache_b200 import patch as patch_mod  # noqa: E402
from oracle import hunyuan_ref as hr  # noqa: E402


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(emu_ops, "dequant_fp8_bf16", f8.emu_dequant_fp8_bf16, raising=False)
    monkeypatch.setattr(mmdit_mod, "ops", emu_ops)
    monkeypatch.setattr(patch_mod, "ops", emu_ops)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def _model(seed=0, depth=(2, 3), guidance=True):
    return hr.HYVideoDiffusionTransformer(hidden_size=256, heads_num=2, mm_double_blocks_depth=depth[0], mm_single_blocks_depth=depth[1],
                                          text_states_dim=96, text_states_dim_2=48, guidance_embed=guidance).init_synthetic(seed)


def _inputs(seed=0, grid=(2, 4, 6), n_txt=16, valid=11):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, 16, grid[0], 2 * grid[1], 2 * grid[2], generator=g).bfloat16()
    txt = torch.randn(1, n_txt, 96, generator=g).bfloat16()
    mask = torch.zeros(1, n_txt, dtype=torch.long)
    mask[0, :valid] = 1
    pooled = torch.randn(1, 48, generator=g).bfloat16()
    cos, sin = hr.rope_cos_sin(grid)
    return x, txt, mask, pooled, cos, sin


def _fresh(model, name):
    m = copy.deepcopy(model)
    m.__class__ = type(name, (m.__class__,), {})
    return m


UPSTREAM_DOUBLE = ("img_mod.linear", "img_attn_qkv", "img_attn_proj", "img_mlp.fc1", "img_mlp.fc2",
                   "txt_mod.linear", "txt_attn_qkv", "txt_attn_proj", "txt_mlp.fc1", "txt_mlp.fc2")
UPSTREAM_SINGLE = ("linear1", "linear2", "modulation.linear")


def test_oracle_converts_exactly_the_block_linears():
    m = f8.to_fp8_checkpoint(_model(depth=(2, 2)))
    fp8 = {n for n, p in m.named_parameters() if p.dtype == torch.float8_e4m3fn}
    want = {f"double_blocks.{i}.{n}.weight" for i in range(2) for n in UPSTREAM_DOUBLE}
    want |= {f"single_blocks.{i}.{n}.weight" for i in range(2) for n in UPSTREAM_SINGLE}
    assert fp8 == want
    for n, p in m.named_parameters():
        if n.split(".")[0] in ("txt_in", "final_layer", "time_in", "vector_in", "guidance_in", "img_in"):
            assert p.dtype == torch.bfloat16, n
    for n in want:
        lin = m.get_submodule(n[:-len(".weight")])
        assert lin.fp8_scale.dtype == torch.bfloat16 and lin.fp8_scale.numel() == 1
    # the restated forward multiplies by the bf16-rounded dequantised weight: the same numbers as the dequantised bf16 model
    lin, ref = m.double_blocks[0].img_attn_qkv, f8.dequantized(m).double_blocks[0].img_attn_qkv
    x = torch.randn(5, 256).bfloat16()
    assert torch.equal(lin(x), ref(x)) and ref.weight.dtype == torch.bfloat16


def test_from_module_keeps_block_weights_in_fp8():
    m = f8.to_fp8_checkpoint(_model())
    w = mmdit_mod.HunyuanWeights.from_module(m, torch.device("cpu"))
    D = 256
    fp8_bytes = 0
    for blk in w.double + w.single:
        for k, v in blk.items():
            if k.endswith("_w"):
                assert isinstance(v, mmdit_mod.Fp8Weight) and v.q.dtype == torch.float8_e4m3fn and v.q.element_size() == 1, k
                fp8_bytes += v.q.numel()
    # row blocks of the fused q|k|v and linear1 matrices are views of the module's own codes
    b0, s0 = w.double[0], w.single[0]
    assert b0["qk_w"].q.data_ptr() == m.double_blocks[0].img_attn_qkv.weight.data_ptr()
    assert b0["v_w"].q.data_ptr() == m.double_blocks[0].img_attn_qkv.weight.data_ptr() + 2 * D * D
    assert s0["mlp_w"].q.data_ptr() == m.single_blocks[0].linear1.weight.data_ptr() + 3 * D * D
    assert b0["o_w"].q.data_ptr() == m.double_blocks[0].img_attn_proj.weight.data_ptr()
    assert torch.equal(s0["v_w"].scale, m.single_blocks[0].linear1.fp8_scale.reshape(1).expand(D))
    assert fp8_bytes == sum(p.numel() for n, p in m.named_parameters() if p.dtype == torch.float8_e4m3fn and "mod" not in n)
    # modulation: block rows stacked as codes with their per-row scales, the final layer's rows bf16
    (r0, mod), (r1, fin) = w.ada_parts
    assert r0 == 0 and isinstance(mod, mmdit_mod.Fp8Weight) and mod.shape == (w.ada_out, D) and r1 == w.ada_out
    assert fin.dtype == torch.bfloat16 and fin.shape == (2 * D, D) and w.ada_rows == w.ada_out + 2 * D
    assert torch.equal(mod.scale[6 * D:12 * D], m.double_blocks[0].txt_mod.linear.fp8_scale.reshape(1).expand(6 * D))
    assert torch.equal(mod.q[6 * D:12 * D].view(torch.uint8), m.double_blocks[0].txt_mod.linear.weight.view(torch.uint8))
    assert w.fp8_scratch.dtype == torch.bfloat16 and w.fp8_scratch.numel() == 5 * D * D  # linear2, D x 5D
    assert not hasattr(w, "ada_w")


def test_from_module_rejects_incomplete_fp8_checkpoints():
    m = f8.to_fp8_checkpoint(_model())
    del m.single_blocks[1].linear2.fp8_scale
    with pytest.raises(ValueError, match="fp8_scale"):
        mmdit_mod.HunyuanWeights.from_module(m, torch.device("cpu"))
    m = f8.to_fp8_checkpoint(_model())
    m.final_layer.linear.weight = torch.nn.Parameter(m.final_layer.linear.weight.detach().to(torch.float8_e4m3fn), requires_grad=False)
    with pytest.raises(NotImplementedError):
        mmdit_mod.HunyuanWeights.from_module(m, torch.device("cpu"))
    # a bf16 module takes the bf16 path: one stacked modulation matrix, no scratch
    w = mmdit_mod.HunyuanWeights.from_module(_model(), torch.device("cpu"))
    assert w.ada_parts is None and w.fp8_scratch is None and w.ada_w.dtype == torch.bfloat16


def _run_loop(model, name, steps, n_calls, x, txt, mask, pooled, cos, sin):
    m = _fresh(model, name)
    mc.init_magcache_hunyuan(m, steps, thresh=0.24, K=6, retention_ratio=0.2)
    outs, state = [], []
    with torch.no_grad():
        for i in range(n_calls):
            t = torch.tensor([1000.0 - 90.0 * (i % steps)])
            outs.append(m(x * (1.0 - 0.03 * i), t, txt, mask, pooled, cos, sin, torch.tensor([6000.0]), return_dict=False).clone())
            state.append(tuple(float(getattr(m, a)) for a in ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps")))
    return outs, state


def test_fp8_engine_bit_equal_to_dequantised_bf16_engine(emulated):
    """Miss and hit calls, controller state, and the oracle criterion of the bf16 emulated test against the oracle's FP8 forward."""
    fp8_model = f8.to_fp8_checkpoint(_model(seed=1))
    bf_model = f8.dequantized(fp8_model)
    x, txt, mask, pooled, cos, sin = _inputs(1)
    steps = 10
    got, st_a = _run_loop(fp8_model, "OurF8", steps, steps + 2, x, txt, mask, pooled, cos, sin)
    want, st_b = _run_loop(bf_model, "OurBF", steps, steps + 2, x, txt, mask, pooled, cos, sin)
    assert st_a == st_b
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    skips = mc.MagCacheConfig("hunyuan", 0.24, 6, 0.2, steps, table="hunyuan_720p").schedule().tolist()
    assert 0 < sum(skips) < steps  # the loop has both kinds of call
    # the first (miss) call against the oracle's FP8 forward and the fp64 evaluation of the dequantised model
    ref_m = _fresh(fp8_model, "RefF8")
    hr.install_magcache(type(ref_m), mc.tables()["hunyuan_720p"], steps)
    m64 = _fresh(bf_model, "RefF864").double()
    hr.install_magcache(type(m64), mc.tables()["hunyuan_720p"], steps)
    t, gd = torch.tensor([1000.0]), torch.tensor([6000.0])
    with torch.no_grad():
        ref = ref_m(x, t, txt, mask, pooled, cos, sin, gd, return_dict=False)
        with hr.exact():
            exact = m64(x.double(), t.double(), txt.double(), mask, pooled.double(), cos.double(), sin.double(), gd.double(), return_dict=False)
    e_ours, e_ref, e_vs = rel_l2(got[0], exact), rel_l2(ref, exact), rel_l2(got[0], ref)
    assert e_ours <= 1.5 * e_ref + 1e-3 and e_vs <= 2.0 * e_ref + 1e-3, (e_ours, e_ref, e_vs)


def test_fp8_calibration_twin_bit_equal(emulated):
    fp8_model = f8.to_fp8_checkpoint(_model(seed=3))
    bf_model = f8.dequantized(fp8_model)
    x, txt, mask, pooled, cos, sin = _inputs(3)
    res = {}
    for name, model in (("CalF8", fp8_model), ("CalBF", bf_model)):
        m = _fresh(model, name)
        mc.init_magcache_hunyuan_calibration(m, 50)
        outs = []
        with torch.no_grad():
            for i in range(3):
                outs.append(m(x * (1.0 - 0.1 * i), torch.tensor([900.0 - 100.0 * i]), txt, mask, pooled, cos, sin, torch.tensor([6000.0]))["x"])
        res[name] = (outs, [list(getattr(m, k)) for k in ("norm_ratio", "norm_std", "cos_dis")])
    assert all(torch.equal(a, b) for a, b in zip(res["CalF8"][0], res["CalBF"][0]))
    assert res["CalF8"][1] == res["CalBF"][1] and len(res["CalF8"][1][0]) == 2


def _shard_worker(rank, world, initfile, results):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import emu_ops as eo
    import hunyuan_fp8_ref as ref
    from magcache_b200 import mmdit
    from magcache_b200 import patch as pm
    dist.init_process_group("gloo", init_method=f"file://{initfile}", rank=rank, world_size=world)
    try:
        eo.dequant_fp8_bf16 = ref.emu_dequant_fp8_bf16
        mmdit.ops = eo
        pm.ops = eo
        torch.Tensor.is_cuda = property(lambda self: True)
        model = ref.to_fp8_checkpoint(_model(seed=0, depth=(2, 2)))
        x, txt, mask, pooled, cos, sin = _inputs(0)
        outs = {}
        for name in ("single", "sharded"):
            m = _fresh(model, "S_" + name)
            mc.init_magcache_hunyuan(m, 6, thresh=10.0, K=2, retention_ratio=0.34, mag_ratios=[1.0] * 6)  # miss miss hit hit miss miss
            if name == "sharded":
                mc.enable_token_shard(m, rank, world)
            with torch.no_grad():
                outs[name] = [m(x * (1 - 0.05 * i), torch.tensor([900.0 - 100 * i]), txt, mask, pooled, cos, sin, torch.tensor([6000.0]),
                                return_dict=False).clone() for i in range(6)]
        results[rank] = [float((a.float() - b.float()).abs().max() / b.float().abs().max()) for a, b in zip(outs["sharded"], outs["single"])]
    finally:
        dist.destroy_process_group()


def test_sharded_fp8_engine_equals_single_world2():
    with tempfile.TemporaryDirectory() as d:
        mgr = mp.get_context("spawn").Manager()
        results = mgr.dict()
        mp.spawn(_shard_worker, args=(2, os.path.join(d, "init"), results), nprocs=2, join=True)
        assert set(results.keys()) == {0, 1}
        for r in (0, 1):
            errs = results[r]
            assert len(errs) == 6 and max(errs) < 1.2e-2, errs  # bf16 streams: a different GEMM row blocking flips roundings
