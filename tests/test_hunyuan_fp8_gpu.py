"""HunyuanVideo FP8-weight checkpoints on the GPU: `mc_dequant_fp8_bf16` against torch bit for bit, `magcache_hunyuan_forward` on an FP8
module bit-equal to the same forward on the dequantised bf16 module (and within the bf16 criterion of tests/test_hunyuan_forward_gpu.py
of the oracle's FP8 forward and the fp64 evaluation), and the device memory an FP8 engine holds."""
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _bits_equal(got, want):
    """Bitwise equality of two bf16 tensors except at NaN, where both must be NaN (payloads are not compared)."""
    nan = torch.isnan(want)
    return torch.equal(torch.isnan(got), nan) and torch.equal(got[~nan].view(torch.int16), want[~nan].view(torch.int16))


@pytest.mark.parametrize("rows,cols,offset", [(4, 256, 0), (3, 257, 0), (5, 100, 0), (6, 48, 1), (4608, 1536, 0)])
def test_dequant_fp8_all_codes_bitwise(rows, cols, offset):
    """Every e4m3 code (including -0 and the NaN codes 0x7F / 0xFF), row lengths that are and are not multiples of 16, a misaligned
    operand, and a large matrix; scales 1, typical amax / 448 values and a different scale per row."""
    from magcache_b200 import ops
    n = rows * cols
    codes = torch.arange(256, dtype=torch.uint8, device=DEV).repeat((n + offset) // 256 + 1)[:n + offset]
    q = codes[offset:].view(rows, cols).view(torch.float8_e4m3fn)
    g = torch.Generator(device=DEV).manual_seed(rows * 1000 + cols)
    amax = torch.tensor([0.05, 0.8, 3.1, 1e-3], device=DEV)
    for scale in (torch.ones(rows, device=DEV),
                  (amax[1] / 448).expand(rows),
                  (amax[rows % 4] / 448).expand(rows),
                  (amax[torch.randint(0, 4, (rows,), device=DEV, generator=g)] / 448) * (1 + torch.rand(rows, device=DEV, generator=g))):
        s = scale.to(torch.bfloat16).contiguous()
        out = torch.full((rows, cols), 7.0, dtype=torch.bfloat16, device=DEV)
        ops.dequant_fp8_bf16(q, s, out)
        want = q.to(torch.bfloat16) * s[:, None]
        assert _bits_equal(out, want)
        flat = codes[offset:]
        assert torch.equal(torch.isnan(out).view(-1), (flat & 0x7F) == 0x7F)
        neg0 = (flat == 0x80).view(rows, cols)
        assert bool((out[neg0].view(torch.int16) == torch.tensor(-32768, dtype=torch.int16, device=DEV)).all())  # -0 stays -0


def _setup(seed, valid=11, hidden=256, heads=2, depth=(2, 3), grid=(3, 8, 12), n_txt=16):
    import hunyuan_fp8_ref as f8
    from oracle import hunyuan_ref as hr
    model = hr.HYVideoDiffusionTransformer(hidden_size=hidden, heads_num=heads, mm_double_blocks_depth=depth[0], mm_single_blocks_depth=depth[1],
                                          text_states_dim=96, text_states_dim_2=48).init_synthetic(seed)
    fp8_model = f8.to_fp8_checkpoint(model)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, 16, grid[0], 2 * grid[1], 2 * grid[2], generator=g).bfloat16()
    txt = torch.randn(1, n_txt, 96, generator=g).bfloat16()
    mask = torch.zeros(1, n_txt, dtype=torch.long)
    mask[0, :valid] = 1
    pooled = torch.randn(1, 48, generator=g).bfloat16()
    cos, sin = hr.rope_cos_sin(grid)
    return hr, f8, fp8_model, (x, txt, mask, pooled, cos, sin)


def _fresh(model, name):
    m = copy.deepcopy(model)
    m.__class__ = type(name, (m.__class__,), {})
    return m


@pytest.mark.parametrize("size", ["reduced", "mid"])
def test_hunyuan_fp8_forward_bit_equal_to_dequantised(size):
    """Miss then two hits: the FP8 engine's outputs and controller state equal the bf16 engine's on the dequantised weights bit for
    bit; both meet the bf16 criterion against the oracle's FP8 forward and the fp64 evaluation of the dequantised model."""
    import magcache_b200 as mc
    from magcache_b200.mmdit import Fp8Weight
    kw = {} if size == "reduced" else dict(valid=37, hidden=1536, heads=12, depth=(2, 4), grid=(3, 16, 24), n_txt=64)
    hr, f8, fp8_model, (x, txt, mask, pooled, cos, sin) = _setup(5, **kw)
    bf_model = f8.dequantized(fp8_model)
    t, gd = torch.tensor([611.0]), torch.tensor([6000.0])
    steps, table = 5, [1.0] + [0.98] * 4
    dev_in = [v.to(DEV) for v in (txt, mask, pooled, cos, sin)]
    ours = {}
    for name, model in (("F8", fp8_model), ("BF", bf_model)):
        m = _fresh(model, "Our" + name).to(DEV)
        mc.init_magcache_hunyuan(m, steps, thresh=10.0, K=3, retention_ratio=0.2, mag_ratios=table)
        outs, state = [], []
        with torch.no_grad():
            for _ in range(3):
                outs.append(m(x.to(DEV), t.to(DEV), *dev_in, gd.to(DEV), return_dict=False).cpu())
                state.append(tuple(float(getattr(m, a)) for a in ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps")))
        ours[name] = (outs, state, m)
    assert ours["F8"][1] == ours["BF"][1]
    assert all(torch.equal(a, b) for a, b in zip(ours["F8"][0], ours["BF"][0]))
    assert isinstance(ours["F8"][2]._mc_hunyuan_engine.w.single[0]["out_w"], Fp8Weight)
    ref_m = _fresh(fp8_model, "RefF8")
    hr.install_magcache(type(ref_m), table, steps, thresh=10.0, K=3, retention_ratio=0.2)
    m64 = _fresh(bf_model, "RefF864").double()
    hr.install_magcache(type(m64), table, steps, thresh=10.0, K=3, retention_ratio=0.2)
    kinds = []
    with torch.no_grad():
        for call in range(3):
            ref = ref_m(x, t, txt, mask, pooled, cos, sin, gd, return_dict=False)
            with hr.exact():
                exact = m64(x.double(), t.double(), txt.double(), mask, pooled.double(), cos.double(), sin.double(), gd.double(), return_dict=False)
            out = ours["F8"][0][call]
            kinds.append(int(ref_m.last_skip))
            e_ours, e_ref, e_vs = rel_l2(out, exact), rel_l2(ref, exact), rel_l2(out, ref)
            print(f"[hunyuan fp8 {size}, call {call}] ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e} | ours vs oracle {e_vs:.3e}")
            assert e_ours <= 1.5 * e_ref + 1e-3 and e_vs <= 2.0 * e_ref + 1e-3, (call, e_ours, e_ref, e_vs)
    assert kinds == [0, 1, 1], kinds


def test_fp8_engine_memory():
    """Building the engine from an FP8 module on the device adds at most: the stacked FP8 modulation codes and the per-row scales, the
    dequantisation scratch, and the non-block weights (bf16 matrices, fp32 copies of every bias / norm vector) — no bf16 copy of a
    block weight."""
    import magcache_b200 as mc  # noqa: F401
    from magcache_b200 import mmdit
    _, _, fp8_model, _ = _setup(7, hidden=1536, heads=12, depth=(2, 4))
    m = fp8_model.to(DEV)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    w = mmdit.HunyuanWeights.from_module(m, torch.device(DEV))
    eng = mmdit.HunyuanEngine(w)
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - before
    params = dict(m.named_parameters())
    fp8_params = {n: p for n, p in params.items() if p.dtype == torch.float8_e4m3fn}
    fp8_rows = sum(p.shape[0] for p in fp8_params.values())
    mod_codes = sum(p.numel() for n, p in fp8_params.items() if "mod" in n)
    other_mats = sum(p.numel() for n, p in params.items() if n not in fp8_params and p.dim() > 1)
    vectors = sum(p.numel() for p in params.values() if p.dim() == 1)
    n_tensors = 4 * len(params) + 16
    bound = mod_codes + 2 * 2 * fp8_rows + w.fp8_scratch.numel() * 2 + 2 * other_mats + 4 * vectors + 512 * n_tensors
    block_bf16 = 2 * sum(p.numel() for p in fp8_params.values())
    print(f"[fp8 engine memory] grown {grown / 2**20:.1f} MiB, bound {bound / 2**20:.1f} MiB, block weights in bf16 would be "
          f"{block_bf16 / 2**20:.1f} MiB")
    assert grown <= bound, (grown, bound)
    assert w.fp8_scratch.numel() == 5 * 1536 * 1536 and eng.w is w
