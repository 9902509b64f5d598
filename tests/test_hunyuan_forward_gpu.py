"""HunyuanVideo MMDiT engine on the GPU: `magcache_hunyuan_forward` against the oracle restatement of
MagCache4HunyuanVideo/magcache_sample_video.py:29-160, and the column-mean kernel against torch.

The orchestration is also pinned on CPU through the kernel emulation
(tests/test_hunyuan_engine_emulated_cpu.py)."""
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


def test_colmean_vs_torch():
    import emu_ops
    from magcache_b200 import ops
    for rows, cols in [(11, 4096), (1, 96), (256, 4096)]:
        x = torch.randn(rows, cols, device=DEV).bfloat16()
        got = ops.colmean(x).cpu()
        want = emu_ops.colmean(x.cpu())
        assert ((got.float() - want.float()).abs() <= want.float().abs() * 2.0 ** -7 + 1e-6).all()


def _setup(seed, guidance=True, valid=11, hidden=256, heads=2, depth=(2, 3), grid=(3, 8, 12), n_txt=16):
    import magcache_b200 as mc
    from oracle import hunyuan_ref as hr
    model = hr.HYVideoDiffusionTransformer(hidden_size=hidden, heads_num=heads, mm_double_blocks_depth=depth[0], mm_single_blocks_depth=depth[1],
                                          text_states_dim=96, text_states_dim_2=48, guidance_embed=guidance).init_synthetic(seed)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, 16, grid[0], 2 * grid[1], 2 * grid[2], generator=g).bfloat16()
    txt = torch.randn(1, n_txt, 96, generator=g).bfloat16()
    mask = torch.zeros(1, n_txt, dtype=torch.long)
    mask[0, :valid] = 1
    pooled = torch.randn(1, 48, generator=g).bfloat16()
    cos, sin = hr.rope_cos_sin(grid)
    return mc, hr, model, (x, txt, mask, pooled, cos, sin)


def test_hunyuan_forward_vs_oracle_and_fp64():
    mc, hr, model, (x, txt, mask, pooled, cos, sin) = _setup(0)
    t, gd = torch.tensor([731.0]), torch.tensor([6000.0])
    ref_m = copy.deepcopy(model)
    ref_m.__class__ = type("RefHY", (ref_m.__class__,), {})
    hr.install_magcache(type(ref_m), mc.tables()["hunyuan_720p"], 50)
    m64 = copy.deepcopy(model).double()
    m64.__class__ = type("RefHY64", (m64.__class__,), {})
    hr.install_magcache(type(m64), mc.tables()["hunyuan_720p"], 50)
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("OurHY", (ours.__class__,), {})
    mc.init_magcache_hunyuan(ours, 50)
    with torch.no_grad():
        ref = ref_m(x, t, txt, mask, pooled, cos, sin, gd)["x"]
        with hr.exact():
            exact = m64(x.double(), t.double(), txt.double(), mask, pooled.double(), cos.double(), sin.double(), gd.double())["x"]
    out = ours(x.to(DEV), t.to(DEV), txt.to(DEV), mask.to(DEV), pooled.to(DEV), cos.to(DEV), sin.to(DEV), gd.to(DEV))["x"].cpu()
    e_ours, e_ref, e_vs = rel_l2(out, exact), rel_l2(ref, exact), rel_l2(out, ref)
    print(f"[hunyuan] ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e} | ours vs oracle {e_vs:.3e}")
    assert e_ours <= 1.5 * e_ref + 1e-3 and e_vs <= 2.0 * e_ref + 1e-3


def test_hunyuan_loop_vs_oracle():
    """12 calls (hits and misses): controller state bit-equal on every call; tensors within twice the bf16 oracle's own distance from an
    fp64 run of the same loop (+1e-3)."""
    mc, hr, model, (x, txt, mask, pooled, cos, sin) = _setup(1, valid=16)
    steps = 10
    ref_m = copy.deepcopy(model)
    ref_m.__class__ = type("RefHYL", (ref_m.__class__,), {})
    hr.install_magcache(type(ref_m), mc.tables()["hunyuan_720p"], steps)
    m64 = copy.deepcopy(model).double()
    m64.__class__ = type("RefHYL64", (m64.__class__,), {})
    hr.install_magcache(type(m64), mc.tables()["hunyuan_720p"], steps)
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("OurHYL", (ours.__class__,), {})
    mc.init_magcache_hunyuan(ours, steps)
    dev_in = [v.to(DEV) for v in (txt, mask, pooled, cos, sin)]
    skips = []
    with torch.no_grad():
        for i in range(steps + 2):
            t = torch.tensor([1000.0 - 90.0 * (i % steps)])
            xi = x * (1.0 - 0.03 * i)
            ref = ref_m(xi, t, txt, mask, pooled, cos, sin, torch.tensor([6000.0]), return_dict=False)
            with hr.exact():
                exact = m64(xi.double(), t.double(), txt.double(), mask, pooled.double(), cos.double(), sin.double(), torch.tensor([6000.0]).double(),
                            return_dict=False)
            out = ours(xi.to(DEV), t.to(DEV), *dev_in, torch.tensor([6000.0], device=DEV), return_dict=False).cpu()
            skips.append(int(ref_m.last_skip))
            e_ref, e_vs, e_ours = rel_l2(ref, exact), rel_l2(out, ref), rel_l2(out, exact)
            assert e_vs <= 2.0 * e_ref + 1e-3, (i, e_vs, e_ref)
            assert e_ours <= 1.5 * e_ref + 1e-3, (i, e_ours, e_ref)
            for attr in ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"):
                assert float(getattr(ours, attr)) == float(getattr(ref_m, attr)), (i, attr)
    assert 0 < sum(skips[:steps]) < steps


def test_hunyuan_mid_size_forward_vs_oracle_and_fp64():
    """A HunyuanVideo-shaped model at a mid size — hidden 1536 (12 heads x 128), 2 double + 4 single blocks, 3 x 16 x 24 = 1152 image
    tokens + 64 text tokens (37 valid): the long attention kernel, multi-tile GEMMs — miss then hit, against the bf16 oracle and the
    fp64 evaluation."""
    mc, hr, model, (x, txt, mask, pooled, cos, sin) = _setup(5, valid=37, hidden=1536, heads=12, depth=(2, 4), grid=(3, 16, 24), n_txt=64)
    t, gd = torch.tensor([611.0]), torch.tensor([6000.0])
    steps, table = 5, [1.0] + [0.98] * 4
    ref_m = copy.deepcopy(model)
    ref_m.__class__ = type("RefHYM", (ref_m.__class__,), {})
    hr.install_magcache(type(ref_m), table, steps, thresh=10.0, K=3, retention_ratio=0.2)
    m64 = copy.deepcopy(model).double()
    m64.__class__ = type("RefHYM64", (m64.__class__,), {})
    hr.install_magcache(type(m64), table, steps, thresh=10.0, K=3, retention_ratio=0.2)
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("OurHYM", (ours.__class__,), {})
    mc.init_magcache_hunyuan(ours, steps, thresh=10.0, K=3, retention_ratio=0.2, mag_ratios=table)
    dev_in = [v.to(DEV) for v in (txt, mask, pooled, cos, sin)]
    kinds = []
    with torch.no_grad():
        for call in range(3):
            ref = ref_m(x, t, txt, mask, pooled, cos, sin, gd, return_dict=False)
            with hr.exact():
                exact = m64(x.double(), t.double(), txt.double(), mask, pooled.double(), cos.double(), sin.double(), gd.double(), return_dict=False)
            out = ours(x.to(DEV), t.to(DEV), *dev_in, gd.to(DEV), return_dict=False).cpu()
            kinds.append(int(ref_m.last_skip))
            e_ours, e_ref, e_vs = rel_l2(out, exact), rel_l2(ref, exact), rel_l2(out, ref)
            print(f"[hunyuan mid, call {call}, {'hit' if kinds[-1] else 'miss'}] ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e} | ours vs oracle {e_vs:.3e}")
            assert e_ours <= 1.5 * e_ref + 1e-3 and e_vs <= 2.0 * e_ref + 1e-3, (call, e_ours, e_ref, e_vs)
            assert float(ours.cnt) == float(ref_m.cnt)
    assert kinds == [0, 1, 1], kinds
