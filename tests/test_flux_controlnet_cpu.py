"""FLUX / Kontext ControlNet residuals on the MMDiT engine, on CPU: `magcache_flux_forward` / `magcache_flux_calibration` with
`controlnet_block_samples` / `controlnet_single_block_samples`, the engine driven through the kernel emulation (tests/emu_ops.py plus
epilogue 8, tests/flux_controlnet_ref.py) against the oracle running the reference's ControlNet statements
(MagCache4FLUX/magcache_flux.py:374-384, :416-423; calibration :145-155, :187-193). The epilogue itself: test_flux_controlnet_gpu.py."""
import copy
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import magcache_b200 as mc
from magcache_b200 import mmdit as flux_mod
from magcache_b200 import patch as patch_mod
from oracle import flux_ref as fr

import flux_controlnet_ref as cref


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


@pytest.fixture()
def emulated(monkeypatch):
    monkeypatch.setattr(flux_mod, "ops", cref.emu)
    monkeypatch.setattr(patch_mod, "ops", cref.emu)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))  # the forward insists on CUDA tensors


def _model(num_layers=2, num_single_layers=3, seed=0):
    return fr.FluxTransformer2DModel(in_channels=64, num_layers=num_layers, num_single_layers=num_single_layers, num_attention_heads=2,
                                     joint_attention_dim=96, pooled_projection_dim=48).init_synthetic(seed)


def _inputs(seed=0, hw=(8, 6), n_txt=19):
    g = torch.Generator().manual_seed(seed)
    n_img = hw[0] * hw[1]
    hs = torch.randn(1, n_img, 64, generator=g).bfloat16()
    enc = torch.randn(1, n_txt, 96, generator=g).bfloat16()
    pooled = torch.randn(1, 48, generator=g).bfloat16()
    img_ids, txt_ids = fr.make_ids(hw[0], hw[1], n_txt)
    return hs, enc, pooled, img_ids, txt_ids


def _samples(n, n_img=48, D=256, seed=0, scale=0.5):
    if n is None:
        return None
    g = torch.Generator().manual_seed(1000 + seed)
    return [(scale * torch.randn(1, n_img, D, generator=g)).bfloat16() for _ in range(n)]


def _as(cls_name, model):
    m = copy.deepcopy(model)
    m.__class__ = type(cls_name, (m.__class__,), {})
    return m


def test_block_to_sample_mapping_is_the_references():
    for n_blocks in range(1, 58):
        for n_samples in range(1, 61):
            for repeat in (False, True):
                want = cref.reference_samples(n_blocks, list(range(n_samples)), repeat)
                got = [flux_mod.controlnet_index(i, n_blocks, n_samples, repeat) for i in range(n_blocks)]
                assert got == want, (n_blocks, n_samples, repeat)
    with pytest.raises(ZeroDivisionError):
        flux_mod.controlnet_index(0, 19, 0, True)


# (double blocks, single blocks, double samples, single samples, controlnet_blocks_repeat, text tokens)
CASES = {
    "double_only": (2, 3, 1, None, False, 19),
    "single_only": (2, 3, None, 3, False, 19),
    "both": (2, 3, 2, 3, False, 19),
    "repeat": (3, 3, 2, 1, True, 19),
    "ceil": (3, 3, 2, 2, False, 19),
    "n_txt_32": (2, 3, 1, 2, False, 32),
}


@pytest.mark.parametrize("case", list(CASES))
def test_controlnet_forward_matches_oracle(emulated, case):
    nd, ns, cd, cs, repeat, n_txt = CASES[case]
    model = _model(nd, ns)
    hs, enc, pooled, img_ids, txt_ids = _inputs(n_txt=n_txt)
    bs, ss = _samples(cd, seed=1), _samples(cs, seed=2)
    t, gd = torch.tensor([0.731]), torch.tensor([3.5])
    ref_m, m64, ours = _as("RefCN", model), _as("RefCN64", copy.deepcopy(model).double()), _as("OurCN", model)
    fr.install_magcache(type(ref_m), mc.tables()["flux_dev"], 28)
    fr.install_magcache(type(m64), mc.tables()["flux_dev"], 28)
    mc.init_magcache_flux(ours, 28)
    dbl = (lambda v: None if v is None else [x.double() for x in v])
    with torch.no_grad():
        with cref.controlnet_blocks(ref_m, bs, ss, n_txt, repeat):
            ref = ref_m(hs, enc, pooled, t, img_ids, txt_ids, gd, return_dict=False)[0]
        with fr.exact(), cref.controlnet_blocks(m64, dbl(bs), dbl(ss), n_txt, repeat):
            exact = m64(hs.double(), enc.double(), pooled.double(), t.double(), img_ids, txt_ids, gd.double(), return_dict=False)[0]
        plain = _as("OurPlain", model)
        mc.init_magcache_flux(plain, 28)
        base = plain(hs, enc, pooled, t, img_ids, txt_ids, gd, return_dict=False)[0]
        out = ours(hs, enc, pooled, t, img_ids, txt_ids, gd, controlnet_block_samples=bs, controlnet_single_block_samples=ss,
                   controlnet_blocks_repeat=repeat).sample
    e_ours, e_ref, e_vs = rel_l2(out, exact), rel_l2(ref, exact), rel_l2(out, ref)
    print(f"[flux controlnet {case}] ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e} | ours vs oracle {e_vs:.3e}")
    assert e_ours <= 1.5 * e_ref + 1e-3
    assert e_vs <= 2.0 * e_ref + 1e-3
    assert rel_l2(base, exact) > 10 * e_ours  # the samples changed the output well beyond the rounding noise
    assert rel_l2(ours.previous_residual[0], ref_m.previous_residual[0]) <= 2.0 * e_ref + 2e-2


def test_zero_samples_change_nothing(emulated):
    model = _model()
    hs, enc, pooled, img_ids, txt_ids = _inputs()
    zeros = [torch.zeros(1, 48, 256, dtype=torch.bfloat16)]
    a, b = _as("OurZ0", model), _as("OurZ1", model)
    mc.init_magcache_flux(a, 28)
    mc.init_magcache_flux(b, 28)
    with torch.no_grad():
        x = a(hs, enc, pooled, torch.tensor([0.5]), img_ids, txt_ids, torch.tensor([3.5]), return_dict=False)[0]
        y = b(hs, enc, pooled, torch.tensor([0.5]), img_ids, txt_ids, torch.tensor([3.5]), return_dict=False,
              controlnet_block_samples=zeros, controlnet_single_block_samples=zeros * 2)[0]
    assert torch.equal(x, y)


@pytest.mark.parametrize("preset", ["flux_dev", "flux_kontext"])
def test_controlnet_loop_hits_ignore_samples(emulated, preset):
    """A 12-step generation with fresh samples on every step: the oracle and the engine take the same skip decisions and keep the
    same controller attributes; on hit steps the samples are not read, so other samples there (even malformed ones) leave every
    output of the generation unchanged."""
    thresh, K, retention = (0.24, 5, 0.1) if preset == "flux_dev" else (0.05, 4, 0.2)
    model = _model(seed=1)
    hs, enc, pooled, img_ids, txt_ids = _inputs(1)
    steps = 12
    ref_m = _as("RefCNL", model)
    fr.install_magcache(type(ref_m), mc.tables()[preset], steps, thresh=thresh, K=K, retention_ratio=retention)
    runs = {}
    for name in ("same", "other_on_hits"):
        m = _as("OurCNL_" + name, model)
        mc.init_magcache_flux(m, steps, thresh=thresh, K=K, retention_ratio=retention, table=preset)
        runs[name] = m
    skips, outs = [], {k: [] for k in runs}
    with torch.no_grad():
        for i in range(steps):
            t = torch.tensor([1.0 - i / steps])
            x = hs * (1.0 - 0.03 * i)
            bs, ss = _samples(2, seed=10 + i, scale=0.1), _samples(3, seed=50 + i, scale=0.1)
            with cref.controlnet_blocks(ref_m, bs, ss, 19):
                ref = ref_m(x, enc, pooled, t, img_ids, txt_ids, torch.tensor([3.5]), return_dict=False)[0]
            skips.append(bool(ref_m.last_skip))
            for name, m in runs.items():
                cb, cs = bs, ss
                if name == "other_on_hits" and skips[-1]:
                    cb, cs = [torch.zeros(1, 1, 256, dtype=torch.bfloat16)], _samples(3, seed=90 + i)
                out = m(x, enc, pooled, t, img_ids, txt_ids, torch.tensor([3.5]), return_dict=False, controlnet_block_samples=cb,
                        controlnet_single_block_samples=cs)[0]
                outs[name].append(out.clone())
                assert rel_l2(out, ref) <= 0.15, (i, name, rel_l2(out, ref))
                for attr in ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"):
                    assert float(getattr(m, attr)) == float(getattr(ref_m, attr)), (i, attr)
    assert 0 < sum(skips) < steps, skips
    for a, b in zip(outs["same"], outs["other_on_hits"]):
        assert torch.equal(a, b)


def test_controlnet_calibration_twin(emulated, capsys):
    model = _model(seed=2)
    hs, enc, pooled, img_ids, txt_ids = _inputs(2)
    steps = 4
    ref_m = _as("RefCNC", model)
    type(ref_m).forward = fr.magcache_calibration
    type(ref_m).cnt, type(ref_m).num_steps = 0, steps
    type(ref_m).norm_ratio, type(ref_m).norm_std, type(ref_m).cos_dis, type(ref_m).previous_residual = [], [], [], None
    ours = _as("OurCNC", model)
    mc.init_magcache_flux_calibration(ours, steps)
    stats_ref, stats_ours = None, None
    with torch.no_grad():
        for i in range(steps):
            t = torch.tensor([1.0 - i / steps])
            x = hs * (1.0 - 0.1 * i)
            bs, ss = _samples(1, seed=20 + i, scale=0.2), _samples(2, seed=60 + i, scale=0.2)
            with cref.controlnet_blocks(ref_m, bs, ss, 19):
                a = ref_m(x, enc, pooled, t, img_ids, txt_ids, torch.tensor([3.5]), return_dict=False)[0]
            if i < steps - 1:
                stats_ref = [list(ref_m.norm_ratio), list(ref_m.norm_std), list(ref_m.cos_dis)]
            b = ours(x, enc, pooled, t, img_ids, txt_ids, torch.tensor([3.5]), return_dict=False, controlnet_block_samples=bs,
                     controlnet_single_block_samples=ss)[0]
            if i < steps - 1:
                stats_ours = [list(ours.norm_ratio), list(ours.norm_std), list(ours.cos_dis)]
            assert rel_l2(b, a) <= 0.15
    assert all(len(v) == steps - 2 for v in stats_ref + stats_ours)
    for r, o in zip(stats_ref, stats_ours):
        for a, b in zip(o, r):
            assert abs(a - b) <= 2e-2 * abs(b) + 2e-3, (stats_ours, stats_ref)
    assert ours.cnt == 0 and "norm ratio" in capsys.readouterr().out


@pytest.mark.parametrize("bad", ["fp32", "broadcast", "tokens", "empty_double", "empty_single"])
def test_controlnet_sample_validation(emulated, bad):
    model = _as("OurCNV", _model())
    mc.init_magcache_flux(model, 28)
    hs, enc, pooled, img_ids, txt_ids = _inputs()
    kw = {"fp32": dict(controlnet_block_samples=[torch.randn(1, 48, 256)]),
          "broadcast": dict(controlnet_single_block_samples=[torch.zeros(1, 1, 256, dtype=torch.bfloat16)]),
          "tokens": dict(controlnet_block_samples=[torch.zeros(1, 47, 256, dtype=torch.bfloat16)]),
          "empty_double": dict(controlnet_block_samples=[]),
          "empty_single": dict(controlnet_single_block_samples=[])}[bad]
    err = ZeroDivisionError if bad.startswith("empty") else NotImplementedError
    with torch.no_grad(), pytest.raises(err) as e:
        model(hs, enc, pooled, torch.tensor([0.5]), img_ids, txt_ids, torch.tensor([3.5]), **kw)
    if err is NotImplementedError:
        assert "got torch." in str(e.value)
    with pytest.raises(NotImplementedError, match="joint_attention_kwargs"):
        model(hs, enc, pooled, torch.tensor([0.5]), img_ids, txt_ids, torch.tensor([3.5]), joint_attention_kwargs={"scale": 0.5})


def _shard_worker(rank, world, initfile, results):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch.distributed as dist
    import flux_controlnet_ref as cr
    dist.init_process_group("gloo", init_method=f"file://{initfile}", rank=rank, world_size=world)
    try:
        flux_mod.ops = cr.emu
        patch_mod.ops = cr.emu
        torch.Tensor.is_cuda = property(lambda self: True)
        model = _model(2, 2)
        hs, enc, pooled, img_ids, txt_ids = _inputs(3)
        outs = {}
        for name in ("single", "sharded"):
            m = _as("S_" + name, model)
            mc.init_magcache_flux(m, 6, thresh=10.0, K=2, retention_ratio=0.34)  # miss miss hit hit miss miss
            if name == "sharded":
                mc.enable_token_shard(m, rank, world)
            got = []
            with torch.no_grad():
                for i in range(6):
                    bs, ss = _samples(2, seed=i, scale=0.2), _samples(1, seed=30 + i, scale=0.2)
                    got.append(m(hs * (1 - 0.05 * i), enc, pooled, torch.tensor([1.0 - i / 6]), img_ids, txt_ids, torch.tensor([3.5]),
                                 return_dict=False, controlnet_block_samples=bs, controlnet_single_block_samples=ss)[0].clone())
            outs[name] = got
        eng = m._mc_flux_engine
        errs = [float((a.float() - b.float()).abs().max() / b.float().abs().max()) for a, b in zip(outs["sharded"], outs["single"])]
        results[rank] = (errs, eng.n_img, eng.n_img_total)
    finally:
        dist.destroy_process_group()


def test_controlnet_sharded_equals_single_world2():
    """Token-sharded (image rows split over 2 ranks, gloo): each rank adds its own rows of every sample (a view, no copy)."""
    with tempfile.TemporaryDirectory() as d:
        results = mp.get_context("spawn").Manager().dict()
        mp.spawn(_shard_worker, args=(2, os.path.join(d, "init"), results), nprocs=2, join=True)
        assert set(results.keys()) == {0, 1}
        for r in (0, 1):
            errs, n_loc, n_tot = results[r]
            assert n_loc * 2 == n_tot == 48
            assert len(errs) == 6 and max(errs) < 1.2e-2, errs   # as the sharded test without samples: row blocking flips roundings
