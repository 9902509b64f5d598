"""Open-Sora 1.2 videos of 8 s and longer (T > 32 latent frames) without a GPU.

* The restatement (tests/opensora_ref.py) against the fixture made by executing the reference's own STDiT3 and `magcache_forward`
  at T = 40 and T = 70 (tests/golden/make_opensora_long_golden.py): fp32 within 1e-6 rel-L2, bf16 bit for bit, the controller
  attributes bit for bit. This pins the temporal RoPE past position 32 and the temporal attention at long T.
* The engine (`magcache_opensora_forward`, `teacache_opensora_forward`) through the kernel emulation at T = 40 and T = 70 against
  the restatement. tests/opensora_emu.py models the T <= 32 kernel only; here `attention_temporal_d72` is replaced by one that, past
  32 frames, models the chain of the tensor-core kernel (fp32 scores, P rounded to bf16 for PV, fp32 accumulation and row sum of
  the unrounded P, bf16 output).
* `mc_attn_temporal_d72` rejects the shapes whose grid or row index it cannot represent before any launch."""
import contextlib
import copy
import io
import json
import math
import os

import numpy as np
import pytest
import torch

import magcache_b200 as mc
from magcache_b200 import _lib as L
from magcache_b200 import opensora as os_mod
from magcache_b200 import patch as patch_mod

import opensora_emu
import opensora_ref as R
import opensora_tea_ref as TR

GOLD = os.path.join(os.path.dirname(__file__), "golden")
DOC = json.load(open(os.path.join(GOLD, "opensora_long.json")))
ARR = np.load(os.path.join(GOLD, "opensora_long.npz"))
ATTRS = ("t", "accumulated_sim", "accumulated_err", "accumulated_steps", "skip_steps")
BF, F32 = torch.bfloat16, torch.float32


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


# ---- the fixture ----------------------------------------------------------------------------------------------------------
def _fixture_inputs(T):
    B, H, W, cfg = DOC["B"], DOC["H"], DOC["W"], DOC["config"]
    g = torch.Generator().manual_seed(T)
    x = torch.randn(B, 4, T, H, W, generator=g)
    y = torch.randn(B, 1, cfg["model_max_length"], cfg["caption_channels"], generator=g)
    mask = torch.ones(B, cfg["model_max_length"], dtype=torch.long)
    return x, y, dict(mask=mask, fps=torch.tensor([24.0]), height=torch.tensor([8.0 * H]), width=torch.tensor([8.0 * W]))


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("T", DOC["frames"])
def test_restatement_matches_reference_execution(T, dtype):
    m = R.STDiT3(**DOC["config"]).init_synthetic(DOC["seed"]).to(F32 if dtype == "fp32" else BF).eval()
    m.__class__ = type(f"LongOracle_{dtype}", (R.STDiT3,), {})
    R.install_magcache(m.__class__, thresh=0.12, K=3, skip_time=6)
    x, y, kw = _fixture_inputs(T)
    gold = ARR[f"T{T}_{dtype}"]
    attrs = DOC[f"T{T}_attrs_{dtype}"]
    hits = []
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        for i in range(DOC["calls"]):
            out = m(x, torch.tensor(DOC["timesteps"][i]), None, y, **kw)
            hits.append(int(m.last_skip))
            if i in DOC["stored"]:
                want = gold[DOC["stored"].index(i)]
                if dtype == "fp32":
                    err = np.linalg.norm(out.numpy().astype(np.float64) - want) / np.linalg.norm(want)
                    assert err <= 1e-6, (T, i, err)
                else:
                    want = torch.from_numpy(want).view(BF).float()
                    assert torch.equal(out, want), (T, i, float((out - want).abs().max()))
            for a in ATTRS:
                assert float(getattr(m, a)) == attrs[i][a], (T, i, a)
    assert hits == DOC[f"T{T}_mask_{dtype}"]
    assert 0 in hits and 1 in hits


# ---- the engine through the emulation -------------------------------------------------------------------------------------
def attention_temporal_d72(q, k, v, heads, B, T, S, scale=None, out=None, tag=None):
    """`ops.attention_temporal_d72`: T <= 32 is the fp32-P kernel (opensora_emu's model); past 32 frames the tensor-core kernel's
    chain: fp32 scores of the bf16 operands, e = 2^(x - max) in fp32, l = sum e in fp32, O = sum bf16(e) v in fp32, bf16(O / l)."""
    if T <= 32:
        return opensora_emu.attention_temporal_d72(q, k, v, heads, B, T, S, scale, out, tag)
    assert q.shape == (B * T * S, heads * 72)
    scale = 1.0 / math.sqrt(72) if scale is None else scale
    if out is None:
        out = torch.empty(q.shape[0], heads * 72, dtype=BF)
    seq = lambda t: t.to(F32).view(B, T, S, heads, 72).permute(0, 2, 3, 1, 4)  # noqa: E731  [B, S, H, T, 72]
    x = (seq(q) @ seq(k).transpose(-1, -2)) * (scale * 1.4426950408889634)
    e = torch.exp2(x - x.max(-1, keepdim=True).values)
    o = (e.to(BF).float() @ seq(v)) / e.sum(-1, keepdim=True)
    out.copy_(o.permute(0, 3, 1, 2, 4).reshape(B * T * S, heads * 72).to(BF))
    return out


def _namespace(base):
    ns = base()
    ns.attention_temporal_d72 = attention_temporal_d72
    return ns


@pytest.fixture()
def cuda_flag(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))


def _video(B, T, H, W, L=12, cy=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, T, H, W, generator=g)
    d = torch.randn(B, 4, T, H, W, generator=g)
    y = torch.randn(B, 1, L, cy, generator=g)
    mask = torch.ones(B, L, dtype=torch.long)
    mask[-1, L // 2:] = 0
    kw = dict(mask=mask, fps=torch.tensor([24.0]), height=torch.tensor([8.0 * H]), width=torch.tensor([8.0 * W]))
    return (lambda i: x + 0.004 * i * d), y, kw


def _check(i, o, r, r64):
    e_ref = rel_l2(r, r64)
    assert rel_l2(o, r64) <= 1.5 * e_ref + 1e-3, (i, rel_l2(o, r64), e_ref)
    assert rel_l2(o, r) <= 2 * e_ref + 1e-3, (i, rel_l2(o, r), e_ref)


@pytest.mark.parametrize("T", [40, 70])
def test_magcache_engine_long_video(cuda_flag, monkeypatch, T):
    """miss, miss, hit, ... over 5 calls at B = 2, 4 x 6 latents (S = 6), distinct per-sample timesteps."""
    monkeypatch.setattr(os_mod, "ops", _namespace(opensora_emu.namespace))
    base = R.STDiT3(**R.CONFIGS["tiny"]).init_synthetic(0)
    kw_mc = dict(thresh=0.5, K=3, skip_time=2)
    ref, ref64 = copy.deepcopy(base).to(BF), copy.deepcopy(base).double()
    for m, name in ((ref, "RefLong"), (ref64, "RefLong64")):
        m.__class__ = type(name, (R.STDiT3,), {})
        R.install_magcache(m.__class__, **kw_mc)
    ours = copy.deepcopy(base).to(BF)
    ours.__class__ = type("OursLong", (R.STDiT3,), {})
    patch_mod.init_magcache_opensora(ours, **kw_mc)
    latents, y, kw = _video(2, T, 4, 6)
    skips = []
    with torch.no_grad():
        for i in range(5):
            ts = torch.tensor([1000.0 - 37.0 * i, 990.0 - 29.0 * i])
            r = ref(latents(0), ts, None, y, **kw)
            r64 = ref64(latents(0).double(), ts.to(BF).double(), None, y.double(), **kw)
            o = ours(latents(0), ts, None, y, **kw)
            skips.append(bool(ref.last_skip))
            assert bool(ref64.last_skip) == skips[-1]
            _check(i, o, r, r64)
            for a in ATTRS:
                assert getattr(ours, a) == getattr(ref, a), (i, a)
    assert skips[:2] == [False, False] and True in skips, skips


@pytest.mark.parametrize("T", [40, 70])
def test_teacache_engine_long_video(cuda_flag, monkeypatch, T):
    """The forced first call, then distance calls (at least one of them a hit), at B = 2, 4 x 6 latents."""
    monkeypatch.setattr(os_mod, "ops", _namespace(TR.namespace))
    base = R.STDiT3(**R.CONFIGS["tiny"]).init_synthetic(0)
    with torch.no_grad():
        for n, p in base.named_parameters():
            if n.startswith("t_block."):
                p.mul_(0.05)
    ref, ref64 = copy.deepcopy(base).to(BF), copy.deepcopy(base).double()
    for m, name in ((ref, "RefTeaLong"), (ref64, "RefTeaLong64")):
        m.__class__ = type(name, (R.STDiT3,), {})
        TR.install_teacache(m.__class__, 0.2)
    ref64.decisions_from = ref
    ours = copy.deepcopy(base).to(BF)
    ours.__class__ = type("OursTeaLong", (R.STDiT3,), {})
    mc.init_teacache_opensora(ours, rel_l1_thresh=0.2)
    latents, y, kw = _video(2, T, 4, 6)
    ts = [torch.tensor([1000.0 - 30.0 * i] * 2) for i in range(4)]
    all_ts = [int(t[0].to(BF).item()) for t in ts] + [100]
    forced, calcs = [], []
    with torch.no_grad():
        for i in range(4):
            r = ref(latents(i), ts[i], all_ts, y, **kw)
            r64 = ref64(latents(i).double(), ts[i].to(BF).double(), all_ts, y.double(), **kw)
            res_before = ours.previous_residual
            o = ours(latents(i), ts[i], all_ts, y, **kw)
            forced.append(ref.last_forced)
            calcs.append(ref.last_calc)
            _check(i, o, r, r64)
            # the same decision (a compute stores a new residual); the accumulated distance is not compared bit for bit here: at
            # 10^5 elements torch's bf16 means and the engine's fp64 sums may round `rel` one bf16 step apart
            assert (ours.previous_residual is not res_before) == ref.last_calc, i
    assert forced == [True, False, False, False], forced
    assert False in calcs, calcs


def test_emulated_long_chain_against_fp64():
    """The restated chain is the attention itself up to bf16 roundings (within 2^-7 of fp64 in rel-L2) and differs from the
    fp32-P chain of the short kernel."""
    g = torch.Generator().manual_seed(3)
    B, T, S, H = 2, 70, 3, 2
    q, k, v = (torch.randn(B * T * S, H * 72, generator=g).to(BF) for _ in range(3))
    got = attention_temporal_d72(q, k, v, H, B, T, S)
    seq = lambda t: t.double().view(B, T, S, H, 72).permute(0, 2, 3, 1, 4)  # noqa: E731
    r64 = torch.softmax(seq(q) @ seq(k).transpose(-1, -2) / math.sqrt(72), -1) @ seq(v)
    assert rel_l2(seq(got), r64) < 2.0 ** -7


# ---- argument checks ------------------------------------------------------------------------------------------------------
def test_temporal_rejects_unrepresentable_shapes():
    """Past 32 frames the grid is one flat dimension of B*S*heads*ceil(T/64) CTAs and the frame rows are int32: a shape beyond
    either returns MC_ERR_INVALID before any launch (the checks need no device)."""
    p = 1 << 20  # any 16-byte aligned non-null address: the call returns before it is read

    def call(B, T, S, heads):
        ld = heads * 72
        return L.lib.mc_attn_temporal_d72(p, ld, p, ld, p, ld, p, ld, B, T, S, heads, 0.1, None)

    assert call(1, 33, 40000, 65535) == L.MC_ERR_INVALID      # 2.6e9 CTAs
    assert call(2, 240, 5_000_000, 1) == L.MC_ERR_INVALID     # 2.4e9 rows
    assert call(1, 0, 1, 1) == L.MC_ERR_INVALID
