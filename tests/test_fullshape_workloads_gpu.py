"""Parity at the full single-GPU shapes of BASELINE.json's other workloads: FLUX.1-dev 1024x1024 (4096 image + 512 text tokens,
hidden 3072, 24 heads), HunyuanVideo 720p x 129 frames (33 x 45 x 80 = 118 800 image tokens + the valid text tokens, hidden 3072,
24 heads, single-stream linear1 3072 -> 21 504, linear2 K = 15 360) and Wan2.1-T2V-14B 1280x720x81 (21 x 45 x 80 = 75 600 tokens,
dim 5120, 40 heads, ffn 13 824).

(a) One-layer, full-width models of each family through the patched forward (miss, miss, hit, hit), against the bf16 oracle and
    an fp64 evaluation of the same network, at DESIGN §5's rule: rel-L2(ours, oracle) <= 2 e_ref + 1e-3 and rel-L2(ours, fp64)
    <= 1.5 e_ref + 1e-3 with e_ref = rel-L2(oracle, fp64), for the output and for the residual cache; controller state bit-equal.
    Both references run on the GPU (test infrastructure, never the product path). The oracle's attention as written cannot run
    at these lengths (HunyuanVideo's `segment_attention` builds a dense L x L mask: 14 GB of bools at 119 k tokens), so
    `_oracle_on_gpu` replaces it, test-locally, by a query-chunked evaluation of the same rule: same-segment keys (HunyuanVideo),
    the first `k_lens` keys (Wan), every key (FLUX); bf16 through SDPA on chunks, fp64 through matmul / softmax. It also runs the
    oracle helpers that build host tensors (timestep sinusoids, FLUX's RoPE table, the segment ids) on host copies of their
    inputs, and evaluates HunyuanVideo's fp64 single-stream block and MLPs in row chunks, which keeps the 20 GB linear1 output
    and the 12 GB MLP activations off the card. CPU tests pin every replacement to the oracle's own function.
(b) Each kernel at the launch shapes only these workloads issue, per element against fp64 with the criteria of the existing
    kernel tests (imported from test_kernel_bounds_gpu.py), with fenced outputs: attention over 119 056 / 75 600 / 4608 keys,
    q|k RMSNorm + RoPE at row offsets past 2^31 elements, the GEMMs of linear1 / linear2 and of Wan-14B's qkv / ffn, K7, the head
    and K3 at 75 600 - 119 056 rows.

`test_shape_table_matches_the_engines` and the chunked-reference tests run without a GPU."""
import contextlib
import copy
import gc
import math
import os
import sys
import time
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_bounds_gpu import (BF, F32, _assert_ulps, _fill_bytes_ok, _ln_chain, _rb, _rms_rope_ref, _rope64, _stats_chain,  # noqa: E402
                                    FENCE_BYTE, check_fence, fenced, gemm_fp64_bounds_ok)
from test_head_readout_gpu import NORTH_STAR, head_chain  # noqa: E402
from oracle import hunyuan_ref as _hr  # noqa: E402

DEV = "cuda"

# ------------------------------------------------------------------------------------------- the shapes
# FLUX.1-dev 1024 x 1024: 128 x 128 latents packed 2 x 2 -> 64 x 64 image tokens, 512 T5 tokens (text rows first).
FLUX = dict(hidden=3072, heads=24, h_tok=64, w_tok=64, n_img=4096, n_txt=512, text_dim=4096, pooled=768, linear1=21504, linear2=15360)
# HunyuanVideo 720p x 129 frames: latents 16 x 33 x 90 x 160, patch (1, 2, 2); 256 text positions, the valid ones a strict
# prefix; image rows first, then the valid text rows. The kernel checks take every text position valid (the longest sequence).
HUNYUAN = dict(hidden=3072, heads=24, latent=(16, 33, 90, 160), grid=(33, 45, 80), n_img=118800, text_len=256, valid=229,
               text_dim=4096, pooled=768, linear1=21504, linear2=15360)
# Wan2.1-T2V-14B 1280 x 720 x 81: latents 16 x 21 x 90 x 160, patch (1, 2, 2).
WAN14B = dict(dim=5120, heads=40, ffn=13824, latent=(16, 21, 90, 160), grid=(21, 45, 80), n_tok=75600, qkv=15360)
HY_ROWS = HUNYUAN["n_img"] + HUNYUAN["text_len"]  # 119 056: the longest HunyuanVideo sequence at this size


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def _need_device_memory(gib):
    total = torch.cuda.get_device_properties(0).total_memory
    if total < gib * 2 ** 30:
        pytest.skip(f"needs a device with {gib} GiB of memory, this one has {total / 2 ** 30:.0f} GiB")
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def _report(what, t0):
    print(f"[{what}] peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB, wall {time.time() - t0:.1f} s")


# ------------------------------------------------------------------------------------------- chunked reference attention
def sdpa_chunked(q, k, v, budget=1 << 30):
    """softmax(q k^T / sqrt(d)) v for q [B, H, Lq, d] and k / v [B, H, Lk, d], one block of query rows at a time. fp64: explicit
    matmul and softmax, blocks sized so one block's scores take at most `budget` bytes; other dtypes: torch SDPA per block (each
    query row's result does not depend on the other rows)."""
    B, H, Lq, d = q.shape
    Lk = k.shape[2]
    out = torch.empty(B, H, Lq, v.shape[-1], dtype=q.dtype, device=q.device)
    if q.dtype == torch.float64:
        kt, v = k.transpose(-1, -2).contiguous(), v.contiguous()
        rows = max(1, budget // (B * H * Lk * 8))
        for r0 in range(0, Lq, rows):
            s = (q[:, :, r0:r0 + rows] @ kt) / math.sqrt(d)
            out[:, :, r0:r0 + rows] = torch.softmax(s, -1) @ v
    else:
        for r0 in range(0, Lq, 16384):
            out[:, :, r0:r0 + 16384] = F.scaled_dot_product_attention(q[:, :, r0:r0 + 16384], k, v)
    return out


def hunyuan_segment_attention(q, k, v, seg_ids):
    """`hunyuan_ref.segment_attention` ([B, L, H, D]; tokens attend inside their own segment) without the dense L x L mask: the
    segments of `get_cu_seqlens` are contiguous row ranges, each evaluated on its own keys."""
    B, L, H, d = q.shape
    out = torch.empty(B, H, L, d, dtype=q.dtype, device=q.device)
    ids = seg_ids.cpu()
    for b in range(B):
        for s in torch.unique(ids[b]).tolist():
            idx = (ids[b] == s).nonzero().flatten()
            r0, r1 = int(idx[0]), int(idx[-1]) + 1
            assert r1 - r0 == idx.numel(), "segments are contiguous"
            out[b:b + 1, :, r0:r1] = sdpa_chunked(*(t[b:b + 1, r0:r1].transpose(1, 2) for t in (q, k, v)))
    return out.transpose(1, 2).reshape(B, L, -1)


def wan_attention(q, k, v, k_lens=None):
    """`wan_ref.attention_ref` ([B, L, H, hd], in the oracle's current dtype) with the `k_lens` mask as a key range."""
    from oracle import wan_ref
    q, k, v = (t.transpose(1, 2).to(wan_ref.BF16) for t in (q, k, v))
    out = torch.empty_like(q)
    for b in range(q.shape[0]):
        n = k.shape[2] if k_lens is None else int(k_lens[b])
        out[b:b + 1] = sdpa_chunked(q[b:b + 1], k[b:b + 1, :, :n], v[b:b + 1, :, :n])
    return out.transpose(1, 2).contiguous()


class _FluxFunctional:
    """torch.nn.functional for `flux_ref`, with `scaled_dot_product_attention` (plain attention, no mask) evaluated in chunks."""

    def __getattr__(self, name):
        return getattr(F, name)

    @staticmethod
    def scaled_dot_product_attention(q, k, v, **kw):
        assert not kw
        return sdpa_chunked(q, k, v)


def _on_host(fn):
    """An oracle helper that builds host tensors (`torch.arange` without a device) run on host copies of its tensor arguments,
    its result moved back to the caller's device: the same arithmetic as on a CPU run of the oracle, only placed elsewhere."""
    def wrapped(*args, **kw):
        dev = next(a.device for a in args if torch.is_tensor(a))
        out = fn(*[a.cpu() if torch.is_tensor(a) else a for a in args], **kw)
        return tuple(o.to(dev) for o in out) if isinstance(out, tuple) else out.to(dev)
    return wrapped


def hunyuan_single_block_rows(self, x, vec, txt_len, seg_ids, freqs_cis, rows=8192):
    """`MMSingleStreamBlock.forward` evaluated in fp64 with its row-local layers (LN + modulation, linear1, q / k RMSNorm, RoPE,
    GELU, linear2, the gated residual) in blocks of `rows` tokens and the attention over the whole sequence. The [L, 21 504] linear1
    output never exists at once: its q | k | v columns are kept, the MLP columns are recomputed per block for linear2. Other
    dtypes take the block as written."""
    from oracle import hunyuan_ref as hr
    if hr.DT != torch.float64:
        return _SINGLE_FORWARD(self, x, vec, txt_len, seg_ids, freqs_cis)
    shift, scale, gate = self.modulation(vec).chunk(3, dim=-1)
    b, l, _ = x.shape
    n_img = l - txt_len
    q, k, v = (torch.empty(b, l, self.heads, self.hidden // self.heads, dtype=x.dtype, device=x.device) for _ in range(3))

    def linear1(r0, r1):
        return torch.split(self.linear1(hr.modulate(hr._ln(x[:, r0:r1]), shift, scale)), [3 * self.hidden, self.mlp_hidden], dim=-1)

    for r0 in range(0, l, rows):
        r1 = min(r0 + rows, l)
        cq, ck, cv = linear1(r0, r1)[0].view(b, r1 - r0, 3, self.heads, -1).unbind(2)
        cq, ck = self.q_norm(cq).to(cv), self.k_norm(ck).to(cv)
        if freqs_cis is not None and r0 < n_img:
            m = min(r1, n_img) - r0
            iq, ik = hr.apply_rotary_emb(cq[:, :m], ck[:, :m], tuple(f[r0:r0 + m] for f in freqs_cis))
            cq, ck = torch.cat((iq, cq[:, m:]), 1), torch.cat((ik, ck[:, m:]), 1)
        q[:, r0:r1], k[:, r0:r1], v[:, r0:r1] = cq, ck, cv
    attn = hr.segment_attention(q, k, v, seg_ids)
    del q, k, v
    out = torch.empty_like(x)
    for r0 in range(0, l, rows):
        r1 = min(r0 + rows, l)
        mlp = linear1(r0, r1)[1]
        out[:, r0:r1] = x[:, r0:r1] + hr.apply_gate(self.linear2(torch.cat((attn[:, r0:r1], self.mlp_act(mlp)), 2)), gate)
    return out


_SINGLE_FORWARD = _hr.MMSingleStreamBlock.forward  # as written, for the bf16 oracle


def hunyuan_mlp_rows(self, x, rows=8192):
    """`hunyuan_ref.MLP.forward` (fc2(act(fc1(x))), row-local) evaluated in fp64 one block of `rows` tokens at a time, so the
    double-stream block's [L, 12 288] hidden activations never exist at once. Other dtypes take the MLP as written."""
    if _hr.DT != torch.float64 or x.shape[1] <= rows:
        return _MLP_FORWARD(self, x)
    return torch.cat([_MLP_FORWARD(self, x[:, r0:r0 + rows]) for r0 in range(0, x.shape[1], rows)], 1)


_MLP_FORWARD = _hr.MLP.forward


def _oracle_on_gpu(monkeypatch):
    """Test-local replacements that let the oracles run at these shapes on the GPU (see the module docstring)."""
    from oracle import flux_ref as fr
    from oracle import hunyuan_ref as hr
    from oracle import wan_ref
    monkeypatch.setattr(hr, "segment_attention", hunyuan_segment_attention)
    monkeypatch.setattr(hr, "seg_ids_from_mask", _on_host(hr.seg_ids_from_mask))
    monkeypatch.setattr(hr, "timestep_embedding", _on_host(hr.timestep_embedding))
    monkeypatch.setattr(hr.MMSingleStreamBlock, "forward", hunyuan_single_block_rows)
    monkeypatch.setattr(hr.MLP, "forward", hunyuan_mlp_rows)
    monkeypatch.setattr(fr, "F", _FluxFunctional())
    monkeypatch.setattr(fr, "get_timestep_embedding", _on_host(fr.get_timestep_embedding))
    monkeypatch.setattr(fr, "rope_freqs", _on_host(fr.rope_freqs))
    monkeypatch.setattr(wan_ref, "attention_ref", wan_attention)


# ------------------------------------------------------------------------------------------- CPU: the replacements and the shapes
def test_chunked_attention_equals_the_oracle_functions():
    """At small shapes on the CPU: the chunked evaluations equal the oracle's dense functions — fp64 within 1e-12 relative, bf16
    within a bf16 rounding — for a HunyuanVideo mask with padded text, Wan `k_lens` shorter than the sequence, and FLUX's plain
    attention; and the row-blocked fp64 single-stream block and MLP equal `MMSingleStreamBlock.forward` / `MLP.forward` within
    1e-12, with blocks that straddle the image / text boundary."""
    from oracle import hunyuan_ref as hr
    from oracle import wan_ref
    g = torch.Generator().manual_seed(0)
    B, L, H, d = 1, 45, 3, 16

    def qkv(dt):
        return [torch.randn(B, L, H, d, generator=g, dtype=torch.float64).to(dt) for _ in range(3)]

    mask = torch.zeros(1, 9, dtype=torch.long)
    mask[0, :5] = 1
    seg = hr.seg_ids_from_mask(mask, L - 9)
    assert len(torch.unique(seg)) == 2
    for dt in (torch.float64, torch.bfloat16):
        tol = 1e-12 if dt == torch.float64 else 2.0 ** -7
        q, k, v = qkv(dt)
        want = hr.segment_attention(q, k, v, seg)
        assert rel_l2(hunyuan_segment_attention(q, k, v, seg), want) <= tol, dt
        kl = torch.tensor([L - 7])
        ctx = wan_ref.exact_fp64() if dt == torch.float64 else contextlib.nullcontext()
        with ctx:
            want = wan_ref.attention_ref(q, k, v, k_lens=kl)
            assert rel_l2(wan_attention(q, k, v, k_lens=kl), want) <= tol, dt
            assert rel_l2(wan_attention(q, k, v), wan_ref.attention_ref(q, k, v)) <= tol, dt
        qh, kh, vh = (t.transpose(1, 2) for t in (q, k, v))
        assert rel_l2(_FluxFunctional.scaled_dot_product_attention(qh, kh, vh), F.scaled_dot_product_attention(qh, kh, vh)) <= tol, dt
    # the budget forces one-row blocks: every block boundary is exercised
    q, k, v = (t.transpose(1, 2) for t in qkv(torch.float64))
    assert rel_l2(sdpa_chunked(q, k, v, budget=1), F.scaled_dot_product_attention(q, k, v)) <= 1e-12

    blk = hr.MMSingleStreamBlock(64, 2).double()
    with torch.no_grad():
        for p in blk.parameters():
            p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64) * 0.2)
    n_img, n_txt = 21, 9
    x = torch.randn(1, n_img + n_txt, 64, generator=g, dtype=torch.float64)
    vec = torch.randn(1, 64, generator=g, dtype=torch.float64)
    cos, sin = (t.double() for t in hr.rope_cos_sin((1, 3, 7), head_dim=32, axes=(8, 12, 12)))
    m = torch.zeros(1, n_txt, dtype=torch.long)
    m[0, :6] = 1
    seg = hr.seg_ids_from_mask(m, n_img)
    with torch.no_grad(), hr.exact():
        want = _SINGLE_FORWARD(blk, x, vec, n_txt, seg, (cos, sin))
        for rows in (4, 7, 30):
            got = hunyuan_single_block_rows(blk, x, vec, n_txt, seg, (cos, sin), rows=rows)
            assert rel_l2(got, want) <= 1e-12, rows
        mlp = hr.MLP(64, 96, torch.nn.GELU(approximate="tanh")).double()
        for rows in (4, 7, 30):
            assert rel_l2(hunyuan_mlp_rows(mlp, x, rows=rows), _MLP_FORWARD(mlp, x)) <= 1e-12, rows


def test_oracle_host_helpers_keep_their_values():
    """`_on_host` returns the helper's own result (bit for bit) on the caller's device."""
    from oracle import flux_ref as fr
    from oracle import hunyuan_ref as hr
    t = torch.tensor([731.0])
    assert torch.equal(_on_host(hr.timestep_embedding)(t), hr.timestep_embedding(t))
    ids = torch.cat(fr.make_ids(4, 5, 3)[::-1])
    for a, b in zip(_on_host(fr.rope_freqs)(ids, (16, 56, 56)), fr.rope_freqs(ids, (16, 56, 56))):
        assert torch.equal(a, b)


def test_shape_table_matches_the_engines():
    """The shapes the GPU tests use are the ones the engines derive from the models and the latents: token counts (the oracle's
    patch embedding on the latent shape), where the text tail sits in the key order (the oracle's segments, the engines' row
    slices), and the widths of the single-stream linear1 / linear2 against the engines' buffers. Models and engine buffers live
    on the meta device: shapes only."""
    from magcache_b200.mmdit import FluxEngine, HunyuanEngine
    from magcache_b200.wan import WAN_CONFIGS, WanEngine
    from oracle import flux_ref as fr
    from oracle import hunyuan_ref as hr
    from oracle import wan_ref
    meta = torch.device("meta")

    # HunyuanVideo
    hy = HUNYUAN
    with meta:
        m = hr.HYVideoDiffusionTransformer(hidden_size=hy["hidden"], heads_num=hy["heads"], mm_double_blocks_depth=1, mm_single_blocks_depth=1,
                                           text_states_dim=hy["text_dim"], text_states_dim_2=hy["pooled"])
        n_img = m.img_in(torch.empty(1, *hy["latent"])).shape[1]
    assert n_img == hy["n_img"] == math.prod(hy["grid"]) and HY_ROWS == 119056
    s = m.single_blocks[0]
    assert s.linear1.out_features == hy["linear1"] and s.linear2.in_features == hy["linear2"] and s.heads * 128 == hy["hidden"]
    mask = torch.zeros(1, hy["text_len"], dtype=torch.long)
    mask[0, :hy["valid"]] = 1
    seg = hr.seg_ids_from_mask(mask, n_img)[0]
    assert int((seg == seg[0]).sum()) == n_img + hy["valid"] and 0 < hy["valid"] < hy["text_len"]  # [image | valid text] | padding
    w = types.SimpleNamespace(device=meta, dim=hy["hidden"], heads=hy["heads"], ada_rows=1, in_channels=16, text_dim=hy["text_dim"],
                              pooled_dim=hy["pooled"], r_ada_w=torch.empty(2 * hy["hidden"], hy["hidden"], device=meta))
    e = HunyuanEngine(w)
    lat = hy["latent"]
    e._workspace((lat[1], lat[2] // 2, lat[3] // 2), hy["valid"])  # the grid `stage_inputs` derives from x [1, 16, T, H, W]
    assert e.img == slice(0, n_img) and e.txt == slice(n_img, n_img + hy["valid"]) and e.S_keys == n_img + hy["valid"]
    # single-stream block: linear1 = q | k (qk), v, MLP (cat[:, D:]); linear2 reads cat = [attention | GELU(MLP)]
    D = hy["hidden"]
    assert e.qk.shape[1] + e.v.shape[1] + (e.cat.shape[1] - D) == hy["linear1"] and e.cat.shape[1] == hy["linear2"]

    # FLUX.1-dev 1024 x 1024
    fl = FLUX
    with meta:
        m = fr.FluxTransformer2DModel(num_layers=1, num_single_layers=1, num_attention_heads=fl["heads"])
    img_ids, txt_ids = fr.make_ids(fl["h_tok"], fl["w_tok"], fl["n_txt"])
    assert img_ids.shape[0] == fl["n_img"] == (1024 // 16) ** 2
    s = m.single_transformer_blocks[0]
    assert 3 * s.attn.to_q.out_features + s.proj_mlp.out_features == fl["linear1"] and s.proj_out.in_features == fl["linear2"]
    w = types.SimpleNamespace(device=meta, dim=fl["hidden"], heads=fl["heads"], ada_rows=1, in_channels=64, joint_dim=fl["text_dim"],
                              pooled_dim=fl["pooled"])
    e = FluxEngine(w)
    e._workspace(fl["n_img"], fl["n_txt"])
    assert e.txt == slice(0, fl["n_txt"]) and e.img == slice(fl["n_txt"], fl["n_txt"] + fl["n_img"]) and e.S_keys == 4608
    assert e.qk.shape[1] + e.v.shape[1] + (e.cat.shape[1] - fl["hidden"]) == fl["linear1"] and e.cat.shape[1] == fl["linear2"]

    # Wan2.1-T2V-14B 1280 x 720 x 81
    wn = WAN14B
    dims = WAN_CONFIGS["t2v-14B"]
    assert (dims.dim, dims.num_heads, dims.ffn_dim) == (wn["dim"], wn["heads"], wn["ffn"])
    with meta:
        m = wan_ref.WanModel(**wan_ref.CONFIGS["t2v-14B"])
        grid = tuple(m.patch_embedding(torch.empty(1, *wn["latent"])).shape[2:])
    assert grid == wn["grid"] and math.prod(grid) == wn["n_tok"]
    e = WanEngine(types.SimpleNamespace(dims=dims, device=meta, head_wt=None, head_b=None))
    e._workspace(wn["n_tok"])
    assert e.qkv.shape == (wn["n_tok"], wn["qkv"]) and e.ffn.shape == (wn["n_tok"], wn["ffn"]) and e.n_keys == wn["n_tok"]


# ------------------------------------------------------------------------------------------- (a) one-layer forwards
def rule_fraction(out, ref, exact):
    """DESIGN §5's rule without the assertion: (e_ref, e_ours, e_vs, the larger of the two errors as a fraction of its bound).
    The rule holds exactly when the fraction is <= 1."""
    e_ref, e_vs, e_ours = rel_l2(ref, exact), rel_l2(out, ref), rel_l2(out, exact)
    return e_ref, e_ours, e_vs, max(e_vs / (2.0 * e_ref + 1e-3), e_ours / (1.5 * e_ref + 1e-3))


def _rule(what, out, ref, exact, verbose=True):
    """DESIGN §5's rule; returns the larger of its two errors as a fraction of its bound."""
    e_ref, e_ours, e_vs, frac = rule_fraction(out, ref, exact)
    if verbose:
        print(f"  {what}: ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e} | ours vs oracle {e_vs:.3e}")
    assert e_vs <= 2.0 * e_ref + 1e-3 and e_ours <= 1.5 * e_ref + 1e-3, (what, e_ours, e_ref, e_vs)
    return frac


def _forward_loop(name, calls, ours, ref_m, m64, exact_ctx, res_attr, attrs, check=None):
    """Per call: our forward, the bf16 oracle, the fp64 oracle (each result moved to the host at once), then DESIGN §5's rule
    on the output and on the residual cache, and the controller attributes bit-equal; `check(i, out, ref, ex, r_ours, r_ref,
    r_ex)`, when given, holds parts of the same host tensors to more rules. Returns the oracle's skip decisions."""
    skips = []
    for i, (args_ours, args_ref, args_64) in enumerate(calls):
        with torch.no_grad():
            out = ours(*args_ours).float().cpu()
            r_ours = res_attr(ours).float().cpu()
            ref = ref_m(*args_ref).float().cpu()
            r_ref = res_attr(ref_m).float().cpu()
            torch.cuda.empty_cache()
            with exact_ctx():
                ex = m64(*args_64).cpu()
            r_ex = res_attr(m64).float().cpu()
            torch.cuda.empty_cache()
        skips.append(int(ref_m.last_skip))
        print(f"[{name}] call {i} ({'hit' if skips[-1] else 'miss'})")
        assert out.shape == ref.shape == ex.shape
        _rule("output", out, ref, ex)
        _rule("residual cache", r_ours, r_ref, r_ex)
        if check is not None:
            check(i, out, ref, ex, r_ours, r_ref, r_ex)
        for a in attrs:
            vals = [np.asarray(getattr(m, a), dtype=np.float64).tolist() for m in (ours, ref_m, m64)]
            assert vals[0] == vals[1] == vals[2], (i, a, vals)
        del out, ref, ex, r_ours, r_ref, r_ex
    return skips


@pytest.mark.gpu
def test_hunyuan_720p_129f_one_layer_forward(monkeypatch):
    """HunyuanVideo at 720p x 129 frames, one double + one single block at hidden 3072 / 24 heads, text 256 x 4096 with 229 valid
    (a strict prefix), pooled 768: miss, miss, hit, hit."""
    import magcache_b200 as mc
    from oracle import hunyuan_ref as hr
    _need_device_memory(75)
    _oracle_on_gpu(monkeypatch)
    t0 = time.time()
    hy = HUNYUAN
    model = hr.HYVideoDiffusionTransformer(hidden_size=hy["hidden"], heads_num=hy["heads"], mm_double_blocks_depth=1, mm_single_blocks_depth=1,
                                           text_states_dim=hy["text_dim"], text_states_dim_2=hy["pooled"], guidance_embed=True).init_synthetic(31)
    g = torch.Generator().manual_seed(31)
    x = torch.randn(1, *hy["latent"], generator=g).bfloat16().to(DEV)
    txt = torch.randn(1, hy["text_len"], hy["text_dim"], generator=g).bfloat16().to(DEV)
    mask = torch.zeros(1, hy["text_len"], dtype=torch.long)
    mask[0, :hy["valid"]] = 1
    mask = mask.to(DEV)
    pooled = torch.randn(1, hy["pooled"], generator=g).bfloat16().to(DEV)
    cos, sin = (t.to(DEV) for t in hr.rope_cos_sin(hy["grid"]))
    gd = torch.tensor([6000.0], device=DEV)
    steps, table = 5, [1.0] + [0.98] * 4  # retention 0.4: calls 0 and 1 miss, thresh 10 / K 3: calls 2 and 3 hit
    kw = dict(thresh=10.0, K=3, retention_ratio=0.4)
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("OurHYFull", (ours.__class__,), {})
    mc.init_magcache_hunyuan(ours, steps, mag_ratios=table, **kw)
    ref_m = copy.deepcopy(model).to(DEV)
    ref_m.__class__ = type("RefHYFull", (ref_m.__class__,), {})
    hr.install_magcache(type(ref_m), table, steps, **kw)
    m64 = copy.deepcopy(model).to(DEV).double()
    m64.__class__ = type("RefHYFull64", (m64.__class__,), {})
    hr.install_magcache(type(m64), table, steps, **kw)
    del model
    calls = []
    for i in range(4):
        t = torch.tensor([900.0 - 110.0 * i], device=DEV)
        calls.append(((x, t, txt, mask, pooled, cos, sin, gd, False), (x, t, txt, mask, pooled, cos, sin, gd, False),
                      (x.double(), t.double(), txt.double(), mask, pooled.double(), cos.double(), sin.double(), gd.double(), False)))
    skips = _forward_loop("hunyuan 720p x 129f", calls, ours, ref_m, m64, hr.exact, lambda m: m.residual_cache,
                          ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"))
    assert skips == [0, 0, 1, 1], skips
    _report("hunyuan 720p x 129f forward", t0)


@pytest.mark.gpu
def test_flux_1024_one_layer_forward(monkeypatch):
    """FLUX.1-dev at 1024 x 1024, one double + one single block at 3072 / 24 heads, 512 text tokens of width 4096, pooled 768:
    miss, miss, hit, hit.

    The reference rounds the timestep and the guidance to bf16 and multiplies them by 1000 in bf16 (magcache_flux.py:292-293);
    the fp64 evaluation does neither. With FLUX-dev's guidance 3.5 the bf16 side embeds 3504 and the fp64 side 3500, the
    sinusoid's fastest channels differ by radians, and e_ref measures that input difference (0.04 on the output, 0.24 on the
    residual) instead of arithmetic error. Guidance 4 and the timesteps 1, 1/2, 1/4, 1/8 are exact in bf16 before and after
    the product, so both references embed the same values."""
    import magcache_b200 as mc
    from oracle import flux_ref as fr
    _need_device_memory(40)
    _oracle_on_gpu(monkeypatch)
    t0 = time.time()
    fl = FLUX
    model = fr.FluxTransformer2DModel(in_channels=64, num_layers=1, num_single_layers=1, num_attention_heads=fl["heads"],
                                      joint_attention_dim=fl["text_dim"], pooled_projection_dim=fl["pooled"], guidance_embeds=True).init_synthetic(21)
    g = torch.Generator().manual_seed(21)
    hs = torch.randn(1, fl["n_img"], 64, generator=g).bfloat16().to(DEV)
    enc = torch.randn(1, fl["n_txt"], fl["text_dim"], generator=g).bfloat16().to(DEV)
    pooled = torch.randn(1, fl["pooled"], generator=g).bfloat16().to(DEV)
    img_ids, txt_ids = (t.to(DEV) for t in fr.make_ids(fl["h_tok"], fl["w_tok"], fl["n_txt"]))
    gd = torch.tensor([4.0], device=DEV)
    steps, table = 5, [1.0] + [0.98] * 4
    kw = dict(thresh=10.0, K=3, retention_ratio=0.4)
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("OurFluxFull", (ours.__class__,), {})
    mc.init_magcache_flux(ours, steps, mag_ratios=table, **kw)
    ref_m = copy.deepcopy(model).to(DEV)
    ref_m.__class__ = type("RefFluxFull", (ref_m.__class__,), {})
    fr.install_magcache(type(ref_m), table, steps, **kw)
    m64 = copy.deepcopy(model).to(DEV).double()
    m64.__class__ = type("RefFluxFull64", (m64.__class__,), {})
    fr.install_magcache(type(m64), table, steps, **kw)
    calls = []
    for tv in (1.0, 0.5, 0.25, 0.125):
        t = torch.tensor([tv], device=DEV)
        a = (hs, enc, pooled, t, img_ids, txt_ids, gd)
        calls.append((a, a, (hs.double(), enc.double(), pooled.double(), t.double(), img_ids, txt_ids, gd.double())))

    assert all(float(v.bfloat16()) == float(v) and float(v.bfloat16() * 1000) == float(v) * 1000 for v in (gd, *(c[0][3] for c in calls)))
    skips = _forward_loop("flux 1024", calls, _Delegate(ours), _Delegate(ref_m), _Delegate(m64), fr.exact, lambda m: m.previous_residual,
                          ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"))
    assert skips == [0, 0, 1, 1], skips
    _report("flux 1024 forward", t0)


class _Delegate:
    """A FLUX model called with return_dict=False, its first output returned; attributes read through."""

    def __init__(self, m):
        object.__setattr__(self, "_m", m)

    def __call__(self, *a):
        return self._m(*a, return_dict=False)[0]

    def __getattr__(self, name):
        return getattr(self._m, name)


@pytest.mark.gpu
def test_wan14b_720p_one_layer_forward(monkeypatch):
    """Wan2.1-T2V-14B at 1280 x 720 x 81, one block at dim 5120 / 40 heads / ffn 13 824: miss, miss, hit, hit over both CFG
    slots (cond, uncond, cond, uncond)."""
    import magcache_b200 as mc
    from oracle import wan_ref
    _need_device_memory(75)
    _oracle_on_gpu(monkeypatch)
    t0 = time.time()
    wn = WAN14B
    model = wan_ref.WanModel(dim=wn["dim"], ffn_dim=wn["ffn"], num_heads=wn["heads"], num_layers=1).init_synthetic(41)
    g = torch.Generator().manual_seed(42)
    lat = torch.randn(*wn["latent"], generator=g).to(DEV)
    ctx, ctx_null = torch.randn(400, 4096, generator=g).to(DEV), torch.randn(77, 4096, generator=g).to(DEV)
    t = torch.tensor([640.0], device=DEV)
    steps, table = 4, [1.0] * 2 + [0.97] * 6  # thresh 10 makes every eligible call a hit (the window opens at cnt 2)
    kw = dict(thresh=10.0, K=3, retention_ratio=0.25)
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("OursWanFull", (ours.__class__,), {})
    mc.init_magcache(ours, steps, mag_ratios=table, **kw)
    ref_m = copy.deepcopy(model).to(DEV)
    ref_m.__class__ = type("RefWanFull", (ref_m.__class__,), {})
    wan_ref.install_magcache(ref_m.__class__, table, steps, **kw)
    m64 = copy.deepcopy(model).to(DEV).double()
    m64.__class__ = type("RefWanFull64", (m64.__class__,), {})
    wan_ref.install_magcache(m64.__class__, table, steps, **kw)
    del model
    n = wn["n_tok"]

    class Call:
        def __init__(self, m, dt):
            self.m, self.dt = m, dt

        def __call__(self, c):
            return self.m([lat.to(self.dt)], t=t.to(self.dt) if self.dt == torch.float64 else t, context=[c.to(self.dt)], seq_len=n)[0]

        def __getattr__(self, name):
            return getattr(self.m, name)

    calls = [((c,), (c,), (c,)) for c in (ctx, ctx_null, ctx, ctx_null)]

    def res(m):  # the residual cache of the slot the call just wrote (cnt has advanced by one)
        return m.residual_cache[(m.cnt - 1) % 2][0]

    skips = _forward_loop("wan2.1-14B 720p", calls, Call(ours, torch.float32), Call(ref_m, torch.float32), Call(m64, torch.float64),
                          wan_ref.exact_fp64, res, ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"))
    assert skips == [0, 0, 1, 1], skips
    _report("wan2.1-14B 720p forward", t0)


# ------------------------------------------------------------------------------------------- (b) kernels at the launch shapes
def _fill(view, g, scale=1.0, shift=0.0, rows=8192):
    """Normal random values into a (possibly huge, strided) view, one block of rows at a time."""
    for r0 in range(0, view.shape[0], rows):
        blk = view[r0:r0 + rows]
        blk.copy_(torch.randn(blk.shape, device=DEV, generator=g) * scale + shift)


def _tiles(M, tile=128):
    """Row indices of the first, a middle and the last (ragged) `tile`-row tile of M rows."""
    mid = (M // 2) // tile * tile
    last = (M - 1) // tile * tile
    return torch.cat([torch.arange(0, min(tile, M)), torch.arange(mid, min(mid + tile, M)), torch.arange(last, M)]).unique().to(DEV)


def _attn_ref64(q, k, v, heads):
    """fp64 softmax(q k^T / sqrt(128)) v over every key, for the query rows given."""
    qh = q.double().view(q.shape[0], heads, 128).transpose(0, 1)[None]
    kh, vh = (t.double().view(t.shape[0], heads, 128).transpose(0, 1)[None] for t in (k, v))
    return sdpa_chunked(qh, kh, vh)[0].transpose(0, 1).reshape(q.shape[0], -1)


def _attention_case(name, L, heads, ld, slices, scaled_slice, g):
    """q | k | v as column slices of one [L, ld] bf16 buffer (NaN columns past v), or with ld None in the MMDiT engine's layout:
    q | k in an [L, 2 W] buffer and v in an [L, W] one (ldq = ldk = 2 W, ldv = W); 128 NaN rows after the key rows either way.
    The output a window of a fenced buffer, the split-KV workspace a fenced buffer of exactly `mc_attn_workspace_bytes`; the
    query `slices` against fp64 over the whole key sequence at test_attention_full_key_sequence_vs_fp64's criterion; then q scaled
    6.5x (peaked softmax) on `scaled_slice`."""
    import ctypes
    from magcache_b200 import _lib as L_
    from magcache_b200 import ops
    W = heads * 128
    if ld is None:
        qk = torch.full((L + 128, 2 * W), float("nan"), dtype=BF, device=DEV)
        vb = torch.full((L + 128, W), float("nan"), dtype=BF, device=DEV)
        q, k, v = qk[:L, :W], qk[:L, W:], vb[:L]
    else:
        buf = torch.full((L + 128, ld), float("nan"), dtype=BF, device=DEV)
        q, k, v = buf[:L, :W], buf[:L, W:2 * W], buf[:L, 2 * W:3 * W]
    for t in (q, k, v):
        _fill(t, g)
    need = ctypes.c_int64(0)
    L_.check(L_.lib.mc_attn_workspace_bytes(L, L, heads, ctypes.byref(need)))
    units = -(-L // 128) * heads
    print(f"[attention {name}] Lq = Lk = {L}, {heads} heads, ldq {q.stride(0)}, ldv {v.stride(0)}: {units} units, "
          f"workspace {need.value} bytes")
    ws, wbuf = fenced((max(need.value, 32),), torch.uint8, (0, 0, 32, 32), fill="fence")
    out, obuf = fenced((L, W), BF, (1, 1, 8, 8), fill="fence")
    worst = 0.0
    for qscale, sl in ((1.0, slices), (6.5, [scaled_slice])):
        if qscale != 1.0:
            q.mul_(qscale)
        L_.check(L_.lib.mc_attn_fwd_ex(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), out.data_ptr(),
                                       out.stride(0), L, L, heads, 1.0 / math.sqrt(128), ws.data_ptr(), need.value, 0, None, None, 0,
                                       ops._stream()))
        check_fence(out, obuf)
        check_fence(ws, wbuf)
        rows = torch.cat([torch.arange(a, b) for a, b in sl]).to(DEV)
        ref = _attn_ref64(q[rows], k, v, heads).float()
        got = out[rows].float()
        sd = F.scaled_dot_product_attention(*(t.view(t.shape[0], heads, 128).transpose(0, 1)[None] for t in (q[rows], k, v)))
        sd = sd[0].transpose(0, 1).reshape(rows.numel(), W).float()
        err, err_sd = (got - ref).abs(), (sd - ref).abs()
        e_ours, e_sdpa = rel_l2(got, ref), rel_l2(sd, ref)
        print(f"  q x{qscale} rows {sl}: rel-L2 vs fp64 ours {e_ours:.3e}, SDPA {e_sdpa:.3e}; max abs ours {float(err.max()):.3e}, "
              f"SDPA {float(err_sd.max()):.3e}")
        assert bool(torch.isfinite(got).all())
        assert e_ours <= 2.0 * e_sdpa + 1e-4, (name, qscale, e_ours, e_sdpa)
        assert float(err.max()) <= 2.0 * float(err_sd.max()) + 1e-3, (name, qscale, float(err.max()), float(err_sd.max()))
        assert e_ours < 8e-3 and float(err.mean()) < 2e-3, (name, qscale, e_ours, float(err.mean()))
        worst = max(worst, e_ours / (2.0 * e_sdpa + 1e-4), float(err.max()) / (2.0 * float(err_sd.max()) + 1e-3))
    print(f"  worst bound ratio {worst:.2f}")


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["engine", "linear1"])
def test_attention_hunyuan_119056_keys(layout):
    """HunyuanVideo's joint attention: 118 800 image + 256 text rows in the engine's [image | text] key order, 24 heads; q | k | v
    in the engine's own buffers (ldq 6144, ldv 3072), and as column slices of a [119 056, 21 504] buffer (the reference's linear1
    layout: row offsets past 2^31 elements). Slices: the first query tile, a middle tile, the last image rows, and the text rows
    (which hold the ragged last tile)."""
    _need_device_memory(40)
    t0 = time.time()
    n_img = HUNYUAN["n_img"]
    _attention_case(f"hunyuan {layout}", HY_ROWS, 24, None if layout == "engine" else HUNYUAN["linear1"],
                    [(0, 128), (59392, 59520), (n_img - 128, n_img), (n_img, HY_ROWS)], (59392, 59520),
                    torch.Generator(device=DEV).manual_seed(61))
    _report(f"attention hunyuan {layout}", t0)


@pytest.mark.gpu
def test_attention_wan14b_75600_keys():
    """Wan-14B's self-attention: 75 600 keys, 40 heads, q | k | v column slices of the [75 600, 15 360] qkv buffer (ldq = 15 360)."""
    _need_device_memory(40)
    t0 = time.time()
    n = WAN14B["n_tok"]
    _attention_case("wan14b", n, 40, WAN14B["qkv"], [(0, 128), (37760, 37888), (n - 80, n)], (n - 80, n),
                    torch.Generator(device=DEV).manual_seed(62))
    _report("attention wan14b", t0)


@pytest.mark.gpu
def test_attention_flux_4608_keys():
    """FLUX's joint attention: 512 text rows then 4096 image rows, 24 heads, in the MMDiT engine's q | k and v buffers."""
    _attention_case("flux", 4608, 24, None, [(0, 512), (2304, 2432), (4480, 4608)], (0, 512),
                    torch.Generator(device=DEV).manual_seed(63))


def _untouched(buf, c0, rows=8192):
    """Do columns c0: of every row of `buf` still hold the fence pattern?"""
    for r0 in range(0, buf.shape[0], rows):
        if not bool(_fill_bytes_ok(buf[r0:r0 + rows, c0:]).all()):
            return False
    return True


@pytest.mark.gpu
def test_hunyuan_qk_norm_rope_past_2_31_elements():
    """`mc_rmsnorm_head_rope` in place on the q and k column slices of a [119 056, 21 504] bf16 buffer (2.56e9 elements): the
    reference's linear1 layout, whose row offsets pass 2^31 elements (the engine keeps q | k in its own [S, 6144] buffer, which
    stays below). Image rows with the (33, 45, 80) RoPE table of `rope_cos_sin`, text rows without, as the engine splits them.
    The first 256 rows, the last 1024 image rows (offsets past 2^31) and the text rows against `_rms_rope_ref`; the v and MLP
    columns must keep their bytes."""
    from magcache_b200 import ops
    from oracle import hunyuan_ref as hr
    _need_device_memory(40)
    t0 = time.time()
    D, H, n_img, L = HUNYUAN["hidden"], HUNYUAN["heads"], HUNYUAN["n_img"], HY_ROWS
    g = torch.Generator(device=DEV).manual_seed(71)
    buf = torch.empty(L, HUNYUAN["linear1"], dtype=BF, device=DEV)
    buf.view(torch.uint8).fill_(FENCE_BYTE)
    _fill(buf[:, :2 * D], g, 2.0)
    assert (n_img - 1024) * buf.stride(0) > 2 ** 31
    checks = [(0, 256, True), (n_img - 1024, n_img, True), (n_img, L, False)]
    x0 = {c: buf[c[0]:c[1], :2 * D].clone() for c in checks}
    cos, sin = hr.rope_cos_sin(HUNYUAN["grid"])
    cs = torch.stack([cos[:, 0::2], sin[:, 0::2]], dim=-1).reshape(n_img, 128).contiguous().to(DEV)  # HunyuanEngine.stage_inputs
    nq, nk = ((1 + 0.2 * torch.randn(128, device=DEV, generator=g)).bfloat16().float() for _ in range(2))
    for c0, w in ((0, nq), (D, nk)):
        ops.rmsnorm_head_rope_(buf[:n_img, c0:c0 + D], w, H, cs)
        ops.rmsnorm_head_rope_(buf[n_img:, c0:c0 + D], w, H, None)
    for (r0, r1, rope) in checks:
        pos = torch.arange(r0, r1, device=DEV) if rope else None
        for c0, w in ((0, nq), (D, nk)):
            _assert_ulps(buf[r0:r1, c0:c0 + D], _rms_rope_ref(x0[(r0, r1, rope)][:, c0:c0 + D], w, H, 128, cs if rope else None, pos), rope,
                         ("hunyuan q|k", r0, r1, c0))
    assert _untouched(buf, 2 * D), "v / MLP columns changed"
    _report("hunyuan q|k RMSNorm + RoPE", t0)


def _segs_ref(x0, w, cs, cols):
    o = _rb(x0.double() * torch.rsqrt(x0.double().pow(2).mean(-1, keepdim=True) + 1e-6)) * w.double()
    return _rb(_rope64(o, cs, cols))


@pytest.mark.gpu
def test_wan14b_qk_norm_rope_segs():
    """`mc_rmsnorm_rope_segs` (segs 2, 5120 columns) in place on q | k of the [75 600, 15 360] qkv buffer with the (21, 45, 80)
    table of `wan.rope_table`: the first 1024 and the last 1024 rows against fp64 at test_rmsnorm_rope_segs_fenced's criterion;
    the v columns must keep their bytes."""
    from magcache_b200 import ops
    from magcache_b200.wan import rope_table
    _need_device_memory(20)
    D, n = WAN14B["dim"], WAN14B["n_tok"]
    g = torch.Generator(device=DEV).manual_seed(72)
    buf = torch.empty(n, WAN14B["qkv"], dtype=BF, device=DEV)
    buf.view(torch.uint8).fill_(FENCE_BYTE)
    _fill(buf[:, :2 * D], g, 2.0)
    rows = torch.cat([torch.arange(0, 1024), torch.arange(n - 1024, n)]).to(DEV)
    x0 = buf[rows, :2 * D].clone()
    cs = rope_table(WAN14B["grid"], 128, DEV)
    w = (1 + 0.2 * torch.randn(2, D, device=DEV, generator=g)).contiguous()
    ops.rmsnorm_rope_segs_(buf, w, 2, cs, 128)
    for sg in range(2):
        sl = slice(sg * D, (sg + 1) * D)
        _assert_ulps(buf[rows, sl], _segs_ref(x0[:, sl], w[sg], cs[rows], D), True, ("wan14b q|k", sg))
    assert _untouched(buf, 2 * D), "v columns changed"


# the GEMMs only these models launch: (epilogue, M, N, K)
_GEMMS = [
    ("hunyuan linear1 mlp", "MC_EPI_BIAS_GELU_BF16", HY_ROWS, 12288, 3072),
    ("hunyuan linear1 q|k", "MC_EPI_BIAS_BF16", HY_ROWS, 6144, 3072),
    ("hunyuan linear1 v", "MC_EPI_BIAS_BF16", HY_ROWS, 3072, 3072),
    ("hunyuan linear2", "MC_EPI_BIAS_GATE_RESID_BF16", HY_ROWS, 3072, 15360),
    ("wan14b qkv", "MC_EPI_BIAS_BF16", 75600, 15360, 5120),
    ("wan14b ffn1", "MC_EPI_BIAS_GELU_BF16", 75600, 13824, 5120),
    ("wan14b ffn2", "MC_EPI_BIAS_GATE_RESID", 75600, 5120, 13824),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,epi,M,N,K", _GEMMS, ids=[c[0].replace(" ", "_") for c in _GEMMS])
def test_gemm_workload_shapes(name, epi, M, N, K):
    """`mc_gemm_bf16` at the engine's shape and epilogue: A / B with NaN columns either side of K, bias / gate fenced with NaN,
    the output a window of a fenced buffer (the residual epilogues update a random stream in place); the first, a middle and the
    ragged last 128-row tile against fp64 within `gemm_fp64_bounds_ok`."""
    from magcache_b200 import _lib as L_
    from magcache_b200 import ops
    _need_device_memory(40)
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    a, _ = fenced((M, K), BF, (0, 1, 8, 8))
    _fill(a, g)
    b, _ = fenced((N, K), BF, (0, 1, 8, 8))
    _fill(b, g, 1.0 / math.sqrt(K))
    bias, _ = fenced((N,), F32, (0, 0, 4, 4))
    bias.copy_(torch.randn(N, device=DEV, generator=g).bfloat16().float())
    gate = None
    if "GATE" in epi:
        gate, _ = fenced((N,), F32, (0, 0, 4, 4))
        gate.copy_(torch.randn(N, device=DEV, generator=g) * 0.5)
    odt = F32 if epi == "MC_EPI_BIAS_GATE_RESID" else BF
    out, obuf = fenced((M, N), odt, (2, 2, 8, 8), fill="fence")
    rows = _tiles(M)
    old = None
    if gate is not None:
        _fill(out, g)
        old = out[rows].double()
    ops.gemm(a, b, bias, getattr(L_, epi), out=out, gate=gate)
    check_fence(out, obuf)
    got = out[rows].double()
    assert bool(torch.isfinite(got).all()), name
    pre = a[rows].double() @ b.double().t() + bias.double()
    ok = gemm_fp64_bounds_ok(epi, got, pre, old, None if gate is None else gate.double())
    print(f"[gemm {name}] {M} x {N} x {K}: {int((~ok).sum())} of {ok.numel()} checked outputs outside the bound")
    assert bool(ok.all()), (name, int((~ok).sum()))


def _sample_rows(rows, head=1024, tail=4096, stride=97):
    """The first `head` rows, the last `tail` rows (the last CTAs' rows) and every `stride`-th row in between."""
    return torch.cat([torch.arange(0, head), torch.arange(0, rows, stride), torch.arange(rows - tail, rows)]).unique().to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols", [(HY_ROWS, 3072), (WAN14B["n_tok"], 5120)])
def test_ln_modulate_workload_rows(rows, cols):
    """K7 (`mc_ln_modulate` modes 0 and 1) at HunyuanVideo's 119 056 x 3072 and Wan-14B's 75 600 x 5120: x bf16 and fp32 with NaN
    rows after it, round_ln on and off, out bf16 a row window of a fenced buffer; sampled rows (always the last 4096) against
    `_ln_chain`'s per-element bound."""
    from magcache_b200 import _lib as L_
    from magcache_b200 import ops
    _need_device_memory(20)
    g = torch.Generator(device=DEV).manual_seed(rows + cols)
    sel = _sample_rows(rows)
    worst = 0.0
    for xdt in (BF, F32):
        x, _ = fenced((rows, cols), xdt, (0, 8, 0, 0), pitch=cols)
        _fill(x, g, 3.0, 0.5)
        p, _ = fenced((6 * cols,), F32, (0, 0, 8, 8))
        p.copy_(torch.randn(6 * cols, device=DEV, generator=g) * 0.3)
        em = p.view(6, cols)
        for mode in (0, 1):
            a, b = (em[4], em[3]) if mode == 0 else (em[0], em[5])
            p0, p1 = (em, None) if mode == 0 else (em[0], em[5])
            for round_ln in (1, 0):
                out, obuf = fenced((rows, cols), BF, (2, 2, 0, 0), fill="fence", pitch=cols)
                L_.check(L_.lib.mc_ln_modulate(x.data_ptr(), L_.MC_BF16 if xdt == BF else L_.MC_F32, rows, cols, 1e-6, mode, p0.data_ptr(),
                                               None if p1 is None else p1.data_ptr(), 4, 3, round_ln, out.data_ptr(), L_.MC_BF16,
                                               ops._stream()))
                check_fence(out, obuf)
                ref, bound = _ln_chain(x[sel], a, b, mode, round_ln, True)
                got = out[sel].double()
                assert bool(torch.isfinite(got).all())
                r = float(((got - ref).abs() / bound).max())
                worst = max(worst, r)
                assert r <= 1.0, ((rows, cols, xdt, mode, round_ln), r)
                del out, obuf
    print(f"[K7 {rows} x {cols}] worst error / bound {worst:.2f}")


def _unpatchify(y, grid):
    Fr, Hp, Wp = grid
    return torch.einsum("fhwpqrc->cfphqwr", y.view(Fr, Hp, Wp, 1, 2, 2, 16)).reshape(16, Fr, Hp * 2, Wp * 2)


def _head_case(kind, w_scale, seed):
    """One head launch per form (fp32 stream, fused cache hit) at D = 5120 on the (21, 45, 80) grid, W = w_scale * randn.
    Returns per form (got, fp64 reference, `head_chain` bound), unpatchified."""
    from magcache_b200 import ops
    D, grid = WAN14B["dim"], WAN14B["grid"]
    rows = math.prod(grid)
    g = torch.Generator(device=DEV).manual_seed(seed)
    head_mod = torch.randn(1, 2, D, device=DEV, generator=g) / math.sqrt(D)
    e = torch.randn(1, D, device=DEV, generator=g) * 0.3
    W = torch.randn(64, D, device=DEV, generator=g) * w_scale
    b = torch.randn(64, device=DEV, generator=g) * 0.1
    x = torch.randn(rows, D, device=DEV, generator=g) * 2
    if kind == "offset":
        x = x + torch.randn(rows, 1, device=DEV, generator=g) * 50.0
    s, t = 1.0 + (head_mod[0, 1] + e[0]), head_mod[0, 0] + e[0]  # fp32, as the kernel forms them
    Wt = W.t().contiguous()
    x0, r = x.bfloat16(), torch.randn(rows, D, device=DEV, generator=g) * 0.3
    res = {}
    for form, out, v in (("stream", ops.head_unpatchify(x, head_mod, e, Wt, b, grid), x),
                         ("hit", ops.head_unpatchify(x0, head_mod, e, Wt, b, grid, residual=r), x0.float() + r)):
        ref, bound = (_unpatchify(z, grid) for z in head_chain(v, s, t, Wt, b))
        assert bool(torch.isfinite(out).all()), (kind, form)
        res[form] = (out.double(), ref, bound)
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["plain", "offset"])
def test_head_wan14b_grid(kind):
    """The head kernel at D = 5120 on Wan-14B's (21, 45, 80) grid (75 600 rows), the fp32-stream form and the fused cache-hit form.

    With W = randn / sqrt(5120) the outputs have unit scale, like the velocity the Wan head predicts: every output within
    test_head_unpatchify_shapes_and_offsets' criterion (rtol 1e-3, atol 1e-4) and within the per-element bound of the kernel's
    rounding chain (`head_chain` of test_head_readout_gpu.py, through the 64-wide Linear).

    The head's absolute error grows with the scale of its outputs: each product of the 3-pass bf16 split is good to about
    2^-16 of itself, so the error is a fraction of sum_k |y_k W_k|. With test_head_unpatchify_shapes_and_offsets' W = 0.05 randn
    the outputs' rms is 0.05 sqrt(5120) ~ 3.6 and a fixed atol of 1e-4 is no longer met on outputs near zero (about 1.5x). So
    at that scale every output is held to the chain bound, and the largest error relative to the outputs' rms must be no
    worse than at unit scale (x 1.25): the error scales with the outputs, it does not grow on its own."""
    _need_device_memory(20)
    seed = 81 + (kind == "offset")
    unit = _head_case(kind, 1.0 / math.sqrt(WAN14B["dim"]), seed)
    wide = _head_case(kind, 0.05, seed)
    rel = {}
    for scale, res in (("unit", unit), ("0.05", wide)):
        for form, (got, ref, bound) in res.items():
            err = (got - ref).abs()
            chain = float(torch.where(err == 0, 0.0, err / bound).max())
            north = float((err / NORTH_STAR(ref)).max())
            rel[scale, form] = float(err.max()) / float(ref.pow(2).mean().sqrt())
            print(f"[head D=5120 {kind} W {scale} {form}] output rms {float(ref.pow(2).mean().sqrt()):.2f}, max error "
                  f"{float(err.max()):.2e}, / chain bound {chain:.2f}, / (1e-3 |ref| + 1e-4) {north:.2f}")
            assert chain <= 1.0, (kind, scale, form, chain)
            if scale == "unit":
                assert torch.allclose(got, ref, rtol=1e-3, atol=1e-4), (kind, form, north)
    for form in ("stream", "hit"):
        assert rel["0.05", form] <= 1.25 * rel["unit", form], (kind, form, rel)


@pytest.mark.gpu
def test_residual_stats_wan14b_rows():
    """K3 (`mc_residual_stats`, `mc_residual_sub_stats`) at 75 600 x 5120 fp32, the calibration statistics of Wan-14B: inputs
    with NaN rows after them, the fused residual a fenced row window bit-equal to x_out - x_in, the three sums against fp64 within
    `_stats_chain`'s bound."""
    from magcache_b200 import _lib as L_
    from magcache_b200 import ops
    _need_device_memory(20)
    rows, cols = WAN14B["n_tok"], WAN14B["dim"]
    g = torch.Generator(device=DEV).manual_seed(91)
    prev, _ = fenced((rows, cols), F32, (0, 8, 0, 0), pitch=cols)
    _fill(prev, g, 0.1)
    cur, _ = fenced((rows, cols), F32, (0, 8, 0, 0), pitch=cols)
    cur.copy_(prev * (0.97 + 0.05 * torch.rand(rows, 1, device=DEV, generator=g)) + torch.randn(rows, cols, device=DEV, generator=g) * 0.01)
    stats = torch.empty(4, dtype=torch.float64, device=DEV)
    L_.check(L_.lib.mc_residual_stats(cur.data_ptr(), L_.MC_F32, prev.data_ptr(), L_.MC_F32, rows, cols, 0.0, stats.data_ptr(), ops._stream()))
    ref, bound = _stats_chain(cur, prev)
    assert float(stats[3]) == rows
    r1 = float(((stats[:3] - ref).abs() / bound).max())
    assert r1 <= 1.0, (stats.tolist(), ref.tolist(), bound.tolist())
    x_in, _ = fenced((rows, cols), BF, (0, 8, 0, 0), pitch=cols)
    _fill(x_in, g)
    x_out, _ = fenced((rows, cols), F32, (0, 8, 0, 0), pitch=cols)
    x_out.copy_(x_in.float() + cur)
    r, rbuf = fenced((rows, cols), F32, (1, 1, 0, 0), fill="fence", pitch=cols)
    L_.check(L_.lib.mc_residual_sub_stats(x_out.data_ptr(), L_.MC_F32, x_in.data_ptr(), L_.MC_BF16, r.data_ptr(), prev.data_ptr(), rows, cols,
                                          0.0, stats.data_ptr(), ops._stream()))
    check_fence(r, rbuf)
    assert torch.equal(r, x_out - x_in.float())
    ref, bound = _stats_chain(r, prev)
    r2 = float(((stats[:3] - ref).abs() / bound).max())
    assert r2 <= 1.0, ("fused", stats.tolist(), ref.tolist(), bound.tolist())
    print(f"[K3 {rows} x {cols}] worst error / bound {max(r1, r2):.2f}")
