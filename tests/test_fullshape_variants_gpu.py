"""Parity at the full shapes of the Wan variants whose code paths are not the t2v one: Wan2.2 TI2V-5B 1280x704x121 (dim 3072,
24 heads, ffn 14 336, 48 latent channels in and out; latent 48 x 31 x 44 x 80 -> 31 x 22 x 40 = 27 280 tokens; `t` per token
with t = 0 on the first frame's 880 tokens), Wan2.1 I2V-14B 1280x720x81 (dim 5120, 40 heads, in_dim 36 = 16 noise + 20 mask
and first-frame channels; 75 600 tokens; 257 CLIP tokens of width 1280) and VACE-1.3B 832x480x81 (dim 1536, 12 heads; 32 760
tokens; a 96-channel control video).

(a) One-layer, full-width models (VACE: one main block and its VACE block) through the patched forwards (`magcache_wan22_forward`,
    `magcache_forward` with `clip_fea` / `y`, `magcache_vace_forward`): miss, miss, hit, hit over both CFG slots against the
    bf16 oracle and the fp64 oracle, both on the GPU, at DESIGN §5's rule for the output and the residual cache, controller
    attributes bit-equal (`_forward_loop` of test_fullshape_workloads_gpu.py). A whole-output rel-L2 moves by about
    1 / sqrt(27 280) = 6e-3 when one row of 27 280 takes the wrong range, which is e_ref's size, so for TI2V the rule is also
    applied to each of the six output blocks (timestep range u x 16-channel group g: what one head launch writes), to each
    range's rows of the residual cache, and to the 256 rows around the range boundary at row 880.
(b) Each kernel at the launch shapes only these variants issue, per element against fp64, outputs fenced:
    1. the TI2V head: six launches (2 ranges x 3 channel groups, row_offset 0 / 880, head-prep slots u * 3 + g) into one NaN-
       filled output; after each launch exactly its block has changed, at the end no NaN is left, every element meets
       `head_chain` and, at unit-scale W, the north star; the fp32-stream and the cache-hit forms;
    2. the gated-residual GEMM (o: K 3072, ffn2: K 14 336) and K7 (LayerNorm + modulation) on the row slices [0, 880) and
       [880, 27 280) with each range's gate / modulation rows, the other slice's rows bit-unchanged;
    3. an engine forward at TI2V width with 8 timestep values in 64 ranges (values recurring in non-adjacent ranges, boundaries
       off the 128-row tile), each range held to the rule: the time MLP at M = 8, head-prep slots up to 23;
    4. the time path: `time_sinusoid` and `linear_f32_small` at every M in 1..8;
    5. I2V's image branch: attention of 75 600 query rows x 40 heads over the 257 CLIP keys (four full 64-key tiles and a 1-key
       one) and over the 512 text keys, in the engine's buffers; `img_emb` (LayerNorm, Linear + GELU(erf), Linear, LayerNorm);
    6. `patchify` at C = 36, 48 and 96 on the full latents, bit-equal to the view / permute statement.

Controls. Each check of (b) is shown to fail when its reference carries one wrong input, in the same test: the range boundary
moved by one row (row 880 with range 0's modulation, i.e. t = 0 on 881 tokens), head groups 1 and 2 swapped, the other range's
gate / modulation on the boundary row, the 257th CLIP key dropped, and M = 8 computed as M = 7 (the eighth timestep value's
rows given the seventh's value).

The bound of `linear_f32_small` (4). The kernel gives each output y[m, n] to one warp: each lane runs a chain of K / 32 fmaf over
its float4 slices of the row, then five shuffle adds combine the lanes, then the bias is added in fp32. Every product passes
through at most L = K / 32 + 5 roundings before the bias, so with u = 2^-24 and gamma_L = L u / (1 - L u) the pre-activation
is within gamma_L sum_k |x_k w_k| + u |y| of the fp64 value (Higham, Thm 3.1; the last term is the bias add). act = 1 applies
SiLU to each input first: `x / (1 + expf(-x))` with expf within 2 ulp, the add and the divide within 1/2 ulp each, so each
SiLU value is within 4 u of itself relative and adds 4 u sum_k |silu(x_k) w_k| (taken 5 u). act = 2 applies SiLU to the
output: |SiLU'| <= 1.1 carries the pre-activation error through, plus 5 u |SiLU(y)| for the SiLU itself.

The oracle needs no replacement beyond `_oracle_on_gpu` (I2V's image cross-attention calls `attention_ref` without `k_lens`,
which `wan_attention` covers; TI2V's per-token time embedding, [27 280, 6, 3072] in fp64, fits on the card as written).

`test_variant_shape_table_matches_the_engines`, `test_timestep_range_limits` and `test_token_layout_inverts_unpatchify` run
without a GPU."""
import copy
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
from test_fullshape_workloads_gpu import (_attn_ref64, _fill, _forward_loop, _need_device_memory, _oracle_on_gpu, _report,  # noqa: E402
                                          _rule, rel_l2)
from test_head_readout_gpu import NORTH_STAR, head_chain  # noqa: E402
from test_kernel_bounds_gpu import BF, F32, _ln_chain, check_fence, fenced, gemm_fp64_bounds_ok  # noqa: E402

DEV = "cuda"
U32 = 2.0 ** -24

# ------------------------------------------------------------------------------------------- the shapes
# Wan2.2 TI2V-5B 1280 x 704 x 121 (tools/bench_ti2v.py): the first latent frame (22 x 40 = 880 tokens) is the conditioning
# image, its tokens at t = 0
TI2V = dict(cfg="ti2v-5B", dim=3072, heads=24, ffn=14336, channels=48, latent=(48, 31, 44, 80), grid=(31, 22, 40), n_tok=27280,
            first=880, table="wan2.2_ti2v_5b_a")
TI2V_RUNS = [(0, 880, 0), (880, 27280, 1)]
# Wan2.1 I2V-14B 1280 x 720 x 81: noise latents 16 x 21 x 90 x 160 and `y` (mask + first-frame latents) 20 x 21 x 90 x 160
I2V = dict(cfg="i2v-14B", dim=5120, heads=40, ffn=13824, latent=(16, 21, 90, 160), y=(20, 21, 90, 160), grid=(21, 45, 80),
           n_tok=75600, clip_len=257, clip_dim=1280, text_len=512, table="wan2.1_i2v_720p")
# VACE-1.3B 832 x 480 x 81: latents 16 x 21 x 60 x 104, control video 96 x 21 x 60 x 104
VACE = dict(cfg="vace-1.3B", dim=1536, heads=12, ffn=8960, latent=(16, 21, 60, 104), control=(96, 21, 60, 104), grid=(21, 30, 52),
            n_tok=32760, table="wan2.1_vace_1.3b")
# more timestep values and ranges than TI2V uses: the engine's limits, at TI2V width on a reduced grid
MANY = dict(latent=(48, 4, 32, 48), grid=(4, 16, 24), n_tok=1536, values=(0.0, 999.0, 731.0, 500.0, 250.0, 900.0, 40.0, 640.0))


def _tokens(out, grid):
    """A head / unpatchify output [C, F, 2 Hp, 2 Wp] as [tokens, 4, C]: token (f, h, w), patch position 2 q + r, channel c."""
    C = out.shape[0]
    f, hp, wp = grid
    return out.reshape(C, f, hp, 2, wp, 2).permute(1, 2, 4, 3, 5, 0).reshape(f * hp * wp, 4, C)


def _untokens(tok, grid):
    f, hp, wp = grid
    C = tok.shape[-1]
    return tok.reshape(f, hp, wp, 2, 2, C).permute(5, 0, 1, 3, 2, 4).reshape(C, f, 2 * hp, 2 * wp)


def _many_ranges(n_tok, n_values, n_runs, seed=0):
    """A per-token t [1, n_tok] with `n_values` distinct values in `n_runs` contiguous ranges: range j carries value j % n_values
    (so neighbours differ and every value recurs in non-adjacent ranges), lengths 24 +- 8 with no boundary on a multiple of 128.
    Returns (t, [(r0, r1, value index)])."""
    rng = np.random.default_rng(seed)
    values = list(MANY["values"]) + [123.0 + 7.0 * i for i in range(max(0, n_values - len(MANY["values"])))]
    cuts = [0]
    base = n_tok // n_runs
    for j in range(1, n_runs):
        c = j * base + int(rng.integers(-8, 9))
        if c % 128 == 0:
            c += 1
        cuts.append(c)
    cuts.append(n_tok)
    assert all(b - a >= 4 for a, b in zip(cuts[:-1], cuts[1:]))
    t = torch.empty(1, n_tok)
    runs = []
    for j in range(n_runs):
        t[0, cuts[j]:cuts[j + 1]] = values[j % n_values]
        runs.append((cuts[j], cuts[j + 1], j % n_values))
    return t, runs


def _meta_engine(cfg):
    from magcache_b200.wan import WAN_CONFIGS, WanEngine
    meta = torch.device("meta")
    d = WAN_CONFIGS[cfg]
    return WanEngine(types.SimpleNamespace(dims=d, device=meta, head_wt=torch.empty(d.dim, 4 * d.out_dim, device=meta),
                                           head_b=torch.empty(4 * d.out_dim, device=meta)))


# ------------------------------------------------------------------------------------------- CPU: the shapes and the host logic
def test_variant_shape_table_matches_the_engines():
    """The shapes the GPU tests use are the ones the engines derive: token counts (the oracle's patch embedding on the latent
    shape), TI2V's row ranges and head groups from `_stage_t` on its per-token t, I2V's CLIP buffers, the VACE hint layers of
    `WAN_CONFIGS` against the model's and `WanWeights.from_module`'s, and the MagCache tables the tests install. Models and
    engine buffers live on the meta device: shapes only."""
    import magcache_b200 as mc
    from magcache_b200.wan import WAN_CONFIGS, WanWeights
    from oracle import wan_ref
    meta = torch.device("meta")
    for v in (TI2V, I2V, VACE):
        d = WAN_CONFIGS[v["cfg"]]
        assert (d.dim, d.num_heads, d.ffn_dim) == (v["dim"], v["heads"], v["ffn"]) and d.head_dim == 128, v["cfg"]
        assert v["table"] in mc.tables(), v["table"]

    # TI2V-5B
    d = WAN_CONFIGS[TI2V["cfg"]]
    assert d.in_dim == d.out_dim == TI2V["channels"]
    with meta:
        m = wan_ref.WanModel(dim=d.dim, ffn_dim=d.ffn_dim, num_heads=d.num_heads, num_layers=1, in_dim=48, out_dim=48)
        grid = tuple(m.patch_embedding(torch.empty(1, *TI2V["latent"])).shape[2:])
    assert grid == TI2V["grid"] and math.prod(grid) == TI2V["n_tok"] and grid[1] * grid[2] == TI2V["first"]
    assert TI2V["first"] % 128 != 0
    eng = _meta_engine(TI2V["cfg"])
    eng._workspace(TI2V["n_tok"])
    t = torch.full((1, TI2V["n_tok"]), 731.0)
    t[0, :TI2V["first"]] = 0.0
    eng._stage_t(t)
    assert eng.t_values == 2 and eng.runs == TI2V_RUNS and len(eng.head_groups) == 3
    assert all(wt.shape == (d.dim, 64) and hb.shape == (64,) for wt, hb in eng.head_groups)

    # I2V-14B
    d = WAN_CONFIGS[I2V["cfg"]]
    assert d.model_type == "i2v" and d.in_dim == I2V["latent"][0] + I2V["y"][0] and (d.clip_len, d.clip_dim) == (I2V["clip_len"], I2V["clip_dim"])
    with meta:
        m = wan_ref.WanModel(dim=d.dim, ffn_dim=d.ffn_dim, num_heads=d.num_heads, num_layers=1, in_dim=36, model_type="i2v",
                             clip_dim=I2V["clip_dim"])
        grid = tuple(m.patch_embedding(torch.empty(1, *((36,) + I2V["latent"][1:]))).shape[2:])
    assert grid == I2V["grid"] and math.prod(grid) == I2V["n_tok"]
    w = WanWeights.from_module(m, meta)
    assert w.dims.model_type == "i2v" and (w.dims.clip_len, w.dims.clip_dim) == (I2V["clip_len"], I2V["clip_dim"])
    eng = _meta_engine(I2V["cfg"])
    eng._workspace(I2V["n_tok"])
    assert eng.clip_in.shape == (I2V["clip_len"], I2V["clip_dim"]) and eng.ckv_img.shape == (I2V["clip_len"], 2 * d.dim)
    assert eng.ckv.shape == (I2V["text_len"], 2 * d.dim) and eng.cq.shape == eng.att_img.shape == (I2V["n_tok"], d.dim)

    # VACE-1.3B
    d = WAN_CONFIGS[VACE["cfg"]]
    assert d.model_type == "vace" and d.vace_in_dim == VACE["control"][0]
    with meta:
        m = wan_ref.WanModel(dim=d.dim, ffn_dim=d.ffn_dim, num_heads=d.num_heads, num_layers=d.num_layers, model_type="vace")
        grid = tuple(m.patch_embedding(torch.empty(1, *VACE["latent"])).shape[2:])
        cgrid = tuple(m.vace_patch_embedding(torch.empty(1, *VACE["control"])).shape[2:])
    assert grid == cgrid == VACE["grid"] and math.prod(grid) == VACE["n_tok"]
    assert tuple(m.vace_layers) == d.vace_layers == tuple(range(0, 30, 2))
    w = WanWeights.from_module(m, meta)
    assert w.dims.vace_layers == d.vace_layers and len(w.vace_blocks) == len(d.vace_layers) and w.dims.vace_in_dim == 96
    with meta:  # the one-layer model of the GPU test: one main block, its hint from the one VACE block
        m1 = wan_ref.WanModel(dim=d.dim, ffn_dim=d.ffn_dim, num_heads=d.num_heads, num_layers=1, model_type="vace")
    assert m1.vace_layers == [0] and len(m1.vace_blocks) == 1


def test_timestep_range_limits():
    """`WanEngine._stage_t` at its limits: the t of (b)3 — 8 values in 64 ranges, boundaries off the 128-row tile — reduces to
    exactly those ranges (value indices in order of first appearance); one more value or one more range is refused."""
    from magcache_b200.wan import MAX_T_RUNS, MAX_T_VALUES
    assert (MAX_T_VALUES, MAX_T_RUNS) == (8, 64)
    n = MANY["n_tok"]
    t, runs = _many_ranges(n, 8, 64)
    assert all(r0 % 128 for r0, _, _ in runs[1:])
    eng = _meta_engine(TI2V["cfg"])
    eng._workspace(n)
    eng._stage_t(t)
    assert eng.t_values == 8 and eng.runs == runs
    for nv, nr in ((9, 64), (8, 65)):
        tt, _ = _many_ranges(n, nv, nr)
        with pytest.raises(NotImplementedError):
            eng._stage_t(tt)


def test_token_layout_inverts_unpatchify():
    """`_tokens` (the per-block view the TI2V checks use) inverts the oracle's `unpatchify`: feature (2 q + r) * C + c of token
    (f, h, w) lands at [token, 2 q + r, c]; `_untokens` is its inverse."""
    from oracle import wan_ref
    grid, C = (3, 4, 5), 48
    n = math.prod(grid)
    u = torch.randn(n, 4 * C, dtype=torch.float64)
    m = types.SimpleNamespace(out_dim=C, patch_size=(1, 2, 2))
    out = wan_ref.WanModel.unpatchify(m, [u], torch.tensor([grid]))[0]
    assert torch.equal(_tokens(out, grid), u.view(n, 4, C))
    assert torch.equal(_untokens(_tokens(out, grid), grid), out)


# ------------------------------------------------------------------------------------------- (a) one-layer forwards
class _Call:
    """One model called the way the pipeline calls it: [latent], t, [context], seq_len, plus the variant's extra inputs, all
    in `dt` (the fp64 oracle takes fp64 inputs); attributes read through."""

    def __init__(self, m, dt, lat, n, **extra):
        self.m, self.dt, self.lat, self.n, self.extra = m, dt, lat, n, extra

    def __call__(self, c, t):
        cast = (lambda v: v.to(self.dt)) if self.dt == torch.float64 else (lambda v: v)  # noqa: E731
        kw = {k: ([cast(v[0])] if isinstance(v, list) else cast(v)) for k, v in self.extra.items()}
        return self.m([cast(self.lat)], t=cast(t), context=[cast(c)], seq_len=self.n, **kw)[0]

    def __getattr__(self, name):
        return getattr(self.m, name)


def _res(m):  # the residual cache of the slot the call just wrote (cnt has advanced by one)
    return m.residual_cache[(int(m.cnt) - 1) % 2][0]


def _three(model, name, install):
    """Our model (patched by `install(model, None)`), the bf16 oracle and the fp64 oracle, each on the GPU in its own class."""
    ours = copy.deepcopy(model).to(DEV)
    ours.__class__ = type("Ours" + name, (ours.__class__,), {})
    install(ours, None)
    ref_m = copy.deepcopy(model).to(DEV)
    ref_m.__class__ = type("Ref" + name, (ref_m.__class__,), {})
    install(ref_m, "oracle")
    m64 = copy.deepcopy(model).to(DEV).double()
    m64.__class__ = type("Ref64" + name, (m64.__class__,), {})
    install(m64, "oracle")
    return ours, ref_m, m64


_ATTRS = ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps")


def _per_range_check(tag, runs, grid, groups, band=None, verbose=True):
    """The `check` of `_forward_loop`: the rule on each (range, 16-channel group) block of the output, on each range's rows of
    the residual cache, and on the rows [band[0], band[1]) of both. Keeps the worst fraction of the bound in `worst`."""
    worst = {}

    def check(i, out, ref, ex, r_ours, r_ref, r_ex):
        o, r, x = (_tokens(v, grid) for v in (out, ref, ex))
        for r0, r1, u in runs:
            for g in range(groups):
                c = slice(16 * g, 16 * g + 16)
                k = ("output", u if verbose else "any", g)
                worst[k] = max(worst.get(k, 0.0), _rule(f"{tag} call {i} rows [{r0}, {r1}) t#{u} channels {16 * g}:{16 * g + 16}",
                                                        o[r0:r1, :, c], r[r0:r1, :, c], x[r0:r1, :, c], verbose))
            k = ("residual", u if verbose else "any")
            worst[k] = max(worst.get(k, 0.0), _rule(f"{tag} call {i} residual rows [{r0}, {r1})", r_ours[r0:r1], r_ref[r0:r1],
                                                    r_ex[r0:r1], verbose))
        if band is not None:
            b0, b1 = band
            worst["band output"] = max(worst.get("band output", 0.0), _rule(f"{tag} call {i} output rows [{b0}, {b1})", o[b0:b1], r[b0:b1], x[b0:b1]))
            worst["band residual"] = max(worst.get("band residual", 0.0), _rule(f"{tag} call {i} residual rows [{b0}, {b1})",
                                                                                r_ours[b0:b1], r_ref[b0:b1], r_ex[b0:b1]))
    check.worst = worst
    return check


@pytest.mark.gpu
def test_ti2v_5b_one_layer_forward(monkeypatch):
    """Wan2.2 TI2V-5B at 1280 x 704 x 121, one block at dim 3072 / 24 heads / ffn 14 336, 48 channels in and out, `t` per token
    with t = 0 on the first frame's 880 tokens: miss, miss, hit, hit over both CFG slots; then the rule per (range, channel
    group) block, per range of the residual cache and on rows [752, 1008) around the boundary."""
    import magcache_b200 as mc
    from oracle import wan_ref
    _need_device_memory(40)
    _oracle_on_gpu(monkeypatch)
    t0 = time.time()
    model = wan_ref.WanModel(dim=TI2V["dim"], ffn_dim=TI2V["ffn"], num_heads=TI2V["heads"], num_layers=1, in_dim=48,
                             out_dim=48).init_synthetic(51)
    g = torch.Generator().manual_seed(52)
    lat = torch.randn(*TI2V["latent"], generator=g).to(DEV)
    ctx, ctx_null = torch.randn(400, 4096, generator=g).to(DEV), torch.randn(77, 4096, generator=g).to(DEV)
    n = TI2V["n_tok"]
    ratios = mc.tables()[TI2V["table"]][2:].tolist()
    kw = dict(thresh=10.0, K=3, retention_ratio=0.25)  # 4 steps = 8 calls: the window opens at call 2, thresh 10 makes it a hit

    def install(m, who):
        if who is None:
            mc.init_magcache_wan22(m, ratios, 4, **kw)
        else:
            wan_ref.install_magcache_wan22(type(m), ratios, 4, **kw)

    ours, ref_m, m64 = _three(model, "TI2VFull", install)
    del model
    calls = []
    for i, c in enumerate((ctx, ctx_null, ctx, ctx_null)):
        t = torch.full((1, n), 900.0 - 100.0 * (i // 2), device=DEV)
        t[0, :TI2V["first"]] = 0.0
        calls.append(((c, t),) * 3)
    check = _per_range_check("ti2v", TI2V_RUNS, TI2V["grid"], 3, band=(TI2V["first"] - 128, TI2V["first"] + 128))
    skips = _forward_loop("wan2.2-ti2v-5B 1280x704x121", calls, _Call(ours, torch.float32, lat, n), _Call(ref_m, torch.float32, lat, n),
                          _Call(m64, torch.float64, lat, n), wan_ref.exact_fp64, _res, _ATTRS, check=check)
    assert skips == [0, 0, 1, 1], skips
    eng = ours._mc_engine
    assert eng.t_values == 2 and eng.runs == TI2V_RUNS and len(eng.head_groups) == 3
    print("[ti2v blocks] worst fraction of the rule's bound:", {str(k): round(v, 3) for k, v in check.worst.items()})
    _report("wan2.2-ti2v-5B forward", t0)


@pytest.mark.gpu
def test_i2v_14b_720p_one_layer_forward(monkeypatch):
    """Wan2.1 I2V-14B at 1280 x 720 x 81, one block at dim 5120 / 40 heads / ffn 13 824: `y` (20 channels) under the 16 noise
    channels, 257 CLIP tokens of width 1280 through `img_emb` and the image cross-attention summed with the text one; miss,
    miss, hit, hit over both CFG slots."""
    import magcache_b200 as mc
    from oracle import wan_ref
    _need_device_memory(75)
    _oracle_on_gpu(monkeypatch)
    t0 = time.time()
    model = wan_ref.WanModel(dim=I2V["dim"], ffn_dim=I2V["ffn"], num_heads=I2V["heads"], num_layers=1, in_dim=36, model_type="i2v",
                             clip_dim=I2V["clip_dim"]).init_synthetic(61)
    g = torch.Generator().manual_seed(62)
    lat, y = torch.randn(*I2V["latent"], generator=g).to(DEV), torch.randn(*I2V["y"], generator=g).to(DEV)
    clip = torch.randn(1, I2V["clip_len"], I2V["clip_dim"], generator=g).to(DEV)
    ctx, ctx_null = torch.randn(400, 4096, generator=g).to(DEV), torch.randn(77, 4096, generator=g).to(DEV)
    table = mc.tables()[I2V["table"]]
    kw = dict(thresh=10.0, K=3, retention_ratio=0.25)

    def install(m, who):
        if who is None:
            mc.init_magcache(m, 4, mag_ratios=table, **kw)
        else:
            wan_ref.install_magcache(type(m), table, 4, **kw)

    ours, ref_m, m64 = _three(model, "I2VFull", install)
    del model
    n = I2V["n_tok"]
    t = torch.tensor([640.0], device=DEV)
    calls = [((c, t),) * 3 for c in (ctx, ctx_null, ctx, ctx_null)]
    skips = _forward_loop("wan2.1-i2v-14B 720p", calls, _Call(ours, torch.float32, lat, n, clip_fea=clip, y=[y]),
                          _Call(ref_m, torch.float32, lat, n, clip_fea=clip, y=[y]), _Call(m64, torch.float64, lat, n, clip_fea=clip, y=[y]),
                          wan_ref.exact_fp64, _res, _ATTRS)
    assert skips == [0, 0, 1, 1], skips
    _report("wan2.1-i2v-14B 720p forward", t0)


@pytest.mark.gpu
def test_vace_1_3b_one_layer_forward(monkeypatch):
    """VACE-1.3B at 832 x 480 x 81, one main block at dim 1536 / 12 heads / ffn 8960 and its VACE block (96-channel control video,
    `before_proj` mixing, the hint added through the `after_proj` GEMM epilogue): miss, miss, hit, hit over both CFG slots."""
    import magcache_b200 as mc
    from oracle import wan_ref
    _need_device_memory(40)
    _oracle_on_gpu(monkeypatch)
    t0 = time.time()
    model = wan_ref.WanModel(dim=VACE["dim"], ffn_dim=VACE["ffn"], num_heads=VACE["heads"], num_layers=1, model_type="vace",
                             vace_in_dim=VACE["control"][0]).init_synthetic(71)
    g = torch.Generator().manual_seed(72)
    lat, vc = torch.randn(*VACE["latent"], generator=g).to(DEV), torch.randn(*VACE["control"], generator=g).to(DEV)
    ctx, ctx_null = torch.randn(400, 4096, generator=g).to(DEV), torch.randn(77, 4096, generator=g).to(DEV)
    table = mc.tables()[VACE["table"]]
    kw = dict(thresh=10.0, K=3, retention_ratio=0.25)

    def install(m, who):
        if who is None:
            mc.init_magcache(m, 4, mag_ratios=table, **kw)
        else:
            wan_ref.install_magcache(type(m), table, 4, vace=True, **kw)

    ours, ref_m, m64 = _three(model, "VaceFull", install)
    del model
    assert type(ours).forward is mc.magcache_vace_forward
    n = VACE["n_tok"]
    t = torch.tensor([777.0], device=DEV)
    calls = [((c, t),) * 3 for c in (ctx, ctx_null, ctx, ctx_null)]
    skips = _forward_loop("wan2.1-vace-1.3B 480p", calls, _Call(ours, torch.float32, lat, n, vace_context=[vc]),
                          _Call(ref_m, torch.float32, lat, n, vace_context=[vc]), _Call(m64, torch.float64, lat, n, vace_context=[vc]),
                          wan_ref.exact_fp64, _res, _ATTRS)
    assert skips == [0, 0, 1, 1], skips
    _report("wan2.1-vace-1.3B 480p forward", t0)


# ------------------------------------------------------------------------------------------- (b)1 the TI2V head
def _bits(t):
    return t.view(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("w_scale", ["unit", "0.05"])
def test_ti2v_head_six_launches(w_scale):
    """The TI2V head as the engine issues it: for each timestep range u and 16-channel group g (`WanEngine.head_groups` of a
    48-channel engine), one `head_unpatchify` on the range's rows with row_offset r0 and the preparation in slot u * 3 + g, into
    the group's channels of one [48, 31, 44, 80] output — a window of a fenced buffer, filled with NaN. After each launch exactly
    that launch's block (range rows x group channels x 4 patch positions) differs from before, bit for bit; at the end the fence
    holds and no NaN is left. Every element meets `head_chain` at D = 3072; with W = randn / sqrt(3072) (unit-scale outputs) also
    the north star. The fp32-stream and the cache-hit form (bf16 x + fp32 residual). Controls: group 1's reference computed with
    group 2's columns, and row 880 with range 0's modulation (the boundary one row late), must both fail."""
    from magcache_b200 import ops
    from magcache_b200.wan import WAN_CONFIGS, WanEngine
    _need_device_memory(20)
    t0 = time.time()
    D, C, grid, n = TI2V["dim"], TI2V["channels"], TI2V["grid"], TI2V["n_tok"]
    g = torch.Generator(device=DEV).manual_seed(101 if w_scale == "unit" else 102)
    hm = torch.randn(2, D, device=DEV, generator=g) / math.sqrt(D)
    e = torch.randn(2, D, device=DEV, generator=g) * 0.3                     # one time embedding per range
    W = torch.randn(D, 4 * C, device=DEV, generator=g) * (1.0 / math.sqrt(D) if w_scale == "unit" else 0.05)
    b = torch.randn(4 * C, device=DEV, generator=g) * 0.1
    eng = WanEngine(types.SimpleNamespace(dims=WAN_CONFIGS[TI2V["cfg"]], device=torch.device(DEV), head_wt=W, head_b=b))
    groups = eng.head_groups
    assert len(groups) == 3
    x = torch.randn(n, D, device=DEV, generator=g) * 2
    x0, r = x.bfloat16(), torch.randn(n, D, device=DEV, generator=g) * 0.3
    st = [(1.0 + (hm[1] + e[u]), hm[0] + e[u]) for u in range(2)]            # fp32, as the preparation forms them
    preps = {(u, gi): ops.head_prepare(hm, e[u], wt, hb, slot=u * 3 + gi) for u in range(2) for gi, (wt, hb) in enumerate(groups)}
    worst = {}
    for form in ("stream", "hit"):
        flat, buf = fenced((C * grid[0] * 4 * grid[1] * grid[2],), F32, (0, 0, 64, 64), fill="fence")
        flat.fill_(float("nan"))
        out = flat.view(C, grid[0], 2 * grid[1], 2 * grid[2])
        for r0, r1, u in TI2V_RUNS:
            for gi, (wt, hb) in enumerate(groups):
                before = out.clone()
                ops.head_unpatchify(x0[r0:r1] if form == "hit" else x[r0:r1], hm, e[u], wt, hb, grid, c_out=16,
                                    residual=r[r0:r1] if form == "hit" else None, row_offset=r0, out=out[16 * gi:16 * gi + 16],
                                    prep=preps[(u, gi)])
                mask = torch.zeros(n, 4, C, dtype=torch.bool, device=DEV)
                mask[r0:r1, :, 16 * gi:16 * gi + 16] = True
                changed = _bits(out) != _bits(before)
                assert torch.equal(changed, _untokens(mask, grid)), (form, u, gi, int((changed ^ _untokens(mask, grid)).sum()))
                del before, changed, mask
        check_fence(flat, buf)
        assert not bool(out.isnan().any()), form
        tok = _tokens(out, grid).double()
        v = (x0.float() + r) if form == "hit" else x
        for r0, r1, u in TI2V_RUNS:
            s, t = st[u]
            for gi, (wt, hb) in enumerate(groups):
                got = tok[r0:r1, :, 16 * gi:16 * gi + 16].reshape(r1 - r0, 64)
                ref, bound = head_chain(v[r0:r1], s, t, wt, hb)
                err = (got - ref).abs()
                ratio = float(torch.where(err == 0, 0.0, err / bound).max())
                worst[form, "chain"] = max(worst.get((form, "chain"), 0.0), ratio)
                assert ratio <= 1.0, (form, u, gi, ratio)
                if w_scale == "unit":
                    north = float((err / NORTH_STAR(ref)).max())
                    worst[form, "north star"] = max(worst.get((form, "north star"), 0.0), north)
                    assert north <= 1.0, (form, u, gi, north)
                if u == 1 and gi == 1:  # control: group 2's columns in group 1's reference
                    ref_sw, bound_sw = head_chain(v[r0:r1], s, t, *groups[2])
                    worst[form, "control swap"] = float(((got - ref_sw).abs() / bound_sw).max())
                    assert worst[form, "control swap"] > 1.0
                if u == 1:  # control: the boundary one row late (row 880 still at range 0's t = 0)
                    ref_b, bound_b = head_chain(v[r0:r0 + 1], *st[0], wt, hb)
                    rb = float(((got[:1] - ref_b).abs() / bound_b).max())
                    worst[form, "control boundary"] = max(worst.get((form, "control boundary"), 0.0), rb)
                del got, ref, bound, err
        assert worst[form, "control boundary"] > 1.0
        del tok, out, flat, buf
    print(f"[ti2v head W {w_scale}] worst |error| / bound:", {f"{k[0]} {k[1]}": round(val, 3) for k, val in worst.items()})
    _report(f"ti2v head W {w_scale}", t0)


# ------------------------------------------------------------------------------------------- (b)2 row-sliced launches
def _check_rows(n):
    """Rows checked against fp64: the first tile, the 256 rows around the boundary at 880, every 97th row and the last 208
    (the last tile and the ragged 80 rows)."""
    f = TI2V["first"]
    return torch.cat([torch.arange(0, 128), torch.arange(f - 128, f + 128), torch.arange(0, n, 97), torch.arange(n - 208, n)]).unique().to(DEV)


_SLICED_GEMMS = [("o", 3072, 3072), ("ffn2", 3072, 14336)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,N,K", _SLICED_GEMMS, ids=[c[0] for c in _SLICED_GEMMS])
def test_ti2v_row_sliced_gated_gemm(name, N, K):
    """`MC_EPI_BIAS_GATE_RESID` as `WanEngine._gemm_gated` issues it for TI2V: a[880:] into xs[880:] with range 1's gate, then
    a[:880] into xs[:880] with range 0's, on fenced [27 280, K] / [27 280, 3072] buffers. After each launch the other slice's
    rows are bit-unchanged; sampled rows within `gemm_fp64_bounds_ok` of fp64 with their range's gate. Control: row 880 held to
    range 0's gate must fail."""
    from magcache_b200 import _lib as L_
    from magcache_b200 import ops
    _need_device_memory(20)
    n = TI2V["n_tok"]
    g = torch.Generator(device=DEV).manual_seed(N + K)
    a, _ = fenced((n, K), BF, (0, 1, 8, 8))
    _fill(a, g)
    w, _ = fenced((N, K), BF, (0, 1, 8, 8))
    _fill(w, g, 1.0 / math.sqrt(K))
    bias, _ = fenced((N,), F32, (0, 0, 4, 4))
    bias.copy_(torch.randn(N, device=DEV, generator=g).bfloat16().float())
    gates = []
    for _ in range(2):
        gt, _ = fenced((N,), F32, (0, 0, 4, 4))
        gt.copy_(torch.randn(N, device=DEV, generator=g) * 0.5)
        gates.append(gt)
    xs, xbuf = fenced((n, N), F32, (2, 2, 8, 8), fill="fence")
    _fill(xs, g)
    rows = _check_rows(n)
    old = xs[rows].double()
    for r0, r1, u in reversed(TI2V_RUNS):
        before = xs.clone()
        ops.gemm(a[r0:r1], w, bias, L_.MC_EPI_BIAS_GATE_RESID, out=xs[r0:r1], gate=gates[u])
        keep = torch.ones(n, dtype=torch.bool, device=DEV)
        keep[r0:r1] = False
        assert torch.equal(_bits(xs[keep]), _bits(before[keep])), (name, "rows outside the slice changed", u)
        del before
    check_fence(xs, xbuf)
    got = xs[rows].double()
    assert bool(torch.isfinite(got).all())
    pre = a[rows].double() @ w.double().t() + bias.double()
    in0 = (rows < TI2V["first"])[:, None]
    gate = torch.where(in0, gates[0].double(), gates[1].double())
    ok = gemm_fp64_bounds_ok("MC_EPI_BIAS_GATE_RESID", got, pre, old, gate)
    print(f"[ti2v gated gemm {name}] {n} x {N} x {K}: {int((~ok).sum())} of {ok.numel()} checked outputs outside the bound")
    assert bool(ok.all()), (name, int((~ok).sum()))
    # control: the boundary row 880 with range 0's gate
    gate_c = gate.clone()
    gate_c[rows == TI2V["first"]] = gates[0].double()
    bad = ~gemm_fp64_bounds_ok("MC_EPI_BIAS_GATE_RESID", got, pre, old, gate_c)
    print(f"  control (row 880 at range 0's gate): {int(bad.sum())} outputs outside the bound, all on row 880: "
          f"{bool(bad[rows != TI2V['first']].sum() == 0)}")
    assert bool(bad[rows == TI2V["first"]].any()) and not bool(bad[rows != TI2V["first"]].any())


@pytest.mark.gpu
def test_ti2v_row_sliced_ln_modulate():
    """K7 (`ops.ln_modulate`, mode 0) as `WanEngine._ln_modulate` issues it for TI2V: xs[880:] with range 1's modulation rows, then
    xs[:880] with range 0's, into row slices of one fenced bf16 output (row pitch 3072, as the engine's `h`), both the
    self-attention (scale 1, shift 0) and the FFN (scale 4, shift 3) rows, round_ln off and on (block 0). After each launch the
    other slice's rows are bit-unchanged; sampled rows within `_ln_chain`'s bound. Control: row 880 held to range 0's modulation
    must fail."""
    from magcache_b200 import ops
    _need_device_memory(20)
    D, n, f = TI2V["dim"], TI2V["n_tok"], TI2V["first"]
    g = torch.Generator(device=DEV).manual_seed(111)
    x, _ = fenced((n, D), F32, (0, 8, 0, 0), pitch=D)
    _fill(x, g, 3.0, 0.5)
    em = torch.randn(2, 6, D, device=DEV, generator=g) * 0.3
    rows = _check_rows(n)
    worst, control = 0.0, 0.0
    for si, hi in ((1, 0), (4, 3)):
        for round_ln in (0, 1):
            out, obuf = fenced((n, D), BF, (2, 2, 0, 0), fill="fence", pitch=D)
            for r0, r1, u in reversed(TI2V_RUNS):
                before = out.clone()
                ops.ln_modulate(x[r0:r1], em[u], si, hi, eps=1e-6, round_ln_to_bf16=bool(round_ln), out=out[r0:r1])
                keep = torch.ones(n, dtype=torch.bool, device=DEV)
                keep[r0:r1] = False
                assert torch.equal(out[keep].view(torch.int16), before[keep].view(torch.int16)), (si, round_ln, u)
                del before
            check_fence(out, obuf)
            got = out[rows].double()
            assert bool(torch.isfinite(got).all())
            for u, sel in enumerate((rows < f, rows >= f)):
                ref, bound = _ln_chain(x[rows[sel]], em[u][si], em[u][hi], 0, round_ln, True)
                r = float(((got[sel] - ref).abs() / bound).max())
                worst = max(worst, r)
                assert r <= 1.0, (si, round_ln, u, r)
            i880 = int((rows == f).nonzero())
            ref, bound = _ln_chain(x[f:f + 1], em[0][si], em[0][hi], 0, round_ln, True)  # control: range 0's rows on row 880
            rc = float(((got[i880:i880 + 1] - ref).abs() / bound).max())
            control = rc if control == 0.0 else min(control, rc)
            assert rc > 1.0, (si, round_ln, rc)
            del out, obuf
    print(f"[ti2v K7 row slices] worst error / bound {worst:.3f}; control (row 880 at range 0's modulation) {control:.1f}x the bound")


# ------------------------------------------------------------------------------------------- (b)3 8 values in 64 ranges
@pytest.mark.gpu
def test_eight_timestep_values_in_64_ranges(monkeypatch):
    """A one-layer TI2V-width model (dim 3072, 24 heads, ffn 14 336, 48 channels) on a 4 x 16 x 24 grid (1536 tokens) with `t`
    carrying 8 distinct values in 64 ranges (`_many_ranges`): the engine's limits, so the time MLP runs at M = 8 and the head
    prepares 8 x 3 = 24 slots. miss, miss, hit, hit through `magcache_wan22_forward` against the bf16 and fp64 oracles, the rule
    on every (range, channel group) block and on every range of the residual cache. Control: against oracles whose eighth value's
    rows carry the seventh value (M = 8 computed as M = 7), the rule must fail on exactly the eighth value's ranges."""
    import magcache_b200 as mc
    from magcache_b200 import ops
    from oracle import wan_ref
    _need_device_memory(20)
    _oracle_on_gpu(monkeypatch)
    t0 = time.time()
    model = wan_ref.WanModel(dim=TI2V["dim"], ffn_dim=TI2V["ffn"], num_heads=TI2V["heads"], num_layers=1, in_dim=48,
                             out_dim=48).init_synthetic(121)
    g = torch.Generator().manual_seed(122)
    lat = torch.randn(*MANY["latent"], generator=g).to(DEV)
    ctx, ctx_null = torch.randn(400, 4096, generator=g).to(DEV), torch.randn(77, 4096, generator=g).to(DEV)
    n, grid = MANY["n_tok"], MANY["grid"]
    t, runs = _many_ranges(n, 8, 64)
    t = t.to(DEV)
    ratios = mc.tables()[TI2V["table"]][2:].tolist()
    kw = dict(thresh=10.0, K=3, retention_ratio=0.25)

    def install(m, who):
        if who is None:
            mc.init_magcache_wan22(m, ratios, 4, **kw)
        else:
            wan_ref.install_magcache_wan22(type(m), ratios, 4, **kw)

    ours, ref_m, m64 = _three(model, "Many", install)
    calls = [((c, t),) * 3 for c in (ctx, ctx_null, ctx, ctx_null)]
    check = _per_range_check("8 values / 64 ranges", runs, grid, 3, verbose=False)
    first = {}
    inner = check

    def keep_first(i, out, *rest):
        if i == 0:
            first["out"] = out
        inner(i, out, *rest)

    skips = _forward_loop("ti2v width, 8 values in 64 ranges", calls, _Call(ours, torch.float32, lat, n), _Call(ref_m, torch.float32, lat, n),
                          _Call(m64, torch.float64, lat, n), wan_ref.exact_fp64, _res, _ATTRS, check=keep_first)
    assert skips == [0, 0, 1, 1], skips
    eng = ours._mc_engine
    assert eng.t_values == 8 and eng.runs == runs
    assert eng.time_embedding()[1].shape == (8, 6, TI2V["dim"])
    assert max(u * 3 + gi for u, gi in eng._head_prep) == 23 and ("head23", torch.device(DEV).index or 0) in ops._WORKSPACES
    print("[8 values / 64 ranges] worst fraction of the rule's bound:", {str(k): round(v, 3) for k, v in check.worst.items()})

    # control: M = 8 computed as M = 7
    del ref_m, m64
    t7 = t.clone()
    t7[t == MANY["values"][7]] = MANY["values"][6]
    _, ref_w, m64_w = _three(model, "ManyM7", install)
    with torch.no_grad():
        ref = _Call(ref_w, torch.float32, lat, n)(ctx, t7).float().cpu()
        with wan_ref.exact_fp64():
            ex = _Call(m64_w, torch.float64, lat, n)(ctx, t7).cpu()
    o, r, x = (_tokens(v, grid) for v in (first["out"], ref, ex))
    failed = []
    for r0, r1, u in runs:
        try:
            _rule("", o[r0:r1], r[r0:r1], x[r0:r1], verbose=False)
        except AssertionError:
            failed.append((r0, u))
    # self-attention carries the eighth value's changed keys into every row, so other ranges may fail too; the eighth's must
    print(f"  control (M = 7): the rule fails on {len(failed)} of {len(runs)} ranges, "
          f"{sum(u == 7 for _, u in failed)} of the {sum(u == 7 for _, _, u in runs)} ranges of the eighth value")
    assert all((r0, u) in failed for r0, _, u in runs if u == 7)
    _report("8 values / 64 ranges", t0)


# ------------------------------------------------------------------------------------------- (b)4 the time path
@pytest.mark.gpu
def test_time_path_per_element():
    """`time_sinusoid` (t = 0 exactly; t = 999; timesteps rounded to bf16 as a bf16 pipeline passes them) against the oracle's
    fp64 `sinusoidal_embedding_1d`: within half an fp32 ulp plus 1e-12 (the kernel evaluates in fp64 and rounds once).
    `linear_f32_small` at every M in 1..8, K in {256, 3072}, N in {3072, 18 432}, act 0 / 1 / 2, per element against fp64 within
    the bound of the module docstring. Control: the M = 8 launch against a reference whose row 7 is row 6's (M computed as 7)
    must fail."""
    from magcache_b200 import ops
    from oracle import wan_ref
    D = TI2V["dim"]
    g = torch.Generator(device=DEV).manual_seed(131)
    ts = torch.tensor([0.0, 999.0, 981.73, 640.31, 1.7, 27.0]).bfloat16().double()
    ts[1] = 999.0
    got = ops.time_sinusoid(ts.to(DEV), 256).double()
    ref = wan_ref.sinusoidal_embedding_1d(256, ts).to(DEV)
    r = float(((got - ref).abs() / (U32 * ref.abs() + 1e-12)).max())
    assert r <= 1.0, r
    assert torch.equal(got[0, :128], torch.ones(128, dtype=torch.float64, device=DEV)) and torch.equal(got[0, 128:], torch.zeros(128, dtype=torch.float64, device=DEV))
    worst = {}
    control = None
    for K in (256, D):
        for N in (D, 6 * D):
            w = torch.randn(N, K, device=DEV, generator=g) * 0.02
            b = torch.randn(N, device=DEV, generator=g) * 0.02
            for act in (0, 1, 2):
                xall = torch.randn(8, K, device=DEV, generator=g)
                for M in range(1, 9):
                    x = xall[:M].contiguous()
                    y = ops.linear_f32_small(x, w, b, act=act).double()
                    x64 = x.double()
                    if act == 1:
                        x64 = F.silu(x64)
                    pre = x64 @ w.double().t() + b.double()
                    L = K // 32 + 5
                    gam = L * U32 / (1 - L * U32)
                    sabs = x64.abs() @ w.double().abs().t()
                    e_pre = (gam + (5 * U32 if act == 1 else 0.0)) * sabs + U32 * pre.abs()
                    if act == 2:
                        ref = F.silu(pre)
                        bound = 1.1 * e_pre + 5 * U32 * ref.abs()
                    else:
                        ref, bound = pre, e_pre
                    err = (y - ref).abs()
                    rr = float((err / bound).max())
                    worst[act] = max(worst.get(act, 0.0), rr)
                    assert rr <= 1.0, (M, K, N, act, rr)
                    if M == 8:  # control: row 7 computed from row 6
                        wrong = ref.clone()
                        wrong[7] = ref[6]
                        rc = float(((y[7] - wrong[7]).abs() / bound[7]).max())
                        control = rc if control is None else min(control, rc)
                        assert rc > 1.0, (K, N, act, rc)
    print(f"[time path] time_sinusoid worst error / bound {r:.3f}; linear_f32_small worst error / bound by act {worst}; "
          f"control (M = 7) at least {control:.0f}x the bound")


# ------------------------------------------------------------------------------------------- (b)5 I2V's image branch
def _sdpa_rule(got, ref, sd):
    """test_attention_full_key_sequence_vs_fp64's criterion (as in test_fullshape_workloads_gpu's `_attention_case`): returns
    (passes, worst fraction of the SDPA-relative bounds, printable numbers)."""
    err, err_sd = (got - ref).abs(), (sd - ref).abs()
    e_ours, e_sdpa = rel_l2(got, ref), rel_l2(sd, ref)
    m, m_sd, mean = float(err.max()), float(err_sd.max()), float(err.mean())
    ok = e_ours <= 2.0 * e_sdpa + 1e-4 and m <= 2.0 * m_sd + 1e-3 and e_ours < 8e-3 and mean < 2e-3
    ratio = max(e_ours / (2.0 * e_sdpa + 1e-4), m / (2.0 * m_sd + 1e-3))
    return ok, ratio, f"rel-L2 vs fp64 ours {e_ours:.3e}, SDPA {e_sdpa:.3e}; max abs ours {m:.3e}, SDPA {m_sd:.3e}; mean {mean:.2e}"


@pytest.mark.gpu
def test_i2v_image_and_text_cross_attention_75600_rows():
    """The i2v block's two cross-attentions at 75 600 query rows x 40 heads, in the engine's buffers: q = cq [75 600, 5120], k | v
    column halves of one [L, 10 240] buffer (ckv_img for the 257 CLIP keys, ckv for the 512 text keys) with 128 NaN rows after
    it, the output a row window (pitch 5120) of a fenced buffer. Every query row against fp64 at the SDPA-relative criterion.
    Control: the CLIP result against a reference without the 257th key (the ragged last 64-key tile) must fail."""
    from magcache_b200 import ops
    _need_device_memory(40)
    t0 = time.time()
    n, H, W = I2V["n_tok"], I2V["heads"], I2V["dim"]
    g = torch.Generator(device=DEV).manual_seed(141)
    q = torch.empty(n, W, dtype=BF, device=DEV)
    _fill(q, g)
    for Lk, what in ((I2V["clip_len"], "clip"), (I2V["text_len"], "text")):
        kv, _ = fenced((Lk, 2 * W), BF, (0, 128, 0, 0))
        _fill(kv, g)
        k, v = kv[:, :W], kv[:, W:]
        out, obuf = fenced((n, W), BF, (1, 1, 0, 0), fill="fence", pitch=W)
        ops.attention(q, k, v, H, out=out)
        check_fence(out, obuf)
        got = out.float()
        assert bool(torch.isfinite(got).all()), what
        ref = _attn_ref64(q, k, v, H).float()
        sd = F.scaled_dot_product_attention(*(t.reshape(t.shape[0], H, 128).transpose(0, 1)[None] for t in (q, k, v)))
        sd = sd[0].transpose(0, 1).reshape(n, W).float()
        ok, ratio, msg = _sdpa_rule(got, ref, sd)
        print(f"[i2v cross-attention {what}: {n} rows x {H} heads over {Lk} keys] {msg}; worst bound ratio {ratio:.2f}")
        assert ok, (what, msg)
        if what == "clip":  # control: the 257th key dropped from the reference (and from SDPA's)
            ref_c = _attn_ref64(q, k[:Lk - 1], v[:Lk - 1], H).float()
            sd_c = F.scaled_dot_product_attention(*(t.reshape(t.shape[0], H, 128).transpose(0, 1)[None] for t in (q, k[:Lk - 1], v[:Lk - 1])))
            sd_c = sd_c[0].transpose(0, 1).reshape(n, W).float()
            ok_c, ratio_c, msg_c = _sdpa_rule(got, ref_c, sd_c)
            print(f"  control (256 keys in the reference): {msg_c}; bound ratio {ratio_c:.2f}")
            assert not ok_c
            del ref_c, sd_c
        del out, obuf, got, ref, sd, kv
    _report("i2v cross-attention", t0)


@pytest.mark.gpu
def test_i2v_img_emb_chain():
    """`img_emb` as `WanEngine.prologue` runs it on the 257 x 1280 CLIP features: `ln_affine` (eps 1e-5) -> bf16, the GELU(erf)
    GEMM 1280 -> 1280, the GEMM 1280 -> 5120, `ln_affine` -> bf16; each stage on the previous stage's output, fenced (the
    LayerNorms write rows of pitch 1280 / 5120 like the engine's buffers, the GEMMs windows of wider buffers), per element against
    fp64: `_ln_chain` for the LayerNorms, `gemm_fp64_bounds_ok` for the GEMMs. Weights at `WanWeights.random`'s scales."""
    from magcache_b200 import _lib as L_
    from magcache_b200 import ops
    Lc, Cd, D = I2V["clip_len"], I2V["clip_dim"], I2V["dim"]
    g = torch.Generator(device=DEV).manual_seed(151)
    clip = torch.randn(Lc, Cd, device=DEV, generator=g) * 2 + 0.3
    ln1_w, ln1_b = 1 + 0.1 * torch.randn(Cd, device=DEV, generator=g), 0.02 * torch.randn(Cd, device=DEV, generator=g)
    w1, b1 = (0.02 * torch.randn(Cd, Cd, device=DEV, generator=g)).bfloat16(), (0.02 * torch.randn(Cd, device=DEV, generator=g)).bfloat16().float()
    w2, b2 = (0.02 * torch.randn(D, Cd, device=DEV, generator=g)).bfloat16(), (0.02 * torch.randn(D, device=DEV, generator=g)).bfloat16().float()
    ln2_w, ln2_b = 1 + 0.1 * torch.randn(D, device=DEV, generator=g), 0.02 * torch.randn(D, device=DEV, generator=g)
    worst = {}

    def ln(x, w, b, cols, what):
        out, obuf = fenced((Lc, cols), BF, (2, 2, 0, 0), fill="fence", pitch=cols)
        ops.ln_affine(x, w, b, eps=1e-5, out=out)
        check_fence(out, obuf)
        ref, bound = _ln_chain(x, w, b, 1, 0, True, eps=1e-5)
        worst[what] = float(((out.double() - ref).abs() / bound).max())
        assert worst[what] <= 1.0, (what, worst[what])
        return out

    def gemm(a, w, b, epi, what):
        out, obuf = fenced((Lc, w.shape[0]), BF, (2, 2, 8, 8), fill="fence")
        ops.gemm(a, w, b, getattr(L_, epi), out=out)
        check_fence(out, obuf)
        pre = a.double() @ w.double().t() + b.double()
        ok = gemm_fp64_bounds_ok(epi, out.double(), pre)
        worst[what] = int((~ok).sum())
        assert bool(ok.all()), (what, int((~ok).sum()))
        return out

    h1 = ln(clip, ln1_w, ln1_b, Cd, "ln1")
    h2 = gemm(h1, w1, b1, "MC_EPI_BIAS_GELU_ERF_BF16", "linear1 + GELU(erf): outputs outside the bound")
    h3 = gemm(h2, w2, b2, "MC_EPI_BIAS_BF16", "linear2: outputs outside the bound")
    ln(h3.contiguous(), ln2_w, ln2_b, D, "ln2")
    print(f"[i2v img_emb 257 x 1280 -> 5120] {worst}")


# ------------------------------------------------------------------------------------------- (b)6 patchify
@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["i2v", "ti2v", "vace"])
def test_patchify_variant_channels(variant):
    """`mc_patchify` at C = 36 (I2V: the noise latents and `y` as the engine stages them), 48 (TI2V) and 96 (VACE's control video)
    on the full latent shapes, into a fenced [tokens, 4 C] bf16 buffer: bit-equal to bf16 of the view / permute statement of the
    (1, 2, 2) patch (column c * 4 + 2 kh + kw of token (f, h, w))."""
    from magcache_b200 import _lib as L_
    from magcache_b200 import ops
    _need_device_memory(10)
    shape = {"i2v": (36,) + I2V["latent"][1:], "ti2v": TI2V["latent"], "vace": VACE["control"]}[variant]
    C, Fr, Hh, Ww = shape
    g = torch.Generator(device=DEV).manual_seed(161 + C)
    lat = torch.randn(*shape, device=DEV, generator=g) * 3
    n = Fr * (Hh // 2) * (Ww // 2)
    out, obuf = fenced((n, 4 * C), BF, (2, 2, 0, 0), fill="fence", pitch=4 * C)
    L_.check(L_.lib.mc_patchify(lat.data_ptr(), C, Fr, Hh, Ww, out.data_ptr(), ops._stream()))
    check_fence(out, obuf)
    ref = lat.bfloat16().view(C, Fr, Hh // 2, 2, Ww // 2, 2).permute(1, 2, 4, 0, 3, 5).reshape(n, 4 * C)
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16)), (variant, int((out.view(torch.int16) != ref.view(torch.int16)).sum()))
    print(f"[patchify {variant}] C = {C}, {n} tokens: bit-equal")
