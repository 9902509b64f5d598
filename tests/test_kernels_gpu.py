"""GPU parity of every hand-written kernel against a plain PyTorch fp32 reference of the same op (called through the C ABI).

Tolerances (stated per test): integer/bit-exact for the fp32 add/sub; <= 1 bf16 ulp for bf16 outputs whose fp32 pre-image is
compared at rtol 1e-3 / atol 1e-4 (the north-star tolerance); statistics at 1e-5 absolute.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ops():
    from magcache_b200 import ops
    return ops


def _lib():
    from magcache_b200 import _lib
    return _lib


def bf16_ulp_close(got, ref_f32, extra_atol=0.0):
    """got (bf16) must equal ref rounded to bf16 up to one bf16 ulp (2^-8 relative) — the rounding of an fp32 value that
    itself carries rtol 1e-3/atol 1e-4 accumulation-order noise."""
    g = got.float()
    tol = ref_f32.abs() * (2.0 ** -7) + 1e-4 + extra_atol
    bad = (g - ref_f32).abs() > tol
    return int(bad.sum().item()), float((g - ref_f32).abs().max().item())


# ------------------------------------------------------------------------------------------- cache kernels
@pytest.mark.parametrize("n", [0, 1, 7, 8, 1000, 4096 * 3 + 5, 32760 * 1536])
def test_cache_hit_add_wan_dtypes(n):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(n % 1000)
    x = torch.randn(n, device=DEV, generator=g).bfloat16()
    r = torch.randn(n, device=DEV, generator=g) * 0.1
    out = ops.cache_hit_add(x, r)
    ref = x + r  # torch promotes bf16 + fp32 -> fp32
    assert out.dtype == torch.float32
    assert torch.equal(out, ref)  # bit-exact


@pytest.mark.parametrize("dx,dr", [(torch.bfloat16, torch.bfloat16), (torch.float32, torch.float32), (torch.float32, torch.bfloat16)])
def test_cache_hit_add_other_dtypes(dx, dr):
    ops = _ops()
    n = 4096 * 3072 + 3
    x = torch.randn(n, device=DEV).to(dx)
    r = (torch.randn(n, device=DEV) * 0.1).to(dr)
    assert torch.equal(ops.cache_hit_add(x, r), x + r)
    assert torch.equal(ops.residual_sub(x, r), x - r)


def test_hit_then_sub_roundtrip_full_size():
    """Size-independent property at the BASELINE config-2 size: (x + r) - x == r exactly when the add did not round,
    and always |((x + r) - x) - r| <= ulp(x + r)."""
    ops = _ops()
    n = 32760 * 1536
    x = torch.randn(n, device=DEV).bfloat16()
    r = torch.randn(n, device=DEV) * 0.05
    y = ops.cache_hit_add(x, r)
    back = ops.residual_sub(y, x)
    assert torch.equal(back, (x + r) - x)
    err = (back - r).abs()
    assert float(err.max()) <= float((y.abs().max() * 2 ** -23) * 2)


def test_residual_sub_unaligned_and_ragged():
    ops = _ops()
    base_o = torch.randn(1024 + 3, device=DEV)
    base_i = torch.randn(1024 + 3, device=DEV).bfloat16()
    xo, xi = base_o[1:1001].contiguous(), base_i[:1000].contiguous()
    assert torch.equal(ops.residual_sub(xo, xi), xo - xi)


def test_cfg_combine_bit_exact():
    """wan_magcache.py:301-302 on the full latent shape and on a ragged/unaligned one."""
    ops = _ops()
    for shape, off in [((16, 21, 60, 104), 0), ((1003,), 1)]:
        n = int(torch.tensor(shape).prod()) + off
        cond = torch.randn(n, device=DEV)[off:].contiguous() if off == 0 else torch.randn(n, device=DEV)[off:]
        uncond = torch.randn(cond.shape, device=DEV)
        cond = cond.contiguous()
        for g in (5.0, 6.0, 1.0, 7.5):
            assert torch.equal(ops.cfg_combine(cond, uncond, g), uncond + g * (cond - uncond))


def _cfg_step_torch(cond, uncond, g, x, coef_v, coef_x=1.0, hist=(), coef_h=(), sigma=0.0):
    f = lambda a: torch.tensor(a, dtype=torch.float32, device=x.device)  # noqa: E731
    v = uncond + f(g) * (cond - uncond)
    acc = f(coef_x) * x + f(coef_v) * v
    for h, c in zip(hist, coef_h):
        acc = acc + f(c) * h
    return acc, x - f(sigma) * v


@pytest.mark.parametrize("n,off", [(16 * 21 * 60 * 104, 0), (1003, 0), (4099, 3), (7, 0)])
def test_cfg_step_bit_exact(n, off):
    """`mc_cfg_step` (CFG combine + scheduler update, wan_magcache.py:301-310) against the chain of torch eager kernels it
    replaces — same rounding order, so bit-equal: Euler form, in-place update, 1..4 history terms, x0 output, ragged and
    unaligned sizes (the unaligned views take the scalar tail kernel)."""
    ops = _ops()
    mk = lambda: torch.randn(n + off, device=DEV)[off:] if off else torch.randn(n, device=DEV)  # noqa: E731
    cond, uncond, x = mk().contiguous(), mk().contiguous(), mk().contiguous()
    if off:  # keep the storage offset (mis-aligned pointers) — .contiguous() above is a no-op for a 1-D slice
        assert cond.data_ptr() % 32 != 0
    d = -0.0123
    want, _ = _cfg_step_torch(cond, uncond, 5.0, x, d)
    assert torch.equal(want, x + d * (uncond + 5.0 * (cond - uncond)))  # the literal caller expression
    assert torch.equal(ops.cfg_step(cond, uncond, 5.0, x, d), want)
    xin = x.clone()
    assert ops.cfg_step(cond, uncond, 5.0, xin, d, out=xin) is xin and torch.equal(xin, want)
    hist = [mk().contiguous() for _ in range(4)]
    coefs = [0.37, -1.9, 0.004, 2.5]
    for k in range(1, 5):
        x0 = torch.empty_like(x)
        got = ops.cfg_step(cond, uncond, 6.5, x, -0.7, coef_x=0.93, hist=hist[:k], coef_h=coefs[:k], sigma=0.81, x0_out=x0)
        want, want0 = _cfg_step_torch(cond, uncond, 6.5, x, -0.7, 0.93, hist[:k], coefs[:k], 0.81)
        assert torch.equal(got, want) and torch.equal(x0, want0), k
    # no-guidance form used by the sampler's predictor launch: cond = uncond = m, g = 0  ->  v = m exactly
    got = ops.cfg_step(x, x, 0.0, cond, 0.25, coef_x=0.5)
    assert torch.equal(got, torch.tensor(0.5, device=DEV) * cond + torch.tensor(0.25, device=DEV) * x)


def test_cfg_step_rejects_aliasing_and_bad_history():
    ops = _ops()
    from magcache_b200._lib import MagCacheError
    a, b, x = (torch.randn(64, device=DEV) for _ in range(3))
    with pytest.raises(MagCacheError):
        ops.cfg_step(a, b, 1.0, x, 0.1, out=a)  # out may alias x only
    with pytest.raises(MagCacheError):
        ops.cfg_step(a, b, 1.0, x, 0.1, x0_out=x)
    with pytest.raises(AssertionError):
        ops.cfg_step(a, b, 1.0, x, 0.1, hist=[a] * 5, coef_h=[1.0] * 5)


def test_unipc_sampler_on_the_kernel_matches_the_oracle():
    """magcache_b200/sampler.py on the real kernel: 20 UniPC steps (two launches each) and 20 Euler steps of a synthetic
    two-branch flow model against oracle/sampler_ref.py in float64."""
    from magcache_b200 import sampler as S
    from oracle import sampler_ref as R
    ops = _ops()

    def model_v(z, sigma, branch):
        c = 0.7 if branch == 0 else -0.2
        return torch.tanh(1.3 * z + c) * (0.5 + float(sigma)) - 0.8 * z * float(sigma)

    sig = S.sampling_sigmas(20, 5.0)
    sig[0] = 0.9999
    x0 = torch.randn(16, 21, 60, 104, device=DEV)
    for name, smp, ref in [("unipc", S.FlowUniPCSampler(sig), R.UniPCRef(torch.tensor(sig, dtype=torch.float64))),
                           ("euler", S.FlowEulerSampler(sig), R.EulerRef(torch.tensor(sig, dtype=torch.float64)))]:
        x, xr = x0.clone(), x0.double()
        launches0 = ops.LAUNCHES
        for i in range(20):
            x = smp.step(model_v(x, sig[i], 0), model_v(x, sig[i], 1), 5.0, x)
            xr = ref.step(R.cfg(model_v(xr, sig[i], 0), model_v(xr, sig[i], 1), 5.0), xr)
            err = float((x.double() - xr).abs().max()) / max(1.0, float(xr.abs().max()))
            assert err < 5e-5, (name, i, err)
        assert ops.LAUNCHES - launches0 == (40 if name == "unipc" else 20)


@pytest.mark.parametrize("n", [1536, 6 * 1536, 6 * 5120, 7])
def test_rel_l1_matches_the_reference_expression(n):
    """`((cur - prev).abs().mean() / prev.abs().mean()).cpu().item()` (wan_teacache.py:543) to fp32 precision."""
    ops = _ops()
    prev = torch.randn(n, device=DEV)
    cur = prev + 0.05 * torch.randn(n, device=DEV)
    want = ((cur - prev).abs().mean() / prev.abs().mean()).cpu().item()
    got = ops.rel_l1(cur, prev)
    exact = float((cur.double() - prev.double()).abs().mean() / prev.double().abs().mean())
    assert abs(got - exact) <= 2e-7 * exact + abs(want - exact), (got, want, exact)  # at least as close to exact as torch's fp32 value
    assert abs(got - want) <= 1e-6 * want


def test_cache_kernels_hunyuan_720p_shape():
    """BASELINE configs[3] (HunyuanVideo 720p x 129 frames: [1, 118800, 3072], all bf16): hit add / residual sub bit-exact."""
    ops = _ops()
    n = 118800 * 3072
    x = torch.randn(n, device=DEV).bfloat16()
    r = (torch.randn(n, device=DEV) * 0.2).bfloat16()
    y = ops.cache_hit_add(x, r)
    assert y.dtype == torch.bfloat16 and torch.equal(y, x + r)
    assert torch.equal(ops.residual_sub(y, x), y - x)


def _ref_stats(r, p, eps=0.0):
    ratio = r.norm(dim=-1) / (p.norm(dim=-1) + eps)
    return ratio.mean().item(), ratio.std().item(), (1 - torch.nn.functional.cosine_similarity(r, p, dim=-1, eps=1e-8)).mean().item()


# fp32 up to ~3000 columns: the staged kernel; 5120 fp32 columns (fewer than two stages fit) and bf16: the warp-per-row kernel
@pytest.mark.parametrize("shape,dtype", [((1, 64, 96), torch.float32), ((2, 33, 1536), torch.float32), ((1, 32760, 1536), torch.float32),
                                         ((1, 777, 5120), torch.float32), ((2, 515, 1536), torch.bfloat16)])
def test_residual_stats(shape, dtype):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(5)
    p = torch.randn(*shape, device=DEV, generator=g) * 0.1
    r = p * (0.97 + 0.05 * torch.rand(shape[0], shape[1], 1, device=DEV, generator=g)) + 0.01 * torch.randn(*shape, device=DEV, generator=g)
    r, p = r.to(dtype), p.to(dtype)
    got = ops.residual_stats(r, p)
    ref = _ref_stats(r.double(), p.double())
    for a, b in zip(got, ref):
        assert abs(a - b) < 1e-5, (got, ref)


def test_residual_sub_stats_fused():
    ops = _ops()
    rows, cols = 4095, 1536
    xi = torch.randn(rows, cols, device=DEV).bfloat16()
    p = torch.randn(rows, cols, device=DEV) * 0.1
    xo = xi.float() + p * 1.02 + 0.003 * torch.randn(rows, cols, device=DEV)
    r, st = ops.residual_sub_stats(xo, xi, p)
    assert torch.equal(r, xo - xi)
    ref = _ref_stats((xo - xi).double(), p.double())
    for a, b in zip(st, ref):
        assert abs(a - b) < 1e-5


# ------------------------------------------------------------------------------------------- row-wise kernels
def test_patchify_matches_conv3d_im2col():
    ops = _ops()
    lat = torch.randn(16, 3, 8, 12, device=DEV)
    tok = ops.patchify(lat)
    # reference: unfold the (1,2,2) patches in (c, kh, kw) order
    C, F, H, W = lat.shape
    ref = lat.view(C, F, H // 2, 2, W // 2, 2).permute(1, 2, 4, 0, 3, 5).reshape(F * (H // 2) * (W // 2), C * 4).bfloat16()
    assert torch.equal(tok, ref)
    # and against an actual Conv3d: tokens @ W.flatten(1).T == conv output
    conv = torch.nn.Conv3d(16, 32, kernel_size=(1, 2, 2), stride=(1, 2, 2), device=DEV)
    y = conv(lat.bfloat16().float().unsqueeze(0))[0].flatten(1).t()
    y2 = tok.float() @ conv.weight.flatten(1).t() + conv.bias
    assert torch.allclose(y, y2, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("rows,cols,xdt", [(37, 1536, torch.float32), (130, 5120, torch.float32), (64, 1536, torch.bfloat16), (5, 256, torch.float32),
                                           # >= 1024 rows: the TMA-staged form (ragged last group of 8 rows, 2-8 ring stages)
                                           (1029, 1536, torch.float32), (4099, 1536, torch.bfloat16), (2050, 384, torch.float32),
                                           (1500, 2048, torch.float32), (1025, 3072, torch.float32),
                                           # cols 1024: four groups per lane (G = 4), the register and the staged form
                                           (300, 1024, torch.bfloat16), (1029, 1024, torch.float32)])
def test_ln_modulate(rows, cols, xdt):
    ops = _ops()
    x = (torch.randn(rows, cols, device=DEV) * 3 + 0.5).to(xdt)
    mod = torch.randn(6, cols, device=DEV) / math.sqrt(cols)
    e = torch.randn(6, cols, device=DEV) * 0.2
    round_ln = xdt == torch.bfloat16
    em = ops.cache_hit_add(mod, e)  # e = modulation + e0 (fp32), as the engine forms it once per layer
    assert torch.equal(em, mod + e)
    out32 = ops.ln_modulate(x, em, 1, 0, round_ln_to_bf16=round_ln, out_dtype=torch.float32)
    ln = torch.nn.functional.layer_norm(x.float(), (cols,), eps=1e-6)
    if round_ln:
        ln = ln.to(xdt).float()
    ee = mod + e
    ref = ln * (1 + ee[1]) + ee[0]
    # tolerance: rtol 1e-3 / atol 1e-4 (north star) -- fp32 LN statistics differ only by summation order; with round_ln the
    # bf16 rounding of LN may flip by one ulp (2^-8 relative) on a handful of elements
    if round_ln:
        assert ((out32 - ref).abs() <= ref.abs() * 2 ** -7 + 1e-2).all()
        assert ((out32 - ref).abs() > 1e-4 + 1e-3 * ref.abs()).float().mean() < 0.01
    else:
        assert torch.allclose(out32, ref, rtol=1e-3, atol=1e-4)
    out16 = ops.ln_modulate(x, em, 1, 0, round_ln_to_bf16=round_ln)
    assert torch.equal(out16, out32.bfloat16())


@pytest.mark.parametrize("rows", [77, 3003])
def test_ln_affine(rows):
    ops = _ops()
    x = torch.randn(rows, 1536, device=DEV) * 2
    w = torch.randn(1536, device=DEV)
    b = torch.randn(1536, device=DEV)
    out = ops.ln_affine(x, w, b, out_dtype=torch.float32)
    ref = torch.nn.functional.layer_norm(x, (1536,), w, b, eps=1e-6)
    assert torch.allclose(out, ref, rtol=1e-3, atol=1e-4)


def _rope_ref(x, cos_sin, heads):
    rows, cols = x.shape
    hd = cols // heads
    xc = torch.view_as_complex(x.double().reshape(rows, heads, hd // 2, 2))
    cs = cos_sin.double().reshape(rows, 1, hd // 2, 2)
    fr = torch.complex(cs[..., 0], cs[..., 1])
    return torch.view_as_real(xc * fr).reshape(rows, cols).float()


@pytest.mark.parametrize("rows,cols,heads,rope", [(100, 1536, 12, True), (512, 1536, 12, False), (33, 5120, 40, True),
                                                  (1027, 1536, 12, True), (4101, 1536, 12, False), (2049, 256, 2, True)])  # TMA-staged form
def test_rmsnorm_rope(rows, cols, heads, rope):
    ops = _ops()
    x = torch.randn(rows, 2 * cols, device=DEV).bfloat16()
    view = x[:, cols:]  # strided view, like q/k inside a fused projection buffer
    w = 1 + 0.1 * torch.randn(cols, device=DEV)
    ang = torch.rand(rows, 64, device=DEV, dtype=torch.float64) * 6.28
    cos_sin = torch.stack([ang.cos(), ang.sin()], -1).reshape(rows, 128).float() if rope else None
    xf = view.float()
    ref = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)).bfloat16().float() * w
    if rope:
        ref = _rope_ref(ref, cos_sin, heads)
    keep = x[:, :cols].clone()
    ops.rmsnorm_rope_(view, w, cos_sin, 128)
    assert torch.equal(x[:, :cols], keep)  # the other half of the buffer is untouched
    # two successive bf16 roundings (after the norm, after weight/RoPE): an fp32-ulp difference in rsqrt can flip the first
    # one, so allow 2 bf16 ulps (2^-6 relative) element-wise but require > 99.99 % of elements within 1 ulp
    err = (view.float() - ref).abs()
    # RoPE mixes the two elements of a pair: a flipped rounding of either one moves BOTH outputs by up to an ulp of the pair's
    # magnitude (which the rotation preserves), however small one output happens to be
    mag = ref.view(rows, -1, 2).norm(dim=-1, keepdim=True).expand(-1, -1, 2).reshape(rows, cols) if rope else ref.abs()
    assert (err <= mag * 2.0 ** -6 + 1e-4).all(), float(err.max())
    nbad, maxerr = bf16_ulp_close(view, ref)
    assert nbad <= 1e-4 * view.numel(), (nbad, maxerr)


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("grid", [(3, 5, 7), (5, 30, 52)])
def test_head_step_epilogue_equals_head_then_cfg_step_bitwise(fused, grid):
    """`mc_head_unpatchify_step` (CFG combine + scheduler update in the head's epilogue, SURVEY §8f-1) == `mc_head_unpatchify_ex`
    followed by `mc_cfg_step`, bit for bit, for the stream form and the cache-hit form, out of place and with the latent updated
    in place."""
    ops = _ops()
    F, Hp, Wp = grid
    D = 1536
    rows = F * Hp * Wp
    g = torch.Generator(device=DEV).manual_seed(rows + int(fused))
    head_mod = torch.randn(1, 2, D, device=DEV, generator=g) / math.sqrt(D)
    e = torch.randn(1, D, device=DEV, generator=g) * 0.3
    wt = (torch.randn(D, 64, device=DEV, generator=g) * 0.05).contiguous()
    b = torch.randn(64, device=DEV, generator=g) * 0.1
    if fused:
        x = torch.randn(rows, D, device=DEV, generator=g).bfloat16()
        kw = dict(residual=torch.randn(rows, D, device=DEV, generator=g) * 0.3)
    else:
        x = torch.randn(rows, D, device=DEV, generator=g) * 2
        kw = {}
    cond = torch.randn(16, F, 2 * Hp, 2 * Wp, device=DEV, generator=g)
    lat = torch.randn(16, F, 2 * Hp, 2 * Wp, device=DEV, generator=g)
    gs, cx, cv = 5.0, 1.0, -0.0371
    uncond = ops.head_unpatchify(x, head_mod, e, wt, b, grid, **kw)
    want = ops.cfg_step(cond, uncond, gs, lat, cv, coef_x=cx)
    got = ops.head_unpatchify(x, head_mod, e, wt, b, grid, step=(cond, lat, gs, cx, cv), **kw)
    assert torch.equal(got, want)
    lat2 = lat.clone()
    got2 = ops.head_unpatchify(x, head_mod, e, wt, b, grid, step=(cond, lat2, gs, 0.9, cv), out=lat2, **kw)
    assert got2.data_ptr() == lat2.data_ptr()
    assert torch.equal(lat2, ops.cfg_step(cond, uncond, gs, lat, cv, coef_x=0.9))


def test_linear_f32_small_and_time_path():
    ops = _ops()
    t = torch.tensor([999.0, 417.25], device=DEV)
    sin = ops.time_sinusoid(t, 256)
    half = 128
    pos = t.double()
    s = torch.outer(pos, torch.pow(10000, -torch.arange(half, device=DEV).double().div(half)))
    ref = torch.cat([s.cos(), s.sin()], 1).float()
    assert torch.allclose(sin, ref, rtol=0, atol=2e-7)
    w = torch.randn(1536, 256, device=DEV) * 0.02
    b = torch.randn(1536, device=DEV) * 0.1
    y = ops.linear_f32_small(sin, w, b, act=2)
    assert torch.allclose(y, torch.nn.functional.silu(sin @ w.t() + b), rtol=1e-3, atol=1e-4)
    w2 = torch.randn(9216, 1536, device=DEV) * 0.02
    y2 = ops.linear_f32_small(y, w2, None, act=1)
    assert torch.allclose(y2, torch.nn.functional.silu(y) @ w2.t(), rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("rows_grid,D", [((1, 1, 1), 256), ((2, 3, 5), 384), ((3, 16, 24), 1536), ((5, 30, 52), 1536)])
@pytest.mark.parametrize("kind", ["plain", "offset", "outlier"])
def test_head_unpatchify_shapes_and_offsets(rows_grid, D, kind):
    """The single-pass tensor-core head (row statistics by Chan's update, 3-pass bf16 split GEMM against the modulated weight)
    against an fp64 evaluation of `Head` + unpatchify: ragged row counts (CTA row ranges and partial 128-row tiles), rows with a
    large common offset (the pilot shift) and rows with a few huge columns, both the fp32-stream and the fused cache-hit form.
    Tolerance = the north-star's rtol 1e-3 / atol 1e-4 on fp32 outputs."""
    ops = _ops()
    F, Hp, Wp = rows_grid
    rows = F * Hp * Wp
    g = torch.Generator(device=DEV).manual_seed(rows + D)
    head_mod = torch.randn(1, 2, D, device=DEV, generator=g) / math.sqrt(D)
    e = torch.randn(1, D, device=DEV, generator=g) * 0.3
    W = torch.randn(64, D, device=DEV, generator=g) * 0.05
    b = torch.randn(64, device=DEV, generator=g) * 0.1
    x = torch.randn(rows, D, device=DEV, generator=g) * 2
    if kind == "offset":
        x = x + torch.randn(rows, 1, device=DEV, generator=g) * 50.0
    if kind == "outlier":
        x[:, 0] *= 300.0
        x[:, D // 2 + 3] += 500.0
    ee = (head_mod + e.unsqueeze(1)).double()

    def ref_of(xx):
        y = torch.nn.functional.layer_norm(xx.double(), (D,), eps=1e-6) * (1 + ee[0, 1]) + ee[0, 0]
        y = y @ W.double().t() + b.double()
        return torch.einsum("fhwpqrc->cfphqwr", y.float().view(F, Hp, Wp, 1, 2, 2, 16)).reshape(16, F, Hp * 2, Wp * 2)

    out = ops.head_unpatchify(x, head_mod, e, W.t().contiguous(), b, rows_grid)
    ref = ref_of(x)
    assert torch.allclose(out, ref, rtol=1e-3, atol=1e-4), (kind, float((out - ref).abs().max()), float(ref.abs().max()))
    x0 = x.bfloat16()
    r = torch.randn(rows, D, device=DEV, generator=g) * 0.3
    out_h = ops.head_unpatchify(x0, head_mod, e, W.t().contiguous(), b, rows_grid, residual=r)
    ref_h = ref_of(x0.float() + r)
    assert torch.allclose(out_h, ref_h, rtol=1e-3, atol=1e-4), (kind, float((out_h - ref_h).abs().max()))
    # the fused hit equals add-then-head bit for bit (same fp32 sum, same pipeline)
    assert torch.equal(out_h, ops.head_unpatchify(ops.cache_hit_add(x0, r), head_mod, e, W.t().contiguous(), b, rows_grid))
    # TeaCache form: sum rounded to bf16 first
    out_t = ops.head_unpatchify(x0, head_mod, e, W.t().contiguous(), b, rows_grid, residual=r, round_sum_to_bf16=True)
    ref_t = ref_of((x0.float() + r).bfloat16().float())
    assert torch.allclose(out_t, ref_t, rtol=1e-3, atol=1e-4)


def test_head_unpatchify_token_range():
    """Token-sharded call: rows [row_offset, row_offset + n) of the grid written into a caller-provided output, other positions
    untouched."""
    ops = _ops()
    F, Hp, Wp, D = 3, 8, 12, 384
    rows = F * Hp * Wp
    g = torch.Generator(device=DEV).manual_seed(7)
    head_mod = torch.randn(1, 2, D, device=DEV, generator=g) / math.sqrt(D)
    e = torch.randn(1, D, device=DEV, generator=g) * 0.3
    Wt = (torch.randn(64, D, device=DEV, generator=g) * 0.05).t().contiguous()
    b = torch.randn(64, device=DEV, generator=g) * 0.1
    x = torch.randn(rows, D, device=DEV, generator=g)
    full = ops.head_unpatchify(x, head_mod, e, Wt, b, (F, Hp, Wp))
    out = torch.full_like(full, 777.0)
    lo, hi = 100, 233
    ops.head_unpatchify(x[lo:hi].contiguous(), head_mod, e, Wt, b, (F, Hp, Wp), row_offset=lo, out=out)
    tok = torch.zeros(rows, dtype=torch.bool, device=DEV)
    tok[lo:hi] = True
    mask = tok.view(F, Hp, Wp)[:, :, None, :, None].expand(F, Hp, 2, Wp, 2).reshape(F, Hp * 2, Wp * 2)[None].expand(16, -1, -1, -1)
    assert torch.equal(out[mask], full[mask])
    assert bool((out[~mask] == 777.0).all())


@pytest.mark.parametrize("fused", [False, True])
def test_head_unpatchify(fused):
    ops = _ops()
    F, Hp, Wp, D = 3, 5, 7, 1536
    rows = F * Hp * Wp
    head_mod = torch.randn(1, 2, D, device=DEV) / math.sqrt(D)
    e = torch.randn(1, D, device=DEV) * 0.3
    W = torch.randn(64, D, device=DEV) * 0.05
    b = torch.randn(64, device=DEV) * 0.1
    if fused:
        x0 = torch.randn(rows, D, device=DEV).bfloat16()
        r = torch.randn(rows, D, device=DEV) * 0.3
        x = x0 + r
        out = ops.head_unpatchify(x0, head_mod, e, W.t().contiguous(), b, (F, Hp, Wp), residual=r)
    else:
        x = torch.randn(rows, D, device=DEV) * 2
        out = ops.head_unpatchify(x, head_mod, e, W.t().contiguous(), b, (F, Hp, Wp))
    ee = head_mod + e.unsqueeze(1)
    y = (torch.nn.functional.layer_norm(x, (D,), eps=1e-6) * (1 + ee[0, 1]) + ee[0, 0]).double() @ W.double().t() + b.double()
    ref = torch.einsum("fhwpqrc->cfphqwr", y.float().view(F, Hp, Wp, 1, 2, 2, 16)).reshape(16, F, Hp * 2, Wp * 2)
    assert out.shape == ref.shape
    assert torch.allclose(out, ref, rtol=1e-3, atol=1e-4), float((out - ref).abs().max())


# ------------------------------------------------------------------------------------------- wgmma GEMM
def _gemm_ref(a, b):
    return a.double() @ b.double().t()


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 128, 256), (256, 384, 1536), (300, 200, 512), (1000, 1536, 1536), (517, 8960, 1536),
                                    (777, 1536, 8960), (64, 64, 64), (512, 1536, 4096), (333, 1536, 64),
                                    (4095, 1536, 1536)])  # a token-sharded rank's o-projection: 192 wide tiles / 384 narrow ones
@pytest.mark.parametrize("bn", [0, 128, 256])  # 0: the launcher's choice by wave count; else the N-tile width forced (MC_GEMM_BN)
def test_gemm_bias_bf16(M, N, K, bn, monkeypatch):
    ops, L = _ops(), _lib()
    if bn:
        monkeypatch.setenv("MC_GEMM_BN", str(bn))
    a = torch.randn(M, K, device=DEV).bfloat16()
    b = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=DEV).bfloat16().float()
    out = ops.gemm(a, b, bias, L.MC_EPI_BIAS_BF16)
    ref = (_gemm_ref(a, b) + bias.double()).float()
    nbad, maxerr = bf16_ulp_close(out, ref)
    assert nbad == 0, (nbad, maxerr)
    # fp32 epilogue: the accumulator itself at rtol 1e-3 / atol 1e-4
    out32 = ops.gemm(a, b, bias, L.MC_EPI_BIAS_F32)
    assert torch.allclose(out32, ref, rtol=1e-3, atol=1e-4), float((out32 - ref).abs().max())


@pytest.mark.parametrize("bn", [128, 256])
def test_gemm_epilogues(bn, monkeypatch):
    ops, L = _ops(), _lib()
    monkeypatch.setenv("MC_GEMM_BN", str(bn))
    M, N, K = 391, 640, 1536
    a = torch.randn(M, K, device=DEV).bfloat16()
    b = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=DEV).bfloat16().float()
    acc = (_gemm_ref(a, b) + bias.double()).float()
    # GELU(tanh) on the bf16-rounded Linear output
    out = ops.gemm(a, b, bias, L.MC_EPI_BIAS_GELU_BF16)
    ref = torch.nn.functional.gelu(acc.bfloat16().float(), approximate="tanh")
    # a 1-ulp flip of the bf16 pre-activation (2^-8 relative to |acc|) moves GELU by at most that much (|GELU'| <= 1.13)
    tol = ref.abs() * 2.0 ** -7 + acc.abs() * 2.0 ** -7 + 1e-3
    assert ((out.float() - ref).abs() <= tol).all(), float((out.float() - ref).abs().max())
    # exact (erf) GELU of the i2v `img_emb` MLP, same bf16 pre-activation rule
    out = ops.gemm(a, b, bias, L.MC_EPI_BIAS_GELU_ERF_BF16)
    ref = torch.nn.functional.gelu(acc.bfloat16().float())
    assert ((out.float() - ref).abs() <= tol).all(), float((out.float() - ref).abs().max())
    # 257 CLIP tokens x K = 1280: ragged M and N, K not a multiple of the 64-wide K block count the block GEMMs use
    a2 = torch.randn(257, 1280, device=DEV).bfloat16()
    b2 = (torch.randn(1280, 1280, device=DEV) / math.sqrt(1280)).bfloat16()
    out2 = ops.gemm(a2, b2, None, L.MC_EPI_BIAS_GELU_ERF_BF16)
    acc2 = _gemm_ref(a2, b2).float()
    ref2 = torch.nn.functional.gelu(acc2.bfloat16().float())
    assert ((out2.float() - ref2).abs() <= ref2.abs() * 2.0 ** -7 + acc2.abs() * 2.0 ** -7 + 1e-3).all()
    # gated residual, fp32 stream updated in place
    x = torch.randn(M, N, device=DEV)
    gate = torch.randn(N, device=DEV) * 0.5
    x_ref = x + acc.bfloat16().float() * gate
    ops.gemm(a, b, bias, L.MC_EPI_BIAS_GATE_RESID, out=x, gate=gate)
    assert ((x - x_ref).abs() <= 1e-4 + gate.abs() * acc.abs() * 2 ** -7).all()
    x2 = torch.randn(M, N, device=DEV)
    x2_ref = x2 + acc.bfloat16().float()
    ops.gemm(a, b, bias, L.MC_EPI_BIAS_GATE_RESID, out=x2, gate=None)
    assert ((x2 - x2_ref).abs() <= 1e-4 + acc.abs() * 2 ** -7).all()
    # row bias (V^T = Wv h^T + bv): A = weight [N, K], B = activations [M, K], padded leading dimension
    rb = torch.randn(N, device=DEV).bfloat16().float()
    buf = torch.zeros(N, M + 9, dtype=torch.bfloat16, device=DEV)
    vt = ops.gemm(b, a, rb, L.MC_EPI_ROWBIAS_BF16, out=buf[:, :M])
    ref_t = (_gemm_ref(b, a) + rb.double()[:, None]).float()
    nbad, maxerr = bf16_ulp_close(vt, ref_t)
    assert nbad == 0, (nbad, maxerr)
    assert float(buf[:, M:].abs().max()) == 0.0  # nothing written past N columns


def test_gemm_strided_operands():
    ops, L = _ops(), _lib()
    big = torch.randn(300, 2 * 512, device=DEV).bfloat16()
    a = big[:, 512:]
    b = (torch.randn(256, 512, device=DEV) / 22).bfloat16()
    out = ops.gemm(a, b, None, L.MC_EPI_BIAS_F32)
    assert torch.allclose(out, _gemm_ref(a, b).float(), rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("rows,D", [(7, 256), (333, 384), (1000, 1536), (515, 2048), (1031, 1536), (3001, 384)])
def test_rmsnorm_rope_two_blocks_one_launch(rows, D):
    """q | k of the fused q|k|v buffer normalised (+ RoPE) by ONE launch over two column blocks == two single-block launches, bit
    for bit (same per-row arithmetic), on a row-strided view; the v block is untouched."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(rows)
    qkv = torch.randn(rows, 3 * D, device=DEV, generator=g).bfloat16()
    w = 1 + 0.1 * torch.randn(2, D, device=DEV, generator=g)
    cs = torch.randn(rows, 128, device=DEV, generator=g)
    a, b = qkv.clone(), qkv.clone()
    ops.rmsnorm_rope_segs_(a, w, 2, cs, 128)
    ops.rmsnorm_rope_(b[:, :D], w[0], cs, 128)
    ops.rmsnorm_rope_(b[:, D:2 * D], w[1], cs, 128)
    assert torch.equal(a, b)
    assert torch.equal(a[:, 2 * D:], qkv[:, 2 * D:])
    assert not torch.equal(a[:, :2 * D], qkv[:, :2 * D])


def test_rmsnorm_rope_staged_form_matches_register_form_bitwise():
    """The TMA-staged kernels (>= 1024 items) and the register-pipelined ones (fewer) run the same per-row arithmetic: the first
    1000 rows of a long input, processed alone, must come out bit-identical; likewise LayerNorm + modulation (mode 0) and the
    affine LayerNorm (mode 1), from fp32 and from bf16 input with the LN value rounded to bf16, into bf16 and into fp32. The widths
    D = 256 / 1024 / 1536 / 2048 cover every per-lane group count G = 2 / 4 / 6 / 8 of both kernels."""
    ops = _ops()
    for D in (256, 1024, 1536, 2048):
        g = torch.Generator(device=DEV).manual_seed(3 + D)
        qkv = torch.randn(2500, 3 * D, device=DEV, generator=g).bfloat16()
        w = 1 + 0.1 * torch.randn(2, D, device=DEV, generator=g)
        cs = torch.randn(2500, 128, device=DEV, generator=g)
        a, b = qkv.clone(), qkv[:500].clone()
        ops.rmsnorm_rope_segs_(a, w, 2, cs, 128)         # 5000 items: staged
        ops.rmsnorm_rope_segs_(b, w, 2, cs[:500], 128)   # 1000 items: register form
        assert torch.equal(a[:500], b), D
        x = torch.randn(2500, D, device=DEV, generator=g) * 2 + 0.3
        em = torch.randn(6, D, device=DEV, generator=g) * 0.2
        ya = ops.ln_modulate(x, em, 4, 3)
        yb = ops.ln_modulate(x[:1000], em, 4, 3)
        assert torch.equal(ya[:1000], yb), D
        xh = x.bfloat16()
        for out_dtype in (torch.bfloat16, torch.float32):
            ya = ops.ln_modulate(xh, em, 1, 0, round_ln_to_bf16=True, out_dtype=out_dtype)
            yb = ops.ln_modulate(xh[:1000], em, 1, 0, round_ln_to_bf16=True, out_dtype=out_dtype)
            assert ya.dtype == out_dtype and torch.equal(ya[:1000], yb), (D, out_dtype)
            for xi in (x, xh):
                ya = ops.ln_affine(xi, em[0], em[5], out_dtype=out_dtype)
                yb = ops.ln_affine(xi[:1000], em[0], em[5], out_dtype=out_dtype)
                assert torch.equal(ya[:1000], yb), (D, out_dtype, xi.dtype)


# ------------------------------------------------------------------------------------------- wgmma attention
def _attn_ref(q, k, v, heads):
    Lq, W = q.shape
    qh = q.double().view(Lq, heads, 128).transpose(0, 1)
    kh = k.double().view(-1, heads, 128).transpose(0, 1)
    vh = v.double().view(-1, heads, 128).transpose(0, 1)
    s = qh @ kh.transpose(1, 2) / math.sqrt(128)
    return (torch.softmax(s, -1) @ vh).transpose(0, 1).reshape(Lq, W).float()


@pytest.mark.parametrize("Lq,Lk,heads,qscale", [(128, 64, 1, 1.0), (128, 128, 1, 1.0), (256, 512, 2, 1.0), (300, 1000, 3, 1.0), (1000, 4095, 12, 1.0),
                                                (200, 777, 2, 6.0), (130, 512, 12, 1.0),
                                                (11, 11, 24, 1.0), (300, 65, 3, 1.0)])  # HunyuanVideo token refiner: Lk < 64 and Lq < 128
def test_attention(Lq, Lk, heads, qscale):
    ops = _ops()
    W = heads * 128
    q = (torch.randn(Lq, W, device=DEV) * qscale).bfloat16()
    k = torch.randn(Lk, W, device=DEV).bfloat16()
    v = torch.randn(Lk, W, device=DEV).bfloat16()
    out = ops.attention(q, k, v, heads)
    ref = _attn_ref(q, k, v, heads)
    # P is rounded to bf16 before the PV product (as in flash-attention): error ~ 2^-9 * sqrt(sum p^2) relative to |v|~1,
    # plus the bf16 rounding of the output.
    err = (out.float() - ref).abs()
    assert float(err.max()) < 2e-2, float(err.max())
    assert float(err.mean()) < 2e-3, float(err.mean())


@pytest.mark.parametrize("emu", [0, 2, 3, 4])
@pytest.mark.parametrize("Lq,Lk,heads,qscale", [(128, 128, 1, 1.0), (256, 256, 1, 1.0), (300, 1000, 3, 1.0), (513, 1285, 2, 6.0), (1000, 4095, 12, 1.0),
                                                (40, 130, 1, 3.0)])
def test_attention_long_kernel(Lq, Lk, heads, qscale, emu, monkeypatch):
    """The 128-wide-KV instantiation forced onto small and ragged shapes (second consumer warpgroup's rows empty or partial, one KV
    tile, ragged last KV tile), for every exponential-emulation fraction it is built with: same bounds as the default path, and each
    variant bit-reproducible."""
    ops = _ops()
    monkeypatch.setenv("MC_ATTN_KERNEL", "2")
    monkeypatch.setenv("MC_ATTN_EMU", str(emu))
    W = heads * 128
    q = (torch.randn(Lq, W, device=DEV) * qscale).bfloat16()
    k = torch.randn(Lk, W, device=DEV).bfloat16()
    v = torch.randn(Lk, W, device=DEV).bfloat16()
    out = ops.attention(q, k, v, heads)
    ref = _attn_ref(q, k, v, heads)
    err = (out.float() - ref).abs()
    assert float(err.max()) < 2e-2, float(err.max())
    assert float(err.mean()) < 2e-3, float(err.mean())
    assert torch.equal(out, ops.attention(q, k, v, heads))


def test_attention_strided_qkv_views_and_rotation(monkeypatch):
    """q, k, v as column slices of one fused [L, 3W] buffer (row pitch 3W), and the rotated key order of the token-sharded form
    (`first_key_row`): softmax is permutation invariant over keys, so the result matches the unrotated one to rounding."""
    ops = _ops()
    L, heads = 1500, 3
    W = heads * 128
    qkv = torch.randn(L, 3 * W, device=DEV).bfloat16()
    q, k, v = qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:]
    ref = _attn_ref(q.contiguous(), k.contiguous(), v.contiguous(), heads)
    out = ops.attention(q, k, v, heads)
    assert float((out.float() - ref).abs().max()) < 2e-2
    for first in (0, 127, 128, 700, 1499):
        rot = ops.attention(q, k, v, heads, first_key_row=first)
        assert float((rot.float() - ref).abs().max()) < 2e-2, first
        assert float((rot.float() - out.float()).abs().mean()) < 1e-3, first
    monkeypatch.setenv("MC_ATTN_SPLITS", "3")
    rot = ops.attention(q, k, v, heads, first_key_row=700)
    assert float((rot.float() - ref).abs().max()) < 2e-2


def test_attention_matches_sdpa_bf16_noise_level():
    """Our error against the fp64 reference must be no worse than 2x torch SDPA's bf16 error on the same inputs."""
    ops = _ops()
    Lq, Lk, heads = 512, 2048, 4
    W = heads * 128
    q, k, v = (torch.randn(n, W, device=DEV).bfloat16() for n in (Lq, Lk, Lk))
    out = ops.attention(q, k, v, heads)
    ref = _attn_ref(q, k, v, heads)
    sd = torch.nn.functional.scaled_dot_product_attention(q.view(Lq, heads, 128).transpose(0, 1)[None], k.view(Lk, heads, 128).transpose(0, 1)[None],
                                                          v.view(Lk, heads, 128).transpose(0, 1)[None])[0].transpose(0, 1).reshape(Lq, W)
    e_ours = (out.float() - ref).pow(2).mean().sqrt().item()
    e_sdpa = (sd.float() - ref).pow(2).mean().sqrt().item()
    assert e_ours <= 2.0 * e_sdpa + 1e-4, (e_ours, e_sdpa)


@pytest.mark.parametrize("Lq,Lk,heads,splits", [(1000, 4095, 12, 0), (300, 2000, 2, 3), (129, 1100, 1, 2), (512, 4100, 4, 8), (256, 700, 2, 5)])
def test_attention_split_kv(Lq, Lk, heads, splits, monkeypatch):
    """Split-KV path (small grids, e.g. the per-rank shape of an 8-way token shard): every split normalises its own partial
    softmax and a second kernel merges them. Checked against the fp64 reference, against the unsplit kernel, and for
    reproducibility; ragged cases where the last split has fewer KV tiles (and a partial tile)."""
    ops = _ops()
    W = heads * 128
    q = (torch.randn(Lq, W, device=DEV) * 3.0).bfloat16()
    k = torch.randn(Lk, W, device=DEV).bfloat16()
    v = torch.randn(Lk, W, device=DEV).bfloat16()
    monkeypatch.setenv("MC_ATTN_SPLITS", "1")
    one = ops.attention(q, k, v, heads).clone()
    if splits:
        monkeypatch.setenv("MC_ATTN_SPLITS", str(splits))
    else:
        monkeypatch.delenv("MC_ATTN_SPLITS")
    outs = [ops.attention(q, k, v, heads).clone() for _ in range(3)]
    ref = _attn_ref(q, k, v, heads)
    err = (outs[0].float() - ref).abs()
    assert float(err.max()) < 2e-2 and float(err.mean()) < 2e-3, (float(err.max()), float(err.mean()))
    # P is rounded to bf16 relative to each CTA's own running max, so split and unsplit results differ at the level of that
    # rounding (not just by the output's bf16 ulp): the split result must be as close to the fp64 reference as the unsplit one
    err_one = (one.float() - ref).abs()
    assert float(err.mean()) <= 1.25 * float(err_one.mean()) + 1e-5, (float(err.mean()), float(err_one.mean()))
    assert float(err.max()) <= 2.0 * float(err_one.max()) + 1e-3, (float(err.max()), float(err_one.max()))
    assert float((outs[0].float() - one.float()).abs().max()) < 2e-2
    assert all(torch.equal(outs[0], o) for o in outs[1:])


@pytest.mark.parametrize("Lq,Lk,heads,qscale", [(4096, 512, 12, 1.0), (2048, 4096, 4, 5.0), (1000, 777, 3, 8.0)])
def test_attention_is_bit_reproducible(Lq, Lk, heads, qscale):
    """Same inputs -> same bits, including short KV sequences (cross-attention shape) and score ranges that force the
    accumulator to be rescaled many times. (A missing ordering between the softmax warps and the PV MMA showed up exactly
    here in round 1: tools/diag_determinism.py.)"""
    ops = _ops()
    W = heads * 128
    q = (torch.randn(Lq, W, device=DEV) * qscale).bfloat16()
    k = torch.randn(Lk, W, device=DEV).bfloat16()
    v = torch.randn(Lk, W, device=DEV).bfloat16()
    outs = [ops.attention(q, k, v, heads).clone() for _ in range(4)]
    assert torch.isfinite(outs[0].float()).all()
    for o in outs[1:]:
        assert torch.equal(outs[0], o)
