"""The hand-written kernels at the edge shapes the engines launch, with poisoned input margins and fenced outputs.

Every operand here is a view into a larger allocation (`fenced`). Input margins hold NaN, so a kernel that reads past a view where
the bytes feed a stored result writes NaN; output margins hold a fixed byte pattern that `check_fence` compares bit for bit after
the call, so a store past a row or past a tensor fails the test instead of landing in allocator slack. The shapes are the ragged
tiles, the wholly out-of-range half tiles, the idle warps and the unaligned tails: K not a multiple of 64 and N = 32 in the GEMM
(Open-Sora's x_embedder and final layer), an 11-key attention (HunyuanVideo's token refiner), key views of longer buffers,
segments of 1 / 63 / 64 / 65 rows, and the like. The staged row kernels, whose copy sizes are worked out at run time, are
here too: LayerNorm + modulation (K7) and RMSNorm + RoPE (K9) either side of the 1024-row switch to the staging ring, with a
ragged last stage, at every per-lane group count and the wide forms, and the residual statistics (K3) with a ragged last chunk
of 4 rows and the fused residual output fenced. Results are compared with fp64 statements of each kernel's rounding chain, at
the criteria of test_kernels_gpu.py and test_opensora_gpu.py; where a result is exact (one key, a 30-logit peak, the
elementwise kernels) it is compared bit for bit.

Only `test_fence_check_catches_a_write_past_each_edge` runs without a GPU; this module imports without initialising CUDA.
"""
import math

import pytest
import torch
import torch.nn.functional as F

DEV = "cuda"
FENCE_BYTE = 0xA5  # output margins: every byte; decodes to a finite bf16 / fp32 value, so only a bit compare sees a stray store
NAN_FP8 = 0x7F     # float8_e4m3fn NaN
BF, F32 = torch.bfloat16, torch.float32


def _ops():
    from magcache_b200 import ops
    return ops


def _lib():
    from magcache_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------- fences
def fenced(shape, dtype, margin=(0, 0, 0, 0), fill="nan", device=DEV, pitch=None):
    """A `shape` view inside a larger buffer; returns (view, buf). `margin` = (rows_before, rows_after, cols_left, cols_right)
    elements around the view (a 1-D shape has only the column margins). The view's contents are left to the caller.

    fill="nan": the whole buffer is NaN (float8_e4m3fn: code 0x7F), poison for inputs. Poison only catches a stray read where
    that read would change a stored output: columns past K of a GEMM operand, key rows past Lk or past a segment, columns past a
    head slice. Rows past M of a GEMM's A, or query rows past a segment, are never combined into a stored row, so NaN there
    catches nothing and no test relies on it.
    fill="fence": every byte is 0xA5, for outputs and in-place operands; `check_fence(view, buf)` after the call.

    The view's first element is 16-byte aligned (cols_left * itemsize is a multiple of 16 on a fresh allocation) and the row
    pitch is the smallest multiple of 8 elements that holds both margins, unless `pitch` is given (an odd ldo)."""
    esize = torch.empty(0, dtype=dtype).element_size()
    rb, ra, cl, cr = margin
    assert (cl * esize) % 16 == 0, "the view must start 16-byte aligned"
    if len(shape) == 1:
        assert rb == ra == 0 and pitch is None
        buf = torch.empty(cl + shape[0] + cr, dtype=dtype, device=device)
    else:
        rows, cols = shape
        if pitch is None:
            pitch = -(-(cl + cols + cr) // 8) * 8
        assert pitch >= cl + cols + cr
        buf = torch.empty(rb + rows + ra, pitch, dtype=dtype, device=device)
    if fill == "fence":
        buf.view(torch.uint8).fill_(FENCE_BYTE)
    elif fill == "nan":
        if dtype == torch.float8_e4m3fn:
            buf.view(torch.uint8).fill_(NAN_FP8)
        else:
            buf.fill_(float("nan"))
    else:
        raise ValueError(fill)
    view = buf[cl:cl + shape[0]] if len(shape) == 1 else buf[rb:rb + shape[0], cl:cl + shape[1]]
    assert view.data_ptr() % 16 == 0, "the view must start 16-byte aligned"
    return view, buf


def _fill_bytes_ok(t):
    """Elementwise: does the (contiguous) tensor still hold the fence pattern in every byte?"""
    raw = t.contiguous().view(torch.uint8).view(*t.shape, t.element_size())
    return (raw == FENCE_BYTE).all(-1)


def check_fence(view, buf):
    """Every element of `buf` outside `view` must still hold the fence pattern, bit for bit. A 1-D buffer may hold a
    contiguous view of any shape."""
    off = view.storage_offset() - buf.storage_offset()
    outside = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    if buf.dim() == 1:
        assert view.is_contiguous()
        outside[off:off + view.numel()] = False
    else:
        r0, c0 = divmod(off, buf.stride(0))
        outside[r0:r0 + view.shape[0], c0:c0 + view.shape[1]] = False
    bad = outside & ~_fill_bytes_ok(buf)
    n = int(bad.sum())
    if n:
        raise AssertionError(f"{n} fence elements overwritten, the first at buffer index {bad.nonzero()[0].tolist()} (view at offset {off})")


def test_fence_check_catches_a_write_past_each_edge():
    """The fence checker itself (CPU): untouched margins pass whatever the view holds; one element written just past the view
    above, below, left or right of it fails, for bf16, fp32 and a 1-D buffer; the fp8 poison decodes to NaN."""
    for dtype in (BF, F32):
        view, buf = fenced((5, 9), dtype, (2, 2, 8, 8), fill="fence", device="cpu")
        view.fill_(1.0)
        check_fence(view, buf)
        for r, c in ((-1, 0), (5, 8), (0, -1), (4, 9)):
            view, buf = fenced((5, 9), dtype, (2, 2, 8, 8), fill="fence", device="cpu")
            buf[2 + r, 8 + c] = 0.0
            with pytest.raises(AssertionError):
                check_fence(view, buf)
    for i in (3, 4 + 7):
        view, buf = fenced((7,), F32, (0, 0, 4, 4), fill="fence", device="cpu")
        view.fill_(0.0)
        buf[i] = 1.0
        with pytest.raises(AssertionError):
            check_fence(view, buf)
    view, buf = fenced((16,), torch.float8_e4m3fn, (0, 0, 16, 16), device="cpu")
    assert bool(buf.float().isnan().all())
    vv, bb = fenced((3, 8), BF, (0, 0, 8, 8), device="cpu")
    assert bool(bb.isnan().all()) and bb.stride(0) == 24


def _rb(t):
    """fp64 -> nearest bf16 (through fp32), kept in fp64."""
    return t.float().bfloat16().double()


def _randn(shape, g, scale=1.0):
    return torch.randn(*shape, device=DEV, generator=g) * scale


# ------------------------------------------------------------------------------------------- GEMM
_EPIS = ["MC_EPI_BIAS_BF16", "MC_EPI_BIAS_GELU_BF16", "MC_EPI_BIAS_GATE_RESID", "MC_EPI_ROWBIAS_BF16", "MC_EPI_BIAS_F32",
         "MC_EPI_BIAS_GELU_ERF_BF16", "MC_EPI_BIAS_GATE_RESID_BF16", "MC_EPI_BIAS_SILU_BF16"]
_F32_OUT = ("MC_EPI_BIAS_GATE_RESID", "MC_EPI_BIAS_F32")


def _gemm_case(epi, M, N, K, g, odd_ldo=False):
    """One fenced `mc_gemm_bf16` launch against fp64: A / B with NaN columns past K (and left of it), bias and gate with NaN on
    both sides, the output a window at column 8 of a wider fenced buffer (ldo > N; odd when asked)."""
    ops, L = _ops(), _lib()
    e = getattr(L, epi)
    a, _ = fenced((M, K), BF, (0, 1, 8, 8))
    a.copy_(_randn((M, K), g))
    b, _ = fenced((N, K), BF, (0, 1, 8, 8))
    b.copy_(_randn((N, K), g, 1.0 / math.sqrt(K)))
    rowbias = epi == "MC_EPI_ROWBIAS_BF16"
    bias, _ = fenced((M if rowbias else N,), F32, (0, 0, 4, 4))
    bias.copy_(_randn(bias.shape, g).bfloat16().float())
    gate = None
    if "GATE" in epi:
        gate, _ = fenced((N,), F32, (0, 0, 4, 4))
        gate.copy_(_randn((N,), g, 0.5))
    odt = F32 if epi in _F32_OUT else BF
    if odd_ldo:
        pitch = 8 + N + 8 + 1 - (N % 2)
        out, obuf = fenced((M, N), odt, (8, 2, 8, 8), fill="fence", pitch=pitch)
        assert out.stride(0) % 2 == 1
    else:
        out, obuf = fenced((M, N), odt, (2, 2, 8, 8), fill="fence")
    old = _randn((M, N), g).to(odt)
    out.copy_(old)

    ops.gemm(a, b, bias, e, out=out, gate=gate)
    check_fence(out, obuf)
    got = out.double()
    assert bool(torch.isfinite(got).all()), (epi, M, N, K)
    acc = a.double() @ b.double().t()
    pre = acc + (bias.double()[:, None] if rowbias else bias.double())
    assert bool(gemm_fp64_bounds_ok(epi, got, pre, old.double(), None if gate is None else gate.double()).all()), (epi, M, N, K, odd_ldo)


def gemm_fp64_bounds_ok(epi, got, pre, old=None, gate=None):
    """Elementwise: is an `mc_gemm_bf16` output `got` within this module's bound of the fp64 pre-activation pre = acc + bias
    (`old`: the output's contents before an in-place epilogue; `gate` broadcast over the rows)? All fp64 tensors."""
    if epi in ("MC_EPI_BIAS_BF16", "MC_EPI_ROWBIAS_BF16"):
        # bf16_ulp_close of test_kernels_gpu: one bf16 ulp of an fp32 value with rtol 1e-3 / atol 1e-4 noise
        return (got - pre).abs() <= pre.abs() * 2.0 ** -7 + 1e-4
    if epi == "MC_EPI_BIAS_F32":  # torch.allclose(got, pre, rtol=1e-3, atol=1e-4)
        return (got - pre).abs() <= 1e-4 + 1e-3 * pre.abs()
    if epi in ("MC_EPI_BIAS_GELU_BF16", "MC_EPI_BIAS_GELU_ERF_BF16", "MC_EPI_BIAS_SILU_BF16"):
        y = _rb(pre)  # the Linear output is bf16 before the activation sees it
        if epi == "MC_EPI_BIAS_GELU_BF16":
            ref = F.gelu(y, approximate="tanh")
        elif epi == "MC_EPI_BIAS_GELU_ERF_BF16":
            ref = F.gelu(y)
        else:
            ref = y * torch.sigmoid(y)
        # a 1-ulp flip of the bf16 pre-activation moves the activation by at most that much (|GELU'|, |SiLU'| <= 1.13)
        return (got - ref).abs() <= ref.abs() * 2.0 ** -7 + pre.abs() * 2.0 ** -7 + 1e-3
    if epi == "MC_EPI_BIAS_GATE_RESID":
        ref = old + _rb(pre) * gate
        return (got - ref).abs() <= 1e-4 + gate.abs() * pre.abs() * 2.0 ** -7
    # MC_EPI_BIAS_GATE_RESID_BF16: bf16(old + bf16(g * bf16(acc + b)))
    gy = gate * _rb(pre)
    ref = _rb(old + _rb(gy))
    # one flip of bf16(acc + b) (<= 2^-7 |g y|), propagated, plus one of bf16(g y) (<= 2^-7 |g y|), plus one of the final rounding
    return (got - ref).abs() <= ref.abs() * 2.0 ** -7 + gy.abs() * 2.0 ** -6 + 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("epi", _EPIS)
def test_gemm_edge_shapes_fenced(epi, bn, monkeypatch):
    """Every epilogue at K in {8, 16, 72, 144, 200, 1000} (the K tail rests on TMA's zero fill, past NaN columns), N in
    {1, 7, 32, 33, 65} (N = 32: the second CTA's B half tile lies wholly past N at BN 128) and M in {1, 129, 257}, both tile widths;
    the bf16 epilogues once more with an odd ldo (scalar stores)."""
    monkeypatch.setenv("MC_GEMM_BN", str(bn))
    g = torch.Generator(device=DEV).manual_seed(_EPIS.index(epi) * 2 + bn)
    for K in (8, 16, 72, 144, 200, 1000):
        for N in (1, 7, 32, 33, 65):
            for M in (1, 129, 257):
                _gemm_case(epi, M, N, K, g)
    if epi not in _F32_OUT:
        for M, N, K in ((129, 65, 72), (257, 33, 144), (1, 32, 16), (300, 200, 512)):
            _gemm_case(epi, M, N, K, g, odd_ldo=True)


# ------------------------------------------------------------------------------------------- head_dim-128 attention
def _attn64(q, k, v, heads, scale, hd=128):
    Lq = q.shape[0]
    qh = q.double().reshape(Lq, heads, hd).transpose(0, 1)
    kh = k.double().reshape(-1, heads, hd).transpose(0, 1)
    vh = v.double().reshape(-1, heads, hd).transpose(0, 1)
    return (torch.softmax(qh @ kh.transpose(1, 2) * scale, -1) @ vh).transpose(0, 1).reshape(Lq, heads * hd)


def _attn_operands(Lq, Lk, heads, g, peak=None, scale=None, hd=128):
    """Fenced q [Lq, W] (NaN columns either side), k / v as [:Lk] views of buffers whose next 128 rows are NaN. With `peak` =
    key index, every query row's scaled logit for that key lies ~40 above all others (q rows near one direction u per head, the
    peak key along u, the other keys short)."""
    W = heads * hd
    q, _ = fenced((Lq, W), BF, (0, 0, 8, 8))
    k, _ = fenced((Lk, W), BF, (0, 128, 8, 8))
    v, _ = fenced((Lk, W), BF, (0, 128, 8, 8))
    v.copy_(_randn((Lk, W), g))
    if peak is None:
        q.copy_(_randn((Lq, W), g))
        k.copy_(_randn((Lk, W), g))
    else:
        u = _randn((heads, hd), g)
        q.copy_((u[None] + _randn((Lq, heads, hd), g, 0.05)).reshape(Lq, W))
        kk = _randn((Lk, heads, hd), g, 0.05)
        kk[peak] = u * (40.0 / scale) / u.pow(2).sum(-1, keepdim=True)
        k.copy_(kk.reshape(Lk, W))
    return q, k, v


def _attn_check(Lq, Lk, heads, scale, g, peak=None):
    ops = _ops()
    W = heads * 128
    q, k, v = _attn_operands(Lq, Lk, heads, g, peak, scale)
    out, obuf = fenced((Lq, W), BF, (1, 1, 8, 8), fill="fence")
    ops.attention(q, k, v, heads, scale=scale, out=out)
    check_fence(out, obuf)
    got = out.float()
    what = (Lq, Lk, heads, scale, peak)
    assert bool(torch.isfinite(got).all()), what
    if Lk == 1:  # P = 1, l = 1: V's row, bit for bit
        assert torch.equal(out, v[0:1].expand(Lq, W)), what
    elif peak is not None:  # the peak key's V row, to the output's bf16 rounding
        vp = v[peak].float()[None]
        assert bool(((got - vp).abs() <= vp.abs() * 2.0 ** -8 + 1e-6).all()), (what, float((got - vp).abs().max()))
    else:  # test_attention's bounds
        err = (got.double() - _attn64(q, k, v, heads, scale)).abs()
        assert float(err.max()) < 2e-2 and float(err.mean()) < 2e-3, (what, float(err.max()), float(err.mean()))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [1, 24])
def test_attention_short_kernel_ragged_fenced(heads):
    """The 64-key kernel at Lk in {1, 11, 63, 64, 65, 127, 129} x Lq in {1, 64, 65, 128, 300}, scale 0.05 and 0.3, K / V as
    views with NaN rows after Lk, the output a fenced window (ldo > W); Lk = 1 is exact, and a 40-logit peak in the last full
    tile and in the ragged tile must return that key's V row."""
    g = torch.Generator(device=DEV).manual_seed(heads)
    for scale in (0.05, 0.3):
        for Lk in (1, 11, 63, 64, 65, 127, 129):
            for Lq in (1, 64, 65, 128, 300):
                _attn_check(Lq, Lk, heads, scale, g)
        for Lk, peak in ((128, 127), (128, 64), (129, 128), (127, 126), (65, 64), (11, 10)):
            _attn_check(65, Lk, heads, scale, g, peak=peak)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["forced64", "default"])
def test_attention_kernel_switch_fenced(kernel, monkeypatch):
    """`MC_ATTN_KERNEL=1` (64-key tiles at Lk 1500, a 28-key ragged tile), and the default choice either side of the switch to
    128-key tiles (Lk 1023 / 1024 / 1025): fp64 bounds and peaks in the last tile / the ragged tile."""
    if kernel == "forced64":
        monkeypatch.setenv("MC_ATTN_KERNEL", "1")
        lks = [(1500, (1499, 1472, 1471))]
    else:
        monkeypatch.delenv("MC_ATTN_KERNEL", raising=False)
        lks = [(1023, (1022, 960)), (1024, (1023, 896)), (1025, (1024, 1023))]
    g = torch.Generator(device=DEV).manual_seed(len(kernel))
    for Lk, peaks in lks:
        for scale in (0.05, 0.3):
            _attn_check(300, Lk, 2, scale, g)
            for p in peaks:
                _attn_check(130, Lk, 2, scale, g, peak=p)


@pytest.mark.gpu
def test_attention_split_kv_fenced(monkeypatch):
    """Split-KV forced (`MC_ATTN_SPLITS=3`) into a fenced output: the fence covers the combine kernel's stores too; peaks
    in the last split's ragged tile."""
    monkeypatch.setenv("MC_ATTN_SPLITS", "3")
    g = torch.Generator(device=DEV).manual_seed(3)
    for Lq, Lk, heads in ((200, 300, 3), (65, 1025, 2), (1, 129, 1), (300, 1500, 2)):
        for scale in (0.05, 0.3):
            _attn_check(Lq, Lk, heads, scale, g)
            _attn_check(Lq, Lk, heads, scale, g, peak=Lk - 1)
    _attn_check(7, 1, 1, 0.3, g)


@pytest.mark.gpu
def test_attention_rejects_a_bad_out():
    ops = _ops()
    q = torch.zeros(16, 256, dtype=BF, device=DEV)
    for bad in (torch.empty(16, 256, dtype=F32, device=DEV), torch.empty(17, 256, dtype=BF, device=DEV),
                torch.empty(16, 264, dtype=BF, device=DEV), torch.empty(256, 16, dtype=BF, device=DEV).t()):
        with pytest.raises(AssertionError):
            ops.attention(q, q, q, 2, out=bad)


# ------------------------------------------------------------------------------------------- Open-Sora kernels (head_dim 72)
def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _heads72(t, H):
    return t.reshape(t.shape[0], H, 72).transpose(0, 1)


@pytest.mark.gpu
def test_varlen_d72_segments_fenced():
    """`mc_attn_varlen_d72` over segments of 1 / 63 / 64 / 65 / 130 query rows and 1 / 63 / 64 / 65 / 300 keys in one launch
    (max_q_len 130: most segments leave q tiles idle), NaN key rows between the segments' key ranges and after the last,
    unassigned output rows between the segments (must stay bit-unchanged), scale 0.3. k_len = 1 returns V exactly, a peaked
    key in the last full / the ragged tile returns its V row; the rest within 2x SDPA's bf16 error of fp64; 3 launches agree
    bit for bit."""
    ops = _ops()
    H, scale = 3, 0.3
    W = H * 72
    g = torch.Generator(device=DEV).manual_seed(11)
    spec = [(1, 1, None), (63, 63, None), (64, 64, None), (65, 65, None), (130, 300, None), (65, 1, None), (1, 300, None),
            (63, 65, None), (1, 64, None), (64, 128, 127), (65, 129, 128), (63, 65, 64)]
    segs, qs, ks = [], 3, 0
    for ql, kl, pk in spec:
        segs.append((qs, ql, ks, kl, pk))
        qs, ks = qs + ql + 5, ks + kl + 7  # 5 unassigned query rows and 7 NaN key rows between segments
    Lq, Lk = qs, ks
    q, _ = fenced((Lq, W), BF, (0, 0, 8, 8))
    k, _ = fenced((Lk, W), BF, (0, 64, 8, 8))
    v, _ = fenced((Lk, W), BF, (0, 64, 8, 8))
    for s0, ql, k0, kl, pk in segs:
        v[k0:k0 + kl] = _randn((kl, W), g).bfloat16()
        if pk is None:
            q[s0:s0 + ql] = _randn((ql, W), g).bfloat16()
            k[k0:k0 + kl] = _randn((kl, W), g).bfloat16()
        else:
            u = _randn((H, 72), g)
            q[s0:s0 + ql] = (u[None] + _randn((ql, H, 72), g, 0.05)).reshape(ql, W).bfloat16()
            kk = _randn((kl, H, 72), g, 0.05)
            kk[pk] = u * (40.0 / scale) / u.pow(2).sum(-1, keepdim=True)
            k[k0:k0 + kl] = kk.reshape(kl, W).bfloat16()
    segs_dev = torch.tensor([s[:4] for s in segs], dtype=torch.int32, device=DEV)
    out, obuf = fenced((Lq, W), BF, (1, 1, 8, 8), fill="fence")
    ops.attention_varlen_d72(q, k, v, H, segs_dev, 130, scale=scale, out=out)
    check_fence(out, obuf)
    assigned = torch.zeros(Lq, dtype=torch.bool, device=DEV)
    for s0, ql, _, _, _ in segs:
        assigned[s0:s0 + ql] = True
    assert bool(_fill_bytes_ok(out[~assigned]).all()), "a store landed on a row that belongs to no segment"
    for s0, ql, k0, kl, pk in segs:
        o, what = out[s0:s0 + ql], (ql, kl, pk)
        assert bool(torch.isfinite(o.float()).all()), what
        if kl == 1:
            assert torch.equal(o, v[k0:k0 + 1].expand(ql, W)), what
            continue
        if pk is not None:
            vp = v[k0 + pk].float()[None]
            assert bool(((o.float() - vp).abs() <= vp.abs() * 2.0 ** -8 + 1e-6).all()), what
            continue
        qh, kh, vh = _heads72(q[s0:s0 + ql], H), _heads72(k[k0:k0 + kl], H), _heads72(v[k0:k0 + kl], H)
        r64 = F.scaled_dot_product_attention(qh.double(), kh.double(), vh.double(), scale=scale)
        if ql >= 16:
            e_sdpa = _rel(F.scaled_dot_product_attention(qh, kh, vh, scale=scale), r64)
            e = _rel(_heads72(o, H), r64)
            assert e <= 2 * e_sdpa + 1e-6, (what, e, e_sdpa)
        else:  # a row or two: the ratio of two tiny samples means little; P's bf16 rounding and the output's, absolutely
            err = (_heads72(o, H).double() - r64).abs()
            assert bool((err <= r64.abs() * 2.0 ** -7 + 1e-2).all()), (what, float(err.max()))
    first = out.clone()
    for _ in range(2):
        ops.attention_varlen_d72(q, k, v, H, segs_dev, 130, scale=scale, out=out)
        assert torch.equal(out, first)
    check_fence(out, obuf)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 2, 15, 31, 32])
def test_temporal_d72_fenced(T):
    """`mc_attn_temporal_d72` at heads 1 / 5 / 16 (warps past the last head return), S 1 / 7, B 1 / 3: q / k / v column views
    with NaN on both sides, fenced output. The kernel is fp32 up to the final bf16 rounding: within one bf16 ulp of fp64
    everywhere; T = 1 returns V exactly."""
    ops = _ops()
    scale = 0.2
    g = torch.Generator(device=DEV).manual_seed(T)
    for heads in (1, 5, 16):
        for S in (1, 7):
            for B in (1, 3):
                rows, W = B * T * S, heads * 72
                qkv = []
                for _ in range(3):
                    t, _ = fenced((rows, W), BF, (0, 1, 8, 8))
                    t.copy_(_randn((rows, W), g, 1.5))
                    qkv.append(t)
                q, k, v = qkv
                out, obuf = fenced((rows, W), BF, (1, 1, 8, 8), fill="fence")
                ops.attention_temporal_d72(q, k, v, heads, B, T, S, scale=scale, out=out)
                check_fence(out, obuf)
                what = (T, heads, S, B)
                assert bool(torch.isfinite(out.float()).all()), what
                if T == 1:
                    assert torch.equal(out, v), what
                    continue
                seq = lambda t: t.reshape(B, T, S, heads, 72).permute(0, 2, 3, 1, 4).reshape(B * S, heads, T, 72)  # noqa: E731
                r64 = F.scaled_dot_product_attention(seq(q).double(), seq(k).double(), seq(v).double(), scale=scale)
                err = (seq(out).double() - r64).abs()
                assert bool((err <= r64.abs() * 2.0 ** -7 + 1e-4).all()), (what, float(err.max()))


def _ulp_err(got, ref, pairs):
    """|got - ref| in bf16 ulps of |ref| (of the RoPE pair's magnitude when `pairs`: a flipped rounding of either element moves
    both outputs by up to an ulp of the pair)."""
    g, r = got.double(), ref.double()
    mag = r.reshape(*r.shape[:-1], -1, 2).norm(dim=-1, keepdim=True).expand(*r.shape[:-1], -1, 2).reshape(r.shape) if pairs else r.abs()
    ulp = (mag.clamp_min(1e-30).log2().floor() - 7).exp2()
    return (g - r).abs() / ulp


def _assert_ulps(got, ref, pairs, what):
    """test_rmsnorm72_rope's criterion: at most 2 ulps anywhere, under 1 % of the elements off at all."""
    err = _ulp_err(got, ref, pairs)
    n_off = int((err > 0).sum())
    assert float(err.max()) <= 2.0 and n_off <= max(1, 0.01 * err.numel()), (what, float(err.max()), n_off)


def _rms_rope_ref(x, w, heads, hd, cs=None, pos=None):
    """fp64 statement of the per-head RMSNorm + RoPE kernels: bf16(bf16(x * rsqrt(mean(x^2) + eps)) * w), then RoPE on
    (even, odd) pairs from the bf16 values, rounded to bf16 once."""
    rows = x.shape[0]
    v = x.double().reshape(rows, heads, hd)
    o = _rb(_rb(v * torch.rsqrt(v.pow(2).mean(-1, keepdim=True) + 1e-6)) * w.double())
    if cs is not None:
        c = cs.double()[pos].reshape(rows, 1, hd // 2, 2)
        re, im = o.reshape(rows, heads, hd // 2, 2).unbind(-1)
        o = torch.stack([re * c[..., 0] - im * c[..., 1], im * c[..., 0] + re * c[..., 1]], -1)
    return _rb(o).reshape(rows, heads * hd)


def _rope_table(P, hd, g):
    ang = torch.rand(P, hd // 2, device=DEV, generator=g, dtype=torch.float64) * 6.28
    return torch.stack([ang.cos(), ang.sin()], -1).reshape(P, hd).float().contiguous()


def _rms72_case(rows, heads, pos_div, P, g):
    ops = _ops()
    W = heads * 72
    x, xbuf = fenced((rows, W), BF, (1, 1, 8, 8), fill="fence")
    x.copy_(_randn((rows, W), g, 2.0))
    x0 = x.clone()
    w = (1 + 0.2 * _randn((72,), g)).bfloat16().float()
    cs = _rope_table(P, 72, g) if P else None
    ops.rmsnorm_head72_rope_(x, w, heads, cs, pos_div=pos_div)
    check_fence(x, xbuf)
    pos = (torch.arange(rows, device=DEV) // pos_div) % P if P else None
    _assert_ulps(x, _rms_rope_ref(x0, w, heads, 72, cs, pos), P > 0, (rows, heads, pos_div, P))


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [1, 5, 16])
def test_rmsnorm_head72_rope_fenced(heads):
    """`mc_rmsnorm_head72_rope` in place on a fenced view: pos_div 1 / S, RoPE tables of 1 and 32 positions, and no RoPE."""
    g = torch.Generator(device=DEV).manual_seed(heads)
    B, T, S = 2, 5, 7
    for pos_div in (1, S):
        for P in (0, 1, 32):
            _rms72_case(B * T * S, heads, pos_div, P, g)
    _rms72_case(1, heads, 1, 32, g)


@pytest.mark.gpu
def test_rmsnorm_head72_rope_grid_stride_wraps():
    """47 700 rows x 16 heads: more items than the grid's num_sms * 16 * 256 threads, so the grid-stride loop wraps."""
    assert 47700 * 16 > torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256
    _rms72_case(47700, 16, 1590, 15, torch.Generator(device=DEV).manual_seed(5))


@pytest.mark.gpu
@pytest.mark.parametrize("cols", [8, 72, 1152, 2048])
def test_ln_t2i_modulate_fenced(cols):
    """LN + t2i_modulate (`mc_ln_modulate` mode 2) at 1 / 7 / 4099 rows up to its 2048-column limit, x between NaN rows, the
    output a row slice of a buffer with sentinel rows either side; against an fp64 evaluation of the bf16 chain
    bf16(bf16(bf16(LN(x)) * bf16(1 + scale)) + shift) at test_ln_t2i_modulate_matches_emulation's ulp criterion."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(cols)
    for rows in (1, 7, 4099):
        x, _ = fenced((rows, cols), BF, (1, 1, 0, 0), pitch=cols)
        x.copy_(_randn((rows, cols), g, 3.0) + 0.5)
        em = _randn((6, cols), g, 0.5).bfloat16().float()
        out, obuf = fenced((rows, cols), BF, (2, 2, 0, 0), fill="fence", pitch=cols)
        assert x.is_contiguous() and out.is_contiguous()
        ops.ln_t2i_modulate(x, em, 4, 3, out=out)
        check_fence(out, obuf)
        ln = F.layer_norm(x.double(), (cols,), eps=1e-6)
        e = em.double()
        want = _rb(_rb(_rb(ln) * _rb(1.0 + e[4])) + e[3])
        mag = torch.maximum(want.abs(), (want - e[3]).abs())  # |result| and |LN(x) * (1 + scale)|
        ulp = (mag.clamp_min(1e-30).log2().floor() - 7).exp2()
        diff = (out.double() - want).abs() / ulp
        n_off = int((diff > 0).sum())
        assert float(diff.max()) <= 2.0 and n_off <= max(2, 1e-3 * diff.numel()), (rows, cols, float(diff.max()), n_off)


# ------------------------------------------------------------------------------------------- row-wise and elementwise kernels
@pytest.mark.gpu
@pytest.mark.parametrize("rope", [False, True])
@pytest.mark.parametrize("rows,heads", [(1, 1), (77, 3), (4609, 24)])
def test_rmsnorm_head_rope_fenced(rows, heads, rope):
    """`mc_rmsnorm_head_rope` (head_dim 128) in place on a fenced view; 1 and 231 items leave the last half-warp idle."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(rows + heads)
    x, xbuf = fenced((rows, heads * 128), BF, (1, 1, 8, 8), fill="fence")
    x.copy_(_randn(x.shape, g, 2.0))
    x0 = x.clone()
    w = (1 + 0.2 * _randn((128,), g)).bfloat16().float()
    cs = _rope_table(rows, 128, g) if rope else None
    ops.rmsnorm_head_rope_(x, w, heads, cs)
    check_fence(x, xbuf)
    pos = torch.arange(rows, device=DEV) if rope else None
    _assert_ulps(x, _rms_rope_ref(x0, w, heads, 128, cs, pos), rope, (rows, heads, rope))


@pytest.mark.gpu
def test_colmean_fenced():
    """`mc_colmean_bf16` (torch: bf16(bf16(sum) / bf16(rows))) on a NaN-fenced view, into a fenced output."""
    ops, L = _ops(), _lib()
    g = torch.Generator(device=DEV).manual_seed(1)
    for rows in (1, 256, 257):
        for cols in (1, 3073):
            x, _ = fenced((rows, cols), BF, (1, 1, 8, 8))
            x.copy_(_randn((rows, cols), g) + 0.3)
            out, obuf = fenced((cols,), BF, (0, 0, 8, 8), fill="fence")
            L.check(L.lib.mc_colmean_bf16(x.data_ptr(), x.stride(0), rows, cols, out.data_ptr(), ops._stream()))
            check_fence(out, obuf)
            s = x.double().sum(0)
            ref = _rb(_rb(s) / _rb(torch.tensor(float(rows), dtype=torch.float64)))
            # the kernel's fp32 running sum may flip bf16(sum) by one ulp: two ulps of the result, plus the fp32 sum's own error
            tol = ref.abs() * 2.0 ** -6 + 3e-5 * x.double().abs().sum(0) / rows
            assert bool(((out.double() - ref).abs() <= tol).all()), (rows, cols)


@pytest.mark.gpu
def test_silu_and_cast_fenced():
    """`mc_silu_bf16` within a bf16 ulp of fp64, `mc_cast` both ways bit for bit: NaN around the input, fenced output."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(2)
    for n in (1, 7, 3073):
        x, _ = fenced((n,), BF, (0, 0, 8, 8))
        x.copy_(_randn((n,), g, 3.0))
        y, ybuf = fenced((n,), BF, (0, 0, 8, 8), fill="fence")
        ops.silu(x, out=y)
        check_fence(y, ybuf)
        xd = x.double()
        ref = xd * torch.sigmoid(xd)
        assert bool(((y.double() - ref).abs() <= ref.abs() * 2.0 ** -7 + 1e-6).all()), n
        for sdt, ddt in ((F32, BF), (BF, F32)):
            s, _ = fenced((n,), sdt, (0, 0, 8, 8))
            s.copy_(_randn((n,), g, 10.0))
            d, dbuf = fenced((n,), ddt, (0, 0, 8, 8), fill="fence")
            ops.cast_into(s, d)
            check_fence(d, dbuf)
            assert torch.equal(d, s.to(ddt)), (n, sdt)


@pytest.mark.gpu
def test_transpose_fenced():
    """`mc_transpose_bf16` at rows, cols in {1, 63, 64, 65, 130} (partial 64x64 tiles), padded lds / ldd: bit-exact."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(3)
    for rows in (1, 63, 64, 65, 130):
        for cols in (1, 63, 64, 65, 130):
            s, _ = fenced((rows, cols), BF, (1, 1, 8, 8))
            s.copy_(_randn((rows, cols), g))
            d, dbuf = fenced((cols, rows), BF, (1, 1, 8, 8), fill="fence")
            ops.transpose(s, d)
            check_fence(d, dbuf)
            assert torch.equal(d, s.t()), (rows, cols)


_AXPB_DTYPES = [(BF, F32, F32), (F32, BF, F32), (F32, F32, F32), (BF, BF, BF), (BF, BF, F32), (F32, BF, BF), (BF, F32, BF), (F32, F32, BF)]
_NS = (1, 7, 8, 9, 4095, 4096 * 3 + 5)


def _cl(dt, mixed):
    """Left margin: fp32 views 32-byte aligned (the vector path), or only 16-byte aligned when `mixed` (the scalar path)."""
    return 16 // torch.empty(0, dtype=dt).element_size() if (mixed and dt == F32) else 8


@pytest.mark.gpu
@pytest.mark.parametrize("da,db,do", _AXPB_DTYPES)
def test_cache_hit_add_and_residual_sub_fenced(da, db, do):
    """Every dtype combination `dispatch_axpb` builds, at ragged sizes, aligned and with fp32 operands 16- but not 32-byte
    aligned: bit-equal to the fp32 sum / difference rounded to the output type, NaN after the inputs, fenced output."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(_AXPB_DTYPES.index((da, db, do)))
    for n in _NS:
        for mixed in (False, True):
            a, _ = fenced((n,), da, (0, 0, _cl(da, mixed), 8))
            a.copy_(_randn((n,), g))
            b, _ = fenced((n,), db, (0, 0, _cl(db, mixed), 8))
            b.copy_(_randn((n,), g, 0.3))
            for fn, sign in ((ops.cache_hit_add, 1.0), (ops.residual_sub, -1.0)):
                o, obuf = fenced((n,), do, (0, 0, _cl(do, mixed), 8), fill="fence")
                fn(a, b, out=o)
                check_fence(o, obuf)
                assert torch.equal(o, (a.float() + sign * b.float()).to(do)), (n, mixed, sign)


@pytest.mark.gpu
def test_cfg_kernels_and_dequant_fenced():
    """`mc_cfg_combine`, `mc_cfg_step` (two history terms, x0 output) and `mc_dequant_fp8_bf16` at ragged sizes, aligned and
    16- but not 32-byte aligned: bit-equal to the torch expressions they replace, NaN after the inputs, fenced outputs."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(4)

    def inp(n, mixed, dt=F32, scale=1.0):
        t, _ = fenced((n,), dt, (0, 0, _cl(dt, mixed), 8))
        t.copy_(_randn((n,), g, scale))
        return t

    f = lambda a: torch.tensor(a, dtype=F32, device=DEV)  # noqa: E731
    for n in _NS:
        for mixed in (False, True):
            cond, uncond, x, h0, h1 = (inp(n, mixed) for _ in range(5))
            o, obuf = fenced((n,), F32, (0, 0, _cl(F32, mixed), 8), fill="fence")
            ops.cfg_combine(cond, uncond, 5.0, out=o)
            check_fence(o, obuf)
            v = uncond + f(5.0) * (cond - uncond)
            assert torch.equal(o, v), (n, mixed)
            o, obuf = fenced((n,), F32, (0, 0, _cl(F32, mixed), 8), fill="fence")
            x0, x0buf = fenced((n,), F32, (0, 0, _cl(F32, mixed), 8), fill="fence")
            ops.cfg_step(cond, uncond, 6.5, x, -0.7, coef_x=0.93, hist=[h0, h1], coef_h=[0.37, -1.9], sigma=0.81, out=o, x0_out=x0)
            check_fence(o, obuf)
            check_fence(x0, x0buf)
            v = uncond + f(6.5) * (cond - uncond)
            want = f(0.93) * x + f(-0.7) * v + f(0.37) * h0 + f(-1.9) * h1
            assert torch.equal(o, want) and torch.equal(x0, x - f(0.81) * v), (n, mixed)
    for rows, cols in ((1, 1), (1, 7), (1, 8), (1, 9), (5, 819), (1, 4096 * 3 + 5), (3, 4096), (12, 1024), (7, 48)):
        n = rows * cols
        q, _ = fenced((n,), torch.float8_e4m3fn, (0, 0, 16, 16))
        q.copy_((_randn((n,), g, 4.0)).to(torch.float8_e4m3fn))
        q = q.view(rows, cols)
        sc, _ = fenced((rows,), BF, (0, 0, 8, 8))
        sc.copy_(_randn((rows,), g, 0.01).bfloat16())
        o, obuf = fenced((n,), BF, (0, 0, 8, 8), fill="fence")
        ops.dequant_fp8_bf16(q, sc, o.view(rows, cols))
        check_fence(o, obuf)
        assert torch.equal(o.view(rows, cols), q.to(BF) * sc[:, None]), (rows, cols)


# ------------------------------------------------------------------------------------------- staged row kernels (K7, K9, K3)
U32 = 2.0 ** -24  # fp32 unit roundoff


def _staged_rows(sms):
    """Row counts either side of the 1024-row switch to the staged forms, a ragged last chunk of 8, and two chunks per CTA
    plus a ragged one."""
    return (1023, 1024, 1025, 1031, 2 * 8 * sms + 3)


def _ln_chain(x, a, b, mode, round_ln, out_bf16, eps=1e-6):
    """fp64 reference and per-element bound of K7 (`mc_ln_modulate` modes 0 / 1) on x [rows, cols]: y = LN(x) (rounded to bf16
    when round_ln) times aa = fp32(1 + a) (mode 0) or a (mode 1), plus b, each rounded in fp32, stored as bf16 or fp32.
    The fp32 two-pass statistics: a lane sums at most cols / 32 values and the warp (or team) adds 5-7 levels, so the mean is
    within (cols / 32 + 8) u mean|x| and the variance relative within (cols / 32 + 10) u, plus the mean error squared; rsqrtf
    2 ulp, (x - mean) * rstd 2 u. round_ln may flip the LN value's bf16 rounding by one ulp (2^-7 relative); the bf16 store
    adds half an ulp (2^-8)."""
    v = x.double()
    cols = v.shape[1]
    k = cols / 32 + 8
    mu = v.mean(1, keepdim=True)
    var = (v - mu).pow(2).mean(1, keepdim=True)
    rstd = (var + eps).rsqrt()
    ln = (v - mu) * rstd
    dmu = k * U32 * v.abs().mean(1, keepdim=True)
    e_r = 0.5 * ((k + 2) * U32 + dmu.pow(2) / (var + eps)) + 3 * U32
    e_ln = dmu * rstd + (e_r + 2 * U32) * ln.abs()
    aa = ((1.0 + a) if mode == 0 else a).double()  # fp32 1 + a, as the kernel forms it
    if round_ln:
        ln = _rb(ln)
        e_ln = e_ln + ln.abs() * 2.0 ** -7
    ref = ln * aa + b.double()
    bound = e_ln * aa.abs() + U32 * (2 * (ln * aa).abs() + ref.abs())
    if out_bf16:
        bound = bound * (1 + 2.0 ** -8) + ref.abs() * 2.0 ** -8
    return ref, bound


@pytest.mark.gpu
@pytest.mark.parametrize("cols", [256, 384, 1024, 1536, 2048, 3072, 5120])
def test_ln_modulate_staged_fenced(cols):
    """K7 (`mc_ln_modulate` modes 0 and 1) at the row counts either side of the staged form (G = 2 / 2 / 4 / 6 / 8 by width,
    the wide team-per-row form at 3072 and 5120): x fp32 and bf16 with NaN rows after it, out fp32 and bf16 a row window of a
    fenced buffer, round_ln on and off; every element against fp64 within `_ln_chain`'s bound."""
    L = _lib()
    ops = _ops()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator(device=DEV).manual_seed(cols)
    for rows in _staged_rows(sms):
        for xdt in (F32, BF):
            x, _ = fenced((rows, cols), xdt, (0, 8, 0, 0), pitch=cols)
            x.copy_(_randn((rows, cols), g, 3.0) + 0.5)
            p, _ = fenced((6 * cols,), F32, (0, 0, 8, 8))
            p.copy_(_randn((6 * cols,), g, 0.3))
            em = p.view(6, cols)
            for mode in (0, 1):
                a, b = (em[4], em[3]) if mode == 0 else (em[0], em[5])
                for round_ln in (0, 1):
                    for odt in (F32, BF):
                        out, obuf = fenced((rows, cols), odt, (2, 2, 0, 0), fill="fence", pitch=cols)
                        p0, p1 = (em, None) if mode == 0 else (em[0], em[5])
                        L.check(L.lib.mc_ln_modulate(x.data_ptr(), L.MC_BF16 if xdt == BF else L.MC_F32, rows, cols, 1e-6, mode,
                                                     p0.data_ptr(), None if p1 is None else p1.data_ptr(), 4, 3, round_ln,
                                                     out.data_ptr(), L.MC_BF16 if odt == BF else L.MC_F32, ops._stream()))
                        check_fence(out, obuf)
                        ref, bound = _ln_chain(x, a, b, mode, round_ln, odt == BF)
                        err = (out.double() - ref).abs()
                        what = (rows, cols, xdt, mode, round_ln, odt)
                        assert bool(torch.isfinite(out.float()).all()), what
                        assert bool((err <= bound).all()), (what, float((err / bound).max()))


def _rope64(o, cs, cols):
    """fp64 RoPE of o [rows, cols] with cos_sin [rows, head_dim] (interleaved cos, sin): column c at position c % head_dim."""
    hd = cs.shape[1]
    c = cs.double()[:, torch.arange(cols, device=cs.device) % hd].reshape(o.shape[0], cols // 2, 2)
    re, im = o.reshape(o.shape[0], cols // 2, 2).unbind(-1)
    return torch.stack([re * c[..., 0] - im * c[..., 1], im * c[..., 0] + re * c[..., 1]], -1).reshape(o.shape)


@pytest.mark.gpu
@pytest.mark.parametrize("segs,rows", [(1, 1031), (2, 515), (4, 257), (3, 401), (1, 33), (2, 33)])
@pytest.mark.parametrize("rope", [False, True])
def test_rmsnorm_rope_segs_fenced(segs, rows, rope):
    """K9 (`mc_rmsnorm_rope_segs`) in place on a strided view: segs 1 / 2 / 4 take the staged ring (ragged last stage), 3 the
    register form; the fenced columns left of the view, between segs * cols and ld, right of it, and the fenced rows above and
    below must keep their bytes; cos_sin has NaN rows after the last. cols 256 / 1024 / 1536 / 2048, and 5120 (one wide launch per
    segment) at 33 rows. Every element of every segment within test_rmsnorm72_rope's ulp criterion of fp64."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(segs * 1000 + rows + rope)
    for cols in ((5120,) if rows == 33 else (256, 1024, 1536, 2048)):
        x, xbuf = fenced((rows, segs * cols), BF, (1, 1, 8, 16), fill="fence")
        x.copy_(_randn(x.shape, g, 2.0))
        x0 = x.clone()
        w, _ = fenced((segs * cols,), F32, (0, 0, 8, 8))
        w.copy_(1 + 0.2 * _randn((segs * cols,), g))
        cs = None
        if rope:
            cs, _ = fenced((rows, 128), F32, (0, 8, 0, 0), pitch=128)
            cs.copy_(_rope_table(rows, 128, g))
        ops.rmsnorm_rope_segs_(x, w.view(segs, cols), segs, cs, 128)
        check_fence(x, xbuf)
        for sg in range(segs):
            v = x0[:, sg * cols:(sg + 1) * cols].double()
            o = _rb(v * torch.rsqrt(v.pow(2).mean(-1, keepdim=True) + 1e-6)) * w[sg * cols:(sg + 1) * cols].double()
            if rope:
                o = _rope64(o, cs, cols)
            _assert_ulps(x[:, sg * cols:(sg + 1) * cols], _rb(o), rope, (segs, rows, cols, sg, rope))


def _stats_chain(c, p, eps=0.0):
    """fp64 (sum ratio, sum ratio^2, sum (1 - cos)) over the rows of c, p and a bound from the per-row fp32 sums: each of
    |c|^2, |p|^2, c.p is a fused multiply-add chain of cols / 32 terms per lane plus 5 shuffle levels, within
    g = (cols / 32 + 6) u of the sum of |terms|; the norms (sqrtf), the ratio and the cosine add a few u."""
    c, p = c.double(), p.double()
    cols = c.shape[1]
    gm = (cols / 32 + 6) * U32
    nc, np_ = c.norm(dim=1), p.norm(dim=1)
    dot = (c * p).sum(1)
    ratio = nc / (np_ + eps)
    cosv = dot / (nc.clamp_min(1e-8) * np_.clamp_min(1e-8))
    e_ratio = ratio * (gm + 4 * U32)
    e_cos = gm * (c * p).abs().sum(1) / (nc.clamp_min(1e-8) * np_.clamp_min(1e-8)) + cosv.abs() * (gm + 4 * U32) + U32
    ref = torch.stack([ratio.sum(), ratio.pow(2).sum(), (1 - cosv).sum()])
    bound = torch.stack([e_ratio.sum(), (2 * ratio * e_ratio + U32 * ratio.pow(2)).sum(), e_cos.sum()]) + 1e-12 * ref.abs()
    return ref, bound


@pytest.mark.gpu
@pytest.mark.parametrize("cols,dt", [(1536, F32), (3072, F32), (5120, F32), (1536, BF)])
def test_residual_stats_fenced(cols, dt):
    """K3 (`mc_residual_stats`, and `mc_residual_sub_stats` in fp32) at 1 / 3 / 4 / 5 / 1027 rows: fp32 1536 and 3072 take the
    staged form (3072: two stages of 4 rows, the fused form the warp-per-row kernel), 5120 and bf16 the warp-per-row kernel;
    inputs with NaN rows after them; the fused r_out a fenced row window, bit-equal to x_out - x_in; the three sums against
    fp64 within `_stats_chain`'s bound."""
    ops, L = _ops(), _lib()
    g = torch.Generator(device=DEV).manual_seed(cols + (dt == BF))
    code = L.MC_BF16 if dt == BF else L.MC_F32
    for rows in (1, 3, 4, 5, 1027):
        prev, _ = fenced((rows, cols), dt, (0, 8, 0, 0), pitch=cols)
        prev.copy_(_randn((rows, cols), g, 0.1))
        cur, _ = fenced((rows, cols), dt, (0, 8, 0, 0), pitch=cols)
        cur.copy_(prev.float() * (0.97 + 0.05 * torch.rand(rows, 1, device=DEV, generator=g)) + _randn((rows, cols), g, 0.01))
        stats = torch.empty(4, dtype=torch.float64, device=DEV)
        L.check(L.lib.mc_residual_stats(cur.data_ptr(), code, prev.data_ptr(), code, rows, cols, 0.0, stats.data_ptr(), ops._stream()))
        ref, bound = _stats_chain(cur, prev)
        assert float(stats[3]) == rows
        assert bool(((stats[:3] - ref).abs() <= bound).all()), (rows, cols, dt, stats.tolist(), ref.tolist())
        if dt == BF:
            continue
        x_in, _ = fenced((rows, cols), BF, (0, 8, 0, 0), pitch=cols)
        x_in.copy_(_randn((rows, cols), g))
        x_out, _ = fenced((rows, cols), F32, (0, 8, 0, 0), pitch=cols)
        x_out.copy_(x_in.float() + cur)
        r, rbuf = fenced((rows, cols), F32, (1, 1, 0, 0), fill="fence", pitch=cols)
        L.check(L.lib.mc_residual_sub_stats(x_out.data_ptr(), L.MC_F32, x_in.data_ptr(), L.MC_BF16, r.data_ptr(), prev.data_ptr(), rows,
                                            cols, 0.0, stats.data_ptr(), ops._stream()))
        check_fence(r, rbuf)
        assert torch.equal(r, x_out - x_in.float()), (rows, cols)
        ref, bound = _stats_chain(r, prev)
        assert bool(((stats[:3] - ref).abs() <= bound).all()), (rows, cols, "fused", stats.tolist(), ref.tolist())
