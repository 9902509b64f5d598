"""PyTorch-tensor front end of the C ABI: tensors in, tensors out, kernels on the current CUDA stream.

PyTorch is used for device memory and streams only; every function below lands in exactly one hand-written
sm_90a kernel of libmagcache_b200.so (see include/magcache_b200.h for the reference statement each one replaces).
"""
import math

import torch

from . import _lib
from ._lib import MC_BF16, MC_F32, check, lib

LAUNCHES = 0  # number of libmagcache_b200 kernel-launching calls made by this process (bench.py reports the delta)
PROFILE = None  # bench.py sets this to a dict: tag -> list of (start_event, end_event) recorded around launches
PROFILE_TAGS = None  # None: every launch is recorded (under its tag, or the op's name when the caller gave none); a set: only these tags


class _Timed:
    """Records a CUDA-event pair on the launching stream around one tagged kernel launch (only when PROFILE is enabled)."""

    def __init__(self, tag, default=None):
        if PROFILE is None:
            self.tag = None
        elif PROFILE_TAGS is None:
            self.tag = tag or default
        else:
            self.tag = tag if tag in PROFILE_TAGS else None

    def __enter__(self):
        if self.tag is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *a):
        if self.tag is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            PROFILE.setdefault(self.tag, []).append((self.e0, e1))


def _dt(t):
    if t.dtype == torch.float32:
        return MC_F32
    if t.dtype == torch.bfloat16:
        return MC_BF16
    raise TypeError(f"unsupported dtype {t.dtype} (fp32 / bf16 only)")


def _dev(t, name="tensor"):
    if not t.is_cuda:
        raise RuntimeError(f"{name} must live on a CUDA device: magcache_b200 has no CPU path")
    return t


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _count(n=1):
    global LAUNCHES
    LAUNCHES += n


def _promote(a, b):
    return torch.promote_types(a.dtype, b.dtype)


def cache_hit_add(x, r, out=None, tag=None):
    """`x + residual_x` (MagCache4Wan2.1/magcache_generate.py:295) with torch's type promotion."""
    _dev(x, "x"), _dev(r, "r")
    assert x.shape == r.shape and x.is_contiguous() and r.is_contiguous()
    if out is None:
        out = torch.empty(x.shape, dtype=_promote(x, r), device=x.device)
    with _Timed(tag, "add"):
        check(lib.mc_cache_hit_add(x.data_ptr(), _dt(x), r.data_ptr(), _dt(r), out.data_ptr(), _dt(out), x.numel(), _stream()))
    _count()
    return out


def residual_sub(x_out, x_in, out=None, tag=None):
    """`residual_x = x - ori_x` (MagCache4Wan2.1/magcache_generate.py:299)."""
    _dev(x_out, "x_out"), _dev(x_in, "x_in")
    assert x_out.shape == x_in.shape and x_out.is_contiguous() and x_in.is_contiguous()
    if out is None:
        out = torch.empty(x_out.shape, dtype=_promote(x_out, x_in), device=x_out.device)
    with _Timed(tag, "residual_sub"):
        check(lib.mc_residual_sub(x_out.data_ptr(), _dt(x_out), x_in.data_ptr(), _dt(x_in), out.data_ptr(), _dt(out), x_out.numel(), _stream()))
    _count()
    return out


def cfg_combine(cond, uncond, guide_scale, out=None):
    """`uncond + guide_scale * (cond - uncond)` (wan_magcache.py:301-302) in one pass, bit-identical to the torch expression."""
    _dev(cond), _dev(uncond)
    assert cond.dtype == uncond.dtype == torch.float32 and cond.shape == uncond.shape and cond.is_contiguous() and uncond.is_contiguous()
    if out is None:
        out = torch.empty_like(cond)
    check(lib.mc_cfg_combine(cond.data_ptr(), uncond.data_ptr(), float(guide_scale), out.data_ptr(), cond.numel(), _stream()))
    _count()
    return out


def cfg_step(cond, uncond, guide_scale, x, coef_v, coef_x=1.0, hist=(), coef_h=(), sigma=0.0, out=None, x0_out=None, tag=None):
    """CFG combine + scheduler update in one kernel (`mc_cfg_step`): `out = coef_x*x + coef_v*v + sum coef_h[i]*hist[i]` with
    `v = uncond + guide_scale*(cond - uncond)` (wan_magcache.py:301-310); `out` may be `x` itself. Euler flow step:
    `cfg_step(cond, uncond, g, x, sigma_next - sigma)` — bit-identical to `x + (sigma_next - sigma) * (uncond + g*(cond - uncond))`.
    With `x0_out` the x0-prediction `x - sigma*v` is written as well."""
    import ctypes
    tensors = [cond, uncond, x, *hist] + ([out] if out is not None else []) + ([x0_out] if x0_out is not None else [])
    for t in tensors:
        _dev(t)
        assert t.dtype == torch.float32 and t.is_contiguous() and t.numel() == cond.numel()
    assert len(hist) == len(coef_h) <= 4
    if out is None:
        out = torch.empty_like(x)
    hp = (ctypes.c_void_p * max(len(hist), 1))(*[h.data_ptr() for h in hist])
    hc = (ctypes.c_float * max(len(hist), 1))(*[float(c) for c in coef_h])
    with _Timed(tag, "cfg_step"):
        check(lib.mc_cfg_step(cond.data_ptr(), uncond.data_ptr(), float(guide_scale), x.data_ptr(), float(coef_x), float(coef_v), hp, hc, len(hist),
                              float(sigma), out.data_ptr(), x0_out.data_ptr() if x0_out is not None else None, cond.numel(), _stream()))
    _count()
    return out


def rel_l1(cur, prev):
    """`((cur - prev).abs().mean() / prev.abs().mean()).cpu().item()` (wan_teacache.py:543): one tiny reduction kernel and the one
    host sync the reference has too. The two means and the quotient are rounded to fp32 like the torch scalars."""
    import numpy as np
    _dev(cur), _dev(prev)
    assert cur.dtype == prev.dtype == torch.float32 and cur.is_contiguous() and prev.is_contiguous() and cur.numel() == prev.numel()
    sums = torch.empty(2, dtype=torch.float64, device=cur.device)
    check(lib.mc_rel_l1(cur.data_ptr(), prev.data_ptr(), cur.numel(), sums.data_ptr(), _stream()))
    _count()
    d, p = sums.tolist()
    n = cur.numel()
    return float(np.float32(d / n) / np.float32(p / n))


def _finish_stats(stats_dev):
    s0, s1, s2, n = stats_dev.tolist()  # the single host sync of the calibration path
    mean = s0 / n
    var = (s1 - s0 * s0 / n) / (n - 1) if n > 1 else float("nan")
    return mean, math.sqrt(max(var, 0.0)), s2 / n


def residual_stats(r_cur, r_prev, denom_eps=0.0, reduce=None):
    """(norm_ratio, norm_std, cos_dis) of MagCache4Wan2.1/magcache_generate.py:167-169 in one pass + one sync. `reduce(stats_dev)` lets
    a token-sharded caller add the four partial sums of every rank before they are finalised."""
    _dev(r_cur), _dev(r_prev)
    assert r_cur.shape == r_prev.shape and r_cur.is_contiguous() and r_prev.is_contiguous()
    cols = r_cur.shape[-1]
    rows = r_cur.numel() // cols
    stats = torch.empty(4, dtype=torch.float64, device=r_cur.device)
    check(lib.mc_residual_stats(r_cur.data_ptr(), _dt(r_cur), r_prev.data_ptr(), _dt(r_prev), rows, cols, float(denom_eps),
                                stats.data_ptr(), _stream()))
    _count(2)
    if reduce is not None:
        stats = reduce(stats)
    return _finish_stats(stats)


def residual_sub_stats(x_out, x_in, r_prev, denom_eps=0.0, reduce=None):
    """Fused `x - ori_x` + statistics against the previous residual (calibration miss epilogue). `reduce(stats_dev)` lets a
    token-sharded caller all-reduce the four partial sums before they are finalised on the host."""
    _dev(x_out), _dev(x_in), _dev(r_prev)
    assert x_out.dtype == torch.float32 and x_in.dtype == torch.bfloat16 and r_prev.dtype == torch.float32
    cols = x_out.shape[-1]
    rows = x_out.numel() // cols
    r = torch.empty_like(x_out)
    stats = torch.empty(4, dtype=torch.float64, device=x_out.device)
    check(lib.mc_residual_sub_stats(x_out.data_ptr(), MC_F32, x_in.data_ptr(), MC_BF16, r.data_ptr(), r_prev.data_ptr(), rows, cols,
                                    float(denom_eps), stats.data_ptr(), _stream()))
    _count(2)
    if reduce is not None:
        stats = reduce(stats)
    return r, _finish_stats(stats)


def patchify(latent, tag=None):
    """latent fp32 [C,F,H,W] -> bf16 [F*(H/2)*(W/2), C*4] (im2col of the (1,2,2) patch embedding)."""
    _dev(latent)
    assert latent.dtype == torch.float32 and latent.dim() == 4 and latent.is_contiguous()
    C, F, H, W = latent.shape
    out = torch.empty(F * (H // 2) * (W // 2), C * 4, dtype=torch.bfloat16, device=latent.device)
    with _Timed(tag, "patchify"):
        check(lib.mc_patchify(latent.data_ptr(), C, F, H, W, out.data_ptr(), _stream()))
    _count()
    return out


def ln_modulate(x, em, scale_idx, shift_idx, eps=1e-6, round_ln_to_bf16=False, out_dtype=torch.bfloat16, out=None, tag=None):
    """bf16/fp32( LN(x) * (1 + em[scale_idx]) + em[shift_idx] ) ; x [rows, cols], em = modulation + e0, fp32 [k, cols]."""
    _dev(x)
    rows, cols = x.shape
    assert x.is_contiguous() and em.dtype == torch.float32 and em.is_contiguous() and em.shape[-1] == cols
    if out is None:
        out = torch.empty(rows, cols, dtype=out_dtype, device=x.device)
    with _Timed(tag, "ln_modulate"):
        check(lib.mc_ln_modulate(x.data_ptr(), _dt(x), rows, cols, eps, 0, em.data_ptr(), None, scale_idx, shift_idx,
                                 int(round_ln_to_bf16), out.data_ptr(), _dt(out), _stream()))
    _count()
    return out


def ln_affine(x, weight, bias, eps=1e-6, out_dtype=torch.bfloat16, out=None, tag=None):
    """LayerNorm with elementwise affine (norm3 of the Wan block)."""
    _dev(x)
    rows, cols = x.shape
    assert x.is_contiguous() and weight.dtype == torch.float32 and bias.dtype == torch.float32
    if out is None:
        out = torch.empty(rows, cols, dtype=out_dtype, device=x.device)
    with _Timed(tag, "ln_affine"):
        check(lib.mc_ln_modulate(x.data_ptr(), _dt(x), rows, cols, eps, 1, weight.data_ptr(), bias.data_ptr(), 0, 0, 0, out.data_ptr(),
                                 _dt(out), _stream()))
    _count()
    return out


def rmsnorm_rope_(x, weight, cos_sin=None, head_dim=128, eps=1e-6, tag=None):
    """In-place WanRMSNorm (+ RoPE when cos_sin [rows, head_dim] is given) on a bf16 [rows, cols] view (row stride allowed)."""
    _dev(x)
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1 and weight.dtype == torch.float32
    rows, cols = x.shape
    if cos_sin is not None:
        assert cos_sin.dtype == torch.float32 and cos_sin.is_contiguous() and cos_sin.shape == (rows, head_dim)
    with _Timed(tag, "rmsnorm_rope"):
        check(lib.mc_rmsnorm_rope(x.data_ptr(), x.stride(0), rows, cols, weight.data_ptr(), eps,
                                  cos_sin.data_ptr() if cos_sin is not None else None, head_dim, _stream()))
    _count()
    return x


def rmsnorm_rope_segs_(x, weights, segs, cos_sin=None, head_dim=128, eps=1e-6, tag=None):
    """`rmsnorm_rope_` over `segs` adjacent column blocks per row in ONE launch (q | k of the fused q|k|v projection): x bf16
    [rows, >= segs*cols] view, weights fp32 [segs, cols]; RoPE applies to every block."""
    _dev(x)
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1 and weights.dtype == torch.float32 and weights.is_contiguous()
    rows = x.shape[0]
    cols = weights.shape[-1]
    assert weights.numel() == segs * cols and x.shape[1] >= segs * cols
    if cos_sin is not None:
        assert cos_sin.dtype == torch.float32 and cos_sin.is_contiguous() and cos_sin.shape == (rows, head_dim)
    with _Timed(tag, "rmsnorm_rope"):
        check(lib.mc_rmsnorm_rope_segs(x.data_ptr(), x.stride(0), rows, segs, cols, weights.data_ptr(), eps,
                                       cos_sin.data_ptr() if cos_sin is not None else None, head_dim, _stream()))
    _count()
    return x


def rmsnorm_head_rope_(x, weight, heads, cos_sin=None, eps=1e-6, tag=None):
    """In-place per-head RMSNorm (head_dim 128) + optional RoPE on a bf16 [rows, heads*128] view (row stride allowed): the q / k
    normalisation of the MMDiT attention. weight fp32 [128]; cos_sin fp32 [rows, 128] (interleaved cos, sin)."""
    _dev(x)
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1 and x.shape[1] == heads * 128
    assert weight.dtype == torch.float32 and weight.numel() == 128 and weight.is_contiguous()
    rows = x.shape[0]
    if cos_sin is not None:
        assert cos_sin.dtype == torch.float32 and cos_sin.is_contiguous() and cos_sin.shape == (rows, 128)
    with _Timed(tag, "rmsnorm_head_rope"):
        check(lib.mc_rmsnorm_head_rope(x.data_ptr(), x.stride(0), rows, heads, weight.data_ptr(), eps,
                                       cos_sin.data_ptr() if cos_sin is not None else None, _stream()))
    _count()
    return x


def rmsnorm_head72_rope_(x, weight, heads, cos_sin=None, pos_div=1, eps=1e-6, tag=None):
    """In-place per-head LlamaRMSNorm(72) + optional RoPE (`mc_rmsnorm_head72_rope`) on a bf16 [rows, heads*72] view (row stride
    allowed): the q / k normalisation of Open-Sora's attention. weight fp32 [72]; cos_sin fp32 [P, 72] (interleaved cos, sin per pair),
    row r uses position (r // pos_div) % P."""
    _dev(x)
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1 and x.shape[1] == heads * 72
    assert weight.dtype == torch.float32 and weight.numel() == 72 and weight.is_contiguous()
    P = 1
    if cos_sin is not None:
        assert cos_sin.dtype == torch.float32 and cos_sin.is_contiguous() and cos_sin.dim() == 2 and cos_sin.shape[1] == 72
        P = cos_sin.shape[0]
    with _Timed(tag, "rmsnorm_head72_rope"):
        check(lib.mc_rmsnorm_head72_rope(x.data_ptr(), x.stride(0), x.shape[0], heads, weight.data_ptr(), eps,
                                         cos_sin.data_ptr() if cos_sin is not None else None, int(pos_div), int(P), _stream()))
    _count()
    return x


def attention_varlen_d72(q, k, v, heads, segs, max_q_len, scale=None, out=None, tag=None):
    """softmax(q k^T * scale) v per head (head_dim 72) over independent segments in one launch (`mc_attn_varlen_d72`). q [Lq, H*72],
    k / v [Lk, H*72] row-major bf16 views (row stride allowed); segs: int32 device tensor [n, 4] of (q_start, q_len, k_start, k_len)."""
    _dev(q), _dev(k), _dev(v), _dev(segs, "segs")
    assert q.dtype == k.dtype == v.dtype == torch.bfloat16 and q.stride(1) == 1 and k.stride(1) == 1 and v.stride(1) == 1
    assert q.shape[1] == k.shape[1] == v.shape[1] == heads * 72 and k.shape[0] == v.shape[0]
    assert segs.dtype == torch.int32 and segs.is_contiguous() and segs.dim() == 2 and segs.shape[1] == 4
    if scale is None:
        scale = 1.0 / math.sqrt(72)
    if out is None:
        out = torch.empty(q.shape[0], heads * 72, dtype=torch.bfloat16, device=q.device)
    assert out.stride(1) == 1 and out.shape == q.shape
    with _Timed(tag, "attn_varlen_d72"):
        check(lib.mc_attn_varlen_d72(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), out.data_ptr(),
                                     out.stride(0), heads, segs.data_ptr(), segs.shape[0], int(max_q_len), float(scale), _stream()))
    _count()
    return out


def attention_temporal_d72(q, k, v, heads, B, T, S, scale=None, out=None, tag=None):
    """Temporal attention (`mc_attn_temporal_d72`): rows in B (T S) C order, sequence (b, s) = rows b*T*S + t*S + s; head_dim 72.
    T <= 32 keeps P in fp32 (one lane per query frame); T > 32 runs on the tensor cores and rounds P to bf16 for the PV product,
    as `attention_varlen_d72` does. The kernel is chosen from T alone."""
    _dev(q), _dev(k), _dev(v)
    for t_ in (q, k, v):
        assert t_.dtype == torch.bfloat16 and t_.stride(1) == 1 and t_.shape == (B * T * S, heads * 72)
    if scale is None:
        scale = 1.0 / math.sqrt(72)
    if out is None:
        out = torch.empty(B * T * S, heads * 72, dtype=torch.bfloat16, device=q.device)
    assert out.stride(1) == 1 and out.shape == q.shape
    with _Timed(tag, "attn_temporal_d72"):
        check(lib.mc_attn_temporal_d72(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), out.data_ptr(),
                                       out.stride(0), B, T, S, heads, float(scale), _stream()))
    _count()
    return out


def ln_t2i_modulate(x, em, scale_idx, shift_idx, eps=1e-6, out=None, tag=None):
    """`t2i_modulate(LayerNorm(x), shift, scale)` with the bf16 rounding of every tensor op (`mc_ln_modulate` mode 2): x bf16
    [rows, cols]; em fp32 [k, cols] holding bf16 values (scale row `scale_idx`, shift row `shift_idx`)."""
    _dev(x)
    rows, cols = x.shape
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and em.dtype == torch.float32 and em.is_contiguous() and em.shape[-1] == cols
    if out is None:
        out = torch.empty(rows, cols, dtype=torch.bfloat16, device=x.device)
    assert out.dtype == torch.bfloat16 and out.is_contiguous() and out.shape == x.shape
    with _Timed(tag, "ln_t2i_modulate"):
        check(lib.mc_ln_modulate(x.data_ptr(), MC_BF16, rows, cols, eps, 2, em.data_ptr(), None, scale_idx, shift_idx, 0, out.data_ptr(),
                                 MC_BF16, _stream()))
    _count()
    return out


def opensora_head(x, mod, w, bias, grid, crop, res=None, step=None, out=None, eps=1e-6, tag=None):
    """Open-Sora's final layer + unpatchify in one pass (`mc_opensora_head`): x bf16 [B*T*H*W, D] (x0 with `res` bf16 on a cache hit,
    the sum never written), mod fp32 [B, 2, D] (shift | scale per sample), w bf16 [32, D], bias fp32 [32], grid (T, H, W), crop
    (Tx, Hx, Wx). Returns fp32 [B, 8, Tx, Hx, Wx], bit-equal to OpenSoraEngine.head. With step = (z, guidance_scale, dt) it returns
    instead `z + (u + g * (c - u)) * dt` over the 4 velocity channels, fp32 [B/2, 4, Tx, Hx, Wx] (c: samples [0, B/2), u: [B/2, B);
    z fp32 of that shape, dt fp32 [B/2] on the device); `out` may be `z`."""
    _dev(x, "x")
    T, H, W = grid
    Tx, Hx, Wx = crop
    rows, D = x.shape
    B = rows // (T * H * W)
    assert Tx == T and B * T * H * W == rows and x.dtype == torch.bfloat16 and x.is_contiguous()
    assert res is None or (res.dtype == torch.bfloat16 and res.shape == x.shape and res.is_contiguous())
    assert mod.dtype == torch.float32 and mod.shape == (B, 2, D) and mod.is_contiguous()
    assert w.dtype == torch.bfloat16 and w.shape == (32, D) and w.is_contiguous() and bias.dtype == torch.float32 and bias.numel() == 32
    z = dt = None
    g = 0.0
    if step is None:
        shape = (B, 8, T, Hx, Wx)
    else:
        z, g, dt = step
        shape = (B // 2, 4, T, Hx, Wx)
        assert B % 2 == 0 and z.dtype == torch.float32 and tuple(z.shape) == shape and z.is_contiguous()
        _dev(z, "z"), _dev(dt, "dt")
        assert dt.dtype == torch.float32 and dt.numel() == B // 2 and dt.is_contiguous()
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=x.device)
    assert out.dtype == torch.float32 and tuple(out.shape) == shape and out.is_contiguous()
    with _Timed(tag, "opensora_head"):
        check(lib.mc_opensora_head(x.data_ptr(), res.data_ptr() if res is not None else None, B, T, H, W, D, mod.data_ptr(), w.data_ptr(),
                                   bias.data_ptr(), 8, eps, Hx, Wx, z.data_ptr() if z is not None else None,
                                   dt.data_ptr() if dt is not None else None, float(g), out.data_ptr(), _stream()))
    _count()
    return out


def opensora_head_frames(x, mod, w, bias, grid, crop, t0, out, res=None, step=None, eps=1e-6, tag=None):
    """`opensora_head` on frames [t0, t0 + T) of a sequence-parallel run (`mc_opensora_head_frames`): x bf16 [B*T*H*W, D] holds those
    frames of every sample, grid = (T, H, W) local, crop = (T_out, Hx, Wx) the full tensor. `out` is the full-size fp32 tensor
    [B, 8, T_out, Hx, Wx] (step mode: [B/2, 4, T_out, Hx, Wx], z of that shape, may alias out): only the window's frames are
    written (and read of z), bit-equal to the same frames of one `opensora_head` over the whole video."""
    _dev(x, "x"), _dev(out, "out")
    T, H, W = grid
    T_out, Hx, Wx = crop
    rows, D = x.shape
    B = rows // (T * H * W)
    assert 0 <= t0 and t0 + T <= T_out and B * T * H * W == rows and x.dtype == torch.bfloat16 and x.is_contiguous()
    assert res is None or (res.dtype == torch.bfloat16 and res.shape == x.shape and res.is_contiguous())
    assert mod.dtype == torch.float32 and mod.shape == (B, 2, D) and mod.is_contiguous()
    assert w.dtype == torch.bfloat16 and w.shape == (32, D) and w.is_contiguous() and bias.dtype == torch.float32 and bias.numel() == 32
    z = dt = None
    g = 0.0
    shape = (B, 8, T_out, Hx, Wx)
    if step is not None:
        z, g, dt = step
        shape = (B // 2, 4, T_out, Hx, Wx)
        assert B % 2 == 0 and z.dtype == torch.float32 and tuple(z.shape) == shape and z.is_contiguous()
        _dev(z, "z"), _dev(dt, "dt")
        assert dt.dtype == torch.float32 and dt.numel() == B // 2 and dt.is_contiguous()
    assert out.dtype == torch.float32 and tuple(out.shape) == shape and out.is_contiguous()
    off = t0 * Hx * Wx * 4
    with _Timed(tag, "opensora_head"):
        check(lib.mc_opensora_head_frames(x.data_ptr(), res.data_ptr() if res is not None else None, B, T, H, W, D, mod.data_ptr(),
                                          w.data_ptr(), bias.data_ptr(), 8, eps, Hx, Wx, T_out, z.data_ptr() + off if z is not None else None,
                                          dt.data_ptr() if dt is not None else None, float(g), out.data_ptr() + off, _stream()))
    _count()
    return out


REL_L1_MAX_CTAS = 4096  # MC_LN_REL_L1_MAX_CTAS


def rel_l1_partials(device):
    """Device scratch for `ln_t2i_modulate_rel_l1`'s per-CTA partial sums."""
    return torch.empty(2 * REL_L1_MAX_CTAS, dtype=torch.float64, device=device)


def ln_t2i_modulate_rel_l1(x, em, scale_idx, shift_idx, prev, out, partials, sums, eps=1e-6, tag=None):
    """`ln_t2i_modulate` into `out` fused with TeaCache's input distance against `prev` (`mc_ln_t2i_modulate_rel_l1`):
    sums (fp64 [2], on the device) += (sum |bf16(out - prev)|, sum |prev|). Deterministic; no host sync."""
    _dev(x), _dev(prev), _dev(out)
    rows, cols = x.shape
    assert x.dtype == prev.dtype == out.dtype == torch.bfloat16 and x.is_contiguous() and prev.is_contiguous() and out.is_contiguous()
    assert prev.shape == out.shape == x.shape and em.dtype == torch.float32 and em.is_contiguous() and em.shape[-1] == cols
    assert sums.dtype == partials.dtype == torch.float64 and sums.numel() >= 2 and partials.numel() >= 2 * REL_L1_MAX_CTAS
    with _Timed(tag, "ln_t2i_modulate_rel_l1"):
        check(lib.mc_ln_t2i_modulate_rel_l1(x.data_ptr(), rows, cols, eps, em.data_ptr(), scale_idx, shift_idx, prev.data_ptr(), out.data_ptr(),
                                            partials.data_ptr(), sums.data_ptr(), _stream()))
    _count(2)
    return out


def colmean(x):
    """bf16 mean over the rows of a bf16 [rows, cols] view -> [1, cols] (torch semantics: bf16 sum, then bf16 division)."""
    _dev(x)
    assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    out = torch.empty(1, x.shape[1], dtype=torch.bfloat16, device=x.device)
    check(lib.mc_colmean_bf16(x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], out.data_ptr(), _stream()))
    _count()
    return out


def silu(x, out=None):
    """bf16 silu(x) (fp32 inside)."""
    _dev(x)
    assert x.dtype == torch.bfloat16 and x.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    check(lib.mc_silu_bf16(x.data_ptr(), out.data_ptr(), x.numel(), _stream()))
    _count()
    return out


def gemm(a, b, bias=None, epilogue=_lib.MC_EPI_BIAS_BF16, out=None, gate=None, tag=None):
    """acc = a @ b.T on wgmma (a [M,K] bf16, b [N,K] bf16, row stride allowed) + fused epilogue (see MC_EPI_*)."""
    _dev(a), _dev(b)
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.stride(1) == 1 and b.stride(1) == 1
    M, K = a.shape
    N, K2 = b.shape
    assert K == K2
    if out is None:
        assert epilogue not in (_lib.MC_EPI_BIAS_GATE_RESID, _lib.MC_EPI_BIAS_GATE_RESID_BF16), "the residual epilogues update `out` in place; pass the stream"
        out = torch.empty(M, N, dtype=torch.float32 if epilogue == _lib.MC_EPI_BIAS_F32 else torch.bfloat16, device=a.device)
    want = torch.float32 if epilogue in (_lib.MC_EPI_BIAS_GATE_RESID, _lib.MC_EPI_BIAS_F32) else torch.bfloat16
    assert out.dtype == want and out.stride(1) == 1 and out.shape == (M, N)
    for v in (bias, gate):
        assert v is None or (v.dtype == torch.float32 and v.is_contiguous())
    with _Timed(tag, "gemm_other"):
        check(lib.mc_gemm_bf16(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), M, N, K, bias.data_ptr() if bias is not None else None,
                               epilogue, out.data_ptr(), out.stride(0), gate.data_ptr() if gate is not None else None, _stream()))
    _count()
    return out


def dequant_fp8_bf16(q, scale, out, tag=None):
    """out = bf16(q * scale[row]) (`mc_dequant_fp8_bf16`): q float8_e4m3fn [rows, cols], scale bf16 [rows], out bf16 [rows, cols],
    all contiguous. Bit-equal to `q.to(bf16) * scale[:, None]`, the weight upstream's fp8_linear_forward multiplies by."""
    _dev(q), _dev(scale), _dev(out)
    assert q.dtype == torch.float8_e4m3fn and scale.dtype == torch.bfloat16 and out.dtype == torch.bfloat16
    assert q.dim() == 2 and q.is_contiguous() and scale.is_contiguous() and out.is_contiguous()
    rows, cols = q.shape
    assert scale.shape == (rows,) and out.shape == (rows, cols)
    with _Timed(tag, "dequant_fp8"):
        check(lib.mc_dequant_fp8_bf16(q.data_ptr(), scale.data_ptr(), out.data_ptr(), rows, cols, _stream()))
    _count()
    return out


_WORKSPACES = {}  # (kind, device index) -> torch.uint8 scratch owned by this module (grown on demand, never shrunk)


def _workspace(kind, device, nbytes):
    """Device scratch a kernel needs besides its operands (split-KV partials, the head's modulated weight). One buffer per kind and
    device, used on the calling stream only (the engines are single-stream, as the reference is). It grows when a larger shape shows
    up — eagerly, i.e. before any CUDA-graph capture of that shape (the engines run every graph key eagerly once first)."""
    key = (kind, device.index)
    buf = _WORKSPACES.get(key)
    if buf is None or buf.numel() < nbytes:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError(f"magcache_b200: the {kind} workspace would have to grow inside a CUDA-graph capture; run the shape eagerly once first")
        buf = torch.empty(max(int(nbytes), 1024), dtype=torch.uint8, device=device)
        _WORKSPACES[key] = buf
    return buf


def attention(q, k, v, heads, scale=None, out=None, tag=None, first_key_row=0, seg_flags=None, seg_epoch=None, seg_rows=0):
    """softmax(q k^T * scale) v per head (head_dim 128). q [Lq, H*128], k [Lk, H*128], v [Lk, H*128]: row-major bf16 views (row
    stride allowed — column slices of one fused q|k|v buffer). `first_key_row` / `seg_*`: token-sharded key order, see
    mc_attn_fwd_ex in include/magcache_b200.h."""
    import ctypes
    _dev(q), _dev(k), _dev(v)
    assert q.dtype == k.dtype == v.dtype == torch.bfloat16 and q.stride(1) == 1 and k.stride(1) == 1 and v.stride(1) == 1
    Lq, W = q.shape
    Lk = k.shape[0]
    assert W == heads * 128 and k.shape[1] == W and v.shape == (Lk, W)
    if scale is None:
        scale = 1.0 / math.sqrt(128)
    if out is None:
        out = torch.empty(Lq, W, dtype=torch.bfloat16, device=q.device)
    assert out.dtype == torch.bfloat16 and out.stride(1) == 1 and out.shape == (Lq, W)
    need = ctypes.c_int64(0)
    check(lib.mc_attn_workspace_bytes(Lq, Lk, heads, ctypes.byref(need)))
    ws = _workspace("attention", q.device, need.value) if need.value > 0 else None
    with _Timed(tag, "attn_other"):
        check(lib.mc_attn_fwd_ex(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), out.data_ptr(),
                                 out.stride(0), Lq, Lk, heads, float(scale), ws.data_ptr() if ws is not None else None,
                                 ws.numel() if ws is not None else 0, int(first_key_row),
                                 seg_flags.data_ptr() if seg_flags is not None else None,
                                 seg_epoch.data_ptr() if seg_epoch is not None else None, int(seg_rows), _stream()))
    _count(2 if need.value > 0 else 1)
    return out


attention_rowmajor_v = attention


def linear_f32_small(x, w, b=None, act=0, tag=None):
    """fp32 y = act(x @ w.T + b) for M <= 8 rows (time embedding path). act: 0 none, 1 SiLU on the input, 2 SiLU on the output."""
    _dev(x), _dev(w)
    assert x.dtype == torch.float32 and w.dtype == torch.float32 and x.is_contiguous() and w.is_contiguous()
    M, K = x.shape
    N = w.shape[0]
    y = torch.empty(M, N, dtype=torch.float32, device=x.device)
    with _Timed(tag, "linear_f32_small"):
        check(lib.mc_linear_f32_small(x.data_ptr(), M, K, w.data_ptr(), b.data_ptr() if b is not None else None, N, act, y.data_ptr(), _stream()))
    _count()
    return y


def time_sinusoid(t, dim, tag=None):
    """sinusoidal_embedding_1d(dim, t) computed in float64 on the device, returned as fp32 [len(t), dim]."""
    _dev(t)
    pos = t.to(torch.float64).contiguous()
    out = torch.empty(pos.numel(), dim, dtype=torch.float32, device=t.device)
    with _Timed(tag, "time_sinusoid"):
        check(lib.mc_time_sinusoid(pos.data_ptr(), pos.numel(), dim, out.data_ptr(), _stream()))
    _count()
    return out


class HeadPrep:
    """The head's per-forward preparation (`mc_head_prepare`): the modulated weight split into bf16 hi / lo and the two per-output
    constants, in a device workspace. Built right after the time embedding, consumed by `head_unpatchify(..., prep=...)`."""

    def __init__(self, ptr, nbytes, cols, keep):
        self.ptr, self.nbytes, self.cols, self._keep = ptr, nbytes, cols, keep


def head_prepare(head_mod, e, w_t, b, tag=None, slot=0):
    """Fold (modulation + e) into head.weight for one forward: head_mod [2, cols] fp32, e [cols] fp32, w_t [cols, 64] fp32, b [64].
    `slot`: which of this module's head workspaces receives it — a forward that needs several preparations alive at once (per-token
    timesteps, more than 16 output channels) numbers them."""
    import ctypes
    _dev(w_t)
    cols = w_t.shape[0]
    assert head_mod.shape[-2:] == (2, cols) and e.numel() == cols and w_t.shape == (cols, 64) and w_t.is_contiguous() and b.numel() == 64
    need = ctypes.c_int64(0)
    check(lib.mc_head_workspace_bytes(cols, ctypes.byref(need)))
    ws = _workspace("head" if slot == 0 else f"head{slot}", w_t.device, need.value + 1024)
    ptr = (ws.data_ptr() + 1023) // 1024 * 1024
    with _Timed(tag, "head_prepare"):
        check(lib.mc_head_prepare(head_mod.data_ptr(), e.data_ptr(), w_t.data_ptr(), b.data_ptr(), cols, ptr, need.value, _stream()))
    _count()
    return HeadPrep(ptr, need.value, cols, ws)


def head_unpatchify(x, head_mod, e, w_t, b, grid, c_out=16, residual=None, eps=1e-6, tag=None, row_offset=0, out=None, round_sum_to_bf16=False,
                    peer_outs=None, prep=None, step=None):
    """head(x, e) + unpatchify (MagCache4Wan2.1/magcache_generate.py:304-305) -> fp32 [c_out, F, 2*Hp, 2*Wp].
    x fp32 (the residual stream), or bf16 with `residual` (fp32): the cache-hit sum x + residual is formed on the fly (fused hit
    path, :295). `prep`: a `head_prepare` result for this forward's time embedding (else it is computed here). A token-sharded
    caller passes its contiguous token range (`row_offset`, x.shape[0] rows) and an `out` whose other positions the peers fill;
    `peer_outs` (device pointers of the peers' outputs) makes the kernel store its rows there as well.
    `step` = (cond, x_latent, guide_scale, coef_x, coef_v): this is the unconditional head of a denoising step and the caller loop's
    CFG combine + scheduler update are applied in the epilogue (`mc_head_unpatchify_step`, SURVEY §8f-1): the result is
    `coef_x * x_latent + coef_v * (y + guide_scale * (cond - y))` instead of y — bit-equal to this head followed by `cfg_step`."""
    import ctypes
    _dev(x)
    F, Hp, Wp = grid
    rows, cols = x.shape
    assert row_offset + rows <= F * Hp * Wp and x.is_contiguous()
    if residual is not None:
        assert x.dtype == torch.bfloat16 and residual.dtype == torch.float32 and residual.is_contiguous() and residual.shape == x.shape
    else:
        assert x.dtype == torch.float32, "head_unpatchify: fp32 stream, or bf16 patch embedding + fp32 residual"
    if prep is None:
        prep = head_prepare(head_mod, e, w_t, b)
    assert prep.cols == cols
    if out is None:
        assert rows == F * Hp * Wp, "a partial token range needs a caller-provided output"
        out = torch.empty(c_out, F, 2 * Hp, 2 * Wp, dtype=torch.float32, device=x.device)
    ptrs = [out.data_ptr()] + [int(p) for p in (peer_outs or [])]
    arr = (ctypes.c_void_p * len(ptrs))(*ptrs)
    rptr = residual.data_ptr() if residual is not None else None
    with _Timed(tag, "head"):
        if step is None:
            check(lib.mc_head_unpatchify_ex(x.data_ptr(), _dt(x), rptr, rows, row_offset, cols, F, Hp, Wp, c_out, eps, arr, len(ptrs), prep.ptr,
                                            prep.nbytes, 1 if round_sum_to_bf16 else 0, _stream()))
        else:
            cond, x_lat, g, cx, cv = step
            for t_ in (cond, x_lat):
                assert t_.dtype == torch.float32 and t_.is_contiguous() and t_.numel() == out.numel() and t_.device == x.device
            check(lib.mc_head_unpatchify_step(x.data_ptr(), _dt(x), rptr, rows, row_offset, cols, F, Hp, Wp, c_out, eps, arr, len(ptrs), prep.ptr,
                                              prep.nbytes, 1 if round_sum_to_bf16 else 0, cond.data_ptr(), x_lat.data_ptr(), float(g), float(cx),
                                              float(cv), _stream()))
    _count()
    return out


def transpose(src, out):
    """out[c, r] = src[r, c] for bf16 2-D views (row strides allowed)."""
    _dev(src), _dev(out)
    assert src.dtype == out.dtype == torch.bfloat16 and src.stride(1) == 1 and out.stride(1) == 1
    rows, cols = src.shape
    assert out.shape == (cols, rows)
    check(lib.mc_transpose_bf16(src.data_ptr(), src.stride(0), rows, cols, out.data_ptr(), out.stride(0), _stream()))
    _count()
    return out


def cast(src, dtype):
    _dev(src)
    assert src.is_contiguous()
    dst = torch.empty(src.shape, dtype=dtype, device=src.device)
    check(lib.mc_cast(src.data_ptr(), _dt(src), dst.data_ptr(), _dt(dst), src.numel(), _stream()))
    _count()
    return dst


def cast_into(src, dst, tag=None):
    """dst[...] = src converted (bf16 <-> fp32), no allocation."""
    _dev(src), _dev(dst)
    assert src.is_contiguous() and dst.is_contiguous() and src.numel() == dst.numel()
    with _Timed(tag, "cast"):
        check(lib.mc_cast(src.data_ptr(), _dt(src), dst.data_ptr(), _dt(dst), src.numel(), _stream()))
    _count()
    return dst
