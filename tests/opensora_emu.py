"""CPU emulation of the Open-Sora ops (magcache_b200.ops: ln_t2i_modulate, rmsnorm_head72_rope_, attention_varlen_d72,
attention_temporal_d72) with the rounding points include/magcache_b200.h documents, on top of tests/emu_ops.py. `namespace()` is a
drop-in for `magcache_b200.opensora.ops`, so the engine's orchestration runs on CPU against the oracle."""
import math
import types

import torch
import torch.nn.functional as F

import emu_ops as E

BF, F32 = torch.bfloat16, torch.float32
_rb = E._rb


def ln_t2i_modulate(x, em, scale_idx, shift_idx, eps=1e-6, out=None, tag=None):
    assert x.dtype == BF and x.is_contiguous() and em.dtype == F32
    y = _rb(F.layer_norm(x.to(F32), (x.shape[-1],), None, None, eps))
    o = _rb(_rb(y * _rb(1.0 + em[scale_idx])) + em[shift_idx]).to(BF)
    if out is None:
        return o
    out.copy_(o)
    return out


def rmsnorm_head72_rope_(x, weight, heads, cos_sin=None, pos_div=1, eps=1e-6, tag=None):
    assert x.dtype == BF and x.stride(1) == 1 and x.shape[1] == heads * 72 and weight.numel() == 72
    rows = x.shape[0]
    v = x.to(F32).view(rows, heads, 72)
    o = _rb(_rb(v * torch.rsqrt(v.pow(2).mean(-1, keepdim=True) + eps)) * weight)
    if cos_sin is not None:
        pos = (torch.arange(rows) // pos_div) % cos_sin.shape[0]
        cs = cos_sin[pos].view(rows, 1, 36, 2)
        re, im = o.view(rows, heads, 36, 2).unbind(-1)
        c, s = cs[..., 0], cs[..., 1]
        o = torch.stack([re * c - im * s, im * c + re * s], dim=-1).view(rows, heads, 72)
    x.copy_(o.reshape(rows, heads * 72))
    return x


def _attn(q, k, v, heads, scale):
    qh = q.to(F32).reshape(q.shape[0], heads, 72).transpose(0, 1)
    kh = k.to(F32).reshape(k.shape[0], heads, 72).transpose(0, 1)
    vh = v.to(F32).reshape(v.shape[0], heads, 72).transpose(0, 1)
    return (torch.softmax(qh @ kh.transpose(1, 2) * scale, -1) @ vh).transpose(0, 1).reshape(q.shape[0], heads * 72)


def attention_varlen_d72(q, k, v, heads, segs, max_q_len, scale=None, out=None, tag=None):
    assert segs.dtype == torch.int32 and segs.shape[1] == 4 and q.stride(1) == 1 and k.stride(1) == 1 and v.stride(1) == 1
    scale = 1.0 / math.sqrt(72) if scale is None else scale
    if out is None:
        out = torch.empty(q.shape[0], heads * 72, dtype=BF)
    for qs, ql, ks, kl in segs.tolist():
        assert 1 <= kl and ql <= max_q_len
        out[qs:qs + ql] = _attn(q[qs:qs + ql], k[ks:ks + kl], v[ks:ks + kl], heads, scale).to(BF)
    return out


def attention_temporal_d72(q, k, v, heads, B, T, S, scale=None, out=None, tag=None):
    assert T <= 32 and q.shape == (B * T * S, heads * 72)
    scale = 1.0 / math.sqrt(72) if scale is None else scale
    if out is None:
        out = torch.empty(q.shape[0], heads * 72, dtype=BF)
    seq = lambda t: t.to(F32).view(B, T, S, heads, 72).permute(0, 2, 3, 1, 4)  # noqa: E731  [B, S, H, T, 72]
    o = torch.softmax(seq(q) @ seq(k).transpose(-1, -2) * scale, -1) @ seq(v)
    out.copy_(o.permute(0, 3, 1, 2, 4).reshape(B * T * S, heads * 72).to(BF))
    return out


def namespace():
    ns = types.SimpleNamespace(**{n: getattr(E, n) for n in dir(E) if not n.startswith("__")})
    for f in (ln_t2i_modulate, rmsnorm_head72_rope_, attention_varlen_d72, attention_temporal_d72):
        setattr(ns, f.__name__, f)
    return ns
