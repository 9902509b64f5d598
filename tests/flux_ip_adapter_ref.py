"""IP-Adapter image prompts for the FLUX tests: diffusers' modules restated under their attribute names, their loading into the
oracle's FluxTransformer2DModel, the reference's statements around the oracle's forward, and `ops.cast` / `ops.ip_attention` in the kernel emulation.

diffusers is not part of this project and the block-level statements sit outside the reference tree (parity unpinned, like
oracle/flux_ref.py). Restated from the current diffusers form:
  - `ImageProjection`: image_embeds Linear(emb_dim -> T*C), `norm` LayerNorm(C) (eps 1e-5); forward LayerNorm(Linear(x).reshape(B, T, C)).
  - `MultiIPAdapterImageProjection`: one ImageProjection per adapter in `image_projection_layers`; embeds [B, num_images, emb_dim]
    per adapter become [B, num_images, T, C].
  - `FluxIPAdapterAttnProcessor` (`to_k_ip`, `to_v_ip`: ModuleLists of Linear(C -> D); `scale`: one float per adapter): in a
    double block, ip_query = the image stream's q after norm_q (before the text rows and RoPE), and
    ip_attn_output = zeros_like(hidden_states); ip_attn_output += scale[a] * SDPA(ip_query, to_k_ip[a](ip_h[a]), to_v_ip[a](ip_h[a]))
    per adapter, all in the stream's dtype.
  - `FluxTransformerBlock`: `hidden_states = hidden_states + ip_attn_output` after the feed-forward residual.
The forward's own statements are the reference's: MagCache4FLUX/magcache_flux.py:321-324 (calibration :108-111; Kontext
magcache_flux_kontext.py:323-326, :110-113) pop the embeds from a copy of joint_attention_kwargs and project them on every call."""
import contextlib
import math
import types

import torch
import torch.nn.functional as F
from torch import nn

import emu_ops
import flux_controlnet_ref as cref
import flux_lora_ref as lref


class ImageProjection(nn.Module):
    def __init__(self, image_embed_dim, cross_attention_dim, num_image_text_embeds):
        super().__init__()
        self.num_image_text_embeds, self.cross_attention_dim = num_image_text_embeds, cross_attention_dim
        self.image_embeds = nn.Linear(image_embed_dim, num_image_text_embeds * cross_attention_dim)
        self.norm = nn.LayerNorm(cross_attention_dim)

    def forward(self, image_embeds):
        b = image_embeds.shape[0]
        x = self.image_embeds(image_embeds.to(self.image_embeds.weight.dtype))
        return self.norm(x.reshape(b, self.num_image_text_embeds, -1))


class MultiIPAdapterImageProjection(nn.Module):
    def __init__(self, layers):
        super().__init__()
        self.image_projection_layers = nn.ModuleList(layers)

    def forward(self, image_embeds):
        out = []
        for e, layer in zip(image_embeds, self.image_projection_layers):
            b, n = e.shape[0], e.shape[1]
            y = layer(e.reshape((b * n,) + e.shape[2:]))
            out.append(y.reshape((b, n) + y.shape[1:]))
        return out


class FluxIPAdapterAttnProcessor(nn.Module):
    def __init__(self, hidden_size, cross_attention_dim, num_tokens=(4,), scale=1.0):
        super().__init__()
        self.num_tokens = list(num_tokens)
        self.scale = scale if isinstance(scale, list) else [scale] * len(self.num_tokens)
        self.to_k_ip = nn.ModuleList([nn.Linear(cross_attention_dim, hidden_size) for _ in self.num_tokens])
        self.to_v_ip = nn.ModuleList([nn.Linear(cross_attention_dim, hidden_size) for _ in self.num_tokens])


class FluxAttnProcessor:
    """The plain processor diffusers leaves on single blocks (not a Module)."""


def load_ip_adapter(model, n_adapters=1, T=16, emb_dim=32, C=64, seed=0, blocks=None):
    """What `pipe.load_ip_adapter(...)` leaves on the transformer: `encoder_hid_proj` and an IP-Adapter processor on every double
    block (`blocks`: only these indices), seeded weights in the model's dtype (bf16)."""
    g = torch.Generator().manual_seed(seed)
    D = model.inner_dim
    T = T if isinstance(T, (list, tuple)) else [T] * n_adapters
    proj = MultiIPAdapterImageProjection([ImageProjection(emb_dim, C, t) for t in T])
    for i, blk in enumerate(model.transformer_blocks):
        if blocks is None or i in blocks:
            blk.attn.processor = FluxIPAdapterAttnProcessor(D, C, T, 1.0)
    for blk in model.single_transformer_blocks:
        blk.attn.processor = FluxAttnProcessor()
    model.encoder_hid_proj = proj
    with torch.no_grad():
        for name, p in list(proj.named_parameters()) + [(n, p) for n, p in model.named_parameters() if "_ip." in n]:
            if name.endswith("bias"):
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            elif p.dim() == 1:
                p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(torch.randn(p.shape, generator=g) / p.shape[1] ** 0.5)
    model.to(next(model.parameters()).dtype)
    return model


def unload_ip_adapter(model):
    """diffusers `unload_ip_adapter`: no image projection, the default processor back on every block."""
    model.encoder_hid_proj = None
    for blk in list(model.transformer_blocks) + list(model.single_transformer_blocks):
        if "processor" in blk.attn._modules:
            del blk.attn._modules["processor"]
        blk.attn.processor = FluxAttnProcessor()


def set_ip_adapter_scale(model, scale):
    """diffusers `set_ip_adapter_scale` on the transformer: one value for every block, or a list with one value per double block;
    each value goes to every adapter."""
    procs = [b.attn.processor for b in model.transformer_blocks if isinstance(getattr(b.attn, "processor", None), FluxIPAdapterAttnProcessor)]
    scales = scale if isinstance(scale, list) else [scale] * len(procs)
    for p, s in zip(procs, scales):
        p.scale = list(s) if isinstance(s, (list, tuple)) else [s] * len(p.to_k_ip)


def make_embeds(n_adapters=1, n_images=1, emb_dim=32, seed=0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed + 101)
    return [torch.randn(1, n_images, emb_dim, generator=g).to(dtype) for _ in range(n_adapters)]


class _DoubleWithIP(nn.Module):
    """A double block with its processor's image-prompt attention added after the block's feed-forward residual."""

    def __init__(self, block, ip_hidden_states):
        super().__init__()
        self.block, self.ip_hidden_states = block, ip_hidden_states

    def forward(self, hidden_states, encoder_hidden_states, temb, image_rotary_emb=None, joint_attention_kwargs=None):
        blk, sample = self.block, None
        if isinstance(blk, cref._DoubleThenAdd):  # ControlNet around the block: its sample is added after the image prompt
            blk, sample = blk.block, blk.sample
        a, proc = blk.attn, getattr(blk.attn, "processor", None)
        if not isinstance(proc, FluxIPAdapterAttnProcessor):
            return self.block(hidden_states=hidden_states, encoder_hidden_states=encoder_hidden_states, temb=temb,
                              image_rotary_emb=image_rotary_emb)
        b, h = hidden_states.shape[0], a.heads
        n = blk.norm1(hidden_states, temb)[0]  # the block's own LN+modulate of the image stream: the same bits as inside it
        ip_query = a.norm_q(a.to_q(n).view(b, -1, h, 128).transpose(1, 2))
        ip_attn_output = torch.zeros_like(hidden_states)
        for ip_h, scale, to_k_ip, to_v_ip in zip(self.ip_hidden_states, proc.scale, proc.to_k_ip, proc.to_v_ip):
            k = to_k_ip(ip_h).view(b, -1, h, 128).transpose(1, 2)
            v = to_v_ip(ip_h).view(b, -1, h, 128).transpose(1, 2)
            o = F.scaled_dot_product_attention(ip_query, k, v)
            o = o.transpose(1, 2).reshape(b, -1, h * 128).to(ip_query.dtype)
            ip_attn_output += scale * o
        encoder_hidden_states, hidden_states = blk(hidden_states=hidden_states, encoder_hidden_states=encoder_hidden_states, temb=temb,
                                                   image_rotary_emb=image_rotary_emb)
        hidden_states = hidden_states + ip_attn_output
        if sample is not None:
            hidden_states = hidden_states + sample
        return encoder_hidden_states, hidden_states


@contextlib.contextmanager
def _ip_blocks(model, ip_hidden_states):
    double = model.transformer_blocks
    model.transformer_blocks = nn.ModuleList([_DoubleWithIP(b, ip_hidden_states) for b in double])
    try:
        yield
    finally:
        model.transformer_blocks = double


def reference_ip(inner):
    """The oracle's forward (or calibration twin, or one already wrapped by flux_lora_ref.reference_lora) `inner` with the
    reference's ip-adapter statements: the embeds are popped from a copy of joint_attention_kwargs and projected on every call."""

    def forward(self, *args, joint_attention_kwargs=None, **kw):
        if joint_attention_kwargs is not None and "ip_adapter_image_embeds" in joint_attention_kwargs:
            joint_attention_kwargs = joint_attention_kwargs.copy()
            ip_hidden_states = self.encoder_hid_proj(joint_attention_kwargs.pop("ip_adapter_image_embeds"))
            with _ip_blocks(self, ip_hidden_states):
                return inner(self, *args, joint_attention_kwargs=joint_attention_kwargs, **kw)
        return inner(self, *args, joint_attention_kwargs=joint_attention_kwargs, **kw)

    return forward


def cast(src, dtype):
    assert src.is_contiguous()
    return src.to(dtype)


def ip_attention(q, weight, heads, kv, n_keys, scales, out=None, eps=1e-6, tag=None):
    """`mc_ip_attn` in torch: the per-head RMSNorm of emu_ops.rmsnorm_head_rope_ on the raw q (no RoPE), then per adapter, in
    order, acc = bf16(acc + bf16(s_a * bf16(softmax(qn K_a^T / sqrt(128)) V_a))) from +0 (P unrounded, fp32)."""
    BF, F32 = torch.bfloat16, torch.float32
    rows, W = q.shape
    assert W == heads * 128 and q.stride(1) == 1 and q.stride(0) % 8 == 0 and q.data_ptr() % 16 == 0
    assert kv.stride(1) == 1 and kv.stride(0) % 8 == 0 and kv.data_ptr() % 16 == 0
    assert len(n_keys) == len(scales) >= 1 and kv.shape[0] == sum(n_keys) and kv.shape[1] >= 2 * W
    assert out is None or (out.shape == q.shape and out.stride(1) == 1 and out.stride(0) % 8 == 0 and out.data_ptr() % 16 == 0)
    qn = q.clone()
    emu_ops.rmsnorm_head_rope_(qn, weight, heads, None, eps)
    emu_ops.LAUNCHES -= 1  # one launch in all, counted below
    qh = qn.to(F32).view(rows, heads, 128).transpose(0, 1)
    acc, k0 = torch.zeros(rows, W, dtype=BF), 0
    for n, s in zip(n_keys, scales):
        k = kv[k0:k0 + n, :W].to(F32).view(n, heads, 128).transpose(0, 1)
        v = kv[k0:k0 + n, W:2 * W].to(F32).view(n, heads, 128).transpose(0, 1)
        o = (torch.softmax(qh @ k.transpose(1, 2) / math.sqrt(128), -1) @ v).transpose(0, 1).reshape(rows, W).to(BF)
        acc = (acc.to(F32) + (torch.tensor(s, dtype=F32) * o.to(F32)).to(BF).to(F32)).to(BF)
        k0 += n
    if out is None:
        out = torch.empty(rows, W, dtype=BF)
    out.copy_(acc)
    emu_ops._count()
    return out


emu = types.ModuleType("emu_ops_ip_adapter")
emu.__dict__.update({k: v for k, v in vars(lref.emu).items() if not k.startswith("__")})
emu.cast = cast
emu.ip_attention = ip_attention
