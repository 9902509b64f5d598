"""CPU-or-GPU restatement of Open-Sora 1.2's STDiT3 under the reference's module tree and parameter names
(videosys/models/transformers/open_sora_transformer_3d.py, videosys/models/modules/{attentions,embeddings,normalization}.py) and of
the paper-evaluation MagCache forward that drives it (eval/magcache/experiments/opensora.py:229-373, installed by `eval_ours`,
:411-437). Used by the tests and tools only; it runs in whatever dtype the module is cast to (fp64 for the accuracy yardstick, bf16
for the reference's own rounding).

Stand-ins for what the reference imports from outside its tree: timm's `Mlp` (fc1 -> act -> fc2) and `DropPath` (identity at
drop_path 0), `rotary_embedding_torch.RotaryEmbedding(dim).rotate_queries_or_keys` [EXT] (interleaved pairs, theta 10000,
position = index along the sequence axis), a parallel manager with sp = cp = 1, PAB off. Attention is torch SDPA; the
cross-attention follows `flash_attn_varlen_func` (each sample attends to its own `y_lens[b]` caption tokens), which equals the
default `torch_impl` (attentions.py:155-166) whenever all samples have the same length."""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

CONFIGS = {
    # STDiT3-XL/2 (hpcai-tech/OpenSora-STDiT-v3)
    "full": dict(hidden_size=1152, depth=28, num_heads=16, caption_channels=4096, model_max_length=300),
    "tiny": dict(hidden_size=144, depth=2, num_heads=2, caption_channels=64, model_max_length=12),
    "wide": dict(hidden_size=1152, depth=1, num_heads=16, caption_channels=256, model_max_length=20),
}

# eval/magcache/experiments/opensora.py:433 (before the `** 0.5`)
OPENSORA_RATIO = [0.93359, 0.96484, 0.99609, 1.0, 0.99609, 0.99609, 0.99219, 1.0, 1.0, 0.99609, 0.99219, 1.0, 0.99219, 0.99609, 0.99219,
                  0.99609, 0.99609, 0.99609, 0.99219, 0.99219, 0.99219, 0.98828, 0.98828, 0.98438, 0.98438, 0.97656, 0.97656, 0.96484, 0.96484]


def synthetic_state(shapes, seed):
    """name -> fp32 tensor for a {parameter name: shape} dict, drawn in sorted-name order from one seeded generator (so any module
    with the reference's parameter names gets the same weights): norm weights 1 + 0.2 N(0, 1), matrices N(0, 1 / fan_in), vectors
    0.1 N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name in sorted(shapes):
        shape = tuple(shapes[name])
        if name.endswith("norm.weight"):
            out[name] = 1.0 + 0.2 * torch.randn(shape, generator=g)
        elif len(shape) >= 2:
            out[name] = torch.randn(shape, generator=g) / math.sqrt(int(np.prod(shape[1:])))
        else:
            out[name] = 0.1 * torch.randn(shape, generator=g)
    return out


def t2i_modulate(x, shift, scale):
    return x * (1 + scale) + shift


class Mlp(nn.Module):  # timm.models.vision_transformer.Mlp with drop=0
    def __init__(self, in_features, hidden_features, out_features=None):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = nn.GELU(approximate="tanh")
        self.fc2 = nn.Linear(hidden_features, out_features or in_features)

    def forward(self, x):
        return self.fc2(self.act(self.fc1(x)))


class LlamaRMSNorm(nn.Module):  # normalization.py:8-22
    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, hidden_states):
        input_dtype = hidden_states.dtype
        hidden_states = hidden_states.to(torch.float32)
        variance = hidden_states.pow(2).mean(-1, keepdim=True)
        hidden_states = hidden_states * torch.rsqrt(variance + self.variance_epsilon)
        return self.weight * hidden_states.to(input_dtype)


class RotaryEmbedding(nn.Module):
    """rotary_embedding_torch.RotaryEmbedding(dim) [EXT] as STDiT3 uses it: `rotate_queries_or_keys(t)` on [..., seq, dim] with
    interleaved pairs; freqs fp32, applied in fp32 (`t * cos + rotate_half(t) * sin`), result cast back to t's dtype."""

    def __init__(self, dim, theta=10000):
        super().__init__()
        self.dim, self.theta = dim, theta

    def rotate_queries_or_keys(self, t):
        ct = torch.float64 if t.dtype == torch.float64 else torch.float32  # the library's fp32 freqs (fp64 for the yardstick)
        inv = 1.0 / (self.theta ** (torch.arange(0, self.dim, 2, device=t.device)[: self.dim // 2].to(ct) / self.dim))
        pos = torch.arange(t.shape[-2], device=t.device, dtype=ct)
        freqs = torch.einsum("i,f->if", pos, inv).repeat_interleave(2, dim=-1)
        x = t.to(ct)
        x1, x2 = x.unflatten(-1, (-1, 2)).unbind(-1)
        rot = torch.stack((-x2, x1), dim=-1).flatten(-2)
        out = x * freqs.cos() + rot * freqs.sin()
        return out.type(t.dtype)


class OpenSoraAttention(nn.Module):  # attentions.py:21-100 (SDPA path, qk_norm_legacy=False)
    def __init__(self, dim, num_heads, qkv_bias=True, qk_norm=True, rope=None):
        super().__init__()
        self.num_heads, self.head_dim = num_heads, dim // num_heads
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.q_norm = LlamaRMSNorm(self.head_dim) if qk_norm else nn.Identity()
        self.k_norm = LlamaRMSNorm(self.head_dim) if qk_norm else nn.Identity()
        self.proj = nn.Linear(dim, dim)
        self.rope = rope is not None
        self.rotary_emb = rope

    def forward(self, x):
        B, N, C = x.shape
        qkv = self.qkv(x).view(B, N, 3, self.num_heads, self.head_dim).permute(2, 0, 3, 1, 4)
        q, k, v = qkv.unbind(0)
        q, k = self.q_norm(q), self.k_norm(k)
        if self.rope:
            q = self.rotary_emb(q)
            k = self.rotary_emb(k)
        x = F.scaled_dot_product_attention(q, k, v)
        return self.proj(x.transpose(1, 2).reshape(B, N, C))


class OpenSoraMultiHeadCrossAttention(nn.Module):  # attentions.py:103-153 (varlen semantics)
    def __init__(self, d_model, num_heads):
        super().__init__()
        self.num_heads, self.head_dim = num_heads, d_model // num_heads
        self.q_linear = nn.Linear(d_model, d_model)
        self.kv_linear = nn.Linear(d_model, d_model * 2)
        self.proj = nn.Linear(d_model, d_model)

    def forward(self, x, cond, mask=None):
        B, N, C = x.shape
        q = self.q_linear(x).view(B, N, self.num_heads, self.head_dim)
        kv = self.kv_linear(cond).view(-1, 2, self.num_heads, self.head_dim)
        k, v = kv.unbind(1)
        outs, k0 = [], 0
        for b in range(B):
            n = int(mask[b])
            qb = q[b].transpose(0, 1)[None]
            kb, vb = k[k0:k0 + n].transpose(0, 1)[None], v[k0:k0 + n].transpose(0, 1)[None]
            outs.append(F.scaled_dot_product_attention(qb, kb, vb)[0].transpose(0, 1).reshape(N, C))
            k0 += n
        return self.proj(torch.stack(outs))


class STDiT3Block(nn.Module):  # open_sora_transformer_3d.py:98-273 with x_mask = None, PAB off, sp = 1
    def __init__(self, hidden_size, num_heads, mlp_ratio=4.0, rope=None, qk_norm=True, temporal=False):
        super().__init__()
        self.temporal = temporal
        self.norm1 = nn.LayerNorm(hidden_size, eps=1e-6, elementwise_affine=False)
        self.attn = OpenSoraAttention(hidden_size, num_heads, qkv_bias=True, qk_norm=qk_norm, rope=rope)
        self.cross_attn = OpenSoraMultiHeadCrossAttention(hidden_size, num_heads)
        self.norm2 = nn.LayerNorm(hidden_size, eps=1e-6, elementwise_affine=False)
        self.mlp = Mlp(hidden_size, int(hidden_size * mlp_ratio))
        self.scale_shift_table = nn.Parameter(torch.randn(6, hidden_size) / hidden_size ** 0.5)

    def forward(self, x, y, t, mask=None, T=None, S=None):
        B, N, C = x.shape
        shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = (self.scale_shift_table[None] + t.reshape(B, 6, -1)).chunk(6, dim=1)
        x_m = t2i_modulate(self.norm1(x), shift_msa, scale_msa)
        if self.temporal:
            x_m = x_m.view(B, T, S, C).transpose(1, 2).reshape(B * S, T, C)
            x_m = self.attn(x_m)
            x_m = x_m.view(B, S, T, C).transpose(1, 2).reshape(B, T * S, C)
        else:
            x_m = self.attn(x_m.reshape(B * T, S, C)).reshape(B, T * S, C)
        x = x + gate_msa * x_m
        x = x + self.cross_attn(x, y, mask)
        x_m = t2i_modulate(self.norm2(x), shift_mlp, scale_mlp)
        x = x + gate_mlp * self.mlp(x_m)
        return x


class TimestepEmbedder(nn.Module):  # embeddings.py:107-146
    def __init__(self, hidden_size, frequency_embedding_size=256):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(frequency_embedding_size, hidden_size), nn.SiLU(), nn.Linear(hidden_size, hidden_size))
        self.frequency_embedding_size = frequency_embedding_size

    @staticmethod
    def timestep_embedding(t, dim, max_period=10000):
        half = dim // 2
        freqs = torch.exp(-math.log(max_period) * torch.arange(start=0, end=half, dtype=torch.float32) / half).to(device=t.device)
        args = t[:, None].float() * freqs[None]
        return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)

    def forward(self, t, dtype):
        t_freq = self.timestep_embedding(t, self.frequency_embedding_size)
        return self.mlp(t_freq.to(dtype))


class SizeEmbedder(TimestepEmbedder):  # embeddings.py:149-180
    def forward(self, s, bs):
        if s.ndim == 1:
            s = s[:, None]
        if s.shape[0] != bs:
            s = s.repeat(bs // s.shape[0], 1)
        b, dims = s.shape[0], s.shape[1]
        s_freq = self.timestep_embedding(s.reshape(-1), self.frequency_embedding_size).to(next(self.parameters()).dtype)
        return self.mlp(s_freq).reshape(b, dims * self.mlp[2].out_features)


class OpenSoraCaptionEmbedder(nn.Module):  # embeddings.py:183-228 (inference: no token drop)
    def __init__(self, in_channels, hidden_size, token_num):
        super().__init__()
        self.y_proj = Mlp(in_channels, hidden_size, hidden_size)
        self.register_buffer("y_embedding", torch.randn(token_num, in_channels) / in_channels ** 0.5)

    def forward(self, caption):
        return self.y_proj(caption)


class OpenSoraPositionEmbedding2D(nn.Module):  # embeddings.py:231-280
    def __init__(self, dim):
        super().__init__()
        self.dim = dim

    def _get_sin_cos_emb(self, t):
        half_dim = self.dim // 2
        inv_freq = 1.0 / (10000 ** (torch.arange(0, half_dim, 2, device=t.device).to(t.dtype) / half_dim))
        out = torch.einsum("i,d->id", t, inv_freq)
        return torch.cat((torch.sin(out), torch.cos(out)), dim=-1)

    def forward(self, x, h, w, scale=1.0, base_size=None):
        grid_h = torch.arange(h, device=x.device) / scale
        grid_w = torch.arange(w, device=x.device) / scale
        if base_size is not None:
            grid_h *= base_size / h
            grid_w *= base_size / w
        grid_h, grid_w = torch.meshgrid(grid_w, grid_h, indexing="ij")
        grid_h = grid_h.t().reshape(-1)
        grid_w = grid_w.t().reshape(-1)
        ct = torch.float64 if x.dtype == torch.float64 else torch.float32
        emb_h = self._get_sin_cos_emb(grid_h.to(ct))
        emb_w = self._get_sin_cos_emb(grid_w.to(ct))
        return torch.concat([emb_h, emb_w], dim=-1).unsqueeze(0).to(x.dtype)


class T2IFinalLayer(nn.Module):  # open_sora_transformer_3d.py:50-86 with x_mask = None
    def __init__(self, hidden_size, num_patch, out_channels):
        super().__init__()
        self.norm_final = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.linear = nn.Linear(hidden_size, num_patch * out_channels, bias=True)
        self.scale_shift_table = nn.Parameter(torch.randn(2, hidden_size) / hidden_size ** 0.5)

    def forward(self, x, t):
        shift, scale = (self.scale_shift_table[None] + t[:, None]).chunk(2, dim=1)
        return self.linear(t2i_modulate(self.norm_final(x), shift, scale))


class _Proj(nn.Module):
    def __init__(self, cin, cout, patch):
        super().__init__()
        self.proj = nn.Conv3d(cin, cout, kernel_size=patch, stride=patch)


class STDiT3(nn.Module):
    def __init__(self, hidden_size=1152, depth=28, num_heads=16, mlp_ratio=4.0, in_channels=4, patch_size=(1, 2, 2), caption_channels=4096,
                 model_max_length=300, input_sq_size=512, pred_sigma=True):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, in_channels * 2 if pred_sigma else in_channels
        self.hidden_size, self.num_heads, self.depth, self.patch_size, self.input_sq_size = hidden_size, num_heads, depth, patch_size, input_sq_size
        self.pos_embed = OpenSoraPositionEmbedding2D(hidden_size)
        self.rope = RotaryEmbedding(dim=hidden_size // num_heads)
        self.x_embedder = _Proj(in_channels, hidden_size, patch_size)
        self.t_embedder = TimestepEmbedder(hidden_size)
        self.fps_embedder = SizeEmbedder(hidden_size)
        self.t_block = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 6 * hidden_size, bias=True))
        self.y_embedder = OpenSoraCaptionEmbedder(caption_channels, hidden_size, model_max_length)
        self.spatial_blocks = nn.ModuleList([STDiT3Block(hidden_size, num_heads, mlp_ratio) for _ in range(depth)])
        self.temporal_blocks = nn.ModuleList([STDiT3Block(hidden_size, num_heads, mlp_ratio, rope=self.rope.rotate_queries_or_keys, temporal=True)
                                              for _ in range(depth)])
        self.final_layer = T2IFinalLayer(hidden_size, int(np.prod(patch_size)), self.out_channels)

    def init_synthetic(self, seed):
        """Seeded weights with every path live (the reference zero-initialises the temporal output projections, :474-478)."""
        with torch.no_grad():
            for name, t in synthetic_state({n: p.shape for n, p in self.named_parameters()}, seed).items():
                dict(self.named_parameters())[name].copy_(t)
        return self

    def get_dynamic_size(self, x):
        _, _, T, H, W = x.size()
        p = self.patch_size
        T, H, W = -(-T // p[0]), -(-H // p[1]), -(-W // p[2])
        return T, H, W

    def encode_text(self, y, mask=None):  # :493-504
        y = self.y_embedder(y)
        if mask is not None:
            if mask.shape[0] != y.shape[0]:
                mask = mask.repeat(y.shape[0] // mask.shape[0], 1)
            mask = mask.squeeze(1).squeeze(1)
            y = y.squeeze(1).masked_select(mask.unsqueeze(-1) != 0).view(1, -1, self.hidden_size)
            y_lens = mask.sum(dim=1).tolist()
        else:
            y_lens = [y.shape[2]] * y.shape[0]
            y = y.squeeze(1).view(1, -1, self.hidden_size)
        return y, y_lens

    def embed(self, x, timestep, y, mask, fps, height, width):
        """Everything before the block stack (:243-293): returns (x, y, y_lens, t, t_mlp, (T, H, W, S), (Tx, Hx, Wx))."""
        dtype = self.x_embedder.proj.weight.dtype
        B = x.size(0)
        x, timestep, y = x.to(dtype), timestep.to(dtype), y.to(dtype)
        _, _, Tx, Hx, Wx = x.size()
        T, H, W = self.get_dynamic_size(x)
        S = H * W
        base_size = round(S ** 0.5)
        scale = (height[0].item() * width[0].item()) ** 0.5 / self.input_sq_size
        pos_emb = self.pos_embed(x, H, W, scale=scale, base_size=base_size)
        t = self.t_embedder(timestep, dtype=x.dtype)
        t = t + self.fps_embedder(fps.unsqueeze(1), B)
        t_mlp = self.t_block(t)
        y, y_lens = self.encode_text(y, mask)
        x = self.x_embedder.proj(x).flatten(2).transpose(1, 2)
        x = (x.view(B, T, S, -1) + pos_emb).view(B, T * S, -1)
        return x, y, y_lens, t, t_mlp, (T, H, W, S), (Tx, Hx, Wx)

    def blocks(self, x, y, t_mlp, y_lens, T, S):
        for sb, tb in zip(self.spatial_blocks, self.temporal_blocks):
            x = sb(x, y, t_mlp, y_lens, T, S)
            x = tb(x, y, t_mlp, y_lens, T, S)
        return x

    def head(self, x, t, T, H, W, Tx, Hx, Wx):
        x = self.final_layer(x, t)
        return self.unpatchify(x, T, H, W, Tx, Hx, Wx).to(torch.float32)

    def unpatchify(self, x, N_t, N_h, N_w, R_t, R_h, R_w):  # :623-647
        B = x.shape[0]
        T_p, H_p, W_p = self.patch_size
        x = x.view(B, N_t, N_h, N_w, T_p, H_p, W_p, self.out_channels).permute(0, 7, 1, 4, 2, 5, 3, 6)
        x = x.reshape(B, self.out_channels, N_t * T_p, N_h * H_p, N_w * W_p)
        return x[:, :, :R_t, :R_h, :R_w]

    def forward(self, x, timestep, all_timesteps, y, mask=None, x_mask=None, fps=None, height=None, width=None, **kwargs):  # :506-621
        x, y, y_lens, t, t_mlp, (T, H, W, S), (Tx, Hx, Wx) = self.embed(x, timestep, y, mask, fps, height, width)
        x = self.blocks(x, y, t_mlp, y_lens, T, S)
        return self.head(x, t, T, H, W, Tx, Hx, Wx)


def push_tensor_roll(cache, x):  # opensora.py: the depth-3 residual FIFO; the newest entry is [..., -1]
    return torch.cat([cache[..., 1:], x.unsqueeze(-1)], dim=-1)


def magcache_forward(self, x, timestep, all_timesteps, y, mask=None, x_mask=None, fps=None, height=None, width=None, **kwargs):
    """eval/magcache/experiments/opensora.py:229-373 (sp = cp = 1, x_mask = None)."""
    x, y, y_lens, t, t_mlp, (T, H, W, S), (Tx, Hx, Wx) = self.embed(x, timestep, y, mask, fps, height, width)
    cache_time = 0
    ori_x = x
    skip_forward = False
    if self.t >= self.skip_time:
        cur_scale = self.ratio[self.t - 1]
        self.accumulated_sim = self.accumulated_sim * cur_scale
        self.accumulated_steps += 1
        self.accumulated_err += 1 - self.accumulated_sim
        if self.accumulated_err <= self.magcache_thresh and self.accumulated_steps <= self.K:
            residual_x = self.residual_cache[..., -1]
            skip_forward = True
        else:
            self.accumulated_sim = 1.0
            self.accumulated_steps = 0
            self.accumulated_err = 0
    if skip_forward:
        x = x + residual_x
        self.skip_steps += 1
    else:
        x = self.blocks(x, y, t_mlp, y_lens, T, S)
        residual_x = x - ori_x
    if self.t >= cache_time:
        if self.residual_cache is None:
            self.residual_cache = torch.zeros((*x.shape, 3), device=x.device, dtype=x.dtype)
        self.residual_cache = push_tensor_roll(self.residual_cache, residual_x)
    self.t += 1
    if self.t >= 30:
        self.t = 0
        self.accumulated_sim = 1.0
        self.accumulated_steps = 0
        self.accumulated_err = 0
        self.skip_steps = 0
    self.last_skip = skip_forward
    return self.head(x, t, T, H, W, Tx, Hx, Wx)


def install_magcache(cls, thresh=0.12, K=3, skip_time=6):
    """The attribute block of `eval_ours` (opensora.py:418-433) on a class."""
    cls.forward = magcache_forward
    cls.magcache_thresh, cls.K, cls.skip_time = thresh, K, skip_time
    cls.t, cls.residual_cache, cls.accumulated_err, cls.accumulated_sim, cls.accumulated_steps, cls.skip_steps = 0, None, 0, 1, 0, 0
    cls.ratio = np.array(OPENSORA_RATIO) ** 0.5
    return cls

