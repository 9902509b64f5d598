"""ORACLE — test infrastructure only. CPU restatement of Qwen-Image's transformer and of the MagCache statements that drive it
(`magcache_forward`, `magcache_calibration`, `init_magcache`, `init_magcache_calibration` of MagCache4QwenImage/magcache_generate.py;
MagCache4QwenImageEdit/magcache_generate.py has the same four).

PARITY UNPINNED for the transformer: `QwenImageTransformer2DModel`, `QwenImageTransformerBlock`, `QwenDoubleStreamAttnProcessor2_0`,
`QwenEmbedRope`, `QwenTimestepProjEmbeddings` live in diffusers (restated here from diffusers 0.35.1, which is not installed and
which the reference does not pin), under diffusers' attribute names so that `QwenImageWeights.from_module` reads a real pipeline's
transformer the same way. The MagCache statements are pinned: tests/golden/make_qwen_image_golden.py runs the reference's own
functions on this model, and tests/test_qwen_image_cpu.py holds these restatements bit-equal to that fixture.

dtype rule of the Qwen scripts: the pipeline is loaded in bf16 and runs without autocast, so every tensor is bf16 and every torch op
rounds to bf16 (`DT`). `exact()` switches the same code to float64 (RoPE angles and the timestep sinusoid included).
"""
import math
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

DT = torch.bfloat16


class exact:
    """Evaluate the same network with no reduced-precision rounding (the point both implementations are measured against)."""

    def __enter__(self):
        global DT
        self._old, DT = DT, torch.float64

    def __exit__(self, *a):
        global DT
        DT = self._old


def _wide():
    return torch.float64 if DT == torch.float64 else torch.float32


# ----------------------------------------------------------------------------------------------- embeddings
def timestep_proj(timesteps, dim=256, max_period=10000, scale=1000):
    """Timesteps(256, flip_sin_to_cos=True, downscale_freq_shift=0, scale=1000): `scale * (t * exp(-ln(P) k / half))` in fp32,
    [cos | sin]."""
    half, wd = dim // 2, _wide()
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=wd, device=timesteps.device) / half)
    emb = scale * (timesteps[:, None].to(wd) * freqs[None, :])
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


class TimestepEmbedding(nn.Module):
    def __init__(self, in_channels, dim):
        super().__init__()
        self.linear_1, self.act, self.linear_2 = nn.Linear(in_channels, dim), nn.SiLU(), nn.Linear(dim, dim)

    def forward(self, x):
        return self.linear_2(self.act(self.linear_1(x)))


class QwenTimestepProjEmbeddings(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.timestep_embedder = TimestepEmbedding(256, dim)

    def forward(self, timestep, hidden_states):
        return self.timestep_embedder(timestep_proj(timestep).to(dtype=hidden_states.dtype))


def rope_angles(index, dim, theta=10000):
    """`torch.outer(index, 1 / theta ** (arange(0, dim, 2) / dim))`, fp32 like upstream (float64 under exact())."""
    wd = _wide()
    return torch.outer(index.to(wd), 1.0 / torch.pow(theta, torch.arange(0, dim, 2).to(wd).div(dim)))


class QwenEmbedRope(nn.Module):
    """scale_rope=True. Returns complex (vid_freqs [sum f*h*w, 64], txt_freqs [max(txt_seq_lens), 64])."""

    def __init__(self, theta=10000, axes_dim=(16, 56, 56)):
        super().__init__()
        self.theta, self.axes_dim = theta, list(axes_dim)

    def _freqs(self, index):
        return torch.cat([torch.polar(torch.ones(len(index), d // 2, dtype=_wide()), rope_angles(index, d, self.theta))
                          for d in self.axes_dim], dim=1)

    def _video_freqs(self, frame, height, width, idx):
        pos = self._freqs(torch.arange(4096)).split([d // 2 for d in self.axes_dim], dim=1)
        neg = self._freqs(torch.arange(4096).flip(0) * -1 - 1).split([d // 2 for d in self.axes_dim], dim=1)
        f = pos[0][idx:idx + frame].view(frame, 1, 1, -1).expand(frame, height, width, -1)
        h = torch.cat([neg[1][-(height - height // 2):], pos[1][:height // 2]], dim=0).view(1, height, 1, -1).expand(frame, height, width, -1)
        w = torch.cat([neg[2][-(width - width // 2):], pos[2][:width // 2]], dim=0).view(1, 1, width, -1).expand(frame, height, width, -1)
        return torch.cat([f, h, w], dim=-1).reshape(frame * height * width, -1)

    def forward(self, video_fhw, txt_seq_lens, device=None):
        if isinstance(video_fhw, list):
            video_fhw = video_fhw[0]
        if not isinstance(video_fhw, list):
            video_fhw = [video_fhw]
        vid, m = [], 0
        for idx, (frame, height, width) in enumerate(video_fhw):
            vid.append(self._video_freqs(frame, height, width, idx))
            m = max(height // 2, width // 2, m)
        txt = self._freqs(torch.arange(4096))[m:m + max(txt_seq_lens)]
        return torch.cat(vid, dim=0), txt


def apply_rotary_emb_qwen(x, freqs_cis):
    """use_real=False: x [B, S, H, D] as complex (real, imag) pairs times freqs [S, D/2]."""
    xc = torch.view_as_complex(x.to(_wide()).reshape(*x.shape[:-1], -1, 2))
    return torch.view_as_real(xc * freqs_cis.to(x.device).unsqueeze(1)).flatten(3).type_as(x)


# ----------------------------------------------------------------------------------------------- norms, attention, blocks
class RMSNorm(nn.Module):
    def __init__(self, dim, eps=1e-6):
        super().__init__()
        self.eps, self.weight = eps, nn.Parameter(torch.ones(dim))

    def forward(self, h):
        variance = h.to(_wide()).pow(2).mean(-1, keepdim=True)
        h = h * torch.rsqrt(variance + self.eps)
        return h.to(self.weight.dtype) * self.weight


def _ln(x, eps=1e-6):
    return F.layer_norm(x, (x.shape[-1],), None, None, eps)


class Attention(nn.Module):
    """diffusers `Attention` as Qwen-Image configures it (added_kv_proj_dim=dim, qk_norm="rms_norm", bias=True) with
    QwenDoubleStreamAttnProcessor2_0 inlined: joint attention over [txt | img]."""

    def __init__(self, dim, heads, head_dim):
        super().__init__()
        self.heads = heads
        self.to_q, self.to_k, self.to_v = nn.Linear(dim, dim), nn.Linear(dim, dim), nn.Linear(dim, dim)
        self.add_q_proj, self.add_k_proj, self.add_v_proj = nn.Linear(dim, dim), nn.Linear(dim, dim), nn.Linear(dim, dim)
        self.norm_q, self.norm_k = RMSNorm(head_dim), RMSNorm(head_dim)
        self.norm_added_q, self.norm_added_k = RMSNorm(head_dim), RMSNorm(head_dim)
        self.to_out = nn.ModuleList([nn.Linear(dim, dim), nn.Dropout(0.0)])
        self.to_add_out = nn.Linear(dim, dim)

    def forward(self, hidden_states, encoder_hidden_states, image_rotary_emb):
        h = self.heads

        def split(t):
            return t.unflatten(-1, (h, -1))  # [B, S, H, D]

        q, k, v = split(self.to_q(hidden_states)), split(self.to_k(hidden_states)), split(self.to_v(hidden_states))
        tq, tk, tv = (split(p(encoder_hidden_states)) for p in (self.add_q_proj, self.add_k_proj, self.add_v_proj))
        q, k, tq, tk = self.norm_q(q), self.norm_k(k), self.norm_added_q(tq), self.norm_added_k(tk)
        img_freqs, txt_freqs = image_rotary_emb
        q, k = apply_rotary_emb_qwen(q, img_freqs), apply_rotary_emb_qwen(k, img_freqs)
        tq, tk = apply_rotary_emb_qwen(tq, txt_freqs), apply_rotary_emb_qwen(tk, txt_freqs)
        jq, jk, jv = (torch.cat([a, b], dim=1).transpose(1, 2) for a, b in ((tq, q), (tk, k), (tv, v)))
        o = F.scaled_dot_product_attention(jq, jk, jv).transpose(1, 2).flatten(2, 3).to(jq.dtype)
        n = encoder_hidden_states.shape[1]
        return self.to_out[0](o[:, n:]), self.to_add_out(o[:, :n])


class FeedForward(nn.Module):
    """FeedForward(dim, dim_out=dim, activation_fn="gelu-approximate"): net[0].proj, tanh GELU, net[2]."""

    def __init__(self, dim, mult=4):
        super().__init__()
        gelu = nn.Module()
        gelu.proj = nn.Linear(dim, dim * mult)
        self.net = nn.ModuleList([gelu, nn.Dropout(0.0), nn.Linear(dim * mult, dim)])

    def forward(self, x):
        return self.net[2](F.gelu(self.net[0].proj(x), approximate="tanh"))


def _modulate(x, mod_params):
    shift, scale, gate = mod_params.chunk(3, dim=-1)
    return x * (1 + scale.unsqueeze(1)) + shift.unsqueeze(1), gate.unsqueeze(1)


class QwenImageTransformerBlock(nn.Module):
    def __init__(self, dim, heads, head_dim):
        super().__init__()
        self.img_mod = nn.Sequential(nn.SiLU(), nn.Linear(dim, 6 * dim))
        self.txt_mod = nn.Sequential(nn.SiLU(), nn.Linear(dim, 6 * dim))
        self.attn = Attention(dim, heads, head_dim)
        self.img_mlp, self.txt_mlp = FeedForward(dim), FeedForward(dim)

    def forward(self, hidden_states, encoder_hidden_states, encoder_hidden_states_mask, temb, image_rotary_emb=None,
                joint_attention_kwargs=None):
        img_mod1, img_mod2 = self.img_mod(temb).chunk(2, dim=-1)
        txt_mod1, txt_mod2 = self.txt_mod(temb).chunk(2, dim=-1)
        img_m, img_gate1 = _modulate(_ln(hidden_states), img_mod1)
        txt_m, txt_gate1 = _modulate(_ln(encoder_hidden_states), txt_mod1)
        img_attn, txt_attn = self.attn(img_m, txt_m, image_rotary_emb)
        hidden_states = hidden_states + img_gate1 * img_attn
        encoder_hidden_states = encoder_hidden_states + txt_gate1 * txt_attn
        img_m2, img_gate2 = _modulate(_ln(hidden_states), img_mod2)
        hidden_states = hidden_states + img_gate2 * self.img_mlp(img_m2)
        txt_m2, txt_gate2 = _modulate(_ln(encoder_hidden_states), txt_mod2)
        encoder_hidden_states = encoder_hidden_states + txt_gate2 * self.txt_mlp(txt_m2)
        return encoder_hidden_states, hidden_states


class AdaLayerNormContinuous(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.silu, self.linear = nn.SiLU(), nn.Linear(dim, 2 * dim)

    def forward(self, x, cond):
        scale, shift = self.linear(self.silu(cond).to(x.dtype)).chunk(2, dim=1)  # scale FIRST
        return _ln(x) * (1 + scale)[:, None, :] + shift[:, None, :]


class QwenImageTransformer2DModel(nn.Module):
    """Attribute names and config of diffusers' QwenImageTransformer2DModel (Qwen-Image: 60 blocks, 24 heads x 128, text 3584)."""

    def __init__(self, patch_size=2, in_channels=64, out_channels=16, num_layers=60, attention_head_dim=128, num_attention_heads=24,
                 joint_attention_dim=3584, guidance_embeds=False, axes_dims_rope=(16, 56, 56)):
        super().__init__()
        dim = attention_head_dim * num_attention_heads
        self.config = types.SimpleNamespace(patch_size=patch_size, in_channels=in_channels, out_channels=out_channels,
                                            num_layers=num_layers, attention_head_dim=attention_head_dim,
                                            num_attention_heads=num_attention_heads, joint_attention_dim=joint_attention_dim,
                                            guidance_embeds=guidance_embeds, axes_dims_rope=tuple(axes_dims_rope))
        self.pos_embed = QwenEmbedRope(10000, axes_dims_rope)
        self.time_text_embed = QwenTimestepProjEmbeddings(dim)
        self.txt_norm = RMSNorm(joint_attention_dim, eps=1e-6)
        self.img_in, self.txt_in = nn.Linear(in_channels, dim), nn.Linear(joint_attention_dim, dim)
        self.transformer_blocks = nn.ModuleList([QwenImageTransformerBlock(dim, num_attention_heads, attention_head_dim)
                                                 for _ in range(num_layers)])
        self.norm_out = AdaLayerNormContinuous(dim)
        self.proj_out = nn.Linear(dim, patch_size * patch_size * out_channels)
        self.gradient_checkpointing = False

    @torch.no_grad()
    def init_synthetic(self, seed=0):
        """Seeded synthetic weights in bf16 (xavier-uniform matrices, modulation projections scaled down, non-zero biases and norm
        weights), drawn in place parameter by parameter (so a full-size model can be filled on the device)."""
        g = torch.Generator(device=next(self.parameters()).device).manual_seed(seed)
        for name, p in self.named_parameters():
            if p.dim() == 1 and "norm" in name and name.endswith("weight"):
                p.normal_(generator=g).mul_(0.1).add_(1.0)
            elif name.endswith("bias"):
                p.normal_(generator=g).mul_(0.02)
            else:
                a = math.sqrt(6.0 / (p.shape[0] + p.shape[1])) * (0.3 if ("_mod." in name or "norm_out" in name) else 1.0)
                p.uniform_(-a, a, generator=g)
        return self.to(torch.bfloat16)


# ----------------------------------------------------------------------------------------------- the MagCache statements
class Output:
    def __init__(self, sample):
        self.sample = sample


def _prologue(self, hidden_states, encoder_hidden_states, timestep, img_shapes, txt_seq_lens):
    hidden_states = self.img_in(hidden_states)
    timestep = timestep.to(hidden_states.dtype)
    encoder_hidden_states = self.txt_in(self.txt_norm(encoder_hidden_states))
    temb = self.time_text_embed(timestep, hidden_states)
    return hidden_states, encoder_hidden_states, temb, self.pos_embed(img_shapes, txt_seq_lens)


def _blocks(self, hidden_states, encoder_hidden_states, encoder_hidden_states_mask, temb, rope, attention_kwargs):
    for block in self.transformer_blocks:
        encoder_hidden_states, hidden_states = block(hidden_states, encoder_hidden_states, encoder_hidden_states_mask, temb, rope,
                                                     attention_kwargs)
    return hidden_states


def magcache_forward(self, hidden_states, encoder_hidden_states=None, encoder_hidden_states_mask=None, timestep=None, img_shapes=None,
                     txt_seq_lens=None, guidance=None, attention_kwargs=None, return_dict=True):
    """magcache_generate.py:173-252 (no guidance, no LoRA: the scripts' own case)."""
    hidden_states, encoder_hidden_states, temb, rope = _prologue(self, hidden_states, encoder_hidden_states, timestep, img_shapes,
                                                                 txt_seq_lens)
    b = self.cnt % 2
    skip = False
    if self.cnt >= int(self.num_steps * self.retention_ratio):                       # :205-219
        self.accumulated_ratio[b] *= self.mag_ratios[self.cnt]
        self.accumulated_steps[b] += 1
        self.accumulated_err[b] += np.abs(1 - self.accumulated_ratio[b])
        if self.accumulated_err[b] < self.magcache_thresh and self.accumulated_steps[b] <= self.K:
            skip, residual_x = True, self.residual_cache[b]
        else:
            self.accumulated_err[b], self.accumulated_steps[b], self.accumulated_ratio[b] = 0.0, 0, 1.0
    if skip:
        hidden_states += residual_x                                                    # :221-222, in place
    else:
        ori = hidden_states
        hidden_states = _blocks(self, hidden_states, encoder_hidden_states, encoder_hidden_states_mask, temb, rope, attention_kwargs)
        residual_x = hidden_states - ori
    self.residual_cache[b] = residual_x
    self.last_skip = skip  # (oracle-only bookkeeping for the tests)
    self.cnt += 1                                                                      # :242-244: counter only
    if self.cnt >= self.num_steps:
        self.cnt = 0
    output = self.proj_out(self.norm_out(hidden_states, temb))
    return Output(output) if return_dict else (output,)


def magcache_calibration(self, hidden_states, encoder_hidden_states=None, encoder_hidden_states_mask=None, timestep=None,
                         img_shapes=None, txt_seq_lens=None, guidance=None, attention_kwargs=None, return_dict=True):
    """magcache_generate.py:94-171: statistics from cnt >= 2 against the same branch's residual, as bf16 tensor ops."""
    hidden_states, encoder_hidden_states, temb, rope = _prologue(self, hidden_states, encoder_hidden_states, timestep, img_shapes,
                                                                 txt_seq_lens)
    ori = hidden_states
    hidden_states = _blocks(self, hidden_states, encoder_hidden_states, encoder_hidden_states_mask, temb, rope, attention_kwargs)
    residual_x = hidden_states - ori
    if self.cnt >= 2:
        prev = self.residual_cache[self.cnt % 2]
        ratio = residual_x.norm(dim=-1) / prev.norm(dim=-1)
        norm_ratio, norm_std = ratio.mean().item(), ratio.std().item()
        cos_dis = (1 - F.cosine_similarity(residual_x, prev, dim=-1, eps=1e-8)).mean().item()
        self.norm_ratio.append(round(norm_ratio, 5))
        self.norm_std.append(round(norm_std, 5))
        self.cos_dis.append(round(cos_dis, 5))
        print(f"Step {self.cnt}: norm_ratio={norm_ratio:.5f}, norm_std={norm_std:.5f}, cos_dis={cos_dis:.5f}")
    self.residual_cache[self.cnt % 2] = residual_x
    self.cnt += 1
    if self.cnt >= self.num_steps:                                                     # :158-163: lists printed, not cleared
        self.cnt = 0
        print("\nCalibration Results:")
        print("norm_ratio:", self.norm_ratio)
        print("norm_std:", self.norm_std)
        print("cos_dis:", self.cos_dis)
    output = self.proj_out(self.norm_out(hidden_states, temb))
    return Output(output) if return_dict else (output,)


def nearest_interp(original, target_length):
    if len(original) == target_length:
        return original.copy()
    return original[np.round(np.linspace(0, len(original) - 1, target_length)).astype(int)]


def init_magcache(model, mag_ratios, sample_steps, thresh=0.06, K=2, retention_ratio=0.2):
    """magcache_generate.py:63-83 with the argparse values as arguments."""
    cls = model.__class__
    cls.forward = magcache_forward
    cls.cnt = torch.tensor(0)
    cls.num_steps = sample_steps * 2
    cls.split_step, cls.mode = None, "t2v"
    cls.magcache_thresh, cls.K = thresh, K
    cls.accumulated_err, cls.accumulated_steps, cls.accumulated_ratio = [0.0, 0.0], [0, 0], [1.0, 1.0]
    cls.retention_ratio = retention_ratio
    cls.residual_cache = [None, None]
    cls.mag_ratios = np.array([1.0] * 2 + list(mag_ratios))
    if len(cls.mag_ratios) != sample_steps * 2:
        con, ucon = nearest_interp(cls.mag_ratios[0::2], sample_steps), nearest_interp(cls.mag_ratios[1::2], sample_steps)
        cls.mag_ratios = np.concatenate([con.reshape(-1, 1), ucon.reshape(-1, 1)], axis=1).flatten()


def init_magcache_calibration(model, sample_steps):
    cls = model.__class__
    cls.forward = magcache_calibration
    cls.cnt = torch.tensor(0)
    cls.num_steps = sample_steps * 2
    cls.norm_ratio, cls.norm_std, cls.cos_dis = [], [], []
    cls.residual_cache = [None, None]


# ----------------------------------------------------------------------------------------------- shared test inputs
TINY = dict(in_channels=16, out_channels=4, num_layers=2, num_attention_heads=2, joint_attention_dim=96)


def tiny_model(seed=0, **kw):
    return QwenImageTransformer2DModel(**{**TINY, **kw}).init_synthetic(seed)


def call_inputs(seed, shapes, n_txt, in_channels=16, joint_dim=96, t=0.5):
    """One call's arguments for `shapes` [(f, h, w), ...] (one grid: T2I's `[(1, h, w)]`; several: Edit's `[[...]]`)."""
    g = torch.Generator().manual_seed(seed)
    n_img = sum(f * h * w for f, h, w in shapes)
    img_shapes = [tuple(shapes[0])] if len(shapes) == 1 else [[tuple(s) for s in shapes]]
    return dict(hidden_states=torch.randn(1, n_img, in_channels, generator=g).bfloat16(),
                encoder_hidden_states=torch.randn(1, n_txt, joint_dim, generator=g).bfloat16(),
                encoder_hidden_states_mask=torch.ones(1, n_txt, dtype=torch.int64),
                timestep=torch.tensor([t]), img_shapes=img_shapes, txt_seq_lens=[n_txt])
