"""Open-Sora 1.2 engine: the STDiT3 forward behind `magcache_forward` of eval/magcache/experiments/opensora.py:229-373 on the sm_90a
kernels — wgmma GEMMs (fused bias / GELU-tanh / bf16 gated-residual epilogues), the head_dim-72 varlen attention (spatial and
cross), the temporal attention read in B (T S) C order, per-head LlamaRMSNorm(72) + RoPE, LayerNorm + t2i_modulate with bf16
rounding (`mc_ln_modulate` mode 2), the K1 / K2 cache kernels.

Block arithmetic is the reference's own (videosys/models/transformers/open_sora_transformer_3d.py: STDiT3Block.forward :154-273,
T2IFinalLayer :50-86, STDiT3.forward / encode_text / unpatchify :493-647), restated for the tests in tests/opensora_ref.py. Everything
is bf16 like the reference pipeline. Batch B > 1 per call (the CFG pair of scheduling_rflow_open_sora.py:238-246); the modulation,
gates and final-layer shift / scale are per sample.

HBM layout (B samples, T frames, S = H*W patches per frame, N = T*S, R = B*N rows in B (T S) order, D = hidden size):
  x    [R, D]   the residual stream              x0  [R, D]  x_embedder + pos_embed (`ori_x`)      res [R, D]  cached residual
  h    [R, D]   LN + t2i_modulate output         qkv [R, 3D] q | k | v, q / k normalised in place  att [R, D]  attention output
  ff   [R, 4D]  MLP hidden                        yk  [L, 2D] cross-attention k | v of the L = sum(y_lens) caption tokens
  mod  [2*depth, B, 6D] per-block `scale_shift_table + t_mlp` (bf16, and an exact fp32 copy for the kernels)

Sequence parallelism (VideoSys DSP, eval/magcache/experiments/opensora.py:284-293, 342-361; `enable_sequence_parallel`): rank r of P
owns frames [t0, t0 + T_r) (`shard.frame_position_shards`, the `split_sequence` partition without its pad). x / x0 / res / h / att
then hold those frames of every sample (N = T_r S rows per sample); the spatial blocks and cross-attention run on them unchanged.
A temporal block switches its modulated input to the position-sharded layout (every frame of positions [s0, s0 + S_r)), runs
qkv, q / k RMSNorm + RoPE and the attention there, switches the attention output back and runs `proj` with its gated residual on
the rank's frames (STDiT3Block.dynamic_switch, open_sora_transformer_3d.py:275-296, moves the same D-wide rows). The final layer
runs on the rank's frames into its window of the full-size output, which the peers then fill in: every rank returns the whole
prediction (or updated latent). Every row is computed by the launches the one-GPU engine uses for it, so the outputs are the same
bits.
"""
import math

import torch

from . import _lib, ops, shard

E = _lib


def _w(t, dev):
    return t.detach().to(device=dev, dtype=torch.bfloat16).contiguous()


def _b(t, dev):
    return t.detach().to(device=dev, dtype=torch.bfloat16).float().contiguous()  # bf16 parameter values, fp32 for the epilogues


class OpenSoraWeights:
    """The STDiT3 parameters by the reference's names (x_embedder.proj, t_embedder.mlp, fps_embedder.mlp, t_block.1, y_embedder.y_proj,
    spatial_blocks.i / temporal_blocks.i, final_layer), on one device in the layout the engine reads."""

    @classmethod
    def from_module(cls, m, dev):
        self = cls()
        self.device = torch.device(dev)
        p = dict(m.named_parameters())
        conv = p["x_embedder.proj.weight"]
        self.dim = conv.shape[0]
        self.in_channels = conv.shape[1]
        self.patch = tuple(conv.shape[2:])
        if self.patch != (1, 2, 2):
            raise NotImplementedError(f"magcache_b200: Open-Sora patch size {self.patch}; the engine embeds (1, 2, 2) patches")
        self.depth = len(m.spatial_blocks)
        self.heads = m.spatial_blocks[0].attn.num_heads
        if self.dim != self.heads * 72:
            raise NotImplementedError(f"magcache_b200: Open-Sora head_dim {self.dim // self.heads}; the attention kernels are built for 72")
        self.input_sq_size = getattr(getattr(m, "config", m), "input_sq_size", 512)
        D = self.dim
        self.x_w, self.x_b = _w(conv.reshape(D, -1), dev), _b(p["x_embedder.proj.bias"], dev)

        def mlp(prefix, a=0, c=2):
            return (_w(p[f"{prefix}.{a}.weight"], dev), _b(p[f"{prefix}.{a}.bias"], dev), _w(p[f"{prefix}.{c}.weight"], dev), _b(p[f"{prefix}.{c}.bias"], dev))

        self.t_mlp, self.fps_mlp = mlp("t_embedder.mlp"), mlp("fps_embedder.mlp")
        self.tb_w, self.tb_b = _w(p["t_block.1.weight"], dev), _b(p["t_block.1.bias"], dev)
        self.y_mlp = (_w(p["y_embedder.y_proj.fc1.weight"], dev), _b(p["y_embedder.y_proj.fc1.bias"], dev),
                      _w(p["y_embedder.y_proj.fc2.weight"], dev), _b(p["y_embedder.y_proj.fc2.bias"], dev))
        self.blocks, tables = [], []
        for i in range(self.depth):
            for kind in ("spatial", "temporal"):
                q = f"{kind}_blocks.{i}."
                self.blocks.append(dict(
                    temporal=kind == "temporal",
                    qkv_w=_w(p[q + "attn.qkv.weight"], dev), qkv_b=_b(p[q + "attn.qkv.bias"], dev),
                    nq=_b(p[q + "attn.q_norm.weight"], dev), nk=_b(p[q + "attn.k_norm.weight"], dev),
                    o_w=_w(p[q + "attn.proj.weight"], dev), o_b=_b(p[q + "attn.proj.bias"], dev),
                    cq_w=_w(p[q + "cross_attn.q_linear.weight"], dev), cq_b=_b(p[q + "cross_attn.q_linear.bias"], dev),
                    ckv_w=_w(p[q + "cross_attn.kv_linear.weight"], dev), ckv_b=_b(p[q + "cross_attn.kv_linear.bias"], dev),
                    co_w=_w(p[q + "cross_attn.proj.weight"], dev), co_b=_b(p[q + "cross_attn.proj.bias"], dev),
                    f1_w=_w(p[q + "mlp.fc1.weight"], dev), f1_b=_b(p[q + "mlp.fc1.bias"], dev),
                    f2_w=_w(p[q + "mlp.fc2.weight"], dev), f2_b=_b(p[q + "mlp.fc2.bias"], dev)))
                tables.append(_w(p[q + "scale_shift_table"], dev).reshape(-1))
        self.tables = torch.stack(tables)                                    # [2*depth, 6D] bf16, block order s0, t0, s1, t1, ...
        self.fin_table = _w(p["final_layer.scale_shift_table"], dev).reshape(-1)  # [2D]: shift | scale
        self.fin_w, self.fin_b = _w(p["final_layer.linear.weight"], dev), _b(p["final_layer.linear.bias"], dev)
        self.out_channels = self.fin_w.shape[0] // 4
        return self


def pos_embed_2d(dim, h, w, scale, base_size, device):
    """OpenSoraPositionEmbedding2D._get_cached_emb (videosys/models/modules/embeddings.py:231-280) -> bf16 [h*w, dim]."""
    half_dim = dim // 2
    inv_freq = (1.0 / (10000 ** (torch.arange(0, half_dim, 2).float() / half_dim))).to(device)
    grid_h = torch.arange(h, device=device) / scale
    grid_w = torch.arange(w, device=device) / scale
    if base_size is not None:
        grid_h *= base_size / h
        grid_w *= base_size / w
    grid_h, grid_w = torch.meshgrid(grid_w, grid_h, indexing="ij")  # w goes first, as upstream
    grid_h = grid_h.t().reshape(-1)
    grid_w = grid_w.t().reshape(-1)

    def sincos(t):
        out = torch.einsum("i,d->id", t, inv_freq)
        return torch.cat((torch.sin(out), torch.cos(out)), dim=-1)

    return torch.concat([sincos(grid_h), sincos(grid_w)], dim=-1).to(torch.bfloat16).contiguous()


def rope_table(T, head_dim, device, theta=10000.0):
    """fp32 [T, head_dim] (cos, sin) per interleaved pair: rotary_embedding_torch RotaryEmbedding(head_dim) [EXT] at positions 0..T-1
    (fp32 freqs `1 / theta^(arange(0, dim, 2) / dim)`, angle = position * freq)."""
    inv = (1.0 / (theta ** (torch.arange(0, head_dim, 2)[: head_dim // 2].float() / head_dim))).to(device)
    ang = torch.einsum("i,f->if", torch.arange(T, device=device, dtype=torch.float32), inv)
    return torch.stack([ang.cos(), ang.sin()], dim=-1).reshape(T, head_dim).contiguous()


class OpenSoraEngine:
    """One STDiT3 on the sm_90a kernels. Buffers are allocated once per (B, T, H, W) shape; the caption buffer grows with the
    number of valid caption tokens."""

    def __init__(self, weights: OpenSoraWeights, shard_world=1, shard_rank=0, shard_group=None, sp_world=1, sp_rank=0, sp_group=None):
        if shard_world > 1:  # no token-sharded path: every rank would compute the whole video
            raise NotImplementedError("magcache_b200: Open-Sora token sharding (enable_token_shard with world > 1) is not supported; "
                                      "enable_sequence_parallel shards frames and positions instead")
        self.w, self.device = weights, weights.device
        self.sp = (sp_rank, sp_world, sp_group) if sp_world > 1 else None  # sequence parallelism: (rank, world, group)
        self.switch = None
        self._shape = None
        self.res_valid = False
        self._step = None  # (z, guidance_scale, dt, out) armed by `arm_step` for the next forward

    # ------------------------------------------------------------------------------------------ buffers
    def _alloc(self, B, T, H, W):
        if self._shape == (B, T, H, W):
            return
        w, dev = self.w, self.device
        D = w.dim
        S = H * W
        self.t0, self.T_loc = 0, T  # this rank's frames (all of them without sequence parallelism)
        if self.sp is not None:
            rank, world, group = self.sp
            frames, positions = shard.frame_position_shards(world, T, S, group)
            self.t0, self.T_loc, self.S_loc = frames[rank].start, frames[rank].n_local, positions[rank].n_local
        N = self.T_loc * S  # rows per sample on this rank
        R = B * N
        bf = dict(dtype=torch.bfloat16, device=dev)
        self.B, self.T, self.H, self.W, self.S, self.N = B, T, H, W, S, N
        self.R = B * T * S  # rows of the whole batch (TeaCache's decision input covers all of them on every rank)
        self.x, self.x0, self.res, self.hit = (torch.empty(R, D, **bf) for _ in range(4))
        self.h, self.att = torch.empty(R, D, **bf), torch.empty(R, D, **bf)
        self.qkv, self.ff = torch.empty(R, 3 * D, **bf), torch.empty(R, 4 * D, **bf)
        self.qc = torch.empty(R, D, **bf)
        if self.sp is not None:
            R_pos = B * T * self.S_loc  # position-sharded rows of the temporal attention
            self.qkv_pos, self.att_pos = torch.empty(R_pos, 3 * D, **bf), torch.empty(R_pos, D, **bf)
        self.mod = torch.empty(2 * w.depth, B, 6 * D, **bf)
        self.mod_t = torch.empty_like(self.mod)
        self.tables_rep = w.tables[:, None, :].expand(2 * w.depth, B, 6 * D).contiguous()
        self.modf = torch.empty(2 * w.depth, B, 6 * D, dtype=torch.float32, device=dev)
        self.fin, self.fin_t = torch.empty(B, 2 * D, **bf), torch.empty(B, 2 * D, **bf)
        self.fin_rep = w.fin_table[None].expand(B, 2 * D).contiguous()
        self.finf = torch.empty(B, 2 * D, dtype=torch.float32, device=dev)
        segs = [(b * N + t * S, S, b * N + t * S, S) for b in range(B) for t in range(self.T_loc)]  # one spatial segment per frame
        self.segs_sp = torch.tensor(segs, dtype=torch.int32, device=dev)
        self.rope = rope_table(T, 72, dev)
        self.s_lat = torch.empty(B, w.in_channels, T, 2 * H, 2 * W, dtype=torch.float32, device=dev)
        self.s_t = torch.empty(2 * B, dtype=torch.float64, device=dev)
        self._pos_key = None
        self._y_key = None
        self.res_valid = False
        self._shape = (B, T, H, W)
        self._crop_key = None

    def rows(self, b):
        return slice(b * self.N, (b + 1) * self.N)

    # ------------------------------------------------------------------------------------------ inputs (:243-293)
    def stage_inputs(self, x, timestep, y, mask, fps, height, width):
        w = self.w
        B, C, Tx, Hx, Wx = x.shape
        if C != w.in_channels:
            raise ValueError(f"x has {C} channels, the model {w.in_channels}")
        T, H, W = Tx, -(-Hx // 2), -(-Wx // 2)
        self._alloc(B, T, H, W)
        self.crop = (Tx, Hx, Wx)
        if self.sp is not None and self._crop_key != (Hx, Wx):  # the output slots are sized by the crop
            if self.switch is not None:
                self.switch.close()
            rank, world, group = self.sp
            self.switch = shard.make_switch(rank, world, B, T, H * W, w.dim, Hx, Wx, self.device, group)
            self._crop_key = (Hx, Wx)
        if Hx % 2 or Wx % 2:
            self.s_lat.zero_()  # OpenSoraPatchEmbed3D zero-pads odd H / W
        self.s_lat[:, :, :, :Hx, :Wx].copy_(x.to(torch.bfloat16))  # `x.to(dtype)` (:245), held exactly in fp32
        # `timestep.to(dtype)` rounds t to bf16 (:246); fps enters the sinusoid as given (SizeEmbedder.forward)
        fps = torch.as_tensor(fps, device=self.device).reshape(-1)
        fps = fps.repeat(B // fps.numel()) if fps.numel() != B else fps
        self.s_t.copy_(torch.cat([timestep.reshape(-1).to(torch.bfloat16).float().double().to(self.device), fps.float().double()]))
        S = H * W
        key = (S, float(height.reshape(-1)[0].item()), float(width.reshape(-1)[0].item()))
        if self._pos_key != key:  # cached per shape like upstream's lru_cache
            scale = (key[1] * key[2]) ** 0.5 / w.input_sq_size
            self.pos = pos_embed_2d(w.dim, H, W, scale, round(S ** 0.5), self.device)
            self._pos_key = key
        # caption rows: `encode_text` (:493-504) keeps the valid tokens of every sample, concatenated
        yb = y.reshape(B, -1, y.shape[-1])
        if mask is not None:
            mk = mask.reshape(mask.shape[0], -1)
            if mk.shape[0] != B:
                mk = mk.repeat(B // mk.shape[0], 1)
            y_lens = [int(v) for v in mk.sum(dim=1).tolist()]
            sel = yb[mk.to(yb.device) != 0]
        else:
            y_lens = [yb.shape[1]] * B
            sel = yb.reshape(-1, yb.shape[-1])
        if min(y_lens) < 1:
            raise ValueError("magcache_b200: every sample needs at least one valid caption token")
        self.y_lens = y_lens
        self.y_in = sel.to(device=self.device, dtype=torch.bfloat16).contiguous()
        key = tuple(y_lens)
        if self._y_key != key:
            starts = [0] + list(torch.tensor(y_lens).cumsum(0)[:-1].tolist())
            self.segs_cross = torch.tensor([(b * self.N, self.N, starts[b], y_lens[b]) for b in range(B)], dtype=torch.int32, device=self.device)
            self._y_key = key

    # ------------------------------------------------------------------------------------------ prologue
    def _time_mlp(self, x_bf16, mlp):
        w1, b1, w2, b2 = mlp
        return ops.gemm(ops.gemm(x_bf16, w1, b1, E.MC_EPI_BIAS_SILU_BF16), w2, b2, E.MC_EPI_BIAS_BF16)

    def _sinusoid(self, t64):
        """[cos | sin] of TimestepEmbedder.timestep_embedding (embeddings.py:122-139), rounded to bf16. The kernel evaluates the
        arguments in float64; the reference forms `t.float() * freqs` in fp32, which at t ~ 1000 moves an argument by up to ~6e-5 rad.
        That is below the bf16 rounding that follows except on rare ties."""
        f = ops.time_sinusoid(t64, 256)
        return ops.cast_into(f, torch.empty(t64.numel(), 256, dtype=torch.bfloat16, device=self.device))

    def prologue(self, kind):
        """x_embedder + pos_embed into x0, t / fps embedders, t_block, the per-block modulation and, on a miss, the caption MLP."""
        w, B, D = self.w, self.B, self.w.dim
        self._embed(self.x0, self.T_loc, self.t0)
        t = self._time_mlp(self._sinusoid(self.s_t[:B]), w.t_mlp)
        t = ops.cache_hit_add(t, self._time_mlp(self._sinusoid(self.s_t[B:]), w.fps_mlp))  # `t = t + fps` (bf16)
        t_mlp = ops.gemm(ops.silu(t), w.tb_w, w.tb_b, E.MC_EPI_BIAS_BF16)               # t_block
        self.mod_t.copy_(t_mlp.view(1, B, 6 * D).expand_as(self.mod_t))
        ops.cache_hit_add(self.tables_rep, self.mod_t, out=self.mod)                      # `scale_shift_table[None] + t.reshape(B, 6, -1)`
        ops.cast_into(self.mod, self.modf)
        self.fin_t.view(B, 2, D).copy_(t.view(B, 1, D).expand(B, 2, D))
        ops.cast_into(ops.cache_hit_add(self.fin_rep, self.fin_t, out=self.fin), self.finf)  # final layer `table[None] + t[:, None]`
        if kind == "miss":
            self.caption()

    def _embed(self, x0, T, t0):
        """x_embedder + pos_embed of frames [t0, t0 + T) of every sample into x0 [B T S, D]."""
        w, B, D, S = self.w, self.B, self.w.dim, self.S
        x0v = x0.view(B, T, S, D)
        x0v.copy_(self.pos.view(1, 1, S, D).expand_as(x0v))
        for b in range(B):  # Conv3d (1,2,2) as a K = 4*C GEMM; `x + pos_emb` in the epilogue (bf16(pos + bf16(acc + bias)))
            tok = ops.patchify(self.s_lat[b])
            if T != self.T:  # the GEMM is row-local: a rank's frames are the same bits as in the whole video
                tok = tok[t0 * S:(t0 + T) * S]
            ops.gemm(tok, w.x_w, w.x_b, E.MC_EPI_BIAS_GATE_RESID_BF16, out=x0[b * T * S:(b + 1) * T * S])

    def caption(self):
        """The caption MLP (`y_embedder`), which only the block stack reads."""
        f1w, f1b, f2w, f2b = self.w.y_mlp
        self.y_emb = ops.gemm(ops.gemm(self.y_in, f1w, f1b, E.MC_EPI_BIAS_GELU_BF16), f2w, f2b, E.MC_EPI_BIAS_BF16)

    # ------------------------------------------------------------------------------------------ blocks (STDiT3Block.forward)
    def _block(self, i, blk, x_m=None):
        """`x_m`: this block's first LN + t2i_modulate output when the caller already has it (TeaCache's decision input is block 0's)."""
        w, B, D, H = self.w, self.B, self.w.dim, self.w.heads
        x, h, qkv, att = self.x, self.h, self.qkv, self.att
        em = [self.modf[i, b].view(6, D) for b in range(B)]  # shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp
        if x_m is None:
            for b in range(B):
                ops.ln_t2i_modulate(x[self.rows(b)], em[b], 1, 0, out=h[self.rows(b)])
            x_m = h
        S = self.S
        if blk["temporal"] and self.sp is not None:  # to every frame of this rank's positions (dynamic_switch, :275-296)
            x_m, qkv, att, S = self.switch.to_positions(x_m), self.qkv_pos, self.att_pos, self.S_loc
        ops.gemm(x_m, blk["qkv_w"], blk["qkv_b"], E.MC_EPI_BIAS_BF16, out=qkv)
        q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        rope = self.rope if blk["temporal"] else None
        ops.rmsnorm_head72_rope_(q, blk["nq"], H, rope, pos_div=S, tag="os_qknorm")
        ops.rmsnorm_head72_rope_(k, blk["nk"], H, rope, pos_div=S, tag="os_qknorm")
        if blk["temporal"]:
            ops.attention_temporal_d72(q, k, v, H, B, self.T, S, out=att, tag="os_attn_temporal")
            if self.sp is not None:  # the attention output back to this rank's frames; `proj` runs there
                att = self.switch.to_frames(att)
        else:
            ops.attention_varlen_d72(q, k, v, H, self.segs_sp, self.S, out=att, tag="os_attn_spatial")
        for b in range(B):  # `x = x + gate_msa * x_m`
            ops.gemm(att[self.rows(b)], blk["o_w"], blk["o_b"], E.MC_EPI_BIAS_GATE_RESID_BF16, out=x[self.rows(b)], gate=em[b][2])
        # cross-attention (varlen over the caption tokens of each sample), `x = x + x_cross`
        ops.gemm(x, blk["cq_w"], blk["cq_b"], E.MC_EPI_BIAS_BF16, out=self.qc)
        kv = ops.gemm(self.y_emb, blk["ckv_w"], blk["ckv_b"], E.MC_EPI_BIAS_BF16)
        ops.attention_varlen_d72(self.qc, kv[:, :D], kv[:, D:], H, self.segs_cross, self.N, out=self.att, tag="os_attn_cross")
        ops.gemm(self.att, blk["co_w"], blk["co_b"], E.MC_EPI_BIAS_GATE_RESID_BF16, out=x)
        # MLP, `x = x + gate_mlp * mlp(t2i_modulate(norm2(x), shift_mlp, scale_mlp))`
        for b in range(B):
            ops.ln_t2i_modulate(x[self.rows(b)], em[b], 4, 3, out=h[self.rows(b)])
        ops.gemm(h, blk["f1_w"], blk["f1_b"], E.MC_EPI_BIAS_GELU_BF16, out=self.ff)
        for b in range(B):
            ops.gemm(self.ff[self.rows(b)], blk["f2_w"], blk["f2_b"], E.MC_EPI_BIAS_GATE_RESID_BF16, out=x[self.rows(b)], gate=em[b][5])

    def run_blocks(self, x_m0=None):
        self.x.copy_(self.x0)
        for i, blk in enumerate(self.w.blocks):
            self._block(i, blk, x_m0 if i == 0 else None)
        return self.x

    # ------------------------------------------------------------------------------------------ output (T2IFinalLayer, unpatchify)
    def head(self, x):
        w, B, D = self.w, self.B, self.w.dim
        for b in range(B):
            ops.ln_t2i_modulate(x[self.rows(b)], self.finf[b].view(2, D), 1, 0, out=self.h[self.rows(b)])
        o = ops.gemm(self.h, w.fin_w, w.fin_b, E.MC_EPI_BIAS_BF16)  # [R, (T_p H_p W_p C_out)]
        C = w.out_channels
        o = o.view(B, self.T, self.H, self.W, 1, 2, 2, C).permute(0, 7, 1, 4, 2, 5, 3, 6).reshape(B, C, self.T, 2 * self.H, 2 * self.W)
        Tx, Hx, Wx = self.crop
        return o[:, :, :Tx, :Hx, :Wx].float()

    def arm_step(self, z, guidance_scale, dt, out):
        """Fold the tail of the sampler's step (scheduling_rflow_open_sora.py:244-251: velocity channels, cond / uncond split, CFG
        combine, `z + v_pred * dt`) into the final layer of the NEXT forward, which then returns `out` = the updated latent fp32
        [B/2, 4, Tx, Hx, Wx] instead of the prediction (`mc_opensora_head` step mode). z: the latent of this step, fp32 of that
        shape; dt: fp32 [B/2] on the device; `out` may be `z`. One-shot; bit-equal to the plain forward followed by the reference's
        statements."""
        if self.w.out_channels != 8:
            raise NotImplementedError("magcache_b200: the fused sampler step is built for 8 output channels (pred_sigma)")
        self._step = (z, float(guidance_scale), dt, out)

    def _final(self, x, hit):
        """The final layer on `x` (None on a hit: x0 + cached residual): `head`, or the armed step in one `mc_opensora_head` pass."""
        step, self._step = self._step, None
        if self.sp is not None:
            return self._final_sp(x, hit, step)
        if step is None:
            return self.head(ops.cache_hit_add(self.x0, self.res, out=self.hit) if hit else x)
        z, g, dt, out = step
        return ops.opensora_head(self.x0 if hit else x, self.finf.view(self.B, 2, self.w.dim), self.w.fin_w, self.w.fin_b,
                                 (self.T, self.H, self.W), self.crop, res=self.res if hit else None, step=(z, g, dt), out=out,
                                 tag="os_head_step")

    def _final_sp(self, x, hit, step):
        """The final layer on this rank's frames into its window of a full-size output (`mc_opensora_head_frames`), then the peers'
        windows: every rank returns the whole prediction, or with a step armed the whole updated latent (into the step's `out`)."""
        _, Hx, Wx = self.crop
        buf = self.switch.output_buffer(step is not None)
        z, g, dt, out = step if step is not None else (None, 0.0, None, None)
        ops.opensora_head_frames(self.x0 if hit else x, self.finf.view(self.B, 2, self.w.dim), self.w.fin_w, self.w.fin_b,
                                 (self.T_loc, self.H, self.W), (self.T, Hx, Wx), self.t0, buf, res=self.res if hit else None,
                                 step=(z, g, dt) if step is not None else None, tag="os_head_frames")
        return self.switch.gather_output(buf, out)

    def forward(self, kind):
        """prologue -> {hit: x0 + cached residual | miss: blocks, residual = x - x0} -> final layer (opensora.py:309-367)."""
        try:
            self.prologue(kind)
            if kind == "hit":
                if not self.res_valid:
                    raise TypeError("magcache_b200: cache hit with an empty residual cache")
                return self._final(None, True)
            x = self.run_blocks()
            ops.residual_sub(x, self.x0, out=self.res)
            self.res_valid = True
            return self._final(x, False)
        finally:
            self._step = None

    # ------------------------------------------------------------------------------------------ TeaCache (opensora.py:34-227)
    def _tea_alloc(self):
        if self.__dict__.get("_tea_shape") == self._shape:
            return
        self.mi = torch.empty(2, self.R, self.w.dim, dtype=torch.bfloat16, device=self.device)  # modulated inputs, alternating
        self.mi_prev = None  # index of the buffer holding `previous_modulated_input`, None: there is none
        if self.sp is not None:  # every frame's x0, for the decision input over all rows
            self.x0_all = torch.empty(self.R, self.w.dim, dtype=torch.bfloat16, device=self.device)
        self.tea_sums = torch.zeros(2, dtype=torch.float64, device=self.device)
        self.tea_partials = ops.rel_l1_partials(self.device)
        self._tea_shape = self._shape

    def take_modulated_input(self, cur):
        """Follow the `previous_modulated_input` attribute: None clears it; a tensor other than the engine's own buffer is copied in."""
        self._tea_alloc()
        if cur is None:
            self.mi_prev = None
        elif self.mi_prev is None or cur.data_ptr() != self.mi[self.mi_prev].data_ptr():
            self.mi_prev = 0 if self.mi_prev is None else self.mi_prev
            self.mi[self.mi_prev].copy_(cur.reshape(self.R, self.w.dim))

    def modulated_input(self, distance):
        """TeaCache's decision input `t2i_modulate(spatial_blocks[0].norm1(x0), shift_msa, scale_msa)` (:89-95) per sample, into the
        buffer that does not hold the previous one, which it then replaces (:108). With `distance`, the same launches also return the
        two sums (sum |cur - prev|, sum |prev|) over all samples (:102), one host sync. Call after `prologue`."""
        self._tea_alloc()
        k = 0 if self.mi_prev is None else 1 - self.mi_prev
        cur, D = self.mi[k], self.w.dim
        x0, rows = self.x0, self.rows
        if self.sp is not None:  # the reference forms it before its split: every rank embeds and modulates all frames
            self._embed(self.x0_all, self.T, 0)
            N = self.T * self.S
            x0, rows = self.x0_all, lambda b: slice(b * N, (b + 1) * N)
        if distance:
            prev = self.mi[self.mi_prev]
            self.tea_sums.zero_()
            for b in range(self.B):
                ops.ln_t2i_modulate_rel_l1(x0[rows(b)], self.modf[0, b].view(6, D), 1, 0, prev[rows(b)], cur[rows(b)],
                                           self.tea_partials, self.tea_sums, tag="os_tea_input")
        else:
            for b in range(self.B):
                ops.ln_t2i_modulate(x0[rows(b)], self.modf[0, b].view(6, D), 1, 0, out=cur[rows(b)], tag="os_tea_input")
        self.mi_prev = k
        return self.tea_sums.tolist() if distance else None

    def forward_teacache(self, calc):
        """After `prologue("hit")` and `modulated_input`: hit `x += previous_residual` (bf16, :114) | miss: the caption MLP, the block
        stack with block 0's first LN-modulate taken from the decision input (the same tensor), `previous_residual = x - origin_x`
        (:156) -> final layer."""
        try:
            if not calc:
                if not self.res_valid:
                    raise TypeError("magcache_b200: TeaCache hit with no previous_residual")
                return self._final(None, True)
            self.caption()
            x_m0 = self.mi[self.mi_prev]
            if self.sp is not None:  # this rank's frames of the decision input
                N, S = self.T * self.S, self.S
                for b in range(self.B):
                    self.h[self.rows(b)].copy_(x_m0[b * N + self.t0 * S:b * N + (self.t0 + self.T_loc) * S])
                x_m0 = self.h
            x = self.run_blocks(x_m0)
            ops.residual_sub(x, self.x0, out=self.res)
            self.res_valid = True
            return self._final(x, False)
        finally:
            self._step = None

    def forward_plain(self):
        """`enable_teacache = False` (:157-197): the block stack, no residual kept."""
        try:
            self.prologue("miss")
            return self._final(self.run_blocks(), False)
        finally:
            self._step = None


def random_opensora_weights(dev, hidden_size=1152, depth=28, num_heads=16, caption_channels=4096, model_max_length=300, seed=0):
    """Seeded full-size STDiT3 weights (bf16 on `dev`) for the benchmark: the module tree of tests/opensora_ref.py is not needed, only
    its parameter names, so the weights are generated straight into the engine's layout."""
    import types
    g = torch.Generator(device="cpu").manual_seed(seed)
    D = hidden_size

    def lin(o, i):
        return (torch.randn(o, i, generator=g) / math.sqrt(i)), 0.02 * torch.randn(o, generator=g)

    params = {}

    def put(name, o, i):
        params[name + ".weight"], params[name + ".bias"] = lin(o, i)

    conv_w, conv_b = lin(D, 16)
    params["x_embedder.proj.weight"], params["x_embedder.proj.bias"] = conv_w.view(D, 4, 1, 2, 2), conv_b
    put("t_embedder.mlp.0", D, 256), put("t_embedder.mlp.2", D, D)
    put("fps_embedder.mlp.0", D, 256), put("fps_embedder.mlp.2", D, D)
    put("t_block.1", 6 * D, D)
    put("y_embedder.y_proj.fc1", D, caption_channels), put("y_embedder.y_proj.fc2", D, D)
    for kind in ("spatial", "temporal"):
        for i in range(depth):
            q = f"{kind}_blocks.{i}."
            put(q + "attn.qkv", 3 * D, D), put(q + "attn.proj", D, D)
            params[q + "attn.q_norm.weight"] = 1 + 0.1 * torch.randn(D // num_heads, generator=g)
            params[q + "attn.k_norm.weight"] = 1 + 0.1 * torch.randn(D // num_heads, generator=g)
            put(q + "cross_attn.q_linear", D, D), put(q + "cross_attn.kv_linear", 2 * D, D), put(q + "cross_attn.proj", D, D)
            put(q + "mlp.fc1", 4 * D, D), put(q + "mlp.fc2", D, 4 * D)
            params[q + "scale_shift_table"] = torch.randn(6, D, generator=g) / D ** 0.5
    params["final_layer.scale_shift_table"] = torch.randn(2, D, generator=g) / D ** 0.5
    put("final_layer.linear", 32, D)
    blk = types.SimpleNamespace(attn=types.SimpleNamespace(num_heads=num_heads))
    m = types.SimpleNamespace(named_parameters=lambda: params.items(), spatial_blocks=[blk] * depth, input_sq_size=512)
    return OpenSoraWeights.from_module(m, dev)
