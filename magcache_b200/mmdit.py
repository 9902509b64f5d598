"""MMDiT engines (SURVEY §8f rank 4): the transformers behind `magcache_forward` of MagCache4FLUX/magcache_flux.py:234-440 (FLUX.1,
FLUX.1-Kontext) and of MagCache4HunyuanVideo/magcache_sample_video.py:29-160 (HunyuanVideo) on the same sm_90a kernels as the Wan path — wgmma GEMMs (fused bias / GELU / SiLU / bf16 gated-residual epilogues), the wgmma flash
attention over the joint text+image sequence, LN+modulate, per-head RMSNorm + RoPE, the K1/K2 cache kernels.

Block arithmetic follows diffusers' `FluxTransformerBlock` / `FluxSingleTransformerBlock` and hyvideo's `MMDoubleStreamBlock` /
`MMSingleStreamBlock` / `SingleTokenRefiner` [EXT, not in the reference tree] as restated in oracle/flux_ref.py and oracle/hunyuan_ref.py;
the forwards' own statements (embedders, controller, hit / miss, residual, final layer, counter) are the reference's (file:line cited in
`magcache_flux_forward` / `magcache_hunyuan_forward`, magcache_b200/patch.py). The two families share one block-stack implementation
(`MMDiTCore`): same modulation chunk order, same per-head q/k RMSNorm, same `cat(attn, act(mlp))` single block; they differ in the
token order of the joint sequence, in which rows get RoPE, and in their embedders.

STATUS (end of round 1): parity-green against the oracles at reduced depth / token counts (tests/test_flux_forward_gpu.py,
tests/test_hunyuan_forward_gpu.py) and pinned on CPU through the kernel emulation
(tests/test_*_engine_emulated_cpu.py); not yet run or timed at the full FLUX 1024^2 / HunyuanVideo 720p shapes. Nothing on the Wan path
depends on this module.

HBM layout (S = n_txt + n_img tokens; FLUX puts the text rows FIRST — `torch.cat([encoder_hidden_states, hidden_states], dim=1)`,
magcache_flux.py:384 — HunyuanVideo the image rows — `torch.cat((img, txt), 1)`, magcache_sample_video.py:123; D = heads*128;
everything bf16 like the reference pipelines, which run without autocast):
  hs   [S, D]    both residual streams; the double-stream blocks work on the two row ranges, the single-stream blocks on all rows
  x0   [n_img, D] x_embedder output (`ori_hidden_states`)         res [n_img, D]  cached residual (`previous_residual`)
  h    [S, D]    LN+modulate output (GEMM A operand)              qk  [S, 2D]     q | k projections, per-head RMSNorm + RoPE in place
  v    [S, D]    row-major V (attention reads it as is)          cat [S, 5D]     single blocks: attention output | GELU(proj_mlp);
                                                                                  double blocks borrow cat[:, D:] as the FF hidden
  ada  [R]       ALL AdaLayerNorm projections of the forward from ONE GEMM over silu(temb) (they depend on temb only)
"""
import numpy as np
import torch

from . import _lib, ops
from .lora import FluxLoraScan, LoraPack, Tailed, base_linear, is_lora_layer
from .ops import IP_ATTN_MAX_ADAPTERS, IP_ATTN_MAX_KEYS

E = _lib


def _w(t, dev):
    return t.detach().to(device=dev, dtype=torch.bfloat16).contiguous()


def _b(t, dev):
    return t.detach().to(device=dev, dtype=torch.bfloat16).float().contiguous()  # bf16 parameter values, kept as fp32 for the epilogues


# ----------------------------------------------------------------------------------------------------------------------
# FP8 block weights (HunyuanVideo `--use-fp8`, MagCache4HunyuanVideo/README.md:76-96). Upstream's `convert_fp8_linear`
# [EXT hyvideo/modules/fp8_optimization.py] stores the weight of every Linear under `double_blocks` / `single_blocks` as
# float8_e4m3fn with a bf16 scalar `fp8_scale`; `fp8_linear_forward` multiplies by `qdata.to(bf16) * scale` in an ordinary bf16
# F.linear. Only `Fp8Weight` and `linear()` below know that format; everything else passes weights through `linear()`.
# ----------------------------------------------------------------------------------------------------------------------
class Fp8Weight:
    """float8_e4m3fn codes [rows, cols] and one bf16 scale per row (the Linear's `fp8_scale` repeated over its rows, so a row block
    of a fused matrix and the stacked modulation rows of several Linears carry their own scales). Indexing takes a row block."""

    def __init__(self, q, scale):
        assert q.dtype == torch.float8_e4m3fn and q.dim() == 2 and scale.dtype == torch.bfloat16 and scale.shape == (q.shape[0],)
        self.q, self.scale = q, scale

    @property
    def shape(self):
        return self.q.shape

    def __getitem__(self, rows):
        return Fp8Weight(self.q[rows], self.scale[rows])


def linear(a, w, bias, epilogue, out, gate=None, scratch=None, addend=None, addend_row0=0):
    """`ops.gemm(a, w, ...)` for a bf16 weight (with an `addend`: the ControlNet epilogue, see ops.gemm). A `lora.Tailed` weight adds
    its LoRA update in the same launch (`ops.gemm(tail=...)`) from the U its group's down-projection left for `a`. For an Fp8Weight: per
    block of rows that fits `scratch` (bf16), one `dequant_fp8_bf16` into the scratch, then the unchanged bf16 GEMM on it for the
    matching output columns. Every epilogue but MC_EPI_ROWBIAS_BF16 is column-wise, so the blocks compute exactly the columns one
    GEMM would."""
    if isinstance(w, Tailed):
        return ops.gemm(a, w.w, bias, epilogue, out=out, gate=gate, addend=addend, addend_row0=addend_row0, tail=w.tail(a))
    if not isinstance(w, Fp8Weight):
        if addend is None:
            return ops.gemm(a, w, bias, epilogue, out=out, gate=gate)
        return ops.gemm(a, w, bias, epilogue, out=out, gate=gate, addend=addend, addend_row0=addend_row0)
    assert addend is None, "no FP8 family has ControlNet residuals"
    assert epilogue != E.MC_EPI_ROWBIAS_BF16 and out is not None and scratch is not None
    rows, cols = w.shape
    step = max(8, scratch.numel() // cols // 8 * 8)  # multiples of 8 rows keep every output column block 16-byte aligned
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        b = scratch[:(r1 - r0) * cols].view(r1 - r0, cols)
        ops.dequant_fp8_bf16(w.q[r0:r1], w.scale[r0:r1], out=b)
        ops.gemm(a, b, None if bias is None else bias[r0:r1], epilogue, out=out[:, r0:r1], gate=None if gate is None else gate[r0:r1])
    return out


class FluxWeights:
    """Weights of one FluxTransformer2DModel (diffusers attribute names), repacked: q|k weights concatenated, every AdaLayerNorm
    projection stacked into one matrix, biases / norm weights as fp32 copies of their bf16 values."""

    ada_parts = None    # bf16 weights only: the modulation table is one GEMM over `ada_w`
    fp8_scratch = None

    def __init__(self):
        self.double, self.single = [], []

    @classmethod
    def from_module(cls, m, dev):
        """Base weights only: a PEFT LoRA layer contributes its `base_layer`; the adapters are read at every call (lora.py)."""
        cfg = m.config
        w = cls()
        B = base_linear
        w.heads, w.head_dim = cfg.num_attention_heads, cfg.attention_head_dim
        if w.head_dim != 128 or tuple(cfg.axes_dims_rope) != (16, 56, 56):
            raise NotImplementedError("FLUX engine: head_dim 128 with RoPE axes (16, 56, 56)")
        w.dim = D = w.heads * w.head_dim
        w.in_channels, w.joint_dim, w.pooled_dim = cfg.in_channels, cfg.joint_attention_dim, cfg.pooled_projection_dim
        w.guidance = bool(cfg.guidance_embeds)
        w.x_w, w.x_b = _w(B(m.x_embedder).weight, dev), _b(B(m.x_embedder).bias, dev)
        w.ctx_w, w.ctx_b = _w(B(m.context_embedder).weight, dev), _b(B(m.context_embedder).bias, dev)
        tte = m.time_text_embed

        def mlp(e):
            return (_w(B(e.linear_1).weight, dev), _b(B(e.linear_1).bias, dev), _w(B(e.linear_2).weight, dev), _b(B(e.linear_2).bias, dev))

        w.t_mlp, w.p_mlp = mlp(tte.timestep_embedder), mlp(tte.text_embedder)
        w.g_mlp = mlp(tte.guidance_embedder) if w.guidance else None
        ada_w, ada_b, off = [], [], 0

        def ada(lin):
            nonlocal off
            ada_w.append(B(lin).weight.detach())
            ada_b.append(B(lin).bias.detach())
            start, off = off, off + B(lin).weight.shape[0]
            return start

        for blk in m.transformer_blocks:
            a = blk.attn
            w.double.append({
                "ada": ada(blk.norm1.linear), "ada_c": ada(blk.norm1_context.linear),
                "qk_w": _w(torch.cat([B(a.to_q).weight, B(a.to_k).weight], 0), dev), "qk_b": _b(torch.cat([B(a.to_q).bias, B(a.to_k).bias], 0), dev),
                "v_w": _w(B(a.to_v).weight, dev), "v_b": _b(B(a.to_v).bias, dev), "o_w": _w(B(a.to_out[0]).weight, dev), "o_b": _b(B(a.to_out[0]).bias, dev),
                "nq": _b(a.norm_q.weight, dev), "nk": _b(a.norm_k.weight, dev),
                "cqk_w": _w(torch.cat([B(a.add_q_proj).weight, B(a.add_k_proj).weight], 0), dev),
                "cqk_b": _b(torch.cat([B(a.add_q_proj).bias, B(a.add_k_proj).bias], 0), dev),
                "cv_w": _w(B(a.add_v_proj).weight, dev), "cv_b": _b(B(a.add_v_proj).bias, dev),
                "co_w": _w(B(a.to_add_out).weight, dev), "co_b": _b(B(a.to_add_out).bias, dev),
                "cnq": _b(a.norm_added_q.weight, dev), "cnk": _b(a.norm_added_k.weight, dev),
                "ff1_w": _w(B(blk.ff.net[0].proj).weight, dev), "ff1_b": _b(B(blk.ff.net[0].proj).bias, dev),
                "ff2_w": _w(B(blk.ff.net[2]).weight, dev), "ff2_b": _b(B(blk.ff.net[2]).bias, dev),
                "cff1_w": _w(B(blk.ff_context.net[0].proj).weight, dev), "cff1_b": _b(B(blk.ff_context.net[0].proj).bias, dev),
                "cff2_w": _w(B(blk.ff_context.net[2]).weight, dev), "cff2_b": _b(B(blk.ff_context.net[2]).bias, dev),
            })
        for blk in m.single_transformer_blocks:
            a = blk.attn
            w.single.append({
                "ada": ada(blk.norm.linear),
                "qk_w": _w(torch.cat([B(a.to_q).weight, B(a.to_k).weight], 0), dev), "qk_b": _b(torch.cat([B(a.to_q).bias, B(a.to_k).bias], 0), dev),
                "v_w": _w(B(a.to_v).weight, dev), "v_b": _b(B(a.to_v).bias, dev), "nq": _b(a.norm_q.weight, dev), "nk": _b(a.norm_k.weight, dev),
                "mlp_w": _w(B(blk.proj_mlp).weight, dev), "mlp_b": _b(B(blk.proj_mlp).bias, dev),
                "out_w": _w(B(blk.proj_out).weight, dev), "out_b": _b(B(blk.proj_out).bias, dev),
            })
        w.ada_out = ada(m.norm_out.linear)
        w.ada_w, w.ada_b, w.ada_rows = _w(torch.cat(ada_w, 0), dev), _b(torch.cat(ada_b, 0), dev), off
        w.out_w, w.out_b = _w(B(m.proj_out).weight, dev), _b(B(m.proj_out).bias, dev)
        w.device = dev
        return w


def rope_table(ids, device, axes_dim=(16, 56, 56), theta=10000.0):
    """cos / sin of `FluxPosEmbed` (float64 angles, fp32 values) for ids [S, 3], stored [S, 128] as interleaved (cos, sin) pairs."""
    pos = ids.detach().double().cpu().numpy()
    ang = [np.outer(pos[:, i], 1.0 / theta ** (np.arange(0, d, 2, dtype=np.float64) / d)) for i, d in enumerate(axes_dim)]
    ang = np.concatenate(ang, axis=1)  # [S, 64]
    cs = np.stack([np.cos(ang), np.sin(ang)], axis=-1).reshape(len(pos), 2 * ang.shape[1])
    return torch.tensor(cs.astype(np.float32)).to(device)  # torch-allocated (aligned) storage on every device


class InputKey:
    """Cache key of a table derived from a caller's tensors (RoPE positions, the valid length of a text mask). The tensors are held,
    so their memory cannot go to another tensor while the key lives, and each is compared by storage, offset, shape, strides, dtype
    and `_version`, which every torch write bumps (`copy_`, in-place ops, a write through any view). An address alone identifies
    nothing: a caller that writes the next generation's ids into the same buffer keeps it, and so does the caching allocator when
    it hands the freed block of one generation's mask to the next one's. Staging through a key adds no host synchronisation. Writes
    torch does not see (through `.data`, DLPack or C, a CUDA graph replay into the tensor) keep the key: call `invalidate_engine`.

    An inference tensor (made under `torch.inference_mode()`) has no version counter, and an in-place write to it inside inference
    mode leaves no trace on the tensor. The key keeps a copy of such a tensor's content and compares it on every call: one small
    comparison and one host synchronisation per call, for inference tensors only."""

    __slots__ = ("held", "meta", "copies")

    def __init__(self, *ts):
        self.held, self.meta = ts, self._meta(ts)
        self.copies = tuple(t.clone() if t.is_inference() else None for t in ts)

    @staticmethod
    def _meta(ts):
        # a held storage stays allocated, so no other live storage can start at its address
        return tuple((t.untyped_storage().data_ptr(), t.storage_offset(), tuple(t.shape), t.stride(), t.dtype, t.device,
                      None if t.is_inference() else t._version) for t in ts)

    def matches(self, *ts):
        return self._meta(ts) == self.meta and all(c is None or torch.equal(c, t) for c, t in zip(self.copies, ts))


def controlnet_index(i, n_blocks, n_samples, repeat=False):
    """Index of the ControlNet sample added after block `i` of `n_blocks`: the reference's expressions (magcache_flux.py:376-384 for
    the double blocks, `repeat` = XLabs' controlnet_blocks_repeat; :418-423 for the single blocks, which never repeat). The interval
    is computed first, as there, so an empty sample list raises ZeroDivisionError either way."""
    interval = int(np.ceil(n_blocks / n_samples))
    return i % n_samples if repeat else i // interval


# diffusers' attention processors of a FLUX block, by class name (no diffusers import): the IP-Adapter processor (current name,
# then the name before diffusers 0.32) and the plain ones, whose arithmetic the engine's blocks restate. The restated oracle
# modules have no `processor` attribute.
IP_PROCESSORS = ("FluxIPAdapterAttnProcessor", "FluxIPAdapterJointAttnProcessor2_0")
PLAIN_PROCESSORS = ("FluxAttnProcessor", "FluxAttnProcessor2_0", "FluxAttnProcessor2_0_NPU")


def ip_processor(attn, name):
    """`attn.processor` when it is an IP-Adapter processor, None when the block runs the plain attention; any other processor
    raises (its arithmetic is not the engine's)."""
    proc = getattr(attn, "processor", None)
    if proc is None or type(proc).__name__ in PLAIN_PROCESSORS:
        return None
    if type(proc).__name__ in IP_PROCESSORS:
        return proc
    raise NotImplementedError(f"magcache_b200: {name}.processor is a {type(proc).__name__}; the FLUX engine runs "
                              f"{', '.join(PLAIN_PROCESSORS + IP_PROCESSORS)}")


class IPAdapterCall:
    """The IP-Adapter side path of one FLUX call, read from the module as it is at that call (processors, scales, weights):
    `ip_hidden_states = encoder_hid_proj(ip_adapter_image_embeds)` (magcache_flux.py:321-324) and, in every double block with an
    IP-Adapter processor, `ip_attn_output = sum_a scale[a] * SDPA(ip_query, to_k_ip[a](ip_h[a]), to_v_ip[a](ip_h[a]))` added to
    the image stream after the feed-forward residual [EXT diffusers FluxIPAdapterAttnProcessor / FluxTransformerBlock]. Nothing
    is kept between calls. The module's bf16 weights are read in place; only biases and norm parameters get fp32 copies."""

    def __init__(self, module, procs, embeds, dim, device):
        """`procs`: ip_processor() of each double block."""
        name = "joint_attention_kwargs['ip_adapter_image_embeds']"
        self.procs = procs
        if not any(p is not None for p in self.procs):
            raise NotImplementedError(f"magcache_b200: {name} given, but no double block has an IP-Adapter attention processor "
                                      "(load the adapter with `load_ip_adapter`)")
        if embeds is None:
            raise NotImplementedError("magcache_b200: the model has IP-Adapter attention processors but the call passes no "
                                      "ip_adapter_image_embeds (the reference's processor cannot run without them either)")
        proj = getattr(module, "encoder_hid_proj", None)
        self.layers = list(getattr(proj, "image_projection_layers", None) or ())
        if not self.layers:
            raise NotImplementedError("magcache_b200: IP-Adapter processors need `encoder_hid_proj` to be a "
                                      "MultiIPAdapterImageProjection with its `image_projection_layers`")
        lora_on = [f"encoder_hid_proj.{n}" for n, m in proj.named_modules() if is_lora_layer(m)]
        for i, p in enumerate(self.procs):
            if p is not None:
                lora_on += [f"transformer_blocks.{i}.attn.processor.{k}.{a}" for k in ("to_k_ip", "to_v_ip")
                            for a, m in enumerate(getattr(p, k)) if is_lora_layer(m)]
        if lora_on:
            raise NotImplementedError(f"magcache_b200: a LoRA adapter on the IP-Adapter's {lora_on[0]} is not supported")
        A = len(self.layers)
        if not isinstance(embeds, (list, tuple)) or len(embeds) != A:
            raise NotImplementedError(f"magcache_b200: {name} must be a list of {A} tensors, one per loaded adapter; got "
                                      f"{type(embeds).__name__}{'' if not isinstance(embeds, (list, tuple)) else f' of {len(embeds)}'}")
        self.embeds, self.n_keys = [], []
        for a, (e, layer) in enumerate(zip(embeds, self.layers)):
            lin, norm = layer.image_embeds, layer.norm
            want = (1, "num_images", lin.in_features)
            if not (torch.is_tensor(e) and e.dim() == 3 and e.shape[0] == 1 and e.shape[1] >= 1 and e.shape[2] == lin.in_features
                    and e.dtype == torch.bfloat16 and e.device == device):
                got = f"{e.dtype} {tuple(e.shape)} on {e.device}" if torch.is_tensor(e) else type(e).__name__
                raise NotImplementedError(f"magcache_b200: {name}[{a}] must be a bf16 tensor of shape {list(want)} on {device} "
                                          f"(one sample per call); got {got}")
            C = norm.normalized_shape[0]
            if norm.weight is None or norm.bias is None or lin.out_features != layer.num_image_text_embeds * C:
                raise NotImplementedError(f"magcache_b200: encoder_hid_proj.image_projection_layers[{a}] is not an ImageProjection "
                                          "(Linear to num_image_text_embeds x C, affine LayerNorm(C))")
            self.embeds.append(e[0].contiguous())
            self.n_keys.append(e.shape[1] * layer.num_image_text_embeds)
        if A > IP_ATTN_MAX_ADAPTERS or sum((n + 15) // 16 * 16 for n in self.n_keys) > IP_ATTN_MAX_KEYS:
            raise NotImplementedError(f"magcache_b200: {A} IP-Adapters with {self.n_keys} image-prompt tokens: the kernel holds at most "
                                      f"{IP_ATTN_MAX_ADAPTERS} adapters and {IP_ATTN_MAX_KEYS} tokens (each adapter's count "
                                      "rounded up to 16)")
        self.scales = []
        for i, p in enumerate(self.procs):
            if p is None:
                self.scales.append(None)
                continue
            s = list(p.scale) if isinstance(p.scale, (list, tuple)) else [p.scale]
            if not (len(s) == len(p.to_k_ip) == len(p.to_v_ip) == A):
                raise NotImplementedError(f"magcache_b200: transformer_blocks.{i}.attn.processor has {len(s)} scales, {len(p.to_k_ip)} "
                                          f"to_k_ip and {len(p.to_v_ip)} to_v_ip for {A} image projections")
            for lin in list(p.to_k_ip) + list(p.to_v_ip):
                wt = lin.weight
                if not (wt.dtype == torch.bfloat16 and wt.device == device and wt.shape == (dim, self.layers[0].norm.normalized_shape[0])
                        and wt.stride(1) == 1 and wt.stride(0) % 8 == 0):
                    raise NotImplementedError(f"magcache_b200: transformer_blocks.{i}.attn.processor weights must be bf16 "
                                              f"[{dim}, C] on {device}; got {wt.dtype} {tuple(wt.shape)} on {wt.device}")
            self.scales.append([float(x) for x in s])
        self.dim, self.device = dim, device

    def project(self):
        """`encoder_hid_proj(ip_adapter_image_embeds)`: per adapter LayerNorm(Linear(x).reshape(num_images * T, C)), on the GEMM
        and LayerNorm kernels. Returns the per-block launches for `MMDiTCore.run_blocks`."""
        f32 = torch.float32
        self.hidden = []
        for x, layer in zip(self.embeds, self.layers):
            lin, norm = layer.image_embeds, layer.norm
            y = ops.gemm(x, lin.weight, None if lin.bias is None else ops.cast(lin.bias, f32), E.MC_EPI_BIAS_BF16)
            y = y.view(-1, norm.normalized_shape[0])
            self.hidden.append(ops.ln_affine(y, ops.cast(norm.weight, f32), ops.cast(norm.bias, f32), eps=norm.eps))
        self.kv = torch.empty(sum(self.n_keys), 2 * self.dim, dtype=torch.bfloat16, device=self.device)
        return [None if p is None else (lambda q, nq, heads, out, i=i: self.attend(i, q, nq, heads, out)) for i, p in enumerate(self.procs)]

    def attend(self, i, q, nq, heads, out):
        """Double block `i`: every adapter's K | V rows from its `to_k_ip` / `to_v_ip`, then `mc_ip_attn` on the raw q into `out`."""
        D, f32, k0 = self.dim, torch.float32, 0
        p = self.procs[i]
        for h, n, tk, tv in zip(self.hidden, self.n_keys, p.to_k_ip, p.to_v_ip):
            for lin, cols in ((tk, slice(0, D)), (tv, slice(D, 2 * D))):
                ops.gemm(h, lin.weight, None if lin.bias is None else ops.cast(lin.bias, f32), E.MC_EPI_BIAS_BF16, out=self.kv[k0:k0 + n, cols])
            k0 += n
        ops.ip_attention(q, nq, heads, self.kv, self.n_keys, self.scales[i], out=out)


class MMDiTCore:
    """Workspace + block stack shared by the FLUX and HunyuanVideo engines. A subclass provides `self.w` (dim, heads, double, single,
    ada_w / ada_b / ada_rows), the token order (`txt_first`), the RoPE table of the rows that get RoPE, and its own prologue / head."""

    txt_first = True
    lora = None  # lora.LoraPack of the current call (FLUX with unmerged adapters), else None
    ip = None    # IPAdapterCall of the current call (FLUX with IP-Adapter processors), else None

    def _controlnet_views(self):
        """`run_blocks`' ControlNet argument for the current call; only the FLUX engine takes ControlNet residuals."""
        return None

    def _ip_blocks(self):
        """`run_blocks`' IP-Adapter argument for the current call (the image projection runs here, on a miss or calibration call only)."""
        return None if self.ip is None else self.ip.project()

    def _alloc_core(self, n_img, n_txt):
        """Buffers for one (image tokens, text tokens) shape. Token-sharded (`self.world > 1`, SURVEY §8e): the IMAGE rows are split over
        the ranks, the (few) text rows are replicated — every rank carries all of them and computes the identical text stream. Per
        attention the K|V rows of a rank's image tokens travel through the same exchange as the Wan engine's (`shard.make_exchange`:
        copy-engine pushes into every peer's gathered buffer, consumed segment by segment inside the attention kernel; or the
        all-gather formulation), and the text K|V rows are written locally behind the image rows of the gathered buffer — the key
        order [image | text] differs from the unsharded engine's, which a softmax over keys cannot see."""
        D, dev = self.w.dim, self.device
        bf = dict(dtype=torch.bfloat16, device=dev)
        self.n_img_total, self.n_txt = n_img, n_txt
        self.shard = None
        if getattr(self, "world", 1) > 1:
            from .shard import TokenShard
            self.shard = TokenShard(self.rank, self.world, n_img, self.group)
            if self.shard.pad:
                raise NotImplementedError(f"magcache_b200: {n_img} image tokens over {self.world} ranks needs the pad rule, built for the Wan engines only")
            n_img = self.shard.n_local
        S = n_img + n_txt                      # rows this rank carries
        Sg = self.n_img_total + n_txt          # keys every query attends to
        self.n_img, self.S, self.S_keys = n_img, S, Sg
        if self.txt_first:
            self.txt, self.img = slice(0, n_txt), slice(n_txt, S)
            self.txt_g, self.img_g = slice(0, n_txt), slice(n_txt, Sg)
        else:
            self.img, self.txt = slice(0, n_img), slice(n_img, S)
            self.img_g, self.txt_g = slice(0, self.n_img_total), slice(self.n_img_total, Sg)
        self.hs, self.h, self.att = torch.empty(S, D, **bf), torch.empty(S, D, **bf), torch.empty(S, D, **bf)
        self.x0, self.res, self.hit = torch.empty(n_img, D, **bf), torch.empty(n_img, D, **bf), torch.empty(n_img, D, **bf)
        if self.shard is None:
            self.qk = torch.empty(S, 2 * D, **bf)
            self.v = torch.empty(S, D, **bf)   # row-major V: the attention kernel consumes it as is (MN-major B operand)
        else:
            from .shard import make_exchange
            self.q_loc, self.k_loc = torch.empty(S, D, **bf), torch.empty(S, D, **bf)  # k_loc: the text refiner's own (local) keys
            self.xch = make_exchange(self.shard, 2 * D, (1,), dev, extra_rows=n_txt)
            self._xi, self._kv_cur = 0, None
        self.cat = torch.empty(S, 5 * D, **bf)
        self.ada = torch.empty(1, self.w.ada_rows, **bf)
        self.adaf = torch.empty(self.w.ada_rows, dtype=torch.float32, device=dev)
        self.res_valid = False

    def _em(self, start, k):
        D = self.w.dim
        return self.adaf[start:start + k * D].view(k, D)

    def _modulation_table(self, vec):
        """Every `Linear(silu(vec))` of the block stack (AdaLayerNormZero / ModulateDiT / final layer) from ONE GEMM: they depend on the
        conditioning vector only. bf16 like the reference, then an exact fp32 copy for the kernels that read modulation / gates."""
        w = self.w
        parts = w.ada_parts if self.lora is None or self.lora.ada_parts is None else self.lora.ada_parts
        if parts is None:
            ops.gemm(ops.silu(vec), w.ada_w, w.ada_b, E.MC_EPI_BIAS_BF16, out=self.ada)
        else:  # FP8 block rows and bf16 final-layer rows, or LoRA-adapted rows apart from the others: each output column still
            s = ops.silu(vec)  # comes from its own row of the stack
            self._down(self.lora.groups if self.lora is not None else {}, "ada", s)
            for r0, wt in parts:
                r1 = r0 + wt.shape[0]
                self._linear(s, wt, w.ada_b[r0:r1], E.MC_EPI_BIAS_BF16, out=self.ada[:, r0:r1])
        ops.cast_into(self.ada.view(-1), self.adaf)

    def _linear(self, a, wt, bias, epilogue, out, gate=None, addend=None, addend_row0=0):
        """A block Linear: bf16 or Fp8Weight (`linear`), through the weights' dequantisation scratch."""
        return linear(a, wt, bias, epilogue, out, gate=gate, scratch=self.w.fp8_scratch, addend=addend, addend_row0=addend_row0)

    def _rope_for(self, rows):
        """RoPE table rows for a token range, or None when that range gets no RoPE (HunyuanVideo text tokens)."""
        raise NotImplementedError

    @staticmethod
    def _down(groups, key, x):
        """The LoRA down-projection U = bf16(x A^T) of the adapters that read the GEMM input `x` (plain GEMM, no bias), if any."""
        g = groups.get(key)
        if g is not None:
            g.u, g.src = ops.gemm(x, g.A), x

    # ------------------------------------------------------------------------------------------ attention over the joint sequence
    def _project(self, rows, h_rows, qk_w, qk_b, v_w, v_b):
        """q | k and V projections of the token range `rows` from its LN+modulate output."""
        D = self.w.dim
        if self.shard is not None:
            # K | V straight into the exchange's gathered buffer: image rows into this rank's segment (pushed to the peers by
            # `_joint_attention`), text rows into the local tail; q stays local
            own, tail = self._kv_views()
            self._linear(h_rows, qk_w[:D], qk_b[:D], E.MC_EPI_BIAS_BF16, out=self.q_loc[rows])
            if rows == self.img:
                parts = ((h_rows, own),)
            elif rows == self.txt:
                parts = ((h_rows, tail),)
            else:  # the whole local sequence (single-stream blocks)
                parts = ((h_rows[self.img], own), (h_rows[self.txt], tail))
            for hp, dst in parts:
                self._linear(hp, qk_w[D:], qk_b[D:], E.MC_EPI_BIAS_BF16, out=dst[:, :D])
                self._linear(hp, v_w, v_b, E.MC_EPI_BIAS_BF16, out=dst[:, D:])
            return
        if isinstance(qk_w, tuple):  # (q, k) weights read in place (QwenImageWeights): one GEMM into each half of qk
            for i, wt in enumerate(qk_w):
                self._linear(h_rows, wt, qk_b[i * D:(i + 1) * D], E.MC_EPI_BIAS_BF16, out=self.qk[rows][:, i * D:(i + 1) * D])
        else:
            self._linear(h_rows, qk_w, qk_b, E.MC_EPI_BIAS_BF16, out=self.qk[rows])
        self._linear(h_rows, v_w, v_b, E.MC_EPI_BIAS_BF16, out=self.v[rows])

    def _qk_norm(self, rows, nq, nk):
        """Per-head RMSNorm of q and k (+ RoPE where the family applies it), in place."""
        D, H = self.w.dim, self.w.heads
        rope = self._rope_for(rows)
        if self.shard is not None:
            own, tail = self._kv_views()
            q, k = self.q_loc[rows], (own if rows == self.img else tail)[:, :D]
        else:
            q, k = self.qk[rows][:, :D], self.qk[rows][:, D:]
        ops.rmsnorm_head_rope_(q, nq, H, rope)
        ops.rmsnorm_head_rope_(k, nk, H, rope)

    def _kv_views(self):
        """(this rank's image segment, the local text tail) of the gathered K|V buffer the NEXT joint attention reads, [rows, 2 D]."""
        if self._kv_cur is None:
            self._kv_cur = (self.xch.own_rows(self._xi), self.xch.tail_rows(self._xi))
        return self._kv_cur

    def _joint_attention(self, out):
        D, H = self.w.dim, self.w.heads
        if self.shard is not None:
            xi = self._xi
            self.xch.begin(xi)  # this rank's normalised image K|V rows start travelling to the peers
            kv_all, kw = self.xch.keys_values(xi)
            ops.attention(self.q_loc, kv_all[:, :D], kv_all[:, D:], H, out=out, tag="mmdit_attn", **kw)
            self._xi, self._kv_cur = xi ^ 1, None
            return
        ops.attention(self.qk[:, :D], self.qk[:, D:], self.v, H, out=out, tag="mmdit_attn")

    def _gather_output(self, o_local):
        """Per-token head output of this rank's image rows -> all image rows, replicated (tiny: 64 features per token)."""
        if self.shard is None:
            return o_local
        from .shard import gather_rows
        full = torch.empty(self.n_img_total, o_local.shape[1], dtype=o_local.dtype, device=o_local.device)
        gather_rows(o_local.contiguous(), full, self.shard.group)
        return full

    def run_blocks(self, ctrl=None, ip=None):
        """Double-stream then single-stream blocks (magcache_flux.py:343-424; magcache_sample_video.py:108-139) on `hs`; the image rows of
        `hs` must hold the embedded image tokens and the text rows the embedded text. Returns the image rows.

        `ctrl`: None, or (double, single) lists with one entry per block — a bf16 [n_img, D] view (this rank's image rows) added to
        the image stream after that block (FLUX ControlNet residuals, magcache_flux.py:374-384 / :416-423), or None. The addition is
        fused into the block's last GEMM on the image rows (MC_EPI_BIAS_GATE_RESID_ADD_BF16): FF2 of the image stream of a double
        block, the `out` GEMM of a single block from row n_txt on (text rows first, FLUX only).

        `ip`: None, or one entry per double block — None, or `f(q, norm_q weight, heads, out)` writing the block's IP-Adapter
        attention output (IPAdapterCall.attend) from the raw q of this rank's image rows, before `_qk_norm` overwrites q. The
        output goes to cat[img, :D] (free in double blocks) and is added after the image stream's feed-forward residual as FF2's
        addend; a ControlNet sample of the same block is added afterwards in its own bf16 add, the reference's order."""
        w, D, S = self.w, self.w.dim, self.S
        double, single = (w.double, w.single) if self.lora is None else (self.lora.double, self.lora.single)
        c_double, c_single = ctrl if ctrl is not None else ((None,) * len(w.double), (None,) * len(w.single))
        c_ip = ip if ip is not None else (None,) * len(w.double)
        txt, img = self.txt, self.img
        hs, h = self.hs, self.h
        down = self._down
        for b, add, ipf in zip(double, c_double, c_ip):
            lg = b.get("lora", {})  # this block's LoRA down-projections, keyed by the GEMM input they read
            em, emc = self._em(b["ada"], 6), self._em(b["ada_c"], 6)  # (shift1, scale1, gate1, shift2, scale2, gate2)
            ops.ln_modulate(hs[img], em, 1, 0, round_ln_to_bf16=True, out=h[img])
            ops.ln_modulate(hs[txt], emc, 1, 0, round_ln_to_bf16=True, out=h[txt])
            down(lg, "h", h[img])
            down(lg, "ch", h[txt])
            self._project(img, h[img], b["qk_w"], b["qk_b"], b["v_w"], b["v_b"])
            self._project(txt, h[txt], b["cqk_w"], b["cqk_b"], b["cv_w"], b["cv_b"])
            ip_out = None
            if ipf is not None:
                ip_out = self.cat[img][:, :D]
                ipf(self.qk[img][:, :D] if self.shard is None else self.q_loc[img], b["nq"], w.heads, ip_out)
            self._qk_norm(img, b["nq"], b["nk"])
            self._qk_norm(txt, b["cnq"], b["cnk"])
            self._joint_attention(self.att)
            down(lg, "att", self.att[img])
            down(lg, "catt", self.att[txt])
            self._linear(self.att[img], b["o_w"], b["o_b"], E.MC_EPI_BIAS_GATE_RESID_BF16, out=hs[img], gate=em[2])
            self._linear(self.att[txt], b["co_w"], b["co_b"], E.MC_EPI_BIAS_GATE_RESID_BF16, out=hs[txt], gate=emc[2])
            for rows, e, f1w, f1b, f2w, f2b, pre in ((img, em, b["ff1_w"], b["ff1_b"], b["ff2_w"], b["ff2_b"], ""),
                                                     (txt, emc, b["cff1_w"], b["cff1_b"], b["cff2_w"], b["cff2_b"], "c")):
                ops.ln_modulate(hs[rows], e, 4, 3, round_ln_to_bf16=True, out=h[rows])
                down(lg, pre + "h2", h[rows])
                ffh = self.cat[rows][:, D:]
                self._linear(h[rows], f1w, f1b, E.MC_EPI_BIAS_GELU_BF16, out=ffh)
                down(lg, pre + "ffh", ffh)
                if rows != img:
                    self._linear(ffh, f2w, f2b, E.MC_EPI_BIAS_GATE_RESID_BF16, out=hs[rows], gate=e[5])
                    continue
                self._linear(ffh, f2w, f2b, E.MC_EPI_BIAS_GATE_RESID_BF16, out=hs[rows], gate=e[5], addend=add if ip_out is None else ip_out)
                if ip_out is not None and add is not None:
                    ops.cache_hit_add(hs[img], add.contiguous(), out=hs[img])
        allr = slice(0, S)
        for b, add in zip(single, c_single):
            lg = b.get("lora", {})
            em = self._em(b["ada"], 3)  # (shift, scale, gate)
            ops.ln_modulate(hs, em, 1, 0, round_ln_to_bf16=True, out=h)
            down(lg, "h", h)
            self._linear(h, b["mlp_w"], b["mlp_b"], E.MC_EPI_BIAS_GELU_BF16, out=self.cat[:, D:])
            self._project(allr, h, b["qk_w"], b["qk_b"], b["v_w"], b["v_b"])
            self._qk_norm(img, b["nq"], b["nk"])
            self._qk_norm(txt, b["nq"], b["nk"])
            self._joint_attention(self.cat[:, :D])
            down(lg, "cat", self.cat)
            self._linear(self.cat, b["out_w"], b["out_b"], E.MC_EPI_BIAS_GATE_RESID_BF16, out=hs, gate=em[2], addend=add,
                         addend_row0=self.n_txt)
        return hs[img]

    def _time_mlp(self, x_bf16, mlp):
        w1, b1, w2, b2 = mlp
        return ops.gemm(ops.gemm(x_bf16, w1, b1, E.MC_EPI_BIAS_SILU_BF16), w2, b2, E.MC_EPI_BIAS_BF16)

    def _sinusoid(self, t64):
        """256-channel [cos | sin] timestep embedding of a float64 device scalar, rounded to bf16 (`.to(dtype=...)` in both families)."""
        f = ops.time_sinusoid(t64, 256)
        return ops.cast_into(f, torch.empty(1, 256, dtype=torch.bfloat16, device=self.device))

    def forward(self, kind):
        """prologue -> {hit: x0 + cached residual | miss: block stack, residual = x - x0} -> family head."""
        x0 = self.prologue()
        if kind == "hit":
            if not self.res_valid:
                raise TypeError("magcache_b200: cache hit with an empty residual cache (reference: Tensor + NoneType)")
            x = ops.cache_hit_add(x0, self.res, out=self.hit)                     # magcache_flux.py:340 ; magcache_sample_video.py:104
        else:
            self.hs[self.img].copy_(x0)                                           # `ori_hidden_states` / `ori_img` stays in x0
            x = self.run_blocks(self._controlnet_views(), self._ip_blocks())
            if self.shard is not None:
                self.xch.join()  # every push of this forward is ordered before its end
            ops.residual_sub(x.contiguous(), x0, out=self.res)                    # :426 ; :140 (x is a contiguous row range of hs)
            self.res_valid = True
        return self.head(x)


    def calibrate(self):
        """The calibration twin of `forward("miss")` (magcache_flux.py:21-231; magcache_sample_video.py:163-290): always runs the block
        stack; returns (head output, (norm_ratio, norm_std, cos_dis) against the previous residual or None on the first call). The
        statistics come from the fused fp32/fp64 reduction kernel — finer than the reference's bf16 tensor ops, which quantise them to
        multiples of 2^-8 (the shipped FLUX table is visibly bf16-quantised, SURVEY §8a row 9)."""
        x0 = self.prologue()
        self.hs[self.img].copy_(x0)
        x = self.run_blocks(self._controlnet_views(), self._ip_blocks())
        reduce = None
        if self.shard is not None:  # the statistics are sums over the image tokens: add the partial sums of every token shard
            from .shard import allreduce_stats
            self.xch.join()
            reduce = lambda st: allreduce_stats(st, self.shard.group)  # noqa: E731
        new = self.hit
        ops.residual_sub(x.contiguous(), x0, out=new)
        stats = ops.residual_stats(new, self.res, reduce=reduce) if self.res_valid else None
        self.res, self.hit = new, self.res
        self.res_valid = True
        return self.head(x), stats


class FluxEngine(MMDiTCore):
    txt_first = True

    def __init__(self, weights: FluxWeights, shard_world=1, shard_rank=0, shard_group=None):
        self.w, self.device = weights, weights.device
        self.world, self.rank, self.group = shard_world, shard_rank, shard_group
        self._shape = None
        self._rope_key, self._rope = None, None
        self.res_valid = False
        self.controlnet = (None, None, False)
        self._lora_scan, self._lora_merged, self._lora_wrappers = None, (), ()
        self.ip = None

    def sync_lora(self, module):
        """Take the module's unmerged LoRA adapters as they are now (lora.FluxLoraScan): called at every forward, after the
        reference's `scale_lora_layers`. Base weights are repacked from the module when a merge or unmerge happened since they
        were packed, and when a LoRA layer seen before has left the module (it may have been merged first: `fuse_lora()` then
        `unload_lora_weights()`); otherwise only what changed is repacked (lora.LoraPack)."""
        first = self._lora_scan is None
        if first:
            self._lora_scan = FluxLoraScan(module)
        spec, merged, wrappers, changed = self._lora_scan.scan()
        now = {id(m) for m in wrappers}
        if not first and (merged != self._lora_merged or any(id(m) not in now for m in self._lora_wrappers)):
            self.w = FluxWeights.from_module(module, self.device)
            self.lora, changed = None, True
        # the layers themselves are kept (not their ids), so an id cannot be reused by a new layer before the next comparison
        self._lora_merged, self._lora_wrappers = merged, wrappers
        if changed:
            self.lora = LoraPack(self.w, spec, self.lora) if spec else None

    def _workspace(self, n_img, n_txt):
        if self._shape == (n_img, n_txt):
            return
        bf = dict(dtype=torch.bfloat16, device=self.device)
        self._alloc_core(n_img, n_txt)
        self.s_hidden = torch.empty(self.n_img, self.w.in_channels, **bf)  # this rank's image tokens
        self.s_enc = torch.empty(n_txt, self.w.joint_dim, **bf)
        self.s_pooled = torch.empty(1, self.w.pooled_dim, **bf)
        self.s_t = torch.zeros(2, dtype=torch.float64, device=self.device)  # timestep*1000, guidance*1000 (already rounded like the reference)
        self._shape = (n_img, n_txt)

    def _rope_for(self, rows):
        if self.shard is None:
            return self._rope[rows]
        if rows == self.txt:
            return self._rope[self.txt_g]
        if rows == self.img:  # this rank's image rows sit at their GLOBAL positions in the table (text rows first)
            return self._rope[self.n_txt + self.shard.start:self.n_txt + self.shard.stop]
        return torch.cat([self._rope[self.txt_g], self._rope[self.n_txt + self.shard.start:self.n_txt + self.shard.stop]])

    # ------------------------------------------------------------------------------------------ inputs (:290-319)
    def stage_inputs(self, hidden_states, encoder_hidden_states, pooled, timestep, guidance, img_ids, txt_ids):
        w = self.w
        assert hidden_states.shape[0] == 1 and encoder_hidden_states.shape[0] == 1, "one sample per call"
        n_img, n_txt = hidden_states.shape[1], encoder_hidden_states.shape[1]
        self._workspace(n_img, n_txt)
        self.s_hidden.copy_(hidden_states[0] if self.shard is None else self.shard.rows(hidden_states[0]))
        self.s_enc.copy_(encoder_hidden_states[0])
        self.s_pooled.copy_(pooled.reshape(1, -1))
        if (w.guidance and guidance is None) or (not w.guidance and guidance is not None):
            raise ValueError("guidance must be given exactly when the model has guidance_embeds")
        # `timestep.to(hidden_states.dtype) * 1000` (:292-294): both the cast and the product round to bf16
        tv = (timestep.reshape(-1)[:1].to(torch.bfloat16) * 1000).double()
        gv = (guidance.reshape(-1)[:1].to(torch.bfloat16) * 1000).double() if guidance is not None else torch.zeros(1, dtype=torch.float64, device=tv.device)
        self.s_t.copy_(torch.cat([tv, gv.to(tv.device)]))
        if self._rope_key is None or not self._rope_key.matches(img_ids, txt_ids):  # ids are constant over a generation
            self._rope = rope_table(torch.cat((txt_ids.reshape(-1, 3), img_ids.reshape(-1, 3)), dim=0), self.device)  # :318
            self._rope_key = InputKey(img_ids, txt_ids)
        assert self._rope.shape == (self.S_keys, 128)

    def stage_controlnet(self, block_samples, single_block_samples, blocks_repeat=False):
        """The call's ControlNet residuals (`controlnet_block_samples`, `controlnet_single_block_samples`,
        `controlnet_blocks_repeat`). Kept as given: they are validated and read only when the block stack runs (a miss or a
        calibration call); a hit ignores them, as the reference does."""
        self.controlnet = (block_samples, single_block_samples, bool(blocks_repeat))

    def stage_ip_adapter(self, module, embeds):
        """The call's IP-Adapter side path: the module's processors, scales and weights as they are now, and the call's
        `ip_adapter_image_embeds` (or None). Checked here, on every call; the projections run only when the block stack runs (a
        hit cannot reach their output). A model without IP-Adapter processors and a call without embeds stage nothing."""
        procs = [ip_processor(b.attn, f"transformer_blocks.{i}.attn") for i, b in enumerate(module.transformer_blocks)]
        for i, b in enumerate(module.single_transformer_blocks):
            if ip_processor(b.attn, f"single_transformer_blocks.{i}.attn") is not None:
                raise NotImplementedError(f"magcache_b200: single_transformer_blocks.{i}.attn has an IP-Adapter processor; FLUX's "
                                          "single blocks take no image prompt")
        self.ip = None
        if embeds is not None or any(p is not None for p in procs):
            self.ip = IPAdapterCall(module, procs, embeds, self.w.dim, self.device)

    def _controlnet_sample(self, sample, what):
        """This rank's rows of one sample as a [n_img, D] view (no copy). Only a CUDA bf16 [1, n_img, D] tensor with unit column
        stride is taken: the reference's `hidden_states + sample` would broadcast other shapes and promote an fp32 sample, changing
        the stream's dtype."""
        want = (1, self.n_img_total, self.w.dim)
        if not (torch.is_tensor(sample) and sample.is_cuda and sample.device == self.hs.device and sample.dtype == torch.bfloat16
                and tuple(sample.shape) == want and sample.stride(-1) == 1):
            got = (f"{sample.dtype} {tuple(sample.shape)} on {sample.device}" if torch.is_tensor(sample) else type(sample).__name__)
            raise NotImplementedError(f"magcache_b200: {what} must be a bf16 CUDA tensor of shape {list(want)} with unit column stride "
                                      f"on {self.hs.device}; got {got}")
        return sample[0] if self.shard is None else sample[0, self.shard.start:self.shard.stop]

    def _controlnet_views(self):
        block_samples, single_samples, repeat = self.controlnet
        if block_samples is None and single_samples is None:
            return None
        w = self.w
        views = []
        for samples, blocks, rep, name in ((block_samples, w.double, repeat, "controlnet_block_samples"),
                                           (single_samples, w.single, False, "controlnet_single_block_samples")):
            if samples is None:
                views.append([None] * len(blocks))
                continue
            idx = [controlnet_index(i, len(blocks), len(samples), rep) for i in range(len(blocks))]
            views.append([self._controlnet_sample(samples[j], f"{name}[{j}]") for j in idx])
        return tuple(views)

    def prologue(self):
        """x_embedder, time_text_embed, context_embedder (:290-303) and every AdaLayerNorm projection of the forward."""
        w = self.w
        top, lg = (self.lora.top, self.lora.groups) if self.lora is not None else ({"x_w": w.x_w, "ctx_w": w.ctx_w}, {})
        self._down(lg, "x", self.s_hidden)
        self._linear(self.s_hidden, top["x_w"], w.x_b, E.MC_EPI_BIAS_BF16, out=self.x0)
        temb = self._time_mlp(self._sinusoid(self.s_t[0:1]), w.t_mlp)
        if w.guidance:
            temb = ops.cache_hit_add(temb, self._time_mlp(self._sinusoid(self.s_t[1:2]), w.g_mlp))
        temb = ops.cache_hit_add(temb, self._time_mlp(self.s_pooled, w.p_mlp))
        self._modulation_table(temb)
        self._down(lg, "ctx", self.s_enc)
        self._linear(self.s_enc, top["ctx_w"], w.ctx_b, E.MC_EPI_BIAS_BF16, out=self.hs[self.txt])
        return self.x0

    def head(self, x_img):
        """`norm_out(hidden_states, temb)`, `proj_out` (:429-430): AdaLayerNormContinuous chunks (scale, shift) in that order."""
        w = self.w
        em = self._em(w.ada_out, 2)
        ops.ln_modulate(x_img, em, 0, 1, round_ln_to_bf16=True, out=self.h[self.img])
        if self.lora is None:
            return self._gather_output(ops.gemm(self.h[self.img], w.out_w, w.out_b, E.MC_EPI_BIAS_BF16))
        self._down(self.lora.groups, "head", self.h[self.img])
        return self._gather_output(self._linear(self.h[self.img], self.lora.top["out_w"], w.out_b, E.MC_EPI_BIAS_BF16, out=None))


# ======================================================================================================================
# HunyuanVideo
# ======================================================================================================================
def _fp8_blocks(m):
    """True when `m` is an FP8 checkpoint as upstream's `convert_fp8_linear` leaves it: every Linear under `double_blocks` /
    `single_blocks` holds float8_e4m3fn codes and an `fp8_scale`. False for a module without FP8 parameters."""
    f8 = {name for name, p in m.named_parameters() if p.dtype == torch.float8_e4m3fn}
    if not f8:
        return False
    lins = {name for name, mod in m.named_modules()
            if name.startswith(("double_blocks.", "single_blocks.")) and isinstance(mod, torch.nn.Linear)}
    outside = sorted(f8 - {f"{n}.weight" for n in lins})
    if outside:
        raise NotImplementedError(f"magcache_b200: FP8 parameters outside the block Linears are not supported: {outside[:4]}")
    missing = sorted(n for n in lins if m.get_submodule(n).weight.dtype != torch.float8_e4m3fn)
    if missing:
        raise NotImplementedError(f"magcache_b200: an FP8 checkpoint must hold every block Linear in FP8; bf16: {missing[:4]}")
    no_scale = sorted(n for n in lins if getattr(m.get_submodule(n), "fp8_scale", None) is None)
    if no_scale:
        raise ValueError(f"magcache_b200: FP8 weight without `fp8_scale` (upstream convert_fp8_linear sets it): {no_scale[:4]}")
    return True


def _fp8_scratch(w, dev):
    """bf16 scratch for the largest FP8 weight one GEMM reads (linear2 of a single block, D x 5D: linear1 is read as its q|k, v and
    mlp row blocks); the modulation table goes through it in row blocks."""
    n = max(v.q.numel() for blk in w.double + w.single for v in blk.values() if isinstance(v, Fp8Weight))
    return torch.empty(n, dtype=torch.bfloat16, device=dev)


class HunyuanWeights:
    """Weights of one HYVideoDiffusionTransformer (hyvideo attribute names), repacked like FluxWeights: fused qkv / linear1 matrices
    split into q|k, v (and mlp) row blocks, every ModulateDiT / final adaLN projection stacked into one matrix.

    An FP8 checkpoint (upstream `convert_fp8_linear`: every Linear under `double_blocks` / `single_blocks` holds float8_e4m3fn codes
    and a bf16 `fp8_scale`) stays in FP8: the block weights become `Fp8Weight`s — row blocks of the module's own codes, 1 byte per
    parameter, no bf16 copy — the block modulation rows are stacked as codes with a per-row scale (`ada_parts`), and one bf16
    scratch for the largest weight a GEMM reads (`fp8_scratch`) is allocated here, once."""

    ada_parts = None    # bf16 weights: the modulation table is one GEMM over `ada_w`
    fp8_scratch = None

    def __init__(self):
        self.double, self.single, self.refiner = [], [], []

    @classmethod
    def from_module(cls, m, dev):
        for name, mod in m.named_modules():  # HunyuanVideo's reference forward has no LoRA path
            if is_lora_layer(mod):
                raise NotImplementedError(f"magcache_b200: the HunyuanVideo engine runs no LoRA adapters; {name} carries one "
                                          "(merge it into the weights first)")
        w = cls()
        w.dim = D = m.hidden_size
        w.heads = m.heads_num
        if D // w.heads != 128:
            raise NotImplementedError("HunyuanVideo engine: head_dim 128")
        if list(m.patch_size) != [1, 2, 2] or m.text_projection != "single_refiner":
            raise NotImplementedError("HunyuanVideo engine: patch (1, 2, 2) and the single_refiner text projection")
        w.in_channels, w.out_channels, w.guidance = m.in_channels, m.out_channels, bool(m.guidance_embed)
        w.patch_w, w.patch_b = _w(m.img_in.proj.weight.flatten(1), dev), _b(m.img_in.proj.bias, dev)

        def mlp2(a, b_):
            return (_w(a.weight, dev), _b(a.bias, dev), _w(b_.weight, dev), _b(b_.bias, dev))

        w.t_mlp = mlp2(m.time_in.mlp[0], m.time_in.mlp[2])
        w.p_mlp = mlp2(m.vector_in.in_layer, m.vector_in.out_layer)
        w.g_mlp = mlp2(m.guidance_in.mlp[0], m.guidance_in.mlp[2]) if w.guidance else None
        w.pooled_dim = m.vector_in.in_layer.in_features
        r = m.txt_in
        w.text_dim = r.input_embedder.in_features
        w.r_in_w, w.r_in_b = _w(r.input_embedder.weight, dev), _b(r.input_embedder.bias, dev)
        w.r_t_mlp = mlp2(r.t_embedder.mlp[0], r.t_embedder.mlp[2])
        w.r_c_mlp = mlp2(r.c_embedder.linear_1, r.c_embedder.linear_2)
        r_ada_w, r_ada_b = [], []
        for blk in r.individual_token_refiner.blocks:
            W = blk.self_attn_qkv.weight
            Bq = blk.self_attn_qkv.bias
            w.refiner.append({
                "n1_w": _b(blk.norm1.weight, dev), "n1_b": _b(blk.norm1.bias, dev), "n2_w": _b(blk.norm2.weight, dev), "n2_b": _b(blk.norm2.bias, dev),
                "qk_w": _w(W[:2 * D], dev), "qk_b": _b(Bq[:2 * D], dev), "v_w": _w(W[2 * D:], dev), "v_b": _b(Bq[2 * D:], dev),
                "nq": _b(blk.self_attn_q_norm.weight, dev), "nk": _b(blk.self_attn_k_norm.weight, dev),
                "o_w": _w(blk.self_attn_proj.weight, dev), "o_b": _b(blk.self_attn_proj.bias, dev),
                "f1_w": _w(blk.mlp.fc1.weight, dev), "f1_b": _b(blk.mlp.fc1.bias, dev), "f2_w": _w(blk.mlp.fc2.weight, dev), "f2_b": _b(blk.mlp.fc2.bias, dev),
            })
            r_ada_w.append(blk.adaLN_modulation[1].weight.detach())
            r_ada_b.append(blk.adaLN_modulation[1].bias.detach())
        w.r_ada_w, w.r_ada_b = _w(torch.cat(r_ada_w, 0), dev), _b(torch.cat(r_ada_b, 0), dev)
        ada_w, ada_b, ada_lins, off = [], [], [], 0
        fp8 = _fp8_blocks(m)

        def lw(lin, rows=slice(None)):
            """A block Linear's weight (row block `rows`): bf16, or in FP8 as views of the module's own codes."""
            if not fp8:
                return _w(lin.weight[rows], dev)
            q = lin.weight.detach()[rows].to(dev)
            return Fp8Weight(q, lin.fp8_scale.detach().to(device=dev, dtype=torch.bfloat16).reshape(1).expand(q.shape[0]).contiguous())

        def ada(lin):
            nonlocal off
            ada_w.append(lin.weight.detach())
            ada_b.append(lin.bias.detach())
            ada_lins.append(lin)
            start, off = off, off + lin.weight.shape[0]
            return start

        for blk in m.double_blocks:
            d = {"ada": ada(blk.img_mod.linear), "ada_c": ada(blk.txt_mod.linear)}
            for pre, key in (("img", ""), ("txt", "c")):
                qkv, proj, mlp = getattr(blk, f"{pre}_attn_qkv"), getattr(blk, f"{pre}_attn_proj"), getattr(blk, f"{pre}_mlp")
                Bq = qkv.bias
                d.update({f"{key}qk_w": lw(qkv, slice(0, 2 * D)), f"{key}qk_b": _b(Bq[:2 * D], dev), f"{key}v_w": lw(qkv, slice(2 * D, None)), f"{key}v_b": _b(Bq[2 * D:], dev),
                          f"{key}nq": _b(getattr(blk, f"{pre}_attn_q_norm").weight, dev), f"{key}nk": _b(getattr(blk, f"{pre}_attn_k_norm").weight, dev),
                          f"{key}o_w": lw(proj), f"{key}o_b": _b(proj.bias, dev),
                          f"{key}ff1_w": lw(mlp.fc1), f"{key}ff1_b": _b(mlp.fc1.bias, dev),
                          f"{key}ff2_w": lw(mlp.fc2), f"{key}ff2_b": _b(mlp.fc2.bias, dev)})
            w.double.append(d)
        for blk in m.single_blocks:
            l1, Bq = blk.linear1, blk.linear1.bias
            w.single.append({
                "ada": ada(blk.modulation.linear),
                "qk_w": lw(l1, slice(0, 2 * D)), "qk_b": _b(Bq[:2 * D], dev), "v_w": lw(l1, slice(2 * D, 3 * D)), "v_b": _b(Bq[2 * D:3 * D], dev),
                "mlp_w": lw(l1, slice(3 * D, None)), "mlp_b": _b(Bq[3 * D:], dev), "nq": _b(blk.q_norm.weight, dev), "nk": _b(blk.k_norm.weight, dev),
                "out_w": lw(blk.linear2), "out_b": _b(blk.linear2.bias, dev),
            })
        w.ada_out = ada(m.final_layer.adaLN_modulation[1])
        w.ada_b, w.ada_rows = _b(torch.cat(ada_b, 0), dev), off
        if not fp8:
            w.ada_w = _w(torch.cat(ada_w, 0), dev)
        else:  # block rows stacked as codes (+ per-row scales), the final layer's rows stay bf16
            mods = [lw(lin) for lin in ada_lins[:-1]]
            q = torch.cat([x.q.view(torch.uint8) for x in mods], 0).view(torch.float8_e4m3fn)
            w.ada_parts = [(0, Fp8Weight(q, torch.cat([x.scale for x in mods], 0))), (w.ada_out, _w(ada_w[-1], dev))]
            w.fp8_scratch = _fp8_scratch(w, dev)
        w.out_w, w.out_b = _w(m.final_layer.linear.weight, dev), _b(m.final_layer.linear.bias, dev)
        w.device = dev
        return w


class HunyuanEngine(MMDiTCore):
    """Image tokens first, RoPE on the image tokens only, text tokens through the two-block token refiner. The padded text tokens form
    their own attention segment in the reference (`get_cu_seqlens`, magcache_sample_video.py:82) and never reach an image token, so only
    the valid ones are embedded and carried."""

    txt_first = False

    def __init__(self, weights: HunyuanWeights, shard_world=1, shard_rank=0, shard_group=None):
        self.w, self.device = weights, weights.device
        self.world, self.rank, self.group = shard_world, shard_rank, shard_group
        self._shape = None
        self._rope_key, self._rope = None, None
        self._mask_key, self._valid = None, None
        self.res_valid = False

    def _workspace(self, grid, n_txt):
        n_img = grid[0] * grid[1] * grid[2]
        if self._shape == (grid, n_txt):
            return
        w, dev = self.w, self.device
        bf = dict(dtype=torch.bfloat16, device=dev)
        self._alloc_core(n_img, n_txt)
        self.grid = grid
        self.s_lat = torch.empty(w.in_channels, grid[0], 2 * grid[1], 2 * grid[2], dtype=torch.float32, device=dev)
        self.s_txt = torch.empty(n_txt, w.text_dim, **bf)
        self.s_pooled = torch.empty(1, w.pooled_dim, **bf)
        self.s_t = torch.zeros(2, dtype=torch.float64, device=dev)
        self.rv = torch.empty(n_txt, w.dim, **bf)  # V of the token refiner's self-attention
        self.rada = torch.empty(1, w.r_ada_w.shape[0], **bf)
        self.radaf = torch.empty(w.r_ada_w.shape[0], dtype=torch.float32, device=dev)
        self._shape = (grid, n_txt)

    def _rope_for(self, rows):
        if rows != self.img or self._rope is None:
            return None  # the text tokens get no RoPE (magcache_sample_video.py:108-120 -> hyvideo blocks)
        return self._rope if self.shard is None else self._rope[self.shard.start:self.shard.stop]

    # ------------------------------------------------------------------------------------------ inputs (:42-86)
    def stage_inputs(self, x, t, text_states, text_mask, text_states_2, freqs_cos, freqs_sin, guidance):
        w = self.w
        assert x.shape[0] == 1 and text_states.shape[0] == 1, "one sample per call"
        _, c, ot, oh, ow = x.shape
        grid = (ot, oh // 2, ow // 2)
        if self._mask_key is None or not self._mask_key.matches(text_mask):  # the mask is constant over a generation: one host read
            m = text_mask.reshape(-1).to(torch.int64).cpu()
            valid = int(m.sum())
            if valid < 1 or not bool((m[:valid] == 1).all()):
                raise NotImplementedError("magcache_b200: the valid text tokens must be a non-empty prefix of text_states (right padding)")
            self._mask_key, self._valid = InputKey(text_mask), valid
        n_txt = self._valid
        self._workspace(grid, n_txt)
        self.s_lat.copy_(x[0])
        self.s_txt.copy_(text_states[0, :n_txt])
        self.s_pooled.copy_(text_states_2.reshape(1, -1))
        if w.guidance and guidance is None:
            raise ValueError("Didn't get guidance strength for guidance distilled model.")  # :58-61
        gv = guidance.reshape(-1)[:1].double() if guidance is not None else torch.zeros(1, dtype=torch.float64, device=t.device)
        self.s_t.copy_(torch.cat([t.reshape(-1)[:1].double(), gv.to(t.device)]))
        if freqs_cos is not None:
            n = self.n_img_total
            assert tuple(freqs_cos.shape) == (n, 128) and tuple(freqs_sin.shape) == (n, 128)
            if self._rope_key is None or not self._rope_key.matches(freqs_cos, freqs_sin):
                cs = torch.stack([freqs_cos.float()[:, 0::2], freqs_sin.float()[:, 0::2]], dim=-1).reshape(n, 128)
                self._rope, self._rope_key = cs.contiguous().to(self.device), InputKey(freqs_cos, freqs_sin)
        else:
            self._rope, self._rope_key = None, None

    # ------------------------------------------------------------------------------------------ token refiner (`self.txt_in`, :69)
    def _refine_text(self):
        """SingleTokenRefiner over the valid text tokens: c = t_embedder(t) + c_embedder(mean of the raw states); two blocks of
        LN(affine) -> qkv -> per-head RMSNorm -> self-attention -> gated proj, LN(affine) -> SiLU MLP -> gated; in place on hs[txt]."""
        w, D, H = self.w, self.w.dim, self.w.heads
        txt, n = self.txt, self.n_txt
        c = ops.cache_hit_add(self._time_mlp(self._sinusoid(self.s_t[0:1]), w.r_t_mlp), self._time_mlp(ops.colmean(self.s_txt), w.r_c_mlp))
        ops.gemm(ops.silu(c), w.r_ada_w, w.r_ada_b, E.MC_EPI_BIAS_BF16, out=self.rada)
        ops.cast_into(self.rada.view(-1), self.radaf)
        x, h = self.hs[txt], self.h[txt]
        ops.gemm(self.s_txt, w.r_in_w, w.r_in_b, E.MC_EPI_BIAS_BF16, out=x)
        sharded = self.shard is not None
        q, k = (self.q_loc[txt], self.k_loc[txt]) if sharded else (self.qk[txt][:, :D], self.qk[txt][:, D:])
        rv = self.rv[:n]
        for i, b in enumerate(w.refiner):
            g = self.radaf[i * 2 * D:(i + 1) * 2 * D].view(2, D)  # gate_msa, gate_mlp
            ops.ln_affine(x, b["n1_w"], b["n1_b"], eps=1e-6, out=h)
            if sharded:
                ops.gemm(h, b["qk_w"][:D], b["qk_b"][:D], E.MC_EPI_BIAS_BF16, out=q)
                ops.gemm(h, b["qk_w"][D:], b["qk_b"][D:], E.MC_EPI_BIAS_BF16, out=k)
            else:
                ops.gemm(h, b["qk_w"], b["qk_b"], E.MC_EPI_BIAS_BF16, out=self.qk[txt])
            ops.gemm(h, b["v_w"], b["v_b"], E.MC_EPI_BIAS_BF16, out=rv)
            ops.rmsnorm_head_rope_(q, b["nq"], H, None)
            ops.rmsnorm_head_rope_(k, b["nk"], H, None)
            ops.attention(q, k, rv, H, out=self.att[txt], tag="refiner_attn")
            ops.gemm(self.att[txt], b["o_w"], b["o_b"], E.MC_EPI_BIAS_GATE_RESID_BF16, out=x, gate=g[0])
            ops.ln_affine(x, b["n2_w"], b["n2_b"], eps=1e-6, out=h)
            ffh = self.cat[txt][:, D:]
            ops.gemm(h, b["f1_w"], b["f1_b"], E.MC_EPI_BIAS_SILU_BF16, out=ffh)
            ops.gemm(ffh, b["f2_w"], b["f2_b"], E.MC_EPI_BIAS_GATE_RESID_BF16, out=x, gate=g[1])

    def prologue(self):
        """time_in + vector_in (+ guidance_in), img_in, txt_in (:52-69) and the modulation table of the whole block stack."""
        w = self.w
        vec = ops.cache_hit_add(self._time_mlp(self._sinusoid(self.s_t[0:1]), w.t_mlp), self._time_mlp(self.s_pooled, w.p_mlp))
        if w.guidance:
            vec = ops.cache_hit_add(vec, self._time_mlp(self._sinusoid(self.s_t[1:2]), w.g_mlp))
        tok = ops.patchify(self.s_lat)
        ops.gemm(tok if self.shard is None else self.shard.rows(tok), w.patch_w, w.patch_b, E.MC_EPI_BIAS_BF16, out=self.x0)
        self._refine_text()
        self._modulation_table(vec)
        return self.x0

    def head(self, x_img):
        """`final_layer(img, vec)` (shift, scale in that order) and `unpatchify` (:144-146): [1, C, T, H, W] bf16."""
        w = self.w
        em = self._em(w.ada_out, 2)
        ops.ln_modulate(x_img, em, 1, 0, round_ln_to_bf16=True, out=self.h[self.img])
        o = self._gather_output(ops.gemm(self.h[self.img], w.out_w, w.out_b, E.MC_EPI_BIAS_BF16))  # [n_img, C*1*2*2], (c, pt, ph, pw)
        t, hh, ww = self.grid
        c = w.out_channels
        o = o.view(1, t, hh, ww, c, 1, 2, 2)
        return torch.einsum("nthwcopq->nctohpwq", o).reshape(1, c, t, 2 * hh, 2 * ww)  # pure data movement


# ======================================================================================================================
# Qwen-Image / Qwen-Image-Edit
# ======================================================================================================================
class QwenImageWeights:
    """Weights of one QwenImageTransformer2DModel (diffusers attribute names). Its 60 double blocks are FLUX double blocks statement
    for statement (per-stream `Linear(silu(temb))` -> (shift, scale, gate) x 2, LayerNorm without affine at eps 1e-6, biased
    q/k/v/o, per-head RMSNorm of q and k, interleaved-pair RoPE, joint attention over [txt | img], GELU(tanh) FF at 4 D), so they
    run on `MMDiTCore.run_blocks` with no single blocks.

    At 20 B parameters (40.9 GB in bf16) nothing large is copied: every block matrix is the module's own bf16 weight, read in
    place. The modulation rows stay one part per Linear (`ada_parts`; a stacked copy would be 13.6 GB), and q and k run as two
    GEMMs into the halves of `qk` instead of one over a fused q|k copy (4.5 GB): 240 more GEMM launches per miss, each over half
    the columns. The engine's own copies are the biases and norm weights, as fp32 (22 MB at full size)."""

    fp8_scratch = None

    def __init__(self):
        self.double, self.single = [], []

    @classmethod
    def from_module(cls, m, dev):
        for name, mod in m.named_modules():
            if is_lora_layer(mod):
                raise NotImplementedError(f"magcache_b200: the Qwen-Image engine runs no LoRA adapters; {name} carries one "
                                          "(merge it into the weights first)")
        cfg = m.config
        if cfg.attention_head_dim != 128 or tuple(cfg.axes_dims_rope) != (16, 56, 56):
            raise NotImplementedError("magcache_b200: the Qwen-Image engine needs head_dim 128 with RoPE axes (16, 56, 56)")
        if getattr(cfg, "guidance_embeds", False):
            raise NotImplementedError("magcache_b200: Qwen-Image with guidance_embeds is not supported (the released checkpoints have none)")
        for name, p in m.named_parameters():
            if p.dtype != torch.bfloat16 or p.device != dev:
                raise NotImplementedError(f"magcache_b200: the Qwen-Image engine reads the module's bf16 weights in place on {dev}; "
                                          f"{name} is {p.dtype} on {p.device}")
        w = cls()
        w.heads = cfg.num_attention_heads
        w.dim = D = w.heads * 128
        w.in_channels, w.joint_dim = cfg.in_channels, cfg.joint_attention_dim
        v = lambda t: t.detach()  # noqa: E731  (the module's own storage)

        def lin(l):
            return v(l.weight), _b(l.bias, dev)

        w.img_w, w.img_b = lin(m.img_in)
        w.txt_norm_w, w.txt_norm_eps = _b(m.txt_norm.weight, dev), m.txt_norm.eps
        w.txt_w, w.txt_b = lin(m.txt_in)
        te = m.time_text_embed.timestep_embedder
        w.t_mlp = (*lin(te.linear_1), *lin(te.linear_2))
        parts, ada_b, off = [], [], 0

        def ada(l):
            nonlocal off
            parts.append((off, v(l.weight)))
            ada_b.append(l.bias.detach())
            start, off = off, off + l.weight.shape[0]
            return start

        for blk in m.transformer_blocks:
            a = blk.attn
            d = {"ada": ada(blk.img_mod[1]), "ada_c": ada(blk.txt_mod[1])}
            for key, q, k, vv, o, nq, nk, mlp in (("", a.to_q, a.to_k, a.to_v, a.to_out[0], a.norm_q, a.norm_k, blk.img_mlp),
                                                  ("c", a.add_q_proj, a.add_k_proj, a.add_v_proj, a.to_add_out, a.norm_added_q,
                                                   a.norm_added_k, blk.txt_mlp)):
                d.update({f"{key}qk_w": (v(q.weight), v(k.weight)), f"{key}qk_b": _b(torch.cat([q.bias, k.bias]), dev),
                          f"{key}v_w": v(vv.weight), f"{key}v_b": _b(vv.bias, dev), f"{key}o_w": v(o.weight), f"{key}o_b": _b(o.bias, dev),
                          f"{key}nq": _b(nq.weight, dev), f"{key}nk": _b(nk.weight, dev),
                          f"{key}ff1_w": v(mlp.net[0].proj.weight), f"{key}ff1_b": _b(mlp.net[0].proj.bias, dev),
                          f"{key}ff2_w": v(mlp.net[2].weight), f"{key}ff2_b": _b(mlp.net[2].bias, dev)})
            w.double.append(d)
        w.ada_out = ada(m.norm_out.linear)
        w.ada_parts, w.ada_b, w.ada_rows = parts, _b(torch.cat(ada_b), dev), off
        w.out_w, w.out_b = lin(m.proj_out)
        w.device = dev
        return w


def qwen_img_shapes(img_shapes):
    """The image grids of a call as `QwenEmbedRope.forward` reads `img_shapes`: [(1, h, w)] (T2I) and [[(1, h, w), (1, h', w')]]
    (Edit: the noised latents, then the reference image) both give a tuple of (frames, height, width) per image."""
    fhw = img_shapes
    if isinstance(fhw, list):
        fhw = fhw[0]
    if not isinstance(fhw, list):
        fhw = [fhw]
    return tuple(tuple(int(x) for x in s) for s in fhw)


def qwen_rope_positions(shapes, n_txt):
    """(frame, height, width) position of every row of the joint sequence [txt | img] (diffusers `QwenEmbedRope`, scale_rope=True):
    image i takes frames i .. i+f-1, row r of an image of height h sits at r - (h - h//2) (centred; the width alike), and text
    token j at m + j on all three axes, m the largest h//2 or w//2 over the images. int64 [n_txt + sum f*h*w, 3]."""
    rows, m = [], 0
    for i, (f, h, w) in enumerate(shapes):
        fr = torch.arange(i, i + f)
        hr = torch.arange(h) - (h - h // 2)
        wr = torch.arange(w) - (w - w // 2)
        rows.append(torch.stack(torch.meshgrid(fr, hr, wr, indexing="ij"), dim=-1).reshape(-1, 3))
        m = max(m, h // 2, w // 2)
    txt = (m + torch.arange(n_txt))[:, None].expand(n_txt, 3)
    return torch.cat([txt] + rows, dim=0)


def qwen_rope_table(shapes, n_txt, device, axes_dim=(16, 56, 56), theta=10000):
    """cos / sin of `QwenEmbedRope` for the joint sequence [txt | img], [S, 128] fp32 as interleaved (cos, sin) pairs. Upstream
    forms each angle in fp32 (`torch.outer(index, 1 / theta ** (arange(0, d, 2) / d))`, then `torch.polar`); the same fp32
    angles are formed here and their cos / sin taken in float64, then rounded to fp32 — within one fp32 ulp of upstream's. This is
    not FLUX's `rope_table`, whose angles are float64."""
    pos = qwen_rope_positions(shapes, n_txt)
    ang = []
    for i, d in enumerate(axes_dim):
        inv = 1.0 / torch.pow(theta, torch.arange(0, d, 2).to(torch.float32).div(d))
        ang.append(torch.outer(pos[:, i].float(), inv))
    ang = torch.cat(ang, dim=1).double()  # [S, 64], fp32 values
    cs = torch.stack([ang.cos(), ang.sin()], dim=-1).reshape(len(pos), 128)
    return cs.float().to(device)


class QwenImageEngine(MMDiTCore):
    """The MMDiT block stack with Qwen-Image's prologue and head, and the per-CFG-branch state of its MagCache forward
    (MagCache4QwenImage/magcache_generate.py:173-252): the cond and the uncond call of a step have their own text length, so the
    engine keeps a workspace (and RoPE table) for each of the two most recent (image tokens, text tokens) shapes and one residual
    slot per branch (`residual_cache[cnt % 2]`), shared by the workspaces. After the first two calls of a generation nothing is
    allocated but each call's output.

    A hit (`hidden_states += residual_x`, then norm_out / proj_out, :221-247) runs img_in, the time MLP, the final layer's
    modulation rows, the add, LN+modulate and proj_out: it reads neither the block modulation weights nor the text path."""

    txt_first = True
    _WS = ("n_img_total", "n_txt", "shard", "n_img", "S", "S_keys", "txt", "img", "txt_g", "img_g", "hs", "h", "att", "x0", "hit",
           "qk", "v", "cat", "ada", "adaf", "s_hidden", "s_enc", "s_t", "_rope", "_rope_shapes")

    def __init__(self, weights: QwenImageWeights):
        self.w, self.device = weights, weights.device
        self.world = 1
        self._spaces = {}       # (n_img, n_txt) -> workspace attributes, most recently used last
        self._shape = None
        self.res, self.spare, self.res_valid = None, None, [False, False]
        self._masks = []        # InputKeys of the last text masks found all ones

    def _workspace(self, n_img, n_txt):
        key = (n_img, n_txt)
        if self._shape == key:
            return
        if self.res is None or self.res[0].shape[0] != n_img:  # the residual slots: one per CFG branch, for every text length
            D = self.w.dim
            self.res = [torch.empty(n_img, D, dtype=torch.bfloat16, device=self.device) for _ in range(2)]
            self.spare = torch.empty_like(self.res[0])  # the calibration twin's new residual, swapped into its slot
            self.res_valid = [False, False]
        ws = self._spaces.pop(key, None)
        if ws is None:
            while len(self._spaces) >= 2:
                self._spaces.pop(next(iter(self._spaces)))
            slots, valid = self.res, self.res_valid
            self._alloc_core(n_img, n_txt)
            self.res, self.res_valid = slots, valid  # (`_alloc_core`'s single residual buffer is not used)
            bf = dict(dtype=torch.bfloat16, device=self.device)
            self.s_hidden = torch.empty(n_img, self.w.in_channels, **bf)
            self.s_enc = torch.empty(n_txt, self.w.joint_dim, **bf)
            self.s_t = torch.empty(1, dtype=torch.float64, device=self.device)
            self._rope, self._rope_shapes = None, None
            ws = {k: getattr(self, k) for k in self._WS}
        self._spaces[key] = ws
        self.__dict__.update(ws)
        self._shape = key

    def _rope_for(self, rows):
        return self._rope[rows]

    def stage_inputs(self, hidden_states, encoder_hidden_states, encoder_hidden_states_mask, timestep, img_shapes, txt_seq_lens):
        """Checks and stages one call's inputs (one sample). Raises ValueError for `txt_seq_lens` other than [text tokens] and for
        image grids that do not add up to the image tokens; NotImplementedError for more than one sample and for a text mask with
        zeros (upstream's attention ignores the mask: its pipeline trims the prompt to the valid tokens of a one-prompt batch)."""
        if hidden_states.dim() != 3 or hidden_states.shape[0] != 1 or encoder_hidden_states.shape[0] != 1 or timestep.numel() != 1:
            raise NotImplementedError("magcache_b200: the Qwen-Image engine runs one sample per call (true CFG as two calls)")
        n_img, n_txt = hidden_states.shape[1], encoder_hidden_states.shape[1]
        if txt_seq_lens is None or list(txt_seq_lens) != [n_txt]:
            raise ValueError(f"magcache_b200: txt_seq_lens must be [{n_txt}] (the text tokens of the call); got {txt_seq_lens}")
        shapes = qwen_img_shapes(img_shapes)
        if sum(f * h * w for f, h, w in shapes) != n_img:
            raise ValueError(f"magcache_b200: img_shapes {list(shapes)} cover {sum(f * h * w for f, h, w in shapes)} tokens, "
                             f"hidden_states has {n_img}")
        m = encoder_hidden_states_mask
        if m is not None and not any(k.matches(m) for k in self._masks):  # one host read per new mask
            if tuple(m.shape) != (1, n_txt) or not bool((m == 1).all()):
                raise NotImplementedError("magcache_b200: encoder_hidden_states_mask must be None or all ones [1, text tokens]: "
                                          "padded prompts are not supported")
            self._masks = self._masks[-1:] + [InputKey(m)]
        self._workspace(n_img, n_txt)
        self.s_hidden.copy_(hidden_states[0])
        self.s_enc.copy_(encoder_hidden_states[0])
        # `timestep.to(bf16)` (:195), then Timesteps(256, scale=1000) forms 1000 * t * freq in fp32 [EXT diffusers]; the sinusoid
        # kernel takes float(bf16(t)) * 1000 and forms its arguments in float64 (finer than upstream's fp32, as for Open-Sora)
        self.s_t.copy_(timestep.reshape(1).to(torch.bfloat16).double() * 1000)
        if self._rope_shapes != shapes:
            self._rope, self._rope_shapes = qwen_rope_table(shapes, n_txt, self.device), shapes
            self._spaces[self._shape].update(_rope=self._rope, _rope_shapes=shapes)

    def prologue(self, full):
        """img_in and the time embedding (:194-202); on a miss or a calibration call (`full`) also the modulation table of every
        block and txt_norm -> txt_in into the text rows. A hit computes only the final layer's two modulation chunks."""
        w = self.w
        ops.gemm(self.s_hidden, w.img_w, w.img_b, E.MC_EPI_BIAS_BF16, out=self.x0)
        temb = self._time_mlp(self._sinusoid(self.s_t), w.t_mlp)
        if full:
            self._modulation_table(temb)
            ops.rmsnorm_rope_(self.s_enc, w.txt_norm_w, None, eps=w.txt_norm_eps)  # RMSNorm(3584): bf16(bf16(x rsqrt(ms + eps)) w)
            ops.gemm(self.s_enc, w.txt_w, w.txt_b, E.MC_EPI_BIAS_BF16, out=self.hs[self.txt])
        else:
            r0, r1 = w.ada_out, w.ada_out + 2 * w.dim
            ops.gemm(ops.silu(temb), w.ada_parts[-1][1], w.ada_b[r0:r1], E.MC_EPI_BIAS_BF16, out=self.ada[:, r0:r1])
            ops.cast_into(self.ada.view(-1)[r0:r1], self.adaf[r0:r1])
        return self.x0

    def head(self, x_img):
        """`norm_out(hidden_states, temb)` (AdaLayerNormContinuous: scale, shift in that order) and `proj_out` (:246-247)."""
        w = self.w
        ops.ln_modulate(x_img, self._em(w.ada_out, 2), 0, 1, round_ln_to_bf16=True, out=self.h[self.img])
        return ops.gemm(self.h[self.img], w.out_w, w.out_b, E.MC_EPI_BIAS_BF16)

    def forward(self, kind, slot):
        """hit: `hidden_states += residual_cache[slot]` (:221-222) | miss: the 60 blocks, residual into the slot (:224-239); then the
        head."""
        if kind == "hit":
            if not self.res_valid[slot]:
                raise TypeError("magcache_b200: cache hit with an empty residual cache (reference: Tensor += NoneType)")
            x = ops.cache_hit_add(self.prologue(full=False), self.res[slot], out=self.hit)
        else:
            x0 = self.prologue(full=True)
            self.hs[self.img].copy_(x0)
            x = self.run_blocks()
            ops.residual_sub(x, x0, out=self.res[slot])
            self.res_valid[slot] = True
        return self.head(x)

    def calibrate(self, slot, compare):
        """The calibration twin (:94-171): the blocks always run; with `compare`, (norm_ratio, norm_std, cos_dis) of the new
        residual against the slot's (fused fp32/fp64 reduction, finer than upstream's bf16 tensor ops), else None. The new residual
        then takes the slot."""
        x0 = self.prologue(full=True)
        self.hs[self.img].copy_(x0)
        x = self.run_blocks()
        new = self.spare
        ops.residual_sub(x, x0, out=new)
        stats = None
        if compare:
            if not self.res_valid[slot]:
                raise TypeError("magcache_b200: calibration statistics against an empty residual slot (reference: NoneType.norm)")
            stats = ops.residual_stats(new, self.res[slot])
        self.res[slot], self.spare = new, self.res[slot]
        self.res_valid[slot] = True
        return self.head(x), stats


# ======================================================================================================================
# Synthetic weights created directly on the device (benchmarks: a FLUX.1-dev / HunyuanVideo-sized nn.Module does not fit a CPU box)
# ======================================================================================================================
def _rand_block_weights(D, dev, g, keys_prefix=("", "c")):
    import math

    def xav(o, i, s=1.0):
        return ((torch.rand(o, i, device=dev, generator=g) * 2 - 1) * (s * math.sqrt(6.0 / (i + o)))).bfloat16()

    def bias(n):
        return (0.02 * torch.randn(n, device=dev, generator=g)).bfloat16().float()

    def nw():
        return (1 + 0.1 * torch.randn(128, device=dev, generator=g)).bfloat16().float()

    d = {}
    for k in keys_prefix:
        d.update({f"{k}qk_w": xav(2 * D, D), f"{k}qk_b": bias(2 * D), f"{k}v_w": xav(D, D), f"{k}v_b": bias(D), f"{k}o_w": xav(D, D), f"{k}o_b": bias(D),
                  f"{k}nq": nw(), f"{k}nk": nw(), f"{k}ff1_w": xav(4 * D, D), f"{k}ff1_b": bias(4 * D), f"{k}ff2_w": xav(D, 4 * D), f"{k}ff2_b": bias(D)})
    return d, xav, bias, nw


def _random_stack(w, D, n_double, n_single, dev, g):
    """Double / single block weights + the stacked modulation matrix (rows: 12D per double block, 3D per single block, 2D final)."""
    off = 0
    for _ in range(n_double):
        d, xav, bias, nw = _rand_block_weights(D, dev, g)
        d["ada"], d["ada_c"] = off, off + 6 * D
        off += 12 * D
        w.double.append(d)
    for _ in range(n_single):
        _, xav, bias, nw = _rand_block_weights(D, dev, g, keys_prefix=())
        w.single.append({"ada": off, "qk_w": xav(2 * D, D), "qk_b": bias(2 * D), "v_w": xav(D, D), "v_b": bias(D), "nq": nw(), "nk": nw(),
                         "mlp_w": xav(4 * D, D), "mlp_b": bias(4 * D), "out_w": xav(D, 5 * D), "out_b": bias(D)})
        off += 3 * D
    w.ada_out = off
    off += 2 * D
    _, xav, bias, nw = _rand_block_weights(D, dev, g, keys_prefix=())
    w.ada_w, w.ada_b, w.ada_rows = xav(off, D, 0.3), bias(off), off
    return xav, bias, nw


def random_flux_weights(dev, heads=24, num_layers=19, num_single_layers=38, in_channels=64, joint_dim=4096, pooled_dim=768, guidance=True, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    w = FluxWeights()
    w.heads, w.head_dim, w.dim = heads, 128, heads * 128
    D = w.dim
    w.in_channels, w.joint_dim, w.pooled_dim, w.guidance, w.device = in_channels, joint_dim, pooled_dim, guidance, dev
    xav, bias, _ = _random_stack(w, D, num_layers, num_single_layers, dev, g)
    w.x_w, w.x_b, w.ctx_w, w.ctx_b = xav(D, in_channels), bias(D), xav(D, joint_dim), bias(D)
    w.t_mlp = (xav(D, 256), bias(D), xav(D, D), bias(D))
    w.p_mlp = (xav(D, pooled_dim), bias(D), xav(D, D), bias(D))
    w.g_mlp = (xav(D, 256), bias(D), xav(D, D), bias(D)) if guidance else None
    w.out_w, w.out_b = xav(in_channels, D), bias(in_channels)
    return w


def random_hunyuan_weights(dev, heads=24, double_depth=20, single_depth=40, in_channels=16, text_dim=4096, pooled_dim=768, guidance=True, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    w = HunyuanWeights()
    w.heads, w.dim = heads, heads * 128
    D = w.dim
    w.in_channels, w.out_channels, w.guidance, w.text_dim, w.pooled_dim, w.device = in_channels, in_channels, guidance, text_dim, pooled_dim, dev
    xav, bias, nw = _random_stack(w, D, double_depth, single_depth, dev, g)
    w.patch_w, w.patch_b = xav(D, in_channels * 4), bias(D)
    w.t_mlp = (xav(D, 256), bias(D), xav(D, D), bias(D))
    w.p_mlp = (xav(D, pooled_dim), bias(D), xav(D, D), bias(D))
    w.g_mlp = (xav(D, 256), bias(D), xav(D, D), bias(D)) if guidance else None
    w.r_in_w, w.r_in_b = xav(D, text_dim), bias(D)
    w.r_t_mlp = (xav(D, 256), bias(D), xav(D, D), bias(D))
    w.r_c_mlp = (xav(D, text_dim), bias(D), xav(D, D), bias(D))
    for _ in range(2):
        w.refiner.append({"n1_w": nw().new_ones(D) + 0.1 * torch.randn(D, device=dev, generator=g), "n1_b": bias(D),
                          "n2_w": nw().new_ones(D) + 0.1 * torch.randn(D, device=dev, generator=g), "n2_b": bias(D),
                          "qk_w": xav(2 * D, D), "qk_b": bias(2 * D), "v_w": xav(D, D), "v_b": bias(D), "nq": nw(), "nk": nw(),
                          "o_w": xav(D, D), "o_b": bias(D), "f1_w": xav(4 * D, D), "f1_b": bias(4 * D), "f2_w": xav(D, 4 * D), "f2_b": bias(D)})
    w.r_ada_w, w.r_ada_b = xav(4 * D, D, 0.3), bias(4 * D)
    w.out_w, w.out_b = xav(in_channels * 4, D), bias(in_channels * 4)
    return w


def random_qwen_weights(dev, heads=24, num_layers=60, in_channels=64, out_channels=16, joint_dim=3584, seed=0):
    """QwenImageWeights of the Qwen-Image shape on synthetic device weights, one tensor per Linear like a loaded module's."""
    g = torch.Generator(device=dev).manual_seed(seed)
    w = QwenImageWeights()
    w.heads, w.dim = heads, heads * 128
    D = w.dim
    w.in_channels, w.joint_dim, w.device, w.txt_norm_eps = in_channels, joint_dim, dev, 1e-6
    d, xav, bias, nw = _rand_block_weights(D, dev, g)
    parts, off = [], 0
    for _ in range(num_layers):
        d, *_ = _rand_block_weights(D, dev, g)
        for k in ("", "c"):
            q, kk = d[f"{k}qk_w"].split(D)
            d[f"{k}qk_w"] = (q.contiguous(), kk.contiguous())
        d["ada"], d["ada_c"] = off, off + 6 * D
        parts += [(off, xav(6 * D, D, 0.3)), (off + 6 * D, xav(6 * D, D, 0.3))]
        off += 12 * D
        w.double.append(d)
    w.ada_out = off
    parts.append((off, xav(2 * D, D, 0.3)))
    w.ada_parts, w.ada_b, w.ada_rows = parts, bias(off + 2 * D), off + 2 * D
    w.img_w, w.img_b, w.txt_w, w.txt_b = xav(D, in_channels), bias(D), xav(D, joint_dim), bias(D)
    w.txt_norm_w = (1 + 0.1 * torch.randn(joint_dim, device=dev, generator=g)).bfloat16().float()
    w.t_mlp = (xav(D, 256), bias(D), xav(D, D), bias(D))
    w.out_w, w.out_b = xav(4 * out_channels, D), bias(4 * out_channels)
    return w


class MMDiTHandle:
    """Stand-in for the pipeline's transformer object when the weights do not come from an nn.Module (benchmarks): carries the engine
    and receives the reference's class attributes through `init_magcache_flux` / `init_magcache_hunyuan`."""

    def __new__(cls, engine):
        sub = type("MMDiTHandle", (cls,), {})
        return object.__new__(sub)

    def __init__(self, engine):
        key = "_mc_flux_engine" if isinstance(engine, FluxEngine) else "_mc_hunyuan_engine"
        object.__setattr__(self, key, engine)

    def __call__(self, *a, **k):
        return self.forward(*a, **k)
