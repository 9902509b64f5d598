"""Drop-in replacements for the reference's monkey-patched transformer forwards.

Usage is the reference's own (MagCache4Wan2.1/magcache_generate.py:896-928): assign the function to the model class and set
the class attributes it reads —

    from magcache_b200 import magcache_forward, init_magcache
    init_magcache(wan_t2v.model, sample_steps=50, thresh=0.12, K=4, retention_ratio=0.2, ckpt_dir=args.ckpt_dir)
    # or, literally as the script does:  wan_t2v.model.__class__.forward = magcache_forward ; ...cnt = 0 ; ...

Signatures, attribute names (`cnt, num_steps, magcache_thresh, K, retention_ratio, accumulated_ratio, accumulated_err,
accumulated_steps, residual_cache, mag_ratios`; calibration: `norm_ratio, norm_std, cos_dis`) and error behaviour follow the
reference. Everything between the Python call and the returned tensors runs on the CUDA kernels of libmagcache_b200.so;
there is no eager/PyTorch fallback — a CPU tensor or a missing library raises.
"""
import contextlib
import os

import numpy as np

import torch

from . import ops
from .config import FAMILIES, interp_cfg, nearest_interp, save_json, table_for_ckpt_dir, table_from_calibration, tables
from .controller import AttrController, OpenSoraTeaController, TeaController, nearest_interp_linspace, opensora_rel_l1
from .lora import is_lora_layer, scale_lora_layers, unscale_lora_layers
from .mmdit import FluxEngine, FluxWeights, HunyuanEngine, HunyuanWeights, QwenImageEngine, QwenImageWeights
from .opensora import OpenSoraEngine, OpenSoraWeights
from .wan import WanEngine, WanWeights

# every engine a patched forward caches on its module (one per model family)
ENGINE_ATTRS = ("_mc_engine", "_mc_flux_engine", "_mc_hunyuan_engine", "_mc_opensora_engine", "_mc_qwen_engine")


def _cached_engine(self, attr, build):
    """The engine cached on the module under `attr` (one of ENGINE_ATTRS); on the first call `build(**shard_kw)` makes it, with the
    keywords `enable_token_shard` left on the module."""
    eng = self.__dict__.get(attr)
    if eng is None:
        eng = build(**self.__dict__.get("_mc_shard_kw", {}))
        object.__setattr__(self, attr, eng)
    return eng


def invalidate_engine(model):
    """Drop the engine cached on `model` (and with it the repacked bf16 copy of the weights, the workspaces and any captured CUDA
    graphs) and its controllers. The engine snapshots the module's parameters at the first forward: call this after anything that
    changes them — a LoRA merge (on a FLUX model only one whose LoRA layers are then removed before the next forward, see
    lora.FluxLoraScan), `load_state_dict`, `.to(...)` — and the next forward repacks. The module's own parameters stay
    resident next to the packed copy (about +2.8 GB for the 1.3B model, +28 GB for 14B); free or offload them yourself if that matters."""
    for name in ENGINE_ATTRS + ("_mc_ctrls",):
        model.__dict__.pop(name, None)
    return model


def enable_token_shard(model, rank, world, group=None):
    """Shard the token axis of `model`'s forwards over `world` ranks of one node (call before the first forward; needs an
    initialised torch.distributed NCCL group). Every rank must then make the same calls with the same inputs; outputs are
    replicated, the residual cache stays sharded. Wan engines shard all tokens; the FLUX / HunyuanVideo engines shard the image tokens and
    replicate the text tokens. The Open-Sora engine has no token-sharded path: its forward raises NotImplementedError for world > 1
    (`enable_sequence_parallel` shards it by frames and positions instead)."""
    if any(k in model.__dict__ for k in ENGINE_ATTRS):
        raise RuntimeError("enable_token_shard must be called before the first forward")
    object.__setattr__(model, "_mc_shard_kw", dict(shard_world=world, shard_rank=rank, shard_group=group))
    return model


def enable_sequence_parallel(model, rank, world, group=None):
    """Run `model`'s Open-Sora forwards (`magcache_opensora_forward`, `teacache_opensora_forward`) and `OpenSoraRFlowSampler.sample`
    with VideoSys's sequence parallelism over `world` ranks of one node: each rank owns a contiguous block of latent frames for the
    spatial blocks and of positions for the temporal blocks (eval/magcache/experiments/opensora.py:284-293, 342-361). Call before the
    first forward, after `init_magcache_opensora` / `init_teacache_opensora`, on every rank with an initialised torch.distributed
    group (`group`, default the world); every rank then makes the same calls with the same inputs (the same latent noise included)
    and receives the whole output. The residual cache stays sharded: `residual_cache` / `previous_residual` hold this rank's frames.
    Every output is bit-equal to the one-GPU engine's. world == 1 is the unsharded engine."""
    if getattr(type(model), "forward", None) not in (magcache_opensora_forward, teacache_opensora_forward):
        raise RuntimeError("enable_sequence_parallel needs an Open-Sora forward installed (init_magcache_opensora / init_teacache_opensora)")
    if any(k in model.__dict__ for k in ENGINE_ATTRS):
        raise RuntimeError("enable_sequence_parallel must be called before the first forward")
    if not 0 <= rank < world:
        raise ValueError(f"enable_sequence_parallel: rank {rank} outside a world of {world}")
    object.__setattr__(model, "_mc_sp_kw", dict(sp_world=world, sp_rank=rank, sp_group=group))
    return model


# the paper-evaluation scripts keep the controller inputs under their own attribute names and hard-code some of them
_ATTR_NAMES = {
    # eval/magcache/experiments/Wan2.1_EVAL/wan_magcache.py:770-786 (`skip_time = int(self.num_steps*0.2)`, :772)
    "wan2.1-eval": (dict(cnt="t", K="magcache_K", mag_ratios="ratio", accumulated_ratio="accumulated_sim"), dict(retention_ratio=0.2)),
    # eval/magcache/experiments/opensora.py:297-308 (30 steps per video, :349-354)
    "opensora": (dict(cnt="t", mag_ratios="ratio", accumulated_ratio="accumulated_sim", split_step="skip_time"),
                 dict(num_steps=30, retention_ratio=0.2)),
}


def _ctrl(self, family):
    """The module's controller for `family` (a key of `config.FAMILIES`)."""
    ctrls = self.__dict__.setdefault("_mc_ctrls", {})
    c = ctrls.get(family)
    if c is None:
        c = ctrls[family] = AttrController(FAMILIES[family], *_ATTR_NAMES.get(family, ()))
    return c


def _take_residual(eng, cur, slot=None):
    """The reference keeps the cached residual in an attribute (`cur`, its current value); the engine keeps it in a fixed buffer that
    the attribute aliases (`eng.res`, or `eng.res[slot]` for the per-CFG-branch engines). If a caller replaced the attribute (or
    cleared it), follow the attribute. A residual of another size is the previous generation's at another shape (the attribute
    outlives a generation, as in the reference): it can serve no hit here, so the cache counts as empty."""
    res = eng.res if slot is None else eng.res[slot]
    if cur is None or (torch.is_tensor(cur) and cur.numel() != res.numel()):
        valid = False
    elif torch.is_tensor(cur) and cur.data_ptr() != res.data_ptr():
        res.copy_(cur.reshape(res.shape))
        valid = True
    else:
        return
    if slot is None:
        eng.res_valid = valid
    else:
        eng.res_valid[slot] = valid


def _record_stats(self, stats):
    """One calibration call's statistics: appended rounded to 5 places and printed like the reference."""
    norm_ratio, norm_std, cos_dis = stats
    self.norm_ratio.append(round(norm_ratio, 5))
    self.norm_std.append(round(norm_std, 5))
    self.cos_dis.append(round(cos_dis, 5))
    print(f"time: {self.cnt}, norm_ratio: {norm_ratio}, norm_std: {norm_std}, cos_dis: {cos_dis}")


def _print_stats(self):
    print("norm ratio")
    print(self.norm_ratio)
    print("norm std")
    print(self.norm_std)
    print("cos_dis")
    print(self.cos_dis)


def _wan_weights(self):
    if not hasattr(self, "patch_embedding"):
        raise TypeError("magcache_b200.magcache_forward expects a Wan2.1 WanModel (or an object carrying `_mc_engine`)")
    dev = self.patch_embedding.weight.device
    if dev.type != "cuda":
        raise RuntimeError("magcache_b200: the model must be on a CUDA device (no CPU path)")
    return WanWeights.from_module(self, dev)


def _engine(self):
    return _cached_engine(self, "_mc_engine", lambda **kw: WanEngine(_wan_weights(self), **kw))


def _stage(self, x, t, context, seq_len, clip_fea, y, pad_ok=True, vace_context=None, vace_scale=1.0, require_clip=True):
    if getattr(self, "model_type", "t2v") == "i2v" and require_clip:
        assert clip_fea is not None and y is not None  # magcache_generate.py:226-227
    if len(x) != 1 or len(context) != 1 or (y is not None and len(y) != 1):
        raise NotImplementedError("magcache_b200: one sample per call (the reference's caller passes [latents], wan_magcache.py:296-299)")
    eng = _engine(self)
    lat = x[0]
    if not lat.is_cuda:
        raise RuntimeError("magcache_b200: latents must be CUDA tensors (no CPU path)")
    n_tok = lat.shape[1] * (lat.shape[2] // 2) * (lat.shape[3] // 2)
    assert n_tok <= seq_len  # reference: assert seq_lens.max() <= seq_len (:242)
    # seq_len > n_tok (upstream rounds seq_len up to a multiple of the sequence-parallel size): the reference appends zero rows
    # (:243-246) that never reach a real token — keys are masked by k_lens = seq_lens, every other op is per token, unpatchify
    # reads the first n_tok rows — so the forwards simply do not compute them; the only visible difference: residual_cache[i] has
    # n_tok rows instead of seq_len. The calibration statistics DO average over the padded rows upstream: there (pad_ok=False) ONE
    # representative pad row is computed — the padded rows are all identical — and weighted by their count.
    pad_row = 1 if (n_tok != seq_len and pad_ok is False) else 0
    if vace_context is not None and len(vace_context) != 1:
        raise NotImplementedError("magcache_b200: one sample per call")
    eng.stage_inputs(lat, t, context[0], clip_fea=clip_fea, y=None if y is None else y[0],
                     vace_context=None if vace_context is None else vace_context[0], vace_scale=vace_scale, pad_row=pad_row)
    eng.pad_weight = (seq_len - n_tok) if pad_row else 0
    return eng


def magcache_forward(self, x, t, context, seq_len, clip_fea=None, y=None):
    r"""MagCache4Wan2.1/magcache_generate.py:198-312 on the H100 kernels.

    Args / returns as the reference: x List[Tensor[C_in, F, H, W]], t Tensor[B], context List[Tensor[L, C]], seq_len int
    -> List[Tensor[C_out, F, H, W]] (float32).
    """
    eng = _stage(self, x, t, context, seq_len, clip_fea, y)
    ctrl = _ctrl(self, "wan2.1")
    slot = self.cnt % 2
    skip_forward = ctrl.decide(self)  # :279-292 (float64 state under the reference's attribute names)
    _take_residual(eng, self.residual_cache[slot], slot)
    # hit : `x = x + residual_x` (:295) feeds only the head, so the sum is formed inside the head kernel (same fp32 arithmetic)
    # miss: block stack (:297-298), `residual_x = x - ori_x` (:299) written into the slot's buffer
    out = eng.forward("hit" if skip_forward else "miss", slot)
    self.residual_cache[slot] = eng.res[slot].view(1, *eng.res[slot].shape)  # :301
    ctrl.advance(self)  # :306-311
    return [out]


def magcache_vace_forward(self, x, t, vace_context, context, seq_len, vace_context_scale=1.0, clip_fea=None, y=None):
    r"""MagCache4Wan2.1/magcache_generate.py:439-560 (installed at :1126-1150 with the VACE tables): the T2V forward plus the
    control branch. `vace_context`: List[Tensor[96, F, H, W]]. On a miss the control blocks run first (`forward_vace`, :541) and
    every second main block adds its hint; on a hit nothing of the control branch is computed, as in the reference. `clip_fea` and
    `y` are accepted and ignored (the reference has those lines commented out, :471-476, :505-507)."""
    eng = _stage(self, x, t, context, seq_len, None, None, vace_context=vace_context, vace_scale=vace_context_scale)
    ctrl = _ctrl(self, "wan2.1")
    slot = self.cnt % 2
    skip_forward = ctrl.decide(self)  # :517-531
    _take_residual(eng, self.residual_cache[slot], slot)
    if skip_forward:
        print("skip: ", self.cnt)  # :527
    out = eng.forward("hit" if skip_forward else "miss", slot)
    self.residual_cache[slot] = eng.res[slot].view(1, *eng.res[slot].shape)  # :549
    ctrl.advance(self)  # :554-559
    return [out]


def magcache_vace_calibration(self, x, t, vace_context, context, seq_len, vace_context_scale=1.0, clip_fea=None, y=None):
    r"""MagCache4Wan2.1/magcache_generate.py:314-436: `magcache_calibration` with the control branch."""
    return _calibrate(self, _stage(self, x, t, context, seq_len, None, None, pad_ok=False, vace_context=vace_context,
                                   vace_scale=vace_context_scale))


def magcache_wan22_forward(self, x, t, context, seq_len, clip_fea=None, y=None):
    r"""MagCache4Wan2.2/magcache_generate.py:209-336 for the A14B experts (T2V and I2V) on the Wan engine: the Wan2.1 forward with the
    two-expert skip windows (`split_step`, `mode`, :294-303) and a counter shared by the high-noise and the low-noise model — two
    instances of one class, one engine (weights) each, one controller state and one residual cache between them (:340-362).
    Wan2.2 gives every token its own timestep (:263-272). A 1-D `t` (the A14B experts) is one value for all tokens; TI2V-5B passes
    [1, seq_len] with t = 0 on the first-frame tokens of an image-conditioned run: the engine reduces it to its distinct values and the
    contiguous token ranges carrying them (`WanEngine._stage_t`), so the arithmetic per token is the reference's. With `split_step` None
    (TI2V, :301-303) the window is the plain `int(num_steps * retention_ratio)`."""
    if getattr(self, "model_type", "t2v") == "i2v":
        assert y is not None  # :239-240
    if t.dim() != 1:
        if t.size(0) != 1:
            raise NotImplementedError("magcache_b200: one sample per call")
        assert t.size(1) == seq_len  # what `.unflatten(0, (bt, seq_len))` (:270) requires
    eng = _stage(self, x, t, context, seq_len, None, y, require_clip=False)
    ctrl = _ctrl(self, "wan2.2-i2v" if getattr(self, "mode", "t2v") == "i2v" else "wan2.2-t2v")
    slot = int(self.cnt) % 2
    skip_forward = ctrl.decide(self)  # :290-317
    _take_residual(eng, self.residual_cache[slot], slot)  # the other expert's residual arrives through the shared class-level list
    out = eng.forward("hit" if skip_forward else "miss", slot)
    self.residual_cache[slot] = eng.res[slot].view(1, *eng.res[slot].shape)  # :324
    ctrl.advance(self)  # :328-334
    return [out]


def init_magcache_wan22(model, mag_ratios, sample_steps, thresh=0.06, K=2, retention_ratio=0.2, split_steps=None, mode="t2v"):
    """`init_magcache(model, mag_ratios, args, split_steps, mode)` of MagCache4Wan2.2/magcache_generate.py:340-362: patches the CLASS the
    two experts share. `mag_ratios`: the list without its `[1.0]*2` prefix like the script passes it, or a key of `tables()` (which
    already carries the prefix)."""
    cls = model.__class__
    cls.forward = magcache_wan22_forward
    cls.cnt = torch.tensor(0)
    cls.num_steps = sample_steps * 2
    cls.split_step = split_steps * 2 if split_steps else None
    cls.mode = mode
    cls.magcache_thresh, cls.K = thresh, K
    cls.accumulated_err, cls.accumulated_steps, cls.accumulated_ratio = [0.0, 0.0], [0, 0], [1.0, 1.0]
    cls.retention_ratio = retention_ratio
    cls.residual_cache = [None, None]
    mr = tables()[mag_ratios] if isinstance(mag_ratios, str) else np.array([1.0] * 2 + list(mag_ratios))
    cls.mag_ratios = interp_cfg(mr, sample_steps)  # :357-361
    return model


def magcache_calibration(self, x, t, context, seq_len, clip_fea=None, y=None):
    r"""MagCache4Wan2.1/magcache_generate.py:80-194: always runs the block stack and records, per forward, the token-mean
    magnitude ratio, its std and the cosine distance to the previous residual of the same CFG branch (one fused pass)."""
    return _calibrate(self, _stage(self, x, t, context, seq_len, clip_fea, y, pad_ok=False))


def _calibrate(self, eng):
    slot = self.cnt % 2
    out, stats = eng.calibrate(slot, self.residual_cache[slot] if self.cnt >= 2 else None)
    if stats is not None:
        _record_stats(self, stats)
    self.residual_cache[slot] = eng.cal_residual
    self.cnt += 1
    if self.cnt >= self.num_steps:
        self.cnt = 0
        self.accumulated_ratio = [1.0, 1.0]
        self.accumulated_err = [0.0, 0.0]
        self.accumulated_steps = [0, 0]
        _print_stats(self)
        # :191-193 `save_json("wan2_1_mag_ratio", self.norm_ratio)` ...: same file names, in `calibration_dir` (default: the
        # working directory, like the reference). `config.table_from_calibration` turns the first file into a `mag_ratios` table.
        out_dir = getattr(self, "calibration_dir", ".")
        if out_dir is not None:
            save_json(os.path.join(out_dir, "wan2_1_mag_ratio"), self.norm_ratio)
            save_json(os.path.join(out_dir, "wan2_1_mag_std"), self.norm_std)
            save_json(os.path.join(out_dir, "wan2_1_cos_dis"), self.cos_dis)
    return [out]


def init_magcache(model, sample_steps, thresh=0.12, K=2, retention_ratio=0.2, mag_ratios=None, ckpt_dir=None, table=None):
    """The installation block of magcache_generate.py:896-919 (i2v :989-1010, VACE :1126-1150) as a helper (same form as Wan2.2's
    `init_magcache`, MagCache4Wan2.2/magcache_generate.py:340-362): patches the CLASS, like the reference. VACE models
    (`model_type == "vace"`) get `magcache_vace_forward`."""
    cls = model.__class__
    cls.forward = magcache_vace_forward if getattr(model, "model_type", "t2v") == "vace" else magcache_forward
    cls.cnt = 0
    cls.num_steps = sample_steps * 2
    cls.magcache_thresh = thresh
    cls.K = K
    cls.accumulated_err = [0.0, 0.0]
    cls.accumulated_steps = [0, 0]
    cls.accumulated_ratio = [1.0, 1.0]
    cls.retention_ratio = retention_ratio
    cls.residual_cache = [None, None]
    if isinstance(mag_ratios, (str, os.PathLike)):  # a calibration dump (`wan2_1_mag_ratio.json`) instead of a pasted literal
        mag_ratios = table_from_calibration(mag_ratios)
    if mag_ratios is None:
        mag_ratios = tables()[table] if table is not None else table_for_ckpt_dir(ckpt_dir)
    cls.mag_ratios = interp_cfg(mag_ratios, sample_steps)  # :915-919
    return model


def reset_magcache(model):
    """Start a new video: cnt = 0 and fresh accumulators (what `pipeline.transformer.__class__.cnt = 0` between prompts is
    meant to do, MagCache4FLUX/magcache_flux.py:478). `self.cnt += 1` in the forward creates INSTANCE attributes that shadow
    the class-level ones the scripts install, so both levels are reset here. The residual cache is kept, as in the reference."""
    cls = model.__class__
    for attr in ("cnt", "accumulated_err", "accumulated_steps", "accumulated_ratio"):
        model.__dict__.pop(attr, None)
    if torch.is_tensor(getattr(cls, "cnt", None)):
        cls.cnt.fill_(0)  # Wan2.2's two experts share one counter tensor (MagCache4Wan2.2/magcache_generate.py:342): keep it shared
    else:
        cls.cnt = 0
    if isinstance(getattr(cls, "accumulated_err", None), list):
        cls.accumulated_err, cls.accumulated_steps, cls.accumulated_ratio = [0.0, 0.0], [0, 0], [1.0, 1.0]
    else:
        cls.accumulated_err, cls.accumulated_steps, cls.accumulated_ratio = 0, 0, 1.0
    return model


def init_magcache_calibration(model, sample_steps):
    """magcache_generate.py:921-928."""
    cls = model.__class__
    cls.forward = magcache_vace_calibration if getattr(model, "model_type", "t2v") == "vace" else magcache_calibration
    cls.cnt = 0
    cls.num_steps = sample_steps * 2
    cls.norm_ratio, cls.norm_std, cls.cos_dis = [], [], []
    cls.residual_cache = [None, None]
    return model


# ------------------------------------------------------------------------------------------------------------------
# Other adapters: controller + cache kernels around a caller-supplied block stack
# ------------------------------------------------------------------------------------------------------------------
def magcache_branch(self, hidden, run_blocks, family, cache_attr):
    """The hit/miss branch of the other adapters' forwards — FLUX / Kontext (magcache_flux.py:326-427), HunyuanVideo
    (magcache_sample_video.py:88-141), FramePack (magcache_demo_gradio.py:252-300), Wan2.2 / Qwen-Image
    (MagCache4Wan2.2/magcache_generate.py:290-334): decides with the family's controller (`config.FAMILIES`), then either adds
    the cached residual (K1 kernel) or calls `run_blocks(hidden)` (the model's own transformer stack) and stores `out - hidden`
    (K2 kernel) under `cache_attr` — a tensor for scalar-state families, a 2-list indexed by `cnt % 2` for per-branch ones.
    Advances the counter. Wan2.2's expert boundary is read from `self.split_step` like upstream (:344)."""
    ctrl = _ctrl(self, family)
    per_branch = FAMILIES[family]["branches"] == 2
    slot = int(self.cnt) % 2 if per_branch else None
    if ctrl.decide(self):
        cur = getattr(self, cache_attr)[slot] if per_branch else getattr(self, cache_attr)
        if cur is None:
            raise TypeError("magcache_b200: cache hit with an empty residual cache (reference: Tensor + NoneType)")
        out = ops.cache_hit_add(hidden.contiguous(), cur)
    else:
        out = run_blocks(hidden)
        cur = ops.residual_sub(out.contiguous(), hidden.contiguous())
    if per_branch:
        getattr(self, cache_attr)[slot] = cur
    else:
        setattr(self, cache_attr, cur)
    ctrl.advance(self)
    return out


# ------------------------------------------------------------------------------------------------------------------
# FLUX: the whole patched forward on the MMDiT engine (magcache_b200/flux.py; opt-in until validated on a GPU, see its header)
# ------------------------------------------------------------------------------------------------------------------
class _Sample:
    """Stand-in for diffusers' Transformer2DModelOutput (`.sample`), which is not importable here."""

    def __init__(self, sample):
        self.sample = sample


def _flux_lora_scale(self, hidden_states, joint_attention_kwargs):
    """The call's LoRA scale (:274-279), after the checks that need no engine: only the "scale" and "ip_adapter_image_embeds"
    keys are built, CUDA inputs only."""
    extra = sorted(k for k in (joint_attention_kwargs or {}) if k not in ("scale", "ip_adapter_image_embeds"))
    if extra:
        raise NotImplementedError(f"magcache_b200: joint_attention_kwargs {extra} are not built for the FLUX engine; only the LoRA "
                                  "'scale' and 'ip_adapter_image_embeds' are")
    if not hidden_states.is_cuda:
        raise RuntimeError("magcache_b200: hidden_states must be CUDA tensors (no CPU path)")
    lora_scale = joint_attention_kwargs.get("scale", 1.0) if joint_attention_kwargs is not None else 1.0
    if lora_scale != 1.0 and not (isinstance(self, torch.nn.Module) and any(is_lora_layer(m) for m in self.modules())):
        # the reference would scale nothing: a scale without adapters is taken for adapters that failed to load
        raise NotImplementedError(f"magcache_b200: joint_attention_kwargs scale={lora_scale} but the model has no LoRA layer to scale")
    return lora_scale


@contextlib.contextmanager
def _lora_scaled(self, lora_scale):
    """The reference's `scale_lora_layers` before the forward (:281-283) and `unscale_lora_layers` after it (:437-439). The unscale
    also runs when the engine refuses an input mid-call (an unsupported adapter, a malformed ControlNet sample), so a caller that
    catches the error never finds the layers' `scaling` left multiplied by the scale."""
    scale_lora_layers(self, lora_scale)
    try:
        yield
    finally:
        unscale_lora_layers(self, lora_scale)


def _flux_stage(self, hidden_states, encoder_hidden_states, pooled_projections, timestep, img_ids, txt_ids, guidance,
                controlnet_block_samples, controlnet_single_block_samples, controlnet_blocks_repeat, joint_attention_kwargs):
    """Stages one FLUX call on the engine (inside `_lora_scaled`) and hands it the adapters as they are now."""
    is_module = isinstance(self, torch.nn.Module)
    eng = _cached_engine(self, "_mc_flux_engine", lambda **kw: FluxEngine(FluxWeights.from_module(self, hidden_states.device), **kw))
    if is_module:  # (a benchmark's MMDiTHandle sets the engine's LoRA pack and IP-Adapter call itself)
        eng.sync_lora(self)
        eng.stage_ip_adapter(self, (joint_attention_kwargs or {}).get("ip_adapter_image_embeds"))
    if txt_ids.ndim == 3:  # :305-316 (deprecated 3-D ids)
        txt_ids = txt_ids[0]
    if img_ids.ndim == 3:
        img_ids = img_ids[0]
    eng.stage_inputs(hidden_states, encoder_hidden_states, pooled_projections, timestep, guidance, img_ids, txt_ids)
    eng.stage_controlnet(controlnet_block_samples, controlnet_single_block_samples, controlnet_blocks_repeat)
    return eng


def magcache_flux_forward(self, hidden_states, encoder_hidden_states=None, pooled_projections=None, timestep=None, img_ids=None,
                          txt_ids=None, guidance=None, joint_attention_kwargs=None, controlnet_block_samples=None,
                          controlnet_single_block_samples=None, return_dict=True, controlnet_blocks_repeat=False):
    r"""MagCache4FLUX/magcache_flux.py:234-440 on the H100 kernels: same signature, same state attributes (`cnt, num_steps,
    magcache_thresh, K, retention_ratio, accumulated_ratio / _err / _steps, previous_residual, mag_ratios`), `(output,)` or an object
    with `.sample`. ControlNet residuals (:374-384, :416-423) are added after their blocks on a miss, fused into each block's last GEMM
    on the image rows; a hit ignores them, as the reference does. Unmerged PEFT LoRA adapters run as tails of the GEMMs of the
    Linears they adapt (magcache_b200/lora.py), scaled by `joint_attention_kwargs["scale"]` with the reference's
    scale / unscale statements (:274-287, :437-439) on every call, hit or miss. IP-Adapter image prompts
    (`joint_attention_kwargs["ip_adapter_image_embeds"]`, :321-324) run on a miss: the image projection, then per double block
    one `mc_ip_attn` launch whose output FF2's epilogue adds (mmdit.IPAdapterCall); a hit ignores them."""
    lora_scale = _flux_lora_scale(self, hidden_states, joint_attention_kwargs)
    with _lora_scaled(self, lora_scale):
        eng = _flux_stage(self, hidden_states, encoder_hidden_states, pooled_projections, timestep, img_ids, txt_ids, guidance,
                          controlnet_block_samples, controlnet_single_block_samples, controlnet_blocks_repeat, joint_attention_kwargs)
        ctrl = _ctrl(self, "flux")
        skip_forward = ctrl.decide(self)  # :326-338
        _take_residual(eng, self.previous_residual)
        out = eng.forward("hit" if skip_forward else "miss")
        self.previous_residual = eng.res.view(1, *eng.res.shape)  # :427
        ctrl.advance(self)  # :431-436
    output = out.view(1, *out.shape)
    if not return_dict:
        return (output,)
    return _Sample(output)


def magcache_flux_calibration(self, hidden_states, encoder_hidden_states=None, pooled_projections=None, timestep=None, img_ids=None,
                              txt_ids=None, guidance=None, joint_attention_kwargs=None, controlnet_block_samples=None,
                              controlnet_single_block_samples=None, return_dict=True, controlnet_blocks_repeat=False):
    r"""MagCache4FLUX/magcache_flux.py:21-231: every call runs the block stack and, from the second call on, records the token-mean
    magnitude ratio, its std and the cosine distance to the previous residual (`norm_ratio / norm_std / cos_dis`, rounded to 5 places);
    the lists are printed on the last call of a generation and cleared at the wrap (:207-221). ControlNet residuals as in the
    forward (:145-155, :187-193); LoRA adapters and scale as in the forward (:62-75, :224-226); IP-Adapter image prompts as in the
    forward (:108-111)."""
    lora_scale = _flux_lora_scale(self, hidden_states, joint_attention_kwargs)
    with _lora_scaled(self, lora_scale):
        eng = _flux_stage(self, hidden_states, encoder_hidden_states, pooled_projections, timestep, img_ids, txt_ids, guidance,
                          controlnet_block_samples, controlnet_single_block_samples, controlnet_blocks_repeat, joint_attention_kwargs)
        if self.cnt == 0:
            eng.res_valid = False  # `if self.cnt>=1` (:199): the first call of a generation has nothing to compare with
        out, stats = eng.calibrate()
        if stats is not None:
            _record_stats(self, stats)
        self.previous_residual = eng.res.view(1, *eng.res.shape)
        if self.cnt >= self.num_steps - 1:
            _print_stats(self)
        self.cnt += 1
        if self.cnt >= self.num_steps:
            self.cnt = 0
            self.norm_ratio, self.norm_std, self.cos_dis = [], [], []
    output = out.view(1, *out.shape)
    return _Sample(output) if return_dict else (output,)


def init_magcache_flux_calibration(transformer, num_inference_steps=28):
    """magcache_flux.py:446-458 with `FluxTransformer2DModel.forward = magcache_calibration`."""
    cls = transformer.__class__
    cls.forward = magcache_flux_calibration
    cls.cnt, cls.num_steps = 0, num_inference_steps
    cls.norm_ratio, cls.norm_std, cls.cos_dis = [], [], []
    cls.previous_residual = None
    return transformer


def init_magcache_flux(transformer, num_inference_steps=28, thresh=0.24, K=5, retention_ratio=0.1, mag_ratios=None, table="flux_dev"):
    """The installation statements of magcache_flux.py:446-471 (Kontext: magcache_flux_kontext.py:445-470 with table "flux_kontext",
    thresh 0.05, K 4, retention 0.2): patches the CLASS."""
    cls = transformer.__class__
    cls.forward = magcache_flux_forward
    cls.cnt, cls.num_steps = 0, num_inference_steps
    mr = np.asarray(tables()[table] if mag_ratios is None else mag_ratios, dtype=np.float64)
    if len(mr) != num_inference_steps:  # :461-463
        mr = nearest_interp(mr, num_inference_steps)
    cls.mag_ratios = mr
    cls.K, cls.magcache_thresh, cls.retention_ratio = K, thresh, retention_ratio
    cls.accumulated_ratio, cls.accumulated_err, cls.accumulated_steps = 1, 0, 0
    cls.previous_residual = None
    return transformer


def _hunyuan_stage(self, x, t, text_states, text_mask, text_states_2, freqs_cos, freqs_sin, guidance):
    if not x.is_cuda:
        raise RuntimeError("magcache_b200: x must be a CUDA tensor (no CPU path)")
    eng = _cached_engine(self, "_mc_hunyuan_engine", lambda **kw: HunyuanEngine(HunyuanWeights.from_module(self, x.device), **kw))
    eng.stage_inputs(x, t, text_states, text_mask, text_states_2, freqs_cos, freqs_sin, guidance)
    return eng


def magcache_hunyuan_forward(self, x, t, text_states=None, text_mask=None, text_states_2=None, freqs_cos=None, freqs_sin=None,
                             guidance=None, return_dict=True):
    r"""MagCache4HunyuanVideo/magcache_sample_video.py:29-160 on the H100 kernels (MMDiT engine, magcache_b200/mmdit.py; opt-in until
    validated on a GPU): same signature and state attributes (`cnt, num_steps, magcache_thresh, K, retention_ratio, accumulated_ratio /
    _err / _steps, residual_cache, mag_ratios`), returns `{"x": img}` or the tensor. x [1, 16, T, H, W]; text_mask marks the valid
    (right-padded) text tokens."""
    eng = _hunyuan_stage(self, x, t, text_states, text_mask, text_states_2, freqs_cos, freqs_sin, guidance)
    ctrl = _ctrl(self, "hunyuan")
    skip_forward = ctrl.decide(self)  # :88-102
    _take_residual(eng, self.residual_cache)
    img = eng.forward("hit" if skip_forward else "miss")
    self.residual_cache = eng.res.view(1, *eng.res.shape)  # :141
    ctrl.advance(self)  # :149-154
    if return_dict:
        return {"x": img}
    return img


def magcache_hunyuan_calibration(self, x, t, text_states=None, text_mask=None, text_states_2=None, freqs_cos=None, freqs_sin=None,
                                 guidance=None, return_dict=True):
    r"""MagCache4HunyuanVideo/magcache_sample_video.py:163-290: the calibration twin (statistics from the second call on, lists printed
    from call 49 on — hard-coded upstream, :266 — and a counter that is never wrapped, :281)."""
    eng = _hunyuan_stage(self, x, t, text_states, text_mask, text_states_2, freqs_cos, freqs_sin, guidance)
    if self.cnt == 0:
        eng.res_valid = False
    img, stats = eng.calibrate()
    if stats is not None:
        _record_stats(self, stats)
    self.residual_cache = eng.res.view(1, *eng.res.shape)
    if self.cnt >= 49:
        _print_stats(self)
    self.cnt += 1
    return {"x": img} if return_dict else img


def init_magcache_hunyuan_calibration(transformer, infer_steps=50):
    """magcache_sample_video.py:307-314 with `forward = magcache_calibration` (:324)."""
    cls = transformer.__class__
    cls.forward = magcache_hunyuan_calibration
    cls.cnt, cls.num_steps = 0, infer_steps
    cls.norm_ratio, cls.norm_std, cls.cos_dis = [], [], []
    cls.residual_cache = None
    return transformer


def init_magcache_hunyuan(transformer, infer_steps=50, thresh=0.24, K=6, retention_ratio=0.2, video_height=720, mag_ratios=None):
    """The installation statements of magcache_sample_video.py:303-328 (table chosen by `args.video_size[0]` in {720, 544}, :315-318)."""
    cls = transformer.__class__
    cls.cnt, cls.num_steps, cls.magcache_thresh, cls.K = 0, infer_steps, thresh, K
    cls.residual_cache = None
    if mag_ratios is None:
        if video_height not in (720, 544):
            raise KeyError(f"no calibrated table for video height {video_height} (the reference would hit AttributeError later)")
        mag_ratios = tables()["hunyuan_720p" if video_height == 720 else "hunyuan_544p"]
    mr = np.asarray(mag_ratios, dtype=np.float64)
    if len(mr) != infer_steps:
        mr = nearest_interp(mr, infer_steps)
    cls.mag_ratios, cls.retention_ratio = mr, retention_ratio
    cls.forward = magcache_hunyuan_forward
    cls.accumulated_ratio, cls.accumulated_err, cls.accumulated_steps = 1, 0, 0
    return transformer


# ------------------------------------------------------------------------------------------------------------------
# Qwen-Image / Qwen-Image-Edit (MagCache4QwenImage/magcache_generate.py, MagCache4QwenImageEdit/magcache_generate.py: the same
# forward, calibration and installation statements) on the MMDiT engine
# ------------------------------------------------------------------------------------------------------------------
def _qwen_stage(self, hidden_states, encoder_hidden_states, encoder_hidden_states_mask, timestep, img_shapes, txt_seq_lens, guidance,
                attention_kwargs):
    if guidance is not None:
        raise NotImplementedError("magcache_b200: Qwen-Image guidance (guidance_embeds checkpoints) is not supported")
    extra = dict(attention_kwargs or {})
    scale = extra.pop("scale", 1.0)
    if extra or scale != 1.0:
        raise NotImplementedError(f"magcache_b200: the Qwen-Image engine takes no attention_kwargs but scale 1.0; got {attention_kwargs}")
    if self.__dict__.get("_mc_shard_kw", {}).get("shard_world", 1) > 1:
        raise NotImplementedError("magcache_b200: the Qwen-Image engine has no token-sharded path; run it on one GPU")
    if not hidden_states.is_cuda:
        raise RuntimeError("magcache_b200: hidden_states must be CUDA tensors (no CPU path)")
    eng = _cached_engine(self, "_mc_qwen_engine", lambda **kw: QwenImageEngine(QwenImageWeights.from_module(self, hidden_states.device)))
    eng.stage_inputs(hidden_states, encoder_hidden_states, encoder_hidden_states_mask, timestep, img_shapes, txt_seq_lens)
    return eng


def magcache_qwen_image_forward(self, hidden_states, encoder_hidden_states=None, encoder_hidden_states_mask=None, timestep=None,
                                img_shapes=None, txt_seq_lens=None, guidance=None, attention_kwargs=None, return_dict=True):
    r"""MagCache4QwenImage/magcache_generate.py:173-252 (Qwen-Image-Edit: the same lines of its script) on the H100 kernels: same
    signature and state attributes (`cnt, num_steps, magcache_thresh, K, retention_ratio, accumulated_ratio / _err / _steps` as
    per-branch lists, `residual_cache` indexed by `cnt % 2`, `mag_ratios`), `(output,)` or an object with `.sample`. One sample per
    call: the pipelines' true CFG makes a cond and an uncond call per step, each with its own text length and residual slot. A
    hit runs only img_in, the time embedding, the add and the final layer (mmdit.QwenImageEngine)."""
    eng = _qwen_stage(self, hidden_states, encoder_hidden_states, encoder_hidden_states_mask, timestep, img_shapes, txt_seq_lens,
                      guidance, attention_kwargs)
    slot = int(self.cnt) % 2
    skip_forward = _ctrl(self, "qwen-image").decide(self)  # :205-219
    _take_residual(eng, self.residual_cache[slot], slot)
    out = eng.forward("hit" if skip_forward else "miss", slot)
    self.residual_cache[slot] = eng.res[slot].view(1, *eng.res[slot].shape)  # :241
    self.cnt += 1  # :242-244, the reference's own statements: the wrap rebinds an int on the instance and keeps the accumulators
    if self.cnt >= self.num_steps:
        self.cnt = 0
    output = out.view(1, *out.shape)
    return _Sample(output) if return_dict else (output,)


def magcache_qwen_image_calibration(self, hidden_states, encoder_hidden_states=None, encoder_hidden_states_mask=None, timestep=None,
                                    img_shapes=None, txt_seq_lens=None, guidance=None, attention_kwargs=None, return_dict=True):
    r"""MagCache4QwenImage/magcache_generate.py:94-171: every call runs the blocks; from `cnt >= 2` on the residual is compared with
    the one of the same CFG branch (`residual_cache[cnt % 2]`) and `norm_ratio / norm_std / cos_dis` get one entry each (rounded to 5
    places), printed per step in the reference's format. At the wrap the lists are printed and only the counter is reset."""
    eng = _qwen_stage(self, hidden_states, encoder_hidden_states, encoder_hidden_states_mask, timestep, img_shapes, txt_seq_lens,
                      guidance, attention_kwargs)
    slot = int(self.cnt) % 2
    _take_residual(eng, self.residual_cache[slot], slot)
    out, stats = eng.calibrate(slot, compare=self.cnt >= 2)
    if stats is not None:  # :143-153
        norm_ratio, norm_std, cos_dis = stats
        self.norm_ratio.append(round(norm_ratio, 5))
        self.norm_std.append(round(norm_std, 5))
        self.cos_dis.append(round(cos_dis, 5))
        print(f"Step {self.cnt}: norm_ratio={norm_ratio:.5f}, norm_std={norm_std:.5f}, cos_dis={cos_dis:.5f}")
    self.residual_cache[slot] = eng.res[slot].view(1, *eng.res[slot].shape)  # :155
    self.cnt += 1
    if self.cnt >= self.num_steps:  # :158-163
        self.cnt = 0
        print("\nCalibration Results:")
        print("norm_ratio:", self.norm_ratio)
        print("norm_std:", self.norm_std)
        print("cos_dis:", self.cos_dis)
    output = out.view(1, *out.shape)
    return _Sample(output) if return_dict else (output,)


def init_magcache_qwen_image(model, mag_ratios, sample_steps=50, thresh=0.06, K=2, retention_ratio=0.2):
    """`init_magcache(model, mag_ratios, args)` of MagCache4QwenImage/magcache_generate.py:63-83 (and the Edit script): patches the
    CLASS. `mag_ratios`: the list without its `[1.0]*2` prefix as the scripts pass it, or a key of `tables()` ("qwen_image",
    "qwen_image_edit"), which carries the prefix. A table of another length is resampled per branch by `np.linspace` rounding."""
    cls = model.__class__
    cls.forward = magcache_qwen_image_forward
    cls.cnt = torch.tensor(0)
    cls.num_steps = sample_steps * 2
    cls.split_step, cls.mode = None, "t2v"
    cls.magcache_thresh, cls.K = thresh, K
    cls.accumulated_err, cls.accumulated_steps, cls.accumulated_ratio = [0.0, 0.0], [0, 0], [1.0, 1.0]
    cls.retention_ratio = retention_ratio
    cls.residual_cache = [None, None]
    mr = tables()[mag_ratios] if isinstance(mag_ratios, str) else np.array([1.0] * 2 + list(mag_ratios))
    if len(mr) != sample_steps * 2:  # :79-83
        con, ucon = nearest_interp_linspace(mr[0::2], sample_steps), nearest_interp_linspace(mr[1::2], sample_steps)
        mr = np.concatenate([con.reshape(-1, 1), ucon.reshape(-1, 1)], axis=1).flatten()
    cls.mag_ratios = mr
    return model


def init_magcache_qwen_image_calibration(model, sample_steps=50):
    """`init_magcache_calibration(model, args)` of MagCache4QwenImage/magcache_generate.py:85-92."""
    cls = model.__class__
    cls.forward = magcache_qwen_image_calibration
    cls.cnt = torch.tensor(0)
    cls.num_steps = sample_steps * 2
    cls.norm_ratio, cls.norm_std, cls.cos_dis = [], [], []
    cls.residual_cache = [None, None]
    return model


# ------------------------------------------------------------------------------------------------------------------
# Open-Sora 1.2 (STDiT3), the paper-evaluation forward behind the published Open-Sora numbers
# ------------------------------------------------------------------------------------------------------------------
def _opensora_unsupported(self, x_mask, kw):
    if x_mask is not None:
        raise NotImplementedError("magcache_b200: Open-Sora x_mask (image / video conditioning with t0) is not supported")
    pm = getattr(self, "parallel_manager", None)
    if pm is not None and (getattr(pm, "sp_size", 1) > 1 or getattr(pm, "cp_size", 1) > 1):
        raise NotImplementedError("magcache_b200: VideoSys's own Open-Sora sequence / CFG parallelism (sp_size or cp_size > 1) is not "
                                  "supported; keep sp_size = cp_size = 1 and call magcache_b200.enable_sequence_parallel")
    try:
        from videosys.core.pab_mgr import enable_pab
        pab = enable_pab()
    except Exception:  # videosys absent or PAB never configured
        pab = False
    if pab:
        raise NotImplementedError("magcache_b200: Open-Sora with PAB enabled is not supported")
    if getattr(getattr(self, "config", None), "skip_y_embedder", False):
        raise NotImplementedError("magcache_b200: Open-Sora with skip_y_embedder is not supported")


def opensora_engine(self, device):
    """The Open-Sora engine cached on the module, built on `device` at first use."""
    sp = self.__dict__.get("_mc_sp_kw", {})  # enable_sequence_parallel
    return _cached_engine(self, "_mc_opensora_engine", lambda **skw: OpenSoraEngine(OpenSoraWeights.from_module(self, device), **skw, **sp))


def _opensora_stage(self, x, timestep, y, mask, x_mask, fps, height, width, kw):
    _opensora_unsupported(self, x_mask, kw)
    if not x.is_cuda:
        raise RuntimeError("magcache_b200: x must be a CUDA tensor (no CPU path)")
    eng = opensora_engine(self, x.device)
    eng.stage_inputs(x, timestep, y, mask, fps, height, width)
    return eng


def magcache_opensora_forward(self, x, timestep, all_timesteps, y, mask=None, x_mask=None, fps=None, height=None, width=None, **kw):
    r"""eval/magcache/experiments/opensora.py:229-373 on the H100 kernels (magcache_b200/opensora.py), with the same signature and
    class attributes (`t, skip_time, K, magcache_thresh, ratio, accumulated_sim / _err / _steps, skip_steps, residual_cache`).
    The decision is the `"opensora"` controller family (`ratio[t-1]`, signed error, explicit `skip_time`), the counter wraps at 30
    (:349-354) and the skip line of :312 is printed. `residual_cache` is the engine's one residual buffer viewed as (B, N, C, 1): the
    reference's depth-3 FIFO is only ever read at [..., -1]; a tensor the caller puts there is honoured through its [..., -1].
    Cross-attention follows `flash_attn_varlen_func`: each sample attends to its own `y_lens[b]` caption tokens (the default
    `torch_impl` agrees whenever the lengths are equal, as for one prompt's CFG pair). Under `enable_sequence_parallel` the cache is
    sharded as in the reference (:342-347): `residual_cache` is (B, N_r, C, 1), this rank's frames."""
    eng = _opensora_stage(self, x, timestep, y, mask, x_mask, fps, height, width, kw)
    skip_forward = self.t >= self.skip_time and _ctrl(self, "opensora").decide(self)  # :297-308
    cur = self.residual_cache
    _take_residual(eng, cur[..., -1] if torch.is_tensor(cur) else cur)
    if skip_forward:
        self.skip_steps += 1
        print(f"skip time {self.t}, cur_scale: {self.ratio[self.t-1]}, acc_sim: {self.accumulated_sim}, total_steps: {self.skip_steps}")  # :312
    out = eng.forward("hit" if skip_forward else "miss")
    self.residual_cache = eng.res.view(eng.B, eng.N, -1, 1)  # :344-347
    self.t += 1                                        # :348-354
    if self.t >= 30:
        self.t = 0
        self.accumulated_sim = 1.0
        self.accumulated_steps = 0
        self.accumulated_err = 0
        self.skip_steps = 0
    return out


def init_magcache_opensora(transformer, thresh=0.12, K=3, skip_time=6, ratio=None):
    """The installation block of `eval_ours` (opensora.py:418-436): the paper's presets are 0.12 / K3 and 0.24 / K5, skip_time 6."""
    cls = transformer.__class__
    cls.forward = magcache_opensora_forward
    cls.magcache_thresh, cls.K, cls.skip_time = thresh, K, skip_time
    cls.t, cls.residual_cache, cls.accumulated_err, cls.accumulated_sim, cls.accumulated_steps, cls.skip_steps = 0, None, 0, 1, 0, 0
    cls.cache_time = 4
    cls.ratio = np.asarray(tables()["opensora_eval"] if ratio is None else ratio, dtype=np.float64)
    return transformer


_TEA_OS = OpenSoraTeaController()


def teacache_opensora_forward(self, x, timestep, all_timesteps, y, mask=None, x_mask=None, fps=None, height=None, width=None, **kw):
    r"""`teacache_forward` of eval/magcache/experiments/opensora.py:34-227 (the paper's TeaCache arm for Open-Sora) on the H100 kernels,
    with the same signature and class attributes (`enable_teacache, rel_l1_thresh, accumulated_rel_l1_distance,
    previous_modulated_input, previous_residual`). The decision input is block 0's first LN + t2i_modulate of `x_embedder(x) + pos_emb`
    over all samples; one fused kernel writes it and takes its relative L1 distance to the previous call's, and a miss feeds that
    same tensor to block 0's qkv projection. A call is forced when `timestep[0]` (rounded to bf16) equals the first or the last of
    `all_timesteps`; there is no counter and nothing is reset between videos. `previous_modulated_input` / `previous_residual` are
    views of the engine's buffers, (B, N, C); a tensor the caller puts there is honoured. With `enable_teacache` False the call is the
    plain forward (`eval_base`). Unsupported inputs raise as in `magcache_opensora_forward`. Under `enable_sequence_parallel` the
    decision input still covers every row on every rank (the reference forms it before its split), but `previous_residual` is
    (B, N_r, C), this rank's frames: the reference gathers it to full size (:199-209) only to add its own frames back after the split,
    so keeping it sharded changes no output."""
    eng = _opensora_stage(self, x, timestep, y, mask, x_mask, fps, height, width, kw)
    if not self.enable_teacache:  # :157-197
        return eng.forward_plain()
    eng.prologue("hit")  # x_embedder + pos_emb, t / fps / t_block; the caption MLP waits for the decision
    ts = timestep.to(torch.bfloat16)  # `timestep = timestep.to(dtype)` (:51)
    forced = bool(ts[0] == all_timesteps[0] or ts[0] == all_timesteps[-1])  # :96
    eng.take_modulated_input(self.previous_modulated_input)
    if not forced and eng.mi_prev is None:
        raise TypeError("magcache_b200: TeaCache distance with no previous_modulated_input (reference: Tensor - NoneType)")
    sums = eng.modulated_input(distance=not forced)
    rel = None if forced else opensora_rel_l1(sums[0], sums[1], eng.R * eng.w.dim)
    calc = _TEA_OS.decide(self, forced, rel)  # :96-107
    self.previous_modulated_input = eng.mi[eng.mi_prev].view(eng.B, -1, eng.w.dim)  # :108 (every row, also under sequence parallelism)
    if not calc:
        _take_residual(eng, self.previous_residual)
    out = eng.forward_teacache(calc)
    if calc:
        self.previous_residual = eng.res.view(eng.B, eng.N, -1)  # :156
    return out


def init_teacache_opensora(transformer, rel_l1_thresh=0.1):
    """The attribute block of `eval_teacache_slow` / `eval_teacache_fast` (opensora.py:389-394, :403-408): thresholds 0.1 / 0.2."""
    cls = transformer.__class__
    cls.enable_teacache = True
    cls.rel_l1_thresh = rel_l1_thresh
    cls.accumulated_rel_l1_distance = 0
    cls.previous_modulated_input = None
    cls.previous_residual = None
    cls.forward = teacache_opensora_forward
    return transformer


# ------------------------------------------------------------------------------------------------------------------
# The paper-evaluation variant of the Wan forward (the code behind the published Wan2.1 numbers)
# ------------------------------------------------------------------------------------------------------------------
def magcache_eval_forward(self, x, t, context, seq_len, clip_fea=None, y=None):
    r"""eval/magcache/experiments/Wan2.1_EVAL/wan_magcache.py:682-817 on the H100 kernels, state under THAT script's attribute
    names (`t, num_steps, magcache_thresh, magcache_K, ratio, accumulated_sim, accumulated_err, accumulated_steps, residual_cache,
    skip_steps, pre_con`). Differences from `magcache_forward`, all reproduced: `<=` threshold compare, table indexed `ratio[t-10]`,
    retention fixed at `int(num_steps*0.2)`, residuals kept from call 10 on (`cache_time`) in a `[2, B, N, D, 1]` tensor — the
    depth-1 `push_tensor_roll` FIFO (:67-85, :796-799) is the engine's two residual slots viewed in place, no roll, no copy —
    and the conditional output of each step remembered in `pre_con` (:804-805)."""
    eng = _stage(self, x, t, context, seq_len, clip_fea, y)
    cache_time = 10                                  # :771
    skip_forward = _ctrl(self, "wan2.1-eval").decide(self)  # :774-786
    slot = self.t % 2
    if skip_forward:
        self.skip_steps += 1
        print(f"skip time {self.t}, cur_scale: {self.ratio[self.t - 10]}, acc_sim: {self.accumulated_sim[slot]}, total_steps: {self.skip_steps}")  # :790
    out = eng.forward("hit" if skip_forward else "miss", slot)
    if self.t >= cache_time:                         # :796-799
        self.residual_cache = eng.res_buf.view(2, 1, *eng.res_buf.shape[1:], 1)
    if self.t % 2 == 0:
        self.pre_con = [out]                         # :804-805
    self.t += 1                                      # :807-815
    if self.t >= self.num_steps:
        self.t = 0
        self.skip_steps = 0
        self.accumulated_sim = [1.0, 1.0]
        self.accumulated_steps = [0, 0]
        self.accumulated_err = [0, 0]
    return [out]


def init_magcache_eval(model, sample_steps, thresh=0.12, K=2, ratio=None):
    """The installation block of wan_magcache.py:1129-1150 as a helper ("slow" = 0.12/K2, "fast" = 0.12/K4, wan_eval.sh:30-31,66-67)."""
    cls = model.__class__
    cls.forward = magcache_eval_forward
    cls.magcache_thresh, cls.magcache_K = thresh, K
    cls.t, cls.accumulated_err, cls.skip_steps, cls.pre_con = 0, [0, 0], 0, None
    cls.num_steps = sample_steps * 2
    cls.ratio = np.asarray(tables()["wan2.1_eval"] if ratio is None else ratio, dtype=np.float64)
    cls.residual_cache = None
    cls.accumulated_sim, cls.accumulated_steps = [1, 1], [0, 0]
    return model


# ------------------------------------------------------------------------------------------------------------------
# TeaCache comparator (the baseline of every published MagCache table) on the same engine
# ------------------------------------------------------------------------------------------------------------------
# coefficients of eval/magcache/experiments/Wan2.1_EVAL/wan_teacache.py:913-926 (t2v) — keyed by (use_ret_steps, model size)
TEACACHE_COEFFICIENTS = {
    (True, "1.3B"): [-5.21862437e+04, 9.23041404e+03, -5.28275948e+02, 1.36987616e+01, -4.99875664e-02],
    (True, "14B"): [-3.03318725e+05, 4.90537029e+04, -2.65530556e+03, 5.87365115e+01, -3.15583525e-01],
    (False, "1.3B"): [2.39676752e+03, -1.31110545e+03, 2.01331979e+02, -8.29855975e+00, 1.37887774e-01],
    (False, "14B"): [-5784.54975374, 5449.50911966, -1811.16591783, 256.27178429, -13.02252404],
}


_TEA = TeaController()


def teacache_forward(self, x, t, context, seq_len, clip_fea=None, y=None):
    r"""eval/magcache/experiments/Wan2.1_EVAL/wan_teacache.py:457-590 on the H100 kernels, state under the reference's attribute
    names (`cnt, num_steps, teacache_thresh, accumulated_rel_l1_distance_even/odd, previous_e0_even/odd,
    previous_residual_even/odd, use_ref_steps, ret_steps, cutoff_steps, coefficients, enable_teacache`). The decision reads the
    relative L1 change of the modulated time embedding (one tiny reduction + the `.item()` sync the reference has), the hit /
    miss branches are the MagCache ones (`x += previous_residual` | block stack, residual = x - ori_x)."""
    eng = _stage(self, x, t, context, seq_len, clip_fea, y)
    if not self.enable_teacache:  # :584-586: plain forward (the counter still advances, :587-589)
        out = eng.forward("miss", self.cnt % 2)
        self.cnt = 0 if self.cnt + 1 >= self.num_steps else self.cnt + 1
        return [out]
    slot = self.cnt % 2
    suffix = "even" if slot == 0 else "odd"
    e, e0 = eng.time_embedding()
    emb = e0 if self.use_ref_steps else e
    modulated = emb.reshape(-1)  # :534
    calc = _TEA.decide(self, lambda: ops.rel_l1(modulated, getattr(self, "previous_e0_" + suffix).reshape(-1)))
    setattr(self, "previous_e0_" + suffix, modulated.clone().view(emb.shape))  # :549 / :564
    _take_residual(eng, getattr(self, "previous_residual_" + suffix), slot)
    eng.hit_sum_bf16 = True  # `x += self.previous_residual_*` in place on the bf16 patch embedding (:569 / :577): the sum is rounded to bf16
    try:
        out = eng.forward("miss" if calc else "hit", slot)
    finally:
        eng.hit_sum_bf16 = False
    setattr(self, "previous_residual_" + suffix, eng.res[slot].view(1, *eng.res[slot].shape))
    _TEA.advance(self)  # :587-589
    return [out]


def init_teacache(model, sample_steps, teacache_thresh=0.2, use_ret_steps=False, ckpt_dir=None, coefficients=None):
    """The installation block of wan_teacache.py:899-928 as a helper: patches the CLASS. Coefficients are chosen by the '1.3B' /
    '14B' substring of `ckpt_dir` like the reference, or passed explicitly."""
    cls = model.__class__
    cls.enable_teacache = True
    cls.forward = teacache_forward
    cls.cnt = 0
    cls.num_steps = sample_steps * 2
    cls.teacache_thresh = teacache_thresh
    cls.accumulated_rel_l1_distance_even = 0
    cls.accumulated_rel_l1_distance_odd = 0
    cls.previous_e0_even = cls.previous_e0_odd = None
    cls.previous_residual_even = cls.previous_residual_odd = None
    cls.use_ref_steps = use_ret_steps
    if coefficients is None:
        size = "1.3B" if "1.3B" in (ckpt_dir or "") else ("14B" if "14B" in (ckpt_dir or "") else None)
        if size is None:
            raise KeyError(f"no TeaCache coefficients match ckpt_dir={ckpt_dir!r} (the reference would hit AttributeError later)")
        coefficients = TEACACHE_COEFFICIENTS[(bool(use_ret_steps), size)]
    cls.coefficients = list(coefficients)
    if use_ret_steps:
        cls.ret_steps, cls.cutoff_steps = 10 * 2, sample_steps * 2
    else:
        cls.ret_steps, cls.cutoff_steps = 1 * 2, sample_steps * 2 - 2
    return model
