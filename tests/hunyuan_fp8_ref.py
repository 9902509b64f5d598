"""ORACLE — test infrastructure only (imported by tests/ and tools/, never by the product).

CPU restatement of HunyuanVideo's FP8 weight mode, the `--use-fp8 --dit-weight ..._fp8.pt` run of MagCache4HunyuanVideo/README.md:76-96,
for models built from oracle/hunyuan_ref.py, plus the emulation of `ops.dequant_fp8_bf16` for the engine tests that run the kernels
emulated (tests/emu_ops.py).

PARITY UNPINNED: `convert_fp8_linear`, `fp8_linear_forward` and `fp8_activation_dequant` live in hyvideo/modules/fp8_optimization.py
[EXT] (github Tencent/HunyuanVideo), which is not under /root/reference and is unpinned by it, like the rest of hyvideo. What follows
restates them:
  - every nn.Linear whose module name contains `double_blocks` or `single_blocks` gets its weight as float8_e4m3fn and a scalar
    `fp8_scale` in the model dtype (bf16); `txt_in`, `final_layer`, `time_in`, `vector_in`, `guidance_in` and `img_in` stay bf16;
  - its forward is `F.linear(input, qdata.to(bf16) * scale.to(bf16), bias)`: the dequantised weight is rounded to bf16, the GEMM is
    the ordinary bf16 one.
One upstream statement is not reproduced: the guard `cls.weight.sum() != 0`, which falls back to the module's own forward. It only
matters for a weight whose values cancel to exactly zero, and torch has no float8 `sum` on CPU.

FP8 checkpoints come quantised upstream; `to_fp8_checkpoint` makes one from a synthetic model with the rule
`scale = bf16(amax / 448)`, `q = (w / scale).to(float8_e4m3fn)` (clamped to the format's range, as upstream's fp8_tensor_quant).
"""
import copy
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

FP8 = torch.float8_e4m3fn
FP8_MAX = 448.0  # torch.finfo(torch.float8_e4m3fn).max


def converted(key, layer):
    """The Linears upstream's convert_fp8_linear converts."""
    return isinstance(layer, nn.Linear) and ("double_blocks" in key or "single_blocks" in key)


def fp8_quantize(w):
    """(codes, scale) of one Linear's weight: scale = bf16(amax / 448), q = (w / scale) clamped to +-448, as float8_e4m3fn."""
    w = w.detach()
    scale = (w.abs().max().float() / FP8_MAX).to(torch.bfloat16)
    q = (w.float() / scale.float()).clamp(-FP8_MAX, FP8_MAX).to(FP8)
    return q, scale


def fp8_activation_dequant(qdata, scale, dtype):
    return qdata.to(dtype) * scale.to(dtype)


def fp8_linear_forward(cls, original_dtype, input):
    w = fp8_activation_dequant(cls.weight, cls.fp8_scale.to(cls.weight.device), original_dtype)
    return F.linear(input, w, cls.bias)


def _forward(self, input):
    return fp8_linear_forward(self, self.fp8_original_dtype, input)


def convert_fp8_linear(module, fp8_map, original_dtype=torch.bfloat16):
    """Upstream's convert_fp8_linear with the `_map.pt` file given as a dict {module name: scale}. A bound method replaces the forward
    (upstream: a lambda), so that copy.deepcopy of the module rebinds it to the copy."""
    module.fp8_matmul_enabled = True
    for key, layer in module.named_modules():
        if converted(key, layer):
            layer.weight = nn.Parameter(layer.weight.detach().to(FP8), requires_grad=False)
            layer.fp8_scale = fp8_map[key].to(dtype=original_dtype)
            layer.fp8_original_dtype = original_dtype
            layer.forward = types.MethodType(_forward, layer)
    return module


def to_fp8_checkpoint(model):
    """`model` (bf16) as an FP8 checkpoint loaded into it and converted: the block Linears hold the codes of `fp8_quantize`."""
    fp8_map = {}
    with torch.no_grad():
        for key, layer in model.named_modules():
            if converted(key, layer):
                q, s = fp8_quantize(layer.weight)
                layer.weight.copy_(q.to(layer.weight.dtype))  # loading the checkpoint into the bf16 model: exact
                fp8_map[key] = s
    return convert_fp8_linear(model, fp8_map)


def dequantized(model):
    """A bf16 copy of an FP8 model whose block Linears hold `qdata.to(bf16) * scale` with the ordinary forward: the bf16 model the
    checkpoint stands for."""
    m = copy.deepcopy(model)
    with torch.no_grad():
        for _, layer in m.named_modules():
            if "fp8_scale" in layer.__dict__:
                layer.weight = nn.Parameter(fp8_activation_dequant(layer.weight, layer.fp8_scale.to(layer.weight.device), torch.bfloat16))
                for attr in ("forward", "fp8_scale", "fp8_original_dtype"):
                    delattr(layer, attr)
    m.__dict__.pop("fp8_matmul_enabled", None)
    return m


def emu_dequant_fp8_bf16(q, scale, out, tag=None):
    """Emulation of `ops.dequant_fp8_bf16` (mc_dequant_fp8_bf16) with its preconditions."""
    import emu_ops
    assert q.dtype == FP8 and scale.dtype == torch.bfloat16 and out.dtype == torch.bfloat16
    assert q.dim() == 2 and q.is_contiguous() and scale.is_contiguous() and out.is_contiguous()
    assert scale.shape == (q.shape[0],) and out.shape == q.shape
    out.copy_((q.to(torch.float32) * scale.to(torch.float32)[:, None]).to(torch.bfloat16))
    emu_ops._count()
    return out
