"""Unmerged LoRA adapters for the FLUX tests: a PEFT-layout LoRA layer, its injection into the oracle's FluxTransformer2DModel, the
reference's scale / unscale statements around the oracle's forward, and the tailed GEMM in the kernel emulation.

PEFT and diffusers are not part of this project: `LoraLinear.forward` restates PEFT's `lora.Linear.forward` (non-DoRA), and
`scale_lora_layers` / `unscale_lora_layers` restate diffusers' functions of those names with PEFT's `scale_layer` /
`unscale_layer` / `set_scale` (parity unpinned, like oracle/sampler_ref.py). `reference_lora` wraps the oracle's forward (or its
calibration twin) in the reference's statements: MagCache4FLUX/magcache_flux.py:274-287 before and :437-439 after (calibration
:62-75, :224-226; Kontext magcache_flux_kontext.py:279-289, :439-441, :64-74, :226-228).

`emu` is tests/flux_controlnet_ref.py's emulation with `gemm(tail=(U, T))`: the tail as more K columns of one fp32 GEMM."""
import math
import types

import torch
from torch import nn

import flux_controlnet_ref as cref
from magcache_b200 import _lib as L


class LoraLinear(nn.Module):
    """The attribute surface of PEFT's `lora.Linear` around an nn.Linear."""

    def __init__(self, base):
        super().__init__()
        self.base_layer = base
        self.lora_A, self.lora_B, self.lora_dropout = nn.ModuleDict(), nn.ModuleDict(), nn.ModuleDict()
        self.scaling, self.lora_alpha, self.r, self.use_dora, self.use_rslora = {}, {}, {}, {}, {}
        self.merged_adapters = []
        self.disable_adapters = False
        self._active = []

    @property
    def weight(self):
        return self.base_layer.weight

    @property
    def bias(self):
        return self.base_layer.bias

    @property
    def merged(self):
        return bool(self.merged_adapters)

    @property
    def active_adapters(self):
        return list(self._active)

    def update_layer(self, name, r, alpha, g, zero_b=False, dropout=0.0, rslora=False):
        base = self.base_layer
        A = nn.Linear(base.in_features, r, bias=False)
        B = nn.Linear(r, base.out_features, bias=False)
        with torch.no_grad():
            A.weight.copy_(torch.randn(r, base.in_features, generator=g) / math.sqrt(base.in_features))
            B.weight.copy_(torch.zeros(base.out_features, r) if zero_b else 0.3 / math.sqrt(r) * torch.randn(base.out_features, r, generator=g))
        dt = base.weight.dtype
        self.lora_A[name], self.lora_B[name] = A.to(dt), B.to(dt)
        self.lora_dropout[name] = nn.Dropout(dropout) if dropout > 0 else nn.Identity()
        self.r[name], self.lora_alpha[name], self.use_rslora[name], self.use_dora[name] = r, alpha, rslora, False
        self.scaling[name] = alpha / (math.sqrt(r) if rslora else r)
        if name not in self._active:
            self._active.append(name)

    def delta(self, a):
        return (self.lora_B[a].weight.float() @ self.lora_A[a].weight.float()) * self.scaling[a]

    def merge(self):
        with torch.no_grad():
            for a in self.active_adapters:
                if a in self.lora_A.keys() and a not in self.merged_adapters:
                    self.base_layer.weight.data += self.delta(a).to(self.base_layer.weight.dtype)
                    self.merged_adapters.append(a)

    def unmerge(self):
        with torch.no_grad():
            while self.merged_adapters:
                a = self.merged_adapters.pop()
                self.base_layer.weight.data -= self.delta(a).to(self.base_layer.weight.dtype)

    def forward(self, x):
        result = self.base_layer(x)
        if self.disable_adapters or self.merged:
            return result
        for a in self.active_adapters:
            if a not in self.lora_A.keys():
                continue
            result = result + self.lora_B[a](self.lora_A[a](self.lora_dropout[a](x))) * self.scaling[a]
        return result


# module-path suffixes of the covered targets inside a block, by set; "all" adds the top-level TOP
ATTN = ("attn.to_q", "attn.to_k", "attn.to_v", "attn.to_out.0", "attn.add_q_proj", "attn.add_k_proj", "attn.add_v_proj", "attn.to_add_out")
BLOCKS = ATTN + ("ff.net.0.proj", "ff.net.2", "ff_context.net.0.proj", "ff_context.net.2", "proj_mlp", "proj_out")
ADA = ("norm1.linear", "norm1_context.linear", "norm.linear")
TOP = ("x_embedder", "context_embedder", "proj_out", "norm_out.linear")
TARGETS = {"attn": ATTN, "blocks": BLOCKS, "ada": BLOCKS + ADA, "all": BLOCKS + ADA}


def target_names(model, targets, blocks=None):
    """Module paths of `model`'s Linears in the target set `targets` (a key of TARGETS). `blocks`: None, or a predicate on the
    path that keeps only some blocks' Linears."""
    names = []
    for name, m in model.named_modules():
        if not isinstance(m, nn.Linear) or any(p in name.split(".") for p in ("base_layer", "lora_A", "lora_B")):
            continue
        if name.startswith(("transformer_blocks.", "single_transformer_blocks.")):
            if name.split(".", 2)[2] in TARGETS[targets] and (blocks is None or blocks(name)):
                names.append(name)
        elif targets == "all" and name in TOP:
            names.append(name)
    return names


def inject_lora(model, targets, adapters=("a",), rank=8, alpha=None, seed=0, names=None, **kw):
    """Wrap every Linear named by `names` (default: target_names(model, targets)) in a LoraLinear and add each adapter of
    `adapters` with rank `rank` (alpha = rank unless given). Returns the wrapped layers."""
    g = torch.Generator().manual_seed(seed)
    names = target_names(model, targets) if names is None else names
    out = []
    for name in names:
        parent, child = name.rsplit(".", 1) if "." in name else ("", name)
        p = model.get_submodule(parent) if parent else model
        m = p._modules[child]
        if not isinstance(m, LoraLinear):
            m = LoraLinear(m)
            p._modules[child] = m
        for a in adapters:
            m.update_layer(a, rank, rank if alpha is None else alpha, g, **kw)
        out.append(m)
    return out


def unload_lora(model):
    """diffusers `unload_lora_weights`: every LoRA layer replaced by its base layer (merged updates stay in the base weights)."""
    for name, m in list(model.named_modules()):
        if isinstance(m, LoraLinear):
            parent, child = name.rsplit(".", 1) if "." in name else ("", name)
            (model.get_submodule(parent) if parent else model)._modules[child] = m.base_layer


def lora_layers(model):
    return [m for m in model.modules() if isinstance(m, LoraLinear)]


def set_adapters(model, names, weights=None):
    """diffusers `set_adapters`: the active adapters and scaling = weight * alpha / r for each."""
    weights = [1.0] * len(names) if weights is None else weights
    for m in lora_layers(model):
        m._active = [n for n in names if n in m.lora_A.keys()]
        for n, w in zip(names, weights):
            if n in m.scaling:
                m.scaling[n] = w * m.lora_alpha[n] / m.r[n]


def scaling_state(model):
    return [dict(m.scaling) for _, m in sorted(((n, m) for n, m in model.named_modules() if isinstance(m, LoraLinear)), key=lambda x: x[0])]


def scale_lora_layers(model, weight):
    if weight == 1.0:
        return
    for m in model.modules():
        if isinstance(m, LoraLinear):
            if weight == 1:
                continue
            for a in m.active_adapters:
                if a not in m.lora_A.keys():
                    continue
                m.scaling[a] *= weight


def unscale_lora_layers(model, weight=None):
    if weight is None or weight == 1.0:
        return
    for m in model.modules():
        if isinstance(m, LoraLinear):
            if weight != 0:
                for a in m.active_adapters:
                    if a not in m.lora_A.keys():
                        continue
                    m.scaling[a] /= weight
            else:
                for a in m.active_adapters:
                    if a not in m.scaling:
                        continue
                    r = m.r[a]
                    m.scaling[a] = 1.0 * m.lora_alpha[a] / (math.sqrt(r) if m.use_rslora.get(a, False) else r)


def reference_lora(inner):
    """The oracle's forward (or calibration twin) `inner` inside the reference's LoRA-scale statements."""

    def forward(self, *args, joint_attention_kwargs=None, **kw):
        if joint_attention_kwargs is not None:
            joint_attention_kwargs = joint_attention_kwargs.copy()
            lora_scale = joint_attention_kwargs.pop("scale", 1.0)
        else:
            lora_scale = 1.0
        scale_lora_layers(self, lora_scale)
        out = inner(self, *args, **kw)
        unscale_lora_layers(self, lora_scale)
        return out

    return forward


def gemm(a, b, bias=None, epilogue=L.MC_EPI_BIAS_BF16, out=None, gate=None, tag=None, addend=None, addend_row0=0, tail=None):
    """flux_controlnet_ref.gemm; with a tail (U [M, R], T [N, R]): acc = a b^T + U T^T, one fp32 sum over [a | U] and [b | T]."""
    if tail is None:
        return cref.gemm(a, b, bias, epilogue, out=out, gate=gate, tag=tag, addend=addend, addend_row0=addend_row0)
    u, t = tail
    R = u.shape[1]
    assert epilogue in (L.MC_EPI_BIAS_BF16, L.MC_EPI_BIAS_GELU_BF16, L.MC_EPI_BIAS_GATE_RESID_BF16)
    assert u.dtype == torch.bfloat16 and t.dtype == torch.bfloat16 and u.shape == (a.shape[0], R) and t.shape == (b.shape[0], R)
    assert R >= 8 and R % 8 == 0 and u.stride(1) == 1 and t.stride(1) == 1 and u.stride(0) % 8 == 0 and t.stride(0) % 8 == 0
    assert u.data_ptr() % 16 == 0 and t.data_ptr() % 16 == 0, "mc_gemm_bf16_lora: U/T must be 16-byte aligned"
    return cref.gemm(torch.cat([a, u], 1), torch.cat([b, t], 1), bias, epilogue, out=out, gate=gate, tag=tag, addend=addend,
                     addend_row0=addend_row0)


emu = types.ModuleType("emu_ops_lora")
emu.__dict__.update({k: v for k, v in vars(cref.emu).items() if not k.startswith("__")})
emu.gemm = gemm

