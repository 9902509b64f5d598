#!/usr/bin/env python
"""Generate tests/golden/opensora_forward.npz and opensora_forward.json by EXECUTING the reference's own Open-Sora code.

Run where the reference tree is present (it is not imported by anything else):

    python tests/golden/make_opensora_golden.py

videosys cannot be imported offline (timm, transformers, flash-attn, rotary_embedding_torch are absent), so this script parses the
sources with `ast`, cuts out these top-level definitions and executes them unmodified:

* videosys/models/transformers/open_sora_transformer_3d.py: t2i_modulate, T2IFinalLayer, auto_grad_checkpoint, STDiT3Block,
  STDiT3Config, STDiT3 (forward, encode_text, unpatchify, get_dynamic_size, initialize_weights, __init__)
* videosys/models/modules/attentions.py: OpenSoraAttention, OpenSoraMultiHeadCrossAttention (forward / torch_impl)
* videosys/models/modules/normalization.py: LlamaRMSNorm
* videosys/models/modules/embeddings.py: OpenSoraPatchEmbed3D, TimestepEmbedder, SizeEmbedder, OpenSoraCaptionEmbedder,
  OpenSoraPositionEmbedding2D
* videosys/models/modules/activations.py: approx_gelu
* eval/magcache/experiments/opensora.py: push_tensor_roll, magcache_forward, and the class-attribute statements of eval_ours
  (:418-433), executed against a stand-in `engine` whose driver_worker.transformer is the model

Stand-ins only for what is absent offline: timm's Mlp / DropPath, transformers' PretrainedConfig / PreTrainedModel (a config
holder over nn.Module), rotary_embedding_torch.RotaryEmbedding (tests/opensora_ref.py's restatement), a parallel manager with
sp = cp = 1, PAB off. The parameters come from `opensora_ref.synthetic_state(seed)` by name; their per-tensor checksums are stored,
not the weights.

Fixture: a tiny STDiT3 (hidden 144, 2 heads x 72, depth 2, 12 caption tokens x 64), B = 2 with distinct per-sample timesteps,
T = 2 latent frames of 6 x 8, over the 30 calls of one video under the slow preset (0.12 / K3 / skip_time 6), in fp32 and in bf16
(parameters cast, buffers left fp32 as `from_pretrained(torch_dtype=bf16)` leaves them); the outputs of every call, the controller
attributes after every call, and the skip masks of both presets.
"""
import ast
import contextlib
import functools
import io
import json
import math
import os
import sys
import types
from collections.abc import Iterable
from functools import partial

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from einops import rearrange

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import opensora_ref as R  # noqa: E402

REF = "/root/reference"
VS = f"{REF}/videosys/models"
SOURCES = {  # in dependency order: default arguments are evaluated when a class body runs
    f"{VS}/modules/normalization.py": ["LlamaRMSNorm"],
    f"{VS}/modules/activations.py": ["approx_gelu"],
    f"{VS}/modules/embeddings.py": ["OpenSoraPatchEmbed3D", "TimestepEmbedder", "SizeEmbedder", "OpenSoraCaptionEmbedder", "OpenSoraPositionEmbedding2D"],
    f"{VS}/modules/attentions.py": ["OpenSoraAttention", "OpenSoraMultiHeadCrossAttention"],
    f"{VS}/transformers/open_sora_transformer_3d.py": ["t2i_modulate", "T2IFinalLayer", "auto_grad_checkpoint", "STDiT3Block", "STDiT3Config", "STDiT3"],
    f"{REF}/eval/magcache/experiments/opensora.py": ["push_tensor_roll", "magcache_forward"],
}
EVAL = f"{REF}/eval/magcache/experiments/opensora.py"
SEED = 0
CFG = dict(hidden_size=144, depth=2, num_heads=2, caption_channels=64, model_max_length=12)
B, T, H, W = 2, 2, 6, 8


def _defs(path, names):
    src = open(path).read()
    out = {}
    for node in ast.parse(src).body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in names:
            out[node.name] = ast.get_source_segment(src, node)
        elif isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id in names for t in node.targets):
            out[node.targets[0].id] = ast.get_source_segment(src, node)
    missing = set(names) - set(out)
    assert not missing, (path, missing)
    return [out[n] for n in names]


def _eval_ours_statements():
    src = open(EVAL).read()
    fn = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "eval_ours")
    keep = [ast.get_source_segment(src, st) for st in fn.body if "driver_worker.transformer.__class__" in ast.get_source_segment(src, st)]
    return "\n".join(keep)


# ---- stand-ins for the modules absent offline --------------------------------------------------------------------
class Mlp(nn.Module):  # timm.models.vision_transformer.Mlp (drop 0, no norm)
    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.0):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = act_layer()
        self.fc2 = nn.Linear(hidden_features, out_features)

    def forward(self, x):
        return self.fc2(self.act(self.fc1(x)))


class DropPath(nn.Identity):
    def __init__(self, *a, **k):
        super().__init__()


class PretrainedConfig:
    def __init__(self, **kwargs):
        for k, v in kwargs.items():
            setattr(self, k, v)


class PreTrainedModel(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config


class _PM:
    sp_size = cp_size = 1


def _namespace():
    rot = types.ModuleType("rotary_embedding_torch")
    rot.RotaryEmbedding = R.RotaryEmbedding
    sys.modules["rotary_embedding_torch"] = rot
    ns = dict(torch=torch, nn=nn, F=F, np=np, math=math, functools=functools, rearrange=rearrange, partial=partial, Iterable=Iterable,
              Optional=__import__("typing").Optional, Mlp=Mlp, DropPath=DropPath, PretrainedConfig=PretrainedConfig,
              PreTrainedModel=PreTrainedModel, enable_pab=lambda: False, checkpoint=None, checkpoint_sequential=None,
              ParallelManager=_PM, batch_func=None, split_sequence=None, gather_sequence=None, set_pad=None, get_pad=None,
              all_to_all_with_pad=None, autocast=torch.amp.autocast)
    for path, names in SOURCES.items():
        for seg in _defs(path, names):
            exec(compile(seg, path, "exec"), ns)  # noqa: S102
    return ns


def build_reference(ns, dtype):
    cfg = ns["STDiT3Config"](**CFG)
    model = ns["STDiT3"](cfg)
    shapes = {n: p.shape for n, p in model.named_parameters()}
    ours = {n for n, _ in R.STDiT3(**CFG).named_parameters()}
    assert set(shapes) == ours, sorted(set(shapes) ^ ours)
    state = R.synthetic_state(shapes, SEED)
    with torch.no_grad():
        for n, p in model.named_parameters():
            p.copy_(state[n])
            p.data = p.data.to(dtype)
    pm = _PM()
    model.parallel_manager = pm
    for blk in list(model.spatial_blocks) + list(model.temporal_blocks):
        blk.parallel_manager = pm
    model.eval()
    model.__class__ = type(f"RefSTDiT3_{dtype}", (ns["STDiT3"],), {})
    engine = types.SimpleNamespace(driver_worker=types.SimpleNamespace(transformer=model))
    exec(_eval_ours_statements(), dict(engine=engine, np=np, magcache_forward=ns["magcache_forward"]))  # noqa: S102
    return model, state


def inputs():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, 4, T, H, W, generator=g)
    y = torch.randn(B, 1, CFG["model_max_length"], CFG["caption_channels"], generator=g)
    mask = torch.ones(B, CFG["model_max_length"], dtype=torch.long)
    kw = dict(mask=mask, fps=torch.tensor([24.0]), height=torch.tensor([8.0 * H]), width=torch.tensor([8.0 * W]))
    return x, y, kw


def timesteps(i):
    return torch.tensor([1000.0 - 33.0 * i, 990.0 - 31.0 * i])


ATTRS = ("t", "accumulated_sim", "accumulated_err", "accumulated_steps", "skip_steps")


def run(model, calls=30):
    x, y, kw = inputs()
    outs, attrs = [], []
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()) as log:
        for i in range(calls):
            outs.append(model(x, timesteps(i), None, y, **kw).numpy())
            attrs.append({a: float(getattr(model, a)) for a in ATTRS})
    return np.stack(outs), attrs, log.getvalue()


def skip_mask(log, calls=30):
    hit = {int(line.split(",")[0].split()[-1]) for line in log.splitlines() if line.startswith("skip time")}
    return [int(i in hit) for i in range(calls)]


def main():
    ns = _namespace()
    doc = {"config": CFG, "B": B, "T": T, "H": H, "W": W, "seed": SEED, "timesteps": [timesteps(i).tolist() for i in range(30)]}
    arrays = {}
    for name, dtype in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        model, state = build_reference(ns, dtype)
        out, attrs, log = run(model)
        arrays[name] = out.astype(np.float32)
        doc[f"attrs_{name}"] = attrs
        doc[f"mask_{name}"] = skip_mask(log)
    doc["checksums"] = {n: [float(t.double().sum()), float(t.double().abs().sum())] for n, t in sorted(state.items())}
    model, _ = build_reference(ns, torch.float32)
    model.__class__.magcache_thresh, model.__class__.K = 0.24, 5  # the fast preset (eval/magcache/README.md:66)
    _, _, log = run(model)
    doc["mask_fast"] = skip_mask(log)
    np.savez_compressed(os.path.join(HERE, "opensora_forward.npz"), **arrays)
    with open(os.path.join(HERE, "opensora_forward.json"), "w") as f:
        json.dump(doc, f, indent=1)
    print("masks", doc["mask_fp32"], doc["mask_fast"])


if __name__ == "__main__":
    main()
