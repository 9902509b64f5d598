#!/usr/bin/env python
"""Generate tests/golden/qwen_image.json and qwen_image.npz by EXECUTING the reference's own Qwen-Image MagCache statements.

Run where the reference tree is present (it is not imported by anything else):

    python tests/golden/make_qwen_image_golden.py [REFERENCE_ROOT]

diffusers is not installed, so the scripts cannot be imported; this parses MagCache4QwenImage/magcache_generate.py and
MagCache4QwenImageEdit/magcache_generate.py with `ast`, cuts out `nearest_interp`, `init_magcache`, `init_magcache_calibration`,
`magcache_calibration` and `magcache_forward`, and executes them unmodified, with stand-ins only for diffusers'
`Transformer2DModelOutput` (an object with `.sample`) and `USE_PEFT_BACKEND = False`, on the tiny model of tests/qwen_image_ref.py
(2 blocks, 2 heads x 128, seed 0). Each run is 2 generations of 50 steps x 2 calls (cond with 7 text tokens, uncond with 3, at
their own timesteps), T2I shape [(1, 3, 4)] and Edit shape [[(1, 3, 4), (1, 2, 3)]]; forward runs use each script's own table
and argparse defaults (0.06 / K2 / 0.2). Stored: the bf16 output bits of every call of the first generation and of every tenth
of the second, the attributes after every call (the calibration lists by length, and whole at the end of each generation),
and everything printed.
"""
import argparse
import ast
import contextlib
import io
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import qwen_image_ref as qr  # noqa: E402
from magcache_b200.config import tables  # noqa: E402

FUNCS = ("nearest_interp", "init_magcache", "init_magcache_calibration", "magcache_calibration", "magcache_forward")
SEED, STEPS, N_COND, N_UNCOND, GENERATIONS = 0, 50, 7, 3, 2


def load(path):
    tree = ast.parse(open(path).read())
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in FUNCS]
    assert sorted(n.name for n in body) == sorted(FUNCS), path
    from typing import Any, Dict, List, Optional, Tuple, Union
    ns = dict(np=np, torch=torch, F=F, Any=Any, Dict=Dict, List=List, Optional=Optional, Tuple=Tuple, Union=Union,
              USE_PEFT_BACKEND=False, Transformer2DModelOutput=qr.Output, scale_lora_layers=None, unscale_lora_layers=None)
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)
    return ns


def attrs(m, names):
    out = {}
    for n in names:
        v = getattr(m, n)
        if torch.is_tensor(v):
            v = ["tensor", int(v)]
        elif isinstance(v, list) and n in ("norm_ratio", "norm_std", "cos_dis"):  # appended to only: the length per call, the
            v = ["len", len(v)]                                                   # whole lists at the end of each generation
        elif isinstance(v, list) and not any(torch.is_tensor(x) or x is None for x in v):
            v = [float(x) for x in v]
        elif isinstance(v, list):
            v = [None if x is None else "tensor" for x in v]
        else:
            v = ["int", int(v)] if isinstance(v, int) else float(v)
        out[n] = v
    return out


def schedule(shapes):
    calls = []
    for s in range(STEPS):
        t = 1.0 - s / STEPS * 0.9
        for b, n in enumerate((N_COND, N_UNCOND)):
            calls.append(qr.call_inputs(SEED + 10 * s + b, shapes, n, t=t))
    return calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("reference", nargs="?", default="/root/reference")
    ref = ap.parse_args().reference
    scripts = {"t2i": (f"{ref}/MagCache4QwenImage/magcache_generate.py", "qwen_image", [(1, 3, 4)]),
               "edit": (f"{ref}/MagCache4QwenImageEdit/magcache_generate.py", "qwen_image_edit", [(1, 3, 4), (1, 2, 3)])}
    meta = dict(seed=SEED, steps=STEPS, n_cond=N_COND, n_uncond=N_UNCOND, generations=GENERATIONS, runs={},
                source="MagCache4QwenImage/magcache_generate.py, MagCache4QwenImageEdit/magcache_generate.py (functions executed via ast)")
    arrays = {}
    for kind, (path, table, shapes) in scripts.items():
        ns = load(path)
        for mode in ("forward", "calibration"):
            run = f"{kind}_{mode}"
            model = qr.tiny_model(SEED)
            model.__class__ = type("Golden", (model.__class__,), {})
            args = types.SimpleNamespace(sample_steps=STEPS, magcache_thresh=0.06, magcache_K=2, retention_ratio=0.2)
            if mode == "forward":
                ns["init_magcache"](model, list(tables()[table][2:]), args)
                names = ["cnt", "accumulated_err", "accumulated_steps", "accumulated_ratio", "residual_cache"]
            else:
                ns["init_magcache_calibration"](model, args)
                names = ["cnt", "norm_ratio", "norm_std", "cos_dis", "residual_cache"]
            calls, buf, att, lists = schedule(shapes), io.StringIO(), [], []
            with torch.no_grad(), contextlib.redirect_stdout(buf):
                for g in range(GENERATIONS):
                    att.append([])
                    for i, kw in enumerate(calls):
                        out = model(**kw, return_dict=False)[0]
                        if g == 0 or i % 10 == 0:
                            arrays[f"{run}_{i}" if g == 0 else f"{run}_g1_{i}"] = out.view(torch.int16).numpy()
                        att[-1].append(attrs(model, names))
                    if mode == "calibration":
                        lists.append({n: list(getattr(model, n)) for n in ("norm_ratio", "norm_std", "cos_dis")})
            meta["runs"][run] = dict(mode=mode, table=table, thresh=0.06, K=2, shapes=[list(s) for s in shapes], attrs=att, lists=lists,
                                     stdout=buf.getvalue())
    with open(os.path.join(HERE, "qwen_image.json"), "w") as f:
        json.dump(meta, f, separators=(",", ":"))
    np.savez_compressed(os.path.join(HERE, "qwen_image.npz"), **arrays)


if __name__ == "__main__":
    main()
