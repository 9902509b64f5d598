#!/usr/bin/env python
"""Generate tests/golden/opensora_long.npz and opensora_long.json by EXECUTING the reference's own Open-Sora code at T > 32.

Run where the reference tree is present (it is not imported by anything else):

    python tests/golden/make_opensora_long_golden.py

The reference's STDiT3 and `magcache_forward` are loaded and set up by make_opensora_golden.py (`_namespace`, `build_reference`:
the same sources executed unmodified, the same stand-ins, the same tiny config and synthetic weights, the `eval_ours` attributes
0.12 / K3 / skip_time 6). This script only changes the video: B = 2 samples with distinct timesteps, 4 x 4 latents (S = 4 tokens
per frame) and T = 40 or T = 70 latent frames, the lengths past the 32 frames the first temporal kernel serves; 70 frames also
cross a 64-key tile of the tensor-core kernel. Over 10 calls of one video (misses, then the hits from call 6 on) in fp32 and in bf16
it records the controller attributes after every call and the outputs of five calls (`STORED`). So the fixture pins the temporal RoPE at positions
past 32 and the temporal attention at long T to the reference's statements.
"""
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_opensora_golden as G  # noqa: E402

B, H, W = 2, 4, 4
FRAMES = (40, 70)
CALLS = 10
STORED = (0, 5, 6, 8, 9)  # outputs kept: the first miss, the last miss before the hits, the first and last hit, the miss after them
ATTRS = G.ATTRS


def inputs(T):
    g = torch.Generator().manual_seed(T)
    x = torch.randn(B, 4, T, H, W, generator=g)
    y = torch.randn(B, 1, G.CFG["model_max_length"], G.CFG["caption_channels"], generator=g)
    mask = torch.ones(B, G.CFG["model_max_length"], dtype=torch.long)
    kw = dict(mask=mask, fps=torch.tensor([24.0]), height=torch.tensor([8.0 * H]), width=torch.tensor([8.0 * W]))
    return x, y, kw


def run(model, T):
    x, y, kw = inputs(T)
    outs, attrs = [], []
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()) as log:
        for i in range(CALLS):
            out = model(x, G.timesteps(i), None, y, **kw).numpy()
            if i in STORED:
                outs.append(out)
            attrs.append({a: float(getattr(model, a)) for a in ATTRS})
    return np.stack(outs), attrs, G.skip_mask(log.getvalue(), CALLS)


def main():
    ns = G._namespace()
    doc = {"config": G.CFG, "B": B, "H": H, "W": W, "frames": list(FRAMES), "calls": CALLS, "stored": list(STORED), "seed": G.SEED,
           "input_seed": "T", "timesteps": [G.timesteps(i).tolist() for i in range(CALLS)]}
    arrays = {}
    for T in FRAMES:
        for name, dtype in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
            model, _ = G.build_reference(ns, dtype)
            out, attrs, mask = run(model, T)
            if name == "fp32":
                arrays[f"T{T}_{name}"] = out.astype(np.float32)
            else:  # the fp32 output of the bf16 model holds bf16 values: stored as their bit patterns, half the bytes
                bits = torch.from_numpy(out).to(torch.bfloat16)
                assert np.array_equal(bits.float().numpy(), out)
                arrays[f"T{T}_{name}"] = bits.view(torch.int16).numpy()
            doc[f"T{T}_attrs_{name}"] = attrs
            doc[f"T{T}_mask_{name}"] = mask
    np.savez_compressed(os.path.join(HERE, "opensora_long.npz"), **arrays)
    with open(os.path.join(HERE, "opensora_long.json"), "w") as f:
        json.dump(doc, f, indent=1)
    print({k: v for k, v in doc.items() if "_mask_" in k})


if __name__ == "__main__":
    main()
