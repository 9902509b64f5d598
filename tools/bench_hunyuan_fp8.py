"""HunyuanVideo FP8-weight checkpoints on the MMDiT engine against bf16: one random full-width model (`random_hunyuan_weights`, 20 double
+ 40 single blocks, D = 3072) quantised like an FP8 checkpoint (tests/hunyuan_fp8_ref.py: scale = bf16(amax / 448) per block Linear,
codes float8_e4m3fn). The bf16 engine runs on the dequantised weights bf16(q * scale) — the model the checkpoint stands for — so
the two engines must agree bit for bit.

Reports, per format: the resident weight bytes the engine reads (block weights separately), the peak allocated memory of building
the engine plus one miss and one hit forward with only that format's weights counted, the miss and hit forward times (CUDA events;
the formats alternated, several repeats), and whether the outputs are bitwise equal. The card's name and power limit are read in the
same run. One JSON line.

usage (GPU): python tools/bench_hunyuan_fp8.py [--frames 33] [--repeats 5]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from hunyuan_fp8_ref import fp8_quantize  # noqa: E402
from magcache_b200 import mmdit  # noqa: E402


def quantise(w16):
    """FP8 weights of the random bf16 weights `w16`, Linear by Linear (a fused q|k|v or linear1 matrix is ONE Linear upstream, so its
    row blocks share a scale). `w16`'s block weights are overwritten with the dequantised values. Non-block weights are shared."""
    D, dev = w16.dim, w16.device
    w8 = mmdit.HunyuanWeights()
    w8.__dict__.update({k: v for k, v in w16.__dict__.items() if k not in ("double", "single", "ada_w")})
    w8.double, w8.single = [dict(b) for b in w16.double], [dict(b) for b in w16.single]

    def linear(parts):  # parts: row blocks of one Linear, bf16 views
        q, s = fp8_quantize(torch.cat(parts, 0))
        scale = s.reshape(1).expand(q.shape[0]).contiguous()
        out, r0 = [], 0
        for p in parts:
            r1 = r0 + p.shape[0]
            p.copy_(q[r0:r1].to(torch.bfloat16) * s)  # fp8_activation_dequant
            out.append(mmdit.Fp8Weight(q[r0:r1], scale[r0:r1]))
            r0 = r1
        return out

    for b8 in w8.double:
        for k in ("", "c"):
            b8[f"{k}qk_w"], b8[f"{k}v_w"] = linear([b8[f"{k}qk_w"], b8[f"{k}v_w"]])
            for n in ("o_w", "ff1_w", "ff2_w"):
                (b8[k + n],) = linear([b8[k + n]])
    for b8 in w8.single:
        b8["qk_w"], b8["v_w"], b8["mlp_w"] = linear([b8["qk_w"], b8["v_w"], b8["mlp_w"]])
        (b8["out_w"],) = linear([b8["out_w"]])
    q = torch.empty(w16.ada_out, D, dtype=torch.float8_e4m3fn, device=dev)
    scale = torch.empty(w16.ada_out, dtype=torch.bfloat16, device=dev)
    starts = sorted([b["ada"] for b in w16.double] + [b["ada_c"] for b in w16.double] + [b["ada"] for b in w16.single] + [w16.ada_out])
    for r0, r1 in zip(starts[:-1], starts[1:]):  # one ModulateDiT Linear per range
        (f,) = linear([w16.ada_w[r0:r1]])
        q[r0:r1], scale[r0:r1] = f.q, f.scale
    w8.ada_parts = [(0, mmdit.Fp8Weight(q, scale)), (w16.ada_out, w16.ada_w[w16.ada_out:].clone())]
    w8.fp8_scratch = mmdit._fp8_scratch(w8, dev)
    return w8


def storages(w):
    """{storage address: bytes} of every device tensor the weights hold, and the same for the block weights alone."""
    seen, block = {}, {}

    def add(t, dst):
        if isinstance(t, mmdit.Fp8Weight):
            add(t.q, dst), add(t.scale, dst)
        elif torch.is_tensor(t):
            st = t.untyped_storage()
            dst[st.data_ptr()] = st.nbytes()
        elif isinstance(t, (list, tuple)):
            for x in t:
                add(x, dst)
        elif isinstance(t, dict):
            for x in t.values():
                add(x, dst)

    for k, v in w.__dict__.items():
        add(v, seen)
    for b in w.double + w.single:
        add({k: v for k, v in b.items() if k.endswith("_w")}, block)
    if w.ada_parts is not None:
        add(w.ada_parts[0][1], block)
    else:
        add(w.ada_w[:w.ada_out], block)  # the whole stack's storage: its final-layer rows are 2 of ~362 D rows
    return seen, block


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=33, help="latent frames (33 = 129 video frames at 720p)")
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_hunyuan_fp8: needs a CUDA device")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    w16 = mmdit.random_hunyuan_weights(dev)
    w8 = quantise(w16)
    torch.cuda.synchronize()
    s16, b16 = storages(w16)
    s8, b8 = storages(w8)
    shared = sum(n for p, n in s16.items() if p in s8)
    own = {"bf16": sum(s16.values()) - shared, "fp8": sum(s8.values()) - shared}

    g = torch.Generator(device=dev).manual_seed(0)
    grid = (args.frames, 45, 80)  # 720 x 1280 -> 90 x 160 latent -> 45 x 80 patches
    n_img = grid[0] * grid[1] * grid[2]
    x = torch.randn(1, 16, grid[0], 2 * grid[1], 2 * grid[2], device=dev, generator=g).bfloat16()
    txt = torch.randn(1, 256, 4096, device=dev, generator=g).bfloat16()
    mask = torch.zeros(1, 256, dtype=torch.long, device=dev)
    mask[0, :48] = 1
    pooled = torch.randn(1, 768, device=dev, generator=g).bfloat16()
    ang = torch.rand(n_img, 64, device=dev, generator=g) * 6.28
    cos, sin = ang.cos().repeat_interleave(2, dim=1), ang.sin().repeat_interleave(2, dim=1)
    t, gd = torch.tensor([870.0], device=dev), torch.tensor([6000.0], device=dev)
    weights = {"bf16": w16, "fp8": w8}

    def engine(fmt):
        e = mmdit.HunyuanEngine(weights[fmt])
        e.stage_inputs(x, t, txt, mask, pooled, cos, sin, gd)
        return e

    # memory: one format's engine at a time; the other format's own weights are subtracted from the peak
    peak, outs = {}, {}
    for fmt in ("fp8", "bf16"):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        e = engine(fmt)
        miss = e.forward("miss").clone()
        hit = e.forward("hit").clone()
        torch.cuda.synchronize()
        peak[fmt] = torch.cuda.max_memory_allocated() - own["bf16" if fmt == "fp8" else "fp8"]
        outs[fmt] = (miss, hit)
        del e
    equal = {k: bool(torch.equal(outs["fp8"][i], outs["bf16"][i])) for i, k in enumerate(("miss", "hit"))}

    engines = {fmt: engine(fmt) for fmt in ("bf16", "fp8")}
    times = {fmt: {"miss": [], "hit": []} for fmt in engines}
    for r in range(args.repeats + 1):  # repeat 0 warms up
        for fmt in (("bf16", "fp8") if r % 2 == 0 else ("fp8", "bf16")):
            for kind in ("miss", "hit"):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                engines[fmt].forward(kind)
                e1.record()
                torch.cuda.synchronize()
                if r:
                    times[fmt][kind].append(round(e0.elapsed_time(e1), 3))
    gib = 2 ** 30
    print(json.dumps({
        "gpu": smi, "frames": args.frames, "image_tokens": n_img, "text_tokens": 48, "repeats": args.repeats,
        "outputs_bitwise_equal": equal,
        "formats": {fmt: {"weight_gib": round(sum((s16 if fmt == "bf16" else s8).values()) / gib, 3),
                          "block_weight_gib": round(sum((b16 if fmt == "bf16" else b8).values()) / gib, 3),
                          "peak_allocated_gib": round(peak[fmt] / gib, 3),
                          "miss_ms": times[fmt]["miss"], "hit_ms": times[fmt]["hit"]} for fmt in ("bf16", "fp8")},
        "fp8_scratch_mib": round(w8.fp8_scratch.numel() * 2 / 2 ** 20, 1),
    }))


if __name__ == "__main__":
    main()
