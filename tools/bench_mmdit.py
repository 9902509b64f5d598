"""Steps/s of the FLUX.1-dev (BASELINE configs[0] shape: 1024x1024, 28 steps, E024K5R01) and HunyuanVideo (configs[3]: 720p x 129
frames, 50 steps, E024K6R02) forwards on the MMDiT engine with synthetic device-side weights, cached vs non-cached, CUDA events.
Not the contract bench (bench.py measures the north-star Wan2.1 workload); written for the first full-size runs of these engines.

usage (GPU): python tools/bench_mmdit.py flux|hunyuan [--steps N] [--no-cache] [--tokens-scale F]
             python tools/bench_mmdit.py flux --controlnet D,S [--controlnet-repeat] [--rounds R] [--steps N]

--controlnet D,S: the FLUX 1024^2 miss forward (the whole block stack) with D double-block and S single-block synthetic bf16
ControlNet samples (S = 0: none for the single blocks) against the same forward without samples, timed in alternating rounds of N
forwards each with CUDA events; prints the card name and power limit beside the times."""
import argparse
import json
import os
import subprocess
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import magcache_b200 as mc  # noqa: E402
from magcache_b200 import mmdit, ops  # noqa: E402


def card():
    """Name and power limit of GPU 0 (read-only query): a time is only worth something next to what it was measured on."""
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    name, _, power = q.partition(",")
    return name.strip() or torch.cuda.get_device_name(0), power.strip() or "unknown"


def bench_controlnet(n_double, n_single, repeat, rounds, per_round):
    """Miss forwards at the FLUX.1-dev 1024^2 shape (4096 image + 512 text tokens), without and with ControlNet samples,
    alternating; the two outputs differ only through the samples."""
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    eng = mmdit.FluxEngine(mmdit.random_flux_weights(dev))
    n_img, n_txt, D = 4096, 512, eng.w.dim
    img_ids = torch.zeros(n_img, 3, device=dev)
    img_ids[:, 1], img_ids[:, 2] = torch.arange(n_img, device=dev) // 64, torch.arange(n_img, device=dev) % 64
    eng.stage_inputs(torch.randn(1, n_img, 64, device=dev, generator=g).bfloat16(), torch.randn(1, n_txt, 4096, device=dev, generator=g).bfloat16(),
                     torch.randn(1, 768, device=dev, generator=g).bfloat16(), torch.tensor([0.6], device=dev), torch.tensor([3.5], device=dev),
                     img_ids, torch.zeros(n_txt, 3, device=dev))

    def samples(n):
        return [(0.05 * torch.randn(1, n_img, D, device=dev, generator=g)).bfloat16() for _ in range(n)] if n else None

    ctrl = (samples(n_double), samples(n_single), repeat)
    modes = {"plain": (None, None, False), "controlnet": ctrl}
    times = {k: [] for k in modes}
    for k, c in modes.items():  # warm-up: every shape and both epilogue paths
        eng.stage_controlnet(*c)
        eng.forward("miss")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for k, c in modes.items():
            eng.stage_controlnet(*c)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(per_round):
                eng.forward("miss")
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / per_round)
    n_reads = sum(x is not None for part in eng._controlnet_views() or () for x in part)
    name, power = card()
    med = {k: statistics.median(v) for k, v in times.items()}
    print(json.dumps({"family": "flux", "workload": "1024x1024 miss forward", "controlnet": [n_double, n_single], "controlnet_blocks_repeat": repeat,
                      "ms_plain": round(med["plain"], 3), "ms_controlnet": round(med["controlnet"], 3),
                      "ms_added": round(med["controlnet"] - med["plain"], 3),
                      "spread_ms": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
                      "sample_reads_per_forward": n_reads, "sample_bytes_per_forward": n_reads * n_img * D * 2,
                      "rounds": rounds, "forwards_per_round": per_round, "gpu": name, "power_limit": power}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("family", choices=["flux", "hunyuan"])
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--no-cache", action="store_true")
    ap.add_argument("--frames", type=int, default=33, help="hunyuan: latent frames (33 = 129 video frames)")
    ap.add_argument("--controlnet", default=None, help="flux: D,S double / single ControlNet samples; times the miss forward with and without")
    ap.add_argument("--controlnet-repeat", action="store_true", help="controlnet_blocks_repeat (XLabs): double block i reads sample i %% D")
    ap.add_argument("--rounds", type=int, default=5, help="--controlnet: alternating rounds")
    args = ap.parse_args()
    if args.controlnet is not None:
        if args.family != "flux":
            ap.error("--controlnet is a FLUX option")
        n_double, n_single = (int(v) for v in args.controlnet.split(","))
        bench_controlnet(n_double, n_single, args.controlnet_repeat, args.rounds, args.steps or 10)
        return
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    if args.family == "flux":
        steps = args.steps or 28
        model = mmdit.MMDiTHandle(mmdit.FluxEngine(mmdit.random_flux_weights(dev)))
        mc.init_magcache_flux(model, steps, thresh=1e-9 if args.no_cache else 0.24, K=5, retention_ratio=0.1)
        n_img, n_txt = 4096, 512
        hs = torch.randn(1, n_img, 64, device=dev, generator=g).bfloat16()
        enc = torch.randn(1, n_txt, 4096, device=dev, generator=g).bfloat16()
        pooled = torch.randn(1, 768, device=dev, generator=g).bfloat16()
        img_ids = torch.zeros(n_img, 3, device=dev)
        img_ids[:, 1], img_ids[:, 2] = torch.arange(n_img, device=dev) // 64, torch.arange(n_img, device=dev) % 64
        txt_ids = torch.zeros(n_txt, 3, device=dev)
        gd = torch.tensor([3.5], device=dev)

        def step(i):
            return model(hs, enc, pooled, torch.tensor([1.0 - i / steps], device=dev), img_ids, txt_ids, gd, return_dict=False)[0]
    else:
        steps = args.steps or 50
        model = mmdit.MMDiTHandle(mmdit.HunyuanEngine(mmdit.random_hunyuan_weights(dev)))
        mc.init_magcache_hunyuan(model, steps, thresh=1e-9 if args.no_cache else 0.24, K=6, retention_ratio=0.2)
        grid = (args.frames, 45, 80)  # 720 x 1280 -> 90 x 160 latent -> 45 x 80 patches
        n_img = grid[0] * grid[1] * grid[2]
        x = torch.randn(1, 16, grid[0], 2 * grid[1], 2 * grid[2], device=dev, generator=g).bfloat16()
        txt = torch.randn(1, 256, 4096, device=dev, generator=g).bfloat16()
        mask = torch.zeros(1, 256, dtype=torch.long, device=dev)
        mask[0, :48] = 1
        pooled = torch.randn(1, 768, device=dev, generator=g).bfloat16()
        ang = torch.rand(n_img, 64, device=dev, generator=g) * 6.28
        cos, sin = ang.cos().repeat_interleave(2, dim=1), ang.sin().repeat_interleave(2, dim=1)
        gd = torch.tensor([6000.0], device=dev)

        def step(i):
            return model(x, torch.tensor([1000.0 * (1 - i / steps)], device=dev), txt, mask, pooled, cos, sin, gd, return_dict=False)

    for i in range(3):  # warm-up inside the retention window, then restart the schedule
        step(i)
    mc.reset_magcache(model)
    n0 = ops.LAUNCHES
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(steps):
        step(i)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    print(json.dumps({"family": args.family, "steps": steps, "cached": not args.no_cache, "steps_per_s": steps / (ms / 1e3), "sec_per_sample": ms / 1e3,
                      "image_tokens": n_img, "gpu_launches": ops.LAUNCHES - n0}))


if __name__ == "__main__":
    main()
