"""Per-step time of Open-Sora's sampler with the step's tail fused into the final layer, against the engine's forward followed by the
reference's statements (scheduling_rflow_open_sora.py:244-251), for a cache-hit step and a miss step.

Workload: 480p 9:16 x 51 frames (a 15 x 60 x 107 latent, 15 x 30 x 54 patches), one prompt (B = 2 with its CFG pair), 300 caption
tokens, full-size seeded random weights (STDiT3-XL/2 shapes), the engine driven directly. One step is
  fused:   OpenSoraEngine.arm_step + forward(kind)                                     (mc_opensora_head in step mode)
  unfused: forward(kind) -> output.chunk(2, 1)[0].chunk(2, 0), uncond + g (cond - uncond), z + v_pred dt   (torch, fp32)
timed with CUDA events around each step, the two forms alternating, after a warm-up of both. The two final layers alone (the fused
kernel against OpenSoraEngine.head + the torch tail) are timed the same way over many launches. Both forms' latents are compared
bit for bit. The card, power limit and SM clocks are read in the same run. Prints one JSON line and writes it to --out.

    python tools/bench_opensora_sampler.py [--miss-reps 6] [--hit-reps 40] [--out results/bench_opensora_sampler.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _smi():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def _timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--miss-reps", type=int, default=6)
    ap.add_argument("--hit-reps", type=int, default=40)
    ap.add_argument("--head-reps", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_opensora_sampler: needs a CUDA device")
    from magcache_b200.opensora import OpenSoraEngine, random_opensora_weights
    dev = torch.device("cuda")
    torch.manual_seed(0)
    eng = OpenSoraEngine(random_opensora_weights(dev))
    B, Tx, Hx, Wx, g = 2, 15, 60, 107, 7.0
    z0 = torch.randn(B // 2, 4, Tx, Hx, Wx, device=dev)
    y = torch.randn(B, 1, 300, 4096, device=dev)
    cap = torch.zeros(B, 300, dtype=torch.long, device=dev)
    cap[:, :37] = 1
    f = dict(device=dev)
    eng.stage_inputs(torch.cat([z0, z0]), torch.tensor([700.0, 700.0], **f), y, cap, torch.tensor([24.0], **f),
                     torch.tensor([480.0], **f), torch.tensor([854.0], **f))
    dt = torch.tensor([0.0331], **f)

    def unfused(kind, z):
        output = eng.forward(kind)
        pred = output.chunk(2, dim=1)[0]
        pred_cond, pred_uncond = pred.chunk(2, dim=0)
        v_pred = pred_uncond + g * (pred_cond - pred_uncond)
        return z + v_pred * dt[:, None, None, None, None]

    def fused(kind, z):
        out = torch.empty_like(z)
        eng.arm_step(z, g, dt, out)
        return eng.forward(kind)

    res = {"card": _smi(), "workload": "480p x 51 frames, latent 15 x 60 x 107, B = 2 (one prompt + CFG), 300 caption tokens"}
    eng.forward("miss")  # fills the residual cache, warms every kernel
    with torch.no_grad():
        for kind, reps in (("miss", a.miss_reps), ("hit", a.hit_reps)):
            for fn in (fused, unfused):
                fn(kind, z0)
            times = {"fused": [], "unfused": []}
            for _ in range(reps):
                for name, fn in (("fused", fused), ("unfused", unfused)):
                    ms, _ = _timed(lambda: fn(kind, z0))
                    times[name].append(ms)
            zf, zu = fused(kind, z0), unfused(kind, z0)
            res[f"{kind}_bit_equal"] = bool(torch.equal(zf, zu))
            for name in times:
                res[f"{kind}_{name}_ms_median"] = round(statistics.median(times[name]), 4)
                res[f"{kind}_{name}_ms_min"] = round(min(times[name]), 4)
            res[f"{kind}_saved_ms_median"] = round(res[f"{kind}_unfused_ms_median"] - res[f"{kind}_fused_ms_median"], 4)
        # the final layers alone: head (+ hit add) + torch tail against one mc_opensora_head, many launches per timing
        from magcache_b200 import ops
        w, D = eng.w, eng.w.dim
        mod = eng.finf.view(B, 2, D)
        out = torch.empty_like(z0)
        for hit in (False, True):
            x = eng.x0 if hit else eng.x

            def tail_unfused():
                for _ in range(a.head_reps):
                    xx = ops.cache_hit_add(eng.x0, eng.res, out=eng.hit) if hit else x
                    pred = eng.head(xx).chunk(2, dim=1)[0]
                    c, u = pred.chunk(2, dim=0)
                    z0 + (u + g * (c - u)) * dt[:, None, None, None, None]

            def tail_fused():
                for _ in range(a.head_reps):
                    ops.opensora_head(x, mod, w.fin_w, w.fin_b, (eng.T, eng.H, eng.W), eng.crop, res=eng.res if hit else None,
                                      step=(z0, g, dt), out=out)
            key = "hit" if hit else "miss"
            for fn in (tail_fused, tail_unfused):
                fn()
            tf, tu = [], []
            for _ in range(5):
                tf.append(_timed(tail_fused)[0] * 1e3 / a.head_reps)
                tu.append(_timed(tail_unfused)[0] * 1e3 / a.head_reps)
            res[f"final_layer_{key}_fused_us_median"] = round(statistics.median(tf), 2)
            res[f"final_layer_{key}_unfused_us_median"] = round(statistics.median(tu), 2)
    rows = B * Tx * 30 * 54
    res["fused_kernel_algorithmic_bytes_miss"] = rows * D * 2 + (B // 2) * 4 * Tx * Hx * Wx * 8
    res["fused_kernel_algorithmic_bytes_hit"] = rows * D * 4 + (B // 2) * 4 * Tx * Hx * Wx * 8
    res["card_after"] = _smi()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
