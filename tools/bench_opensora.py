"""Open-Sora 1.2 (STDiT3-XL/2) on the H100 kernels against the reference's own forward on the same card.

Workload: the default of OpenSoraPipeline.generate under the paper's eval settings — 480p 9:16 (480 x 854 -> a 60 x 106 latent,
30 x 53 = 1590 patches per frame), 51 frames (T = 15 latent frames), B = 2 (the CFG pair), 300 caption tokens, 30 sampling steps,
full-size seeded random weights. Prints one JSON line: miss / hit forward ms (CUDA events), seconds per 30-step video for both paper
presets from their skip schedules, spatial-attention TFLOP/s, temporal-attention GB/s and the GEMMs' share of a miss (from per-launch
events in a separate profiled call), each next to the algorithmic figure computed here from the shapes, and the same forward through
tests/opensora_ref.py in bf16 with torch SDPA (the reference's own path). The card, power limit and SM clock are read in the same run.

    python tools/bench_opensora.py [--reps 3] [--frames 15] [--teacache]

--teacache adds TeaCache's hit and miss (`teacache_opensora_forward`'s engine path: decision input + distance, one host sync, then
the residual add or the block stack), and the fused decision-input kernel (`mc_ln_t2i_modulate_rel_l1`, both samples) in µs and GB/s
against its algorithmic bytes (x0 read, prev read, cur written), next to the unfused pair: `mc_ln_modulate` mode 2 followed by a
separate distance pass (torch's `(cur - prev).abs().sum()` and `prev.abs().sum()`), against its algorithmic bytes (+ cur read back).
No TeaCache seconds per video: with random weights its data-dependent hit count says nothing about the real model.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def _smi():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def _time(fn, reps):
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return min(ts), sorted(ts)[len(ts) // 2]


def _teacache(eng, reps, ops):
    """TeaCache hit / miss ms and the decision-input kernel, fused and unfused, at the engine's staged shape."""
    B, R, D = eng.B, eng.R, eng.w.dim
    eng.prologue("hit")
    eng.modulated_input(distance=False)  # a forced call: fills previous_modulated_input
    eng.forward_teacache(True)

    def call(calc):
        eng.prologue("hit")
        eng.modulated_input(distance=True)
        eng.forward_teacache(calc)

    call(False), call(True)
    torch.cuda.synchronize()
    tmiss = _time(lambda: call(True), reps)
    thit = _time(lambda: call(False), reps)
    prev, cur = eng.mi[eng.mi_prev], eng.mi[1 - eng.mi_prev]
    em = [eng.modf[0, b].view(6, D) for b in range(B)]

    def fused():
        eng.tea_sums.zero_()
        for b in range(B):
            ops.ln_t2i_modulate_rel_l1(eng.x0[eng.rows(b)], em[b], 1, 0, prev[eng.rows(b)], cur[eng.rows(b)], eng.tea_partials, eng.tea_sums)

    def unfused():
        for b in range(B):
            ops.ln_t2i_modulate(eng.x0[eng.rows(b)], em[b], 1, 0, out=cur[eng.rows(b)])
        torch.stack([(cur - prev).abs().sum(dtype=torch.float32), prev.abs().sum(dtype=torch.float32)])

    n = 200
    out = {}
    for name, fn, nbytes in (("fused", fused, 3 * R * D * 2), ("unfused", unfused, 4 * R * D * 2)):
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        best = min(_time(lambda: [fn() for _ in range(n)], 3)) / n  # ms per call pair
        out[f"tea_input_{name}_us"] = round(best * 1e3, 1)
        out[f"tea_input_{name}_mb"] = round(nbytes / 1e6, 1)
        out[f"tea_input_{name}_gbps"] = round(nbytes / (best * 1e-3) / 1e9, 1)
    return {"tea_miss_ms_min": round(tmiss[0], 2), "tea_miss_ms_median": round(tmiss[1], 2), "tea_hit_ms_min": round(thit[0], 2),
            "tea_hit_ms_median": round(thit[1], 2), **out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=15)
    ap.add_argument("--skip-oracle", action="store_true")
    ap.add_argument("--teacache", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_opensora needs a CUDA device")
    import magcache_b200 as mc
    from magcache_b200 import ops
    import opensora_ref as R

    dev = "cuda"
    B, T, Hl, Wl, L = 2, a.frames, 60, 106, 300
    D, depth, heads = 1152, 28, 16
    S, N = (Hl // 2) * (Wl // 2), a.frames * (Hl // 2) * (Wl // 2)
    rows = B * N
    # algorithmic work of one miss forward (multiply-adds x 2)
    lin = 2 * rows * D * (3 * D + D + D + D + 4 * D + 4 * D) * 2 * depth + 2 * B * L * D * 2 * D * 2 * depth
    sp_flops = 4 * B * T * S * S * 72 * heads                   # one spatial-attention launch (QK^T + PV)
    cr_flops = 4 * rows * L * 72 * heads
    tp_flops = 4 * B * S * T * T * 72 * heads
    tp_bytes = 4 * rows * D * 2                                 # q, k, v in, out back
    model = R.STDiT3(**R.CONFIGS["full"]).init_synthetic(0).to(dev, torch.bfloat16).eval()
    eng = mc.opensora.OpenSoraEngine(mc.opensora.OpenSoraWeights.from_module(model, dev))
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(B, 4, T, Hl, Wl, device=dev, generator=g)
    y = torch.randn(B, 1, L, 4096, device=dev, generator=g)
    mask = torch.ones(B, L, dtype=torch.long, device=dev)
    ts = torch.full((B,), 800.0, device=dev)
    fps, hh, ww = torch.tensor([24.0], device=dev), torch.tensor([480.0], device=dev), torch.tensor([854.0], device=dev)
    with torch.no_grad():
        eng.stage_inputs(x, ts, y, mask, fps, hh, ww)
        eng.forward("miss")
        eng.forward("hit")
        torch.cuda.synchronize()
        miss = _time(lambda: eng.forward("miss"), a.reps)
        hit = _time(lambda: eng.forward("hit"), a.reps)
        ops.PROFILE, ops.PROFILE_TAGS = {}, None
        eng.forward("miss")
        torch.cuda.synchronize()
        prof = {k: sum(e0.elapsed_time(e1) for e0, e1 in v) for k, v in ops.PROFILE.items()}
        counts = {k: len(v) for k, v in ops.PROFILE.items()}
        ops.PROFILE = None
        total = sum(prof.values())
        sp_ms = prof.get("os_attn_spatial", 0) / max(counts.get("os_attn_spatial", 1), 1)
        tp_ms = prof.get("os_attn_temporal", 0) / max(counts.get("os_attn_temporal", 1), 1)
        res = {"workload": f"opensora-480p-9:16 B={B} T={T} S={S} rows={rows}", "gpu": _smi(),
               "miss_ms_min": round(miss[0], 2), "miss_ms_median": round(miss[1], 2), "hit_ms_min": round(hit[0], 2), "hit_ms_median": round(hit[1], 2),
               "gemm_tflop_per_miss": round(lin / 1e12, 2), "gemm_share_of_launch_time": round(prof.get("gemm_other", 0) / total, 3),
               "spatial_attn_tflop_per_launch": round(sp_flops / 1e12, 3), "spatial_attn_ms": round(sp_ms, 3),
               "spatial_attn_tflops": round(sp_flops / sp_ms / 1e9, 1) if sp_ms else None,
               "cross_attn_tflop_per_launch": round(cr_flops / 1e12, 3),
               "temporal_attn_gflop_per_launch": round(tp_flops / 1e9, 2), "temporal_attn_mb_per_launch": round(tp_bytes / 1e6, 1),
               "temporal_attn_ms": round(tp_ms, 3), "temporal_attn_gbps": round(tp_bytes / tp_ms / 1e6, 1) if tp_ms else None,
               "launch_ms_by_tag": {k: round(v, 2) for k, v in sorted(prof.items(), key=lambda kv: -kv[1])}}
        for preset in ("opensora-slow-E012K3", "opensora-fast-E024K5"):
            m = mc.PRESETS[preset].schedule()
            hits = int(m.sum())
            res[f"{preset}_hits"] = hits
            res[f"{preset}_s_per_video"] = round(((30 - hits) * miss[1] + hits * hit[1]) / 1e3, 2)
        res["no_cache_s_per_video"] = round(30 * miss[1] / 1e3, 2)
        if a.teacache:
            res.update(_teacache(eng, a.reps, ops))
        if not a.skip_oracle:
            R.install_magcache(model.__class__, thresh=0.0, K=0, skip_time=100)
            call = lambda: model(x, ts, None, y, mask=mask, fps=fps, height=hh, width=ww)  # noqa: E731
            call()
            oracle = _time(call, max(1, a.reps - 1))
            res["oracle_sdpa_miss_ms"] = round(oracle[1], 2)
            res["speedup_miss_vs_oracle"] = round(oracle[1] / miss[1], 3)
        res["gpu_after"] = _smi()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
