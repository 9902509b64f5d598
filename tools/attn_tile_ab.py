"""Self-attention at the benchmarked shape (32760 x 32760 keys, 12 heads of 128) with 128-key and with 176-key KV tiles, alternated
in one process over several rounds (MC_ATTN_KERNEL = 2 / 3), while nvidia-smi samples SM clock and board power. Prints one JSON
line: per width and round ms per launch, TFLOP/s, SM clock, power and J per launch, the card's name and power limit, and the
rel-L2 between the two widths' outputs.   python tools/attn_tile_ab.py [--rounds 5] [--seconds 3]"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magcache_b200 import ops  # noqa: E402

N, D, H = 32760, 1536, 12
FLOPS = 4.0 * N * N * D
WIDTHS = {128: "2", 176: "3"}  # KV tile width -> MC_ATTN_KERNEL


def smi(query):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    return [f.strip() for f in r.stdout.strip().split(",")]


def sample(stop, rows):
    while not stop.is_set():
        try:
            rows.append(tuple(float(f) for f in smi("clocks.sm,power.draw")[:2]))
        except ValueError:
            pass
        time.sleep(0.1)


def timed(fn, secs):
    """Launches fn in batches of 10 for `secs` seconds; CUDA events around the whole loop, nvidia-smi sampling alongside."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    stop, rows = threading.Event(), []
    th = threading.Thread(target=sample, args=(stop, rows))
    th.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n, t0 = 0, time.time()
    e0.record()
    while time.time() - t0 < secs:
        for _ in range(10):
            fn()
        n += 10
        torch.cuda.synchronize()
    e1.record()
    torch.cuda.synchronize()
    stop.set()
    th.join()
    ms = e0.elapsed_time(e1) / n
    rows = rows[len(rows) // 3:]  # the settled part
    med = lambda xs: sorted(xs)[len(xs) // 2] if xs else float("nan")  # noqa: E731
    clk, pw = med([r[0] for r in rows]), med([r[1] for r in rows])
    return {"ms": round(ms, 4), "tflops": round(FLOPS / ms / 1e9, 1), "sm_mhz": clk, "power_w": pw, "j_per_launch": round(ms * pw / 1e3, 3),
            "launches": n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=3.0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "attn_tile_ab.py times the H100 kernels: it needs a CUDA device"
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(N, 3 * D, device="cuda", generator=g).bfloat16()
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]  # column slices of one fused buffer, as the engine launches them
    out = torch.empty(N, D, device="cuda", dtype=torch.bfloat16)
    name, limit = smi("name,power.limit")[:2]
    saved = os.environ.get("MC_ATTN_KERNEL")
    outs = {}
    for w, sel in WIDTHS.items():
        os.environ["MC_ATTN_KERNEL"] = sel
        outs[w] = ops.attention(q, k, v, H).float()
    rel_l2 = float((outs[176] - outs[128]).norm() / outs[128].norm())
    del outs
    rounds = {w: [] for w in WIDTHS}
    for r in range(args.rounds):
        order = list(WIDTHS) if r % 2 == 0 else list(WIDTHS)[::-1]  # alternate which width runs first
        for w in order:
            os.environ["MC_ATTN_KERNEL"] = WIDTHS[w]
            rounds[w].append(timed(lambda: ops.attention(q, k, v, H, out=out), args.seconds))
    if saved is None:
        os.environ.pop("MC_ATTN_KERNEL", None)
    else:
        os.environ["MC_ATTN_KERNEL"] = saved
    ms = {w: [x["ms"] for x in rounds[w]] for w in WIDTHS}
    per_round = [a / b for a, b in zip(ms[176], ms[128])]
    line = {"shape": f"Lq=Lk={N} heads={H} head_dim=128", "gpu": name, "power_limit_w": float(limit), "tflop_per_launch": round(FLOPS / 1e12, 3),
            "rounds": {str(w): rounds[w] for w in WIDTHS},
            "ms_range": {str(w): [min(ms[w]), max(ms[w])] for w in WIDTHS},
            "ratio_176_over_128_per_round": [round(x, 4) for x in per_round],
            "faster_in_every_round": all(x < 1.0 for x in per_round),
            "separated": max(ms[176]) < min(ms[128]),
            "rel_l2_176_vs_128": rel_l2}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
