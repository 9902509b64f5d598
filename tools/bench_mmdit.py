"""Steps/s of the FLUX.1-dev (BASELINE configs[0] shape: 1024x1024, 28 steps, E024K5R01) and HunyuanVideo (configs[3]: 720p x 129
frames, 50 steps, E024K6R02) forwards on the MMDiT engine with synthetic device-side weights, cached vs non-cached, CUDA events.
Not the contract bench (bench.py measures the north-star Wan2.1 workload); written for the first full-size runs of these engines.

usage (GPU): python tools/bench_mmdit.py flux|hunyuan [--steps N] [--no-cache] [--tokens-scale F]
             python tools/bench_mmdit.py flux --controlnet D,S [--controlnet-repeat] [--rounds R] [--steps N]
             python tools/bench_mmdit.py flux --lora RANK [--rounds R] [--steps N]
             python tools/bench_mmdit.py flux --ip-adapter A[,T] [--rounds R] [--steps N]
             python tools/bench_mmdit.py qwen-image [--edit] [--rounds R] [--steps N]
             python tools/bench_mmdit.py qwen-image [--edit] --lora RANK [--rounds R] [--steps N]

--controlnet D,S: the FLUX 1024^2 miss forward (the whole block stack) with D double-block and S single-block synthetic bf16
ControlNet samples (S = 0: none for the single blocks) against the same forward without samples, timed in alternating rounds of N
forwards each with CUDA events; prints the card name and power limit beside the times.

--lora RANK: the FLUX 1024^2 miss and hit forwards with one synthetic rank-RANK LoRA adapter on every covered target (every block
Linear, every AdaLayerNorm projection, x_embedder, context_embedder, proj_out; magcache_b200/lora.py) against the same forwards
without adapters, alternating rounds as for --controlnet.

--ip-adapter A[,T]: the FLUX 1024^2 miss and hit forwards with A synthetic XLabs-shaped IP-Adapters (768-wide image embeds projected
to T tokens of 4096, default T = 16; `to_k_ip` / `to_v_ip` on all 19 double blocks) against the same forwards without them,
alternating rounds as for --controlnet; then `mc_ip_attn` alone at 4096 rows with its bytes per launch and rate.

qwen-image: Qwen-Image (60 blocks, 3072 wide, synthetic weights) at 1328^2 (6889 image tokens; --edit: Qwen-Image-Edit's 1024^2
noised latents plus a 1024^2 reference image, 8192 tokens) with a 200-token cond and a 6-token uncond prompt: cond miss, uncond
miss and hit medians (CUDA events, alternating rounds of N forwards), peak memory, and the 50-step transformer time of the
qwen-image-E006K2R02 schedule from those medians.

qwen-image --lora RANK: the cond (200-token) miss and hit forwards with one synthetic rank-RANK adapter on every covered target
(every block attention and MLP Linear, img_mod.1 / txt_mod.1, img_in, txt_in, norm_out.linear, proj_out; lora.QWEN) against the
same forwards without adapters, alternating rounds as for --controlnet; then the miss's down-projections alone (one plain GEMM per
distinct adapted input, N = the padded rank), so the added miss time splits into down-projections and tails."""
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


def _flux_1024_engine():
    """A FLUX.1-dev engine on synthetic weights, staged at 1024^2 (4096 image + 512 text tokens)."""
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    eng = mmdit.FluxEngine(mmdit.random_flux_weights(dev))
    n_img, n_txt, D = 4096, 512, eng.w.dim
    img_ids = torch.zeros(n_img, 3, device=dev)
    img_ids[:, 1], img_ids[:, 2] = torch.arange(n_img, device=dev) // 64, torch.arange(n_img, device=dev) % 64
    eng.stage_inputs(torch.randn(1, n_img, 64, device=dev, generator=g).bfloat16(), torch.randn(1, n_txt, 4096, device=dev, generator=g).bfloat16(),
                     torch.randn(1, 768, device=dev, generator=g).bfloat16(), torch.tensor([0.6], device=dev), torch.tensor([3.5], device=dev),
                     img_ids, torch.zeros(n_txt, 3, device=dev))
    return eng, g, n_img, D


def _alternate(eng, modes, kinds, rounds, per_round):
    """Median / spread of the forward time (ms) of each (mode, kind), modes set by `modes[k]()`, alternating rounds."""
    times = {(k, kind): [] for k in modes for kind in kinds}
    for k, set_mode in modes.items():  # warm-up: every shape and every epilogue path
        set_mode()
        for kind in ("miss",) + tuple(kinds):
            eng.forward(kind)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for k, set_mode in modes.items():
            set_mode()
            for kind in kinds:
                torch.cuda.synchronize()
                e0.record()
                for _ in range(per_round):
                    eng.forward(kind)
                e1.record()
                torch.cuda.synchronize()
                times[(k, kind)].append(e0.elapsed_time(e1) / per_round)
    return times


def bench_controlnet(n_double, n_single, repeat, rounds, per_round):
    """Miss forwards at the FLUX.1-dev 1024^2 shape (4096 image + 512 text tokens), without and with ControlNet samples,
    alternating; the two outputs differ only through the samples."""
    eng, g, n_img, D = _flux_1024_engine()
    dev = eng.device

    def samples(n):
        return [(0.05 * torch.randn(1, n_img, D, device=dev, generator=g)).bfloat16() for _ in range(n)] if n else None

    ctrl = (samples(n_double), samples(n_single), repeat)
    modes = {"plain": lambda: eng.stage_controlnet(None, None, False), "controlnet": lambda: eng.stage_controlnet(*ctrl)}
    times = {k: v for (k, _), v in _alternate(eng, modes, ("miss",), rounds, per_round).items()}
    n_reads = sum(x is not None for part in eng._controlnet_views() or () for x in part)
    name, power = card()
    med = {k: statistics.median(v) for k, v in times.items()}
    print(json.dumps({"family": "flux", "workload": "1024x1024 miss forward", "controlnet": [n_double, n_single], "controlnet_blocks_repeat": repeat,
                      "ms_plain": round(med["plain"], 3), "ms_controlnet": round(med["controlnet"], 3),
                      "ms_added": round(med["controlnet"] - med["plain"], 3),
                      "spread_ms": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
                      "sample_reads_per_forward": n_reads, "sample_bytes_per_forward": n_reads * n_img * D * 2,
                      "rounds": rounds, "forwards_per_round": per_round, "gpu": name, "power_limit": power}))


def bench_lora(rank, rounds, per_round):
    """Miss and hit forwards at the FLUX.1-dev 1024^2 shape without adapters and with one rank-`rank` adapter (scaling 1) on every
    covered target, alternating."""
    from magcache_b200.lora import LoraPack
    eng, g, n_img, D = _flux_1024_engine()
    w, dev = eng.w, eng.device

    def ad(n_out, n_in):
        A = (torch.randn(rank, n_in, device=dev, generator=g) / n_in ** 0.5).bfloat16()
        return [(A, (0.02 * torch.randn(n_out, rank, device=dev, generator=g)).bfloat16(), 1.0)]

    spec = {}
    for i in range(len(w.double)):
        for t, (o, k) in {"attn.to_q": (D, D), "attn.to_k": (D, D), "attn.to_v": (D, D), "attn.to_out.0": (D, D), "attn.add_q_proj": (D, D),
                          "attn.add_k_proj": (D, D), "attn.add_v_proj": (D, D), "attn.to_add_out": (D, D), "ff.net.0.proj": (4 * D, D),
                          "ff.net.2": (D, 4 * D), "ff_context.net.0.proj": (4 * D, D), "ff_context.net.2": (D, 4 * D),
                          "norm1.linear": (6 * D, D), "norm1_context.linear": (6 * D, D)}.items():
            spec[("double", i, t)] = ad(o, k)
    for i in range(len(w.single)):
        for t, (o, k) in {"attn.to_q": (D, D), "attn.to_k": (D, D), "attn.to_v": (D, D), "proj_mlp": (4 * D, D), "proj_out": (D, 5 * D),
                          "norm.linear": (3 * D, D)}.items():
            spec[("single", i, t)] = ad(o, k)
    for t, (o, k) in {"x_embedder": (D, w.in_channels), "context_embedder": (D, w.joint_dim), "proj_out": (w.in_channels, D),
                      "norm_out.linear": (2 * D, D)}.items():
        spec[("top", 0, t)] = ad(o, k)
    pack = LoraPack(w, spec)

    def set_lora(p):
        eng.lora = p

    times = _alternate(eng, {"plain": lambda: set_lora(None), "lora": lambda: set_lora(pack)}, ("miss", "hit"), rounds, per_round)
    name, power = card()
    med = {f"ms_{k}_{kind}": round(statistics.median(v), 3) for (k, kind), v in times.items()}
    print(json.dumps({"family": "flux", "workload": "1024x1024 forward", "lora_rank": rank, "lora_targets": len(spec), **med,
                      "ms_added_miss": round(med["ms_lora_miss"] - med["ms_plain_miss"], 3),
                      "ms_added_hit": round(med["ms_lora_hit"] - med["ms_plain_hit"], 3),
                      "spread_ms": {f"{k}_{kind}": [round(min(v), 3), round(max(v), 3)] for (k, kind), v in times.items()},
                      "rounds": rounds, "forwards_per_round": per_round, "gpu": name, "power_limit": power}))


class FluxIPAdapterAttnProcessor(torch.nn.Module):
    """diffusers' processor surface the engine reads (its class name, `to_k_ip`, `to_v_ip`, `scale`)."""

    def __init__(self, D, C, n, dev):
        super().__init__()
        kw = dict(device=dev, dtype=torch.bfloat16)
        self.to_k_ip = torch.nn.ModuleList([torch.nn.Linear(C, D, **kw) for _ in range(n)])
        self.to_v_ip = torch.nn.ModuleList([torch.nn.Linear(C, D, **kw) for _ in range(n)])
        self.scale = [1.0] * n


def bench_ip_adapter(n_adapters, T, rounds, per_round):
    """Miss and hit forwards at the FLUX.1-dev 1024^2 shape without and with `n_adapters` IP-Adapters of T tokens, alternating;
    then the kernel alone."""
    import types
    eng, g, n_img, D = _flux_1024_engine()
    dev, C, emb = eng.device, 4096, 768
    kw = dict(device=dev, dtype=torch.bfloat16)
    with torch.no_grad():
        layers = torch.nn.ModuleList()
        for _ in range(n_adapters):
            layer = torch.nn.Module()
            layer.image_embeds, layer.norm, layer.num_image_text_embeds = torch.nn.Linear(emb, T * C, **kw), torch.nn.LayerNorm(C, **kw), T
            layers.append(layer)
        proj = torch.nn.Module()
        proj.image_projection_layers = layers
        procs = [FluxIPAdapterAttnProcessor(D, C, n_adapters, dev) for _ in eng.w.double]
        for p in list(proj.parameters()) + [q for pr in procs for q in pr.parameters()]:
            if p.dim() == 2:
                p.normal_(0.0, p.shape[1] ** -0.5, generator=g)
    module = types.SimpleNamespace(encoder_hid_proj=proj)
    embeds = [torch.randn(1, 1, emb, device=dev, generator=g).bfloat16() for _ in range(n_adapters)]
    call = mmdit.IPAdapterCall(module, procs, embeds, D, dev)

    def set_ip(c):
        eng.ip = c

    times = _alternate(eng, {"plain": lambda: set_ip(None), "ip": lambda: set_ip(call)}, ("miss", "hit"), rounds, per_round)
    # the kernel alone at 4096 rows: q the q half of a q|k buffer, out the 5D-pitch buffer the engine writes
    q = torch.randn(n_img, 2 * D, device=dev, generator=g).bfloat16()[:, :D]
    out = torch.empty(n_img, 5 * D, **kw)[:, :D]
    kv = torch.randn(n_adapters * T, 2 * D, device=dev, generator=g).bfloat16()
    w = torch.ones(128, device=dev)
    args = (q, w, eng.w.heads, kv, [T] * n_adapters, [1.0] * n_adapters)
    for _ in range(10):
        ops.ip_attention(*args, out=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 200
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        ops.ip_attention(*args, out=out)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / n * 1e3
    kernel_bytes = 2 * n_img * D * 2 + n_adapters * T * 2 * D * 2  # q read, output written, K|V read once per head (L2 after that)
    name, power = card()
    med = {f"ms_{k}_{kind}": round(statistics.median(v), 3) for (k, kind), v in times.items()}
    print(json.dumps({"family": "flux", "workload": "1024x1024 forward", "ip_adapters": n_adapters, "ip_tokens": T, **med,
                      "ms_added_miss": round(med["ms_ip_miss"] - med["ms_plain_miss"], 3),
                      "ms_added_hit": round(med["ms_ip_hit"] - med["ms_plain_hit"], 3),
                      "spread_ms": {f"{k}_{kind}": [round(min(v), 3), round(max(v), 3)] for (k, kind), v in times.items()},
                      "ip_attn_us_4096_rows": round(us, 2), "ip_attn_bytes": kernel_bytes,
                      "ip_attn_GBps": round(kernel_bytes / (us * 1e-6) / 1e9, 1),
                      "rounds": rounds, "forwards_per_round": per_round, "gpu": name, "power_limit": power}))


def bench_qwen_image(edit, rounds, per_round):
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    torch.cuda.reset_peak_memory_stats()
    eng = mmdit.QwenImageEngine(mmdit.random_qwen_weights(dev))
    weights = torch.cuda.memory_allocated()
    shapes = [[(1, 64, 64), (1, 64, 64)]] if edit else [(1, 83, 83)]
    n_img = 8192 if edit else 6889
    hs = torch.randn(1, n_img, 64, device=dev, generator=g).bfloat16()
    enc = {n: torch.randn(1, n, 3584, device=dev, generator=g).bfloat16() for n in (200, 6)}
    t = torch.tensor([0.6], device=dev)
    slot = {200: 0, 6: 1}
    modes = {n: (lambda n=n: eng.stage_inputs(hs, enc[n], None, t, shapes, [n])) for n in enc}

    class Slotted:  # `_alternate` calls forward(kind); the slot follows the branch
        def __init__(self):
            self.n = 200

        def forward(self, kind):
            return eng.forward(kind, slot[self.n])

    sl = Slotted()
    modes = {n: (lambda n=n, f=f: (setattr(sl, "n", n), f())) for n, f in modes.items()}
    times = _alternate(sl, modes, ("miss", "hit"), rounds, per_round)
    med = {k: statistics.median(v) for k, v in times.items()}
    mask = mc.PRESETS["qwen-image-edit-E006K2R02" if edit else "qwen-image-E006K2R02"].schedule()
    total = sum(med[(200 if i % 2 == 0 else 6, "hit" if s else "miss")] for i, s in enumerate(mask))
    name, power = card()
    print(json.dumps({"family": "qwen-image-edit" if edit else "qwen-image", "gpu": name, "power_limit": power, "image_tokens": n_img,
                      "miss_cond_ms": med[(200, "miss")], "miss_uncond_ms": med[(6, "miss")], "hit_ms": med[(200, "hit")],
                      "spread_ms": {f"{k[0]}_{k[1]}": [min(v), max(v)] for k, v in times.items()},
                      "peak_gib": torch.cuda.max_memory_allocated() / 2**30, "engine_weights_gib": weights / 2**30,
                      "E006K2R02_50_steps_s": total / 1e3, "hits": int(sum(mask)), "calls": len(mask)}))


def _qwen_engine(edit):
    """A Qwen-Image engine on synthetic weights with the cond (200 text tokens) and uncond (6) inputs of one step: (engine, its
    `_alternate` stand-in, {text tokens: staging function}, image tokens, generator)."""
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    eng = mmdit.QwenImageEngine(mmdit.random_qwen_weights(dev))
    shapes = [[(1, 64, 64), (1, 64, 64)]] if edit else [(1, 83, 83)]
    n_img = 8192 if edit else 6889
    hs = torch.randn(1, n_img, 64, device=dev, generator=g).bfloat16()
    enc = {n: torch.randn(1, n, 3584, device=dev, generator=g).bfloat16() for n in (200, 6)}
    t = torch.tensor([0.6], device=dev)
    slot = {200: 0, 6: 1}
    stage = {n: (lambda n=n: eng.stage_inputs(hs, enc[n], None, t, shapes, [n])) for n in enc}

    class Slotted:  # `_alternate` calls forward(kind); the slot follows the branch
        def __init__(self):
            self.n = 200

        def forward(self, kind):
            return eng.forward(kind, slot[self.n])

    sl = Slotted()
    return eng, sl, {n: (lambda n=n, f=f: (setattr(sl, "n", n), f())) for n, f in stage.items()}, n_img, g


def bench_qwen_lora(edit, rank, rounds, per_round):
    """Cond miss and hit forwards at 1328^2 (Edit: 2 x 1024^2) without adapters and with one rank-`rank` adapter (scaling 1) on
    every covered target, alternating; then the down-projections of one miss alone."""
    from magcache_b200.lora import QWEN, LoraPack
    torch.cuda.reset_peak_memory_stats()
    eng, sl, stage, n_img, g = _qwen_engine(edit)
    w, dev, D = eng.w, eng.device, eng.w.dim
    weights = torch.cuda.memory_allocated()

    def ad(n_out, n_in):
        A = (torch.randn(rank, n_in, device=dev, generator=g) / n_in ** 0.5).bfloat16()
        return [(A, (0.02 * torch.randn(n_out, rank, device=dev, generator=g)).bfloat16(), 1.0)]

    spec = {}
    for i in range(len(w.double)):
        for t, (o, k) in {"attn.to_q": (D, D), "attn.to_k": (D, D), "attn.to_v": (D, D), "attn.to_out.0": (D, D), "attn.add_q_proj": (D, D),
                          "attn.add_k_proj": (D, D), "attn.add_v_proj": (D, D), "attn.to_add_out": (D, D), "img_mlp.net.0.proj": (4 * D, D),
                          "img_mlp.net.2": (D, 4 * D), "txt_mlp.net.0.proj": (4 * D, D), "txt_mlp.net.2": (D, 4 * D),
                          "img_mod.1": (6 * D, D), "txt_mod.1": (6 * D, D)}.items():
            spec[("double", i, t)] = ad(o, k)
    for t, (o, k) in {"img_in": (D, w.in_channels), "txt_in": (D, w.joint_dim), "proj_out": (w.out_w.shape[0], D),
                      "norm_out.linear": (2 * D, D)}.items():
        spec[("top", 0, t)] = ad(o, k)
    adapters = torch.cuda.memory_allocated() - weights
    pack = LoraPack(w, spec, family=QWEN)
    packed = torch.cuda.memory_allocated() - weights - adapters

    def set_lora(p):
        stage[200]()
        eng.lora = p

    stage[6]()  # both workspaces exist, as in a pipeline run
    times = _alternate(sl, {"plain": lambda: set_lora(None), "lora": lambda: set_lora(pack)}, ("miss", "hit"), rounds, per_round)
    # the down-projections of one miss alone: every group's input is still staged from the last miss
    set_lora(pack)
    sl.forward("miss")
    groups = list(pack.groups.values()) + [gr for b in pack.double for gr in b["lora"].values()]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    down = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(per_round):
            for gr in groups:
                ops.gemm(gr.src, gr.A, out=gr.u)
        e1.record()
        torch.cuda.synchronize()
        down.append(e0.elapsed_time(e1) / per_round)
    down_bytes = sum(gr.src.shape[0] * gr.src.shape[1] * 2 + gr.A.numel() * 2 + gr.u.numel() * 2 for gr in groups)
    name, power = card()
    med = {f"ms_{k}_{kind}": round(statistics.median(v), 3) for (k, kind), v in times.items()}
    added = med["ms_lora_miss"] - med["ms_plain_miss"]
    print(json.dumps({"family": "qwen-image-edit" if edit else "qwen-image", "workload": "cond (200-token) forward", "image_tokens": n_img,
                      "lora_rank": rank, "lora_targets": len(spec), **med, "ms_added_miss": round(added, 3),
                      "ms_added_hit": round(med["ms_lora_hit"] - med["ms_plain_hit"], 3),
                      "ms_down_projections_miss": round(statistics.median(down), 3),
                      "ms_tails_and_rest_miss": round(added - statistics.median(down), 3),
                      "down_projection_launches": len(groups), "down_projection_GB": round(down_bytes / 1e9, 2),
                      "spread_ms": {f"{k}_{kind}": [round(min(v), 3), round(max(v), 3)] for (k, kind), v in times.items()},
                      "spread_down_ms": [round(min(down), 3), round(max(down), 3)],
                      "adapter_weights_gb": round(adapters / 1e9, 3), "packed_gb": round(packed / 1e9, 3),
                      "peak_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2),
                      "rounds": rounds, "forwards_per_round": per_round, "gpu": name, "power_limit": power}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("family", choices=["flux", "hunyuan", "qwen-image"])
    ap.add_argument("--edit", action="store_true", help="qwen-image: Qwen-Image-Edit's two 1024^2 images")
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--no-cache", action="store_true")
    ap.add_argument("--frames", type=int, default=33, help="hunyuan: latent frames (33 = 129 video frames)")
    ap.add_argument("--controlnet", default=None, help="flux: D,S double / single ControlNet samples; times the miss forward with and without")
    ap.add_argument("--controlnet-repeat", action="store_true", help="controlnet_blocks_repeat (XLabs): double block i reads sample i %% D")
    ap.add_argument("--lora", type=int, default=None, help="flux, qwen-image: rank of one adapter on every covered target; times miss and hit forwards with and without")
    ap.add_argument("--ip-adapter", default=None, help="flux: A[,T] IP-Adapters of T image-prompt tokens (default 16); times miss and hit forwards with and without")
    ap.add_argument("--rounds", type=int, default=5, help="--controlnet / --lora / --ip-adapter: alternating rounds")
    args = ap.parse_args()
    if args.family == "qwen-image" and args.lora is not None:
        bench_qwen_lora(args.edit, args.lora, args.rounds, args.steps or 3)
        return
    if args.family == "qwen-image":
        bench_qwen_image(args.edit, args.rounds, args.steps or 3)
        return
    if args.ip_adapter is not None:
        if args.family != "flux":
            ap.error("--ip-adapter is a FLUX option")
        a_t = [int(v) for v in args.ip_adapter.split(",")]
        bench_ip_adapter(a_t[0], a_t[1] if len(a_t) > 1 else 16, args.rounds, args.steps or 10)
        return
    if args.lora is not None:
        if args.family != "flux":
            ap.error("--lora is a FLUX option")
        bench_lora(args.lora, args.rounds, args.steps or 10)
        return
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
