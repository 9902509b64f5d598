"""Per-kernel timings at the Wan2.1-1.3B 832x480x81 shapes (CUDA events, L2 flushed between iterations)."""
import json
import math
import sys

import torch

sys.path.insert(0, ".")
from magcache_b200 import _lib, ops  # noqa: E402

dev = "cuda"
N_TOK, D, FFN, HEADS = 32760, 1536, 8960, 12
flush_buf = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10, warmup=3, flush=True):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush:
            flush_buf.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


res = {}


def rec(name, ms, best, bytes_=None, flops=None):
    d = {"ms_median": round(ms, 4), "ms_best": round(best, 4)}
    if bytes_:
        d["GBps"] = round(bytes_ / ms / 1e6, 1)
    if flops:
        d["TFLOPs"] = round(flops / ms / 1e9, 1)
    res[name] = d
    print(name, d, flush=True)


which = sys.argv[1] if len(sys.argv) > 1 else "all"
n = N_TOK * D
if which in ("all", "cache"):
    x = torch.randn(n, device=dev).bfloat16()
    r = torch.randn(n, device=dev) * 0.1
    out = torch.empty(n, device=dev)
    rec("k1_hit_add_bf16_f32", *timeit(lambda: ops.cache_hit_add(x, r, out=out), iters=20), bytes_=n * 10)
    rec("torch_add_bf16_f32", *timeit(lambda: torch.add(x, r, out=out), iters=20), bytes_=n * 10)
    xo = torch.randn(n, device=dev)
    rec("k2_residual_sub", *timeit(lambda: ops.residual_sub(xo, x, out=out), iters=20), bytes_=n * 10)
    rec("torch_copy_f32", *timeit(lambda: out.copy_(r), iters=20), bytes_=n * 8)
    r2, p2 = r.view(N_TOK, D), (r * 1.01).view(N_TOK, D)
    rec("k3_stats_with_host_sync", *timeit(lambda: ops.residual_stats(r2, p2), iters=10), bytes_=n * 8)
    from magcache_b200._lib import check, lib
    st = torch.empty(4, dtype=torch.float64, device=dev)
    rec("k3_stats_kernels_only", *timeit(lambda: check(lib.mc_residual_stats(r2.data_ptr(), 0, p2.data_ptr(), 0, N_TOK, D, 0.0, st.data_ptr(),
                                                                            torch.cuda.current_stream().cuda_stream)), iters=20), bytes_=n * 8)
    xo2 = torch.randn(N_TOK, D, device=dev)
    xi2 = torch.randn(N_TOK, D, device=dev).bfloat16()
    ro = torch.empty(N_TOK, D, device=dev)
    rec("k2k3_sub_stats_fused_kernels_only", *timeit(lambda: check(lib.mc_residual_sub_stats(xo2.data_ptr(), 0, xi2.data_ptr(), 1, ro.data_ptr(), p2.data_ptr(),
                                                                                         N_TOK, D, 0.0, st.data_ptr(), torch.cuda.current_stream().cuda_stream)), iters=20),
        bytes_=n * 14)
    xb = torch.randn(n, device=dev).bfloat16()
    ob = torch.empty_like(xb)
    rec("k1_hit_add_bf16_all", *timeit(lambda: ops.cache_hit_add(x, xb, out=ob), iters=20), bytes_=n * 6)

if which in ("all", "rows"):
    xs = torch.randn(N_TOK, D, device=dev)
    mod, e = torch.randn(6, D, device=dev) * 0.03, torch.randn(6, D, device=dev) * 0.2
    h = torch.empty(N_TOK, D, dtype=torch.bfloat16, device=dev)
    rec("ln_modulate", *timeit(lambda: ops.ln_modulate(xs, mod, 1, 0, out=h)), bytes_=n * 6)
    qk = torch.randn(N_TOK, D, device=dev).bfloat16()
    w = torch.ones(D, device=dev)
    cs = torch.randn(N_TOK, 128, device=dev)
    rec("rmsnorm_rope", *timeit(lambda: ops.rmsnorm_rope_(qk, w, cs, 128)), bytes_=n * 4 + N_TOK * 512)
    hm, ee = torch.randn(1, 2, D, device=dev) * 0.03, torch.randn(1, D, device=dev)
    Wt, b = torch.randn(D, 64, device=dev) * 0.02, torch.zeros(64, device=dev)
    rec("head_unpatchify", *timeit(lambda: ops.head_unpatchify(xs, hm, ee, Wt, b, (21, 30, 52))), bytes_=n * 4)
    x0 = torch.randn(N_TOK, D, device=dev).bfloat16()
    rec("head_unpatchify_fused_hit", *timeit(lambda: ops.head_unpatchify(x0, hm, ee, Wt, b, (21, 30, 52), residual=xs)), bytes_=n * 6)

if which in ("all", "gemm"):
    # the block GEMMs of one Wan2.1-1.3B layer (wan.py tags), each with the epilogue the engine runs it with, next to
    # torch.matmul (cuBLAS, plain bf16 output) on the same operands; a rate is only worth something with the card it ran on
    import subprocess
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        card = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {ex})"
    res["card"] = card
    print("card:", card, flush=True)
    E = _lib
    for tag, N, K, epi in [("gemm_qkv", 3 * D, D, E.MC_EPI_BIAS_BF16), ("gemm_o", D, D, E.MC_EPI_BIAS_GATE_RESID),
                           ("gemm_cq", D, D, E.MC_EPI_BIAS_BF16), ("gemm_co", D, D, E.MC_EPI_BIAS_GATE_RESID),
                           ("gemm_ffn1", FFN, D, E.MC_EPI_BIAS_GELU_BF16), ("gemm_ffn2", D, FFN, E.MC_EPI_BIAS_GATE_RESID)]:
        a = torch.randn(N_TOK, K, device=dev).bfloat16()
        b = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
        bias = torch.randn(N, device=dev) * 0.01
        gate = torch.randn(N, device=dev) * 0.01 if tag in ("gemm_o", "gemm_ffn2") else None
        if epi == E.MC_EPI_BIAS_GATE_RESID:  # fp32 residual stream, updated in place
            o = torch.randn(N_TOK, N, device=dev)
        else:
            o = torch.empty(N_TOK, N, dtype=torch.bfloat16, device=dev)
        flops = 2.0 * N_TOK * N * K
        rec(f"{tag}_{N_TOK}x{N}x{K}", *timeit(lambda: ops.gemm(a, b, bias, epi, out=o, gate=gate)), flops=flops)
        rec(f"{tag}_cublas", *timeit(lambda: torch.matmul(a, b.t())), flops=flops)
        del a, b, o

if which in ("all", "attn"):
    q = torch.randn(N_TOK, D, device=dev).bfloat16()
    k = torch.randn(N_TOK, D, device=dev).bfloat16()
    vt = torch.randn(N_TOK, D, device=dev).bfloat16()
    o = torch.empty_like(q)
    rec("attn_self_32760", *timeit(lambda: ops.attention(q, k, vt, HEADS, out=o), iters=5, warmup=2), flops=4.0 * N_TOK * N_TOK * D)
    try:
        qh = q.view(1, N_TOK, HEADS, 128).transpose(1, 2)
        kh = k.view(1, N_TOK, HEADS, 128).transpose(1, 2)
        vh = vt.view(1, N_TOK, HEADS, 128).transpose(1, 2)
        rec("attn_self_sdpa_torch", *timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qh, kh, vh), iters=5, warmup=2),
            flops=4.0 * N_TOK * N_TOK * D)
    except Exception as ex:  # noqa: BLE001
        print("sdpa failed", ex)
    kc = torch.randn(512, D, device=dev).bfloat16()
    vtc = torch.randn(512, D, device=dev).bfloat16()
    rec("attn_cross_512", *timeit(lambda: ops.attention(q, kc, vtc, HEADS, out=o)), flops=4.0 * N_TOK * 512 * D)

import os  # noqa: E402
os.makedirs("gpurun_out", exist_ok=True)
with open(f"gpurun_out/microbench_{which}.json", "w") as f:
    json.dump(res, f, indent=1)
