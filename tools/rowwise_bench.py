"""HBM-bound row kernels at the benchmarked shape (32760 tokens x 1536): achieved GB/s against their algorithmic bytes. Also one
case per other launch form: 512 rows (the register-pipelined forms, below the 1024 rows of the staged ones) and 5120 columns
(the Wan-14B width: the wide forms).
python tools/rowwise_bench.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magcache_b200 import ops  # noqa: E402

N, D, H = 32760, 1536, 12
dev = "cuda"
g = torch.Generator(device=dev).manual_seed(0)
x32 = torch.randn(N, D, device=dev, generator=g)
em = torch.randn(6, D, device=dev, generator=g) * 0.1
out16 = torch.empty(N, D, device=dev, dtype=torch.bfloat16)
qkv = torch.randn(N, 3 * D, device=dev, generator=g).bfloat16()
cq = torch.randn(N, D, device=dev, generator=g).bfloat16()
w2 = torch.ones(2, D, device=dev)
w1 = torch.ones(D, device=dev)
bias = torch.zeros(D, device=dev)
cs = torch.randn(N, 128, device=dev, generator=g)
p32 = torch.randn(N, D, device=dev, generator=g)
xi16 = torch.randn(N, D, device=dev, generator=g).bfloat16()
NS, DW = 512, 5120
xw = torch.randn(N, DW, device=dev, generator=g)
ow = torch.empty(N, DW, device=dev, dtype=torch.bfloat16)
emw = torch.randn(6, DW, device=dev, generator=g) * 0.1
qw = torch.randn(N, DW, device=dev, generator=g).bfloat16()
w1w = torch.ones(DW, device=dev)
flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        flush.zero_()  # L2 flush between timed launches
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters


cases = {
    "ln_modulate fp32->bf16": (lambda: ops.ln_modulate(x32, em, 1, 0, out=out16), N * D * (4 + 2)),
    "ln_affine fp32->bf16": (lambda: ops.ln_affine(x32, w1, bias, out=out16), N * D * (4 + 2)),
    "rmsnorm_rope q|k in place": (lambda: ops.rmsnorm_rope_segs_(qkv[:, :2 * D], w2, 2, cos_sin=cs), N * 2 * D * 4 + N * 128 * 4),
    "rmsnorm (no rope) in place": (lambda: ops.rmsnorm_rope_(cq, w1), N * D * 4),
    "cache_hit_add bf16": (lambda: ops.cache_hit_add(out16, cq), N * D * 6),
    "residual_stats fp32": (lambda: ops.residual_stats(x32, p32), N * D * 8),
    "residual_sub_stats fp32": (lambda: ops.residual_sub_stats(x32, xi16, p32), N * D * (4 + 2 + 4 + 4)),
    f"ln_modulate {NS} rows": (lambda: ops.ln_modulate(x32[:NS], em, 1, 0, out=out16[:NS]), NS * D * (4 + 2)),
    f"rmsnorm_rope {NS} rows": (lambda: ops.rmsnorm_rope_segs_(qkv[:NS, :2 * D], w2, 2, cos_sin=cs[:NS]), NS * 2 * D * 4 + NS * 128 * 4),
    f"ln_modulate x{DW}": (lambda: ops.ln_modulate(xw, emw, 1, 0, out=ow), N * DW * (4 + 2)),
    f"rmsnorm_rope x{DW}": (lambda: ops.rmsnorm_rope_(qw, w1w, cos_sin=cs), N * DW * 4 + N * 128 * 4),
}
for name, (fn, nbytes) in cases.items():
    ms = timeit(fn)
    print(f"{name:28s} {ms * 1e3:8.1f} us   {nbytes / ms / 1e6:8.1f} GB/s")
