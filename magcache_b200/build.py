"""Build libmagcache_b200.so (sm_90a only) in-tree with nvcc. `python magcache_b200/build.py [--force]`."""
import os
import re
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmagcache_b200.so")
SOURCES = ["controller.cu", "cache_kernels.cu", "rowwise_kernels.cu", "gemm_wgmma.cu", "attn_wgmma.cu", "head_wgmma.cu", "p2p.cu", "dit_forward.cu", "nccl_gather.cu", "opensora_kernels.cu",
           "opensora_head.cu", "ip_attn.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
              "-Xptxas", "-v", "--expt-relaxed-constexpr"]
# Entry functions that keep tensor-core accumulators in registers (wgmma; mma.sync for attn_varlen_d72_kernel,
# attn_temporal_mma_d72_kernel and ip_attn_kernel) and must not spill. head_tc_kernel issues wgmma too but still spills (~350 B, in its
# 104-register converter warps, not next to its accumulators); it joins this list once that is fixed (DESIGN §8).
NO_SPILL_KERNELS = ("attn_kernel", "gemm_bf16_kernel", "attn_varlen_d72_kernel", "attn_temporal_mma_d72_kernel", "opensora_head_kernel",
                    "ip_attn_kernel")


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "magcache_b200.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps)


def _check_ptxas(log):
    """Reject the ptxas outcomes that silently cost the tensor-core kernels a large part of their rate.

    C7510: ptxas serialised a kernel's wgmmas (a wait after every one) because the kernel contains a function call, e.g. a
    device printf. C7512: it serialised them for want of registers. Spills in the kernels that hold their accumulators in
    registers put local-memory traffic into the main loop or epilogue; the log reports them per entry function."""
    serialised = [line.strip() for line in log.splitlines() if "C7510" in line or "C7512" in line]
    if serialised:
        raise RuntimeError("ptxas serialised wgmma (C7510: the kernel contains a function call such as device printf, see "
                           "MC_DEVICE_DIAG in csrc/ptx.cuh; C7512: not enough registers). Full log: build/ptxas.log\n" +
                           "\n".join(serialised[:8]))
    spills, fn = [], None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m and fn is not None:
            if int(m.group(1)) > 0 and any(k in fn for k in NO_SPILL_KERNELS):
                spills.append(f"{fn}: {line.strip()}")
            fn = None
    if spills:
        raise RuntimeError("ptxas spilled registers in a kernel that issues wgmma. Full log: build/ptxas.log\n" + "\n".join(spills))


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    objs = []
    bdir = os.path.join(HERE, "build")
    os.makedirs(bdir, exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = os.path.join(bdir, src.replace(".cu", ".o"))
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {src}\n{out}")
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {src}")
    with open(os.path.join(bdir, "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    _check_ptxas("\n".join(log))
    cmd = [_nvcc(), "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static", "-ldl"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
