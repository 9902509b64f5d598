"""Open-Sora 1.2 (STDiT3-XL/2) with sequence parallelism over the GPUs of one node, against the one-GPU engine in the same job.

    torchrun --nproc-per-node N tools/bench_opensora_sp.py [--frames 15] [--reps 5]

Workload: full-size seeded random weights, 480p 9:16 (60 x 106 latent, 1590 patches per frame), B = 2, 300 caption tokens (200 valid),
--frames latent frames (15 / 30 / 60 / 120 / 240 for 2 ... 32 s). Prints one JSON line per rank: miss and hit ms (CUDA events, median
of --reps, the forward alone: inputs staged before the events), rank 0's one-GPU miss ms and the speedup, bf16 bytes this rank sends
per miss (two switches per temporal block), the stream time of the exchanges of one miss split into issue + copies (bump, 2-D pushes,
flags) and the flag wait kernel (events around each part of a separate profiled miss), whether the gathered output is
bit-equal to the one-GPU engine's, and the card, power limit and SM clocks (query only). With fewer GPUs than ranks, ranks share
devices (rank r on GPU r mod count): the parity holds, the timings then say nothing about scaling.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]


def _smi(idx):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={idx}", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def _median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=15)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    ngpu = torch.cuda.device_count()
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)) % ngpu)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo")  # IPC handles and the barrier only: the data moves over the copy engines (P2P switch)
    from magcache_b200 import ops
    from magcache_b200 import opensora as os_mod

    w = os_mod.random_opensora_weights(dev)
    g = torch.Generator().manual_seed(1)
    T = a.frames
    x = torch.randn(2, 4, T, 60, 106, generator=g).to(dev)
    y = torch.randn(2, 1, 300, 4096, generator=g).to(dev)
    mask = torch.ones(2, 300, dtype=torch.long, device=dev)
    mask[:, 200:] = 0
    args = (torch.tensor([700.0, 700.0], device=dev), y, mask, torch.tensor([24.0], device=dev), torch.tensor([480.0], device=dev),
            torch.tensor([854.0], device=dev))
    rec = dict(rank=rank, world=world, frames=T, device=str(dev), card=_smi(dev.index))

    ref_out, one_ms = None, None
    if rank == 0:
        one = os_mod.OpenSoraEngine(w)
        one.stage_inputs(x, *args)
        ref_out = one.forward("miss")
        one_ms = _median_ms(lambda: one.forward("miss"), a.reps)
        ref_out = ref_out.cpu()
        del one
        torch.cuda.empty_cache()
    dist.barrier()

    sp = os_mod.OpenSoraEngine(w, sp_world=world, sp_rank=rank)
    sp.stage_inputs(x, *args)
    out = sp.forward("miss")
    torch.cuda.synchronize()
    box = [None]
    if rank == 0:
        box = [ref_out]
    dist.broadcast_object_list(box, src=0)
    rec["parity_bit_equal"] = bool(torch.equal(out.cpu(), box[0]))
    rec["miss_ms"] = _median_ms(lambda: sp.forward("miss"), a.reps)
    rec["hit_ms"] = _median_ms(lambda: sp.forward("hit"), a.reps)
    if rank == 0:
        rec["one_gpu_miss_ms"] = one_ms
        rec["speedup_miss"] = one_ms / rec["miss_ms"]
    sw = sp.switch
    rec["switch_bytes_per_miss"] = 2 * sp.w.depth * sw.bytes_per_switch()
    rec["frames_owned"] = sp.T_loc
    # one profiled miss: events around the pushes (bump, 2-D copies, flags) and around the flag wait kernel of every exchange
    import types
    real = sw._lib
    pushes, waits = [], []

    def bracketed(fn, into):
        def call(*args_):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(*args_)
            e1.record()
            into.append((e0, e1))
            return r
        return call

    if sw.p2p:  # this switch's own view of the library, with the two entry points bracketed
        lib = types.SimpleNamespace(mc_p2p_bump=real.lib.mc_p2p_bump, mc_p2p_push2d=bracketed(real.lib.mc_p2p_push2d, pushes),
                                    mc_p2p_wait=bracketed(real.lib.mc_p2p_wait, waits))
        sw._lib = types.SimpleNamespace(lib=lib, check=real.check, Copy2D=real.Copy2D)
    try:
        sp.forward("miss")
        torch.cuda.synchronize()
    finally:
        sw._lib = real
    rec["switch_push_ms_per_miss"] = sum(e0.elapsed_time(e1) for e0, e1 in pushes)
    rec["switch_flag_wait_ms_per_miss"] = sum(e0.elapsed_time(e1) for e0, e1 in waits)
    rec["switch_p2p"] = sw.p2p
    rec["launches"] = ops.LAUNCHES
    print(json.dumps(rec), flush=True)
    sw.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
