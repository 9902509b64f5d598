#!/usr/bin/env python
"""Generate tests/golden/opensora_sp.json and opensora_sp.npz by EXECUTING the reference's own sequence-parallel (DSP) Open-Sora code
under gloo process groups of 2 and 4 ranks. Run where the reference tree is present:

    python tests/golden/make_opensora_sp_golden.py

It builds on the loader of make_opensora_golden.py (the STDiT3 modules and `magcache_forward` / `teacache_forward` executed
unmodified) and adds, from videosys/core/comm.py, `_all_to_all_func`, `_AllToAll`, `_split_sequence_func`, `_gather_sequence_func`,
`_GatherForwardSplitBackward`, `_SplitForwardGatherBackward`, `split_sequence`, `gather_sequence`, `PAD_DICT`, `set_pad`, `get_pad`
and `all_to_all_with_pad`, executed unmodified with two exceptions: `dist.all_to_all` (gloo has no list form) is provided through
`all_to_all_single`, moving the same chunks; and the `assert input_.device.type == "cuda"` of `_gather_sequence_func` is cut out of
the source. A stand-in ParallelManager carries sp_size, sp_group (the world group) and cp_size = 1.

The reference's DSP path passes `x_mask` through `split_sequence` (eval/magcache/experiments/opensora.py:288-291), which fails on
None, so every call here gives an all-True x_mask [B, T]: every row then takes the t (not t0) modulation, and the fixture records
that the sp = 1 outputs with that mask are bit-equal to the sp = 1 outputs without one.

Shapes: the tiny STDiT3, B = 2, a 12 x 14 latent (S = 6 x 7 = 42, a position pad at P = 4); T = 7 on 2 ranks (frames 4 | 3) and
4 ranks (2 | 2 | 2 | 1), T = 35 on 2 ranks. Calls: MagCache (thresh 0.5, K 3, skip_time 2, 10 calls with hits) and TeaCache
(`rel_l1_thresh` 0.1 and 10, 10 and 6 calls; `enable_teacache` False, 2 calls), fp32 and bf16, inputs from tests/opensora_sp_cases.py.
Recorded: each rank's frame range after the split, each rank's controller attributes per call, whether each rank's output equals the
sp = 1 output (bf16: bit-equal; fp32: the largest difference), and the bf16 sp = 1 outputs of the T = 7 MagCache run.
"""
import ast
import contextlib
import io
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
import make_opensora_golden as G  # noqa: E402
import opensora_sp_cases as C  # noqa: E402

COMM = f"{G.REF}/videosys/core/comm.py"
COMM_DEFS = ["_all_to_all_func", "_AllToAll", "_split_sequence_func", "_gather_sequence_func", "_GatherForwardSplitBackward",
             "_SplitForwardGatherBackward", "split_sequence", "gather_sequence", "PAD_DICT", "set_pad", "get_pad", "all_to_all_with_pad"]
CUDA_ASSERT = '    assert input_.device.type == "cuda"\n'
B, HX, WX = 2, 12, 14
CASES = [(7, 2), (7, 4), (35, 2)]
RUNS = [("magcache", None, 10), ("teacache", 0.1, 10), ("teacache", 10.0, 6), ("plain", None, 2)]


def _all_to_all(output_list, input_list, group=None):
    """`dist.all_to_all` through `all_to_all_single`: the same chunks to and from the same ranks."""
    send = torch.cat([t.reshape(-1) for t in input_list])
    recv = torch.empty(sum(t.numel() for t in output_list), dtype=send.dtype)
    dist.all_to_all_single(recv, send, [t.numel() for t in output_list], [t.numel() for t in input_list], group=group)
    for o, c in zip(output_list, recv.split([t.numel() for t in output_list])):
        o.copy_(c.view(o.shape))


def _namespace():
    ns = G._namespace()
    for seg in G._defs(G.EVAL, ["teacache_forward"]):
        exec(compile(seg, G.EVAL, "exec"), ns)  # noqa: S102
    shim = types.SimpleNamespace(**{n: getattr(dist, n) for n in dir(dist) if not n.startswith("__")})
    shim.all_to_all = _all_to_all
    ns.update(dist=shim, Tensor=torch.Tensor, Any=object, Tuple=tuple, ProcessGroup=object, Optional=__import__("typing").Optional)
    for name, seg in zip(COMM_DEFS, G._defs(COMM, COMM_DEFS)):
        if name == "_gather_sequence_func":
            assert seg.count(CUDA_ASSERT) == 1
            seg = seg.replace(CUDA_ASSERT, "")
        exec(compile(seg, COMM, "exec"), ns)  # noqa: S102
    return ns


class _PM:
    def __init__(self, world):
        self.sp_size, self.cp_size = world, 1
        self.sp_group = dist.group.WORLD if world > 1 else None


def _model(ns, kind, thresh, dtype, world):
    model, state = G.build_reference(ns, dtype)
    if kind != "magcache":
        with torch.no_grad():
            for n, p in model.named_parameters():
                if n.startswith("t_block."):
                    p.data = (state[n] * 0.05).to(dtype)
    pm = _PM(world)
    model.parallel_manager = pm
    for blk in list(model.spatial_blocks) + list(model.temporal_blocks):
        blk.parallel_manager = pm
    cls = model.__class__
    if kind == "magcache":
        cls.forward = ns["magcache_forward"]
        cls.magcache_thresh, cls.K, cls.skip_time = 0.5, 3, 2
    else:
        cls.forward = ns["teacache_forward"]
        cls.enable_teacache, cls.rel_l1_thresh = kind == "teacache", thresh if thresh is not None else 0.1
        cls.accumulated_rel_l1_distance, cls.previous_modulated_input, cls.previous_residual = 0, None, None
    return model


def _calls(model, kind, n, T, dtype, x_mask, cy=64):
    lat, y, kw = C.video(B, T, HX, WX, cy=cy)
    ts, all_ts = C.timesteps(n, B, "cpu")
    names = C.MAG_ATTRS if kind == "magcache" else C.TEA_ATTRS
    outs, attrs = [], []
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        for i in range(n):
            mk = torch.ones(B, T, dtype=torch.bool) if x_mask else None
            o = model(lat(i).to(dtype), ts[i], all_ts, y.to(dtype), x_mask=mk, **kw)
            outs.append(o.float().clone())
            attrs.append({a: float(getattr(model, a)) for a in names})
    return outs, attrs


def _frame_range(T, world, rank):
    chunk = (T + (world - T % world) % world) // world
    return [rank * chunk, min((rank + 1) * chunk, T)]


def _worker(rank, world, initfile, cases, outdir):
    dist.init_process_group("gloo", init_method=f"file://{initfile}", rank=rank, world_size=world)
    torch.set_num_threads(max(1, (os.cpu_count() or 1) // world))
    try:
        ns = _namespace()
        split_seen = []
        orig_split = ns["split_sequence"]

        def split(input_, process_group, dim, grad_scale=1.0, pad=0):  # records the frame range this rank receives
            out = orig_split(input_, process_group, dim, grad_scale, pad)
            if dim == 1 and input_.dim() == 4:
                chunk = (input_.shape[1] + pad) // world
                split_seen.append([rank * chunk, rank * chunk + out.shape[1] - max(0, rank * chunk + chunk - input_.shape[1])])
            return out

        ns["split_sequence"] = split
        rec = {}
        for T in cases:
            for kind, thresh, n in RUNS:
                for dname, dtype in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
                    split_seen.clear()
                    outs, attrs = _calls(_model(ns, kind, thresh, dtype, world), kind, n, T, dtype, True)
                    rec[f"T{T}_{kind}_{thresh}_{dname}"] = dict(outs=torch.stack(outs), attrs=attrs, split=split_seen[:1])
        torch.save(rec, os.path.join(outdir, f"w{world}_r{rank}.pt"))
    finally:
        dist.destroy_process_group()


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    ns = _namespace()
    doc = {"config": G.CFG, "seed": G.SEED, "B": B, "Hx": HX, "Wx": WX, "cases": CASES, "runs": {}}
    arrays = {}
    one = {}
    for T in sorted({t for t, _ in CASES}):
        for kind, thresh, n in RUNS:
            for dname, dtype in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
                key = f"T{T}_{kind}_{thresh}_{dname}"
                outs, attrs = _calls(_model(ns, kind, thresh, dtype, 1), kind, n, T, dtype, True)
                outs0, _ = _calls(_model(ns, kind, thresh, dtype, 1), kind, n, T, dtype, False)
                assert all(torch.equal(a, b) for a, b in zip(outs, outs0)), key  # the all-True x_mask changes no bit
                one[key] = (torch.stack(outs), attrs)
                if T == 7 and kind == "magcache" and dname == "bf16":
                    arrays[key] = torch.stack(outs).to(torch.bfloat16).view(torch.int16).numpy()
    for T, world in CASES:
        with tempfile.TemporaryDirectory() as d:
            mp.spawn(_worker, args=(world, os.path.join(d, "init"), [T], d), nprocs=world, join=True)
            ranks = [torch.load(os.path.join(d, f"w{world}_r{r}.pt")) for r in range(world)]
        for key, (o1, a1) in one.items():
            if not key.startswith(f"T{T}_"):
                continue
            per_rank = []
            for r, rec in enumerate(ranks):
                o, a = rec[key]["outs"], rec[key]["attrs"]
                per_rank.append(dict(split=rec[key]["split"][0], attrs=a, attrs_equal_sp1=a == a1,
                                     bit_equal_sp1=bool(torch.equal(o, o1)), max_abs_diff_sp1=float((o - o1).abs().max())))
                assert per_rank[-1]["split"] == _frame_range(T, world, r), (key, r, per_rank[-1]["split"])
            doc["runs"][f"P{world}_{key}"] = dict(T=T, world=world, sp1_attrs=a1, ranks=per_rank)
            print(f"P{world}_{key}", [(p["bit_equal_sp1"], p["max_abs_diff_sp1"]) for p in per_rank], flush=True)
    np.savez_compressed(os.path.join(HERE, "opensora_sp.npz"), **arrays)
    with open(os.path.join(HERE, "opensora_sp.json"), "w") as f:
        json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
