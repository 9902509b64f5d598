#!/usr/bin/env python
"""Generate tests/golden/opensora_teacache.npz and opensora_teacache.json by EXECUTING the reference's own Open-Sora TeaCache code.

Run where the reference tree is present (it is not imported by anything else):

    python tests/golden/make_opensora_teacache_golden.py

Reuses make_opensora_golden.py's `ast` loader, stand-ins and STDiT3 build, and executes these unmodified as well:

* eval/magcache/experiments/opensora.py: `teacache_forward`, and the class-attribute statements of `eval_teacache_slow` (0.1) and
  `eval_teacache_fast` (0.2), executed against a stand-in `engine` whose driver_worker.transformer is the model
* videosys/schedulers/scheduling_rflow_open_sora.py: `timestep_transform`, and the statements of `RFLOW.sample` that build the
  timesteps and `all_timesteps` (:208-213, :221-222)

Fixture: the tiny STDiT3 of opensora_forward.json at B = 2 (the CFG pair, one timestep for both samples like the sampler), two
consecutive 30-call videos with no reset between them, the latents moved between calls (tests/opensora_tea_ref.video_inputs), in fp32
and in bf16, under both thresholds and two timestep schedules: "transform" (Open-Sora 1.2's default `use_timestep_transform` at 480p
x 51 frames: its last timestep rounds to a whole bf16 number, so the bf16 model's last call is forced as well as its first) and
"linear" (no transform: the last timestep, 33.33, rounds to bf16 33.25 while `all_timesteps[-1]` is 33, so only the first call is
forced). The t_block weights are scaled by 0.05: with random weights the modulation would otherwise change by ~20 % between sampler
steps, far outside TeaCache's working range, and every call would compute. Per call: forced, calc, the `rel` the polynomial saw, the
accumulated distance after the call and the output (float32; the bf16 model's outputs are bf16 values, stored as their bit patterns).
"""
import ast
import contextlib
import io
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_opensora_golden as G  # noqa: E402
import opensora_tea_ref as TR  # noqa: E402

EVAL = G.EVAL
RFLOW = f"{G.REF}/videosys/schedulers/scheduling_rflow_open_sora.py"
B, T, H, W = 2, 2, 4, 4
CALLS, VIDEOS = 30, 2
INPUT_SEED, LATENT_STEP = 3, 0.004
T_BLOCK_SCALE = 0.05
SCHEDULES = {"transform": dict(use_timestep_transform=True, use_discrete_timesteps=False),
             "linear": dict(use_timestep_transform=False, use_discrete_timesteps=False)}
MODEL_ARGS = dict(height=480, width=854, num_frames=51)  # the paper's 480p 9:16, 51 frames


def _attribute_statements(fn_name):
    src = open(EVAL).read()
    fn = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == fn_name)
    return "\n".join(ast.get_source_segment(src, st) for st in fn.body if "driver_worker.transformer.__class__" in ast.get_source_segment(src, st))


def _timestep_statements():
    """The statements of RFLOW.sample that form `timesteps` and `all_timesteps`, in source order."""
    src = open(RFLOW).read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "RFLOW")
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "sample")
    keep = []
    for st in fn.body:
        seg = ast.get_source_segment(src, st)
        if isinstance(st, (ast.Assign, ast.If)) and ("timesteps" in seg.split("=")[0] or seg.startswith("dtype =") or
                                                     seg.startswith("if self.use_")):
            keep.append(seg)
    assert len(keep) == 6, keep
    return "\n".join(keep)


def schedule(ns, name, model):
    sched = types.SimpleNamespace(num_sampling_steps=CALLS, num_timesteps=1000, **SCHEDULES[name])
    model_args = {k: torch.tensor([float(v)]) if k != "num_frames" else torch.tensor([v]) for k, v in MODEL_ARGS.items()}
    env = dict(self=sched, torch=torch, z=torch.zeros(B // 2, 4, T, H, W), device="cpu", model_args=model_args, model=model,
               timestep_transform=ns["timestep_transform"])
    exec(_timestep_statements(), env)  # noqa: S102
    steps = [torch.cat([t, t], 0) for t in env["timesteps"]]  # :238-239
    return steps, env["all_timesteps"]


def run(model, steps, all_timesteps, doc):
    latents, y, kw = TR.video_inputs(doc)
    outs, rec = [], []
    log = io.StringIO()
    with torch.no_grad(), contextlib.redirect_stdout(log):
        for v in range(VIDEOS):
            for i in range(CALLS):
                prev, res = model.previous_modulated_input, model.previous_residual
                seen = []
                orig = np.poly1d.__call__

                def spy(self, val, _orig=orig, _seen=seen):  # the value the rescale polynomial is evaluated at
                    _seen.append(float(val))
                    return _orig(self, val)

                np.poly1d.__call__ = spy
                try:
                    out = model(latents(i + v * CALLS), steps[i], all_timesteps, y, **kw)
                finally:
                    np.poly1d.__call__ = orig
                forced = len(seen) == 0
                calc = model.previous_residual is not res  # a miss stores a new residual (:156)
                rec.append(dict(forced=forced, calc=calc, rel=None if forced else seen[0],
                                acc=float(model.accumulated_rel_l1_distance)))
                assert prev is None or model.previous_modulated_input is not prev
                outs.append(out.numpy().astype(np.float32))
    return np.stack(outs), rec


def main():
    ns = G._namespace()
    for seg in G._defs(EVAL, ["teacache_forward"]):
        exec(compile(seg, EVAL, "exec"), ns)  # noqa: S102
    for seg in G._defs(RFLOW, ["timestep_transform"]):
        exec(compile(seg, RFLOW, "exec"), ns)  # noqa: S102
    doc = {"config": G.CFG, "B": B, "T": T, "H": H, "W": W, "seed": G.SEED, "input_seed": INPUT_SEED, "latent_step": LATENT_STEP,
           "t_block_scale": T_BLOCK_SCALE,
           "height": MODEL_ARGS["height"], "width": MODEL_ARGS["width"], "calls": CALLS, "videos": VIDEOS, "runs": {}}
    arrays = {}
    for dname, dtype in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        for sname in SCHEDULES:
            for preset, thresh in (("eval_teacache_slow", 0.1), ("eval_teacache_fast", 0.2)):
                model, state = G.build_reference(ns, dtype)
                with torch.no_grad():
                    for n, p in model.named_parameters():
                        if n.startswith("t_block."):
                            p.data = (state[n] * T_BLOCK_SCALE).to(dtype)
                model.__class__ = type(f"RefTea_{dname}_{sname}_{thresh}", (ns["STDiT3"],), {})
                engine = types.SimpleNamespace(driver_worker=types.SimpleNamespace(transformer=model))
                exec(_attribute_statements(preset), dict(engine=engine, teacache_forward=ns["teacache_forward"]))  # noqa: S102
                assert model.rel_l1_thresh == thresh
                steps, all_ts = schedule(ns, sname, model)
                out, rec = run(model, steps, all_ts, doc)
                key = f"{dname}_{sname}_{thresh}"
                calcs = [r["calc"] for r in rec]
                assert True in calcs and False in calcs, (key, calcs)
                arrays[key] = out if dname == "fp32" else torch.from_numpy(out).to(torch.bfloat16).view(torch.int16).numpy()
                doc["runs"][key] = dict(dtype=dname, schedule=sname, thresh=thresh, records=rec,
                                        timesteps=[s.tolist() for s in steps], all_timesteps=all_ts, discrete=False)
                print(key, "".join("F" if r["forced"] else ("c" if r["calc"] else ".") for r in rec))
    forced_last = {k: r["records"][CALLS - 1]["forced"] for k, r in doc["runs"].items()}
    assert all(forced_last[k] == (k.split("_")[1] == "transform") for k in forced_last if k.startswith("bf16")), forced_last
    np.savez_compressed(os.path.join(HERE, "opensora_teacache.npz"), **arrays)
    with open(os.path.join(HERE, "opensora_teacache.json"), "w") as f:
        json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
