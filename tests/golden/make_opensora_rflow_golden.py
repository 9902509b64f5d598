#!/usr/bin/env python
"""Generate tests/golden/opensora_rflow.npz and opensora_rflow.json by EXECUTING the reference's own Open-Sora sampler.

Run where the reference tree is present (it is not imported by anything else):

    python tests/golden/make_opensora_rflow_golden.py

Executes these unmodified, extracted with make_opensora_golden.py's `ast` loader, from
videosys/schedulers/scheduling_rflow_open_sora.py: `timestep_transform`, `RFlowScheduler`, `RFLOW` (whose `sample` is run whole,
progress off), and the two `dt` statements of its loop (:249-250), evaluated once more per step for the record. The model is the
deterministic stub of tests/opensora_rflow_stub.py, the inputs are the pipeline's (bf16 latent and bf16 height / width / num_frames).

Per case (tests/opensora_rflow_stub.CASES: 480p and 720p, 51 / 102 / 408 frames, cfg 7.0 and 4.5, discrete timesteps on and off,
the transform on and off, B = 1 and 2 prompts): every step's timestep tensor (the first half of the model's `t`), `all_timesteps`,
`dt`, and the latent z entering every step plus the returned one (fp32; the first is the bf16 input's values). With two prompts the
reference raises at `all_timesteps` (`.item()` of a 2-element tensor, :222): the error is recorded, and the record is each prompt's own
run through the reference, side by side (the stub, like every statement of the sampler, works per sample).
"""
import ast
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_opensora_golden as G  # noqa: E402
import opensora_rflow_stub as S  # noqa: E402

RFLOW_SRC = f"{G.REF}/videosys/schedulers/scheduling_rflow_open_sora.py"


def _namespace():
    ns = dict(torch=torch, dist=types.SimpleNamespace(get_rank=lambda: 0), rearrange=None, LogisticNormal=None, tqdm=lambda x: x)
    for seg in G._defs(RFLOW_SRC, ["timestep_transform", "RFlowScheduler", "RFLOW"]):
        exec(compile(seg, RFLOW_SRC, "exec"), ns)  # noqa: S102
    return ns


def _dt_statements():
    src = open(RFLOW_SRC).read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "RFLOW")
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "sample")
    loop = next(st for st in fn.body if isinstance(st, ast.For))
    segs = [ast.get_source_segment(src, st) for st in loop.body
            if isinstance(st, ast.Assign) and isinstance(st.targets[0], ast.Name) and st.targets[0].id == "dt"]
    assert len(segs) == 2, segs
    return "\n".join(segs)


def main():
    ns = _namespace()
    dt_src = _dt_statements()
    doc = {"steps": S.STEPS, "latent": S.LATENT, "cases": {}}
    arrays = {}
    for name in S.CASES:
        z, model_args, y_null = S.case_inputs(name)
        B = z.shape[0]
        rec = dict(reference_error=None)
        if B > 1:  # `int(t.to(dtype).item())` (:222) of a [B] tensor: the reference cannot sample two prompts at once
            try:
                ns["RFLOW"](**S.scheduler_kwargs(name)).sample(S.StubSTDiT3(), z, dict(model_args), y_null, "cpu", progress=False)
            except RuntimeError as e:
                rec["reference_error"] = str(e)
            assert rec["reference_error"] is not None
        # every prompt alone (the stub and the sampler's statements are per sample, so B prompts are these runs side by side)
        runs = []
        for b in range(B):
            sched = ns["RFLOW"](**S.scheduler_kwargs(name))
            model = S.StubSTDiT3()
            args_b = {k: v[b:b + 1] for k, v in model_args.items()}
            with torch.no_grad():
                out = sched.sample(model, z[b:b + 1], args_b, y_null[b:b + 1], "cpu", progress=False)
            timesteps = [t[:1] for _, t, _ in model.calls]
            dts = []
            for i in range(S.STEPS):
                env = dict(timesteps=timesteps, i=i, self=sched)
                exec(dt_src, env)  # noqa: S102
                dts.append(env["dt"])
            assert all(c[2] == model.calls[0][2] for c in model.calls)
            runs.append(dict(timesteps=timesteps, dt=dts, all_timesteps=model.calls[0][2], out=out,
                             zs=[x[:1].float() for x, _, _ in model.calls] + [out.float()]))
        assert all(r["all_timesteps"] == runs[0]["all_timesteps"] for r in runs)
        cat = lambda key, i: torch.cat([r[key][i] for r in runs])  # noqa: E731
        rec.update(timesteps=[cat("timesteps", i).tolist() for i in range(S.STEPS)], timestep_dtype=str(runs[0]["timesteps"][0].dtype),
                   all_timesteps=runs[0]["all_timesteps"], dt=[cat("dt", i).tolist() for i in range(S.STEPS)],
                   dt_dtype=str(runs[0]["dt"][0].dtype), out_dtype=str(runs[0]["out"].dtype))
        doc["cases"][name] = rec
        arrays[name] = torch.stack([cat("zs", i) for i in range(S.STEPS + 1)]).numpy().astype(np.float32)
        print(name, rec["all_timesteps"][:3], rec["dt"][0], rec["dt"][-1], rec["timestep_dtype"], rec["dt_dtype"], rec["out_dtype"])
    np.savez_compressed(os.path.join(HERE, "opensora_rflow.npz"), **arrays)
    with open(os.path.join(HERE, "opensora_rflow.json"), "w") as f:
        json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
