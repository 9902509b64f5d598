"""The tail of a DPM++ 2M step whose two calls both hit the cache, at the benchmarked latent (16 x 21 x 60 x 104: 32 760 tokens of
dim 1536, Wan2.1-1.3B), fused against unfused:
  fused:   head(hit, cond); mc_head_unpatchify_step_hist(hit, uncond)      (CFG combine + DPM++ update + x0 in the head's epilogue)
  unfused: head(hit, cond); head(hit, uncond) -> y; mc_cfg_step(cond, y, hist = [m1], x0_out = m0)
The rest of a hit forward (patch embedding, time MLP, head preparation) is the same launch sequence in both forms and is left out.
The flow-Euler step (mc_head_unpatchify_step against head + mc_cfg_step) is timed alongside for comparison. Each form runs `--steps`
steps back to back between two CUDA events, the forms alternating over `--rounds` rounds after a warm-up of each; the latent is
updated in place and the two x0 buffers swap every step, as FlowDPMSolverSampler does. One step of each form from the same inputs
is compared bit for bit first. By arithmetic the fused form saves the unconditional prediction's write and
re-read (2 x 16 x 21 x 120 x 208 x 4 B = 16.8 MB) and one launch per step: about 5 us at the data sheet's 3.35 TB/s. The card,
power limit and SM clocks are read in the same run. Prints one JSON line (and writes it to --out).

    python tools/bench_dpm_step.py [--steps 50] [--rounds 10] [--out bench_out/bench_dpm_step.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _smi():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dpm_step: needs a CUDA device")
    from magcache_b200 import ops
    from magcache_b200.sampler import FlowDPMSolverSampler, sampling_sigmas
    dev = torch.device("cuda")
    F, Hp, Wp, D = 21, 30, 52, 1536
    rows, shape = F * Hp * Wp, (16, F, 2 * Hp, 2 * Wp)
    g = torch.Generator(device=dev).manual_seed(0)
    x0 = torch.randn(rows, D, generator=g, device=dev).to(torch.bfloat16)  # the patch embedding a hit reads
    res = [0.1 * torch.randn(rows, D, generator=g, device=dev) for _ in range(2)]  # the cached residual of each CFG branch
    hm = 0.3 * torch.randn(2, D, generator=g, device=dev)
    e = 0.3 * torch.randn(D, generator=g, device=dev)
    W = 0.05 * torch.randn(D, 64, generator=g, device=dev)
    b = 0.1 * torch.randn(64, generator=g, device=dev)
    prep = ops.head_prepare(hm, e, W, b)
    grid = (F, Hp, Wp)
    smp = FlowDPMSolverSampler(sampling_sigmas(50, 5.0))
    cx, cv, ch = smp.coeffs(20)
    sig, gs = smp.sigmas[20], 5.0
    lat0 = torch.randn(shape, generator=g, device=dev)
    m1_0 = torch.randn(shape, generator=g, device=dev)

    def head(slot, **kw):
        return ops.head_unpatchify(x0, hm, e, W, b, grid, residual=res[slot], prep=prep, **kw)

    d_euler = smp.sigmas[21] - smp.sigmas[20]

    class Form:
        def __init__(self, fused, euler=False):
            self.fused, self.euler = fused, euler
            self.x = lat0.clone()
            self.m = [m1_0.clone(), torch.empty_like(lat0)]
            self.cond, self.y = torch.empty_like(lat0), torch.empty_like(lat0)

        def step(self):
            m1, m0 = self.m
            head(0, out=self.cond)
            if self.euler:  # the flow-Euler step of the same shape (mc_head_unpatchify_step / head + mc_cfg_step), for comparison
                if self.fused:
                    head(1, out=self.x, step=(self.cond, self.x, gs, 1.0, d_euler))
                else:
                    head(1, out=self.y)
                    ops.cfg_step(self.cond, self.y, gs, self.x, d_euler, out=self.x)
            elif self.fused:
                head(1, out=self.x, step=(self.cond, self.x, gs, cx, cv), step_hist=(m1, ch, sig, m0))
            else:
                head(1, out=self.y)
                ops.cfg_step(self.cond, self.y, gs, self.x, cv, coef_x=cx, hist=[m1], coef_h=[ch], sigma=sig, out=self.x, x0_out=m0)
            self.m.reverse()

    fused, unfused, e_fused, e_unfused = Form(True), Form(False), Form(True, True), Form(False, True)
    for form in (fused, unfused, e_fused, e_unfused):
        form.step()
    torch.cuda.synchronize()
    bit_equal = torch.equal(fused.x, unfused.x) and torch.equal(fused.m[0], unfused.m[0]) and torch.equal(e_fused.x, e_unfused.x)
    names = {id(fused): "fused", id(unfused): "unfused", id(e_fused): "euler_fused", id(e_unfused): "euler_unfused"}

    def batch(form):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            form.step()
        e1.record()
        e1.synchronize()
        return 1e3 * e0.elapsed_time(e1) / a.steps  # us per step

    forms = [fused, unfused, e_fused, e_unfused]
    for form in forms:  # warm-up
        batch(form)
    us = {n: [] for n in names.values()}
    for r in range(a.rounds):
        for form in (forms if r % 2 == 0 else forms[::-1]):
            us[names[id(form)]].append(batch(form))
    med = {k: statistics.median(v) for k, v in us.items()}
    saved_bytes = 2 * 16 * F * 2 * Hp * 2 * Wp * 4
    res_json = {
        "what": "DPM++ 2M hit-step tail (two hit heads [+ mc_cfg_step]) at 16x21x60x104, dim 1536",
        "gpu": _smi(), "device": torch.cuda.get_device_name(0), "steps_per_batch": a.steps, "rounds": a.rounds,
        "bit_equal": bool(bit_equal),
        "us_per_step_median": {k: round(v, 2) for k, v in med.items()},
        "us_per_step_min": {k: round(min(v), 2) for k, v in us.items()},
        "us_per_step_rounds": {k: [round(x, 2) for x in v] for k, v in us.items()},
        "saved_us_median": round(med["unfused"] - med["fused"], 2),
        "euler_saved_us_median": round(med["euler_unfused"] - med["euler_fused"], 2),
        "saved_bytes_by_arithmetic": saved_bytes,
        "saved_us_at_datasheet_hbm": round(saved_bytes / 3.35e12 * 1e6, 2),
    }
    line = json.dumps(res_json)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    if not bit_equal:
        raise SystemExit("bench_dpm_step: the fused and unfused steps differ")


if __name__ == "__main__":
    main()
