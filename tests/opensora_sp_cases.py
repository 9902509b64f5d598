"""The calls the sequence-parallel Open-Sora tests make, shared by the gloo CPU runs (tests/test_opensora_sp_cpu.py) and the GPU runs
(tests/test_opensora_sp_gpu.py): a sharded module (`enable_sequence_parallel`) and an unsharded twin built from the same weights
make the same calls; `compare` holds every rank's outputs, attributes and residual rows bit-equal to the twin's."""
import copy

import torch
import torch.distributed as dist

import magcache_b200 as mc
from magcache_b200 import patch as patch_mod
from magcache_b200.sampler import OpenSoraRFlowSampler

import opensora_ref as R

MAG_ATTRS = ("t", "accumulated_sim", "accumulated_err", "accumulated_steps", "skip_steps")
TEA_ATTRS = ("accumulated_rel_l1_distance",)


def build(kind, cfg="tiny", seed=0, thresh=None, device="cpu"):
    """kind: "magcache" (thresh / K as the slow preset unless given), "teacache" (rel_l1_thresh) or "plain" (enable_teacache False)."""
    base = R.STDiT3(**(R.CONFIGS[cfg] if isinstance(cfg, str) else cfg)).init_synthetic(seed)
    if kind != "magcache":
        with torch.no_grad():
            for n, p in base.named_parameters():
                if n.startswith("t_block."):
                    p.mul_(0.05)  # keeps the modulated input's step-to-step change in TeaCache's working range
    pair = []
    for tag in ("sp", "one"):
        m = copy.deepcopy(base).to(torch.bfloat16).to(device)
        m.__class__ = type(f"SP_{kind}_{tag}", (R.STDiT3,), {})
        if kind == "magcache":
            patch_mod.init_magcache_opensora(m, thresh=0.5 if thresh is None else thresh, K=3, skip_time=2)
        else:
            patch_mod.init_teacache_opensora(m, rel_l1_thresh=0.1 if thresh is None else thresh)
            if kind == "plain":
                m.__class__.enable_teacache = False
        pair.append(m)
    return pair


def video(B, T, Hx, Wx, L=12, cy=64, seed=0, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, T, Hx, Wx, generator=g)
    d = torch.randn(B, 4, T, Hx, Wx, generator=g)
    y = torch.randn(B, 1, L, cy, generator=g).to(device)
    mask = torch.ones(B, L, dtype=torch.long)
    mask[-1, L // 2:] = 0
    kw = dict(mask=mask.to(device), fps=torch.tensor([24.0], device=device), height=torch.tensor([8.0 * Hx], device=device),
              width=torch.tensor([8.0 * Wx], device=device))
    return (lambda i: (x + 0.004 * i * d).to(device)), y, kw


def timesteps(n, B, device):
    ts = [torch.full((B,), 1000.0 - 31.5 * i, device=device) for i in range(n)]
    return ts, [int(t[0].to(torch.bfloat16).item()) for t in ts]


def calls(model, kind, n, B, T, Hx, Wx, device, seed=0, cy=64):
    """n calls of the patched forward; per call (output, attributes, residual rows as the module exposes them)."""
    lat, y, kw = video(B, T, Hx, Wx, cy=cy, seed=seed, device=device)
    ts, all_ts = timesteps(n, B, device)
    names = MAG_ATTRS if kind == "magcache" else TEA_ATTRS
    rec = []
    with torch.no_grad():
        for i in range(n):
            o = model(lat(i), ts[i], all_ts, y, **kw)
            res = model.residual_cache[..., -1] if kind == "magcache" else model.previous_residual
            rec.append((o.clone(), {a: float(getattr(model, a)) for a in names},
                        None if res is None else res.reshape(B, -1, res.shape[-1]).clone()))
    return rec


def sample(model, T, Hx, Wx, device, seed=0, L=12, cy=64):
    """A 30-step OpenSoraRFlowSampler video (the fused step), with the latent entering each step recorded."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(1, 4, T, Hx, Wx, generator=g).to(torch.bfloat16)
    y = torch.randn(1, 1, L, cy, generator=g)
    y_null = torch.randn(1, 1, L, cy, generator=g)
    bf = dict(dtype=torch.bfloat16, device=device)
    args = dict(y=y.to(device), mask=torch.ones(1, L, dtype=torch.long, device=device), fps=torch.tensor([24], **bf),
                height=torch.tensor([480], **bf), width=torch.tensor([854], **bf), num_frames=torch.tensor([51], **bf))
    seen = []
    hook = model.register_forward_hook(lambda mod, a, out: seen.append(a[0][:1].float().clone()))
    try:
        with torch.no_grad():
            out = OpenSoraRFlowSampler().sample(model, z.to(device), args, y_null.to(device), device, progress=False)
    finally:
        hook.remove()
    return seen, out


def compare(got, want, T, t0, t1, what, group=None):
    """Sharded rank's records against the unsharded twin's: whole outputs and attributes bit-equal, residuals equal to the twin's rows of
    this rank's frames; attributes the same on every rank."""
    assert len(got) == len(want), what
    for i, ((o, a, r), (o1, a1, r1)) in enumerate(zip(got, want)):
        assert o.shape == o1.shape and o.dtype == o1.dtype, (what, i)
        assert torch.equal(o, o1), (what, i, float((o.double() - o1.double()).abs().max()))
        assert a == a1, (what, i, a, a1)
        if r1 is not None:
            B, C = r1.shape[0], r1.shape[-1]
            assert torch.equal(r, r1.view(B, T, -1, C)[:, t0:t1].reshape(B, -1, C)), (what, i)
    if dist.is_initialized():
        every = [None] * dist.get_world_size(group)
        dist.all_gather_object(every, [a for _, a, _ in got], group=group)
        assert all(e == every[0] for e in every), what


def enable(model, rank, world, group=None):
    return mc.enable_sequence_parallel(model, rank, world, group)
