"""A deterministic stand-in for STDiT3 behind the Open-Sora sampler fixture (tests/golden/make_opensora_rflow_golden.py) and its tests:
the model's call signature `(x, timestep, all_timesteps, y, **model_args)` and output layout ([2B, 8, T, H, W] fp32, velocity in
channels 0-3), no weights. The conditional and unconditional halves differ through `y`."""
import types

import torch

# the pipeline's model_args (prepare_multi_resolution_info: height / width / num_frames as bf16 tensors repeated over the batch)
RESOLUTIONS = {"480p": (480, 854), "720p": (720, 1280)}
CASES = {  # name -> (resolution, num_frames, cfg_scale, use_discrete_timesteps, use_timestep_transform, B)
    "480p_51_cfg7_B1": ("480p", 51, 7.0, False, True, 1),
    "480p_102_cfg4.5_discrete_B2": ("480p", 102, 4.5, True, True, 2),
    "480p_408_cfg7_discrete_B1": ("480p", 408, 7.0, True, True, 1),
    "720p_51_cfg4.5_B2": ("720p", 51, 4.5, False, True, 2),
    "720p_102_cfg7_B1": ("720p", 102, 7.0, False, True, 1),
    "720p_408_cfg4.5_B2": ("720p", 408, 4.5, False, True, 2),
    "480p_51_cfg7_linear_B2": ("480p", 51, 7.0, False, False, 2),
    "720p_51_cfg4.5_linear_discrete_B1": ("720p", 51, 4.5, True, False, 1),
}
STEPS = 30
LATENT = (4, 2, 3, 5)  # C, T, H, W: odd H / W like a cropped latent


class StubSTDiT3:
    def __init__(self):
        self.x_embedder = types.SimpleNamespace(proj=types.SimpleNamespace(weight=torch.zeros(1, dtype=torch.bfloat16)))
        self.calls = []  # (x, timestep, all_timesteps) of every call

    def __call__(self, x, timestep, all_timesteps, y, **kw):
        self.calls.append((x.clone(), timestep.clone(), list(all_timesteps)))
        s = y.float().mean(dim=(1, 2, 3)).view(-1, 1, 1, 1, 1)
        base = torch.cat([x, torch.cos(x)], 1).float()
        return torch.tanh(base * (1 + s)) - 0.0005 * timestep.float().view(-1, 1, 1, 1, 1) * base


def case_inputs(name, seed=0):
    """(z bf16 [B, 4, T, H, W] like the pipeline's `torch.randn(..., dtype=self._dtype)`, model_args, y_null) of one case."""
    res, frames, _, _, _, B = CASES[name]
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, *LATENT, generator=g).to(torch.bfloat16)
    y = torch.randn(B, 1, 6, 8, generator=g)
    y_null = torch.randn(B, 1, 6, 8, generator=g) + 0.5
    h, w = RESOLUTIONS[res]
    bf = dict(dtype=torch.bfloat16)
    model_args = dict(y=y, height=torch.tensor([h], **bf).repeat(B), width=torch.tensor([w], **bf).repeat(B),
                      num_frames=torch.tensor([frames], **bf).repeat(B), fps=torch.tensor([24], **bf).repeat(B))
    return z, model_args, y_null


def scheduler_kwargs(name):
    _, _, cfg, discrete, transform, _ = CASES[name]
    return dict(num_sampling_steps=STEPS, cfg_scale=cfg, num_timesteps=1000, use_timestep_transform=transform,
                use_discrete_timesteps=discrete)
