"""Restatement of Open-Sora's TeaCache forward (`teacache_forward`, eval/magcache/experiments/opensora.py:34-227, sp = cp = 1,
x_mask = None) and of its installation (`eval_teacache_slow` / `_fast`, :383-409) on tests/opensora_ref.py's STDiT3, the CPU
emulation of the fused decision-input kernel (`mc_ln_t2i_modulate_rel_l1`), and the input schedule of the TeaCache fixture
(tests/golden/opensora_teacache.{npz,json}, written by tests/golden/make_opensora_teacache_golden.py)."""
import numpy as np
import torch

import opensora_emu
import opensora_ref as R

COEFFICIENTS = [2.17546007e+02, -1.18329252e+02, 2.68662585e+01, -4.59364272e-02, 4.84426240e-02]  # :100


def teacache_forward(self, x, timestep, all_timesteps, y, mask=None, x_mask=None, fps=None, height=None, width=None, **kwargs):
    """:34-227. Records `last_forced`, `last_rel` (the value the polynomial saw, None when forced) and `last_calc`."""
    x, y, y_lens, t, t_mlp, (T, H, W, S), (Tx, Hx, Wx) = self.embed(x, timestep, y, mask, fps, height, width)
    timestep = timestep.to(self.x_embedder.proj.weight.dtype)  # :51
    should_calc, rel, forced = True, None, False
    if self.enable_teacache:
        inp = x.clone()
        B = inp.shape[0]
        shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = (
            self.spatial_blocks[0].scale_shift_table[None] + t_mlp.reshape(B, 6, -1)).chunk(6, dim=1)
        modulated_inp = R.t2i_modulate(self.spatial_blocks[0].norm1(inp), shift_msa, scale_msa)
        if timestep[0] == all_timesteps[0] or timestep[0] == all_timesteps[-1]:
            forced = True
            should_calc = True
            self.accumulated_rel_l1_distance = 0
        else:
            rescale_func = np.poly1d(COEFFICIENTS)
            rel = ((modulated_inp - self.previous_modulated_input).abs().mean() / self.previous_modulated_input.abs().mean()).cpu().item()
            self.accumulated_rel_l1_distance += rescale_func(rel)
            if self.accumulated_rel_l1_distance < self.rel_l1_thresh:
                should_calc = False
            else:
                should_calc = True
                self.accumulated_rel_l1_distance = 0
        leader = getattr(self, "decisions_from", None)  # the fp64 yardstick takes the decisions of the bf16 run it measures
        if leader is not None:
            should_calc = leader.last_calc
        self.previous_modulated_input = modulated_inp
        if not should_calc:
            x += self.previous_residual
        else:
            origin_x = x.clone().detach()
            x = self.blocks(x, y, t_mlp, y_lens, T, S)
            self.previous_residual = x - origin_x
    else:
        x = self.blocks(x, y, t_mlp, y_lens, T, S)
    self.last_forced, self.last_rel, self.last_calc = forced, rel, should_calc
    return self.head(x, t, T, H, W, Tx, Hx, Wx)


def opensora_rel_bf16(v):
    """A float rounded to bf16, as `.item()` of a bf16 scalar returns it."""
    return torch.tensor(float(v), dtype=torch.float32).to(torch.bfloat16).item()


def install_teacache(cls, rel_l1_thresh=0.1, enable=True):
    """The attribute block of `eval_teacache_slow` (0.1) / `eval_teacache_fast` (0.2) on a class."""
    cls.enable_teacache = enable
    cls.rel_l1_thresh = rel_l1_thresh
    cls.accumulated_rel_l1_distance = 0
    cls.previous_modulated_input = None
    cls.previous_residual = None
    cls.forward = teacache_forward
    return cls


# ---- the fused decision-input kernel, emulated --------------------------------------------------------------------------------
def ln_t2i_modulate_rel_l1(x, em, scale_idx, shift_idx, prev, out, partials, sums, eps=1e-6, tag=None):
    """`mc_ln_t2i_modulate_rel_l1`: mode-2 output into `out`, sums += (sum |bf16(out - prev)|, sum |prev|) in fp64."""
    o = opensora_emu.ln_t2i_modulate(x, em, scale_idx, shift_idx, eps)
    out.copy_(o)
    d = opensora_emu._rb(o.float() - prev.float()).abs().double().sum()
    sums[0] += d
    sums[1] += prev.float().abs().double().sum()
    return out


def rel_l1_partials(device):
    return torch.empty(2 * 4096, dtype=torch.float64)


def namespace():
    """opensora_emu.namespace() with the fused TeaCache op: a drop-in for `magcache_b200.opensora.ops`."""
    ns = opensora_emu.namespace()
    ns.ln_t2i_modulate_rel_l1 = ln_t2i_modulate_rel_l1
    ns.rel_l1_partials = rel_l1_partials
    return ns


# ---- the fixture's inputs -----------------------------------------------------------------------------------------------------
def video_inputs(doc):
    """(latents(i), y, kw) of the fixture: latents(i) = x + step * i * d, so the input moves between calls independently of the
    outputs, and every restatement or engine run sees the same inputs."""
    B, T, H, W, cfg = doc["B"], doc["T"], doc["H"], doc["W"], doc["config"]
    g = torch.Generator().manual_seed(doc["input_seed"])
    x = torch.randn(B, 4, T, H, W, generator=g)
    d = torch.randn(B, 4, T, H, W, generator=g)
    y = torch.randn(B, 1, cfg["model_max_length"], cfg["caption_channels"], generator=g)
    mask = torch.ones(B, cfg["model_max_length"], dtype=torch.long)
    kw = dict(mask=mask, fps=torch.tensor([24.0]), height=torch.tensor([float(doc["height"])]), width=torch.tensor([float(doc["width"])]))
    step = doc["latent_step"]
    return (lambda i: x + step * i * d), y, kw


def timestep_tensor(sched, i):
    """The sampler's `t` of call i (`torch.cat([t, t], 0)` of the CFG pair, scheduling_rflow_open_sora.py:239)."""
    return torch.tensor(sched["timesteps"][i], dtype=torch.int64 if sched["discrete"] else torch.float32)
