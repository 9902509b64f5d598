"""FLUX ControlNet residuals for the tests: the reference's statements around the oracle's blocks, and the kernel's epilogue 8 in torch.

`controlnet_blocks` makes the oracle's patched forward (oracle/flux_ref.py) run the reference's ControlNet statements after each
block — MagCache4FLUX/magcache_flux.py:374-384 (double blocks) and :416-423 (single blocks); the calibration twin's are :145-155 and
:187-193, and MagCache4FLUX_Kontext/magcache_flux_kontext.py:147-157, :189-195, :376-386, :418-424 are the same lines. The oracle
calls `self.transformer_blocks` / `self.single_transformer_blocks` only on the miss branch and in the calibration twin, where the
reference has them, so wrapping the blocks adds the samples exactly where the reference does.

`emu` is tests/emu_ops.py with `gemm` taking the addend of MC_EPI_BIAS_GATE_RESID_ADD_BF16 (include/magcache_b200.h)."""
import contextlib
import types

import numpy as np
import torch
from torch import nn

import emu_ops
from magcache_b200 import _lib as L


class _DoubleThenAdd(nn.Module):
    def __init__(self, block, sample):
        super().__init__()
        self.block, self.sample = block, sample

    def forward(self, hidden_states, encoder_hidden_states, temb, image_rotary_emb=None, joint_attention_kwargs=None):
        encoder_hidden_states, hidden_states = self.block(hidden_states=hidden_states, encoder_hidden_states=encoder_hidden_states, temb=temb,
                                                          image_rotary_emb=image_rotary_emb)
        if self.sample is not None:
            hidden_states = hidden_states + self.sample                                            # :382-384
        return encoder_hidden_states, hidden_states


class _SingleThenAdd(nn.Module):
    def __init__(self, block, sample, n_txt):
        super().__init__()
        self.block, self.sample, self.n_txt = block, sample, n_txt

    def forward(self, hidden_states, temb, image_rotary_emb=None, joint_attention_kwargs=None):
        hidden_states = self.block(hidden_states=hidden_states, temb=temb, image_rotary_emb=image_rotary_emb)
        if self.sample is not None:                                                                # :420-423
            hidden_states[:, self.n_txt:, ...] = hidden_states[:, self.n_txt:, ...] + self.sample
        return hidden_states


def reference_samples(n_blocks, samples, repeat):
    """The sample each block adds (None without samples): magcache_flux.py:376-384 (`repeat`: XLabs) and :418-423 (never repeats)."""
    if samples is None:
        return [None] * n_blocks
    interval_control = n_blocks / len(samples)
    interval_control = int(np.ceil(interval_control))
    return [samples[i % len(samples)] if repeat else samples[i // interval_control] for i in range(n_blocks)]


@contextlib.contextmanager
def controlnet_blocks(model, block_samples, single_samples, n_txt, repeat=False):
    """Within the block, `model`'s oracle forward adds the ControlNet samples after its blocks as the reference does."""
    double, single = model.transformer_blocks, model.single_transformer_blocks
    model.transformer_blocks = nn.ModuleList(
        [_DoubleThenAdd(b, s) for b, s in zip(double, reference_samples(len(double), block_samples, repeat))])
    model.single_transformer_blocks = nn.ModuleList(
        [_SingleThenAdd(b, s, n_txt) for b, s in zip(single, reference_samples(len(single), single_samples, False))])
    try:
        yield model
    finally:
        model.transformer_blocks, model.single_transformer_blocks = double, single


def gemm(a, b, bias=None, epilogue=L.MC_EPI_BIAS_BF16, out=None, gate=None, tag=None, addend=None, addend_row0=0):
    """emu_ops.gemm; with an addend, MC_EPI_BIAS_GATE_RESID_ADD_BF16: epilogue 6, then out[m] = bf16(out[m] + addend[m - row0]) for
    m >= row0 (rows below are epilogue 6's)."""
    if addend is None:
        return emu_ops.gemm(a, b, bias, epilogue, out=out, gate=gate, tag=tag)
    assert epilogue == L.MC_EPI_BIAS_GATE_RESID_BF16 and out is not None
    assert addend.dtype == torch.bfloat16 and addend.stride(1) == 1 and addend.shape == (out.shape[0] - addend_row0, out.shape[1])
    emu_ops.gemm(a, b, bias, epilogue, out=out, gate=gate, tag=tag)
    out[addend_row0:] = (out[addend_row0:].float() + addend.float()).bfloat16()
    return out


emu = types.ModuleType("emu_ops_controlnet")
emu.__dict__.update({k: v for k, v in vars(emu_ops).items() if not k.startswith("__")})
emu.gemm = gemm
