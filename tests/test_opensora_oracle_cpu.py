"""The Open-Sora restatement (tests/opensora_ref.py) against fixtures produced by executing the reference's own code
(tests/golden/make_opensora_golden.py: STDiT3 and its modules from videosys, `magcache_forward` and the `eval_ours` attributes from
eval/magcache/experiments/opensora.py): a tiny STDiT3 over the 30 calls of one video at B = 2 with distinct per-sample timesteps,
in fp32 and bf16, plus the controller attributes after every call and the skip masks of both paper presets."""
import contextlib
import io
import json
import os

import numpy as np
import pytest
import torch

import magcache_b200 as mc

import opensora_ref as R

GOLD = os.path.join(os.path.dirname(__file__), "golden")
DOC = json.load(open(os.path.join(GOLD, "opensora_forward.json")))
ARR = np.load(os.path.join(GOLD, "opensora_forward.npz"))
PAPER = json.load(open(os.path.join(GOLD, "paper_eval_adapters.json")))
ATTRS = ("t", "accumulated_sim", "accumulated_err", "accumulated_steps", "skip_steps")


def _model(dtype):
    m = R.STDiT3(**DOC["config"]).init_synthetic(DOC["seed"]).to(dtype).eval()
    m.__class__ = type(f"Oracle_{dtype}", (R.STDiT3,), {})
    R.install_magcache(m.__class__, thresh=0.12, K=3, skip_time=6)
    return m


def _inputs():
    B, T, H, W, cfg = DOC["B"], DOC["T"], DOC["H"], DOC["W"], DOC["config"]
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, 4, T, H, W, generator=g)
    y = torch.randn(B, 1, cfg["model_max_length"], cfg["caption_channels"], generator=g)
    mask = torch.ones(B, cfg["model_max_length"], dtype=torch.long)
    return x, y, dict(mask=mask, fps=torch.tensor([24.0]), height=torch.tensor([8.0 * H]), width=torch.tensor([8.0 * W]))


def test_weights_match_the_fixture_checksums():
    m = R.STDiT3(**DOC["config"]).init_synthetic(DOC["seed"])
    params = dict(m.named_parameters())
    assert sorted(params) == sorted(DOC["checksums"])
    for n, (s, a) in DOC["checksums"].items():
        t = params[n].detach().double()
        assert float(t.sum()) == s and float(t.abs().sum()) == a, n


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_oracle_matches_reference_execution(dtype):
    m = _model(torch.float32 if dtype == "fp32" else torch.bfloat16)
    x, y, kw = _inputs()
    gold = ARR[dtype]
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        for i in range(30):
            out = m(x, torch.tensor(DOC["timesteps"][i]), None, y, **kw).numpy()
            if dtype == "fp32":
                err = np.linalg.norm(out.astype(np.float64) - gold[i]) / np.linalg.norm(gold[i])
                assert err <= 1e-6, (i, err)
            else:
                assert np.array_equal(out, gold[i]), (i, np.abs(out - gold[i]).max())
            for a in ATTRS:
                assert float(getattr(m, a)) == DOC[f"attrs_{dtype}"][i][a], (i, a)
    assert [int(v) for v in DOC[f"mask_{dtype}"]] == DOC["mask_fp32"]


def test_preset_masks_match_the_golden_schedules():
    osr = {(c["thresh"], c["K"], c["skip_time"]): [int(v) for v in c["mask"][:30]] for c in PAPER["opensora_masks"]}
    assert DOC["mask_fp32"] == osr[(0.12, 3, 6)] == [int(v) for v in mc.PRESETS["opensora-slow-E012K3"].schedule()]
    assert DOC["mask_fast"] == osr[(0.24, 5, 6)] == [int(v) for v in mc.PRESETS["opensora-fast-E024K5"].schedule()]
