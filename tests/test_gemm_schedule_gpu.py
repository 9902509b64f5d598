"""GPU checks of the wgmma GEMM's tile schedule (clusters of 2 CTAs along M walking 256-row tiles, 128 rows per CTA, 64 per
consumer warpgroup, the B tile multicast over the cluster), beyond the fp64 tolerance tests of test_kernels_gpu.py:

* placement invariance, bit for bit: the rows of a tile must not depend on which CTA of a cluster, which warpgroup or which
  step of the persistent walk computed them, so the GEMM of A[r0:r1] equals rows r0:r1 of the full GEMM exactly;
* shape edges of the cluster walk (odd numbers of 64- and 128-row tiles, a cluster partner without rows, tile counts around the grid,
  a single k-block), against fp64 with the criteria of test_kernels_gpu.py;
* determinism of a full-size launch.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ops():
    from magcache_b200 import ops
    return ops


def _lib():
    from magcache_b200 import _lib
    return _lib


def _gemm_ref(a, b):
    return a.double() @ b.double().t()


def _bf16_bad(got, ref_f32):
    """Elements of a bf16 output further than one bf16 ulp (plus the fp32 accumulation noise) from the fp64 reference."""
    tol = ref_f32.abs() * (2.0 ** -7) + 1e-4
    return int(((got.float() - ref_f32).abs() > tol).sum().item())


def _epilogues():
    L = _lib()
    return {"bias_bf16": L.MC_EPI_BIAS_BF16, "gelu_tanh": L.MC_EPI_BIAS_GELU_BF16, "gate_resid_f32": L.MC_EPI_BIAS_GATE_RESID,
            "rowbias_bf16": L.MC_EPI_ROWBIAS_BF16, "bias_f32": L.MC_EPI_BIAS_F32, "gelu_erf": L.MC_EPI_BIAS_GELU_ERF_BF16,
            "gate_resid_bf16": L.MC_EPI_BIAS_GATE_RESID_BF16, "silu": L.MC_EPI_BIAS_SILU_BF16}


def _run(epi_name, a, b, bias, gate, stream0):
    """One GEMM with the named epilogue; the residual epilogues update a copy of `stream0` (rows matching a) in place."""
    ops, L = _ops(), _lib()
    epi = _epilogues()[epi_name]
    if epi in (L.MC_EPI_BIAS_GATE_RESID, L.MC_EPI_BIAS_GATE_RESID_BF16):
        out = stream0.clone()
        ops.gemm(a, b, bias, epi, out=out, gate=gate)
        return out
    return ops.gemm(a, b, bias, epi)


@pytest.mark.parametrize("epi_name", ["bias_bf16", "gelu_tanh", "gate_resid_f32", "rowbias_bf16", "bias_f32", "gelu_erf",
                                      "gate_resid_bf16", "silu"])
@pytest.mark.parametrize("bn", [128, 256])
def test_gemm_rows_do_not_depend_on_placement(epi_name, bn, monkeypatch):
    monkeypatch.setenv("MC_GEMM_BN", str(bn))
    M, N, K = 1000, 640, 512
    a = torch.randn(M, K, device=DEV).bfloat16()
    b = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    bias_n = torch.randn(N, device=DEV)
    bias_m = torch.randn(M, device=DEV)  # the row-bias epilogue indexes its bias by output row
    gate = torch.randn(N, device=DEV) * 0.5
    resid_bf16 = epi_name == "gate_resid_bf16"
    stream = torch.randn(M, N, device=DEV)
    if resid_bf16:
        stream = stream.bfloat16()
    rowbias = epi_name == "rowbias_bf16"
    full = _run(epi_name, a, b, bias_m if rowbias else bias_n, gate, stream)
    # starts at odd multiples of 64 and 128 (the other warpgroup / the other CTA of a cluster than in the full launch), off
    # any tile boundary, a single row, and a range of fewer than 64 rows
    for r0, r1 in [(64, 192), (128, 1000), (192, 1000), (384, 700), (37, 600), (1, 65), (448, 449), (960, 1000)]:
        part = _run(epi_name, a[r0:r1], b, bias_m[r0:r1] if rowbias else bias_n, gate, stream[r0:r1])
        assert torch.equal(part, full[r0:r1]), (epi_name, bn, r0, r1)


@pytest.mark.parametrize("case", ["odd_row_tiles", "m_le_128", "partner_without_rows", "tiles_around_grid", "single_k_block"])
@pytest.mark.parametrize("bn", [128, 256])
def test_gemm_cluster_walk_shape_edges(case, bn, monkeypatch):
    ops, L = _ops(), _lib()
    monkeypatch.setenv("MC_GEMM_BN", str(bn))
    # shapes are (M, N, K); the walk counts 256-row cluster tiles x N tiles, and the grid holds at most SMs / 2 clusters
    g = torch.cuda.get_device_properties(0).multi_processor_count // 2
    shapes = {
        "odd_row_tiles": [(3 * 64 + 1, 384, 256), (5 * 64, 256, 128), (3 * 128 + 1, 384, 256), (5 * 128, 256, 128)],
        "m_le_128": [(1, 256, 128), (40, 640, 256), (64, 1536, 64), (100, 384, 128), (128, 256, 256)],
        "partner_without_rows": [(256 * 3 + 40, 512, 192), (256 * 2 + 128, 256, 128)],
        # one n tile of 256 (two of 128): cluster tile counts just below and above one and two waves of clusters
        "tiles_around_grid": [(256 * t - 50, 256, 128) for t in (g - 1, g + 1, 2 * g - 1, 2 * g + 1)],
        "single_k_block": [(3 * 64 + 1, 384, 64), (4095, 1536, 64)],
    }[case]
    for M, N, K in shapes:
        a = torch.randn(M, K, device=DEV).bfloat16()
        b = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
        bias = torch.randn(N, device=DEV).bfloat16().float()
        ref = (_gemm_ref(a, b) + bias.double()).float()
        out = ops.gemm(a, b, bias, L.MC_EPI_BIAS_BF16)
        assert _bf16_bad(out, ref) == 0, (case, M, N, K)
        out32 = ops.gemm(a, b, bias, L.MC_EPI_BIAS_F32)
        assert torch.allclose(out32, ref, rtol=1e-3, atol=1e-4), (case, M, N, K, float((out32 - ref).abs().max()))


@pytest.mark.parametrize("bn", [128, 256])
def test_gemm_inplace_stream_ragged_padded(bn, monkeypatch):
    """fp32 residual stream updated in place (o-projection / ffn2 epilogue) on a ragged shape with a padded row stride: every
    row and column inside M x N is updated once, the columns past N are left exactly as they were."""
    ops, L = _ops(), _lib()
    monkeypatch.setenv("MC_GEMM_BN", str(bn))
    M, N, K, pad = 3 * 128 + 1, 200, 320, 24
    a = torch.randn(M, K, device=DEV).bfloat16()
    b = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=DEV).bfloat16().float()
    gate = torch.randn(N, device=DEV) * 0.5
    buf = torch.randn(M, N + pad, device=DEV)
    before = buf.clone()
    acc = (_gemm_ref(a, b) + bias.double()).float()
    ops.gemm(a, b, bias, L.MC_EPI_BIAS_GATE_RESID, out=buf[:, :N], gate=gate)
    x_ref = before[:, :N] + acc.bfloat16().float() * gate
    assert ((buf[:, :N] - x_ref).abs() <= 1e-4 + gate.abs() * acc.abs() * 2 ** -7).all()
    assert torch.equal(buf[:, N:], before[:, N:])


def test_gemm_ffn2_shape_is_deterministic():
    """Two launches at the Wan2.1-1.3B ffn2 shape (32 760 x 1536 x 8960, gated fp32 residual) give bit-equal streams."""
    ops, L = _ops(), _lib()
    M, N, K = 32760, 1536, 8960
    a = torch.randn(M, K, device=DEV).bfloat16()
    b = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=DEV)
    gate = torch.randn(N, device=DEV)
    x0 = torch.randn(M, N, device=DEV)
    x1, x2 = x0.clone(), x0.clone()
    ops.gemm(a, b, bias, L.MC_EPI_BIAS_GATE_RESID, out=x1, gate=gate)
    ops.gemm(a, b, bias, L.MC_EPI_BIAS_GATE_RESID, out=x2, gate=gate)
    assert torch.equal(x1, x2)
    assert not torch.equal(x1, x0)
