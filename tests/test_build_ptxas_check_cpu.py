"""build.py rejects ptxas logs in which a tensor-core kernel lost its wgmma pipeline or spilled (no GPU, no nvcc needed)."""
import importlib.util
import os

import pytest

_spec = importlib.util.spec_from_file_location(
    "mc_build", os.path.join(os.path.dirname(__file__), "..", "magcache_b200", "build.py"))
build = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(build)

ATTN = "_ZN2mc11attn_kernelILi128ELj0EEEv14CUtensorMap_stS1_S1_NS_10AttnParamsE"
GEMM = "_ZN2mc16gemm_bf16_kernelILi2ELi256EEEv14CUtensorMap_stS1_NS_10GemmParamsE"
OTHER = "_ZN2mc22ln_modulate_tma_kernelILi8ELi2EEEvPKvilifiPKfS4_iiiPvii"


def entry(name, spill_stores, spill_loads=None):
    loads = spill_stores if spill_loads is None else spill_loads
    return (f"ptxas info    : Compiling entry function '{name}' for 'sm_90a'\n"
            f"ptxas info    : Function properties for {name}\n"
            f"    0 bytes stack frame, {spill_stores} bytes spill stores, {loads} bytes spill loads\n"
            f"ptxas info    : Used 168 registers, used 16 barriers\n")


def test_clean_log_passes():
    build._check_ptxas(entry(ATTN, 0) + entry(GEMM, 0) + entry(OTHER, 144))  # spills elsewhere are not this check's business


@pytest.mark.parametrize("code", ["C7510", "C7512"])
def test_serialised_wgmma_is_rejected(code):
    log = (f"ptxas info    : ({code}) Potential Performance Loss: wgmma.mma_async instructions are serialized for the function "
           f"'{ATTN}'\n" + entry(ATTN, 0))
    with pytest.raises(RuntimeError, match=code):
        build._check_ptxas(log)


@pytest.mark.parametrize("name", [ATTN, GEMM])
def test_spill_in_tensor_core_kernel_is_rejected(name):
    with pytest.raises(RuntimeError, match="spill"):
        build._check_ptxas(entry(OTHER, 0) + entry(name, 88, 112))
