"""build.py holds the 176-key attention kernel to the same no-spill, no-serialised-wgmma rule as the other widths."""
import importlib.util
import os

import pytest

_spec = importlib.util.spec_from_file_location(
    "mc_build", os.path.join(os.path.dirname(__file__), "..", "magcache_b200", "build.py"))
build = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(build)

ATTN176 = "_ZN2mc11attn_kernelILi176ELj0EEEv14CUtensorMap_stS1_S1_NS_10AttnParamsE"


def entry(name, spill):
    return (f"ptxas info    : Compiling entry function '{name}' for 'sm_90a'\n"
            f"ptxas info    : Function properties for {name}\n"
            f"    0 bytes stack frame, {spill} bytes spill stores, {spill} bytes spill loads\n"
            f"ptxas info    : Used 168 registers, used 16 barriers\n")


def test_wide_tile_clean_log_passes():
    build._check_ptxas(entry(ATTN176, 0))


def test_wide_tile_spill_is_rejected():
    with pytest.raises(RuntimeError, match="spill"):
        build._check_ptxas(entry(ATTN176, 176))


@pytest.mark.parametrize("code", ["C7510", "C7512"])
def test_wide_tile_serialised_wgmma_is_rejected(code):
    log = (f"ptxas info    : ({code}) Potential Performance Loss: wgmma.mma_async instructions are serialized for the function "
           f"'{ATTN176}'\n" + entry(ATTN176, 0))
    with pytest.raises(RuntimeError, match=code):
        build._check_ptxas(log)


def test_built_log_has_every_attn_width_without_spills():
    """When the library has been built here, its ptxas log lists all six attn_kernel instantiations, each with 0 spill bytes."""
    log_path = os.path.join(os.path.dirname(build.LIB), "build", "ptxas.log")
    if not os.path.exists(log_path):
        pytest.skip("library not built in this tree")
    with open(log_path) as f:
        log = f.read()
    import re
    props = re.findall(r"Function properties for (_ZN2mc11attn_kernelILi(\d+)E\S+)\n\s+\d+ bytes stack frame, (\d+) bytes spill stores", log)
    assert sorted({int(w) for _, w, _ in props}) == [64, 128, 176], props
    assert len(props) == 6 and all(s == "0" for _, _, s in props), props
