"""CPU tests: the oracle and the product's host logic (C ABI) against the golden vectors produced from the reference's own
statements (tests/golden/make_golden.py). The skip mask is the bit-exact integer contract."""
import ctypes
import json
import os

import numpy as np
import pytest

from oracle.controller_ref import ControllerRef, interp_cfg, nearest_interp

G = os.path.join(os.path.dirname(__file__), "golden")


def load(name):
    with open(os.path.join(G, name)) as f:
        return json.load(f)


TABLES = load("tables.json")
MASKS = load("masks.json")
INTERP = load("nearest_interp.json")


def _src(case):
    if case["table"] is None:
        return np.array(case["src"])
    t = np.array(TABLES[case["table"]]["values"])
    return {"cond": t[0::2], "uncond": t[1::2], "all": t}[case["slice"]]


# ------------------------------------------------------------------------------------------------ oracle vs golden
@pytest.mark.parametrize("case", INTERP, ids=lambda c: f"{c['table']}-{c['slice']}-{c['L']}to{c['T']}")
def test_oracle_nearest_interp(case):
    out = nearest_interp(_src(case), case["T"])
    assert out.tolist() == case["out"]


def _table_for(case):
    t = np.array(TABLES[case["table"]]["values"])
    if case["family"] == "wan2.1":
        return interp_cfg(t, case["steps"]), case["steps"] * 2
    return (t if len(t) == case["steps"] else nearest_interp(t, case["steps"])), case["steps"]


@pytest.mark.parametrize("case", MASKS, ids=lambda c: f"{c['table']}-s{c['steps']}-E{c['thresh']}K{c['K']}R{c['R']}")
def test_oracle_mask(case):
    ratios, n = _table_for(case)
    ctl = ControllerRef(case["family"], ratios, n, case["thresh"], case["K"], case["R"])
    got = "".join(map(str, ctl.mask(case["calls"])))
    assert got == case["mask"]
    assert ctl.cnt == case["final"]["cnt"]


def test_survey_headline_masks():
    """SURVEY §8c: Wan-1.3B E012K4R02 skips 58/100, per-branch mask as published in BASELINE.md."""
    c = [m for m in MASKS if m["table"] == "wan2.1_t2v_1.3b" and m["steps"] == 50 and m["thresh"] == 0.12 and m["K"] == 4][0]
    assert c["skipped_first_video"] == 58
    assert c["mask"][0:100:2] == "00000000001111011110111101111011110111011011010100"
    assert c["mask"][0:100:2] == c["mask"][1:100:2]
    f = [m for m in MASKS if m["family"] == "flux" and m["steps"] == 28 and m["thresh"] == 0.24 and m["K"] == 5][0]
    assert f["skipped_first_video"] == 19 and f["mask"][:28] == "0001101110101111101111101101"


# ------------------------------------------------------------------------------------------------ C ABI vs golden
@pytest.fixture(scope="module")
def L():
    from magcache_b200 import _lib
    return _lib


def _cfg(L, family, ratios, n, thresh, K, R):
    arr = (ctypes.c_double * len(ratios))(*ratios)
    cfg = L.CtrlConfig()
    cfg.num_steps, cfg.K, cfg.thresh, cfg.retention_ratio = n, K, thresh, R
    cfg.branches = 2 if family == "wan2.1" else 1
    cfg.cmp = L.MC_CMP_LT if family == "wan2.1" else L.MC_CMP_LE
    cfg.retention_mode = L.MC_RETAIN_HALF_UP if family == "flux" else L.MC_RETAIN_FLOOR
    cfg.veto_index, cfg.veto_base = (11, 28) if family == "flux" else (-1, 0)
    cfg.mag_ratios = ctypes.cast(arr, ctypes.POINTER(ctypes.c_double))
    cfg._keep = arr
    return cfg


@pytest.mark.parametrize("case", INTERP, ids=lambda c: f"{c['table']}-{c['slice']}-{c['L']}to{c['T']}")
def test_cabi_nearest_interp(L, case):
    src = _src(case)
    a = (ctypes.c_double * len(src))(*src)
    out = (ctypes.c_double * case["T"])()
    L.check(L.lib.mc_nearest_interp(a, len(src), out, case["T"]))
    assert list(out) == case["out"]


@pytest.mark.parametrize("case", MASKS, ids=lambda c: f"{c['table']}-s{c['steps']}-E{c['thresh']}K{c['K']}R{c['R']}")
def test_cabi_mask_and_stepwise_state(L, case):
    t = TABLES[case["table"]]["values"]
    steps = case["steps"]
    if case["family"] == "wan2.1":
        n = steps * 2
        if len(t) == n:
            ratios = list(t)
        else:
            src = (ctypes.c_double * len(t))(*t)
            dst = (ctypes.c_double * n)()
            L.check(L.lib.mc_nearest_interp_cfg(src, len(t), dst, steps))
            ratios = list(dst)
    else:
        n = steps
        ratios = list(t) if len(t) == n else nearest_interp(np.array(t), n).tolist()
    cfg = _cfg(L, case["family"], ratios, n, case["thresh"], case["K"], case["R"])
    mask = (ctypes.c_uint8 * case["calls"])()
    L.check(L.lib.mc_ctrl_mask(ctypes.byref(cfg), case["calls"], mask))
    assert "".join(str(int(v)) for v in mask) == case["mask"]
    # step-wise API (what the Python shim uses) reproduces the same decisions and the same final accumulator state
    st = L.CtrlState()
    st.accumulated_ratio[0] = st.accumulated_ratio[1] = 1.0
    skip = ctypes.c_int32()
    got = []
    for _ in range(case["calls"]):
        L.check(L.lib.mc_ctrl_decide(ctypes.byref(cfg), ctypes.byref(st), ctypes.byref(skip)))
        got.append(str(skip.value))
        L.check(L.lib.mc_ctrl_advance(ctypes.byref(cfg), ctypes.byref(st)))
    assert "".join(got) == case["mask"]
    fin = case["final"]
    assert st.cnt == fin["cnt"]
    nb = 2 if case["family"] == "wan2.1" else 1
    exp = {k: (fin[k] if isinstance(fin[k], list) else [fin[k]]) for k in ("accumulated_err", "accumulated_steps", "accumulated_ratio")}
    assert [st.accumulated_err[i] for i in range(nb)] == exp["accumulated_err"]          # float64, bit-exact
    assert [st.accumulated_ratio[i] for i in range(nb)] == exp["accumulated_ratio"]
    assert [float(st.accumulated_steps[i]) for i in range(nb)] == exp["accumulated_steps"]


def test_cabi_rejects_bad_configs(L):
    ratios = [1.0] * 10
    cfg = _cfg(L, "wan2.1", ratios, 10, 0.12, 2, 0.0)  # retention 0: reference would add None (Appendix A quirk 4)
    assert L.lib.mc_ctrl_validate(ctypes.byref(cfg)) == L.MC_ERR_STATE
    assert b"residual" in L.lib.mc_last_error()
    cfg = _cfg(L, "wan2.1", ratios, 10, 0.12, 2, 0.2)
    assert L.lib.mc_ctrl_validate(ctypes.byref(cfg)) == 0
    cfg.mag_ratios = ctypes.POINTER(ctypes.c_double)()
    assert L.lib.mc_ctrl_validate(ctypes.byref(cfg)) == L.MC_ERR_INVALID
    st = L.CtrlState()
    st.cnt = 99
    skip = ctypes.c_int32()
    cfg = _cfg(L, "wan2.1", ratios, 10, 0.12, 2, 0.2)
    assert L.lib.mc_ctrl_decide(ctypes.byref(cfg), ctypes.byref(st), ctypes.byref(skip)) == L.MC_ERR_STATE
    out = (ctypes.c_double * 1)()
    assert L.lib.mc_nearest_interp(None, 3, out, 1) == L.MC_ERR_INVALID


def test_oracle_c_restatement_matches(L):
    """The plain-C oracle (oracle/magcache_ref.c) agrees with the golden masks too (it is the cpu_baseline 'port')."""
    so = os.path.join(os.path.dirname(__file__), "..", "oracle", "_build", "libmagcache_ref.so")
    if not os.path.exists(so):
        pytest.skip("oracle/_build not built (python -c 'import __graft_entry__ as g; g.build()')")
    ref = ctypes.CDLL(so)
    fam = {"wan2.1": 0, "flux": 1, "hunyuan": 2}
    for case in MASKS[::7]:
        ratios, n = _table_for(case)
        arr = (ctypes.c_double * len(ratios))(*ratios)
        mask = (ctypes.c_uint8 * case["calls"])()
        ref.ref_ctrl_mask(fam[case["family"]], arr, n, ctypes.c_double(case["thresh"]), case["K"], ctypes.c_double(case["R"]), case["calls"], mask)
        assert "".join(str(int(v)) for v in mask) == case["mask"]


def test_handle_form_equals_the_struct_form(L):
    """mc_ctrl_create / step / reset / destroy (SURVEY §8b) against the golden schedules, plus table ownership and reset."""
    for case in [m for m in MASKS if m["steps"] in (50, 28)][:24]:
        t = TABLES[case["table"]]["values"]
        steps = case["steps"]
        if case["family"] == "wan2.1":
            n = steps * 2
            from magcache_b200.config import interp_cfg
            ratios = list(interp_cfg(np.array(t), steps))
        else:
            n = steps
            ratios = list(t)
        cfg = _cfg(L, case["family"], ratios, n, case["thresh"], case["K"], case["R"])
        h = L.lib.mc_ctrl_create(ctypes.byref(cfg), 0)
        assert h
        cfg.mag_ratios = None  # the handle owns a copy of the table
        skip, cnt = ctypes.c_int32(), ctypes.c_int32()
        got = []
        for _ in range(case["calls"]):
            L.check(L.lib.mc_ctrl_step(h, ctypes.byref(skip), ctypes.byref(cnt)))
            got.append(str(skip.value))
        assert "".join(got) == case["mask"]
        st = L.lib.mc_ctrl_state_of(h).contents
        assert st.cnt == cnt.value == case["final"]["cnt"]
        L.check(L.lib.mc_ctrl_reset(h))
        assert L.lib.mc_ctrl_state_of(h).contents.cnt == 0 and L.lib.mc_ctrl_state_of(h).contents.accumulated_ratio[0] == 1.0
        again = []
        for _ in range(n):
            L.check(L.lib.mc_ctrl_step(h, ctypes.byref(skip), None))
            again.append(str(skip.value))
        assert "".join(again) == case["mask"][:n]
        L.lib.mc_ctrl_destroy(h)
    bad = _cfg(L, "wan2.1", [1.0] * 4, 4, 0.1, 2, 0.0)  # retention 0: the first call would hit an empty cache
    assert not L.lib.mc_ctrl_create(ctypes.byref(bad), 0) and b"mc_ctrl_validate" in L.lib.mc_last_error()
    L.lib.mc_ctrl_destroy(None)


@pytest.mark.parametrize("attr", ["_mc_engine", "_mc_flux_engine", "_mc_hunyuan_engine", "_mc_opensora_engine"])
def test_engine_cache_attrs(attr):
    """Every engine kind a patched forward caches: `enable_token_shard` refuses to come after it, `invalidate_engine` drops it."""
    import magcache_b200 as mc
    m = type("M", (), {})()
    m.__dict__[attr] = object()
    m.__dict__["_mc_ctrls"] = {}
    with pytest.raises(RuntimeError, match="before the first forward"):
        mc.enable_token_shard(m, 0, 2)
    mc.invalidate_engine(m)
    assert attr not in m.__dict__ and "_mc_ctrls" not in m.__dict__
    mc.enable_token_shard(m, 0, 2)
