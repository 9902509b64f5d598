"""MagCache configuration: one parameterised description of every controller variant the reference ships
(SURVEY.md Appendix A), the calibrated `mag_ratios` tables, and the presets the reference's READMEs quote."""
import json
import os
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np

from . import _lib
from .controller import interp_cfg, make_ctrl_config, nearest_interp, nearest_interp_linspace, schedule_from

_TABLES = None


def tables():
    """Calibrated magnitude-ratio tables of every adapter (data extracted from the reference literals by
    tests/golden/make_golden.py; each entry of tables.json carries its `source` file:line), e.g.
    MagCache4Wan2.1/magcache_generate.py:910,912,1002,1004,1142,1144; MagCache4FLUX/magcache_flux.py:459;
    MagCache4HunyuanVideo/magcache_sample_video.py:316,318; MagCache4Wan2.2/magcache_generate.py:695,736,738,771."""
    global _TABLES
    if _TABLES is None:
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "tables.json")) as f:
            _TABLES = {k: np.array(v["values"], dtype=np.float64) for k, v in json.load(f).items()}
    return _TABLES


def table_for_ckpt_dir(ckpt_dir: str, task: str = "t2v"):
    """The reference picks the table by substring of --ckpt_dir (magcache_generate.py:909-912, :1001-1004, :1141-1144)."""
    t = tables()
    if "VACE-1.3B" in ckpt_dir:
        return t["wan2.1_vace_1.3b"]
    if "VACE-14B" in ckpt_dir:
        return t["wan2.1_vace_14b"]
    if "T2V-14B" in ckpt_dir:
        return t["wan2.1_t2v_14b"]
    if "T2V-1.3B" in ckpt_dir:
        return t["wan2.1_t2v_1.3b"]
    if "480P" in ckpt_dir:
        return t["wan2.1_i2v_480p"]
    if "720P" in ckpt_dir:
        return t["wan2.1_i2v_720p"]
    raise KeyError(f"no calibrated mag_ratios table matches ckpt_dir={ckpt_dir!r} (the reference would hit AttributeError later)")


def save_json(filename, obj_list):
    """MagCache4Wan2.1/magcache_generate.py:36-38 (appends ".json" like the reference)."""
    with open(str(filename) + ".json", "w") as f:
        json.dump(obj_list, f)


def table_from_calibration(ratios, branches=2):
    """A `mag_ratios` table from a calibration run: the reference prints / dumps `norm_ratio` (one entry per forward from the
    third call on, :165-175) and its authors paste it behind `[1.0]*2` (`np.array([1.0]*2+[...])`, :910-912; `[1.0]+[...]` for the
    scalar-state families, magcache_flux.py:459). `ratios`: the list itself or the path of `wan2_1_mag_ratio.json`."""
    if isinstance(ratios, (str, os.PathLike)):
        with open(ratios) as f:
            ratios = json.load(f)
    arr = np.asarray(ratios, dtype=np.float64)
    if arr.ndim != 1 or len(arr) == 0 or not np.all(np.isfinite(arr)):
        raise ValueError("calibration ratios must be a non-empty 1-D list of finite numbers")
    return np.concatenate([np.ones(branches), arr])


# One row per adapter of the reference (SURVEY Appendix A): the controller parameters that differ between them.
#   branches 2 = state per CFG branch (`cnt % 2`), 1 = scalar state. `interp`: how the table is resampled to another step count.
_LT, _LE = _lib.MC_CMP_LT, _lib.MC_CMP_LE
FAMILIES = {
    # MagCache4Wan2.1/magcache_generate.py:277-292 (T2V), :522-537 (VACE), I2V alike
    "wan2.1": dict(branches=2, cmp=_LT, retention_mode=_lib.MC_RETAIN_FLOOR),
    # eval/magcache/experiments/Wan2.1_EVAL/wan_magcache.py:770-786 — `<=`, `ratio[t-10]`, retention fixed at int(n*0.2)
    "wan2.1-eval": dict(branches=2, cmp=_LE, retention_mode=_lib.MC_RETAIN_FLOOR, table_offset=10),
    # MagCache4Wan2.2/magcache_generate.py:294-317 — two-expert windows; split_step = 2*high_noise_steps
    "wan2.2-t2v": dict(branches=2, cmp=_LT, retention_mode=_lib.MC_RETAIN_WAN22_T2V),
    "wan2.2-i2v": dict(branches=2, cmp=_LT, retention_mode=_lib.MC_RETAIN_WAN22_I2V),
    "wan2.2-ti2v": dict(branches=2, cmp=_LT, retention_mode=_lib.MC_RETAIN_FLOOR),
    # MagCache4QwenImage/magcache_generate.py:205-219 (+ Edit): Wan2.1's controller, np.linspace interpolation (:14-21)
    # the wrap resets ONLY the counter (:243-244): the accumulators carry over into the next image of the same process
    "qwen-image": dict(branches=2, cmp=_LT, retention_mode=_lib.MC_RETAIN_FLOOR, flags=_lib.MC_CTRL_WRAP_KEEPS_ACC),
    # MagCache4FLUX/magcache_flux.py:326-338 ; MagCache4FLUX_Kontext/magcache_flux_kontext.py:328-340 (same statements)
    "flux": dict(branches=1, cmp=_LE, retention_mode=_lib.MC_RETAIN_HALF_UP, veto_index=11, veto_base=28),
    "flux-kontext": dict(branches=1, cmp=_LE, retention_mode=_lib.MC_RETAIN_HALF_UP, veto_index=11, veto_base=28),
    # MagCache4HunyuanVideo/magcache_sample_video.py:88-102
    "hunyuan": dict(branches=1, cmp=_LE, retention_mode=_lib.MC_RETAIN_FLOOR),
    # MagCache4FramePack/magcache_demo_gradio.py:252-270 (and _f1)
    "framepack": dict(branches=1, cmp=_LE, retention_mode=_lib.MC_RETAIN_FLOOR, min_cnt=1, flags=_lib.MC_CTRL_RESET_AT_ZERO, ratio_veto=0.06),
    # MagCache4OmniGen2/magcache/magcache_utils.py:342-354 — one state object per CFG branch, each scalar; accumulated_steps starts at 3 (:44)
    "omnigen2": dict(branches=1, cmp=_LE, retention_mode=_lib.MC_RETAIN_CEIL),
    # eval/magcache/experiments/opensora.py:297-308 — explicit skip_time, `ratio[t-1]`, signed error
    "opensora": dict(branches=1, cmp=_LE, retention_mode=_lib.MC_RETAIN_EXPLICIT, table_offset=1, flags=_lib.MC_CTRL_SIGNED_ERR),
}
INITIAL_ACCUMULATED_STEPS = {"omnigen2": 3}  # MagCacheParams dataclass default, magcache_utils.py:44


@dataclass
class MagCacheConfig:
    """One MagCache setup: `family` is a key of FAMILIES (the adapter whose controller arithmetic applies), the rest are the
    reference's hyper-parameters under the reference's names. `high_noise_steps` is Wan2.2's expert boundary
    (MagCache4Wan2.2/magcache_generate.py:697-698), `skip_time` Open-Sora's explicit retention (opensora.py:424)."""
    family: str = "wan2.1"
    thresh: float = 0.12
    K: int = 2
    retention_ratio: float = 0.2
    sample_steps: int = 50
    mag_ratios: Optional[Sequence[float]] = None
    table: Optional[str] = None  # key into tables() when mag_ratios is not given
    high_noise_steps: Optional[int] = None
    skip_time: Optional[int] = None

    def __post_init__(self):
        if self.family not in FAMILIES:
            raise KeyError(f"unknown MagCache family {self.family!r}; known: {sorted(FAMILIES)}")

    @property
    def branches(self):
        return FAMILIES[self.family]["branches"]

    @property
    def num_steps(self):  # forward calls per video
        return self.sample_steps * self.branches

    def resolved_ratios(self):
        """The table as the controller indexes it: resampled per CFG branch (Wan :915-919) or whole (FLUX :461-463) when the step
        count differs from the calibrated one; the paper-evaluation tables are fixed-length (no interpolation upstream)."""
        src = np.asarray(self.mag_ratios if self.mag_ratios is not None else tables()[self.table], dtype=np.float64)
        off = FAMILIES[self.family].get("table_offset", 0)
        if off:
            if len(src) != self.num_steps - off:
                raise IndexError(f"{self.family}: the table has {len(src)} entries, the forward indexes ratio[t-{off}] for {self.num_steps} calls")
            return src
        if self.branches == 2:
            if self.family == "qwen-image" and len(src) != 2 * self.sample_steps:
                con, ucon = nearest_interp_linspace(src[0::2], self.sample_steps), nearest_interp_linspace(src[1::2], self.sample_steps)
                return np.stack([con, ucon], axis=1).reshape(-1)
            return interp_cfg(src, self.sample_steps)
        return src if len(src) == self.sample_steps else nearest_interp(src, self.sample_steps)

    def ctrl_kwargs(self):
        kw = dict(FAMILIES[self.family])
        if self.family in ("wan2.2-t2v", "wan2.2-i2v"):
            if self.high_noise_steps is None:
                raise ValueError(f"{self.family} needs high_noise_steps (calls made to the high-noise expert per video)")
            kw["split_step"] = 2 * self.high_noise_steps
        if self.family == "opensora":
            kw["split_step"] = 6 if self.skip_time is None else self.skip_time
        return kw

    def schedule(self, calls=None):
        """Skip mask (uint8 per forward call) of one video, from a fresh controller state."""
        R = 0.2 if self.family == "wan2.1-eval" else self.retention_ratio  # hard-coded upstream: `skip_time = int(self.num_steps*0.2)`, :772
        cfg = make_ctrl_config(self.num_steps, self.thresh, self.K, R, self.resolved_ratios(), **self.ctrl_kwargs())
        return schedule_from(cfg, self.num_steps if calls is None else calls, INITIAL_ACCUMULATED_STEPS.get(self.family, 0))


PRESETS = {
    # MagCache4Wan2.1/README.md:13,19,60-65 ; naming E<thresh>K<K>R<retention>
    "wan2.1-1.3b-E012K2R02": MagCacheConfig("wan2.1", 0.12, 2, 0.2, 50, table="wan2.1_t2v_1.3b"),
    "wan2.1-1.3b-E012K4R02": MagCacheConfig("wan2.1", 0.12, 4, 0.2, 50, table="wan2.1_t2v_1.3b"),
    "wan2.1-14b-E024K6R02": MagCacheConfig("wan2.1", 0.24, 6, 0.2, 50, table="wan2.1_t2v_14b"),
    "wan2.1-vace-1.3b-E002K3R02": MagCacheConfig("wan2.1", 0.02, 3, 0.2, 50, table="wan2.1_vace_1.3b"),
    # eval/magcache/experiments/Wan2.1_EVAL/wan_eval.sh:30-31,66-67 ("slow" / "fast" rows of the paper table)
    "wan2.1-eval-slow-E012K2": MagCacheConfig("wan2.1-eval", 0.12, 2, 0.2, 50, table="wan2.1_eval"),
    "wan2.1-eval-fast-E012K4": MagCacheConfig("wan2.1-eval", 0.12, 4, 0.2, 50, table="wan2.1_eval"),
    # MagCache4Wan2.2/README.md:70,94,110
    "wan2.2-ti2v-5b-E006K2R02": MagCacheConfig("wan2.2-ti2v", 0.06, 2, 0.2, 50, table="wan2.2_ti2v_5b_a"),
    "wan2.2-t2v-a14b-E006K2R04": MagCacheConfig("wan2.2-t2v", 0.06, 2, 0.4, 40, table="wan2.2_t2v_a14b", high_noise_steps=13),
    "wan2.2-i2v-a14b-E006K2R01": MagCacheConfig("wan2.2-i2v", 0.06, 2, 0.1, 40, table="wan2.2_i2v_a14b", high_noise_steps=13),
    # MagCache4QwenImage/magcache_generate.py:35-49 (argparse defaults)
    "qwen-image-E006K2R02": MagCacheConfig("qwen-image", 0.06, 2, 0.2, 50, table="qwen_image"),
    "qwen-image-edit-E006K2R02": MagCacheConfig("qwen-image", 0.06, 2, 0.2, 50, table="qwen_image_edit"),
    # MagCache4FLUX/magcache_flux.py:466-468 ; MagCache4FLUX_Kontext/magcache_flux_kontext.py:465-467
    "flux-E024K5R01": MagCacheConfig("flux", 0.24, 5, 0.1, 28, table="flux_dev"),
    "flux-kontext-E005K4R02": MagCacheConfig("flux-kontext", 0.05, 4, 0.2, 28, table="flux_kontext"),
    # MagCache4HunyuanVideo/magcache_sample_video.py:303-305
    "hunyuan-720p-E024K6R02": MagCacheConfig("hunyuan", 0.24, 6, 0.2, 50, table="hunyuan_720p"),
    "hunyuan-720p-E012K4R02": MagCacheConfig("hunyuan", 0.12, 4, 0.2, 50, table="hunyuan_720p"),
    # MagCache4FramePack/magcache_demo_gradio.py:707-710 (UI defaults)
    "framepack-E010K3R02": MagCacheConfig("framepack", 0.10, 3, 0.2, 25, table="framepack"),
    "framepack-f1-E010K3R02": MagCacheConfig("framepack", 0.10, 3, 0.2, 25, table="framepack_f1"),
    # MagCache4OmniGen2/magcache/magcache_utils.py:81-83 (K 3, R 0.2; threshold from the CLI)
    "omnigen2-t2i-cond-E006K3R02": MagCacheConfig("omnigen2", 0.06, 3, 0.2, 50, table="omnigen2_t2i_cond"),
    # eval/magcache/README.md:66, opensora.py:420-433
    "opensora-slow-E012K3": MagCacheConfig("opensora", 0.12, 3, 0.2, 30, table="opensora_eval", skip_time=6),
    "opensora-fast-E024K5": MagCacheConfig("opensora", 0.24, 5, 0.2, 30, table="opensora_eval", skip_time=6),
}
