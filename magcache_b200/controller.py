"""Skip controller front end. The decision arithmetic lives in the C ABI (`mc_ctrl_decide` / `mc_ctrl_advance`, `mc_tea_*`, float64,
bit-exact with the reference); this module is the only one that knows the layout of the C structs: it moves state between the
reference's attribute names and them, and wraps the table resampling entry points."""
import ctypes
import operator

import numpy as np

from . import _lib
from ._lib import CtrlConfig, CtrlState, TeaConfig, TeaState, check, lib

_DP = ctypes.POINTER(ctypes.c_double)


def _resample(fn, src, n_out, arg):
    src = np.ascontiguousarray(src, dtype=np.float64)
    out = np.empty(n_out, dtype=np.float64)
    check(fn(src.ctypes.data_as(_DP), len(src), out.ctypes.data_as(_DP), arg))
    return out


def nearest_interp(src, target_length):
    """C-ABI `mc_nearest_interp` (MagCache4Wan2.1/magcache_generate.py:27-34)."""
    return _resample(lib.mc_nearest_interp, src, target_length, target_length)


def interp_cfg(table, sample_steps):
    """Per-CFG-branch interpolation (magcache_generate.py:915-919) through `mc_nearest_interp_cfg`."""
    table = np.ascontiguousarray(table, dtype=np.float64)
    if len(table) == 2 * sample_steps:
        return table
    return _resample(lib.mc_nearest_interp_cfg, table, 2 * sample_steps, sample_steps)


def nearest_interp_linspace(src, target_length):
    """C-ABI `mc_nearest_interp_linspace`: Qwen-Image's form (MagCache4QwenImage/magcache_generate.py:14-21)."""
    return _resample(lib.mc_nearest_interp_linspace, src, target_length, target_length)


def make_ctrl_config(num_steps, thresh, K, retention_ratio, mag_ratios, branches, cmp, retention_mode, veto_index=-1, veto_base=0,
                     split_step=0, table_offset=0, min_cnt=0, flags=0, ratio_veto=None):
    arr = np.ascontiguousarray(mag_ratios, dtype=np.float64)
    if len(arr) < num_steps - table_offset:
        raise IndexError(f"mag_ratios has {len(arr)} entries but num_steps={num_steps}, table_offset={table_offset} "
                         "(interpolate first, magcache_generate.py:915-919)")
    cfg = CtrlConfig()
    cfg.num_steps, cfg.branches, cfg.K, cfg.cmp, cfg.retention_mode = int(num_steps), int(branches), int(K), int(cmp), int(retention_mode)
    cfg.veto_index, cfg.veto_base, cfg.split_step = int(veto_index), int(veto_base), int(split_step)
    if ratio_veto is not None:
        flags |= _lib.MC_CTRL_RATIO_VETO
    cfg.table_offset, cfg.min_cnt, cfg.flags, cfg.reserved = int(table_offset), int(min_cnt), int(flags), 0
    cfg.thresh, cfg.retention_ratio, cfg.ratio_veto = float(thresh), float(retention_ratio), float(ratio_veto or 0.0)
    cfg.mag_ratios = arr.ctypes.data_as(_DP)
    cfg._keepalive = arr
    return cfg


def schedule_mask(cfg, calls):
    """Whole skip schedule (uint8 0/1 per forward call) from a fresh state."""
    mask = np.zeros(calls, dtype=np.uint8)
    check(lib.mc_ctrl_mask(ctypes.byref(cfg), calls, mask.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))))
    return mask


def schedule_from(cfg, calls, initial_steps=0):
    """`schedule_mask` from a fresh state whose first accumulated step count is `initial_steps` (OmniGen2's MagCacheParams start
    at 3, magcache_utils.py:44), one decide / advance pair per call."""
    st = CtrlState()
    st.accumulated_ratio[0] = st.accumulated_ratio[1] = 1.0
    st.accumulated_steps[0] = initial_steps
    skip, out = ctypes.c_int32(), np.zeros(calls, dtype=np.uint8)
    for i in range(calls):
        check(lib.mc_ctrl_decide(ctypes.byref(cfg), ctypes.byref(st), ctypes.byref(skip)))
        out[i] = skip.value
        check(lib.mc_ctrl_advance(ctypes.byref(cfg), ctypes.byref(st)))
    return out


class AttrController:
    """Runs the controller on state stored under the reference's attribute names of `owner` (a model instance whose class
    carries `cnt`, `accumulated_ratio`, ... exactly as MagCache4Wan2.1/magcache_generate.py:897-906 installs them).
    Scalar families (FLUX/Hunyuan) keep scalars, Wan keeps 2-element lists — whatever form the script wrote is preserved.

    `names` maps a canonical input (`cnt, num_steps, magcache_thresh, K, retention_ratio, mag_ratios, split_step,
    accumulated_ratio, accumulated_err, accumulated_steps`) to the attribute a script keeps it under when that differs (the
    paper-evaluation scripts say `t`, `ratio`, `accumulated_sim`, ...); `fixed` gives the value of an input the script hard-codes."""

    _INPUTS = ("mag_ratios", "num_steps", "magcache_thresh", "K", "retention_ratio")

    def __init__(self, family_kwargs, names=None, fixed=None):
        self.kw = family_kwargs
        self.names = names or {}
        self.fixed = fixed or {}
        self._cnt = self.names.get("cnt", "cnt")
        self._acc = tuple(self.names.get(n, n) for n in ("accumulated_ratio", "accumulated_err", "accumulated_steps"))
        self._read = operator.attrgetter(*(self.names.get(n, n) for n in self._INPUTS))  # one call per forward on the hot path
        self._cfg = None
        self._key = None

    def _get(self, o, name, *default):
        if name in self.fixed:
            return self.fixed[name]
        return getattr(o, self.names.get(name, name), *default)

    def _inputs(self, o):
        if not self.fixed:
            return self._read(o)
        return tuple(self._get(o, n) for n in self._INPUTS)

    def _config(self, o):
        kw = self.kw
        if kw["retention_mode"] in (_lib.MC_RETAIN_WAN22_T2V, _lib.MC_RETAIN_WAN22_I2V, _lib.MC_RETAIN_EXPLICIT):
            # MagCache4Wan2.2/magcache_generate.py:344 `split_step = split_steps*2`; None (TI2V-5B) falls back to int(n*R), :301-303.
            # Open-Sora's `skip_time` (opensora.py:424) is the same explicit window
            split = self._get(o, "split_step", None)
            kw = dict(kw, split_step=int(split)) if split is not None else dict(kw, retention_mode=_lib.MC_RETAIN_FLOOR)
        # keyed on the table's CONTENT (a few hundred bytes): an in-place edit of the installed table — the reference's suggested
        # `**0.5` smoothing, say — keeps id() and len() but must reach the controller
        mr, n, thresh, K, R = self._inputs(o)
        arr = np.ascontiguousarray(np.asarray(mr, dtype=np.float64))
        key = (hash(arr.tobytes()), len(arr), n, float(thresh), int(K), float(R), kw.get("split_step"))
        if self._key != key:
            self._cfg = make_ctrl_config(n, thresh, K, R, arr, **kw)
            self._key = key
        return self._cfg

    def _load(self, o):
        st = CtrlState()
        st.cnt = int(getattr(o, self._cnt))
        ratio, err, steps = self._acc
        if self.kw["branches"] == 2:
            r, e, s = getattr(o, ratio), getattr(o, err), getattr(o, steps)
            for i in range(2):
                st.accumulated_ratio[i] = float(r[i])
                st.accumulated_err[i] = float(e[i])
                st.accumulated_steps[i] = int(s[i])
        else:
            # FramePack's `initialize_magcache` does not create the accumulators; its forward does at cnt == 0
            # (magcache_demo_gradio.py:63-74, :253-256) — absent attributes are the fresh state
            st.accumulated_ratio[0] = float(getattr(o, ratio, 1.0))
            st.accumulated_err[0] = float(getattr(o, err, 0.0))
            st.accumulated_steps[0] = int(getattr(o, steps, 0))
            st.accumulated_ratio[1] = 1.0
        return st

    def _store(self, o, st, with_cnt):
        ratio, err, steps = self._acc
        if self.kw["branches"] == 2:
            # the reference mutates the class-level lists in place (self.accumulated_ratio[i] = ...)
            r, e, s = getattr(o, ratio), getattr(o, err), getattr(o, steps)
            for i in range(2):
                r[i] = st.accumulated_ratio[i]
                e[i] = st.accumulated_err[i]
                s[i] = st.accumulated_steps[i]
        else:
            setattr(o, ratio, st.accumulated_ratio[0])
            setattr(o, err, st.accumulated_err[0])
            setattr(o, steps, st.accumulated_steps[0])
        if with_cnt:
            self._set_cnt(o, st.cnt)

    def _set_cnt(self, o, value):
        """`self.cnt += 1`. Wan2.2 / Qwen-Image install `cnt = torch.tensor(0)` on the CLASS (MagCache4Wan2.2/magcache_generate.py:342): the
        in-place add mutates that one tensor, which is how the high-noise and the low-noise expert (two instances of one class) share a
        counter. Keep that: a tensor counter is updated in place, anything else is rebound on the instance like a Python int."""
        cur = getattr(type(o), self._cnt, None)
        if hasattr(cur, "fill_") and self._cnt not in o.__dict__:
            cur.fill_(value)
        else:
            setattr(o, self._cnt, value)

    def decide(self, o):
        cfg = self._config(o)
        st = self._load(o)
        skip = ctypes.c_int32(0)
        check(lib.mc_ctrl_decide(ctypes.byref(cfg), ctypes.byref(st), ctypes.byref(skip)))
        self._store(o, st, with_cnt=False)
        return bool(skip.value)

    def advance(self, o):
        cfg = self._config(o)
        st = self._load(o)
        check(lib.mc_ctrl_advance(ctypes.byref(cfg), ctypes.byref(st)))
        if st.cnt == 0 and self.kw["branches"] == 2 and not (self.kw.get("flags", 0) & _lib.MC_CTRL_WRAP_KEEPS_ACC):
            # end of video: the reference REBINDS fresh lists (magcache_generate.py:308-311)
            for name, fresh in zip(self._acc, ([1.0, 1.0], [0.0, 0.0], [0, 0])):
                setattr(o, name, fresh)
            self._set_cnt(o, 0)
        else:
            self._store(o, st, with_cnt=True)


def _bf16(v):
    """fp32 -> bf16 (round to nearest even), as a Python float."""
    b = np.array([v], dtype=np.float32).view(np.uint32)
    b = (b + np.uint32(0x7FFF) + ((b >> np.uint32(16)) & np.uint32(1))) & np.uint32(0xFFFF0000)
    return float(b.view(np.float32)[0])


def opensora_rel_l1(sum_d, sum_p, n):
    """`((cur - prev).abs().mean() / prev.abs().mean()).cpu().item()` on bf16 tensors (eval/magcache/experiments/opensora.py:102) from
    the two sums over n elements: each mean is an fp32 quotient rounded to a bf16 scalar, and so is their quotient."""
    with np.errstate(divide="ignore", invalid="ignore"):
        m_d = _bf16(np.float32(sum_d) / np.float32(n))
        m_p = _bf16(np.float32(sum_p) / np.float32(n))
        return _bf16(np.float32(m_d) / np.float32(m_p))


class OpenSoraTeaController:
    """Open-Sora's TeaCache rule (eval/magcache/experiments/opensora.py:96-107) through `mc_tea_opensora_decide`, on state under the
    reference's attribute names: `rel_l1_thresh`, `accumulated_rel_l1_distance`. No counter: a call is forced by its timestep."""

    COEFFICIENTS = (2.17546007e+02, -1.18329252e+02, 2.68662585e+01, -4.59364272e-02, 4.84426240e-02)  # :100

    def __init__(self, coefficients=COEFFICIENTS):
        self._coef = (ctypes.c_double * len(coefficients))(*[float(c) for c in coefficients])
        self._n = len(coefficients)

    def decide(self, o, forced, rel):
        """True = compute the blocks. `rel` (the bf16 distance, `opensora_rel_l1`) is ignored on a forced call."""
        calc, acc = ctypes.c_int32(), ctypes.c_double()
        check(lib.mc_tea_opensora_decide(int(bool(forced)), 0.0 if rel is None else float(rel), float(o.accumulated_rel_l1_distance),
                                         float(o.rel_l1_thresh), self._coef, self._n, ctypes.byref(calc), ctypes.byref(acc)))
        o.accumulated_rel_l1_distance = acc.value
        return bool(calc.value)


class TeaController:
    """TeaCache's rule (eval/magcache/experiments/Wan2.1_EVAL/wan_teacache.py:535-564, 587-589) on state under that script's attribute
    names: `cnt, num_steps, ret_steps, cutoff_steps, coefficients, teacache_thresh, accumulated_rel_l1_distance_even / _odd`."""

    @staticmethod
    def _load(o):
        coef = [float(c) for c in o.coefficients]
        cfg = TeaConfig()
        cfg.num_steps, cfg.ret_steps, cfg.cutoff_steps, cfg.n_coef, cfg.thresh = int(o.num_steps), int(o.ret_steps), int(o.cutoff_steps), len(coef), float(o.teacache_thresh)
        for i, c in enumerate(coef):
            cfg.coef[i] = c
        st = TeaState()
        st.cnt = int(o.cnt)
        st.accumulated[0], st.accumulated[1] = float(o.accumulated_rel_l1_distance_even), float(o.accumulated_rel_l1_distance_odd)
        return cfg, st

    def decide(self, o, distance):
        """True = compute the blocks. `distance()` (the relative L1 change of the modulated input) is called only when the rule reads it."""
        cfg, st = self._load(o)
        needs, calc = ctypes.c_int32(), ctypes.c_int32()
        check(lib.mc_tea_needs_distance(ctypes.byref(cfg), ctypes.byref(st), ctypes.byref(needs)))
        check(lib.mc_tea_decide(ctypes.byref(cfg), ctypes.byref(st), distance() if needs.value else 0.0, ctypes.byref(calc)))
        o.accumulated_rel_l1_distance_even, o.accumulated_rel_l1_distance_odd = st.accumulated[0], st.accumulated[1]
        return bool(calc.value)

    def advance(self, o):
        cfg, st = self._load(o)
        check(lib.mc_tea_advance(ctypes.byref(cfg), ctypes.byref(st)))
        o.cnt = st.cnt
