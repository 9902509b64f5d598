"""ctypes binding of libmagcache_b200.so (the C ABI declared in include/magcache_b200.h).

There is no fallback: if the shared library has not been built (`python magcache_b200/build.py`) importing
this module raises, and every device entry point raises `MagCacheError` when CUDA reports a failure.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int32, c_int64, c_uint8, c_uint32, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmagcache_b200.so")

MC_OK = 0
MC_ERR_INVALID, MC_ERR_CUDA, MC_ERR_STATE = -1, -2, -3
MC_F32, MC_BF16 = 0, 1
MC_CMP_LT, MC_CMP_LE = 0, 1
MC_RETAIN_FLOOR, MC_RETAIN_HALF_UP, MC_RETAIN_CEIL, MC_RETAIN_WAN22_T2V, MC_RETAIN_WAN22_I2V, MC_RETAIN_EXPLICIT = 0, 1, 2, 3, 4, 5
MC_CTRL_SIGNED_ERR, MC_CTRL_RESET_AT_ZERO, MC_CTRL_RATIO_VETO, MC_CTRL_WRAP_KEEPS_ACC = 1, 2, 4, 8
ABI_VERSION = 11
MC_EPI_BIAS_BF16, MC_EPI_BIAS_GELU_BF16, MC_EPI_BIAS_GATE_RESID, MC_EPI_ROWBIAS_BF16, MC_EPI_BIAS_F32, MC_EPI_BIAS_GELU_ERF_BF16 = 0, 1, 2, 3, 4, 5
MC_EPI_BIAS_GATE_RESID_BF16, MC_EPI_BIAS_SILU_BF16, MC_EPI_BIAS_GATE_RESID_ADD_BF16 = 6, 7, 8


class MagCacheError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libmagcache_b200 error {code}: {msg}")
        self.code = code


class CtrlConfig(Structure):
    _fields_ = [("num_steps", c_int32), ("branches", c_int32), ("K", c_int32), ("cmp", c_int32), ("retention_mode", c_int32),
                ("veto_index", c_int32), ("veto_base", c_int32), ("split_step", c_int32), ("table_offset", c_int32),
                ("min_cnt", c_int32), ("flags", c_int32), ("reserved", c_int32), ("thresh", c_double), ("retention_ratio", c_double),
                ("ratio_veto", c_double), ("mag_ratios", POINTER(c_double))]


class TeaConfig(Structure):
    _fields_ = [("num_steps", c_int32), ("ret_steps", c_int32), ("cutoff_steps", c_int32), ("n_coef", c_int32), ("thresh", c_double),
                ("coef", c_double * 8)]


class TeaState(Structure):
    _fields_ = [("cnt", c_int32), ("pad", c_int32), ("accumulated", c_double * 2)]


class DitDims(Structure):
    _fields_ = [("dim", c_int32), ("ffn_dim", c_int32), ("num_heads", c_int32), ("num_layers", c_int32), ("in_dim", c_int32),
                ("out_dim", c_int32), ("freq_dim", c_int32), ("text_dim", c_int32), ("text_len", c_int32), ("eps", c_float)]


DIT_BLOCK_FIELDS = ("mod", "w_qkv", "b_qkv", "w_o", "b_o", "nqk", "n3_w", "n3_b", "c_wq", "c_bq", "c_wkv", "c_bkv", "c_wo", "c_bo", "c_nq",
                    "c_nk", "w_f1", "b_f1", "w_f2", "b_f2")
DIT_TOP_FIELDS = ("patch_w", "patch_b", "text_w1", "text_b1", "text_w2", "text_b2", "time_w1", "time_b1", "time_w2", "time_b2", "tproj_w",
                  "tproj_b", "head_mod", "head_wt", "head_b")


class DitBlock(Structure):
    _fields_ = [(n, c_void_p) for n in DIT_BLOCK_FIELDS]


class DitWeights(Structure):
    _fields_ = [(n, c_void_p) for n in DIT_TOP_FIELDS] + [("blocks", POINTER(DitBlock))]


class Copy2D(Structure):
    _fields_ = [("dst", c_void_p), ("dpitch", c_int64), ("src", c_void_p), ("spitch", c_int64), ("width", c_int64), ("height", c_int64)]


class CtrlState(Structure):
    _fields_ = [("cnt", c_int32), ("accumulated_steps", c_int32 * 2), ("pad", c_int32), ("accumulated_ratio", c_double * 2),
                ("accumulated_err", c_double * 2)]


# name -> argtypes ; every function returns int32 except mc_last_error. Kept in one table so the CPU test-suite can check
# that the library exports exactly what the header declares.
SIGNATURES = {
    "mc_abi_version": [],
    "mc_nearest_interp": [POINTER(c_double), c_int32, POINTER(c_double), c_int32],
    "mc_nearest_interp_cfg": [POINTER(c_double), c_int32, POINTER(c_double), c_int32],
    "mc_nearest_interp_linspace": [POINTER(c_double), c_int32, POINTER(c_double), c_int32],
    "mc_ctrl_decide": [POINTER(CtrlConfig), POINTER(CtrlState), POINTER(c_int32)],
    "mc_ctrl_advance": [POINTER(CtrlConfig), POINTER(CtrlState)],
    "mc_ctrl_mask": [POINTER(CtrlConfig), c_int32, POINTER(c_uint8)],
    "mc_ctrl_validate": [POINTER(CtrlConfig)],
    "mc_ctrl_step": [c_void_p, POINTER(c_int32), POINTER(c_int32)],
    "mc_ctrl_reset": [c_void_p],
    "mc_tea_needs_distance": [POINTER(TeaConfig), POINTER(TeaState), POINTER(c_int32)],
    "mc_tea_decide": [POINTER(TeaConfig), POINTER(TeaState), c_double, POINTER(c_int32)],
    "mc_tea_advance": [POINTER(TeaConfig), POINTER(TeaState)],
    "mc_rel_l1": [c_void_p, c_void_p, c_int64, c_void_p, c_void_p],
    "mc_tea_opensora_decide": [c_int32, c_double, c_double, c_double, POINTER(c_double), c_int32, POINTER(c_int32), POINTER(c_double)],
    "mc_ln_t2i_modulate_rel_l1": [c_void_p, c_int64, c_int32, c_float, c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p],
    "mc_cache_hit_add": [c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_int64, c_void_p],
    "mc_residual_sub": [c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_int64, c_void_p],
    "mc_cfg_combine": [c_void_p, c_void_p, c_float, c_void_p, c_int64, c_void_p],
    "mc_cfg_step": [c_void_p, c_void_p, c_float, c_void_p, c_float, c_float, POINTER(c_void_p), POINTER(c_float), c_int32, c_float, c_void_p,
                    c_void_p, c_int64, c_void_p],
    "mc_residual_stats": [c_void_p, c_int32, c_void_p, c_int32, c_int64, c_int32, c_double, c_void_p, c_void_p],
    "mc_residual_sub_stats": [c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_void_p, c_int64, c_int32, c_double, c_void_p, c_void_p],
    "mc_dequant_fp8_bf16": [c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_void_p],
    "mc_patchify": [c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p],
    "mc_ln_modulate": [c_void_p, c_int32, c_int64, c_int32, c_float, c_int32, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p,
                       c_int32, c_void_p],
    "mc_rmsnorm_rope": [c_void_p, c_int64, c_int64, c_int32, c_void_p, c_float, c_void_p, c_int32, c_void_p],
    "mc_rmsnorm_rope_segs": [c_void_p, c_int64, c_int64, c_int32, c_int32, c_void_p, c_float, c_void_p, c_int32, c_void_p],
    "mc_rmsnorm_head_rope": [c_void_p, c_int64, c_int64, c_int32, c_void_p, c_float, c_void_p, c_void_p],
    "mc_ip_attn": [c_void_p, c_int64, c_int64, c_int32, c_void_p, c_float, c_void_p, c_int64, POINTER(c_int32), POINTER(c_float), c_int32,
                   c_void_p, c_int64, c_void_p],
    "mc_rmsnorm_head72_rope": [c_void_p, c_int64, c_int64, c_int32, c_void_p, c_float, c_void_p, c_int64, c_int32, c_void_p],
    "mc_attn_varlen_d72": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int32, c_void_p, c_int32, c_int32,
                           c_float, c_void_p],
    "mc_attn_temporal_d72": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int32, c_int32, c_int32, c_int32,
                             c_float, c_void_p],
    "mc_colmean_bf16": [c_void_p, c_int64, c_int32, c_int32, c_void_p, c_void_p],
    "mc_silu_bf16": [c_void_p, c_void_p, c_int64, c_void_p],
    "mc_gemm_bf16": [c_void_p, c_int64, c_void_p, c_int64, c_int32, c_int32, c_int32, c_void_p, c_int32, c_void_p, c_int64, c_void_p,
                     c_void_p],
    "mc_gemm_bf16_add": [c_void_p, c_int64, c_void_p, c_int64, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_int64, c_void_p, c_void_p,
                         c_int64, c_int32, c_void_p],
    "mc_gemm_bf16_lora": [c_void_p, c_int64, c_void_p, c_int64, c_int32, c_int32, c_int32, c_void_p, c_int32, c_void_p, c_int64, c_void_p,
                          c_void_p, c_int64, c_int32, c_void_p, c_int64, c_void_p, c_int64, c_int32, c_void_p],
    "mc_attn_workspace_bytes": [c_int32, c_int32, c_int32, POINTER(c_int64)],
    "mc_attn_fwd": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int32, c_int32, c_int32, c_float,
                    c_void_p, c_int64, c_void_p],
    "mc_attn_fwd_ex": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int32, c_int32, c_int32, c_float,
                       c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_int32, c_void_p],
    "mc_p2p_alloc": [c_int64, POINTER(c_void_p), c_void_p],
    "mc_p2p_open": [c_void_p, POINTER(c_void_p)],
    "mc_p2p_close": [c_void_p],
    "mc_p2p_free": [c_void_p],
    "mc_p2p_bump": [c_void_p, c_void_p, c_void_p],
    "mc_p2p_push": [c_void_p, POINTER(c_void_p), POINTER(c_void_p), c_int32, c_int64, c_void_p, c_void_p],
    "mc_p2p_wait": [c_void_p, c_int32, c_void_p, c_void_p],
    "mc_p2p_push2d": [POINTER(Copy2D), c_int32, POINTER(c_void_p), c_int32, c_void_p, c_void_p],
    "mc_linear_f32_small": [c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_void_p],
    "mc_head_workspace_bytes": [c_int32, POINTER(c_int64)],
    "mc_head_unpatchify": [c_void_p, c_int32, c_void_p, c_int64, c_int64, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p,
                           c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_int64, c_int32, c_void_p],
    "mc_head_prepare": [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_int64, c_void_p],
    "mc_head_unpatchify_ex": [c_void_p, c_int32, c_void_p, c_int64, c_int64, c_int32, c_int32, c_int32, c_int32, c_int32, c_float,
                              POINTER(c_void_p), c_int32, c_void_p, c_int64, c_int32, c_void_p],
    "mc_head_unpatchify_step": [c_void_p, c_int32, c_void_p, c_int64, c_int64, c_int32, c_int32, c_int32, c_int32, c_int32, c_float,
                                POINTER(c_void_p), c_int32, c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_float, c_float, c_float, c_void_p],
    "mc_head_unpatchify_step_hist": [c_void_p, c_int32, c_void_p, c_int64, c_int64, c_int32, c_int32, c_int32, c_int32, c_int32, c_float,
                                     POINTER(c_void_p), c_int32, c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_float, c_float, c_float,
                                     c_void_p, c_float, c_float, c_void_p, c_void_p],
    "mc_opensora_head": [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_int32, c_float,
                         c_int32, c_int32, c_void_p, c_void_p, c_float, c_void_p, c_void_p],
    "mc_opensora_head_frames": [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_int32,
                                c_float, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_float, c_void_p, c_void_p],
    "mc_transpose_bf16": [c_void_p, c_int64, c_int32, c_int32, c_void_p, c_int64, c_void_p],
    "mc_time_sinusoid": [c_void_p, c_int32, c_int32, c_void_p, c_void_p],
    "mc_cast": [c_void_p, c_int32, c_void_p, c_int32, c_int64, c_void_p],
    "mc_nccl_unique_id": [c_void_p],
    "mc_nccl_destroy": [c_void_p],
    "mc_allgather_kv": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p],
    "mc_dit_workspace_bytes": [c_void_p, c_int32, c_int32, c_int32, POINTER(c_int64)],
    "mc_dit_bind": [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_int64, c_void_p],
    "mc_dit_forward": [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_void_p],
    "mc_dit_plan": [c_void_p, c_int32, c_void_p, c_int64, POINTER(c_int64)],
}

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: the CUDA extension has not been built. Run `python magcache_b200/build.py` "
        "(needs nvcc; cross-compiles for sm_90a without a GPU). There is no CPU/eager fallback by design.")

lib = ctypes.CDLL(LIB_PATH)
lib.mc_last_error.restype = c_char_p
lib.mc_last_error.argtypes = []
for _name, _args in SIGNATURES.items():
    _fn = getattr(lib, _name)
    _fn.restype = c_int32
    _fn.argtypes = _args


# entry points that do not return an int32 status
lib.mc_ctrl_create.restype, lib.mc_ctrl_create.argtypes = c_void_p, [POINTER(CtrlConfig), c_int32]
lib.mc_ctrl_state_of.restype, lib.mc_ctrl_state_of.argtypes = POINTER(CtrlState), [c_void_p]
lib.mc_ctrl_destroy.restype, lib.mc_ctrl_destroy.argtypes = None, [c_void_p]
lib.mc_dit_create.restype, lib.mc_dit_create.argtypes = c_void_p, [POINTER(DitDims), POINTER(DitWeights)]
lib.mc_dit_destroy.restype, lib.mc_dit_destroy.argtypes = None, [c_void_p]
lib.mc_nccl_init.restype, lib.mc_nccl_init.argtypes = c_void_p, [c_int32, c_int32, c_void_p]
OTHER_EXPORTS = ("mc_last_error", "mc_ctrl_create", "mc_ctrl_state_of", "mc_ctrl_destroy", "mc_dit_create", "mc_dit_destroy", "mc_nccl_init")

if lib.mc_abi_version() != ABI_VERSION:
    raise ImportError(f"{LIB_PATH} has ABI version {lib.mc_abi_version()}, this package needs {ABI_VERSION}: rebuild with "
                      "`python magcache_b200/build.py`")


def check(rc):
    if rc != MC_OK:
        raise MagCacheError(rc, lib.mc_last_error().decode("utf-8", "replace"))
