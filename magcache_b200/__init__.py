"""magcache_b200 — H100-native (sm_90a) MagCache denoising hot path behind the reference's monkey-patch API.

    from magcache_b200 import magcache_forward, magcache_calibration, init_magcache

Importing this package loads libmagcache_b200.so (build it with `python magcache_b200/build.py`); there is no CPU fallback.
"""
from . import config  # noqa: F401
from .config import FAMILIES, PRESETS, MagCacheConfig, interp_cfg, nearest_interp, tables  # noqa: F401
from .patch import (enable_sequence_parallel, enable_token_shard, invalidate_engine, init_magcache, init_magcache_calibration, magcache_branch, magcache_calibration,  # noqa: F401
                    init_magcache_eval, init_magcache_flux, init_magcache_flux_calibration, init_magcache_hunyuan, init_magcache_hunyuan_calibration, init_magcache_qwen_image, init_magcache_qwen_image_calibration, init_magcache_wan22, init_teacache, magcache_eval_forward, magcache_flux_calibration, magcache_flux_forward, magcache_forward, magcache_hunyuan_calibration, magcache_hunyuan_forward, magcache_opensora_forward, magcache_qwen_image_calibration, magcache_qwen_image_forward, init_magcache_opensora, magcache_vace_calibration, magcache_vace_forward, magcache_wan22_forward, reset_magcache,
                    teacache_forward, teacache_opensora_forward, init_teacache_opensora)
from .sampler import FlowDPMSolverSampler, FlowEulerSampler, FlowUniPCSampler, cfg_denoise_step, sampling_sigmas  # noqa: F401
from .wan import WAN_CONFIGS, WanDims, WanEngine, WanModelHandle, WanWeights  # noqa: F401
from .native import NativeWanForward  # noqa: F401
from .opensora import OpenSoraEngine, OpenSoraWeights, random_opensora_weights  # noqa: F401
from . import opensora  # noqa: F401

__version__ = "0.1.0"
