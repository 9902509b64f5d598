// Shared host/device helpers for libmagcache_b200.so
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "../../include/magcache_b200.h"

namespace mc {

void set_error(const char* fmt, ...);  // defined in controller.cu

inline int32_t cuda_fail(cudaError_t e, const char* what) {
  set_error("%s: %s", what, cudaGetErrorString(e));
  return MC_ERR_CUDA;
}

#define MC_CHECK_ARG(cond, ...)        \
  do {                                 \
    if (!(cond)) {                     \
      ::mc::set_error(__VA_ARGS__);    \
      return MC_ERR_INVALID;           \
    }                                  \
  } while (0)

#define MC_CHECK_LAUNCH(what)                                      \
  do {                                                             \
    cudaError_t e__ = cudaGetLastError();                          \
    if (e__ != cudaSuccess) return ::mc::cuda_fail(e__, what);     \
  } while (0)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int num_sms();  // cudaDevAttrMultiProcessorCount of the current device, cached per device (controller.cu)

constexpr int kMaxDevices = 64;
inline int current_device() {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= kMaxDevices) d = 0;
  return d;
}
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per device: remember it per (kernel, device), not per process.
struct PerDeviceOnce {
  bool done[kMaxDevices] = {};
};
template <typename Kernel>
inline int32_t set_max_smem_once(Kernel kernel, int bytes, PerDeviceOnce& once, const char* what) {
  const int d = current_device();
  if (once.done[d]) return MC_OK;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return cuda_fail(e, what);
  once.done[d] = true;
  return MC_OK;
}

// ---- device-side dtype helpers -----------------------------------------------------------------
__device__ __forceinline__ float bf16_bits_to_f32(uint32_t hi16) { return __uint_as_float(hi16 << 16); }

// unpack 8 bf16 (one uint4) to 8 floats
__device__ __forceinline__ void unpack_bf16x8(const uint4& v, float (&f)[8]) {
  f[0] = __uint_as_float(v.x << 16);
  f[1] = __uint_as_float(v.x & 0xFFFF0000u);
  f[2] = __uint_as_float(v.y << 16);
  f[3] = __uint_as_float(v.y & 0xFFFF0000u);
  f[4] = __uint_as_float(v.z << 16);
  f[5] = __uint_as_float(v.z & 0xFFFF0000u);
  f[6] = __uint_as_float(v.w << 16);
  f[7] = __uint_as_float(v.w & 0xFFFF0000u);
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {  // round-to-nearest-even, like torch
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ uint4 pack_bf16x8(const float (&f)[8]) {
  uint4 v;
  v.x = pack_bf16x2(f[0], f[1]);
  v.y = pack_bf16x2(f[2], f[3]);
  v.z = pack_bf16x2(f[4], f[5]);
  v.w = pack_bf16x2(f[6], f[7]);
  return v;
}
__device__ __forceinline__ float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }  // nn.SiLU in fp32
__device__ __forceinline__ float bf16_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

// torch.nn.GELU() (exact, erf form) in fp32: 0.5*x*(1+erf(x/sqrt(2))) — `img_emb` of the i2v models
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// torch.nn.GELU(approximate='tanh') in fp32, in the operation order of torch's CUDA kernel (ActivationGeluKernel.cu):
// 0.5*x*(1+tanh(kBeta*(x+kKappa*x_cube))), x_cube = x*x*x, with an accurate tanhf. The old tanh.approx.f32 (MUFU.TANH) was
// not good enough: for x < 0, t -> -1 and the output 0.5*x*(1+t) shrinks like exp(-x^2/2), so its error in t became up to
// 13 596 bf16 ulps of the output (at x = -4.875). On every bf16 input this matches torch's F.gelu bit for bit, whether or not
// `x + kKappa*x_cube` is contracted into an FMA; it is written with one rounding per op so that no compiler setting decides.
__device__ __forceinline__ float gelu_tanh(float x) {
  const float kBeta = 0.7978845608028654f;  // sqrt(2/pi)
  const float kKappa = 0.044715f;
  const float x3 = x * x * x;
  const float inner = kBeta * __fadd_rn(x, __fmul_rn(kKappa, x3));
  return 0.5f * x * (1.0f + tanhf(inner));
}

// RoPE in fp32 on four consecutive (real, imag) pairs, cs holding (cos, sin) per pair: every product and every sum rounded on
// its own (no FMA contraction), as torch computes `x * cos +- rotate(x) * sin` elementwise.
__device__ __forceinline__ void rope_pairs4(float (&o)[8], const float (&cs)[8]) {
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const float re = o[2 * p], im = o[2 * p + 1], c = cs[2 * p], sn = cs[2 * p + 1];
    o[2 * p] = __fsub_rn(__fmul_rn(re, c), __fmul_rn(im, sn));
    o[2 * p + 1] = __fadd_rn(__fmul_rn(re, sn), __fmul_rn(im, c));
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace mc
