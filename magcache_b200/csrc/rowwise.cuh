// Per-row arithmetic of the LayerNorm kernels (rowwise_kernels.cu) and of the kernels that run a LayerNorm in front of their own
// work (opensora_head.cu): every form calls these, so all of them give the same bits.
#pragma once
#include "common.cuh"

namespace mc {

__device__ __forceinline__ void load_param8(const float* p, float (&f)[8]) {  // per-column parameters: L1-resident, reused by every row
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

// LayerNorm statistics of a row held in registers. Group i of this lane is column group lane + i * lanes; groups at or past
// `groups` are left out. `reduce` sums over the lanes of the row. Two passes: the mean, then the variance from the squared
// deviations. Returns rsqrt(var + eps) and sets `mean`.
template <int G, typename Reduce>
__device__ __forceinline__ float ln_rstd(const float (&v)[G][8], int lane, int lanes, int groups, float inv_n, float eps, Reduce reduce,
                                         float& mean) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < G; ++i)
    if (lane + i * lanes < groups) {
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    }
  mean = reduce(s) * inv_n;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < G; ++i)
    if (lane + i * lanes < groups) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[i][j] - mean;
        q = fmaf(d, d, q);
      }
    }
  return rsqrtf(reduce(q) * inv_n + eps);
}

struct WarpReduce {  // the `reduce` of the warp-per-row forms
  __device__ __forceinline__ float operator()(float v) const { return warp_sum(v); }
};

// `t2i_modulate(LayerNorm(x), shift, scale)` of 8 elements with every step a bf16 tensor op (mc_ln_modulate mode 2):
// o = bf16(bf16(bf16(LN(x)) * bf16(1 + scale)) + shift), scale / shift the per-column parameters at sc / sh (bf16 values).
__device__ __forceinline__ void t2i_modulate8(const float (&v)[8], float mean, float rstd, const float* sc, const float* sh, float (&o)[8]) {
  float a[8], b[8];
  load_param8(sc, a);
  load_param8(sh, b);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float y = round_bf16((v[j] - mean) * rstd);
    o[j] = round_bf16(__fadd_rn(round_bf16(__fmul_rn(y, round_bf16(__fadd_rn(1.0f, a[j])))), b[j]));
  }
}

}  // namespace mc
