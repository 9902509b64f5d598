// Residual-cache kernels — the HBM-bound half of the MagCache hot path.
//   K1 cache-hit add     `x = x + residual_x`            MagCache4Wan2.1/magcache_generate.py:295
//   K2 residual sub      `residual_x = x - ori_x`        MagCache4Wan2.1/magcache_generate.py:299
//   K3 calibration stats  norm ratio / std / cos distance MagCache4Wan2.1/magcache_generate.py:167-169
//   FP8 weight dequantisation of HunyuanVideo --use-fp8 checkpoints (MagCache4HunyuanVideo/README.md:76-96)
// Layout: flat contiguous tensors; every thread moves 128-bit words with L1::no_allocate (streamed once),
// UNROLL independent word-groups in flight per thread, grid = a multiple of the SM count (persistent grid-stride).
#include <cuda_fp16.h>

#include "common.cuh"
#include "ptx.cuh"
#include "ring.cuh"

namespace mc {

// ---- 8-element group load/store for fp32 and bf16 ----------------------------------------------------------
template <int DT>
struct Elem;
template <>
struct Elem<MC_F32> {
  static constexpr int kBytes = 4;
  static constexpr int kAlign = 32;  // 8 fp32 move as ONE 256-bit access per lane
  __device__ static __forceinline__ void load8(const void* base, int64_t i, float (&f)[8]) {
    ptx::ld_nc_v8_f32(static_cast<const float*>(base) + i, f);
  }
  __device__ static __forceinline__ void store8(void* base, int64_t i, const float (&f)[8]) {
    ptx::st_na_v8_f32(static_cast<float*>(base) + i, f);
  }
  __device__ static __forceinline__ float load1(const void* base, int64_t i) { return static_cast<const float*>(base)[i]; }
  __device__ static __forceinline__ void store1(void* base, int64_t i, float v) { static_cast<float*>(base)[i] = v; }
};
template <>
struct Elem<MC_BF16> {
  static constexpr int kBytes = 2;
  static constexpr int kAlign = 16;
  __device__ static __forceinline__ void load8(const void* base, int64_t i, float (&f)[8]) {
    uint4 a = ptx::ld_nc_v4(static_cast<const __nv_bfloat16*>(base) + i);
    unpack_bf16x8(a, f);
  }
  __device__ static __forceinline__ void store8(void* base, int64_t i, const float (&f)[8]) {
    ptx::st_na_v4(static_cast<__nv_bfloat16*>(base) + i, pack_bf16x8(f));
  }
  __device__ static __forceinline__ float load1(const void* base, int64_t i) {
    return __bfloat162float(static_cast<const __nv_bfloat16*>(base)[i]);
  }
  __device__ static __forceinline__ void store1(void* base, int64_t i, float v) {
    static_cast<__nv_bfloat16*>(base)[i] = __float2bfloat16_rn(v);
  }
};

// out = a + sign * b  (fp32 arithmetic, one rounding into the output type: torch's promoted add/sub)
template <int DA, int DB, int DO, int UNROLL>
__global__ void __launch_bounds__(256) axpb_kernel(const void* __restrict__ a, const void* __restrict__ b, void* __restrict__ out,
                                                   int64_t n_groups /* of 8 */, float sign) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  int64_t g = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  // main: UNROLL groups per thread per trip, all loads issued before any store
  for (; g + (UNROLL - 1) * stride < n_groups; g += UNROLL * stride) {
    float fa[UNROLL][8], fb[UNROLL][8];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      Elem<DA>::load8(a, (g + u * stride) * 8, fa[u]);
      Elem<DB>::load8(b, (g + u * stride) * 8, fb[u]);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
#pragma unroll
      for (int j = 0; j < 8; ++j) fa[u][j] = fa[u][j] + sign * fb[u][j];
      Elem<DO>::store8(out, (g + u * stride) * 8, fa[u]);
    }
  }
  for (; g < n_groups; g += stride) {
    float fa[8], fb[8];
    Elem<DA>::load8(a, g * 8, fa);
    Elem<DB>::load8(b, g * 8, fb);
#pragma unroll
    for (int j = 0; j < 8; ++j) fa[j] = fa[j] + sign * fb[j];
    Elem<DO>::store8(out, g * 8, fa);
  }
}

template <int DA, int DB, int DO>
__global__ void axpb_scalar_kernel(const void* __restrict__ a, const void* __restrict__ b, void* __restrict__ out, int64_t begin,
                                   int64_t n, float sign) {
  int64_t i = begin + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) Elem<DO>::store1(out, i, Elem<DA>::load1(a, i) + sign * Elem<DB>::load1(b, i));
}

template <int DA, int DB, int DO>
static int32_t launch_axpb(const void* a, const void* b, void* out, int64_t n, float sign, cudaStream_t s) {
  constexpr int kUnroll = 4;
  auto al = [](const void* p, int a_) { return (reinterpret_cast<uintptr_t>(p) & static_cast<uintptr_t>(a_ - 1)) == 0; };
  const bool vec_ok = al(a, Elem<DA>::kAlign) && al(b, Elem<DB>::kAlign) && al(out, Elem<DO>::kAlign);
  const int64_t n_groups = vec_ok ? n / 8 : 0;
  if (n_groups > 0) {
    const int threads = 256;
    int64_t want = (n_groups + static_cast<int64_t>(threads) * kUnroll - 1) / (static_cast<int64_t>(threads) * kUnroll);
    const int64_t cap = static_cast<int64_t>(num_sms()) * 8;  // 8 resident CTAs of 256 threads per SM = full occupancy
    int grid = static_cast<int>(want < cap ? (want < 1 ? 1 : want) : cap);
    axpb_kernel<DA, DB, DO, kUnroll><<<grid, threads, 0, s>>>(a, b, out, n_groups, sign);
    MC_CHECK_LAUNCH("axpb_kernel launch");
  }
  const int64_t done = n_groups * 8;
  if (done < n) {
    const int64_t rem = n - done;
    axpb_scalar_kernel<DA, DB, DO><<<static_cast<int>((rem + 255) / 256), 256, 0, s>>>(a, b, out, done, n, sign);
    MC_CHECK_LAUNCH("axpb_scalar_kernel launch");
  }
  return MC_OK;
}

static int32_t dispatch_axpb(const void* a, int da, const void* b, int db, void* out, int dout, int64_t n, float sign,
                             cudaStream_t s, const char* who) {
  MC_CHECK_ARG(n >= 0, "%s: negative element count", who);
  if (n == 0) return MC_OK;  // empty tensors have null data pointers
  MC_CHECK_ARG(a && b && out, "%s: null pointer", who);
#define MC_CASE(A, B, O) \
  if (da == A && db == B && dout == O) return launch_axpb<A, B, O>(a, b, out, n, sign, s);
  MC_CASE(MC_BF16, MC_F32, MC_F32)    // Wan hit: bf16 patch-embed output + fp32 residual
  MC_CASE(MC_F32, MC_BF16, MC_F32)    // Wan miss: fp32 stream - bf16 ori_x
  MC_CASE(MC_F32, MC_F32, MC_F32)
  MC_CASE(MC_BF16, MC_BF16, MC_BF16)  // FLUX / Hunyuan (all bf16)
  MC_CASE(MC_BF16, MC_BF16, MC_F32)
  MC_CASE(MC_F32, MC_BF16, MC_BF16)
  MC_CASE(MC_BF16, MC_F32, MC_BF16)
  MC_CASE(MC_F32, MC_F32, MC_BF16)
#undef MC_CASE
  set_error("%s: unsupported dtype combination (%d, %d) -> %d", who, da, db, dout);
  return MC_ERR_INVALID;
}

// ---- CFG combine of the caller loop: out = uncond + g * (cond - uncond), each op rounded separately like torch eager --------
__global__ void __launch_bounds__(256) cfg_combine_kernel(const float* __restrict__ cond, const float* __restrict__ uncond, float g,
                                                          float* __restrict__ out, int64_t n_groups) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_groups; i += stride) {
    float c[8], u[8];
    Elem<MC_F32>::load8(cond, i * 8, c);
    Elem<MC_F32>::load8(uncond, i * 8, u);
#pragma unroll
    for (int j = 0; j < 8; ++j) c[j] = __fadd_rn(u[j], __fmul_rn(g, __fsub_rn(c[j], u[j])));
    Elem<MC_F32>::store8(out, i * 8, c);
  }
}
__global__ void cfg_combine_tail_kernel(const float* __restrict__ cond, const float* __restrict__ uncond, float g,
                                        float* __restrict__ out, int64_t begin, int64_t n) {
  const int64_t i = begin + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __fadd_rn(uncond[i], __fmul_rn(g, __fsub_rn(cond[i], uncond[i])));
}

// ---- CFG combine + scheduler update of the caller loop in one pass (SURVEY §8f rank 1) ------------------------------------
// Flow-matching samplers (Euler, FlowUniPC, FlowDPM++) all update the latent by a linear combination of the current sample,
// the guided model output and a few stored tensors with host-computed scalar coefficients:
//   v   = uncond + g * (cond - uncond)
//   out = coef_x * x + coef_v * v + sum_i coef_h[i] * hist[i]            (Euler: coef_x = 1, coef_v = sigma_next - sigma)
//   x0  = x - sigma * v                                                  (optional: the x0-prediction multistep solvers keep)
// Every product and sum is rounded separately, in this order, like the chain of torch eager kernels it replaces.
struct CfgStepArgs {
  const float* cond;
  const float* uncond;
  const float* x;
  const float* hist[4];
  float coef_h[4];
  float* out;
  float* x0_out;
  float g, coef_x, coef_v, sigma;
  int n_hist;
};

template <int NH>
__device__ __forceinline__ float cfg_step_one(const CfgStepArgs& a, float c, float u, float x, const float (&h)[4], float* x0) {
  const float v = __fadd_rn(u, __fmul_rn(a.g, __fsub_rn(c, u)));
  float acc = __fadd_rn(__fmul_rn(a.coef_x, x), __fmul_rn(a.coef_v, v));
#pragma unroll
  for (int k = 0; k < NH; ++k) acc = __fadd_rn(acc, __fmul_rn(a.coef_h[k], h[k]));
  *x0 = __fsub_rn(x, __fmul_rn(a.sigma, v));
  return acc;
}

template <int NH>
__global__ void __launch_bounds__(256) cfg_step_kernel(const CfgStepArgs a, int64_t n_groups) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_groups; i += stride) {
    float c[8], u[8], x[8], h[NH > 0 ? NH : 1][8], o[8], x0[8];
    Elem<MC_F32>::load8(a.cond, i * 8, c);
    Elem<MC_F32>::load8(a.uncond, i * 8, u);
    ptx::ld_v8_f32(a.x + i * 8, x);  // x may alias out: coherent load
#pragma unroll
    for (int k = 0; k < NH; ++k) ptx::ld_v8_f32(a.hist[k] + i * 8, h[k]);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float hj[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < NH; ++k) hj[k] = h[k][j];
      o[j] = cfg_step_one<NH>(a, c[j], u[j], x[j], hj, &x0[j]);
    }
    Elem<MC_F32>::store8(a.out, i * 8, o);
    if (a.x0_out) Elem<MC_F32>::store8(a.x0_out, i * 8, x0);
  }
}
template <int NH>
__global__ void cfg_step_tail_kernel(const CfgStepArgs a, int64_t begin, int64_t n) {
  const int64_t i = begin + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) {
    float hj[4] = {0.f, 0.f, 0.f, 0.f}, x0;
#pragma unroll
    for (int k = 0; k < NH; ++k) hj[k] = a.hist[k][i];
    const float o = cfg_step_one<NH>(a, a.cond[i], a.uncond[i], a.x[i], hj, &x0);
    a.out[i] = o;
    if (a.x0_out) a.x0_out[i] = x0;
  }
}

template <int NH>
static int32_t launch_cfg_step(const CfgStepArgs& a, int64_t groups, int64_t n, cudaStream_t s) {
  if (groups > 0) {
    const int64_t want = (groups + 255) / 256, cap = static_cast<int64_t>(num_sms()) * 8;
    cfg_step_kernel<NH><<<static_cast<int>(want < cap ? want : cap), 256, 0, s>>>(a, groups);
    MC_CHECK_LAUNCH("cfg_step_kernel launch");
  }
  if (groups * 8 < n) {
    const int64_t rem = n - groups * 8;
    cfg_step_tail_kernel<NH><<<static_cast<int>((rem + 255) / 256), 256, 0, s>>>(a, groups * 8, n);
    MC_CHECK_LAUNCH("cfg_step_tail_kernel launch");
  }
  return MC_OK;
}

// ---- TeaCache distance: sum |cur - prev| and sum |prev| of the (tiny) modulated time embedding, one CTA --------------------
__global__ void __launch_bounds__(256) rel_l1_kernel(const float* __restrict__ cur, const float* __restrict__ prev, int64_t n,
                                                     double* __restrict__ sums) {
  __shared__ double s_d[8], s_p[8];
  double d = 0.0, p = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const float c = cur[i], q = prev[i];
    d += static_cast<double>(fabsf(c - q));  // the difference is rounded to fp32 like torch's `modulated_inp - previous`
    p += static_cast<double>(fabsf(q));
  }
  for (int o = 16; o > 0; o >>= 1) {
    d += __shfl_xor_sync(0xffffffffu, d, o);
    p += __shfl_xor_sync(0xffffffffu, p, o);
  }
  if ((threadIdx.x & 31) == 0) s_d[threadIdx.x >> 5] = d, s_p[threadIdx.x >> 5] = p;
  __syncthreads();
  if (threadIdx.x == 0) {
    double td = 0.0, tp = 0.0;
    for (int w = 0; w < 8; ++w) td += s_d[w], tp += s_p[w];
    sums[0] = td;
    sums[1] = tp;
  }
}

// ---- K3: per-row norms / cosine, single pass ---------------------------------------------------------------
// Lane partial sums of one row: cur^2, prev^2 and cur * prev over 8 elements
__device__ __forceinline__ void stats_acc8(const float (&c)[8], const float (&p)[8], float& cc, float& pp, float& cp) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    cc = fmaf(c[j], c[j], cc);
    pp = fmaf(p[j], p[j], pp);
    cp = fmaf(c[j], p[j], cp);
  }
}

// End of one row (whole warp): reduce the lane partial sums, then lane 0 adds the row's norm ratio, its square and its cosine
// distance to acc[0..2] in double.
__device__ __forceinline__ void stats_row(float cc, float pp, float cp, double denom_eps, int lane, double (&acc)[3]) {
  cc = warp_sum(cc);
  pp = warp_sum(pp);
  cp = warp_sum(cp);
  if (lane == 0) {
    const float n_cur = sqrtf(cc), n_prev = sqrtf(pp);
    const float ratio = n_cur / (n_prev + static_cast<float>(denom_eps));
    // F.cosine_similarity(eps=1e-8): sum((a/max(|a|,eps)) * (b/max(|b|,eps)))
    const float cosv = cp / (fmaxf(n_cur, 1e-8f) * fmaxf(n_prev, 1e-8f));
    acc[0] += static_cast<double>(ratio);
    acc[1] += static_cast<double>(ratio) * static_cast<double>(ratio);
    acc[2] += static_cast<double>(1.0f - cosv);
  }
}

// One warp per row; lanes stride over 8-element groups. Optionally also forms cur = xo - xi on the fly and stores it.
template <int DCUR, int DPREV, bool FUSE_SUB>
__global__ void __launch_bounds__(256) stats_kernel(const void* __restrict__ cur_or_xo, const void* __restrict__ xi_bf16,
                                                    void* __restrict__ r_out, const void* __restrict__ prev, int64_t rows, int cols,
                                                    double denom_eps, double* __restrict__ stats) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps_per_block = blockDim.x >> 5;
  const int groups = cols >> 3;
  double acc[3] = {0.0, 0.0, 0.0};
  for (int64_t row = static_cast<int64_t>(blockIdx.x) * warps_per_block + warp; row < rows;
       row += static_cast<int64_t>(gridDim.x) * warps_per_block) {
    const int64_t base = row * cols;
    float cc = 0.f, pp = 0.f, cp = 0.f;
    // kBatch groups per lane are loaded before any of them is reduced: 2 x kBatch independent 128/256-bit loads in flight
    constexpr int kBatch = 3;
    for (int g0 = lane; g0 < groups; g0 += 32 * kBatch) {
      float c[kBatch][8], p[kBatch][8];
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int g = g0 + 32 * u;
        if (g < groups) {
          Elem<DCUR>::load8(cur_or_xo, base + g * 8, c[u]);
          if (FUSE_SUB) {
            float xi[8];
            Elem<MC_BF16>::load8(xi_bf16, base + g * 8, xi);
#pragma unroll
            for (int j = 0; j < 8; ++j) c[u][j] = c[u][j] - xi[j];
          }
          Elem<DPREV>::load8(prev, base + g * 8, p[u]);
        }
      }
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int g = g0 + 32 * u;
        if (g < groups) {
          if (FUSE_SUB) Elem<MC_F32>::store8(r_out, base + g * 8, c[u]);
          stats_acc8(c[u], p[u], cc, pp, cp);
        }
      }
    }
    stats_row(cc, pp, cp, denom_eps, lane, acc);
  }
  __shared__ double sh[3][8];
  if (lane == 0) {
    sh[0][warp] = acc[0];
    sh[1][warp] = acc[1];
    sh[2][warp] = acc[2];
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    double t = 0.0;
    for (int w = 0; w < warps_per_block; ++w) t += sh[threadIdx.x][w];
    atomicAdd(&stats[threadIdx.x], t);
  }
}

// TMA-staged variant for fp32 residuals (the Wan stream): the producer of a StageRing keeps kStages x (4 rows of each tensor) in
// flight, so the bytes in flight per SM (~150 KB) no longer depend on how many warps happen to be in their load phase; four
// consumer warps (one row each) reduce out of shared memory with warp shuffles. Same arithmetic as stats_kernel. FUSE_SUB
// additionally stages x_in (bf16) and writes r = x_out - x_in.
constexpr int kStatRows = 4;  // rows per stage = consumer warps
constexpr int kStatMaxStages = 6;

template <bool FUSE_SUB>
__global__ void __launch_bounds__(160) stats_tma_kernel(const float* __restrict__ cur_or_xo, const __nv_bfloat16* __restrict__ xi,
                                                        float* __restrict__ r_out, const float* __restrict__ prev, int64_t rows, int cols,
                                                        int stages, double denom_eps, double* __restrict__ stats) {
  extern __shared__ __align__(128) uint8_t smem_dyn[];
  const int row_f32 = cols * 4, row_bf16 = cols * 2;
  const StageRing ring(smem_dyn, stages, kStatRows * (2 * row_f32 + (FUSE_SUB ? row_bf16 : 0)), kStatRows);
  double* red = reinterpret_cast<double*>(ring.end());  // [3][kStatRows]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n_chunks = (rows + kStatRows - 1) / kStatRows;

  if (warp == kStatRows) {
    // ---- producer warp (one thread): bulk copies of whole row groups, rows are contiguous in memory
    if (lane == 0) {
      auto rows_in = [&](int64_t c) {
        const int64_t left = rows - c * kStatRows;
        return left < kStatRows ? static_cast<int>(left) : kStatRows;
      };
      ring.produce(
          n_chunks, [&](int64_t c) { return static_cast<uint32_t>(rows_in(c)) * (2 * row_f32 + (FUSE_SUB ? row_bf16 : 0)); },
          [&](int64_t c, uint8_t* slot, uint64_t* bar) {
            const int64_t row0 = c * kStatRows;
            const int nr = rows_in(c);
            ptx::bulk_load_1d(slot, cur_or_xo + row0 * cols, nr * row_f32, bar);
            ptx::bulk_load_1d(slot + kStatRows * row_f32, prev + row0 * cols, nr * row_f32, bar);
            if (FUSE_SUB) ptx::bulk_load_1d(slot + 2 * kStatRows * row_f32, xi + row0 * cols, nr * row_bf16, bar);
          });
    }
  } else {
    // ---- consumer warps: warp w owns row w of every stage
    double acc[3] = {0.0, 0.0, 0.0};
    const int groups = cols >> 3;
    ring.consume<1>(n_chunks, 0, [&](int64_t c, const uint8_t* stage, auto release) {
      const int64_t row = c * kStatRows + warp;
      if (row < rows) {
        const float4* cp4 = reinterpret_cast<const float4*>(stage + warp * row_f32);
        const float4* pp4 = reinterpret_cast<const float4*>(stage + kStatRows * row_f32 + warp * row_f32);
        const uint4* xp = reinterpret_cast<const uint4*>(stage + 2 * kStatRows * row_f32 + warp * row_bf16);
        float cc = 0.f, pp = 0.f, cp = 0.f;
        for (int g = lane; g < groups; g += 32) {
          float cv[8], pv[8];
          const float4 c0 = cp4[2 * g], c1 = cp4[2 * g + 1], p0 = pp4[2 * g], p1 = pp4[2 * g + 1];
          cv[0] = c0.x; cv[1] = c0.y; cv[2] = c0.z; cv[3] = c0.w; cv[4] = c1.x; cv[5] = c1.y; cv[6] = c1.z; cv[7] = c1.w;
          pv[0] = p0.x; pv[1] = p0.y; pv[2] = p0.z; pv[3] = p0.w; pv[4] = p1.x; pv[5] = p1.y; pv[6] = p1.z; pv[7] = p1.w;
          if (FUSE_SUB) {
            float xv[8];
            unpack_bf16x8(xp[g], xv);
#pragma unroll
            for (int j = 0; j < 8; ++j) cv[j] = cv[j] - xv[j];
            Elem<MC_F32>::store8(r_out, row * cols + g * 8, cv);
          }
          stats_acc8(cv, pv, cc, pp, cp);
        }
        stats_row(cc, pp, cp, denom_eps, lane, acc);
      }
      release();  // this warp is done reading the stage
    });
    if (lane == 0) {
      red[0 * kStatRows + warp] = acc[0];
      red[1 * kStatRows + warp] = acc[1];
      red[2 * kStatRows + warp] = acc[2];
    }
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    double t = 0.0;
    for (int w = 0; w < kStatRows; ++w) t += red[threadIdx.x * kStatRows + w];
    atomicAdd(&stats[threadIdx.x], t);
  }
}

__global__ void stats_init_kernel(double* stats, double rows) {
  if (threadIdx.x < 3) stats[threadIdx.x] = 0.0;
  if (threadIdx.x == 3) stats[3] = rows;
}

template <int DCUR, int DPREV, bool FUSE>
static int32_t launch_stats(const void* cur, const void* xi, void* r_out, const void* prev, int64_t rows, int cols, double eps,
                            double* stats, cudaStream_t s) {
  stats_init_kernel<<<1, 32, 0, s>>>(stats, static_cast<double>(rows));
  MC_CHECK_LAUNCH("stats_init_kernel launch");
  if (DCUR == MC_F32 && DPREV == MC_F32) {
    // TMA-staged path when at least two stages of 4 rows fit in shared memory (cols <= ~3000 for the plain statistics)
    const int stage_bytes = kStatRows * (2 * cols * 4 + (FUSE ? cols * 2 : 0));
    const int stages = ring_stages(stage_bytes, kStatMaxStages);
    if (stages > 0)
      return launch_ring<stats_tma_kernel<FUSE>>(stages, stage_bytes, 3 * kStatRows * 8, (rows + kStatRows - 1) / kStatRows, (kStatRows + 1) * 32,
                                                 s, "stats_tma_kernel", static_cast<const float*>(cur), static_cast<const __nv_bfloat16*>(xi),
                                                 static_cast<float*>(r_out), static_cast<const float*>(prev), rows, cols, stages, eps, stats);
  }
  const int threads = 256, wpb = threads / 32;
  int64_t want = (rows + wpb - 1) / wpb;
  const int64_t cap = static_cast<int64_t>(num_sms()) * 8;
  const int grid = static_cast<int>(want < cap ? (want < 1 ? 1 : want) : cap);
  stats_kernel<DCUR, DPREV, FUSE><<<grid, threads, 0, s>>>(cur, xi, r_out, prev, rows, cols, eps, stats);
  MC_CHECK_LAUNCH("stats_kernel launch");
  return MC_OK;
}

// ---- FP8 weight dequantisation: out[r, c] = bf16_rn(float(q[r, c]) * float(scale[r])) ----------------------------------------
// float(e4m3) is exact in fp16 and fp32, and the product of a 4-bit and an 8-bit significand is exact in fp32, so the one rounding
// is the bf16 one: bit-equal to `q.to(bf16) * scale.to(bf16)` (hyvideo fp8_activation_dequant). e4m3 0x7F / 0xFF decode to NaN.
__device__ __forceinline__ float2 e4m3x2_to_f32x2(uint32_t pair) {  // low byte -> .x, high byte -> .y
  uint32_t h2;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(static_cast<unsigned short>(pair & 0xFFFFu)));
  __half2 h;
  memcpy(&h, &h2, 4);
  return __half22float2(h);
}

// one 16-byte word of codes (16 elements of one row) -> two 16-byte words of bf16; grid-stride over the words
__global__ void __launch_bounds__(256) dequant_fp8_kernel(const uint8_t* __restrict__ q, const __nv_bfloat16* __restrict__ scale,
                                                          __nv_bfloat16* __restrict__ out, int64_t n_words, int64_t words_per_row) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t g = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; g < n_words; g += stride) {
    const uint4 w = ptx::ld_nc_v4(q + g * 16);
    const float s = __bfloat162float(scale[g / words_per_row]);
    const uint32_t wd[4] = {w.x, w.y, w.z, w.w};
    float f[2][8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 a = e4m3x2_to_f32x2(wd[k]), b = e4m3x2_to_f32x2(wd[k] >> 16);
      f[k / 2][(k % 2) * 4 + 0] = __fmul_rn(a.x, s);
      f[k / 2][(k % 2) * 4 + 1] = __fmul_rn(a.y, s);
      f[k / 2][(k % 2) * 4 + 2] = __fmul_rn(b.x, s);
      f[k / 2][(k % 2) * 4 + 3] = __fmul_rn(b.y, s);
    }
    // plain stores: the GEMM that follows reads this scratch right away, so whatever of it stays in L2 is a hit
    uint4* o = reinterpret_cast<uint4*>(out + g * 16);
    o[0] = pack_bf16x8(f[0]);
    o[1] = pack_bf16x8(f[1]);
  }
}

// any row length / alignment: one element per thread
__global__ void __launch_bounds__(256) dequant_fp8_scalar_kernel(const uint8_t* __restrict__ q, const __nv_bfloat16* __restrict__ scale,
                                                                 __nv_bfloat16* __restrict__ out, int64_t n, int64_t cols) {
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = __float2bfloat16_rn(__fmul_rn(e4m3x2_to_f32x2(q[i]).x, __bfloat162float(scale[i / cols])));
}

}  // namespace mc

extern "C" {

int32_t mc_dequant_fp8_bf16(const void* q, const void* scale, void* out, int64_t rows, int32_t cols, void* stream) {
  MC_CHECK_ARG(rows >= 0 && cols >= 1, "mc_dequant_fp8_bf16: rows=%lld cols=%d", static_cast<long long>(rows), cols);
  if (rows == 0) return MC_OK;
  MC_CHECK_ARG(q && scale && out, "mc_dequant_fp8_bf16: null pointer");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t n = rows * cols;
  const int64_t cap = static_cast<int64_t>(mc::num_sms()) * 8;  // 8 resident CTAs of 256 threads per SM
  if (cols % 16 == 0 && mc::aligned16(q) && mc::aligned16(out)) {
    const int64_t words = n / 16, want = (words + 255) / 256;
    mc::dequant_fp8_kernel<<<static_cast<int>(want < cap ? want : cap), 256, 0, s>>>(
        static_cast<const uint8_t*>(q), static_cast<const __nv_bfloat16*>(scale), static_cast<__nv_bfloat16*>(out), words, cols / 16);
    MC_CHECK_LAUNCH("dequant_fp8_kernel launch");
    return MC_OK;
  }
  const int64_t want = (n + 255) / 256;
  mc::dequant_fp8_scalar_kernel<<<static_cast<int>(want < cap ? want : cap), 256, 0, s>>>(
      static_cast<const uint8_t*>(q), static_cast<const __nv_bfloat16*>(scale), static_cast<__nv_bfloat16*>(out), n, cols);
  MC_CHECK_LAUNCH("dequant_fp8_scalar_kernel launch");
  return MC_OK;
}

int32_t mc_cache_hit_add(const void* x, int32_t x_dtype, const void* r, int32_t r_dtype, void* out, int32_t out_dtype, int64_t n,
                         void* stream) {
  return mc::dispatch_axpb(x, x_dtype, r, r_dtype, out, out_dtype, n, 1.0f, static_cast<cudaStream_t>(stream), "mc_cache_hit_add");
}

int32_t mc_residual_sub(const void* x_out, int32_t xo_dtype, const void* x_in, int32_t xi_dtype, void* r, int32_t r_dtype, int64_t n,
                        void* stream) {
  return mc::dispatch_axpb(x_out, xo_dtype, x_in, xi_dtype, r, r_dtype, n, -1.0f, static_cast<cudaStream_t>(stream),
                           "mc_residual_sub");
}

int32_t mc_cfg_combine(const float* cond, const float* uncond, float guide_scale, float* out, int64_t n, void* stream) {
  MC_CHECK_ARG(n >= 0, "mc_cfg_combine: negative element count");
  if (n == 0) return MC_OK;
  MC_CHECK_ARG(cond && uncond && out, "mc_cfg_combine: null pointer");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  auto al32 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 31u) == 0; };
  const int64_t groups = (al32(cond) && al32(uncond) && al32(out)) ? n / 8 : 0;
  if (groups > 0) {
    int64_t want = (groups + 255) / 256;
    const int64_t cap = static_cast<int64_t>(mc::num_sms()) * 8;
    mc::cfg_combine_kernel<<<static_cast<int>(want < cap ? want : cap), 256, 0, s>>>(cond, uncond, guide_scale, out, groups);
    MC_CHECK_LAUNCH("cfg_combine_kernel launch");
  }
  if (groups * 8 < n) {
    const int64_t rem = n - groups * 8;
    mc::cfg_combine_tail_kernel<<<static_cast<int>((rem + 255) / 256), 256, 0, s>>>(cond, uncond, guide_scale, out, groups * 8, n);
    MC_CHECK_LAUNCH("cfg_combine_tail_kernel launch");
  }
  return MC_OK;
}

int32_t mc_rel_l1(const float* cur, const float* prev, int64_t n, double* sums_dev, void* stream) {
  MC_CHECK_ARG(cur && prev && sums_dev && n >= 1, "mc_rel_l1: bad arguments");
  mc::rel_l1_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(cur, prev, n, sums_dev);
  MC_CHECK_LAUNCH("rel_l1_kernel launch");
  return MC_OK;
}

int32_t mc_cfg_step(const float* cond, const float* uncond, float guide_scale, const float* x, float coef_x, float coef_v,
                    const float* const* hist, const float* coef_h, int32_t n_hist, float sigma, float* out, float* x0_out, int64_t n,
                    void* stream) {
  MC_CHECK_ARG(n >= 0, "mc_cfg_step: negative element count");
  MC_CHECK_ARG(n_hist >= 0 && n_hist <= 4, "mc_cfg_step: n_hist=%d outside [0, 4]", n_hist);
  if (n == 0) return MC_OK;
  MC_CHECK_ARG(cond && uncond && x && out, "mc_cfg_step: null pointer");
  MC_CHECK_ARG(n_hist == 0 || (hist && coef_h), "mc_cfg_step: null history arrays");
  MC_CHECK_ARG(out != cond && out != uncond && x0_out != cond && x0_out != uncond && (x0_out == nullptr || (x0_out != out && x0_out != x)),
               "mc_cfg_step: out may alias x only; x0_out must be a separate buffer");
  mc::CfgStepArgs a{};
  a.cond = cond, a.uncond = uncond, a.x = x, a.out = out, a.x0_out = x0_out;
  a.g = guide_scale, a.coef_x = coef_x, a.coef_v = coef_v, a.sigma = sigma, a.n_hist = n_hist;
  auto al32 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 31u) == 0; };
  bool aligned = al32(cond) && al32(uncond) && al32(x) && al32(out) && (x0_out == nullptr || al32(x0_out));
  for (int k = 0; k < n_hist; ++k) {
    MC_CHECK_ARG(hist[k] != nullptr && hist[k] != out && hist[k] != x0_out, "mc_cfg_step: hist[%d] is null or aliases an output", k);
    a.hist[k] = hist[k], a.coef_h[k] = coef_h[k];
    aligned = aligned && al32(hist[k]);
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t groups = aligned ? n / 8 : 0;
  switch (n_hist) {
    case 0: return mc::launch_cfg_step<0>(a, groups, n, s);
    case 1: return mc::launch_cfg_step<1>(a, groups, n, s);
    case 2: return mc::launch_cfg_step<2>(a, groups, n, s);
    case 3: return mc::launch_cfg_step<3>(a, groups, n, s);
    default: return mc::launch_cfg_step<4>(a, groups, n, s);
  }
}

int32_t mc_residual_stats(const void* r_cur, int32_t cur_dtype, const void* r_prev, int32_t prev_dtype, int64_t rows, int32_t cols,
                          double denom_eps, double* stats_dev, void* stream) {
  MC_CHECK_ARG(r_cur && r_prev && stats_dev, "mc_residual_stats: null pointer");
  MC_CHECK_ARG(rows >= 1 && cols >= 8 && cols % 8 == 0, "mc_residual_stats: rows=%lld cols=%d (cols must be a multiple of 8)",
               static_cast<long long>(rows), cols);
  MC_CHECK_ARG((reinterpret_cast<uintptr_t>(r_cur) & 31u) == 0 && (reinterpret_cast<uintptr_t>(r_prev) & 31u) == 0,
               "mc_residual_stats: pointers must be 32-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (cur_dtype == MC_F32 && prev_dtype == MC_F32)
    return mc::launch_stats<MC_F32, MC_F32, false>(r_cur, nullptr, nullptr, r_prev, rows, cols, denom_eps, stats_dev, s);
  if (cur_dtype == MC_BF16 && prev_dtype == MC_BF16)
    return mc::launch_stats<MC_BF16, MC_BF16, false>(r_cur, nullptr, nullptr, r_prev, rows, cols, denom_eps, stats_dev, s);
  mc::set_error("mc_residual_stats: unsupported dtypes (%d, %d)", cur_dtype, prev_dtype);
  return MC_ERR_INVALID;
}

int32_t mc_residual_sub_stats(const void* x_out, int32_t xo_dtype, const void* x_in, int32_t xi_dtype, void* r, const void* r_prev,
                              int64_t rows, int32_t cols, double denom_eps, double* stats_dev, void* stream) {
  MC_CHECK_ARG(x_out && x_in && r && r_prev && stats_dev, "mc_residual_sub_stats: null pointer");
  MC_CHECK_ARG(xo_dtype == MC_F32 && xi_dtype == MC_BF16, "mc_residual_sub_stats: only fp32 - bf16 -> fp32 (the Wan stream) is built");
  MC_CHECK_ARG(rows >= 1 && cols >= 8 && cols % 8 == 0, "mc_residual_sub_stats: cols must be a multiple of 8");
  MC_CHECK_ARG((reinterpret_cast<uintptr_t>(x_out) & 31u) == 0 && mc::aligned16(x_in) && (reinterpret_cast<uintptr_t>(r) & 31u) == 0 &&
                   (reinterpret_cast<uintptr_t>(r_prev) & 31u) == 0,
               "mc_residual_sub_stats: fp32 pointers must be 32-byte aligned, bf16 16-byte");
  return mc::launch_stats<MC_F32, MC_F32, true>(x_out, x_in, r, r_prev, rows, cols, denom_eps, stats_dev,
                                                static_cast<cudaStream_t>(stream));
}

}  // extern "C"
