// Row-wise (token-local) kernels of the cache-miss branch — all HBM-bound, fp32 statistics, 128-bit accesses.
// Arithmetic follows upstream Wan2.1 wan/modules/model.py as restated in SURVEY.md Appendix B.1; call sites in the
// reference: MagCache4Wan2.1/magcache_generate.py:237 (patch_embedding), :249-254 (time embedding),
// :297-298 (block stack), :304-305 (head, unpatchify).
#include <type_traits>

#include "common.cuh"
#include "ptx.cuh"
#include "ring.cuh"
#include "rowwise.cuh"

namespace mc {

// A row's 8-element groups are spread over the lanes that share the row, each lane keeping up to kMaxG groups in registers: one
// warp per row covers cols <= 2048; the wide forms, a team of kWideWarps warps per row, cover cols <= 8192.
constexpr int kMaxG = 8;
constexpr int kWideWarps = 4;

// sum over the kWideWarps warps of a team (scratch: [teams per block][kWideWarps])
__device__ __forceinline__ float team_sum(float v, float* scratch, int team, int lane_in_team) {
  v = warp_sum(v);
  const int w = lane_in_team >> 5;
  __syncthreads();  // protect scratch reuse between consecutive reductions
  if ((lane_in_team & 31) == 0) scratch[team * kWideWarps + w] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < kWideWarps; ++i) t += scratch[team * kWideWarps + i];
  return t;
}

__device__ __forceinline__ void load_row_group(const void* x, int dtype_bf16, int64_t off, float (&f)[8]) {
  if (dtype_bf16) {
    uint4 v = ptx::ld_nc_v4(static_cast<const __nv_bfloat16*>(x) + off);
    unpack_bf16x8(v, f);
  } else {
    ptx::ld_nc_v8_f32(static_cast<const float*>(x) + off, f);
  }
}

// ---- per-row arithmetic: every launch form below calls these (and ln_rstd / t2i_modulate8 of rowwise.cuh), so all forms give
// the same bits -------------------------------------------------------------------------------------------------------------
// Output of modes 0 / 1 for 8 elements of a row: y = LN(x) * (1 + a) + b (mode 0) or LN(x) * a + b (mode 1), a and b the
// per-column parameters at pa / pb, the LN value first rounded to bf16 when round_ln; stored at out + off as bf16 or fp32.
__device__ __forceinline__ void ln_modulate_store8(const float (&v)[8], float mean, float rstd, const float* pa, const float* pb, int mode,
                                                   int round_ln, void* out, int out_bf16, int64_t off) {
  float a[8], b[8], o[8];
  load_param8(pa, a);
  load_param8(pb, b);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float y = (v[j] - mean) * rstd;
    if (round_ln) y = round_bf16(y);
    const float aa = (mode == 0) ? 1.0f + a[j] : a[j];
    o[j] = __fadd_rn(__fmul_rn(y, aa), b[j]);  // torch eager: separate mul and add, no FMA contraction
  }
  if (out_bf16) {
    ptx::st_na_v4(static_cast<__nv_bfloat16*>(out) + off, pack_bf16x8(o));
  } else {
    ptx::st_na_v8_f32(static_cast<float*>(out) + off, o);
  }
}

// WanRMSNorm of 8 elements given r = rsqrt(mean(x^2) + eps): _norm(x.float()).type_as(x) * weight, the weight at w
__device__ __forceinline__ void rms_weight8(const float (&x)[8], float r, const float* w, float (&o)[8]) {
  float wv[8];
  load_param8(w, wv);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = round_bf16(x[j] * r) * wv[j];
}

// ---- K7: LayerNorm (no affine) + modulation / affine, optional bf16 rounding of the LN output -----------------
//   mode 0: y = LN(x) * (1 + p0[scale_idx]) + p0[shift_idx]   with p0 = e = modulation + e0, fp32 [k, cols]
//   mode 1: y = LN(x) * p0 + p1                               (elementwise affine)
// Wide form (cols > 2048): a team of kWideWarps warps per row.
__global__ void __launch_bounds__(256) ln_modulate_kernel(const void* __restrict__ x, int x_bf16, int64_t rows, int cols, float eps,
                                                          int mode, const float* __restrict__ p0, const float* __restrict__ p1,
                                                          int scale_idx, int shift_idx, int round_ln, void* __restrict__ out,
                                                          int out_bf16) {
  constexpr int TPR = 32 * kWideWarps, RPB = 256 / TPR;  // threads per row, rows per block
  __shared__ float scratch[RPB * kWideWarps];
  const int team = threadIdx.x / TPR, lt = threadIdx.x % TPR;
  const int groups = cols >> 3;
  const float inv_n = 1.0f / static_cast<float>(cols);
  const float* pa = (mode == 0) ? p0 + static_cast<int64_t>(scale_idx) * cols : p0;
  const float* pb = (mode == 0) ? p0 + static_cast<int64_t>(shift_idx) * cols : p1;
  for (int64_t row0 = static_cast<int64_t>(blockIdx.x) * RPB; row0 < rows; row0 += static_cast<int64_t>(gridDim.x) * RPB) {
    const int64_t row = row0 + team;
    const int live_groups = row < rows ? groups : 0;  // a team past the last row still takes part in the block's reductions
    float v[kMaxG][8];
#pragma unroll
    for (int i = 0; i < kMaxG; ++i) {
      const int g = lt + i * TPR;
      if (g < live_groups) load_row_group(x, x_bf16, row * cols + g * 8, v[i]);
    }
    float mean;
    const float rstd = ln_rstd<kMaxG>(v, lt, TPR, live_groups, inv_n, eps, [&](float t) { return team_sum(t, scratch, team, lt); }, mean);
#pragma unroll
    for (int i = 0; i < kMaxG; ++i) {
      const int g = lt + i * TPR;
      if (g < live_groups) ln_modulate_store8(v[i], mean, rstd, pa + g * 8, pb + g * 8, mode, round_ln, out, out_bf16, row * cols + g * 8);
    }
  }
}

// ---- mode 2: LayerNorm + t2i_modulate with every step a bf16 tensor op (STDiT3Block.forward, open_sora_transformer_3d.py:187, :248;
// T2IFinalLayer, :80): y = bf16(bf16(bf16(LN(x)) * bf16(1 + p0[scale_idx])) + p0[shift_idx]), p0 holding bf16 values.
// One warp per row, x and out bf16, cols <= 2048.
// kRelL1: TeaCache's input distance (eval/magcache/experiments/opensora.py:102) against `prev`, the previous call's output of the
// same shape, taken while the output row is in registers: each warp adds Σ float(|bf16(out - prev)|) and Σ float(|prev|) of its rows
// (fp32 within a row, fp64 across rows), the CTA's warps are added in warp order into partials[blockIdx.x] = {Σ|d|, Σ|prev|}, and
// rel_l1_finish_kernel adds the partials in a fixed order: no floating-point atomics, the same bits on every launch.
// G: 8-element groups per lane (cols <= 256 G); the plain form is instantiated at kMaxG. The distance forms up to G = 6 fit two
// CTAs per SM (<= 128 registers), like the plain form.
template <int G, bool kRelL1>
__global__ void __launch_bounds__(256, (kRelL1 && G < 8) ? 2 : 0) ln_t2i_modulate_kernel(const __nv_bfloat16* __restrict__ x, int64_t rows, int cols, float eps,
                                                              const float* __restrict__ sc, const float* __restrict__ sh,
                                                              __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ prev,
                                                              double2* __restrict__ partials) {
  const int lane = threadIdx.x & 31;
  const int groups = cols >> 3;
  const float inv_n = 1.0f / static_cast<float>(cols);
  double acc_d = 0.0, acc_p = 0.0;  // kRelL1: this warp's rows (lane 0)
  for (int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; row < rows;
       row += (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5) {
    float v[G][8];
    uint4 pv[kRelL1 ? G : 1];
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int g = lane + i * 32;
      if (g < groups) {
        unpack_bf16x8(ptx::ld_nc_v4(x + row * cols + g * 8), v[i]);
        if constexpr (kRelL1) pv[i] = ptx::ld_nc_v4(prev + row * cols + g * 8);
      }
    }
    float mean;
    const float rstd = ln_rstd<G>(v, lane, 32, groups, inv_n, eps, WarpReduce(), mean);
    float sd = 0.f, sp = 0.f;
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int g = lane + i * 32;
      if (g < groups) {
        float o[8];
        t2i_modulate8(v[i], mean, rstd, sc + g * 8, sh + g * 8, o);
        ptx::st_na_v4(out + row * cols + g * 8, pack_bf16x8(o));
        if constexpr (kRelL1) {
          float p[8];
          unpack_bf16x8(pv[i], p);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            sd += fabsf(round_bf16(__fsub_rn(o[j], p[j])));  // `(cur - prev)` is a bf16 tensor op, then `.abs()`
            sp += fabsf(p[j]);
          }
        }
      }
    }
    if constexpr (kRelL1) {
      sd = warp_sum(sd);
      sp = warp_sum(sp);
      acc_d += static_cast<double>(sd);
      acc_p += static_cast<double>(sp);
    }
  }
  if constexpr (kRelL1) {
    __shared__ double2 warp_acc[8];
    if (lane == 0) warp_acc[threadIdx.x >> 5] = make_double2(acc_d, acc_p);
    __syncthreads();
    if (threadIdx.x == 0) {
      double2 t = warp_acc[0];
      for (int w = 1; w < static_cast<int>(blockDim.x >> 5); ++w) {
        t.x += warp_acc[w].x;
        t.y += warp_acc[w].y;
      }
      partials[blockIdx.x] = t;
    }
  }
}

// sums[0..1] += the n partials of ln_t2i_modulate_kernel<true>, added in a fixed order: 256 threads each take a fixed strided
// subset, then a shared-memory tree. One CTA.
__global__ void __launch_bounds__(256) rel_l1_finish_kernel(const double2* __restrict__ partials, int n, double* __restrict__ sums) {
  __shared__ double2 s[256];
  double2 t = make_double2(0.0, 0.0);
  for (int i = threadIdx.x; i < n; i += 256) {
    t.x += partials[i].x;
    t.y += partials[i].y;
  }
  s[threadIdx.x] = t;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (static_cast<int>(threadIdx.x) < h) {
      s[threadIdx.x].x += s[threadIdx.x + h].x;
      s[threadIdx.x].y += s[threadIdx.x + h].y;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    sums[0] += s[0].x;
    sums[1] += s[0].y;
  }
}

// ---- WanRMSNorm over the model dim (+ optional 3-axis RoPE), in place on bf16 ---------------------------------
// Wide form (cols > 2048): a team of kWideWarps warps per row.
__global__ void __launch_bounds__(256) rmsnorm_rope_kernel(__nv_bfloat16* __restrict__ x, int64_t ld, int64_t rows, int cols,
                                                           const float* __restrict__ w, float eps,
                                                           const float* __restrict__ cos_sin, int head_dim) {
  constexpr int TPR = 32 * kWideWarps, RPB = 256 / TPR;
  __shared__ float scratch[RPB * kWideWarps];
  const int team = threadIdx.x / TPR, lt = threadIdx.x % TPR;
  const int groups = cols >> 3;
  const float inv_n = 1.0f / static_cast<float>(cols);
  for (int64_t row0 = static_cast<int64_t>(blockIdx.x) * RPB; row0 < rows; row0 += static_cast<int64_t>(gridDim.x) * RPB) {
    const int64_t row = row0 + team;
    const bool live = row < rows;
    float v[kMaxG][8];
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxG; ++i) {
      const int g = lt + i * TPR;
      if (live && g < groups) {
        const uint4 raw = *reinterpret_cast<const uint4*>(x + row * ld + g * 8);  // coherent: updated in place below
        unpack_bf16x8(raw, v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) q = fmaf(v[i][j], v[i][j], q);
      }
    }
    const float r = rsqrtf(team_sum(q, scratch, team, lt) * inv_n + eps);
#pragma unroll
    for (int i = 0; i < kMaxG; ++i) {
      const int g = lt + i * TPR;
      if (live && g < groups) {
        const int c0 = g * 8;
        float o[8];
        rms_weight8(v[i], r, w + c0, o);
        if (cos_sin != nullptr) {
          float cs[8];
          ptx::ld_nc_v8_f32(cos_sin + row * head_dim + c0 % head_dim, cs);  // position inside the head; 8 elements = 4 pairs
          rope_pairs4(o, cs);
        }
        *reinterpret_cast<uint4*>(x + row * ld + c0) = pack_bf16x8(o);
      }
    }
  }
}

// ---- warp-per-row forms of the two kernels above with the NEXT row's loads in flight while the current row is reduced and
// stored (two register buffers in ping-pong). The plain forms keep one row per warp in flight and spend half their time
// in the reduce / store phase: ~3.4 TB/s on 32760 x 1536; with 2 rows x 16 warps per SM in flight the loads never drain.
// G = 8-element groups per lane (cols <= 256 G); instantiated for the widths the engines use. (fp32 rows of G >= 6 groups need
// 2 x 48+ registers for the two buffers: one block of 8 warps per SM, 96 KB of loads in flight.)
template <int G>
__global__ void __launch_bounds__(256, (G >= 6 ? 1 : 2)) ln_modulate_pipe_kernel(const void* __restrict__ x, int x_bf16, int64_t rows, int cols, float eps,
                                                                  int mode, const float* __restrict__ p0, const float* __restrict__ p1,
                                                                  int scale_idx, int shift_idx, int round_ln, void* __restrict__ out,
                                                                  int out_bf16) {
  const int lane = threadIdx.x & 31;
  const int groups = cols >> 3;
  const float inv_n = 1.0f / static_cast<float>(cols);
  const float* pa = (mode == 0) ? p0 + static_cast<int64_t>(scale_idx) * cols : p0;
  const float* pb = (mode == 0) ? p0 + static_cast<int64_t>(shift_idx) * cols : p1;
  const int64_t stride = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  auto load = [&](int64_t row, float (&v)[G][8]) {
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int g = lane + i * 32;
      if (g < groups) load_row_group(x, x_bf16, row * cols + g * 8, v[i]);
    }
  };
  auto process = [&](int64_t row, float (&v)[G][8]) {
    float mean;
    const float rstd = ln_rstd<G>(v, lane, 32, groups, inv_n, eps, WarpReduce(), mean);
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int c0 = (lane + i * 32) * 8;
      if (c0 < cols) ln_modulate_store8(v[i], mean, rstd, pa + c0, pb + c0, mode, round_ln, out, out_bf16, row * cols + c0);
    }
  };
  float va[G][8], vb[G][8];
  int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (row < rows) load(row, va);
  for (; row < rows; row += 2 * stride) {
    const int64_t r1 = row + stride, r2 = row + 2 * stride;
    if (r1 < rows) load(r1, vb);
    process(row, va);
    if (r1 < rows) {
      if (r2 < rows) load(r2, va);
      process(r1, vb);
    }
  }
}

// In-place WanRMSNorm (+ RoPE) over `segs` adjacent column blocks of `cols` columns per token (q | k of the fused projection in
// one launch: weight [segs, cols]); one warp per (token, block), the next one's loads in flight.
template <int G>
__global__ void __launch_bounds__(256, 2) rmsnorm_rope_pipe_kernel(__nv_bfloat16* __restrict__ x, int64_t ld, int64_t rows, int segs, int cols,
                                                                   const float* __restrict__ w, float eps,
                                                                   const float* __restrict__ cos_sin, int head_dim) {
  const int lane = threadIdx.x & 31;
  const int groups = cols >> 3;
  const float inv_n = 1.0f / static_cast<float>(cols);
  const int64_t items = rows * segs;
  const int64_t stride = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  auto load = [&](int64_t it, uint4 (&v)[G]) {
    const int64_t row = it / segs;
    const int seg = static_cast<int>(it - row * segs);
    const __nv_bfloat16* px = x + row * ld + static_cast<int64_t>(seg) * cols;
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int g = lane + i * 32;
      if (g < groups) v[i] = *reinterpret_cast<const uint4*>(px + g * 8);  // coherent: updated in place below
    }
  };
  auto process = [&](int64_t it, uint4 (&raw)[G]) {
    const int64_t row = it / segs;
    const int seg = static_cast<int>(it - row * segs);
    __nv_bfloat16* px = x + row * ld + static_cast<int64_t>(seg) * cols;
    const float* ws = w + static_cast<int64_t>(seg) * cols;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < G; ++i)
      if (lane + i * 32 < groups) {
        float f[8];
        unpack_bf16x8(raw[i], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) q = fmaf(f[j], f[j], q);
      }
    const float r = rsqrtf(warp_sum(q) * inv_n + eps);
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int g = lane + i * 32;
      if (g < groups) {
        const int c0 = g * 8;
        float f[8], o[8];
        unpack_bf16x8(raw[i], f);
        rms_weight8(f, r, ws + c0, o);
        if (cos_sin != nullptr) {
          float cs[8];
          ptx::ld_nc_v8_f32(cos_sin + row * head_dim + c0 % head_dim, cs);  // position inside the head; 8 elements = 4 pairs
          rope_pairs4(o, cs);
        }
        *reinterpret_cast<uint4*>(px + c0) = pack_bf16x8(o);
      }
    }
  };
  uint4 va[G], vb[G];
  int64_t it = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (it < items) load(it, va);
  for (; it < items; it += 2 * stride) {
    const int64_t i1 = it + stride, i2 = it + 2 * stride;
    if (i1 < items) load(i1, vb);
    process(it, va);
    if (i1 < items) {
      if (i2 < items) load(i2, va);
      process(i1, vb);
    }
  }
}

// ---- TMA-staged forms of the same two kernels: the register-pipelined forms above keep one row per warp in flight (48-96 KB
// per SM), which is short of the ~60 KB x latency a 6.5 TB/s stream needs once the warps also reduce, compute and store
// (3.2-3.9 TB/s measured on 32760 x 1536). Here the producer of a StageRing keeps `stages` x 8 rows in flight (144-192 KB per
// SM); NG groups of eight consumer warps take the stages in turn, one row of the stage per warp: copy it to registers, hand the
// slot back at once, then run the same arithmetic as the forms above. One CTA per SM, chunks of 8 rows strided over the grid.
// The consumers, not the loads, bound these kernels: 8 warps 4.2 TB/s, 16 warps 4.7 TB/s on fp32 rows (24 warps spill at 80
// registers); the bf16 RMSNorm rows take 24 warps: 3.2 -> 5.1 TB/s.
constexpr int kRingRows = 8;                                                   // rows (or (token, block) items) per stage
constexpr int ring_threads(int groups) { return (groups * kRingRows + 1) * 32; }  // + the producer warp
constexpr int kLnRingGroups = 2, kRmsRingGroups = 3;
constexpr int kRowRingMaxStages = 8;

template <int G, int NG>
__global__ void __launch_bounds__(ring_threads(NG), 1) ln_modulate_tma_kernel(const void* __restrict__ x, int x_bf16, int64_t rows, int cols, float eps,
                                                                         int mode, const float* __restrict__ p0, const float* __restrict__ p1,
                                                                         int scale_idx, int shift_idx, int round_ln, void* __restrict__ out,
                                                                         int out_bf16, int stages) {
  extern __shared__ __align__(128) uint8_t smem_dyn[];
  const int row_bytes = cols * (x_bf16 ? 2 : 4);
  const StageRing ring(smem_dyn, stages, kRingRows * row_bytes, kRingRows);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n_chunks = (rows + kRingRows - 1) / kRingRows;

  if (warp == NG * kRingRows) {
    if (lane == 0) {
      auto bytes = [&](int64_t c) {
        const int64_t left = rows - c * kRingRows;
        return static_cast<uint32_t>(left < kRingRows ? left : kRingRows) * row_bytes;
      };
      ring.produce(n_chunks, bytes, [&](int64_t c, uint8_t* slot, uint64_t* bar) {  // rows are contiguous: one copy
        ptx::bulk_load_1d(slot, static_cast<const uint8_t*>(x) + c * kRingRows * row_bytes, bytes(c), bar);
      });
    }
    return;
  }

  const int groups = cols >> 3;
  const float inv_n = 1.0f / static_cast<float>(cols);
  const float* pa = (mode == 0) ? p0 + static_cast<int64_t>(scale_idx) * cols : p0;
  const float* pb = (mode == 0) ? p0 + static_cast<int64_t>(shift_idx) * cols : p1;
  const int grp = warp / kRingRows, wr = warp - grp * kRingRows;  // consumer group, row of the stage
  ring.consume<NG>(n_chunks, grp, [&](int64_t c, const uint8_t* stage, auto release) {
    const int64_t row = c * kRingRows + wr;
    const uint8_t* rp = stage + wr * row_bytes;
    float v[G][8];
    if (row < rows) {
#pragma unroll
      for (int i = 0; i < G; ++i) {
        const int g = lane + i * 32;
        if (g < groups) {
          if (x_bf16) {
            unpack_bf16x8(*reinterpret_cast<const uint4*>(rp + g * 16), v[i]);
          } else {
            const float4 a = *reinterpret_cast<const float4*>(rp + g * 32), b = *reinterpret_cast<const float4*>(rp + g * 32 + 16);
            v[i][0] = a.x; v[i][1] = a.y; v[i][2] = a.z; v[i][3] = a.w; v[i][4] = b.x; v[i][5] = b.y; v[i][6] = b.z; v[i][7] = b.w;
          }
        }
      }
    }
    release();  // the row is in registers: the slot can be refilled while it is processed
    if (row >= rows) return;
    float mean;
    const float rstd = ln_rstd<G>(v, lane, 32, groups, inv_n, eps, WarpReduce(), mean);
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int g = lane + i * 32;
      if (g < groups) ln_modulate_store8(v[i], mean, rstd, pa + g * 8, pb + g * 8, mode, round_ln, out, out_bf16, row * cols + g * 8);
    }
  });
}

// items = (token, block); the `segs` blocks of a token are adjacent in memory, so a stage of 8 items is 8 / segs pitched rows of
// segs * cols elements (one bulk copy each) plus their RoPE rows (contiguous: one bulk copy).
template <int G, int NG>
__global__ void __launch_bounds__(ring_threads(NG), 1) rmsnorm_rope_tma_kernel(__nv_bfloat16* __restrict__ x, int64_t ld, int64_t rows, int segs, int cols,
                                                                          const float* __restrict__ w, float eps,
                                                                          const float* __restrict__ cos_sin, int head_dim, int stages) {
  extern __shared__ __align__(128) uint8_t smem_dyn[];
  const int item_bytes = cols * 2;
  const int rows_per_stage = kRingRows / segs;  // segs in {1, 2, 4}
  const int cs_row_bytes = cos_sin != nullptr ? head_dim * 4 : 0;
  const StageRing ring(smem_dyn, stages, kRingRows * item_bytes + rows_per_stage * cs_row_bytes, kRingRows);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n_chunks = (rows + rows_per_stage - 1) / rows_per_stage;

  if (warp == NG * kRingRows) {
    if (lane == 0) {
      const uint32_t per_row = static_cast<uint32_t>(segs) * item_bytes;
      auto rows_in = [&](int64_t c) {
        const int64_t left = rows - c * rows_per_stage;
        return left < rows_per_stage ? static_cast<int>(left) : rows_per_stage;
      };
      ring.produce(
          n_chunks, [&](int64_t c) { return static_cast<uint32_t>(rows_in(c)) * (per_row + cs_row_bytes); },
          [&](int64_t c, uint8_t* slot, uint64_t* bar) {
            const int64_t row0 = c * rows_per_stage;
            const int nr = rows_in(c);
            for (int r = 0; r < nr; ++r) ptx::bulk_load_1d(slot + r * per_row, x + (row0 + r) * ld, per_row, bar);
            if (cs_row_bytes) ptx::bulk_load_1d(slot + kRingRows * item_bytes, cos_sin + row0 * head_dim, nr * cs_row_bytes, bar);
          });
    }
    return;
  }

  const int groups = cols >> 3;
  const float inv_n = 1.0f / static_cast<float>(cols);
  const int grp = warp / kRingRows, wr = warp - grp * kRingRows;  // consumer group, item of the stage
  const int r_in_stage = wr / segs, seg = wr - r_in_stage * segs;
  const float* ws = w + static_cast<int64_t>(seg) * cols;
  ring.consume<NG>(n_chunks, grp, [&](int64_t c, const uint8_t* stage, auto release) {
    const int64_t row = c * rows_per_stage + r_in_stage;
    const uint8_t* rp = stage + wr * item_bytes;  // item wr of the stage = (row r_in_stage, block seg)
    uint4 raw[G];
    float cs[8] = {1.f, 0.f, 1.f, 0.f, 1.f, 0.f, 1.f, 0.f};
    if (row < rows) {
#pragma unroll
      for (int i = 0; i < G; ++i) {
        const int g = lane + i * 32;
        if (g < groups) raw[i] = *reinterpret_cast<const uint4*>(rp + g * 16);
      }
      if (cs_row_bytes) {
        // a lane's groups are 256 columns apart: with head_dim dividing 256 they all sit at the same position inside their head
        const float4* cp = reinterpret_cast<const float4*>(stage + kRingRows * item_bytes + r_in_stage * cs_row_bytes + ((lane * 8) % head_dim) * 4);
        const float4 a = cp[0], b = cp[1];
        cs[0] = a.x; cs[1] = a.y; cs[2] = a.z; cs[3] = a.w; cs[4] = b.x; cs[5] = b.y; cs[6] = b.z; cs[7] = b.w;
      }
    }
    release();
    if (row >= rows) return;
    __nv_bfloat16* px = x + row * ld + static_cast<int64_t>(seg) * cols;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < G; ++i)
      if (lane + i * 32 < groups) {
        float f[8];
        unpack_bf16x8(raw[i], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) q = fmaf(f[j], f[j], q);
      }
    const float r = rsqrtf(warp_sum(q) * inv_n + eps);
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int g = lane + i * 32;
      if (g < groups) {
        const int c0 = g * 8;
        float f[8], o[8];
        unpack_bf16x8(raw[i], f);
        rms_weight8(f, r, ws + c0, o);
        if (cs_row_bytes) rope_pairs4(o, cs);
        *reinterpret_cast<uint4*>(px + c0) = pack_bf16x8(o);
      }
    }
  });
}

// ---- per-HEAD RMSNorm (head_dim 128, bf16 weight semantics) + RoPE, in place on bf16: the q / k normalisation of the MMDiT
// attention (diffusers `RMSNorm(head_dim)` on [B, H, L, 128] followed by `apply_rotary_emb`, upstream of
// MagCache4FLUX/magcache_flux.py:361-366). 16 threads per (token, head), 8 elements each.
//   y = bf16( bf16(x * rsqrt(mean(x^2) + eps)) * w )      (variance in fp32; the product is cast to the bf16 weight dtype first)
//   RoPE in fp32 on consecutive (real, imag) pairs, result rounded to bf16
__global__ void __launch_bounds__(256) rmsnorm_head_rope_kernel(__nv_bfloat16* __restrict__ x, int64_t ld, int64_t rows, int heads,
                                                                const float* __restrict__ w, float eps,
                                                                const float* __restrict__ cos_sin) {
  const int sub = threadIdx.x & 15;
  const int64_t n_items = rows * heads;
  // a warp handles two items per trip; the trip count is the same for all 32 lanes (full-mask shuffles below)
  const int64_t warps_total = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  for (int64_t item0 = ((static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5) * 2; item0 < n_items; item0 += warps_total * 2) {
    const int64_t item = item0 + ((threadIdx.x >> 4) & 1);
    const bool live = item < n_items;  // all 16 lanes of a segment share `item`
    const int64_t row = live ? item / heads : 0;
    const int head = live ? static_cast<int>(item % heads) : 0;
    __nv_bfloat16* px = x + row * ld + head * 128 + sub * 8;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (live) unpack_bf16x8(*reinterpret_cast<const uint4*>(px), v);
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) q = fmaf(v[j], v[j], q);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);  // stays inside the 16-lane segment
    if (!live) continue;
    const float r = rsqrtf(q * (1.0f / 128.0f) + eps);
    float wv[8], o[8];
    load_param8(w + sub * 8, wv);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = round_bf16(round_bf16(v[j] * r) * wv[j]);
    if (cos_sin != nullptr) {
      float cs[8];
      ptx::ld_nc_v8_f32(cos_sin + row * 128 + sub * 8, cs);
      rope_pairs4(o, cs);
    }
    *reinterpret_cast<uint4*>(px) = pack_bf16x8(o);
  }
}

// ---- column mean of a bf16 matrix: the masked mean of the text states that conditions HunyuanVideo's token refiner
// (`(x * mask).sum(dim=1) / mask.sum(dim=1)` over the valid tokens [EXT hyvideo SingleTokenRefiner], called at
// MagCache4HunyuanVideo/magcache_sample_video.py:69). One thread per column (coalesced across a warp), fp32 accumulation.
__global__ void colmean_bf16_kernel(const __nv_bfloat16* __restrict__ x, int64_t ld, int rows, int cols, __nv_bfloat16* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float s = 0.f;
  for (int r = 0; r < rows; ++r) s += __bfloat162float(x[static_cast<int64_t>(r) * ld + c]);
  // torch: the bf16 sum is rounded to bf16, then divided by the (bf16) count and rounded again
  out[c] = __float2bfloat16_rn(round_bf16(s) / round_bf16(static_cast<float>(rows)));
}

// ---- y = silu(x) on a bf16 vector (the `self.silu(emb)` in front of every AdaLayerNorm linear) ------------------------------
__global__ void silu_bf16_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int64_t n) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float v = __bfloat162float(x[i]);
    y[i] = __float2bfloat16_rn(v / (1.0f + expf(-v)));
  }
}

// ---- patchify: latent fp32 [C,F,H,W] -> tokens bf16 [F*Hp*Wp, C*4] ----------------------------------------------
__global__ void patchify_kernel(const float* __restrict__ lat, int C, int F, int H, int W, __nv_bfloat16* __restrict__ tok) {
  const int Hp = H >> 1, Wp = W >> 1;
  const int64_t total = static_cast<int64_t>(F) * Hp * Wp * C;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    int64_t t = i / C;
    const int wp = static_cast<int>(t % Wp);
    t /= Wp;
    const int hp = static_cast<int>(t % Hp);
    const int f = static_cast<int>(t / Hp);
    const float* src = lat + ((static_cast<int64_t>(c) * F + f) * H + hp * 2) * W + wp * 2;
    const float2 r0 = *reinterpret_cast<const float2*>(src);
    const float2 r1 = *reinterpret_cast<const float2*>(src + W);
    uint2 o;
    o.x = pack_bf16x2(r0.x, r0.y);
    o.y = pack_bf16x2(r1.x, r1.y);
    *reinterpret_cast<uint2*>(tok + i * 4) = o;
  }
}

// ---- small fp32 linear (M <= 8): one warp per output feature -------------------------------------------------
template <int M>
__global__ void __launch_bounds__(256) linear_f32_small_kernel(const float* __restrict__ x, int K, const float* __restrict__ Wt,
                                                               const float* __restrict__ b, int N, int act, float* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  float acc[M];
#pragma unroll
  for (int m = 0; m < M; ++m) acc[m] = 0.f;
  const float4* wrow = reinterpret_cast<const float4*>(Wt + static_cast<int64_t>(n) * K);
  for (int k4 = lane; k4 < (K >> 2); k4 += 32) {
    const float4 wv = wrow[k4];
#pragma unroll
    for (int m = 0; m < M; ++m) {
      float4 xv = reinterpret_cast<const float4*>(x + static_cast<int64_t>(m) * K)[k4];
      if (act == 1) {
        xv.x = silu_f(xv.x); xv.y = silu_f(xv.y); xv.z = silu_f(xv.z); xv.w = silu_f(xv.w);
      }
      acc[m] = fmaf(xv.x, wv.x, acc[m]);
      acc[m] = fmaf(xv.y, wv.y, acc[m]);
      acc[m] = fmaf(xv.z, wv.z, acc[m]);
      acc[m] = fmaf(xv.w, wv.w, acc[m]);
    }
  }
#pragma unroll
  for (int m = 0; m < M; ++m) {
    float t = warp_sum(acc[m]);
    if (lane == 0) {
      t += (b != nullptr) ? b[n] : 0.f;
      if (act == 2) t = silu_f(t);
      y[static_cast<int64_t>(m) * N + n] = t;
    }
  }
}

// ---- elementwise --------------------------------------------------------------------------------------------
__global__ void cast_f32_to_bf16_kernel(const float* __restrict__ s, __nv_bfloat16* __restrict__ d, int64_t n) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    d[i] = __float2bfloat16_rn(s[i]);
}
__global__ void cast_bf16_to_f32_kernel(const __nv_bfloat16* __restrict__ s, float* __restrict__ d, int64_t n) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    d[i] = __bfloat162float(s[i]);
}
// sinusoidal_embedding_1d(dim, position) in float64, cos first (Appendix B.1); out fp32 [n_pos, dim]
__global__ void time_sinusoid_kernel(const double* __restrict__ pos, int n_pos, int dim, float* __restrict__ out) {
  const int half = dim / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pos * half) return;
  const int p = i / half, k = i % half;
  const double freq = pow(10000.0, -static_cast<double>(k) / static_cast<double>(half));
  const double s = pos[p] * freq;
  out[static_cast<int64_t>(p) * dim + k] = static_cast<float>(cos(s));
  out[static_cast<int64_t>(p) * dim + half + k] = static_cast<float>(sin(s));
}

// ---- bf16 transpose [rows, cols] -> [cols, rows] through a padded smem tile (token-sharded runs: gathered V -> V^T) ----
__global__ void __launch_bounds__(256) transpose_bf16_kernel(const __nv_bfloat16* __restrict__ src, int64_t lds, int rows, int cols,
                                                             __nv_bfloat16* __restrict__ dst, int64_t ldd) {
  __shared__ __nv_bfloat16 tile[64][66];
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int i = ty; i < 64; i += 8) {
    const int r = r0 + i;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = c0 + tx * 2 + h;  // two adjacent columns per lane
      tile[i][tx * 2 + h] = (r < rows && c < cols) ? src[static_cast<int64_t>(r) * lds + c] : __float2bfloat16(0.f);
    }
  }
  __syncthreads();
  for (int i = ty; i < 64; i += 8) {
    const int c = c0 + i;  // output row
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + tx * 2 + h;  // output column
      if (c < cols && r < rows) dst[static_cast<int64_t>(c) * ldd + r] = tile[tx * 2 + h][i];
    }
  }
}

// warp-per-row pipelined kernels: 2 blocks of 8 warps per SM, every warp walks rows with a stride of the total warp count
static int pipe_grid(int64_t rows, int blocks_per_sm = 2) {
  const int64_t want = (rows + 7) / 8, cap = static_cast<int64_t>(num_sms()) * blocks_per_sm;
  return static_cast<int>(want < 1 ? 1 : (want < cap ? want : cap));
}

static int grid_for(int64_t work_items, int per_block) {
  int64_t want = (work_items + per_block - 1) / per_block;
  const int64_t cap = static_cast<int64_t>(num_sms()) * 8;
  if (want < 1) want = 1;
  return static_cast<int>(want < cap ? want : cap);
}

// f(std::integral_constant<int, G>{}) for the smallest G in {2, 4, 6, 8} with 32 lanes x G groups >= `groups` (groups <= 32 * kMaxG):
// the per-lane register arrays the warp-per-row kernels are instantiated with
template <typename F>
static auto with_lane_groups(int groups, F f) {
  if (groups <= 32 * 2) return f(std::integral_constant<int, 2>{});
  if (groups <= 32 * 4) return f(std::integral_constant<int, 4>{});
  if (groups <= 32 * 6) return f(std::integral_constant<int, 6>{});
  return f(std::integral_constant<int, 8>{});
}

}  // namespace mc

extern "C" {

int32_t mc_patchify(const float* latent, int32_t C, int32_t F, int32_t H, int32_t W, void* tokens_bf16, void* stream) {
  MC_CHECK_ARG(latent && tokens_bf16, "mc_patchify: null pointer");
  MC_CHECK_ARG(C >= 1 && F >= 1 && H >= 2 && W >= 2 && H % 2 == 0 && W % 2 == 0, "mc_patchify: bad shape C=%d F=%d H=%d W=%d", C, F, H, W);
  MC_CHECK_ARG((reinterpret_cast<uintptr_t>(latent) & 7u) == 0 && (reinterpret_cast<uintptr_t>(tokens_bf16) & 7u) == 0,
               "mc_patchify: pointers must be 8-byte aligned");
  const int64_t total = static_cast<int64_t>(F) * (H / 2) * (W / 2) * C;
  mc::patchify_kernel<<<mc::grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      latent, C, F, H, W, static_cast<__nv_bfloat16*>(tokens_bf16));
  MC_CHECK_LAUNCH("patchify_kernel launch");
  return MC_OK;
}

int32_t mc_ln_modulate(const void* x, int32_t x_dtype, int64_t rows, int32_t cols, float eps, int32_t mode, const float* p0,
                       const float* p1, int32_t scale_idx, int32_t shift_idx, int32_t round_ln_to_bf16, void* out,
                       int32_t out_dtype, void* stream) {
  MC_CHECK_ARG(x && p0 && out && (mode != 1 || p1), "mc_ln_modulate: null pointer");
  MC_CHECK_ARG(mode == 0 || mode == 1 || mode == 2, "mc_ln_modulate: bad mode %d", mode);
  if (mode == 2) {
    MC_CHECK_ARG(x_dtype == MC_BF16 && out_dtype == MC_BF16 && cols >= 8 && cols % 8 == 0 && cols <= 32 * 8 * mc::kMaxG && rows >= 1,
                 "mc_ln_modulate: mode 2 needs bf16 x / out and cols %% 8 == 0, cols <= 2048 (cols=%d)", cols);
    MC_CHECK_ARG(mc::aligned16(x) && mc::aligned16(out) && mc::aligned16(p0) && cols % 4 == 0, "mc_ln_modulate: mode 2 pointers must be 16-byte aligned");
    const int64_t want = (rows + 7) / 8, cap = static_cast<int64_t>(mc::num_sms()) * 16;
    mc::ln_t2i_modulate_kernel<mc::kMaxG, false><<<static_cast<int>(want < cap ? want : cap), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(x), rows, cols, eps, p0 + static_cast<int64_t>(scale_idx) * cols,
        p0 + static_cast<int64_t>(shift_idx) * cols, static_cast<__nv_bfloat16*>(out), nullptr, nullptr);
    MC_CHECK_LAUNCH("ln_t2i_modulate_kernel launch");
    return MC_OK;
  }
  MC_CHECK_ARG(rows >= 1 && cols >= 8 && cols % 8 == 0 && cols <= 32 * mc::kWideWarps * 8 * mc::kMaxG, "mc_ln_modulate: cols=%d unsupported", cols);
  MC_CHECK_ARG(mc::aligned16(p0) && (p1 == nullptr || mc::aligned16(p1)), "mc_ln_modulate: parameters must be 16-byte aligned");
  MC_CHECK_ARG((x_dtype == MC_F32 || x_dtype == MC_BF16) && (out_dtype == MC_F32 || out_dtype == MC_BF16), "mc_ln_modulate: bad dtype");
  MC_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 31u) == 0 && (reinterpret_cast<uintptr_t>(out) & 31u) == 0,
               "mc_ln_modulate: x/out must be 32-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int groups = cols / 8;
  const int x_bf16 = x_dtype == MC_BF16, o_bf16 = out_dtype == MC_BF16;
  // long inputs: the TMA-staged form (needs >= 2 stages of 8 rows in shared memory and 16-byte aligned rows)
  const int stage_bytes = mc::kRingRows * cols * (x_bf16 ? 2 : 4);
  const int ring = rows >= 1024 && groups <= 32 * mc::kMaxG ? mc::ring_stages(stage_bytes, mc::kRowRingMaxStages) : 0;
  if (ring > 0)
    return mc::with_lane_groups(groups, [&](auto G) {
      return mc::launch_ring<mc::ln_modulate_tma_kernel<decltype(G)::value, mc::kLnRingGroups>>(
          ring, stage_bytes, 0, (rows + mc::kRingRows - 1) / mc::kRingRows, mc::ring_threads(mc::kLnRingGroups), s, "ln_modulate_tma_kernel",
          x, x_bf16, rows, cols, eps, mode, p0, p1, scale_idx, shift_idx, round_ln_to_bf16, out, o_bf16, ring);
    });
  if (groups <= 32 * mc::kMaxG) {
    mc::with_lane_groups(groups, [&](auto G) {
      constexpr int g = decltype(G)::value;
      mc::ln_modulate_pipe_kernel<g><<<mc::pipe_grid(rows, g >= 6 ? 1 : 2), 256, 0, s>>>(x, x_bf16, rows, cols, eps, mode, p0, p1, scale_idx,
                                                                                       shift_idx, round_ln_to_bf16, out, o_bf16);
    });
  } else {
    mc::ln_modulate_kernel<<<mc::grid_for(rows, 256 / (32 * mc::kWideWarps)), 256, 0, s>>>(x, x_bf16, rows, cols, eps, mode, p0, p1, scale_idx,
                                                                                          shift_idx, round_ln_to_bf16, out, o_bf16);
  }
  MC_CHECK_LAUNCH("ln_modulate_kernel launch");
  return MC_OK;
}

int32_t mc_ln_t2i_modulate_rel_l1(const void* x, int64_t rows, int32_t cols, float eps, const float* p0, int32_t scale_idx, int32_t shift_idx,
                                  const void* prev, void* out, double* partials_dev, double* sums_dev, void* stream) {
  MC_CHECK_ARG(x && p0 && prev && out && partials_dev && sums_dev, "mc_ln_t2i_modulate_rel_l1: null pointer");
  MC_CHECK_ARG(rows >= 1 && cols >= 8 && cols % 8 == 0 && cols <= 32 * 8 * mc::kMaxG, "mc_ln_t2i_modulate_rel_l1: cols %% 8 == 0, cols <= 2048 (cols=%d)",
               cols);
  MC_CHECK_ARG(mc::aligned16(x) && mc::aligned16(out) && mc::aligned16(prev) && mc::aligned16(p0) && mc::aligned16(partials_dev),
               "mc_ln_t2i_modulate_rel_l1: pointers must be 16-byte aligned");
  MC_CHECK_ARG(prev != out && x != out, "mc_ln_t2i_modulate_rel_l1: out may not alias x or prev");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int64_t grid = (rows + 7) / 8;
  const int64_t cap = static_cast<int64_t>(mc::num_sms()) * 16;
  if (grid > cap) grid = cap;
  if (grid > MC_LN_REL_L1_MAX_CTAS) grid = MC_LN_REL_L1_MAX_CTAS;
  double2* parts = reinterpret_cast<double2*>(partials_dev);
  mc::with_lane_groups(cols / 8, [&](auto G) {
    mc::ln_t2i_modulate_kernel<decltype(G)::value, true><<<static_cast<int>(grid), 256, 0, s>>>(
        static_cast<const __nv_bfloat16*>(x), rows, cols, eps, p0 + static_cast<int64_t>(scale_idx) * cols,
        p0 + static_cast<int64_t>(shift_idx) * cols, static_cast<__nv_bfloat16*>(out), static_cast<const __nv_bfloat16*>(prev), parts);
  });
  MC_CHECK_LAUNCH("ln_t2i_modulate_kernel<rel_l1> launch");
  mc::rel_l1_finish_kernel<<<1, 256, 0, s>>>(parts, static_cast<int>(grid), sums_dev);
  MC_CHECK_LAUNCH("rel_l1_finish_kernel launch");
  return MC_OK;
}

int32_t mc_rmsnorm_rope_segs(void* x_bf16, int64_t ld, int64_t rows, int32_t segs, int32_t cols, const float* w, float eps, const float* cos_sin,
                             int32_t head_dim, void* stream);

int32_t mc_rmsnorm_rope(void* x_bf16, int64_t ld, int64_t rows, int32_t cols, const float* w, float eps, const float* cos_sin,
                        int32_t head_dim, void* stream) {
  return mc_rmsnorm_rope_segs(x_bf16, ld, rows, 1, cols, w, eps, cos_sin, head_dim, stream);
}

int32_t mc_rmsnorm_rope_segs(void* x_bf16, int64_t ld, int64_t rows, int32_t segs, int32_t cols, const float* w, float eps, const float* cos_sin,
                             int32_t head_dim, void* stream) {
  MC_CHECK_ARG(x_bf16 && w, "mc_rmsnorm_rope: null pointer");
  MC_CHECK_ARG(segs >= 1 && segs <= 4, "mc_rmsnorm_rope: segs=%d outside [1, 4]", segs);
  MC_CHECK_ARG(rows >= 1 && cols >= 8 && cols % 8 == 0 && cols <= 32 * mc::kWideWarps * 8 * mc::kMaxG && ld >= static_cast<int64_t>(segs) * cols && ld % 8 == 0,
               "mc_rmsnorm_rope: cols=%d ld=%lld unsupported", cols, static_cast<long long>(ld));
  MC_CHECK_ARG(mc::aligned16(x_bf16), "mc_rmsnorm_rope: x must be 16-byte aligned");
  MC_CHECK_ARG(mc::aligned16(w), "mc_rmsnorm_rope: weight must be 16-byte aligned");
  MC_CHECK_ARG(cos_sin == nullptr || (head_dim >= 8 && head_dim % 8 == 0 && cols % head_dim == 0 && (reinterpret_cast<uintptr_t>(cos_sin) & 31u) == 0),
               "mc_rmsnorm_rope: bad head_dim %d", head_dim);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int groups = cols / 8;
  __nv_bfloat16* xp = static_cast<__nv_bfloat16*>(x_bf16);
  const bool ring_ok = rows * segs >= 1024 && groups <= 32 * mc::kMaxG && (segs == 1 || segs == 2 || segs == 4) &&
                       (cos_sin == nullptr || 256 % head_dim == 0);
  const int rows_per_stage = mc::kRingRows / (segs == 3 ? 1 : segs);
  const int ring_stage_bytes = mc::kRingRows * cols * 2 + (cos_sin != nullptr ? rows_per_stage * head_dim * 4 : 0);
  const int ring = ring_ok ? mc::ring_stages(ring_stage_bytes, mc::kRowRingMaxStages) : 0;
  if (ring > 0)
    return mc::with_lane_groups(groups, [&](auto G) {
      return mc::launch_ring<mc::rmsnorm_rope_tma_kernel<decltype(G)::value, mc::kRmsRingGroups>>(
          ring, ring_stage_bytes, 0, (rows + rows_per_stage - 1) / rows_per_stage, mc::ring_threads(mc::kRmsRingGroups), s,
          "rmsnorm_rope_tma_kernel", xp, ld, rows, segs, cols, w, eps, cos_sin, head_dim, ring);
    });
  if (groups <= 32 * mc::kMaxG) {
    mc::with_lane_groups(groups, [&](auto G) {
      mc::rmsnorm_rope_pipe_kernel<decltype(G)::value><<<mc::pipe_grid(rows * segs), 256, 0, s>>>(xp, ld, rows, segs, cols, w, eps, cos_sin, head_dim);
    });
  } else {
    // wide rows (Wan-14B: 5120): four warps per row, one column block per launch
    for (int sg = 0; sg < segs; ++sg)
      mc::rmsnorm_rope_kernel<<<mc::grid_for(rows, 256 / (32 * mc::kWideWarps)), 256, 0, s>>>(
          xp + static_cast<int64_t>(sg) * cols, ld, rows, cols, w + static_cast<int64_t>(sg) * cols, eps, cos_sin, head_dim);
  }
  MC_CHECK_LAUNCH("rmsnorm_rope_kernel launch");
  return MC_OK;
}

int32_t mc_rmsnorm_head_rope(void* x_bf16, int64_t ld, int64_t rows, int32_t heads, const float* w, float eps, const float* cos_sin,
                             void* stream) {
  MC_CHECK_ARG(x_bf16 && w, "mc_rmsnorm_head_rope: null pointer");
  MC_CHECK_ARG(rows >= 1 && heads >= 1 && ld >= static_cast<int64_t>(heads) * 128 && ld % 8 == 0, "mc_rmsnorm_head_rope: rows=%lld heads=%d ld=%lld",
               static_cast<long long>(rows), heads, static_cast<long long>(ld));
  MC_CHECK_ARG(mc::aligned16(x_bf16) && (cos_sin == nullptr || (reinterpret_cast<uintptr_t>(cos_sin) & 31u) == 0),
               "mc_rmsnorm_head_rope: x must be 16-byte and cos_sin 32-byte aligned");
  const int64_t items = rows * heads;
  const int64_t want = (items + 15) / 16, cap = static_cast<int64_t>(mc::num_sms()) * 8;
  mc::rmsnorm_head_rope_kernel<<<static_cast<int>(want < cap ? want : cap), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<__nv_bfloat16*>(x_bf16), ld, rows, heads, w, eps, cos_sin);
  MC_CHECK_LAUNCH("rmsnorm_head_rope_kernel launch");
  return MC_OK;
}

int32_t mc_colmean_bf16(const void* x, int64_t ld, int32_t rows, int32_t cols, void* out, void* stream) {
  MC_CHECK_ARG(x && out && rows >= 1 && cols >= 1 && ld >= cols, "mc_colmean_bf16: bad arguments");
  mc::colmean_bf16_kernel<<<(cols + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const __nv_bfloat16*>(x), ld, rows, cols,
                                                                                             static_cast<__nv_bfloat16*>(out));
  MC_CHECK_LAUNCH("colmean_bf16_kernel launch");
  return MC_OK;
}

int32_t mc_silu_bf16(const void* x, void* y, int64_t n, void* stream) {
  MC_CHECK_ARG(x && y && n >= 1, "mc_silu_bf16: bad arguments");
  const int64_t want = (n + 255) / 256, cap = static_cast<int64_t>(mc::num_sms()) * 8;
  mc::silu_bf16_kernel<<<static_cast<int>(want < cap ? want : cap), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), n);
  MC_CHECK_LAUNCH("silu_bf16_kernel launch");
  return MC_OK;
}

int32_t mc_linear_f32_small(const float* x, int32_t M, int32_t K, const float* W, const float* b, int32_t N, int32_t act, float* y,
                            void* stream) {
  MC_CHECK_ARG(x && W && y, "mc_linear_f32_small: null pointer");
  MC_CHECK_ARG(M >= 1 && M <= 8 && K >= 4 && K % 4 == 0 && N >= 1, "mc_linear_f32_small: M=%d K=%d N=%d unsupported", M, K, N);
  MC_CHECK_ARG(mc::aligned16(x) && mc::aligned16(W), "mc_linear_f32_small: x/W must be 16-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int grid = (N + 7) / 8;
  switch (M) {
#define MC_LS(MM) case MM: mc::linear_f32_small_kernel<MM><<<grid, 256, 0, s>>>(x, K, W, b, N, act, y); break;
    MC_LS(1) MC_LS(2) MC_LS(3) MC_LS(4) MC_LS(5) MC_LS(6) MC_LS(7) MC_LS(8)
#undef MC_LS
  }
  MC_CHECK_LAUNCH("linear_f32_small_kernel launch");
  return MC_OK;
}

int32_t mc_transpose_bf16(const void* src, int64_t lds, int32_t rows, int32_t cols, void* dst, int64_t ldd, void* stream) {
  MC_CHECK_ARG(src && dst && rows >= 1 && cols >= 1 && lds >= cols && ldd >= rows, "mc_transpose_bf16: bad arguments");
  dim3 grid((cols + 63) / 64, (rows + 63) / 64);
  mc::transpose_bf16_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const __nv_bfloat16*>(src), lds, rows, cols,
                                                                                static_cast<__nv_bfloat16*>(dst), ldd);
  MC_CHECK_LAUNCH("transpose_bf16_kernel launch");
  return MC_OK;
}

int32_t mc_cast(const void* src, int32_t src_dtype, void* dst, int32_t dst_dtype, int64_t n, void* stream) {
  MC_CHECK_ARG(src && dst && n >= 0, "mc_cast: bad arguments");
  if (n == 0) return MC_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (src_dtype == MC_F32 && dst_dtype == MC_BF16)
    mc::cast_f32_to_bf16_kernel<<<mc::grid_for(n, 256), 256, 0, s>>>(static_cast<const float*>(src), static_cast<__nv_bfloat16*>(dst), n);
  else if (src_dtype == MC_BF16 && dst_dtype == MC_F32)
    mc::cast_bf16_to_f32_kernel<<<mc::grid_for(n, 256), 256, 0, s>>>(static_cast<const __nv_bfloat16*>(src), static_cast<float*>(dst), n);
  else {
    mc::set_error("mc_cast: unsupported %d -> %d", src_dtype, dst_dtype);
    return MC_ERR_INVALID;
  }
  MC_CHECK_LAUNCH("cast kernel launch");
  return MC_OK;
}

int32_t mc_time_sinusoid(const double* pos_dev, int32_t n_pos, int32_t dim, float* out, void* stream) {
  MC_CHECK_ARG(pos_dev && out && n_pos >= 1 && dim >= 2 && dim % 2 == 0, "mc_time_sinusoid: bad arguments");
  const int total = n_pos * (dim / 2);
  mc::time_sinusoid_kernel<<<(total + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(pos_dev, n_pos, dim, out);
  MC_CHECK_LAUNCH("time_sinusoid_kernel launch");
  return MC_OK;
}

}  // extern "C"
