// Row-wise (token-local) kernels of the cache-miss branch — all HBM-bound, fp32 statistics, 128-bit accesses.
// Arithmetic follows upstream Wan2.1 wan/modules/model.py as restated in SURVEY.md Appendix B.1; call sites in the
// reference: MagCache4Wan2.1/magcache_generate.py:237 (patch_embedding), :249-254 (time embedding),
// :297-298 (block stack), :304-305 (head, unpatchify).
#include "common.cuh"
#include "ptx.cuh"

namespace mc {

// A "team" of TPR threads owns one row; each thread keeps up to kMaxG groups of 8 elements in registers.
// TPR = 32 (one warp per row, shuffle-only reductions) covers cols <= 2048; TPR = 128 covers cols <= 8192.
constexpr int kMaxG = 8;

template <int TPR>
__device__ __forceinline__ float team_sum(float v, float* scratch /* [rows_per_block][TPR/32] */, int team, int lane_in_team) {
  v = warp_sum(v);
  if (TPR == 32) return v;
  constexpr int W = TPR / 32;
  const int w = lane_in_team >> 5;
  __syncthreads();  // protect scratch reuse between consecutive reductions
  if ((lane_in_team & 31) == 0) scratch[team * W + w] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < W; ++i) t += scratch[team * W + i];
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
__device__ __forceinline__ void load_param8(const float* p, float (&f)[8]) {  // per-column parameters: L1-resident, reused by every row
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

// ---- K7: LayerNorm (no affine) + modulation / affine, optional bf16 rounding of the LN output -----------------
//   mode 0: y = LN(x) * (1 + p0[scale_idx]) + p0[shift_idx]   with p0 = e = modulation + e0, fp32 [k, cols]
//   mode 1: y = LN(x) * p0 + p1                               (elementwise affine)
template <int TPR>
__global__ void __launch_bounds__(256) ln_modulate_kernel(const void* __restrict__ x, int x_bf16, int64_t rows, int cols, float eps,
                                                          int mode, const float* __restrict__ p0, const float* __restrict__ p1,
                                                          int scale_idx, int shift_idx, int round_ln, void* __restrict__ out,
                                                          int out_bf16) {
  constexpr int RPB = 256 / TPR;  // rows per block
  __shared__ float scratch[RPB * (TPR / 32 > 0 ? TPR / 32 : 1)];
  const int team = threadIdx.x / TPR, lt = threadIdx.x % TPR;
  const int groups = cols >> 3;
  const float inv_n = 1.0f / static_cast<float>(cols);
  const float* pa = (mode == 0) ? p0 + static_cast<int64_t>(scale_idx) * cols : p0;
  const float* pb = (mode == 0) ? p0 + static_cast<int64_t>(shift_idx) * cols : p1;
  for (int64_t row0 = static_cast<int64_t>(blockIdx.x) * RPB; row0 < rows; row0 += static_cast<int64_t>(gridDim.x) * RPB) {
    const int64_t row = row0 + team;
    const bool live = row < rows;
    float v[kMaxG][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxG; ++i) {
      const int g = lt + i * TPR;
      if (live && g < groups) {
        load_row_group(x, x_bf16, row * cols + g * 8, v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[i][j];
      }
    }
    const float mean = team_sum<TPR>(s, scratch, team, lt) * inv_n;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxG; ++i) {
      const int g = lt + i * TPR;
      if (live && g < groups) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[i][j] - mean;
          q = fmaf(d, d, q);
        }
      }
    }
    const float var = team_sum<TPR>(q, scratch, team, lt) * inv_n;
    const float rstd = rsqrtf(var + eps);
#pragma unroll
    for (int i = 0; i < kMaxG; ++i) {
      const int g = lt + i * TPR;
      if (live && g < groups) {
        const int c0 = g * 8;
        float a[8], b[8], o[8];
        load_param8(pa + c0, a);
        load_param8(pb + c0, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float y = (v[i][j] - mean) * rstd;
          if (round_ln) y = round_bf16(y);
          const float aa = (mode == 0) ? 1.0f + a[j] : a[j];
          o[j] = __fadd_rn(__fmul_rn(y, aa), b[j]);  // torch eager: separate mul and add, no FMA contraction
        }
        if (out_bf16) {
          ptx::st_na_v4(static_cast<__nv_bfloat16*>(out) + row * cols + c0, pack_bf16x8(o));
        } else {
          ptx::st_na_v8_f32(static_cast<float*>(out) + row * cols + c0, o);
        }
      }
    }
  }
}

// ---- mode 2: LayerNorm + t2i_modulate with every step a bf16 tensor op (STDiT3Block.forward, open_sora_transformer_3d.py:187, :248;
// T2IFinalLayer, :80): y = bf16(bf16(bf16(LN(x)) * bf16(1 + p0[scale_idx])) + p0[shift_idx]), p0 holding bf16 values.
// One warp per row, x and out bf16, cols <= 2048.
__global__ void __launch_bounds__(256) ln_t2i_modulate_kernel(const __nv_bfloat16* __restrict__ x, int64_t rows, int cols, float eps,
                                                              const float* __restrict__ sc, const float* __restrict__ sh,
                                                              __nv_bfloat16* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int groups = cols >> 3;
  const float inv_n = 1.0f / static_cast<float>(cols);
  for (int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; row < rows;
       row += (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5) {
    float v[kMaxG][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxG; ++i) {
      const int g = lane + i * 32;
      if (g < groups) {
        unpack_bf16x8(ptx::ld_nc_v4(x + row * cols + g * 8), v[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[i][j];
      }
    }
    const float mean = warp_sum(s) * inv_n;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxG; ++i) {
      if (lane + i * 32 < groups) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[i][j] - mean;
          q = fmaf(d, d, q);
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(q) * inv_n + eps);
#pragma unroll
    for (int i = 0; i < kMaxG; ++i) {
      const int g = lane + i * 32;
      if (g < groups) {
        float a[8], b[8], o[8];
        load_param8(sc + g * 8, a);
        load_param8(sh + g * 8, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float y = round_bf16((v[i][j] - mean) * rstd);
          o[j] = round_bf16(__fadd_rn(round_bf16(__fmul_rn(y, round_bf16(__fadd_rn(1.0f, a[j])))), b[j]));
        }
        ptx::st_na_v4(out + row * cols + g * 8, pack_bf16x8(o));
      }
    }
  }
}

// ---- WanRMSNorm over the model dim (+ optional 3-axis RoPE), in place on bf16 ---------------------------------
template <int TPR>
__global__ void __launch_bounds__(256) rmsnorm_rope_kernel(__nv_bfloat16* __restrict__ x, int64_t ld, int64_t rows, int cols,
                                                           const float* __restrict__ w, float eps,
                                                           const float* __restrict__ cos_sin, int head_dim) {
  constexpr int RPB = 256 / TPR;
  __shared__ float scratch[RPB * (TPR / 32 > 0 ? TPR / 32 : 1)];
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
    const float ms = team_sum<TPR>(q, scratch, team, lt) * inv_n;
    const float r = rsqrtf(ms + eps);
#pragma unroll
    for (int i = 0; i < kMaxG; ++i) {
      const int g = lt + i * TPR;
      if (live && g < groups) {
        const int c0 = g * 8;
        float wv[8], o[8];
        load_param8(w + c0, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = round_bf16(v[i][j] * r) * wv[j];  // _norm(x.float()).type_as(x) * weight
        if (cos_sin != nullptr) {
          const int d0 = c0 % head_dim;  // position inside the head; 8 elements = 4 complex pairs
          float cs[8];
          ptx::ld_nc_v8_f32(cos_sin + row * head_dim + d0, cs);
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            const float re = o[2 * p], im = o[2 * p + 1], c = cs[2 * p], sn = cs[2 * p + 1];
            o[2 * p] = __fsub_rn(__fmul_rn(re, c), __fmul_rn(im, sn));
            o[2 * p + 1] = __fadd_rn(__fmul_rn(re, sn), __fmul_rn(im, c));
          }
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
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < G; ++i)
      if (lane + i * 32 < groups) {
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[i][j];
      }
    const float mean = warp_sum(s) * inv_n;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < G; ++i)
      if (lane + i * 32 < groups) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[i][j] - mean;
          q = fmaf(d, d, q);
        }
      }
    const float rstd = rsqrtf(warp_sum(q) * inv_n + eps);
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int g = lane + i * 32;
      if (g < groups) {
        const int c0 = g * 8;
        float a[8], b[8], o[8];
        load_param8(pa + c0, a);
        load_param8(pb + c0, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float y = (v[i][j] - mean) * rstd;
          if (round_ln) y = round_bf16(y);
          const float aa = (mode == 0) ? 1.0f + a[j] : a[j];
          o[j] = __fadd_rn(__fmul_rn(y, aa), b[j]);  // torch eager: separate mul and add, no FMA contraction
        }
        if (out_bf16) {
          ptx::st_na_v4(static_cast<__nv_bfloat16*>(out) + row * cols + c0, pack_bf16x8(o));
        } else {
          ptx::st_na_v8_f32(static_cast<float*>(out) + row * cols + c0, o);
        }
      }
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
        float f[8], wv[8], o[8];
        unpack_bf16x8(raw[i], f);
        load_param8(ws + c0, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = round_bf16(f[j] * r) * wv[j];  // _norm(x.float()).type_as(x) * weight
        if (cos_sin != nullptr) {
          const int d0 = c0 % head_dim;  // position inside the head; 8 elements = 4 complex pairs
          float cs[8];
          ptx::ld_nc_v8_f32(cos_sin + row * head_dim + d0, cs);
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            const float re = o[2 * pp], im = o[2 * pp + 1], c = cs[2 * pp], sn = cs[2 * pp + 1];
            o[2 * pp] = __fsub_rn(__fmul_rn(re, c), __fmul_rn(im, sn));
            o[2 * pp + 1] = __fadd_rn(__fmul_rn(re, sn), __fmul_rn(im, c));
          }
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
// (3.2-3.9 TB/s measured on 32760 x 1536). Here one producer thread keeps `stages` x 8 rows in flight with cp.async.bulk into a
// shared-memory ring (144-192 KB per SM, independent of what the consumer warps are doing); NG groups of eight consumer warps
// take the stages in turn (stage `it` belongs to group it % NG), one row of the stage per warp: copy it to registers, hand the
// slot back at once, then run the same arithmetic as the forms above (bit-identical results). One CTA per SM, chunks of 8 rows
// strided over the grid. The consumers, not the loads, bound these kernels: 8 warps 4.2 TB/s, 16 warps 4.7 TB/s on fp32 rows
// (24 warps spill at 80 registers); the bf16 RMSNorm rows take 24 warps: 3.2 -> 5.1 TB/s.
constexpr int kRingRows = 8;                                                   // rows (or (token, block) items) per stage
constexpr int ring_threads(int groups) { return (groups * kRingRows + 1) * 32; }  // + the producer warp
constexpr int kLnRingGroups = 2, kRmsRingGroups = 3;

template <int G, int NG>
__global__ void __launch_bounds__(ring_threads(NG), 1) ln_modulate_tma_kernel(const void* __restrict__ x, int x_bf16, int64_t rows, int cols, float eps,
                                                                         int mode, const float* __restrict__ p0, const float* __restrict__ p1,
                                                                         int scale_idx, int shift_idx, int round_ln, void* __restrict__ out,
                                                                         int out_bf16, int stages) {
  extern __shared__ __align__(128) uint8_t smem_dyn[];
  const int row_bytes = cols * (x_bf16 ? 2 : 4);
  const int stage_bytes = kRingRows * row_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_dyn + static_cast<size_t>(stages) * stage_bytes);
  uint64_t* empty = full + stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n_chunks = (rows + kRingRows - 1) / kRingRows;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], kRingRows);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp == NG * kRingRows) {
    if (lane == 0) {
      uint32_t it = 0;
      for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x, ++it) {
        const int s = it % stages;
        ptx::mbar_wait(&empty[s], ((it / stages) & 1) ^ 1);
        const int64_t row0 = c * kRingRows;
        const int64_t left = rows - row0;
        const uint32_t bytes = static_cast<uint32_t>(left < kRingRows ? left : kRingRows) * row_bytes;  // rows are contiguous
        ptx::mbar_expect_tx(&full[s], bytes);
        ptx::bulk_load_1d(smem_dyn + static_cast<size_t>(s) * stage_bytes, static_cast<const uint8_t*>(x) + row0 * row_bytes, bytes, &full[s]);
      }
    }
    return;
  }

  const int groups = cols >> 3;
  const float inv_n = 1.0f / static_cast<float>(cols);
  const float* pa = (mode == 0) ? p0 + static_cast<int64_t>(scale_idx) * cols : p0;
  const float* pb = (mode == 0) ? p0 + static_cast<int64_t>(shift_idx) * cols : p1;
  const int grp = warp / kRingRows, wr = warp - grp * kRingRows;  // consumer group, row of the stage
  uint32_t it = grp;
  for (int64_t c = blockIdx.x + static_cast<int64_t>(grp) * gridDim.x; c < n_chunks; c += static_cast<int64_t>(NG) * gridDim.x, it += NG) {
    const int s = it % stages;
    ptx::mbar_wait(&full[s], (it / stages) & 1);
    const int64_t row = c * kRingRows + wr;
    const uint8_t* rp = smem_dyn + static_cast<size_t>(s) * stage_bytes + wr * row_bytes;
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
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty[s]);  // the row is in registers: the slot can be refilled while it is processed
    if (row >= rows) continue;
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < G; ++i)
      if (lane + i * 32 < groups) {
#pragma unroll
        for (int j = 0; j < 8; ++j) sum += v[i][j];
      }
    const float mean = warp_sum(sum) * inv_n;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < G; ++i)
      if (lane + i * 32 < groups) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[i][j] - mean;
          q = fmaf(d, d, q);
        }
      }
    const float rstd = rsqrtf(warp_sum(q) * inv_n + eps);
#pragma unroll
    for (int i = 0; i < G; ++i) {
      const int g = lane + i * 32;
      if (g < groups) {
        const int c0 = g * 8;
        float a[8], b[8], o[8];
        load_param8(pa + c0, a);
        load_param8(pb + c0, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float y = (v[i][j] - mean) * rstd;
          if (round_ln) y = round_bf16(y);
          const float aa = (mode == 0) ? 1.0f + a[j] : a[j];
          o[j] = __fadd_rn(__fmul_rn(y, aa), b[j]);  // torch eager: separate mul and add, no FMA contraction
        }
        if (out_bf16) {
          ptx::st_na_v4(static_cast<__nv_bfloat16*>(out) + row * cols + c0, pack_bf16x8(o));
        } else {
          ptx::st_na_v8_f32(static_cast<float*>(out) + row * cols + c0, o);
        }
      }
    }
  }
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
  const int stage_bytes = kRingRows * item_bytes + rows_per_stage * cs_row_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_dyn + static_cast<size_t>(stages) * stage_bytes);
  uint64_t* empty = full + stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n_chunks = (rows + rows_per_stage - 1) / rows_per_stage;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], kRingRows);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp == NG * kRingRows) {
    if (lane == 0) {
      uint32_t it = 0;
      for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x, ++it) {
        const int s = it % stages;
        ptx::mbar_wait(&empty[s], ((it / stages) & 1) ^ 1);
        const int64_t row0 = c * rows_per_stage;
        const int64_t left = rows - row0;
        const int nr = left < rows_per_stage ? static_cast<int>(left) : rows_per_stage;
        uint8_t* base = smem_dyn + static_cast<size_t>(s) * stage_bytes;
        const uint32_t per_row = static_cast<uint32_t>(segs) * item_bytes;
        ptx::mbar_expect_tx(&full[s], static_cast<uint32_t>(nr) * (per_row + cs_row_bytes));
        for (int r = 0; r < nr; ++r) ptx::bulk_load_1d(base + r * per_row, x + (row0 + r) * ld, per_row, &full[s]);
        if (cs_row_bytes) ptx::bulk_load_1d(base + kRingRows * item_bytes, cos_sin + row0 * head_dim, nr * cs_row_bytes, &full[s]);
      }
    }
    return;
  }

  const int groups = cols >> 3;
  const float inv_n = 1.0f / static_cast<float>(cols);
  const int grp = warp / kRingRows, wr = warp - grp * kRingRows;  // consumer group, item of the stage
  const int r_in_stage = wr / segs, seg = wr - r_in_stage * segs;
  const float* ws = w + static_cast<int64_t>(seg) * cols;
  uint32_t it = grp;
  for (int64_t c = blockIdx.x + static_cast<int64_t>(grp) * gridDim.x; c < n_chunks; c += static_cast<int64_t>(NG) * gridDim.x, it += NG) {
    const int s = it % stages;
    ptx::mbar_wait(&full[s], (it / stages) & 1);
    const int64_t row = c * rows_per_stage + r_in_stage;
    const uint8_t* base = smem_dyn + static_cast<size_t>(s) * stage_bytes;
    const uint8_t* rp = base + wr * item_bytes;  // item wr of the stage = (row r_in_stage, block seg)
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
        const float4* cp = reinterpret_cast<const float4*>(base + kRingRows * item_bytes + r_in_stage * cs_row_bytes + ((lane * 8) % head_dim) * 4);
        const float4 a = cp[0], b = cp[1];
        cs[0] = a.x; cs[1] = a.y; cs[2] = a.z; cs[3] = a.w; cs[4] = b.x; cs[5] = b.y; cs[6] = b.z; cs[7] = b.w;
      }
    }
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty[s]);
    if (row >= rows) continue;
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
        float f[8], wv[8], o[8];
        unpack_bf16x8(raw[i], f);
        load_param8(ws + c0, wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = round_bf16(f[j] * r) * wv[j];  // _norm(x.float()).type_as(x) * weight
        if (cs_row_bytes) {
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            const float re = o[2 * pp], im = o[2 * pp + 1], cc = cs[2 * pp], sn = cs[2 * pp + 1];
            o[2 * pp] = __fsub_rn(__fmul_rn(re, cc), __fmul_rn(im, sn));
            o[2 * pp + 1] = __fadd_rn(__fmul_rn(re, sn), __fmul_rn(im, cc));
          }
        }
        *reinterpret_cast<uint4*>(px + c0) = pack_bf16x8(o);
      }
    }
  }
}

// number of ring stages that fit (0: the staged form does not apply)
static int ring_stages(int stage_bytes) {
  int stages = (200 * 1024) / stage_bytes;
  if (stages > 8) stages = 8;
  return stages >= 2 ? stages : 0;
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
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const float re = o[2 * p], im = o[2 * p + 1], c = cs[2 * p], sn = cs[2 * p + 1];
        o[2 * p] = __fsub_rn(__fmul_rn(re, c), __fmul_rn(im, sn));
        o[2 * p + 1] = __fadd_rn(__fmul_rn(im, c), __fmul_rn(re, sn));
      }
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
__device__ __forceinline__ float silu(float x) { return x / (1.0f + expf(-x)); }

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
        xv.x = silu(xv.x); xv.y = silu(xv.y); xv.z = silu(xv.z); xv.w = silu(xv.w);
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
      if (act == 2) t = silu(t);
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
    mc::ln_t2i_modulate_kernel<<<static_cast<int>(want < cap ? want : cap), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(x), rows, cols, eps, p0 + static_cast<int64_t>(scale_idx) * cols,
        p0 + static_cast<int64_t>(shift_idx) * cols, static_cast<__nv_bfloat16*>(out));
    MC_CHECK_LAUNCH("ln_t2i_modulate_kernel launch");
    return MC_OK;
  }
  MC_CHECK_ARG(rows >= 1 && cols >= 8 && cols % 8 == 0 && cols <= 128 * 8 * mc::kMaxG, "mc_ln_modulate: cols=%d unsupported", cols);
  MC_CHECK_ARG(mc::aligned16(p0) && (p1 == nullptr || mc::aligned16(p1)), "mc_ln_modulate: parameters must be 16-byte aligned");
  MC_CHECK_ARG((x_dtype == MC_F32 || x_dtype == MC_BF16) && (out_dtype == MC_F32 || out_dtype == MC_BF16), "mc_ln_modulate: bad dtype");
  MC_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 31u) == 0 && (reinterpret_cast<uintptr_t>(out) & 31u) == 0,
               "mc_ln_modulate: x/out must be 32-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int groups = cols / 8;
#define MC_LN(TPR)                                                                                                             \
  mc::ln_modulate_kernel<TPR><<<mc::grid_for(rows, 256 / TPR), 256, 0, s>>>(x, x_dtype == MC_BF16, rows, cols, eps, mode,       \
                                                                            p0, p1, scale_idx, shift_idx,                      \
                                                                            round_ln_to_bf16, out, out_dtype == MC_BF16)
#define MC_LNP(G)                                                                                                              \
  mc::ln_modulate_pipe_kernel<G><<<mc::pipe_grid(rows, (G) >= 6 ? 1 : 2), 256, 0, s>>>(x, x_dtype == MC_BF16, rows, cols, eps, mode, p0, p1,      \
                                                                     scale_idx, shift_idx, round_ln_to_bf16, out, out_dtype == MC_BF16)
  // long inputs: the TMA-staged form (needs >= 2 stages of 8 rows in shared memory and 16-byte aligned rows)
  const int ring = rows >= 1024 && groups <= 32 * mc::kMaxG ? mc::ring_stages(mc::kRingRows * cols * (x_dtype == MC_BF16 ? 2 : 4)) : 0;
  if (ring > 0) {
    const int smem = ring * mc::kRingRows * cols * (x_dtype == MC_BF16 ? 2 : 4) + ring * 16 + 64;
    const int64_t chunks = (rows + mc::kRingRows - 1) / mc::kRingRows;
    const int grid = static_cast<int>(chunks < mc::num_sms() ? chunks : mc::num_sms());
    int32_t rc = MC_OK;
#define MC_LNT(G, IDX)                                                                                                                 \
  do {                                                                                                                                 \
    static mc::PerDeviceOnce once_##IDX;                                                                                               \
    rc = mc::set_max_smem_once(mc::ln_modulate_tma_kernel<G, mc::kLnRingGroups>, 208 * 1024, once_##IDX, "cudaFuncSetAttribute(ln_modulate_tma smem)");   \
    if (rc == MC_OK)                                                                                                                   \
      mc::ln_modulate_tma_kernel<G, mc::kLnRingGroups><<<grid, mc::ring_threads(mc::kLnRingGroups), smem, s>>>(x, x_dtype == MC_BF16, rows, cols, eps, mode, p0, p1, scale_idx, \
                                                                        shift_idx, round_ln_to_bf16, out, out_dtype == MC_BF16, ring); \
  } while (0)
    if (groups <= 32 * 2) MC_LNT(2, 2);
    else if (groups <= 32 * 4) MC_LNT(4, 4);
    else if (groups <= 32 * 6) MC_LNT(6, 6);
    else MC_LNT(8, 8);
#undef MC_LNT
    if (rc) return rc;
    MC_CHECK_LAUNCH("ln_modulate_tma_kernel launch");
    return MC_OK;
  }
  if (groups <= 32 * 2) MC_LNP(2);
  else if (groups <= 32 * 4) MC_LNP(4);
  else if (groups <= 32 * 6) MC_LNP(6);
  else if (groups <= 32 * mc::kMaxG) MC_LNP(8);
  else MC_LN(128);
#undef MC_LNP
#undef MC_LN
  MC_CHECK_LAUNCH("ln_modulate_kernel launch");
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
  MC_CHECK_ARG(rows >= 1 && cols >= 8 && cols % 8 == 0 && cols <= 128 * 8 * mc::kMaxG && ld >= static_cast<int64_t>(segs) * cols && ld % 8 == 0,
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
  const int ring = ring_ok ? mc::ring_stages(ring_stage_bytes) : 0;
  if (ring > 0) {
    const int smem = ring * ring_stage_bytes + ring * 16 + 64;
    const int64_t chunks = (rows + rows_per_stage - 1) / rows_per_stage;
    const int grid = static_cast<int>(chunks < mc::num_sms() ? chunks : mc::num_sms());
    int32_t rc = MC_OK;
#define MC_RMST(G, IDX)                                                                                                                 \
  do {                                                                                                                                  \
    static mc::PerDeviceOnce once_##IDX;                                                                                                \
    rc = mc::set_max_smem_once(mc::rmsnorm_rope_tma_kernel<G, mc::kRmsRingGroups>, 208 * 1024, once_##IDX, "cudaFuncSetAttribute(rmsnorm_rope_tma smem)"); \
    if (rc == MC_OK)                                                                                                                    \
      mc::rmsnorm_rope_tma_kernel<G, mc::kRmsRingGroups><<<grid, mc::ring_threads(mc::kRmsRingGroups), smem, s>>>(xp, ld, rows, segs, cols, w, eps, cos_sin, head_dim, ring);   \
  } while (0)
    if (groups <= 32 * 2) MC_RMST(2, 2);
    else if (groups <= 32 * 4) MC_RMST(4, 4);
    else if (groups <= 32 * 6) MC_RMST(6, 6);
    else MC_RMST(8, 8);
#undef MC_RMST
    if (rc) return rc;
    MC_CHECK_LAUNCH("rmsnorm_rope_tma_kernel launch");
    return MC_OK;
  }
#define MC_RMSP(G) mc::rmsnorm_rope_pipe_kernel<G><<<mc::pipe_grid(rows * segs), 256, 0, s>>>(xp, ld, rows, segs, cols, w, eps, cos_sin, head_dim)
  if (groups <= 32 * 2) MC_RMSP(2);
  else if (groups <= 32 * 4) MC_RMSP(4);
  else if (groups <= 32 * 6) MC_RMSP(6);
  else if (groups <= 32 * mc::kMaxG) MC_RMSP(8);
  else {
    // wide rows (Wan-14B: 5120): four warps per row, one column block per launch
    for (int sg = 0; sg < segs; ++sg)
      mc::rmsnorm_rope_kernel<128><<<mc::grid_for(rows, 2), 256, 0, s>>>(xp + static_cast<int64_t>(sg) * cols, ld, rows, cols,
                                                                        w + static_cast<int64_t>(sg) * cols, eps, cos_sin, head_dim);
  }
#undef MC_RMSP
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
