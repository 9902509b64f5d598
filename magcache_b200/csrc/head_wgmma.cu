// Head of the Wan forward — LayerNorm (no affine) + modulation + fp32 Linear(cols -> 64) + unpatchify — and the cache-hit branch
// in front of it, as ONE streaming pass (MagCache4Wan2.1/magcache_generate.py:293-295 `x = x + residual_x`, :304-305 `head`,
// `unpatchify`; `Head` itself is upstream wan/modules/model.py [EXT], restated in oracle/wan_ref.py::Head).
//
// The row statistics and the Linear commute:   with  s_k = 1 + e1_k,  t_k = e0_k,  W'_ck = s_k W_ck,
//     y_c = sum_k ((x_k - mu) rstd s_k + t_k) W_ck + b_c = rstd * (sum_k x_k W'_ck - mu * sum_k W'_ck) + (sum_k t_k W_ck + b_c)
// so every row is read exactly ONCE: while its 64-column chunks stream through registers the kernel (a) accumulates the row's
// mean / M2 (Chan's pairwise update, fp32) and (b) feeds the raw values to the tensor cores as the A operand of a
// [rows x cols] x [cols x 64] GEMM against W'. The reference runs this Linear in fp32 (`amp.autocast(dtype=torch.float32)`), so
// the GEMM uses a 3-pass split: x = x_hi + x_lo, W' = W'_hi + W'_lo (bf16 pairs), acc = x_hi W'_hi + x_lo W'_hi + x_hi W'_lo in
// fp32 accumulators — products carry ~2^-17 relative error instead of bf16's 2^-9. To keep `acc - mu * c1` from cancelling when
// a row has a large common offset, every row is shifted by a pilot value p (the mean of its first 64 elements) before the split;
// LayerNorm is shift invariant, so only mu changes to mu - p.
//
// HBM-bound: per row cols * 4 B (fp32 stream), or cols * (2 + 4) B on a cache hit (bf16 patch embedding + fp32 cached residual,
// the sum never materialised), + 256 B out. One CTA per SM, each owning a contiguous row range (balanced to one row). A TMA warp
// streams the rows in [128 x 64] chunks into a shared-memory ring (96 KB in flight per SM, no registers tied up in loads) next to
// the W' chunks; 16 converter warps (4 threads per row) read the staged values, update the statistics and write the hi / lo
// operand tiles. The first converter warpgroup also issues the wgmmas of each chunk once all operand tiles are written (two
// m64n64 accumulators in its registers, rows 0-63 and 64-127) and runs them while it converts the next chunk; at the end of a
// row tile it parks the accumulator in shared memory for the epilogue. Warp-shuffle reductions merge the four threads of a row.
#include <type_traits>

#include "common.cuh"
#include "ptx.cuh"
#include "tma_host.cuh"

namespace mc {
namespace hd {
constexpr int kRows = 128, kKC = 64, kOut = 64;
constexpr int kATile = kRows * kKC * 2;      // 16 KB: one bf16 operand tile (hi or lo), 128-byte rows, 128-byte swizzle
constexpr int kWTile = kOut * kKC * 2;       // 8 KB
constexpr int kOpStage = 2 * kATile + 2 * kWTile;  // 48 KB: A_hi, A_lo, W'_hi, W'_lo of one 64-column chunk
constexpr int kOpStages = 2;
constexpr int kRawF32 = kRows * kKC * 4;     // 32 KB: the fp32 chunk as two TMA boxes [128 rows x 32 fp32] (128-byte rows, swizzled)
constexpr int kRawBf16 = kRows * kKC * 2;    // 16 KB: the bf16 chunk (cache hit: patch embedding), one box [128 x 64 bf16]
constexpr int kConvWarps = 16;
constexpr int kConvThreads = kConvWarps * 32;  // 512: 4 threads per row
constexpr int kThreads = kConvThreads + 128;   // + one data-path warpgroup: TMA warp, three idle warps
constexpr int kIssueRegs = 144, kConvRegs = 104, kDataRegs = 24;  // setmaxnreg: 24 * 128 + 144 * 128 + 104 * 384 = 96 * 640
constexpr int kAccPad = kOut + 1;              // floats per parked accumulator row (conflict-free row reads)
constexpr int kMaxPeers = 8;
template <bool HIT>
struct Layout {
  static constexpr int kRawStage = kRawF32 + (HIT ? kRawBf16 : 0);  // 48 KB on a hit, 32 KB otherwise
  static constexpr int kRawStages = HIT ? 2 : 3;                    // 96 KB of loads in flight per SM either way
  static constexpr int kOffRaw = kOpStages * kOpStage;              // 96 KB
  static constexpr int kOffStats = kOffRaw + kRawStages * kRawStage;  // 192 KB
  static constexpr int kOffAcc = kOffStats + 2 * kRows * 8;          // row statistics, double-buffered by row tile
  static constexpr int kOffBars = kOffAcc + kRows * kAccPad * 4;
  static constexpr int kSmem = kOffBars + 256;      // 232192 of the 232448 an H100 block may use
};
}  // namespace hd

struct HeadParams {
  int round_sum_bf16;
  int64_t rows, row_offset;
  int cols, F, Hp, Wp;
  int rows_per_cta, tail_rows;  // rows of the last 128-row tile of a CTA's range (its own TMA box height; 0: the range is a multiple of 128)
  const float* c1;     // [64] sum_k W'_ck
  const float* c0;     // [64] sum_k t_k W_ck + b_c
  float eps;
  float* out[hd::kMaxPeers];  // fp32 [16, F, 2Hp, 2Wp] — the caller's own and, token-sharded, every peer's (P2P stores)
  int n_out;
  // Caller-loop step folded into the epilogue (SURVEY §8f-1; eval/.../wan_magcache.py:301-310): this launch is the UNCONDITIONAL
  // head of a step; instead of its prediction it writes  out = coef_x * x + coef_v * (y + g * (cond - y))  with `cond` the
  // conditional prediction of the same step and `x` the current latent (both in the output layout; x may alias out).
  const float* step_cond;  // nullptr: plain head
  const float* step_x;
  float step_g, step_cx, step_cv;
  // head_tc_kernel<HIT, true> only (mc_head_unpatchify_step_hist): one history term of a multistep solver, out += coef_h * hist,
  // and the x0-prediction x - sigma * v stored to step_x0 when it is given (DPM++ 2M keeps it for the next step)
  const float* step_hist;
  float* step_x0;
  float step_ch, step_sigma;
};

// ---- per-forward preparation: W' = (1 + e1) * W split into bf16 hi / lo, K-major [64, cols]; c1, c0 ----------------------------
__global__ void __launch_bounds__(256) head_prep_kernel(const float* __restrict__ head_mod, const float* __restrict__ e,
                                                        const float* __restrict__ Wt, const float* __restrict__ bias, int cols,
                                                        __nv_bfloat16* __restrict__ w_hi, __nv_bfloat16* __restrict__ w_lo,
                                                        float* __restrict__ c1, float* __restrict__ c0) {
  __shared__ double red[2][8];
  const int c = blockIdx.x;
  double s1 = 0.0, s0 = 0.0;
  for (int k = threadIdx.x; k < cols; k += blockDim.x) {
    const float sk = 1.0f + (head_mod[cols + k] + e[k]);  // e[1] = modulation[1] + e
    const float tk = head_mod[k] + e[k];                  // e[0] = modulation[0] + e
    const float w = Wt[static_cast<int64_t>(k) * hd::kOut + c];
    const float wp = sk * w;
    const __nv_bfloat16 hi = __float2bfloat16_rn(wp);
    const __nv_bfloat16 lo = __float2bfloat16_rn(wp - __bfloat162float(hi));
    w_hi[static_cast<int64_t>(c) * cols + k] = hi;
    w_lo[static_cast<int64_t>(c) * cols + k] = lo;
    s1 += static_cast<double>(__bfloat162float(hi)) + static_cast<double>(__bfloat162float(lo));  // what the MMA multiplies by
    s0 += static_cast<double>(tk) * static_cast<double>(w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = s1;
    red[1][threadIdx.x >> 5] = s0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int i = 0; i < 8; ++i) a += red[0][i], b += red[1][i];
    c1[c] = static_cast<float>(a);
    c0[c] = static_cast<float>(b + static_cast<double>(bias[c]));
  }
}

// Host: 2-D fp32 tensor map [rows, cols], box [box_rows, 32 fp32] (128-byte rows), 128-byte swizzle, zero fill out of bounds.
static int32_t make_tmap_f32_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return MC_ERR_CUDA;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {cols * 4};
  cuuint32_t box[2] = {32, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(fp32) failed (CUresult %d): base=%p rows=%llu cols=%llu box_rows=%u", static_cast<int>(r), base,
              static_cast<unsigned long long>(rows), static_cast<unsigned long long>(cols), box_rows);
    return MC_ERR_CUDA;
  }
  return MC_OK;
}

// Tensor maps of one launch: the fp32 rows (residual stream, or the cached residual on a hit) and the bf16 rows (hit only), each with
// a full-height (128-row) box and a tail box for the last tile of a CTA's row range — so no CTA fetches a row it does not own.
struct HeadMaps {
  CUtensorMap f32_full, f32_tail, bf16_full, bf16_tail, w_hi, w_lo;
};

// HIST: the fused step with a history operand and the x0 output (mc_head_unpatchify_step_hist); the HIST = false instantiations are
// the plain head and mc_head_unpatchify_step, whose code the HIST branches do not touch.
template <bool HIT, bool HIST = false>
__global__ void __launch_bounds__(hd::kThreads, 1) head_tc_kernel(const __grid_constant__ HeadMaps maps, const HeadParams p) {
  using namespace hd;
  using L = Layout<HIT>;
  extern __shared__ __align__(1024) uint8_t smem[];
  // (mean - pilot, rstd) per tile row, [2][kRows]: tile st uses half st & 1. A converter warp publishes tile st + 1's statistics
  // before the barrier of tile st + 1, while an epilogue warp may still read tile st's: with one or two chunks per row (cols <=
  // 128) nothing else holds the converter back. It cannot reach tile st + 2 before every epilogue warp has passed that barrier.
  float2* stats_buf = reinterpret_cast<float2*>(smem + L::kOffStats);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBars);
  uint64_t* raw_full = bars + 0;    // [kRawStages] TMA
  uint64_t* raw_empty = bars + 3;   // [kRawStages] 16 arrivals (one per converter warp): the raw chunk has been read into registers
  uint64_t* a_full = bars + 6;      // [kOpStages] 16 arrivals: hi / lo operand tiles written
  uint64_t* w_full = bars + 8;      // [kOpStages] TMA
  uint64_t* op_empty = bars + 10;   // [kOpStages] 4 arrivals (issuing warps): the wgmmas that read A and W' of this stage have retired
  float* acc_park = reinterpret_cast<float*>(smem + L::kOffAcc);  // [kRows][kAccPad] accumulator of the current row tile

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkc = p.cols / kKC;
  const int64_t cta_row0 = static_cast<int64_t>(blockIdx.x) * p.rows_per_cta;
  const int64_t cta_row1 = min(cta_row0 + p.rows_per_cta, p.rows);
  const int n_sub = cta_row1 > cta_row0 ? static_cast<int>((cta_row1 - cta_row0 + kRows - 1) / kRows) : 0;
  const int n_sub_full = (p.rows_per_cta + kRows - 1) / kRows;  // tiles of a full range: the last of them uses the tail box

  if (threadIdx.x == 0) {
    if ((ptx::smem_u32(smem) & 1023u) != 0) {
      MC_DIAG("head_tc_kernel: dynamic smem base not 1024-aligned\n");
      __trap();
    }
    ptx::prefetch_tmap(&maps.f32_full);
    ptx::prefetch_tmap(&maps.w_hi);
    ptx::prefetch_tmap(&maps.w_lo);
    for (int s = 0; s < L::kRawStages; ++s) {
      ptx::mbar_init(&raw_full[s], 1);
      ptx::mbar_init(&raw_empty[s], kConvWarps);
    }
    for (int s = 0; s < kOpStages; ++s) {
      ptx::mbar_init(&a_full[s], kConvWarps);
      ptx::mbar_init(&w_full[s], 1);
      ptx::mbar_init(&op_empty[s], 4);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp >= kConvWarps + 1) {
    ptx::setmaxnreg_dec<kDataRegs>();  // idle warps of the data-path warpgroup
  } else if (warp == kConvWarps) {
    // ------------------------------------------------ TMA producer: raw row chunks and W' hi / lo chunks ------------------------
    ptx::setmaxnreg_dec<kDataRegs>();
    int rs = 0, os = 0;
    uint32_t rph = 0, oph = 0;
    for (int st = 0; st < n_sub; ++st) {
      const bool tail = p.tail_rows != 0 && st == n_sub_full - 1;
      const int r0 = static_cast<int>(cta_row0) + st * kRows;
      const uint32_t raw_bytes = static_cast<uint32_t>((tail ? p.tail_rows : kRows) * kKC * (HIT ? 6 : 4));
      for (int kc = 0; kc < nkc; ++kc) {
        ptx::mbar_wait(&raw_empty[rs], rph ^ 1);
        if (ptx::elect_one()) {
          uint8_t* dst = smem + L::kOffRaw + rs * L::kRawStage;
          ptx::mbar_expect_tx(&raw_full[rs], raw_bytes);
          const CUtensorMap* mf = tail ? &maps.f32_tail : &maps.f32_full;
          ptx::tma_load_2d(dst, mf, &raw_full[rs], kc * kKC, r0);
          ptx::tma_load_2d(dst + kRawF32 / 2, mf, &raw_full[rs], kc * kKC + 32, r0);
          if (HIT) ptx::tma_load_2d(dst + kRawF32, tail ? &maps.bf16_tail : &maps.bf16_full, &raw_full[rs], kc * kKC, r0);
        }
        __syncwarp();
        if (++rs == L::kRawStages) rs = 0, rph ^= 1;
        ptx::mbar_wait(&op_empty[os], oph ^ 1);
        if (ptx::elect_one()) {
          uint8_t* wdst = smem + os * kOpStage + 2 * kATile;
          ptx::mbar_expect_tx(&w_full[os], 2 * kWTile);
          ptx::tma_load_2d(wdst, &maps.w_hi, &w_full[os], kc * kKC, 0);
          ptx::tma_load_2d(wdst + kWTile, &maps.w_lo, &w_full[os], kc * kKC, 0);
        }
        __syncwarp();
        if (++os == kOpStages) os = 0, oph ^= 1;
      }
    }
  } else {
    // ------------------------------------------------ converter warps (+ wgmma issue, epilogue) --------------------------------
    // instantiated twice: ISSUE for the first warpgroup (which also holds the accumulators), plain for the other three
    auto convert = [&](auto issue_tag) {
    constexpr bool ISSUE = decltype(issue_tag)::value;
    float acc_a[32], acc_b[32];  // ISSUE only: rows [0, 64) and [64, 128) of the row tile
    const int tid = threadIdx.x;
    const int rt = tid >> 2, sub = tid & 3;  // tile row; this thread owns columns [8 sub, 8 sub + 8) and [32 + 8 sub, 32 + 8 sub + 8) of a chunk
    const int sw = rt & 7;
    const uint32_t row_off = static_cast<uint32_t>((rt >> 3) * 1024 + sw * 128);
    // 16-byte chunk offsets inside a 128-byte swizzled row (chunk index XOR row % 8):
    const uint32_t f0 = static_cast<uint32_t>(((2 * sub) ^ sw) * 16), f1 = static_cast<uint32_t>(((2 * sub + 1) ^ sw) * 16);  // fp32 box: 8 floats = 2 chunks
    const uint32_t h0 = static_cast<uint32_t>((sub ^ sw) * 16), h1 = static_cast<uint32_t>(((4 + sub) ^ sw) * 16);            // bf16 rows: 8 elements = 1 chunk
    int rs = 0, os = 0;
    uint32_t rph = 0, oph = 0;
    const float inv_cols = 1.0f / static_cast<float>(p.cols);
    for (int st = 0; st < n_sub; ++st) {
      int prev_os = -1;
      float2* stats = stats_buf + (st & 1) * kRows;
      const int64_t row = cta_row0 + static_cast<int64_t>(st) * kRows + rt;
      const bool live = row < cta_row1;
      float pilot = 0.f, mean = 0.f, m2 = 0.f;  // running mean / M2 of the shifted values over the slices this thread has seen
      for (int kc = 0; kc < nkc; ++kc) {
        // ---- this thread's 16 values of the chunk, from the TMA-staged rows
        float v[16];
        ptx::mbar_wait(&raw_full[rs], rph);
        {
          const uint8_t* raw = smem + L::kOffRaw + rs * L::kRawStage + row_off;
          const float4 a0 = *reinterpret_cast<const float4*>(raw + f0), a1 = *reinterpret_cast<const float4*>(raw + f1);
          const float4 b0 = *reinterpret_cast<const float4*>(raw + kRawF32 / 2 + f0), b1 = *reinterpret_cast<const float4*>(raw + kRawF32 / 2 + f1);
          v[0] = a0.x, v[1] = a0.y, v[2] = a0.z, v[3] = a0.w, v[4] = a1.x, v[5] = a1.y, v[6] = a1.z, v[7] = a1.w;
          v[8] = b0.x, v[9] = b0.y, v[10] = b0.z, v[11] = b0.w, v[12] = b1.x, v[13] = b1.y, v[14] = b1.z, v[15] = b1.w;
          if (HIT) {
            const uint4 x0 = *reinterpret_cast<const uint4*>(raw + kRawF32 + h0), x1 = *reinterpret_cast<const uint4*>(raw + kRawF32 + h1);
            const uint32_t xb[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) {  // `x + residual_x`: bf16 -> fp32 promotion, fp32 add (exactly torch's promoted add)
              v[2 * i] = bf16_lo(xb[i]) + v[2 * i];
              v[2 * i + 1] = bf16_hi(xb[i]) + v[2 * i + 1];
            }
            if (p.round_sum_bf16) {  // in-place `x += residual` on a bf16 tensor (TeaCache comparator, wan_teacache.py:569/577)
#pragma unroll
              for (int i = 0; i < 16; ++i) v[i] = round_bf16(v[i]);
            }
          }
        }
        if (!live) {
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] = 0.f;  // rows past the range (tail box: not loaded; zero-filled or stale smem)
        }
        // ---- statistics
        if (kc == 0) {  // pilot = mean of the row's first 64 elements (4 adjacent lanes)
          float s = 0.f;
#pragma unroll
          for (int i = 0; i < 16; ++i) s += v[i];
          s += __shfl_xor_sync(0xffffffffu, s, 1);
          s += __shfl_xor_sync(0xffffffffu, s, 2);
          pilot = s * (1.0f / 64.0f);
        }
        float cs = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          v[i] -= pilot;
          cs += v[i];
        }
        // every staged value has been consumed by the sum above (the loads have completed, not merely issued): hand the stage back
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&raw_empty[rs]);
        if (++rs == L::kRawStages) rs = 0, rph ^= 1;
        const float cm = cs * (1.0f / 16.0f);
        float cq = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const float d = v[i] - cm;
          cq = fmaf(d, d, cq);
        }
        // Chan: combine (n_a = 16*kc, mean, m2) with (16, cm, cq)
        const float na = 16.0f * static_cast<float>(kc), rn = 1.0f / (na + 16.0f);
        const float delta = cm - mean;
        mean = fmaf(delta, 16.0f * rn, mean);
        m2 += fmaf(delta * delta, na * 16.0f * rn, cq);

        // ---- hi / lo split into the swizzled operand tiles: columns [8 sub, +8) -> chunk sub, [32 + 8 sub, +8) -> chunk 4 + sub
        ptx::mbar_wait(&op_empty[os], oph ^ 1);
        uint8_t* arow = smem + os * kOpStage + row_off;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float a = v[hf * 8 + 2 * i], b = v[hf * 8 + 2 * i + 1];
            hi[i] = pack_bf16x2(a, b);
            lo[i] = pack_bf16x2(a - bf16_lo(hi[i]), b - bf16_hi(hi[i]));
          }
          const uint32_t ch = hf == 0 ? h0 : h1;
          *reinterpret_cast<uint4*>(arow + ch) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
          *reinterpret_cast<uint4*>(arow + kATile + ch) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
        ptx::fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&a_full[os]);
        if constexpr (ISSUE) {
          ptx::mbar_wait(&a_full[os], oph);
          ptx::mbar_wait(&w_full[os], oph);
          const uint32_t base = ptx::smem_u32(smem + os * kOpStage);
          const uint64_t a_hi = ptx::gmma_desc_sw128_kmajor(base), a_lo = ptx::gmma_desc_sw128_kmajor(base + kATile);
          const uint64_t w_hi = ptx::gmma_desc_sw128_kmajor(base + 2 * kATile), w_lo = ptx::gmma_desc_sw128_kmajor(base + 2 * kATile + kWTile);
          constexpr uint64_t kHalf = (64 * 128) >> 4;  // rows 64-127: 8 row groups of 1024 B further
          ptx::wgmma_fence();
#pragma unroll
          for (int k = 0; k < kKC / 16; ++k) {
            const uint32_t first = (kc | k) != 0 ? 1u : 0u;
            ptx::wgmma_m64n64k16_ss(acc_a, a_hi + 2 * k, w_hi + 2 * k, first);
            ptx::wgmma_m64n64k16_ss(acc_b, a_hi + kHalf + 2 * k, w_hi + 2 * k, first);
            ptx::wgmma_m64n64k16_ss(acc_a, a_lo + 2 * k, w_hi + 2 * k, 1u);
            ptx::wgmma_m64n64k16_ss(acc_b, a_lo + kHalf + 2 * k, w_hi + 2 * k, 1u);
            ptx::wgmma_m64n64k16_ss(acc_a, a_hi + 2 * k, w_lo + 2 * k, 1u);
            ptx::wgmma_m64n64k16_ss(acc_b, a_hi + kHalf + 2 * k, w_lo + 2 * k, 1u);
          }
          ptx::wgmma_commit();
          ptx::wgmma_wait<1>();  // the previous chunk's wgmmas have retired: its operand stage can be refilled
          ptx::fence_regs(acc_a);
          ptx::fence_regs(acc_b);
          if (prev_os >= 0 && lane == 0) ptx::mbar_arrive(&op_empty[prev_os]);
          prev_os = os;
        }
        if (++os == kOpStages) os = 0, oph ^= 1;
      }
      if constexpr (ISSUE) {
        ptx::wgmma_wait<0>();
        ptx::fence_regs(acc_a);
        ptx::fence_regs(acc_b);
        if (lane == 0) ptx::mbar_arrive(&op_empty[prev_os]);
        // park the accumulator for the epilogue warps (their reads of the previous tile's are done: they arrived on this tile's
        // a_full barriers after them)
        const int ar = (warp & 3) * 16 + (lane >> 2), ac = 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < kOut / 8; ++i) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int rr = ar + (e >> 1) * 8, cc = 8 * i + ac + (e & 1);
            acc_park[rr * kAccPad + cc] = acc_a[4 * i + e];
            acc_park[(rr + 64) * kAccPad + cc] = acc_b[4 * i + e];
          }
        }
      }
      // row statistics: merge the four slices of the row (Chan again, equal counts), publish (mean_shifted, rstd)
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, mean, o), oq = __shfl_xor_sync(0xffffffffu, m2, o);
        const float cnt = static_cast<float>(p.cols) * (o == 1 ? 0.25f : 0.5f);  // elements behind each side
        const float delta = om - mean;
        mean = 0.5f * (mean + om);
        m2 = m2 + oq + delta * delta * (cnt * 0.5f);
      }
      if (sub == 0) stats[rt] = make_float2(mean, rsqrtf(m2 * inv_cols + p.eps));
      asm volatile("bar.sync 1, %0;" ::"n"(kConvThreads) : "memory");
      if (warp < 8) {
        // ---- epilogue: y = rstd * (acc - mean_shifted * c1) + c0 -> unpatchify. Warp = (32-row quarter, 32-column half);
        // output feature j = (q*2 + rr)*16 + c -> out[c, f, 2*hp+q, 2*wp+rr]: columns [32q, 32q+32) hold rr = 0 | rr = 1 for the
        // same 16 channels, so every store is one float2 and a warp writes 256 contiguous bytes per channel row.
        const int qtr = warp & 3, qh = warp >> 2;
        const int er = qtr * 32 + lane;
        const int64_t erow = cta_row0 + static_cast<int64_t>(st) * kRows + er;
        const bool elive = erow < cta_row1;
        const int64_t tok = p.row_offset + erow;
        const int wp = static_cast<int>(tok % p.Wp);
        const int hp = static_cast<int>((tok / p.Wp) % p.Hp);
        const int f = static_cast<int>(tok / (static_cast<int64_t>(p.Wp) * p.Hp));
        const int H2 = p.Hp * 2, W2 = p.Wp * 2;
        const int64_t plane = static_cast<int64_t>(p.F) * H2 * W2;
        const int64_t off = (static_cast<int64_t>(f) * H2 + hp * 2 + qh) * W2 + wp * 2;
        const bool step = (HIST || p.step_cond != nullptr) && elive;
        // fused caller step: the conditional prediction and the latent at this thread's 16 output positions, fetched in two batches
        // of 8 channels; the first batch is in flight while the last MMAs of the tile finish (x may alias out: every position is
        // read by the thread that later writes it, before it writes it). HIST: the history term at the same positions too, in four
        // batches of 4 channels (three operands per position: the registers of two batches of 8)
        constexpr int kB = HIST ? 4 : 8;
        float2 cc[kB], xl[kB];
        [[maybe_unused]] float2 hl[kB];
        auto fetch = [&](int c0) {
#pragma unroll
          for (int c = 0; c < kB; ++c) {
            cc[c] = *reinterpret_cast<const float2*>(p.step_cond + (c0 + c) * plane + off);
            xl[c] = *reinterpret_cast<const float2*>(p.step_x + (c0 + c) * plane + off);
            if constexpr (HIST) hl[c] = *reinterpret_cast<const float2*>(p.step_hist + (c0 + c) * plane + off);
          }
        };
        if (step) fetch(0);
        const float* acc = acc_park + er * kAccPad + qh * 32;
        if (elive) {
          const float2 ms = stats[er];
#pragma unroll
          for (int cb = 0; cb < 16; cb += kB) {
            if (step && cb != 0) fetch(cb);
#pragma unroll
            for (int ci = 0; ci < kB; ++ci) {
              const int c = cb + ci;
              const int j0 = qh * 32 + c, j1 = j0 + 16;
              float y0 = fmaf(ms.y, acc[c] - ms.x * __ldg(p.c1 + j0), __ldg(p.c0 + j0));
              float y1 = fmaf(ms.y, acc[16 + c] - ms.x * __ldg(p.c1 + j1), __ldg(p.c0 + j1));
              if (step) {
                // same operations, same order, each rounded separately, as mc_cfg_step (cache_kernels.cu::cfg_step_one): bit-identical
                const float v0 = __fadd_rn(y0, __fmul_rn(p.step_g, __fsub_rn(cc[ci].x, y0)));
                const float v1 = __fadd_rn(y1, __fmul_rn(p.step_g, __fsub_rn(cc[ci].y, y1)));
                y0 = __fadd_rn(__fmul_rn(p.step_cx, xl[ci].x), __fmul_rn(p.step_cv, v0));
                y1 = __fadd_rn(__fmul_rn(p.step_cx, xl[ci].y), __fmul_rn(p.step_cv, v1));
                if constexpr (HIST) {  // cfg_step_one with one history term: + coef_h * h, then x0 = x - sigma * v
                  y0 = __fadd_rn(y0, __fmul_rn(p.step_ch, hl[ci].x));
                  y1 = __fadd_rn(y1, __fmul_rn(p.step_ch, hl[ci].y));
                  if (p.step_x0)
                    *reinterpret_cast<float2*>(p.step_x0 + c * plane + off) =
                        make_float2(__fsub_rn(xl[ci].x, __fmul_rn(p.step_sigma, v0)), __fsub_rn(xl[ci].y, __fmul_rn(p.step_sigma, v1)));
                }
              }
              for (int o = 0; o < p.n_out; ++o) *reinterpret_cast<float2*>(p.out[o] + c * plane + off) = make_float2(y0, y1);
            }
          }
        }
      }
    }
    };
    if (warp < 4) {
      ptx::setmaxnreg_inc<kIssueRegs>();
      convert(std::true_type{});
    } else {
      ptx::setmaxnreg_inc<kConvRegs>();
      convert(std::false_type{});
    }
  }
}

}  // namespace mc

extern "C" {

int32_t mc_head_workspace_bytes(int32_t cols, int64_t* bytes_out) {
  MC_CHECK_ARG(bytes_out != nullptr && cols >= 64, "mc_head_workspace_bytes: bad arguments");
  *bytes_out = static_cast<int64_t>(2) * 64 * cols * 2 + 1024;  // W'_hi, W'_lo [64, cols] bf16; c1, c0 [64] fp32
  return MC_OK;
}

static int32_t head_workspace_split(void* workspace, int64_t workspace_bytes, int32_t cols, __nv_bfloat16** w_hi, __nv_bfloat16** w_lo, float** c1,
                                    float** c0) {
  int64_t need = 0;
  mc_head_workspace_bytes(cols, &need);
  MC_CHECK_ARG(workspace != nullptr && workspace_bytes >= need && (reinterpret_cast<uintptr_t>(workspace) & 1023u) == 0,
               "mc_head: workspace of %lld bytes, 1024-byte aligned, needed (mc_head_workspace_bytes)", static_cast<long long>(need));
  *w_hi = static_cast<__nv_bfloat16*>(workspace);
  *w_lo = *w_hi + static_cast<size_t>(64) * cols;
  *c1 = reinterpret_cast<float*>(*w_lo + static_cast<size_t>(64) * cols);
  *c0 = *c1 + 64;
  return MC_OK;
}

int32_t mc_head_prepare(const float* head_mod, const float* e, const float* Wt, const float* b, int32_t cols, void* workspace,
                        int64_t workspace_bytes, void* stream) {
  using namespace mc;
  MC_CHECK_ARG(head_mod && e && Wt && b, "mc_head_prepare: null pointer");
  MC_CHECK_ARG(cols >= hd::kKC && cols % hd::kKC == 0, "mc_head_prepare: cols=%d must be a multiple of %d", cols, hd::kKC);
  __nv_bfloat16 *w_hi, *w_lo;
  float *c1, *c0;
  const int32_t rc = head_workspace_split(workspace, workspace_bytes, cols, &w_hi, &w_lo, &c1, &c0);
  if (rc) return rc;
  head_prep_kernel<<<hd::kOut, 256, 0, static_cast<cudaStream_t>(stream)>>>(head_mod, e, Wt, b, cols, w_hi, w_lo, c1, c0);
  MC_CHECK_LAUNCH("head_prep_kernel launch");
  return MC_OK;
}

static int32_t head_launch(const void* x, int32_t x_dtype, const float* r_or_null, int64_t rows, int64_t row_offset, int32_t cols, int32_t F,
                           int32_t Hp, int32_t Wp, int32_t C_out, float eps, float* const* outs, int32_t n_out, const void* prepared,
                           int64_t prepared_bytes, int32_t flags, const float* step_cond, const float* step_x, float step_g, float step_cx,
                           float step_cv, const float* step_hist, float step_ch, float step_sigma, float* step_x0, void* stream) {
  using namespace mc;
  MC_CHECK_ARG(x && outs && prepared, "mc_head_unpatchify: null pointer");
  MC_CHECK_ARG(n_out >= 1 && n_out <= hd::kMaxPeers, "mc_head_unpatchify: n_out=%d outside [1, %d]", n_out, hd::kMaxPeers);
  MC_CHECK_ARG(cols >= hd::kKC && cols % hd::kKC == 0, "mc_head_unpatchify: cols=%d must be a multiple of %d", cols, hd::kKC);
  MC_CHECK_ARG(C_out * 4 == hd::kOut, "mc_head_unpatchify: only patch (1,2,2) x C_out=16 (64 output features) is built, got C_out=%d", C_out);
  MC_CHECK_ARG(F >= 1 && Hp >= 1 && Wp >= 1, "mc_head_unpatchify: bad grid");
  MC_CHECK_ARG(rows >= 1 && row_offset >= 0 && row_offset + rows <= static_cast<int64_t>(F) * Hp * Wp,
               "mc_head_unpatchify: token range [%lld, %lld) outside the %d x %d x %d grid", static_cast<long long>(row_offset),
               static_cast<long long>(row_offset + rows), F, Hp, Wp);
  MC_CHECK_ARG((x_dtype == MC_F32 && r_or_null == nullptr) || (x_dtype == MC_BF16 && r_or_null != nullptr),
               "mc_head_unpatchify: x must be fp32 (stream) or bf16 together with an fp32 residual (cache hit)");
  MC_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15u) == 0 && (r_or_null == nullptr || (reinterpret_cast<uintptr_t>(r_or_null) & 15u) == 0),
               "mc_head_unpatchify: x / r must be 16-byte aligned");
  __nv_bfloat16 *w_hi, *w_lo;
  float *c1, *c0;
  int32_t rc = head_workspace_split(const_cast<void*>(prepared), prepared_bytes, cols, &w_hi, &w_lo, &c1, &c0);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);

  HeadParams p{};
  p.round_sum_bf16 = (flags & 1) != 0;
  p.rows = rows, p.row_offset = row_offset, p.cols = cols, p.F = F, p.Hp = Hp, p.Wp = Wp;
  const int sms = num_sms();
  p.rows_per_cta = static_cast<int>((rows + sms - 1) / sms);  // contiguous row range per CTA: HBM bytes balanced to one row
  if (p.rows_per_cta < 16) p.rows_per_cta = 16;
  p.tail_rows = p.rows_per_cta % hd::kRows;
  p.c1 = c1, p.c0 = c0, p.eps = eps;
  for (int i = 0; i < n_out; ++i) {
    MC_CHECK_ARG(outs[i] != nullptr && (reinterpret_cast<uintptr_t>(outs[i]) & 7u) == 0, "mc_head_unpatchify: out[%d] null or not 8-byte aligned", i);
    p.out[i] = outs[i];
  }
  p.n_out = n_out;
  p.step_cond = step_cond, p.step_x = step_x, p.step_g = step_g, p.step_cx = step_cx, p.step_cv = step_cv;
  p.step_hist = step_hist, p.step_x0 = step_x0, p.step_ch = step_ch, p.step_sigma = step_sigma;

  HeadMaps maps{};
  rc = make_tmap_bf16_2d(&maps.w_hi, w_hi, 64, static_cast<uint64_t>(cols), static_cast<uint64_t>(cols), hd::kOut, hd::kKC);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&maps.w_lo, w_lo, 64, static_cast<uint64_t>(cols), static_cast<uint64_t>(cols), hd::kOut, hd::kKC);
  if (rc) return rc;
  const void* f32_rows = r_or_null ? static_cast<const void*>(r_or_null) : x;  // the fp32 operand: cached residual on a hit, else the stream
  const uint32_t tail_box = p.tail_rows ? static_cast<uint32_t>(p.tail_rows) : hd::kRows;
  rc = make_tmap_f32_2d(&maps.f32_full, f32_rows, static_cast<uint64_t>(rows), static_cast<uint64_t>(cols), hd::kRows);
  if (rc) return rc;
  rc = make_tmap_f32_2d(&maps.f32_tail, f32_rows, static_cast<uint64_t>(rows), static_cast<uint64_t>(cols), tail_box);
  if (rc) return rc;
  if (r_or_null) {
    rc = make_tmap_bf16_2d(&maps.bf16_full, x, static_cast<uint64_t>(rows), static_cast<uint64_t>(cols), static_cast<uint64_t>(cols), hd::kRows, hd::kKC);
    if (rc) return rc;
    rc = make_tmap_bf16_2d(&maps.bf16_tail, x, static_cast<uint64_t>(rows), static_cast<uint64_t>(cols), static_cast<uint64_t>(cols), tail_box, hd::kKC);
    if (rc) return rc;
  }
  const int grid = static_cast<int>((rows + p.rows_per_cta - 1) / p.rows_per_cta);
  static PerDeviceOnce once_hit, once_stream, once_hist_hit, once_hist_stream;
  if (step_hist && r_or_null) {
    rc = set_max_smem_once(head_tc_kernel<true, true>, hd::Layout<true>::kSmem, once_hist_hit, "cudaFuncSetAttribute(head smem)");
    if (rc) return rc;
    head_tc_kernel<true, true><<<grid, hd::kThreads, hd::Layout<true>::kSmem, s>>>(maps, p);
  } else if (step_hist) {
    rc = set_max_smem_once(head_tc_kernel<false, true>, hd::Layout<false>::kSmem, once_hist_stream, "cudaFuncSetAttribute(head smem)");
    if (rc) return rc;
    head_tc_kernel<false, true><<<grid, hd::kThreads, hd::Layout<false>::kSmem, s>>>(maps, p);
  } else if (r_or_null) {
    rc = set_max_smem_once(head_tc_kernel<true>, hd::Layout<true>::kSmem, once_hit, "cudaFuncSetAttribute(head smem)");
    if (rc) return rc;
    head_tc_kernel<true><<<grid, hd::kThreads, hd::Layout<true>::kSmem, s>>>(maps, p);
  } else {
    rc = set_max_smem_once(head_tc_kernel<false>, hd::Layout<false>::kSmem, once_stream, "cudaFuncSetAttribute(head smem)");
    if (rc) return rc;
    head_tc_kernel<false><<<grid, hd::kThreads, hd::Layout<false>::kSmem, s>>>(maps, p);
  }
  MC_CHECK_LAUNCH("head_tc_kernel launch");
  return MC_OK;
}

int32_t mc_head_unpatchify_ex(const void* x, int32_t x_dtype, const float* r_or_null, int64_t rows, int64_t row_offset, int32_t cols,
                              int32_t F, int32_t Hp, int32_t Wp, int32_t C_out, float eps, float* const* outs, int32_t n_out,
                              const void* prepared, int64_t prepared_bytes, int32_t flags, void* stream) {
  return head_launch(x, x_dtype, r_or_null, rows, row_offset, cols, F, Hp, Wp, C_out, eps, outs, n_out, prepared, prepared_bytes, flags, nullptr,
                     nullptr, 0.f, 0.f, 0.f, nullptr, 0.f, 0.f, nullptr, stream);
}

int32_t mc_head_unpatchify_step(const void* x, int32_t x_dtype, const float* r_or_null, int64_t rows, int64_t row_offset, int32_t cols,
                                int32_t F, int32_t Hp, int32_t Wp, int32_t C_out, float eps, float* const* outs, int32_t n_out,
                                const void* prepared, int64_t prepared_bytes, int32_t flags, const float* cond, const float* x_latent,
                                float guide_scale, float coef_x, float coef_v, void* stream) {
  MC_CHECK_ARG(cond != nullptr && x_latent != nullptr, "mc_head_unpatchify_step: null cond / latent");
  MC_CHECK_ARG((reinterpret_cast<uintptr_t>(cond) & 7u) == 0 && (reinterpret_cast<uintptr_t>(x_latent) & 7u) == 0,
               "mc_head_unpatchify_step: cond / latent must be 8-byte aligned");
  return head_launch(x, x_dtype, r_or_null, rows, row_offset, cols, F, Hp, Wp, C_out, eps, outs, n_out, prepared, prepared_bytes, flags, cond,
                     x_latent, guide_scale, coef_x, coef_v, nullptr, 0.f, 0.f, nullptr, stream);
}

int32_t mc_head_unpatchify_step_hist(const void* x, int32_t x_dtype, const float* r_or_null, int64_t rows, int64_t row_offset, int32_t cols,
                                     int32_t F, int32_t Hp, int32_t Wp, int32_t C_out, float eps, float* const* outs, int32_t n_out,
                                     const void* prepared, int64_t prepared_bytes, int32_t flags, const float* cond, const float* x_latent,
                                     float guide_scale, float coef_x, float coef_v, const float* hist, float coef_h, float sigma,
                                     float* x0_out, void* stream) {
  auto al8 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 7u) == 0; };
  MC_CHECK_ARG(cond != nullptr && x_latent != nullptr && hist != nullptr, "mc_head_unpatchify_step_hist: null cond / latent / hist");
  MC_CHECK_ARG(al8(cond) && al8(x_latent) && al8(hist) && (x0_out == nullptr || al8(x0_out)),
               "mc_head_unpatchify_step_hist: cond / latent / hist / x0_out must be 8-byte aligned");
  MC_CHECK_ARG(outs != nullptr && n_out >= 1 && n_out <= mc::hd::kMaxPeers, "mc_head_unpatchify_step_hist: outs null or n_out=%d outside [1, %d]",
               n_out, mc::hd::kMaxPeers);
  MC_CHECK_ARG(hist != x0_out, "mc_head_unpatchify_step_hist: hist aliases x0_out");
  MC_CHECK_ARG(x0_out == nullptr || (x0_out != x_latent && x0_out != cond),
               "mc_head_unpatchify_step_hist: x0_out may not alias the latent or cond (out may alias the latent)");
  for (int i = 0; i < n_out; ++i) {
    MC_CHECK_ARG(outs[i] != hist, "mc_head_unpatchify_step_hist: hist aliases out[%d]", i);
    MC_CHECK_ARG(outs[i] != cond, "mc_head_unpatchify_step_hist: cond aliases out[%d]", i);
    MC_CHECK_ARG(x0_out == nullptr || outs[i] != x0_out, "mc_head_unpatchify_step_hist: x0_out aliases out[%d]", i);
  }
  return head_launch(x, x_dtype, r_or_null, rows, row_offset, cols, F, Hp, Wp, C_out, eps, outs, n_out, prepared, prepared_bytes, flags, cond,
                     x_latent, guide_scale, coef_x, coef_v, hist, coef_h, sigma, x0_out, stream);
}

int32_t mc_head_unpatchify(const void* x, int32_t x_dtype, const float* r_or_null, int64_t rows, int64_t row_offset, int32_t cols,
                           int32_t F, int32_t Hp, int32_t Wp, int32_t C_out, const float* head_mod, const float* e, const float* Wt,
                           const float* b, float eps, float* out, void* workspace, int64_t workspace_bytes, int32_t flags, void* stream) {
  const int32_t rc = mc_head_prepare(head_mod, e, Wt, b, cols, workspace, workspace_bytes, stream);
  if (rc) return rc;
  float* outs[1] = {out};
  return mc_head_unpatchify_ex(x, x_dtype, r_or_null, rows, row_offset, cols, F, Hp, Wp, C_out, eps, outs, 1, workspace, workspace_bytes, flags,
                               stream);
}

}  // extern "C"
