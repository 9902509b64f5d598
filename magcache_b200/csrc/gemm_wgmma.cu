// bf16 GEMM on the Hopper tensor cores (wgmma): acc[m,n] = sum_k A[m,k] * B[n,k], fp32 accumulation in registers.
// Replaces the cuBLAS calls behind every nn.Linear / Conv3d of the cache-miss branch
// (`for block in self.blocks: x = block(x, **kwargs)`, MagCache4Wan2.1/magcache_generate.py:297-298; patch_embedding :237;
// text_embedding :257-262), with the reference's elementwise follow-ups fused into the epilogue (SURVEY §2.2 K8/K12/K13).
//
// Persistent kernel, one CTA per SM, clusters of 2 CTAs along M. A cluster walks 256 (M) x BN (N) tiles, BN = 256 or 128; at
// each step CTA rank r of the cluster computes rows [128 r, 128 r + 128) of the tile, 64 (K) per stage:
//   warpgroup 0  TMA producer (one warp): per stage its own A tile (128x64) and one half of the B tile (BN/2 x 64), the B half
//                multicast into both CTAs of the cluster, so each CTA reads 16 + BN/2 * 128 bytes from L2 per stage (a third
//                less per FLOP than loading the whole B tile) and still receives it all; 128-byte swizzle, 4-stage smem ring
//   warpgroups 1-2  consumers: each owns 64 rows of the CTA's tile, wgmma m64nBNk16 x4 per stage with both operands in shared
//                memory and the accumulator in registers; a stage goes back to the producers of both CTAs as soon as the wgmmas
//                reading it have retired (one group kept in flight). Epilogue: each warp's 16 accumulator rows -> its own 16x32
//                smem patch -> lane = column, so every global access is a coalesced row segment and all eight warps drain at
//                the same time, with no barrier between warps.
// Tiles are walked in waves of (number of clusters) consecutive tiles with N fastest: the CTAs of one wave share A row-panels in
// L2. The 128-wide instantiation serves grids that would leave a wave of 256-wide tiles mostly empty (pick_bn).
#include <cstdlib>

#include "common.cuh"
#include "ptx.cuh"
#include "tma_host.cuh"

namespace mc {

TmapCacheEntry* tmap_cache() {
  static TmapCacheEntry table[kTmapCacheSize] = {};
  return table;
}
std::mutex& tmap_cache_mutex() {
  static std::mutex m;
  return m;
}

constexpr int kCluster = 2;                    // CTAs per cluster, stacked along M
constexpr int kBM = 128, kBK = 64, kStages = 4;  // kBM: rows of one CTA step, 64 per consumer warpgroup
constexpr int kClusterBM = kCluster * kBM;     // rows of one cluster step (the tile the walk and pick_bn count)
constexpr int kTileABytes = kBM * kBK * 2;     // 16 KB
constexpr int kStagePad = 33;                                 // floats per staged row (conflict-free transpose)
constexpr int kEpiWarps = 8;                                   // the two consumer warpgroups
constexpr int kPatchRows = 16;                                 // a warp's rows of the accumulator fragment
constexpr int kStagingBytes = kEpiWarps * kPatchRows * kStagePad * 4;  // one 16x32 fp32 patch per consumer warp
constexpr int kGemmThreads = 128 + 32 * kEpiWarps;             // producer warpgroup + two consumer warpgroups
constexpr int kProducerRegs = 40, kConsumerRegs = 232;         // setmaxnreg: 40 * 128 + 232 * 256 <= 64K
template <int BN>
struct GemmTile {  // BN = 256 (default) or 128
  static constexpr int kTileBBytes = BN * kBK * 2;                 // 32 / 16 KB, half of it loaded by each CTA of the cluster
  static constexpr int kHalfBBytes = kTileBBytes / kCluster;
  static constexpr int kStageBytes = kTileABytes + kTileBBytes;    // 48 / 32 KB: what lands in each CTA per stage
  static constexpr int kOffStaging = kStages * kStageBytes;        // 196608 / 131072
  static constexpr int kOffBars = kOffStaging + kStagingBytes;     // + 16896
  static constexpr int kSmem = kOffBars + 128;                     // 213632 / 148096 of the 232448 an H100 block may use
};

struct GemmParams {
  int M, N, K;
  const float* bias;
  void* out;
  int64_t ldo;
  const float* gate;
  int total_tiles;  // 256-row m tiles x n tiles (cluster steps), set by launch_gemm_bn: read from the parameter bank
  const __nv_bfloat16* add;  // MC_EPI_BIAS_GATE_RESID_ADD_BF16 only: addend rows [add_row0, M), row stride ld_add
  int64_t ld_add;
  int add_row0;
  int R;  // gemm_bf16_kernel_tail only: width of the second K segment, acc += U[m, :R] . T[n, :R]
};

// One ROWS-row x 32-column patch: `stage` holds acc[r][c] at stage[r*33 + c]; lane = column. All global accesses below
// touch 128 (fp32) or 64 (bf16, two rows per instruction) contiguous bytes per row.
template <int EPI, int ROWS>
__device__ __forceinline__ void epilogue_patch(const GemmParams& p, const float* stage, int row0, int col0, int lane) {
  const int rows = min(ROWS, p.M - row0);
  if (rows <= 0) return;
  constexpr bool kAdd = EPI == MC_EPI_BIAS_GATE_RESID_ADD_BF16;
  constexpr bool kGateResidBf16 = EPI == MC_EPI_BIAS_GATE_RESID_BF16 || kAdd;  // epilogue 8 is epilogue 6, then the addend
  const int col = col0 + lane;
  const bool col_ok = col < p.N;

  if (EPI == MC_EPI_BIAS_GATE_RESID) {
    // x[m,n] = x[m,n] + float(bf16(acc + bias[n])) * gate[n]   (`x = x + y * e[2]`: y is the bf16 Linear output, fp32 stream)
    const float b = (p.bias && col_ok) ? p.bias[col] : 0.f;
    const float g = (p.gate && col_ok) ? p.gate[col] : 1.f;
    float* xcol = static_cast<float*>(p.out) + static_cast<int64_t>(row0) * p.ldo + col;
    // 16 rows at a time, 16 loads in flight: all 32 rows at once spilled next to the 256-wide tile's 128 accumulator registers
#pragma unroll
    for (int h = 0; h < ROWS; h += 16) {
      float xv[16];
#pragma unroll
      for (int r = 0; r < 16; ++r) xv[r] = (col_ok && h + r < rows) ? xcol[static_cast<int64_t>(h + r) * p.ldo] : 0.f;
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        const float y = round_bf16(stage[(h + r) * kStagePad + lane] + b);
        xv[r] = __fadd_rn(xv[r], __fmul_rn(y, g));
      }
#pragma unroll
      for (int r = 0; r < 16; ++r)
        if (col_ok && h + r < rows) xcol[static_cast<int64_t>(h + r) * p.ldo] = xv[r];
    }
    return;
  }

  if (EPI == MC_EPI_BIAS_F32) {
    const float b = (p.bias && col_ok) ? p.bias[col] : 0.f;
    float* ocol = static_cast<float*>(p.out) + static_cast<int64_t>(row0) * p.ldo + col;
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
      if (col_ok && r < rows) ocol[static_cast<int64_t>(r) * p.ldo] = stage[r * kStagePad + lane] + b;
    return;
  }

  // bf16 outputs: each instruction writes two rows x 16 column pairs (lane -> row parity = lane/16, column pair = lane%16)
  const int half = lane >> 4, cp = (lane & 15) * 2;
  const int c0 = col0 + cp;
  float b0 = 0.f, b1 = 0.f;
  if (EPI != MC_EPI_ROWBIAS_BF16 && p.bias) {
    if (c0 < p.N) b0 = p.bias[c0];
    if (c0 + 1 < p.N) b1 = p.bias[c0 + 1];
  }
  float g0 = 1.f, g1 = 1.f;
  if (kGateResidBf16 && p.gate) {
    if (c0 < p.N) g0 = p.gate[c0];
    if (c0 + 1 < p.N) g1 = p.gate[c0 + 1];
  }
  __nv_bfloat16* obase = static_cast<__nv_bfloat16*>(p.out) + static_cast<int64_t>(row0 + half) * p.ldo + c0;
  const float* sbase = stage + half * kStagePad + cp;
  const float* rbias = (EPI == MC_EPI_ROWBIAS_BF16 && p.bias) ? p.bias + row0 + half : nullptr;

  // epilogue 8: the patch lies wholly at or past add_row0 (every row adds) or wholly before it (none reads the addend)
  const bool add_rows = kAdd && row0 >= p.add_row0;
  const bool add_uniform = !kAdd || row0 + ROWS <= p.add_row0 ||
                           (add_rows && (p.ld_add & 1) == 0 && (reinterpret_cast<uintptr_t>(p.add) & 3u) == 0);
  if (rows == ROWS && col0 + 32 <= p.N && (p.ldo & 1) == 0 && add_uniform) {
    // interior patch: branch-free, ROWS / 2 independent iterations for the scheduler to interleave
    uint32_t w[ROWS / 2];
#pragma unroll
    for (int i = 0; i < ROWS / 2; ++i) {
      float v0 = sbase[2 * i * kStagePad], v1 = sbase[2 * i * kStagePad + 1];
      if (EPI == MC_EPI_ROWBIAS_BF16) {
        const float rb = rbias ? rbias[2 * i] : 0.f;  // V^T = Wv h^T + bv: bias indexed by the output ROW
        v0 += rb;
        v1 += rb;
      } else {
        v0 += b0;
        v1 += b1;
      }
      if (EPI == MC_EPI_BIAS_GELU_BF16) {  // the Linear output is bf16 before nn.GELU(tanh) sees it
        v0 = gelu_tanh(round_bf16(v0));
        v1 = gelu_tanh(round_bf16(v1));
      }
      if (EPI == MC_EPI_BIAS_GELU_ERF_BF16) {
        v0 = gelu_erf(round_bf16(v0));
        v1 = gelu_erf(round_bf16(v1));
      }
      if (EPI == MC_EPI_BIAS_SILU_BF16) {
        v0 = silu_f(round_bf16(v0));
        v1 = silu_f(round_bf16(v1));
      }
      if (kGateResidBf16) {  // x = x + g * y with every tensor bf16 (MMDiT streams): three roundings
        const uint32_t old = *reinterpret_cast<const uint32_t*>(obase + static_cast<int64_t>(2 * i) * p.ldo);
        v0 = bf16_lo(old) + round_bf16(g0 * round_bf16(v0));
        v1 = bf16_hi(old) + round_bf16(g1 * round_bf16(v1));
      }
      w[i] = pack_bf16x2(v0, v1);
    }
    if (add_rows) {  // out = bf16(x1 + add): the second rounding, on the bf16 x1 just packed (32-bit pairs, like the `old` loads)
      const __nv_bfloat16* abase = p.add + static_cast<int64_t>(row0 + half - p.add_row0) * p.ld_add + c0;
#pragma unroll
      for (int i = 0; i < ROWS / 2; ++i) {
        const uint32_t a = *reinterpret_cast<const uint32_t*>(abase + static_cast<int64_t>(2 * i) * p.ld_add);
        w[i] = pack_bf16x2(bf16_lo(w[i]) + bf16_lo(a), bf16_hi(w[i]) + bf16_hi(a));
      }
    }
#pragma unroll
    for (int i = 0; i < ROWS / 2; ++i) *reinterpret_cast<uint32_t*>(obase + static_cast<int64_t>(2 * i) * p.ldo) = w[i];
    return;
  }

  const bool pair_ok = (c0 + 1 < p.N) && ((p.ldo & 1) == 0);
  for (int i = 0; i < ROWS / 2; ++i) {
    const int r = 2 * i + half;
    if (r >= rows) continue;
    float v0 = sbase[2 * i * kStagePad], v1 = sbase[2 * i * kStagePad + 1];
    if (EPI == MC_EPI_ROWBIAS_BF16) {
      const float rb = rbias ? rbias[2 * i] : 0.f;
      v0 += rb;
      v1 += rb;
    } else {
      v0 += b0;
      v1 += b1;
    }
    if (EPI == MC_EPI_BIAS_GELU_BF16) {
      v0 = gelu_tanh(round_bf16(v0));
      v1 = gelu_tanh(round_bf16(v1));
    }
    if (EPI == MC_EPI_BIAS_GELU_ERF_BF16) {
      v0 = gelu_erf(round_bf16(v0));
      v1 = gelu_erf(round_bf16(v1));
    }
    if (EPI == MC_EPI_BIAS_SILU_BF16) {
      v0 = silu_f(round_bf16(v0));
      v1 = silu_f(round_bf16(v1));
    }
    __nv_bfloat16* o = obase + static_cast<int64_t>(2 * i) * p.ldo;
    if (kGateResidBf16) {
      if (c0 < p.N) v0 = __bfloat162float(o[0]) + round_bf16(g0 * round_bf16(v0));
      if (c0 + 1 < p.N) v1 = __bfloat162float(o[1]) + round_bf16(g1 * round_bf16(v1));
    }
    if (kAdd && row0 + r >= p.add_row0) {  // scalar loads: ragged rows / columns, odd ld_add, 2-byte-aligned addend
      const __nv_bfloat16* a = p.add + static_cast<int64_t>(row0 + r - p.add_row0) * p.ld_add + c0;
      if (c0 < p.N) v0 = round_bf16(v0) + __bfloat162float(a[0]);
      if (c0 + 1 < p.N) v1 = round_bf16(v1) + __bfloat162float(a[1]);
    }
    if (pair_ok) {
      *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(v0, v1);
    } else {
      if (c0 < p.N) o[0] = __float2bfloat16_rn(v0);
      if (c0 + 1 < p.N) o[1] = __float2bfloat16_rn(v1);
    }
  }
}

// The kernel body. kTail: after the ceil(K / 64) k-blocks of (A, B) the same main loop runs ceil(R / 64) more from (U, T), so
// every epilogue sees acc = A B^T + U T^T (a LoRA update as extra K blocks). Without it tmap_u / tmap_t are never read.
template <int EPI, int kBN, bool kTail>
__device__ __forceinline__ void gemm_body(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, const CUtensorMap& tmap_u,
                                          const CUtensorMap& tmap_t, const GemmParams& p) {
  using T = GemmTile<kBN>;
  constexpr int kStageBytes = T::kStageBytes, kOffStaging = T::kOffStaging, kOffBars = T::kOffBars;
  extern __shared__ __align__(1024) uint8_t smem[];
  float* staging = reinterpret_cast<float*>(smem + kOffStaging);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kOffBars);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = (p.N + kBN - 1) / kBN;
  const int num_kb = (p.K + kBK - 1) / kBK;
  // k-blocks per tile: TMA zero-fills the ragged ends of both segments, so every stage still carries its full byte count
  const int total_kb = kTail ? num_kb + (p.R + kBK - 1) / kBK : num_kb;
  // Both CTAs of a cluster walk the same cluster tiles in lock step (the launch makes the grid at most one cluster per tile, so
  // every cluster has at least one step); rank r takes rows [64 r, 64 r + 64) of each, computing on TMA's zero fill where
  // those rows lie past M (the epilogue then writes nothing).
  const uint32_t rank = ptx::cluster_ctarank();
  const int cluster = static_cast<int>(ptx::cluster_id_x()), n_clusters = static_cast<int>(ptx::num_clusters_x());
  const int steps = (p.total_tiles - cluster + n_clusters - 1) / n_clusters;

  if (threadIdx.x == 0) {
    if ((ptx::smem_u32(smem) & 1023u) != 0) {
      MC_DIAG("gemm_bf16_kernel: dynamic smem base not 1024-aligned\n");
      __trap();
    }
    ptx::prefetch_tmap(&tmap_a);
    ptx::prefetch_tmap(&tmap_b);
    if constexpr (kTail) {
      ptx::prefetch_tmap(&tmap_u);
      ptx::prefetch_tmap(&tmap_t);
    }
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], kCluster * kEpiWarps);  // one arrival per consumer warp, in each CTA
    }
    ptx::fence_mbar_init();
  }
  // the peer multicasts into this CTA's ring and arrives on its empty barriers: both CTAs' barriers must be initialised first
  ptx::cluster_arrive();
  ptx::cluster_wait();

  if (warp < 4) {
    ptx::setmaxnreg_dec<kProducerRegs>();
    if (warp == 0) {
      // TMA producer: the whole warp walks the loop in uniform control flow, one elected lane issues the copies (ptx::elect_one)
      uint32_t it = 0;  // running k-block counter across steps -> smem stage / phase (the same sequence in both CTAs)
      for (int i = 0; i < steps; ++i) {
        const int tile = cluster + i * n_clusters;
        const int m0 = (tile / n_tiles) * kClusterBM + static_cast<int>(rank) * kBM, n0 = (tile % n_tiles) * kBN;
        const int nb = n0 + static_cast<int>(rank) * (kBN / kCluster);  // this CTA's half of the B tile
        for (int kb = 0; kb < total_kb; ++kb, ++it) {
          const int s = it % kStages;
          const uint32_t ph = (it / kStages) & 1;
          ptx::mbar_wait(&empty_bar[s], ph ^ 1);  // released by the consumers of both CTAs: the multicast writes into both
          if (ptx::elect_one()) {
            uint8_t* sa = smem + s * kStageBytes;
            const bool tail = kTail && kb >= num_kb;
            const CUtensorMap* ma = tail ? &tmap_u : &tmap_a;
            const CUtensorMap* mb = tail ? &tmap_t : &tmap_b;
            const int k0 = (tail ? kb - num_kb : kb) * kBK;
            ptx::mbar_expect_tx(&full_bar[s], kStageBytes);  // own A + both B halves
            ptx::tma_load_2d(sa, ma, &full_bar[s], k0, m0);
            ptx::tma_load_2d_multicast(sa + kTileABytes + rank * T::kHalfBBytes, mb, &full_bar[s], k0, nb,
                                       static_cast<uint16_t>((1u << kCluster) - 1));
          }
          __syncwarp();
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1;  // consumer warpgroup: rows [64 wg, 64 wg + 64) of the CTA's tile
    const int wq = warp & 3;         // warp inside the warpgroup
    float acc[kBN / 2];
    // The mbarrier waits record a timeout instead of trapping (ptx::mbar_wait_or_flag: a trap on a wait inside a loop that
    // keeps wgmmas in flight makes ptxas spill and serialise them); the trap comes after the last wgmma_wait.
    bool timed_out = false;
    for (int i = 0; i < steps; ++i) {
      const int tile = cluster + i * n_clusters;
      const int m0 = (tile / n_tiles) * kClusterBM + static_cast<int>(rank) * kBM, n0 = (tile % n_tiles) * kBN;
      uint32_t it = static_cast<uint32_t>(i) * total_kb;
      int prev_s = -1;
      for (int kb = 0; kb < total_kb; ++kb, ++it) {
        const int s = it % kStages;
        const uint32_t ph = (it / kStages) & 1;
        ptx::mbar_wait_or_flag(&full_bar[s], ph, timed_out);
        const uint32_t sa = ptx::smem_u32(smem + s * kStageBytes);
        const uint64_t da = ptx::gmma_desc_sw128_kmajor(sa + wg * (64 * 128));  // this warpgroup's 64 rows: 8 row groups of 1024 B
        const uint64_t db = ptx::gmma_desc_sw128_kmajor(sa + kTileABytes);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k) {
          if constexpr (kBN == 256) {
            ptx::wgmma_m64n256k16_ss(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
          } else {
            ptx::wgmma_m64n128k16_ss(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
          }
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();  // the previous stage's wgmmas have retired: hand that stage back to both producers
        ptx::fence_regs(acc);
        if (prev_s >= 0 && lane == 0)
          for (uint32_t c = 0; c < kCluster; ++c) ptx::mbar_arrive_cluster(&empty_bar[prev_s], c);
        prev_s = s;
      }
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc);
      if (lane == 0)
        for (uint32_t c = 0; c < kCluster; ++c) ptx::mbar_arrive_cluster(&empty_bar[prev_s], c);

      // epilogue, 32 columns at a time. Each warp stages its own 16 rows of the fragment in its own 16x32 patch and drains it,
      // so the four warps of the warpgroup write (and, for the residual stream, load) global memory at the same time, with no
      // barrier between warps.
      float* patch = staging + (4 * wg + wq) * kPatchRows * kStagePad;
      const int row0 = m0 + wg * 64 + wq * kPatchRows;
      const int r_lo = lane >> 2;  // this lane's first row inside the patch (the second is r_lo + 8)
#pragma unroll  // static accumulator indices: the accumulator must stay in registers
      for (int c = 0; c < kBN / 32; ++c) {
        __syncwarp();  // the previous patch has been read
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int i = 4 * c + q;
          const int col = 8 * q + 2 * (lane & 3);
          patch[r_lo * kStagePad + col] = acc[4 * i + 0];
          patch[r_lo * kStagePad + col + 1] = acc[4 * i + 1];
          patch[(r_lo + 8) * kStagePad + col] = acc[4 * i + 2];
          patch[(r_lo + 8) * kStagePad + col + 1] = acc[4 * i + 3];
        }
        __syncwarp();
        epilogue_patch<EPI, kPatchRows>(p, patch, row0, n0 + c * 32, lane);
      }
    }
    if (timed_out) __trap();
  }
  // no CTA may exit while its peer can still multicast into its ring or arrive on its empty barriers
  ptx::cluster_arrive();
  ptx::cluster_wait();
}

template <int EPI, int kBN>
__global__ void __cluster_dims__(kCluster, 1, 1) __launch_bounds__(kGemmThreads, 1)
    gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const GemmParams p) {
  gemm_body<EPI, kBN, false>(tmap_a, tmap_b, tmap_a, tmap_b, p);
}

// acc = A B^T + U T^T: tmap_u / tmap_t have the boxes of tmap_a / tmap_b (128 x 64; BN/2 x 64, multicast over the cluster)
template <int EPI, int kBN>
__global__ void __cluster_dims__(kCluster, 1, 1) __launch_bounds__(kGemmThreads, 1)
    gemm_bf16_kernel_tail(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const GemmParams p,
                          const __grid_constant__ CUtensorMap tmap_u, const __grid_constant__ CUtensorMap tmap_t) {
  gemm_body<EPI, kBN, true>(tmap_a, tmap_b, tmap_u, tmap_t, p);
}

// Clusters of this instantiation that fit on the device at once (1 CTA per SM at this shared-memory size), cached per device.
// Clusters live inside a GPC, so this can be less than SMs / 2; a grid of SMs / 2 clusters would then run a second, nearly
// empty wave.
template <int EPI, int BN, bool kTail>
static int32_t max_active_clusters(int* out) {
  static int cached[kMaxDevices] = {};
  const int d = current_device();
  if (cached[d] > 0) {
    *out = cached[d];
    return MC_OK;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(kCluster * num_sms(), 1, 1);
  cfg.blockDim = dim3(kGemmThreads, 1, 1);
  cfg.dynamicSmemBytes = GemmTile<BN>::kSmem;
  int n = 0;
  cudaError_t e;
  if constexpr (kTail) {
    e = cudaOccupancyMaxActiveClusters(&n, gemm_bf16_kernel_tail<EPI, BN>, &cfg);
  } else {
    e = cudaOccupancyMaxActiveClusters(&n, gemm_bf16_kernel<EPI, BN>, &cfg);
  }
  if (e != cudaSuccess) return cuda_fail(e, "cudaOccupancyMaxActiveClusters(gemm)");
  if (n < 1) {
    set_error("gemm_bf16_kernel: no cluster of %d CTAs with %d B of shared memory fits on this device", kCluster, GemmTile<BN>::kSmem);
    return MC_ERR_CUDA;
  }
  cached[d] = n;
  *out = n;
  return MC_OK;
}

// kTail: gemm_bf16_kernel_tail with tu / tt (non-null), otherwise gemm_bf16_kernel
template <int EPI, int BN, bool kTail = false>
static int32_t launch_gemm_bn(const CUtensorMap& ta, const CUtensorMap& tb, GemmParams p, cudaStream_t s, const CUtensorMap* tu = nullptr,
                              const CUtensorMap* tt = nullptr) {
  static PerDeviceOnce once;
  int32_t rc;
  if constexpr (kTail) {
    rc = set_max_smem_once(gemm_bf16_kernel_tail<EPI, BN>, GemmTile<BN>::kSmem, once, "cudaFuncSetAttribute(gemm smem)");
  } else {
    rc = set_max_smem_once(gemm_bf16_kernel<EPI, BN>, GemmTile<BN>::kSmem, once, "cudaFuncSetAttribute(gemm smem)");
  }
  if (rc) return rc;
  int clusters = 0;
  rc = max_active_clusters<EPI, BN, kTail>(&clusters);
  if (rc) return rc;
  const int m_tiles = (p.M + kClusterBM - 1) / kClusterBM, n_tiles = (p.N + BN - 1) / BN;
  const int total = m_tiles * n_tiles;
  p.total_tiles = total;
  const int grid = kCluster * (total < clusters ? total : clusters);
  if constexpr (kTail) {
    gemm_bf16_kernel_tail<EPI, BN><<<grid, kGemmThreads, GemmTile<BN>::kSmem, s>>>(ta, tb, p, *tu, *tt);
    MC_CHECK_LAUNCH("gemm_bf16_kernel_tail launch");
  } else {
    gemm_bf16_kernel<EPI, BN><<<grid, kGemmThreads, GemmTile<BN>::kSmem, s>>>(ta, tb, p);
    MC_CHECK_LAUNCH("gemm_bf16_kernel launch");
  }
  return MC_OK;
}

// N-tile width for an M x N output: waves of num_sms() tiles, a wave of 128-wide tiles costed at 0.62 of a wave of 256-wide ones
// (the same A panel moves for half the math, so a narrow tile is not half the cost of a wide one); the narrow width is taken only
// where it makes the estimate at least 8 % cheaper. MC_GEMM_BN = 128 | 256 forces one (tests, A/B timing).
static int pick_bn(int M, int N) {
  const char* e = getenv("MC_GEMM_BN");
  if (e && *e) {
    const int v = atoi(e);
    if (v == 128 || v == 256) return v;
  }
  const int64_t sms = num_sms(), m_tiles = (M + 127) / 128;  // waves of SMs 128-row CTA steps
  const int64_t t256 = m_tiles * ((N + 255) / 256), t128 = m_tiles * ((N + 127) / 128);
  const int64_t cost256 = ((t256 + sms - 1) / sms) * 100, cost128 = ((t128 + sms - 1) / sms) * 62;
  return cost128 * 100 <= cost256 * 92 ? 128 : 256;
}

// The argument checks and tensor maps every GEMM entry point shares; `fn` names the entry point in the error text.
static int32_t gemm_prepare(const char* fn, const void* A, int64_t lda, const void* B, int64_t ldb, int32_t M, int32_t N, int32_t K,
                            const void* out, int64_t ldo, CUtensorMap* ta, CUtensorMap* tb, int* bn) {
  MC_CHECK_ARG(A && B && out, "%s: null pointer", fn);
  MC_CHECK_ARG(M >= 1 && N >= 1 && K >= 8, "%s: M=%d N=%d K=%d", fn, M, N, K);
  MC_CHECK_ARG(K % 8 == 0 && lda % 8 == 0 && ldb % 8 == 0 && lda >= K && ldb >= K, "%s: K/lda/ldb must be multiples of 8 (16-byte TMA pitch)", fn);
  MC_CHECK_ARG(aligned16(A) && aligned16(B) && aligned16(out), "%s: A/B/out must be 16-byte aligned", fn);
  MC_CHECK_ARG(ldo >= N, "%s: ldo=%lld < N=%d", fn, static_cast<long long>(ldo), N);
  int32_t rc = make_tmap_bf16_2d(ta, A, static_cast<uint64_t>(M), static_cast<uint64_t>(K), static_cast<uint64_t>(lda), kBM, kBK);
  if (rc) return rc;
  *bn = pick_bn(M, N);
  // each CTA of a cluster loads (and multicasts) one half of the B tile: the box is bn / 2 rows
  return make_tmap_bf16_2d(tb, B, static_cast<uint64_t>(N), static_cast<uint64_t>(K), static_cast<uint64_t>(ldb), *bn / kCluster, kBK);
}

}  // namespace mc

extern "C" int32_t mc_gemm_bf16(const void* A, int64_t lda, const void* B, int64_t ldb, int32_t M, int32_t N, int32_t K,
                                const float* bias, int32_t epilogue, void* out, int64_t ldo, const float* gate, void* stream) {
  CUtensorMap ta, tb;
  int bn = 0;
  const int32_t rc = mc::gemm_prepare("mc_gemm_bf16", A, lda, B, ldb, M, N, K, out, ldo, &ta, &tb, &bn);
  if (rc) return rc;
  mc::GemmParams p{M, N, K, bias, out, ldo, gate, 0, nullptr, 0, 0, 0};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
#define MC_GEMM_CASE(E) \
  case E: return bn == 128 ? mc::launch_gemm_bn<E, 128>(ta, tb, p, s) : mc::launch_gemm_bn<E, 256>(ta, tb, p, s)
  switch (epilogue) {
    MC_GEMM_CASE(MC_EPI_BIAS_BF16);
    MC_GEMM_CASE(MC_EPI_BIAS_GELU_BF16);
    MC_GEMM_CASE(MC_EPI_BIAS_GATE_RESID);
    MC_GEMM_CASE(MC_EPI_ROWBIAS_BF16);
    MC_GEMM_CASE(MC_EPI_BIAS_F32);
    MC_GEMM_CASE(MC_EPI_BIAS_GELU_ERF_BF16);
    MC_GEMM_CASE(MC_EPI_BIAS_GATE_RESID_BF16);
    MC_GEMM_CASE(MC_EPI_BIAS_SILU_BF16);
#undef MC_GEMM_CASE
    default:
      mc::set_error("mc_gemm_bf16: unknown epilogue %d", epilogue);
      return MC_ERR_INVALID;
  }
}

extern "C" int32_t mc_gemm_bf16_add(const void* A, int64_t lda, const void* B, int64_t ldb, int32_t M, int32_t N, int32_t K,
                                    const float* bias, void* out, int64_t ldo, const float* gate, const void* add, int64_t ld_add,
                                    int32_t add_row0, void* stream) {
  CUtensorMap ta, tb;
  int bn = 0;
  const int32_t rc = mc::gemm_prepare("mc_gemm_bf16_add", A, lda, B, ldb, M, N, K, out, ldo, &ta, &tb, &bn);
  if (rc) return rc;
  MC_CHECK_ARG(add, "mc_gemm_bf16_add: null addend");
  MC_CHECK_ARG(ld_add >= N, "mc_gemm_bf16_add: ld_add=%lld < N=%d", static_cast<long long>(ld_add), N);
  MC_CHECK_ARG(add_row0 >= 0 && add_row0 < M, "mc_gemm_bf16_add: add_row0=%d outside [0, M=%d)", add_row0, M);
  const mc::GemmParams p{M, N, K, bias, out, ldo, gate, 0, static_cast<const __nv_bfloat16*>(add), ld_add, add_row0, 0};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return bn == 128 ? mc::launch_gemm_bn<MC_EPI_BIAS_GATE_RESID_ADD_BF16, 128>(ta, tb, p, s)
                   : mc::launch_gemm_bn<MC_EPI_BIAS_GATE_RESID_ADD_BF16, 256>(ta, tb, p, s);
}

extern "C" int32_t mc_gemm_bf16_lora(const void* A, int64_t lda, const void* B, int64_t ldb, int32_t M, int32_t N, int32_t K,
                                     const float* bias, int32_t epilogue, void* out, int64_t ldo, const float* gate, const void* add,
                                     int64_t ld_add, int32_t add_row0, const void* U, int64_t ldu, const void* T, int64_t ldt, int32_t R,
                                     void* stream) {
  CUtensorMap ta, tb, tu, tt;
  int bn = 0;
  int32_t rc = mc::gemm_prepare("mc_gemm_bf16_lora", A, lda, B, ldb, M, N, K, out, ldo, &ta, &tb, &bn);
  if (rc) return rc;
  MC_CHECK_ARG(U && T, "mc_gemm_bf16_lora: null U / T");
  MC_CHECK_ARG(R >= 8 && R % 8 == 0, "mc_gemm_bf16_lora: R=%d must be a positive multiple of 8", R);
  MC_CHECK_ARG(ldu % 8 == 0 && ldt % 8 == 0 && ldu >= R && ldt >= R, "mc_gemm_bf16_lora: ldu=%lld / ldt=%lld must be multiples of 8 and >= R=%d",
               static_cast<long long>(ldu), static_cast<long long>(ldt), R);
  MC_CHECK_ARG(mc::aligned16(U) && mc::aligned16(T), "mc_gemm_bf16_lora: U/T must be 16-byte aligned");
  if (epilogue == MC_EPI_BIAS_GATE_RESID_ADD_BF16) {
    MC_CHECK_ARG(add, "mc_gemm_bf16_lora: null addend");
    MC_CHECK_ARG(ld_add >= N, "mc_gemm_bf16_lora: ld_add=%lld < N=%d", static_cast<long long>(ld_add), N);
    MC_CHECK_ARG(add_row0 >= 0 && add_row0 < M, "mc_gemm_bf16_lora: add_row0=%d outside [0, M=%d)", add_row0, M);
  } else {
    MC_CHECK_ARG(!add, "mc_gemm_bf16_lora: an addend needs epilogue %d", MC_EPI_BIAS_GATE_RESID_ADD_BF16);
  }
  rc = mc::make_tmap_bf16_2d(&tu, U, static_cast<uint64_t>(M), static_cast<uint64_t>(R), static_cast<uint64_t>(ldu), mc::kBM, mc::kBK);
  if (rc) return rc;
  rc = mc::make_tmap_bf16_2d(&tt, T, static_cast<uint64_t>(N), static_cast<uint64_t>(R), static_cast<uint64_t>(ldt), bn / mc::kCluster, mc::kBK);
  if (rc) return rc;
  const mc::GemmParams p{M, N, K, bias, out, ldo, gate, 0, static_cast<const __nv_bfloat16*>(add), ld_add, add_row0, R};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
#define MC_GEMM_TAIL_CASE(E)                                                            \
  case E:                                                                               \
    return bn == 128 ? mc::launch_gemm_bn<E, 128, true>(ta, tb, p, s, &tu, &tt)        \
                     : mc::launch_gemm_bn<E, 256, true>(ta, tb, p, s, &tu, &tt)
  switch (epilogue) {
    MC_GEMM_TAIL_CASE(MC_EPI_BIAS_BF16);
    MC_GEMM_TAIL_CASE(MC_EPI_BIAS_GELU_BF16);
    MC_GEMM_TAIL_CASE(MC_EPI_BIAS_GATE_RESID_BF16);
    MC_GEMM_TAIL_CASE(MC_EPI_BIAS_GATE_RESID_ADD_BF16);
#undef MC_GEMM_TAIL_CASE
    default:
      mc::set_error("mc_gemm_bf16_lora: epilogue %d has no LoRA tail (0, 1, 6 and 8 do)", epilogue);
      return MC_ERR_INVALID;
  }
}
