// Non-causal flash-attention forward on the Hopper tensor cores (wgmma), head_dim 128 — the self-/cross-attention of the Wan
// DiT block (SURVEY §2.2 K10/K11; reference call chain MagCache4Wan2.1/magcache_generate.py:297-298 -> WanSelfAttention.forward ->
// flash_attention / SDPA, upstream wan/modules/{model,attention}.py) and the joint attention of the MMDiT blocks
// (MagCache4FLUX/magcache_flux.py:343-425, MagCache4HunyuanVideo/magcache_sample_video.py:108-140).
//
// q [Lq, H*128], k [Lk, H*128], v [Lk, H*128] are all ROW-MAJOR bf16 views (row pitch allowed: they are column slices of the
// fused q|k|v projection buffer). K is the B operand of S = Q K^T in K-major form; V is the B operand of O += P V in MN-major
// form (d contiguous, the transposed-B form of wgmma) — the same [rows][64 bf16] 128-byte-swizzled TMA boxes for both, no
// transposed copy of V anywhere.
//
// One kernel, instantiated for three KV tile widths: 176 keys per tile for long key sequences (Lk >= kLongMinLk), 64 for short
// ones (text / image cross-attention, refiner), and 128 (MC_ATTN_KERNEL=2, the FMA-pipe exponential variants). The wider the
// tile, the more keys share each tile's fixed cost (row max, O rescale, fences, barrier turns, mbarrier waits); 176 is the
// widest whose two-stage K/V ring (2 x 2 x 44 KB + the 32 KB Q tile) fits in shared memory and whose S, P and O fragments fit
// the consumers' 240 registers without spilling. One CTA = one 128-row query tile of one head:
//   warpgroup 0     TMA producer (one warp): the Q tile once, then K and V tiles through a two-stage ring
//   warpgroups 1-2  consumers, 64 query rows each: S = Q K^T (wgmma, both operands in shared memory) into registers, online
//                   softmax in the exp2 domain on the accumulator fragment (a row spans the 4 lanes of a quad), P rounded to bf16
//                   and fed back as the REGISTER A operand of O += P V, O in registers.
//                   The two warpgroups take turns issuing their GEMMs (ping-pong on named barriers), so one's softmax runs
//                   while the tensor cores work on the other's GEMM.
// The units of a partially filled last wave are split over the KV range and merged by attn_combine_kernel.
// The 128-key variant can evaluate a fixed fraction of the softmax exponentials on the FMA pipe (ptx::ex2_emul) instead of the
// MUFU unit; MC_ATTN_EMU selects the fraction per call. The 64- and 176-key variants use the MUFU only.
#include <cstdlib>

#include "common.cuh"
#include "ptx.cuh"
#include "tma_host.cuh"

#ifndef MC_ATTN_EMU_DEFAULT
#define MC_ATTN_EMU_DEFAULT 0  // eighths of the softmax exponentials on the FMA pipe (128-key tiles); MC_ATTN_EMU overrides per call
#endif

namespace mc {

constexpr int kHD = 128;
constexpr int kLongMinLk = 1024;

struct AttnParams {
  int Lq, Lk, heads;
  // Work decomposition (plan_attention): a unit = one query block of one head. CTAs [0, full_units) each own a whole unit;
  // the remaining `tail_units` units (the part of the grid that would not fill a last wave) are split `tail_split` ways over
  // the KV range, CTA full_units + u * tail_split + s owning split s of tail unit u and writing a partial result.
  int q_blocks, full_units, tail_units, tail_split;
  float* part_o;   // [tail_split][tail_units][rows per CTA][128] fp32, each split's output normalised by its own row sum
  float2* part_ml; // [tail_split][tail_units][rows per CTA]      (row max in the scaled log2 domain, row sum)
  float scale_log2;  // softmax scale * log2(e)
  __nv_bfloat16* out;
  int64_t ldo;
  // KV tile order. Token-sharded runs consume the LOCAL keys first and the peers' keys in arrival order: tile j of this CTA is
  // global tile (tile_rot + j) mod total. seg_flags != nullptr: before a tile that touches rows of source segment s
  // (rows [s*seg_rows, (s+1)*seg_rows)) is loaded, seg_flags[s] must have reached seg_epoch (written by the peer copy).
  int tile_rot;
  const uint32_t* seg_flags;
  const uint32_t* seg_epoch;  // device memory: the epoch the flags must have reached (read at run time, so graph replays work)
  int seg_rows;
};

struct WorkItem {
  int q_block, head;
  int split, nsplit;  // nsplit > 1: this CTA covers KV tiles [split * per, ...) of its unit and writes a partial
  int tail_unit;
};

__device__ __forceinline__ WorkItem work_item(const AttnParams& p) {
  WorkItem w;
  int c = blockIdx.x, unit;
  if (c < p.full_units) {
    unit = c, w.split = 0, w.nsplit = 1, w.tail_unit = 0;
  } else {
    c -= p.full_units;
    w.tail_unit = c / p.tail_split;
    w.split = c - w.tail_unit * p.tail_split;
    w.nsplit = p.tail_split;
    unit = p.full_units + w.tail_unit;
  }
  // query blocks of one head are adjacent in launch order: the CTAs resident together stream the same K/V through L2
  w.head = unit / p.q_blocks;
  w.q_block = unit - w.head * p.q_blocks;
  return w;
}

// 2^x through the MUFU, or through the FMA-pipe polynomial when bit (group & 7) of EMU_MASK is set
template <uint32_t EMU_MASK>
__device__ __forceinline__ float exp2_sel(float x, int group) {
  return ((EMU_MASK >> (group & 7)) & 1u) ? ptx::ex2_emul(x) : ptx::ex2_approx(x);
}

// token-sharded runs: block until every source segment a KV tile touches has landed (flag written by the peer's copy stream
// AFTER the segment's data, same stream). Called by the single TMA-issuing thread; the acquire load orders the flag before the
// tile loads in the generic proxy, the proxy fence carries that order over to the async proxy the TMA reads through.
__device__ __forceinline__ void wait_segments(const AttnParams& p, int row0, int rows) {
  if (p.seg_flags == nullptr) return;
  const uint32_t want = *reinterpret_cast<const volatile uint32_t*>(p.seg_epoch);
  const int last = min(row0 + rows, p.Lk) - 1;
  const int s0 = row0 / p.seg_rows, s1 = last / p.seg_rows;
  for (int s = s0; s <= s1; ++s) {
    const uint32_t* f = p.seg_flags + s;
    const long long t0 = clock64();
    for (;;) {
      uint32_t v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
      if (static_cast<int32_t>(v - want) >= 0) break;
      __nanosleep(100);
      if (clock64() - t0 > MC_MBAR_TIMEOUT_CYCLES) {
        MC_DIAG("attention: key segment %d never arrived (flag %u, epoch %u)\n", s, v, want);
        __trap();
      }
    }
  }
  asm volatile("fence.proxy.async;" ::: "memory");
}

namespace ak {
constexpr int kBQ = 128;                     // query rows per CTA (64 per consumer warpgroup)
constexpr int kQBytes = kBQ * kHD * 2;       // 32 KB (two 64-column boxes)
constexpr int kThreads = 384;                // producer warpgroup + two consumer warpgroups
constexpr int kProducerRegs = 24, kConsumerRegs = 240;  // setmaxnreg: 24 * 128 + 240 * 256 <= 64K
template <int BKV>
struct Layout {
  static constexpr int kKBytes = BKV * kHD * 2;  // two boxes [BKV kv x 64 hd]
  static constexpr int kVBytes = BKV * kHD * 2;  // two boxes [BKV kv x 64 d]
  static constexpr int kOffK = kQBytes;
  static constexpr int kOffV = kOffK + 2 * kKBytes;
  static constexpr int kOffBar = kOffV + 2 * kVBytes;  // 208 KB (BKV 176) / 160 KB (BKV 128) / 96 KB (BKV 64)
  static_assert(kKBytes % 2048 == 0, "every K / V box must start on a 1024-byte swizzle atom");
  static_assert(kOffBar + 128 <= 227 * 1024, "shared memory per CTA");
  static constexpr int kSmem = kOffBar + 128;
};
}  // namespace ak

template <int BKV, uint32_t EMU_MASK>
__global__ void __launch_bounds__(ak::kThreads, 1)
    attn_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const AttnParams p) {
  using namespace ak;
  using L = Layout<BKV>;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBar);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;   // [2]
  uint64_t* k_empty = bars + 3;  // [2] one arrival per consumer warp
  uint64_t* v_full = bars + 5;   // [2]
  uint64_t* v_empty = bars + 7;  // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const WorkItem wi = work_item(p);
  const int q0 = wi.q_block * kBQ;
  const int head = wi.head;
  const int total_tiles = (p.Lk + BKV - 1) / BKV;
  const int per_split = (total_tiles + wi.nsplit - 1) / wi.nsplit;
  const int t0 = wi.split * per_split;                   // first KV tile (in rotated order) of this CTA
  const int n_tiles = min(per_split, total_tiles - t0);  // >= 1, guaranteed by the host
  auto tile_of = [&](int j) {  // global KV tile index of this CTA's j-th tile
    int t = p.tile_rot + t0 + j;
    return t >= total_tiles ? t - total_tiles : t;
  };

  if (threadIdx.x == 0) {
    if ((ptx::smem_u32(smem) & 1023u) != 0) {
      MC_DIAG("attn_kernel: dynamic smem base not 1024-aligned\n");
      __trap();
    }
    ptx::prefetch_tmap(&tmap_q);
    ptx::prefetch_tmap(&tmap_k);
    ptx::prefetch_tmap(&tmap_v);
    ptx::mbar_init(q_full, 1);
    for (int s = 0; s < 2; ++s) {
      ptx::mbar_init(&k_full[s], 1);
      ptx::mbar_init(&k_empty[s], 8);
      ptx::mbar_init(&v_full[s], 1);
      ptx::mbar_init(&v_empty[s], 8);
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------ TMA producer ------------------------------------------------
    ptx::setmaxnreg_dec<kProducerRegs>();
    if (warp == 0) {
      if (ptx::elect_one()) {
        ptx::mbar_expect_tx(q_full, kQBytes);
        ptx::tma_load_2d(smem, &tmap_q, q_full, head * kHD, q0);
        ptx::tma_load_2d(smem + kQBytes / 2, &tmap_q, q_full, head * kHD + 64, q0);
      }
      __syncwarp();
      for (int j = 0; j < n_tiles; ++j) {
        const int s = j & 1;
        const uint32_t ph = (j >> 1) & 1;
        const int kv0 = tile_of(j) * BKV;
        if (p.seg_flags != nullptr) {
          if (lane == 0) wait_segments(p, kv0, BKV);
          __syncwarp();
        }
        ptx::mbar_wait(&k_empty[s], ph ^ 1);
        if (ptx::elect_one()) {
          ptx::mbar_expect_tx(&k_full[s], L::kKBytes);
          ptx::tma_load_2d(smem + L::kOffK + s * L::kKBytes, &tmap_k, &k_full[s], head * kHD, kv0);
          ptx::tma_load_2d(smem + L::kOffK + s * L::kKBytes + L::kKBytes / 2, &tmap_k, &k_full[s], head * kHD + 64, kv0);
        }
        __syncwarp();
        ptx::mbar_wait(&v_empty[s], ph ^ 1);
        if (ptx::elect_one()) {
          ptx::mbar_expect_tx(&v_full[s], L::kVBytes);
          ptx::tma_load_2d(smem + L::kOffV + s * L::kVBytes, &tmap_v, &v_full[s], head * kHD, kv0);
          ptx::tma_load_2d(smem + L::kOffV + s * L::kVBytes + L::kVBytes / 2, &tmap_v, &v_full[s], head * kHD + 64, kv0);
        }
        __syncwarp();
      }
    }
  } else {
    // ------------------------------------------------ consumer warpgroups -----------------------------------------
    ptx::setmaxnreg_inc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1;                       // query rows [64 wg, 64 wg + 64) of the tile
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's first row in the tile; the second is r + 8
    const int cq = 2 * (lane & 3);                        // this thread's first column inside each group of 8
    const uint32_t q_base = ptx::smem_u32(smem) + wg * (64 * 128);  // 64 rows = 8 row groups of 1024 B inside each box
    const uint32_t k_base = ptx::smem_u32(smem + L::kOffK), v_base = ptx::smem_u32(smem + L::kOffV);
    // the globally last KV tile is the only one that can hold padding columns (keys >= Lk): its position in this CTA's order
    int j_ragged = -1;
    if (p.Lk % BKV != 0) {
      int jr = total_tiles - 1 - p.tile_rot - t0;
      if (jr < 0) jr += total_tiles;
      if (jr < n_tiles) j_ragged = jr;
    }
    float o[kHD / 2];
#pragma unroll
    for (int i = 0; i < kHD / 2; ++i) o[i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows r and r + 8 (l: this thread's columns only)
    // The consumer's mbarrier waits record a timeout instead of trapping (ptx::mbar_wait_or_flag: a trap on them makes
    // ptxas spill P and serialise the wgmmas of the pipelined loop below); the trap comes after the last wgmma_wait.
    bool timed_out = false;
    ptx::mbar_wait_or_flag(q_full, 0, timed_out);

    // Each warpgroup runs the flash-attention recurrence per KV tile j: S(j) = Q K(j)^T, online softmax, O = f(j) O + P(j) V(j),
    // software-pipelined by one tile: S(j) and PV(j-1) are issued back to back, the softmax of tile j runs while PV(j-1) is on
    // the tensor cores, then O is rescaled by f(j) and P(j) packed for the next turn. Every row still sees rescale by f(j),
    // then + P(j) V(j), in tile order, so the result is bit-identical to the serial loop. Live across the wait: O (64 fp32),
    // S(j) (BKV / 2 fp32) and P(j-1) (BKV / 4 packed bf16x2): 160 registers for 128-key tiles, 196 for 176-key tiles, within
    // setmaxnreg's 240.
    //
    // The two consumer warpgroups also take turns: warpgroup w issues its GEMMs only between bar.sync on barrier 1 + w and
    // bar.arrive on the other's barrier 2 - w, so one warpgroup's softmax runs while the tensor cores work through the other's
    // GEMMs. Each warpgroup makes n_tiles + 1 turns (S(0); S(j) + PV(j-1) for j in [1, n_tiles); PV(n_tiles-1)) whatever rows
    // it holds (a warpgroup whose rows are past Lq computes on TMA's zero fill), since n_tiles is uniform over the CTA.
    // Warpgroup 0 pre-arrives once on its own barrier and warpgroup 1 skips its arrival after its last turn, so on each
    // barrier the arrivals equal the syncs (n_tiles + 1) and both are at rest when the CTA exits. The K/V mbarrier waits come
    // before a turn is taken, never inside one, so a warpgroup holding the turn never waits on the producer.
    constexpr uint32_t kTurnThreads = 256;
    const uint32_t bar_own = 1 + wg, bar_other = 2 - wg;
    auto turn_begin = [&] { ptx::named_bar_sync(bar_own, kTurnThreads); };
    auto turn_end = [&] { ptx::named_bar_arrive(bar_other, kTurnThreads); };
    if (wg == 0) ptx::named_bar_arrive(bar_own, kTurnThreads);

    float sc[BKV / 2];
    uint32_t pa[BKV / 16][4];  // P of the tile whose PV is issued next, as the register A operand
    const int valid = p.Lk - (total_tiles - 1) * BKV;
    auto issue_s = [&](int j) {
      const int s = j & 1;
      ptx::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kHD / 16; ++kk) {
        // 64-column half (kk >> 2) is a separate TMA box; inside a box one K16 step is 32 B (+2 in the >> 4 field)
        const uint64_t da = ptx::gmma_desc_sw128_kmajor(q_base + (kk >> 2) * (kQBytes / 2)) + 2 * (kk & 3);
        const uint64_t db = ptx::gmma_desc_sw128_kmajor(k_base + s * L::kKBytes + (kk >> 2) * (L::kKBytes / 2)) + 2 * (kk & 3);
        if constexpr (BKV == 176) {
          ptx::wgmma_m64n176k16_ss(sc, da, db, kk != 0 ? 1u : 0u);
        } else if constexpr (BKV == 128) {
          ptx::wgmma_m64n128k16_ss(sc, da, db, kk != 0 ? 1u : 0u);
        } else {
          static_assert(BKV == 64, "KV tile widths: 64, 128, 176");
          ptx::wgmma_m64n64k16_ss(sc, da, db, kk != 0 ? 1u : 0u);
        }
      }
      ptx::wgmma_commit();
    };
    auto issue_pv = [&](int j) {
      const int s = j & 1;
      ptx::fence_regs(o);
      ptx::wgmma_fence();
      const uint64_t dv = ptx::gmma_desc_sw128_mnmajor(v_base + s * L::kVBytes, BKV * 128);  // LBO = one [BKV kv x 64 d] box
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk)  // one K16 step = 16 kv rows = 2048 B of the MN-major tile
        ptx::wgmma_m64n128k16_rs_tb(o, pa[kk], dv + static_cast<uint64_t>(kk * (2048 / 16)), 1u);
      ptx::wgmma_commit();
    };
    // S(j) has retired (the caller's wgmma_wait): hand K(j) back, then the online softmax of tile j, P(j) in fp32 in place of
    // S(j); returns the factors O is scaled by
    auto softmax = [&](int j, float& f0, float& f1) {
      ptx::fence_regs(sc);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&k_empty[j & 1]);
      if (j == j_ragged) {  // keys past Lk (zero-filled by TMA) must not take part in the softmax
#pragma unroll
        for (int i = 0; i < BKV / 8; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (8 * i + cq + (e & 1) >= valid) sc[4 * i + e] = -INFINITY;
      }
      // row max over the quad (the 4 lanes holding a row's columns)
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int i = 0; i < BKV / 8; ++i) {
        mx0 = fmaxf(mx0, fmaxf(sc[4 * i], sc[4 * i + 1]));
        mx1 = fmaxf(mx1, fmaxf(sc[4 * i + 2], sc[4 * i + 3]));
      }
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
      }
      const float mn0 = fmaxf(m0, mx0 * p.scale_log2), mn1 = fmaxf(m1, mx1 * p.scale_log2);
      f0 = ptx::ex2_approx(m0 - mn0), f1 = ptx::ex2_approx(m1 - mn1);  // 0 on the first tile (m = -inf)
      m0 = mn0, m1 = mn1;
      l0 *= f0, l1 *= f1;
      // P = 2^(s*scale - m), row sum in fp32 before the bf16 rounding (as flash-attention does)
#pragma unroll
      for (int i = 0; i < BKV / 8; ++i) {
        sc[4 * i] = exp2_sel<EMU_MASK>(fmaf(sc[4 * i], p.scale_log2, -m0), i);
        sc[4 * i + 1] = exp2_sel<EMU_MASK>(fmaf(sc[4 * i + 1], p.scale_log2, -m0), i);
        sc[4 * i + 2] = exp2_sel<EMU_MASK>(fmaf(sc[4 * i + 2], p.scale_log2, -m1), i);
        sc[4 * i + 3] = exp2_sel<EMU_MASK>(fmaf(sc[4 * i + 3], p.scale_log2, -m1), i);
        l0 += sc[4 * i] + sc[4 * i + 1];
        l1 += sc[4 * i + 2] + sc[4 * i + 3];
      }
    };
    // P(j) rounded to bf16 and packed as the A operand
    auto pack_p = [&] {
#pragma unroll
      for (int i = 0; i < BKV / 8; ++i) {
        pa[i >> 1][(i & 1) * 2] = pack_bf16x2(sc[4 * i], sc[4 * i + 1]);
        pa[i >> 1][(i & 1) * 2 + 1] = pack_bf16x2(sc[4 * i + 2], sc[4 * i + 3]);
      }
    };
    // PV(j) has retired (the caller's wgmma_wait<0>): hand V(j) back
    auto release_v = [&](int j) {
      ptx::fence_regs(o);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&v_empty[j & 1]);
    };
    auto rescale_o = [&](float f0, float f1) {
#pragma unroll
      for (int i = 0; i < kHD / 8; ++i) {
        o[4 * i] *= f0, o[4 * i + 1] *= f0;
        o[4 * i + 2] *= f1, o[4 * i + 3] *= f1;
      }
    };
    {  // prologue: S(0), its softmax and P(0)
      ptx::mbar_wait_or_flag(&k_full[0], 0, timed_out);
      turn_begin();
      issue_s(0);
      turn_end();
      ptx::wgmma_wait<0>();
      float f0, f1;
      softmax(0, f0, f1);
      rescale_o(f0, f1);
      pack_p();
    }
    for (int j = 1; j < n_tiles; ++j) {  // steady state: S(j) and PV(j-1) in one turn, softmax(j) under PV(j-1)
      ptx::mbar_wait_or_flag(&k_full[j & 1], (j >> 1) & 1, timed_out);
      ptx::mbar_wait_or_flag(&v_full[(j - 1) & 1], ((j - 1) >> 1) & 1, timed_out);
      turn_begin();
      issue_s(j);
      issue_pv(j - 1);
      turn_end();
      ptx::wgmma_wait<1>();  // S(j) has retired, PV(j-1) may still run
      float f0, f1;
      softmax(j, f0, f1);
      ptx::wgmma_wait<0>();
      release_v(j - 1);
      rescale_o(f0, f1);
      pack_p();
    }
    {  // epilogue: PV(n-1)
      const int j = n_tiles - 1;
      ptx::mbar_wait_or_flag(&v_full[j & 1], (j >> 1) & 1, timed_out);
      turn_begin();
      issue_pv(j);
      if (wg == 0) turn_end();  // warpgroup 1's last turn has no successor to release
      ptx::wgmma_wait<0>();
      release_v(j);
    }
    if (timed_out) __trap();

    // ---- epilogue: O / l -> bf16 -> global (or the normalised fp32 partial of this split)
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      l0 += __shfl_xor_sync(0xffffffffu, l0, off);
      l1 += __shfl_xor_sync(0xffffffffu, l1, off);
    }
    const bool partial = wi.nsplit > 1;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float inv_l = 1.0f / (h ? l1 : l0);
      const int rt = r + 8 * h;
      const int row = q0 + rt;
      if (row >= p.Lq) continue;
      if (partial) {
        const int64_t prow = (static_cast<int64_t>(wi.split) * p.tail_units + wi.tail_unit) * kBQ + rt;
        if ((lane & 3) == 0) p.part_ml[prow] = make_float2(h ? m1 : m0, h ? l1 : l0);
        float* dst = p.part_o + prow * kHD + cq;
#pragma unroll
        for (int i = 0; i < kHD / 8; ++i)
          *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(o[4 * i + 2 * h] * inv_l, o[4 * i + 2 * h + 1] * inv_l);
      } else {
        __nv_bfloat16* dst = p.out + static_cast<int64_t>(row) * p.ldo + head * kHD + cq;
#pragma unroll
        for (int i = 0; i < kHD / 8; ++i)
          *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_bf16x2(o[4 * i + 2 * h] * inv_l, o[4 * i + 2 * h + 1] * inv_l);
      }
    }
  }
}

// Merge of the split-KV partials of the tail units: out = sum_s w_s O_s / sum_s w_s with w_s = l_s * 2^(m_s - max_s m_s).
__global__ void __launch_bounds__(256) attn_combine_kernel(const float* __restrict__ part_o, const float2* __restrict__ part_ml, int nsplit,
                                                           int tail_units, int full_units, int q_blocks, int rows_per_cta, int Lq,
                                                           __nv_bfloat16* __restrict__ out, int64_t ldo) {
  constexpr int kGroups = kHD / 8;
  const int64_t total = static_cast<int64_t>(tail_units) * rows_per_cta * kGroups;
  const int64_t split_stride = static_cast<int64_t>(tail_units) * rows_per_cta;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t prow = i / kGroups;
    const int g = static_cast<int>(i - prow * kGroups);
    const int tu = static_cast<int>(prow / rows_per_cta), r = static_cast<int>(prow - static_cast<int64_t>(tu) * rows_per_cta);
    const int unit = full_units + tu;
    const int head = unit / q_blocks, row = (unit - head * q_blocks) * rows_per_cta + r;
    if (row >= Lq) continue;
    float mmax = -INFINITY;
    for (int s = 0; s < nsplit; ++s) mmax = fmaxf(mmax, part_ml[s * split_stride + prow].x);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float wsum = 0.f;
    for (int s = 0; s < nsplit; ++s) {
      const float2 ml = part_ml[s * split_stride + prow];
      const float w = ml.y * ptx::ex2_approx(ml.x - mmax);
      wsum += w;
      float v[8];
      ptx::ld_nc_v8_f32(part_o + (s * split_stride + prow) * kHD + g * 8, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(w, v[j], acc[j]);
    }
    const float inv = 1.0f / wsum;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= inv;
    *reinterpret_cast<uint4*>(out + static_cast<int64_t>(row) * ldo + head * kHD + g * 8) = pack_bf16x8(acc);
  }
}

// ---- host side: work decomposition ----------------------------------------------------------------------------------
struct AttnPlan {
  int q_blocks, kv_tile, total_tiles, rows_per_cta;
  int full_units, tail_units, tail_split;  // see AttnParams
  size_t ws_bytes;                         // workspace for the split partials (0 when nothing is split)
  int grid() const { return full_units + tail_units * tail_split; }
};

static int env_int(const char* name, int lo, int hi, int dflt) {
  const char* e = getenv(name);
  if (!e || !*e) return dflt;
  const int v = atoi(e);
  return (v < lo || v > hi) ? dflt : v;
}

// KV tile width of a call: 176 keys for long key sequences and for the rotated / flag-gated key order of token-sharded runs, 64
// for short ones. MC_ATTN_KERNEL forces a width (tests, A-B timing in one process): 1 = 64 keys (not for the rotated /
// flag-gated order, which keeps 176), 2 = 128 keys (the kernel with the FMA-pipe exponential variants), 3 = 176 keys.
static int attn_kv_tile(int Lk, bool need_long) {
  switch (env_int("MC_ATTN_KERNEL", 0, 3, 0)) {
    case 1: return need_long ? 176 : 64;
    case 2: return 128;
    case 3: return 176;
    default: return (need_long || Lk >= kLongMinLk) ? 176 : 64;
  }
}

// One CTA = 128 query rows of one head (one CTA per SM), every unit the same length, so the grid runs in rounds of `slots` CTAs
// and a partially filled last round costs a whole one (32760 rows x 12 heads = 3072 units on 132 SMs: 23.3 rounds of work take
// 24; a token-sharded rank's 4095 rows: 384 units, 2.9 rounds take 3). The units
// of that last round are therefore split over the KV range, floor(slots / units) ways, so that they fill the SMs once at a
// fraction of the length; a second kernel merges their partial softmaxes. Units of the full rounds are never split, and no
// split gets fewer than 512 keys (8 / 4 / 3 tiles of 64 / 128 / 176): below that the pipeline's prologue and epilogue and the
// merge outweigh the shorter split. At the benchmarked shape: 187 tiles of 176, the 36 units of the last round split 3 ways.
static AttnPlan plan_attention(int Lq, int Lk, int heads, int kv_tile) {
  AttnPlan pl;
  const int forced_splits = env_int("MC_ATTN_SPLITS", 1, 16, 0);  // MC_ATTN_SPLITS=n: every unit split n ways (1 = never split)
  pl.rows_per_cta = ak::kBQ;
  pl.kv_tile = kv_tile;
  pl.q_blocks = (Lq + pl.rows_per_cta - 1) / pl.rows_per_cta;
  pl.total_tiles = (Lk + pl.kv_tile - 1) / pl.kv_tile;
  const int64_t units = static_cast<int64_t>(pl.q_blocks) * heads;
  const int slots = num_sms();
  const int min_tiles_per_split = (512 + pl.kv_tile - 1) / pl.kv_tile;
  int full = static_cast<int>(units), tail = 0, split = 1;
  if (forced_splits > 0) {
    if (forced_splits > 1) full = 0, tail = static_cast<int>(units), split = forced_splits;
  } else {
    const int rem = static_cast<int>(units % slots);
    const int by_tiles = pl.total_tiles / min_tiles_per_split;
    int f = rem > 0 ? slots / rem : 1;
    if (f > 8) f = 8;
    if (f > by_tiles) f = by_tiles;
    if (f >= 2) full = static_cast<int>(units) - rem, tail = rem, split = f;
  }
  if (split > pl.total_tiles) split = pl.total_tiles;
  if (split > 1) {
    const int per = (pl.total_tiles + split - 1) / split;
    split = (pl.total_tiles + per - 1) / per;  // no empty split
  }
  if (split <= 1) full = static_cast<int>(units), tail = 0, split = 1;
  pl.full_units = full, pl.tail_units = tail, pl.tail_split = split;
  pl.ws_bytes = tail > 0 ? static_cast<size_t>(split) * tail * pl.rows_per_cta * (kHD * sizeof(float) + sizeof(float2)) : 0;
  return pl;
}

}  // namespace mc

extern "C" int32_t mc_attn_workspace_bytes(int32_t Lq, int32_t Lk, int32_t heads, int64_t* bytes_out) {
  MC_CHECK_ARG(bytes_out != nullptr && Lq >= 1 && Lk >= 1 && heads >= 1, "mc_attn_workspace_bytes: bad arguments");
  // the largest decomposition over every tile width the launcher may pick, whatever MC_ATTN_KERNEL and the key order, so a
  // workspace sized once for a shape serves every later call of that shape
  size_t most = 0;
  for (const int kv_tile : {64, 128, 176}) {
    const size_t b = mc::plan_attention(Lq, Lk, heads, kv_tile).ws_bytes;
    most = b > most ? b : most;
  }
  *bytes_out = static_cast<int64_t>(most);
  return MC_OK;
}

extern "C" int32_t mc_attn_fwd_ex(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out,
                                  int64_t ldo, int32_t Lq, int32_t Lk, int32_t heads, float scale, void* workspace,
                                  int64_t workspace_bytes, int32_t first_key_row, const uint32_t* seg_flags, const uint32_t* seg_epoch,
                                  int32_t seg_rows, void* stream) {
  MC_CHECK_ARG(q && k && v && out, "mc_attn_fwd: null pointer");
  MC_CHECK_ARG(Lq >= 1 && Lk >= 1 && heads >= 1, "mc_attn_fwd: Lq=%d Lk=%d heads=%d", Lq, Lk, heads);
  const int64_t width = static_cast<int64_t>(heads) * mc::kHD;
  MC_CHECK_ARG(ldq >= width && ldk >= width && ldo >= width && ldv >= width, "mc_attn_fwd: leading dimensions too small");
  MC_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, "mc_attn_fwd: leading dimensions must be multiples of 8");
  MC_CHECK_ARG(mc::aligned16(q) && mc::aligned16(k) && mc::aligned16(v) && mc::aligned16(out), "mc_attn_fwd: pointers must be 16-byte aligned");
  MC_CHECK_ARG(first_key_row >= 0 && first_key_row < Lk, "mc_attn_fwd: first_key_row=%d outside [0, %d)", first_key_row, Lk);
  MC_CHECK_ARG(seg_flags == nullptr || (seg_rows >= 1 && seg_epoch != nullptr), "mc_attn_fwd: seg_rows=%d / null epoch", seg_rows);
  const mc::AttnPlan pl = mc::plan_attention(Lq, Lk, heads, mc::attn_kv_tile(Lk, first_key_row != 0 || seg_flags != nullptr));
  MC_CHECK_ARG(static_cast<int64_t>(pl.q_blocks) * heads * 8 < INT32_MAX, "mc_attn_fwd: grid too large");
  if (pl.tail_units > 0) {
    MC_CHECK_ARG(workspace != nullptr && workspace_bytes >= static_cast<int64_t>(pl.ws_bytes) && (reinterpret_cast<uintptr_t>(workspace) & 31u) == 0,
                 "mc_attn_fwd: split-KV needs a 32-byte aligned workspace of %lld bytes (mc_attn_workspace_bytes), got %lld",
                 static_cast<long long>(pl.ws_bytes), static_cast<long long>(workspace_bytes));
  }
  const int q_box = mc::ak::kBQ;
  CUtensorMap tq, tk, tv;
  int32_t rc = mc::make_tmap_bf16_2d(&tq, q, static_cast<uint64_t>(Lq), static_cast<uint64_t>(width), static_cast<uint64_t>(ldq), q_box, 64);
  if (rc) return rc;
  rc = mc::make_tmap_bf16_2d(&tk, k, static_cast<uint64_t>(Lk), static_cast<uint64_t>(width), static_cast<uint64_t>(ldk), pl.kv_tile, 64);
  if (rc) return rc;
  rc = mc::make_tmap_bf16_2d(&tv, v, static_cast<uint64_t>(Lk), static_cast<uint64_t>(width), static_cast<uint64_t>(ldv), pl.kv_tile, 64);
  if (rc) return rc;

  float* part_o = static_cast<float*>(workspace);
  const size_t part_rows = static_cast<size_t>(pl.tail_split) * pl.tail_units * pl.rows_per_cta;
  float2* part_ml = pl.tail_units > 0 ? reinterpret_cast<float2*>(part_o + part_rows * mc::kHD) : nullptr;
  mc::AttnParams p{};
  p.Lq = Lq, p.Lk = Lk, p.heads = heads;
  p.q_blocks = pl.q_blocks, p.full_units = pl.full_units, p.tail_units = pl.tail_units, p.tail_split = pl.tail_split;
  p.part_o = pl.tail_units > 0 ? part_o : nullptr, p.part_ml = part_ml;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = static_cast<__nv_bfloat16*>(out), p.ldo = ldo;
  // start with the first tile that lies entirely inside the caller's own (already resident) rows; the tile straddling the segment
  // boundary before it comes last in the rotated order
  p.tile_rot = ((first_key_row + pl.kv_tile - 1) / pl.kv_tile) % pl.total_tiles;
  p.seg_flags = seg_flags, p.seg_epoch = seg_epoch, p.seg_rows = seg_rows > 0 ? seg_rows : Lk;

  dim3 grid(pl.grid(), 1, 1);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // one PerDeviceOnce per instantiation: [0] 64 keys, [1] 176 keys, [2..5] 128 keys with MC_ATTN_EMU 0 / 2 / 3 / 4
  static mc::PerDeviceOnce once[6];
#define MC_LAUNCH(BKV, MASK, IDX)                                                                                                    \
  do {                                                                                                                               \
    rc = mc::set_max_smem_once(mc::attn_kernel<BKV, MASK>, mc::ak::Layout<BKV>::kSmem, once[IDX], "cudaFuncSetAttribute(attn smem)"); \
    if (rc) return rc;                                                                                                               \
    mc::attn_kernel<BKV, MASK><<<grid, mc::ak::kThreads, mc::ak::Layout<BKV>::kSmem, st>>>(tq, tk, tv, p);                           \
  } while (0)
  if (pl.kv_tile == 176) {
    MC_LAUNCH(176, 0x00u, 1);
  } else if (pl.kv_tile == 128) {
    // MC_ATTN_EMU = eighths of the exponentials evaluated on the FMA pipe: 0, 2 (25 %), 3 (37.5 %), 4 (50 %)
    switch (mc::env_int("MC_ATTN_EMU", 0, 4, MC_ATTN_EMU_DEFAULT)) {
      case 2: MC_LAUNCH(128, 0x88u, 3); break;
      case 3: MC_LAUNCH(128, 0x92u, 4); break;
      case 4: MC_LAUNCH(128, 0xAAu, 5); break;
      default: MC_LAUNCH(128, 0x00u, 2); break;
    }
  } else {
    MC_LAUNCH(64, 0x00u, 0);
  }
#undef MC_LAUNCH
  MC_CHECK_LAUNCH("attn_kernel launch");
  if (pl.tail_units > 0) {
    const int64_t total = static_cast<int64_t>(pl.tail_units) * pl.rows_per_cta * (mc::kHD / 8);
    const int64_t want = (total + 255) / 256, cap = static_cast<int64_t>(mc::num_sms()) * 8;
    mc::attn_combine_kernel<<<static_cast<int>(want < cap ? want : cap), 256, 0, st>>>(
        p.part_o, p.part_ml, pl.tail_split, pl.tail_units, pl.full_units, pl.q_blocks, pl.rows_per_cta, Lq, static_cast<__nv_bfloat16*>(out), ldo);
    MC_CHECK_LAUNCH("attn_combine_kernel launch");
  }
  return MC_OK;
}

extern "C" int32_t mc_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out,
                               int64_t ldo, int32_t Lq, int32_t Lk, int32_t heads, float scale, void* workspace,
                               int64_t workspace_bytes, void* stream) {
  return mc_attn_fwd_ex(q, ldq, k, ldk, v, ldv, out, ldo, Lq, Lk, heads, scale, workspace, workspace_bytes, 0, nullptr, nullptr, 0, stream);
}
