// Open-Sora 1.2 (STDiT3) attention kernels, head_dim 72 (videosys/models/transformers/open_sora_transformer_3d.py, called from
// eval/magcache/experiments/opensora.py:314-341):
//   * attn_varlen_d72_kernel: many independent (query rows, key rows) segments in one launch — the spatial self-attention over
//     B*T frames (`rearrange(x_m, "B (T S) C -> (B T) S C")` + OpenSoraAttention, :202-204) and the cross-attention with per-sample
//     caption lengths (OpenSoraMultiHeadCrossAttention.flash_attn_impl, attentions.py:136-153).
//   * attn_temporal_d72_kernel: the temporal self-attention over B*S sequences of T <= 32 frames, read in place from the B (T S) C
//     row order (the reference's `rearrange` copies around it, :196-198, are not made).
//   * rmsnorm_head72_rope_kernel: the q / k LlamaRMSNorm(72) and the temporal RoPE (attentions.py:71-75).
//
// The varlen kernel is a separate mma.sync (m16n8k16) kernel rather than a head_dim template of attn_kernel, so that attn_kernel's
// code and its tuned register budget stay exactly as they are: its 128-wide TMA boxes, m64n128 PV GEMM and one key range per
// launch are all fixed by head_dim 128. The cost is speed: at the 480p workload this kernel runs the spatial attention at about a
// third of attn_kernel's rate on head_dim 128, and spatial + cross attention are ~27 % of a miss forward (DESIGN §4). A wgmma form
// is recorded in DESIGN §8 as the next step.
//
// attn_temporal_d72_kernel is HBM-bound by its algorithm but reaches only about a quarter of the HBM rate: at T = 15 only 15 of 32
// lanes compute, and each warp loads 144-byte head slices S rows apart.
#include "common.cuh"
#include "ptx.cuh"

namespace mc {

namespace os {

constexpr int kD = 72;        // head dim
constexpr int kDP = 80;       // head dim padded to a multiple of 16 (QK^T k-steps); columns 72..79 are zero in shared memory
constexpr int kLd = 88;       // shared-memory row pitch in elements (176 B: ldmatrix rows fall on distinct bank groups)
constexpr int kBQ = 64;       // query rows per CTA (4 warps x 16)
constexpr int kBK = 64;       // keys per tile
constexpr int kThreads = 128;
constexpr int kTileElems = kBK * kLd;
constexpr int kSmemBytes = (kBQ * kLd + 4 * kTileElems) * 2;  // Q + 2 stages of (K, V)

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const uint32_t s = ptx::smem_u32(smem);
  const int n = valid ? 16 : 0;  // src-size 0: the 16 bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(ptx::smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x2(uint32_t (&r)[2], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];\n" : "=r"(r[0]), "=r"(r[1]) : "r"(ptx::smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x2_t(uint32_t (&r)[2], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];\n" : "=r"(r[0]), "=r"(r[1]) : "r"(ptx::smem_u32(p)));
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// rows [row0, row0 + 64) of one head (72 columns) -> shared [64][kLd]; rows at or past `n` are zero-filled
__device__ __forceinline__ void load_tile(__nv_bfloat16* dst, const __nv_bfloat16* src, int64_t ld, int64_t row0, int n, int tid) {
  for (int i = tid; i < kBK * 9; i += kThreads) {
    const int r = i / 9, c = i - r * 9;
    const bool ok = r < n;
    cp_async16(dst + r * kLd + c * 8, ok ? src + (row0 + r) * ld + c * 8 : src, ok);
  }
}

}  // namespace os

// segs: int32 [n_seg, 4] = (q_start, q_len, k_start, k_len). grid (q tiles of the longest segment, n_seg, heads).
__global__ void __launch_bounds__(os::kThreads) attn_varlen_d72_kernel(const __nv_bfloat16* __restrict__ q, int64_t ldq,
                                                                       const __nv_bfloat16* __restrict__ k, int64_t ldk,
                                                                       const __nv_bfloat16* __restrict__ v, int64_t ldv,
                                                                       __nv_bfloat16* __restrict__ out, int64_t ldo,
                                                                       const int32_t* __restrict__ segs, float scale_log2) {
  using namespace os;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* sKV = sQ + kBQ * kLd;  // stage s: K at sKV + (2s) * kTileElems, V at sKV + (2s+1) * kTileElems
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int4 sg = reinterpret_cast<const int4*>(segs)[blockIdx.y];
  const int q_start = sg.x, q_len = sg.y, k_start = sg.z, k_len = sg.w;
  const int q0 = blockIdx.x * kBQ;
  if (q0 >= q_len || k_len <= 0) return;
  const int h = blockIdx.z;
  const __nv_bfloat16* qh = q + h * kD;
  const __nv_bfloat16* kh = k + h * kD;
  const __nv_bfloat16* vh = v + h * kD;

  // zero the pad columns 72..79 of Q and of both K stages (never written by the loads)
  for (int r = tid; r < kBQ + 4 * kBK; r += kThreads) {
    __nv_bfloat16* row = (r < kBQ) ? sQ + r * kLd : sKV + (r - kBQ) * kLd;
    *reinterpret_cast<uint4*>(row + kD) = make_uint4(0u, 0u, 0u, 0u);
  }
  const int n_tiles = (k_len + kBK - 1) / kBK;
  load_tile(sQ, qh, ldq, static_cast<int64_t>(q_start) + q0, q_len - q0, tid);
  load_tile(sKV, kh, ldk, k_start, k_len, tid);
  load_tile(sKV + kTileElems, vh, ldv, k_start, k_len, tid);
  cp_async_commit();

  uint32_t qf[5][4];
  float o[9][4];
#pragma unroll
  for (int j = 0; j < 9; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows lane/4 and lane/4 + 8 of this warp's 16

  for (int t = 0; t < n_tiles; ++t) {
    if (t + 1 < n_tiles) {
      const int st = (t + 1) & 1;
      const int kr = (t + 1) * kBK;
      load_tile(sKV + (2 * st) * kTileElems, kh, ldk, static_cast<int64_t>(k_start) + kr, k_len - kr, tid);
      load_tile(sKV + (2 * st + 1) * kTileElems, vh, ldv, static_cast<int64_t>(k_start) + kr, k_len - kr, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (t == 0) {
#pragma unroll
      for (int ks = 0; ks < 5; ++ks) ldsm_x4(qf[ks], sQ + (warp * 16 + (lane & 15)) * kLd + ks * 16 + (lane >> 4) * 8);
    }
    const __nv_bfloat16* sK = sKV + (2 * (t & 1)) * kTileElems;
    const __nv_bfloat16* sV = sK + kTileElems;

    // S = Q K^T : 16 x 64 per warp
    float s[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 5; ++ks) {
        uint32_t b[2];
        ldsm_x2(b, sK + (n * 8 + (lane & 7)) * kLd + ks * 16 + ((lane >> 3) & 1) * 8);
        mma_bf16(s[n], qf[ks], b);
      }
    }
    // mask the keys past the segment, online softmax (base-2, scale folded in)
    const int kvalid = k_len - t * kBK;
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const int c = n * 8 + (lane & 3) * 2;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float x = s[n][e] * scale_log2;
        if (c + (e & 1) >= kvalid) x = -INFINITY;
        s[n][e] = x;
      }
      mx0 = fmaxf(mx0, fmaxf(s[n][0], s[n][1]));
      mx1 = fmaxf(mx1, fmaxf(s[n][2], s[n][3]));
    }
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
    }
    const float c0 = exp2f(m0 - mx0), c1 = exp2f(m1 - mx1);  // m = -inf on the first tile: exp2(-inf) = 0
    m0 = mx0, m1 = mx1;
    float rs0 = 0.f, rs1 = 0.f;
    uint32_t p[4][4];  // P as the A operand of the four 16-key k-steps
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const float p0 = exp2f(s[n][0] - mx0), p1 = exp2f(s[n][1] - mx0);
      const float p2 = exp2f(s[n][2] - mx1), p3 = exp2f(s[n][3] - mx1);
      rs0 += p0 + p1;
      rs1 += p2 + p3;
      p[n >> 1][(n & 1) * 2 + 0] = pack_bf16x2(p0, p1);
      p[n >> 1][(n & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
    l0 = l0 * c0 + rs0;
    l1 = l1 * c1 + rs1;
#pragma unroll
    for (int j = 0; j < 9; ++j) {
      o[j][0] *= c0, o[j][1] *= c0, o[j][2] *= c1, o[j][3] *= c1;
    }
    // O += P V : k = 64 keys (4 steps), n = 72 (9 tiles of 8)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint32_t a[4] = {p[ks][0], p[ks][1], p[ks][2], p[ks][3]};
#pragma unroll
      for (int j = 0; j < 9; ++j) {
        uint32_t b[2];
        ldsm_x2_t(b, sV + (ks * 16 + (lane & 15)) * kLd + j * 8);
        mma_bf16(o[j], a, b);
      }
    }
    __syncthreads();  // the stage read here is refilled by the next iteration's loads
  }
  // row sums over the quad, normalise, store bf16
#pragma unroll
  for (int off = 1; off <= 2; off <<= 1) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, off);
    l1 += __shfl_xor_sync(0xffffffffu, l1, off);
  }
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  const int r0 = q0 + warp * 16 + (lane >> 2), r1 = r0 + 8;
  __nv_bfloat16* oh = out + h * kD + (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    if (r0 < q_len)
      *reinterpret_cast<uint32_t*>(oh + (static_cast<int64_t>(q_start) + r0) * ldo + j * 8) = pack_bf16x2(o[j][0] * i0, o[j][1] * i0);
    if (r1 < q_len)
      *reinterpret_cast<uint32_t*>(oh + (static_cast<int64_t>(q_start) + r1) * ldo + j * 8) = pack_bf16x2(o[j][2] * i1, o[j][3] * i1);
  }
}

// Temporal attention: one warp per (sequence b*S + s, head), lane = query frame. The T key / value rows of the sequence (S rows
// apart in HBM) are staged in shared memory; each lane runs an fp32 online softmax over them.
constexpr int kTempMaxT = 32;
constexpr int kTempWarps = 4;
__global__ void __launch_bounds__(kTempWarps * 32) attn_temporal_d72_kernel(const __nv_bfloat16* __restrict__ q, int64_t ldq,
                                                                            const __nv_bfloat16* __restrict__ k, int64_t ldk,
                                                                            const __nv_bfloat16* __restrict__ v, int64_t ldv,
                                                                            __nv_bfloat16* __restrict__ out, int64_t ldo, int T, int S,
                                                                            int heads, float scale_log2) {
  __shared__ __align__(16) __nv_bfloat16 sk[kTempWarps][kTempMaxT * os::kD];
  __shared__ __align__(16) __nv_bfloat16 sv[kTempWarps][kTempMaxT * os::kD];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y * kTempWarps + warp;
  if (h >= heads) return;
  const int64_t seq = blockIdx.x;  // b * S + s
  const int64_t b = seq / S, s = seq - b * S;
  const int64_t row0 = b * T * S + s;  // row of frame t: row0 + t * S
  for (int i = lane; i < T * 9; i += 32) {
    const int t = i / 9, c = i - t * 9;
    const int64_t r = row0 + static_cast<int64_t>(t) * S;
    *reinterpret_cast<uint4*>(&sk[warp][t * os::kD + c * 8]) = ptx::ld_nc_v4(k + r * ldk + h * os::kD + c * 8);
    *reinterpret_cast<uint4*>(&sv[warp][t * os::kD + c * 8]) = ptx::ld_nc_v4(v + r * ldv + h * os::kD + c * 8);
  }
  __syncwarp();
  if (lane >= T) return;
  const int64_t r = row0 + static_cast<int64_t>(lane) * S;
  uint32_t qp[36];
#pragma unroll
  for (int c = 0; c < 9; ++c) {
    const uint4 u = ptx::ld_nc_v4(q + r * ldq + h * os::kD + c * 8);
    qp[4 * c] = u.x, qp[4 * c + 1] = u.y, qp[4 * c + 2] = u.z, qp[4 * c + 3] = u.w;
  }
  float acc[os::kD];
#pragma unroll
  for (int d = 0; d < os::kD; ++d) acc[d] = 0.f;
  float m = -INFINITY, l = 0.f;
  for (int j = 0; j < T; ++j) {
    const uint32_t* kr = reinterpret_cast<const uint32_t*>(&sk[warp][j * os::kD]);
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < 36; ++i) {
      const uint32_t kw = kr[i];
      dot = fmaf(bf16_lo(qp[i]), bf16_lo(kw), dot);
      dot = fmaf(bf16_hi(qp[i]), bf16_hi(kw), dot);
    }
    const float x = dot * scale_log2;
    const float mn = fmaxf(m, x);
    const float corr = exp2f(m - mn), p = exp2f(x - mn);
    m = mn;
    l = l * corr + p;
    const uint32_t* vr = reinterpret_cast<const uint32_t*>(&sv[warp][j * os::kD]);
#pragma unroll
    for (int i = 0; i < 36; ++i) {
      const uint32_t vw = vr[i];
      acc[2 * i] = fmaf(p, bf16_lo(vw), acc[2 * i] * corr);
      acc[2 * i + 1] = fmaf(p, bf16_hi(vw), acc[2 * i + 1] * corr);
    }
  }
  const float il = 1.f / l;
  __nv_bfloat16* po = out + r * ldo + h * os::kD;
#pragma unroll
  for (int c = 0; c < 9; ++c) {
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = acc[c * 8 + e] * il;
    *reinterpret_cast<uint4*>(po + c * 8) = pack_bf16x8(f);
  }
}

// LlamaRMSNorm(72) per head (videosys/models/modules/normalization.py:17-22: fp32 variance, `weight * x.to(bf16)`), then, with
// cos_sin, RoPE on interleaved pairs as rotary_embedding_torch's rotate_queries_or_keys [EXT] computes it in fp32:
//   y[2i] = x[2i]*cos - x[2i+1]*sin ; y[2i+1] = x[2i+1]*cos + x[2i]*sin ; rounded to bf16.
// One thread per (row, head); position of a row = (row / pos_div) % pos_mod, cos_sin fp32 [pos_mod, 72] = (cos, sin) per pair.
__global__ void __launch_bounds__(256) rmsnorm_head72_rope_kernel(__nv_bfloat16* __restrict__ x, int64_t ld, int64_t rows, int heads,
                                                                  const float* __restrict__ w, float eps,
                                                                  const float* __restrict__ cos_sin, int64_t pos_div, int pos_mod) {
  const int64_t items = rows * heads;
  for (int64_t it = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; it < items; it += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t row = it / heads;
    const int head = static_cast<int>(it - row * heads);
    __nv_bfloat16* px = x + row * ld + head * os::kD;
    float v[os::kD];
    float ss = 0.f;
#pragma unroll
    for (int c = 0; c < 9; ++c) {
      float f[8];
      unpack_bf16x8(*reinterpret_cast<const uint4*>(px + c * 8), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        v[c * 8 + e] = f[e];
        ss = fmaf(f[e], f[e], ss);
      }
    }
    const float r = rsqrtf(ss * (1.0f / os::kD) + eps);
#pragma unroll
    for (int d = 0; d < os::kD; ++d) v[d] = round_bf16(round_bf16(v[d] * r) * __ldg(w + d));
    if (cos_sin != nullptr) {
      const float* cs = cos_sin + ((row / pos_div) % pos_mod) * os::kD;
#pragma unroll
      for (int i = 0; i < os::kD / 2; ++i) {
        const float re = v[2 * i], im = v[2 * i + 1], c = __ldg(cs + 2 * i), sn = __ldg(cs + 2 * i + 1);
        v[2 * i] = __fsub_rn(__fmul_rn(re, c), __fmul_rn(im, sn));
        v[2 * i + 1] = __fadd_rn(__fmul_rn(im, c), __fmul_rn(re, sn));
      }
    }
#pragma unroll
    for (int c = 0; c < 9; ++c) {
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = v[c * 8 + e];
      *reinterpret_cast<uint4*>(px + c * 8) = pack_bf16x8(f);
    }
  }
}

}  // namespace mc

static bool ld_ok(int64_t ld, int heads) { return ld % 8 == 0 && ld >= static_cast<int64_t>(heads) * mc::os::kD; }

int32_t mc_attn_varlen_d72(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out, int64_t ldo,
                           int32_t heads, const int32_t* segs_dev, int32_t n_segs, int32_t max_q_len, float scale, void* stream) {
  MC_CHECK_ARG(q && k && v && out && segs_dev, "mc_attn_varlen_d72: null pointer");
  MC_CHECK_ARG(heads >= 1 && heads <= 65535 && n_segs >= 1 && n_segs <= 65535 && max_q_len >= 1, "mc_attn_varlen_d72: heads=%d n_segs=%d max_q_len=%d",
               heads, n_segs, max_q_len);
  MC_CHECK_ARG(ld_ok(ldq, heads) && ld_ok(ldk, heads) && ld_ok(ldv, heads) && ld_ok(ldo, heads),
               "mc_attn_varlen_d72: leading dimensions must be multiples of 8 and >= heads*72");
  MC_CHECK_ARG(mc::aligned16(q) && mc::aligned16(k) && mc::aligned16(v) && mc::aligned16(out) && mc::aligned16(segs_dev),
               "mc_attn_varlen_d72: pointers must be 16-byte aligned");
  static mc::PerDeviceOnce once;
  int32_t rc = mc::set_max_smem_once(mc::attn_varlen_d72_kernel, mc::os::kSmemBytes, once, "cudaFuncSetAttribute(attn_varlen_d72 smem)");
  if (rc) return rc;
  const dim3 grid((max_q_len + mc::os::kBQ - 1) / mc::os::kBQ, n_segs, heads);
  mc::attn_varlen_d72_kernel<<<grid, mc::os::kThreads, mc::os::kSmemBytes, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(q), ldq, static_cast<const __nv_bfloat16*>(k), ldk, static_cast<const __nv_bfloat16*>(v), ldv,
      static_cast<__nv_bfloat16*>(out), ldo, segs_dev, scale * 1.4426950408889634f);
  MC_CHECK_LAUNCH("attn_varlen_d72_kernel launch");
  return MC_OK;
}

int32_t mc_attn_temporal_d72(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out, int64_t ldo,
                             int32_t B, int32_t T, int32_t S, int32_t heads, float scale, void* stream) {
  MC_CHECK_ARG(q && k && v && out, "mc_attn_temporal_d72: null pointer");
  MC_CHECK_ARG(B >= 1 && S >= 1 && T >= 1 && T <= mc::kTempMaxT && heads >= 1, "mc_attn_temporal_d72: B=%d T=%d S=%d heads=%d (T <= 32)", B, T, S, heads);
  MC_CHECK_ARG(static_cast<int64_t>(B) * S <= 0x7fffffff, "mc_attn_temporal_d72: B*S too large");
  MC_CHECK_ARG(ld_ok(ldq, heads) && ld_ok(ldk, heads) && ld_ok(ldv, heads) && ld_ok(ldo, heads),
               "mc_attn_temporal_d72: leading dimensions must be multiples of 8 and >= heads*72");
  MC_CHECK_ARG(mc::aligned16(q) && mc::aligned16(k) && mc::aligned16(v) && mc::aligned16(out), "mc_attn_temporal_d72: pointers must be 16-byte aligned");
  const dim3 grid(static_cast<unsigned>(static_cast<int64_t>(B) * S), (heads + mc::kTempWarps - 1) / mc::kTempWarps);
  mc::attn_temporal_d72_kernel<<<grid, mc::kTempWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(q), ldq, static_cast<const __nv_bfloat16*>(k), ldk, static_cast<const __nv_bfloat16*>(v), ldv,
      static_cast<__nv_bfloat16*>(out), ldo, T, S, heads, scale * 1.4426950408889634f);
  MC_CHECK_LAUNCH("attn_temporal_d72_kernel launch");
  return MC_OK;
}

int32_t mc_rmsnorm_head72_rope(void* x_bf16, int64_t ld, int64_t rows, int32_t heads, const float* w, float eps, const float* cos_sin,
                               int64_t pos_div, int32_t pos_mod, void* stream) {
  MC_CHECK_ARG(x_bf16 && w, "mc_rmsnorm_head72_rope: null pointer");
  MC_CHECK_ARG(rows >= 1 && heads >= 1 && ld_ok(ld, heads), "mc_rmsnorm_head72_rope: rows=%lld heads=%d ld=%lld", static_cast<long long>(rows),
               heads, static_cast<long long>(ld));
  MC_CHECK_ARG(cos_sin == nullptr || (pos_div >= 1 && pos_mod >= 1), "mc_rmsnorm_head72_rope: pos_div=%lld pos_mod=%d",
               static_cast<long long>(pos_div), pos_mod);
  MC_CHECK_ARG(mc::aligned16(x_bf16), "mc_rmsnorm_head72_rope: x must be 16-byte aligned");
  const int64_t items = rows * heads;
  const int64_t want = (items + 255) / 256, cap = static_cast<int64_t>(mc::num_sms()) * 16;
  mc::rmsnorm_head72_rope_kernel<<<static_cast<int>(want < cap ? want : cap), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<__nv_bfloat16*>(x_bf16), ld, rows, heads, w, eps, cos_sin, pos_div, pos_mod);
  MC_CHECK_LAUNCH("rmsnorm_head72_rope_kernel launch");
  return MC_OK;
}
