// IP-Adapter image-prompt attention of the FLUX double blocks (mc_ip_attn; the statements and the rounding chain are in
// include/magcache_b200.h). One launch per double block covers every adapter: per CTA 64 image rows of one head, 4 warps of 16
// rows. The head's K and V rows of every adapter are staged once in shared memory; the warp normalises its raw q rows with the
// per-head RMSNorm of mc_rmsnorm_head_rope (rowwise.cuh) into shared memory, runs QK^T and PV on mma.sync m16n8k16 with an online
// softmax over 64-key tiles, and folds each adapter's output into the bf16 sum in registers. The output goes out through the
// warp's Q rows in shared memory as 16-byte row stores.
#include "common.cuh"
#include "ptx.cuh"
#include "rowwise.cuh"

namespace mc {

namespace ip {

constexpr int kBQ = 64;        // image rows per CTA (4 warps x 16)
constexpr int kThreads = 128;
constexpr int kBK = 64;        // keys per softmax tile
constexpr int kLd = 136;       // shared-memory row pitch in elements (272 B: ldmatrix rows fall on distinct bank groups)
constexpr int kMaxKeys = MC_IP_ATTN_MAX_KEYS;
constexpr int kMaxAdapters = MC_IP_ATTN_MAX_ADAPTERS;

__host__ __device__ constexpr int pad16(int n) { return (n + 15) / 16 * 16; }
__host__ __device__ constexpr int smem_bytes(int key_rows) { return (kBQ + 2 * key_rows) * kLd * 2; }

struct Args {
  const __nv_bfloat16* q;
  int64_t ldq, rows;
  int heads;
  const float* w;
  float eps;
  const __nv_bfloat16* kv;
  int64_t ldkv;
  __nv_bfloat16* out;
  int64_t ldo;
  float scale_log2;
  int n_adapters, key_rows;           // key_rows: sum of pad16(n_keys) (shared-memory rows of K, and of V)
  int n_keys[kMaxAdapters];
  int kv_row0[kMaxAdapters];          // first row of adapter a in kv
  int smem_row0[kMaxAdapters];        // first shared-memory row of adapter a (16-row aligned)
  float scale[kMaxAdapters];
};

}  // namespace ip

__global__ void __launch_bounds__(ip::kThreads) ip_attn_kernel(const ip::Args p) {
  using namespace ip;
  using namespace ptx;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* sK = sQ + kBQ * kLd;
  __nv_bfloat16* sV = sK + p.key_rows * kLd;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int h = blockIdx.y;
  const int64_t row0 = static_cast<int64_t>(blockIdx.x) * kBQ;

  // K / V of head h for every adapter; the rows past each adapter's keys are zero-filled (P is 0 there, and 0 * V must stay 0)
  for (int a = 0; a < p.n_adapters; ++a) {
    const int n = p.n_keys[a], r_pad = pad16(n);
    const __nv_bfloat16* src = p.kv + static_cast<int64_t>(p.kv_row0[a]) * p.ldkv + h * 128;
    for (int i = tid; i < r_pad * 16; i += kThreads) {
      const int r = i >> 4, c = (i & 15) * 8;
      const bool ok = r < n;
      const __nv_bfloat16* g = ok ? src + r * p.ldkv + c : p.kv;
      const int s = (p.smem_row0[a] + r) * kLd + c;
      cp_async16(sK + s, g, ok);
      cp_async16(sV + s, ok ? g + p.heads * 128 : p.kv, ok);
    }
  }
  cp_async_commit();

  // q: per-head RMSNorm of the raw projection, a half-warp per row, all eight row loads of the warp in flight first
  const int half = lane >> 4, sub = lane & 15;
  uint4 raw[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const int64_t r = row0 + warp * 16 + 2 * t + half;
    raw[t] = r < p.rows ? ptx::ld_nc_v4(p.q + r * p.ldq + h * 128 + sub * 8) : make_uint4(0u, 0u, 0u, 0u);
  }
  __nv_bfloat16* sQw = sQ + warp * 16 * kLd;  // this warp's 16 rows
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    float v[8], o[8];
    unpack_bf16x8(raw[t], v);
    head_rmsnorm8(v, p.w + sub * 8, p.eps, o);
    *reinterpret_cast<uint4*>(sQw + (2 * t + half) * kLd + sub * 8) = pack_bf16x8(o);
  }
  cp_async_wait<0>();
  __syncthreads();

  uint32_t acc[16][2];  // the bf16 sum over adapters, packed pairs: [dim tile j][row lane/4, row lane/4 + 8], from +0
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j][0] = acc[j][1] = 0u;

  for (int a = 0; a < p.n_adapters; ++a) {
    const int n_keys = p.n_keys[a];
    float o[16][4];
#pragma unroll
    for (int j = 0; j < 16; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows lane/4 and lane/4 + 8 of this warp's 16
    for (int kt = 0; kt < n_keys; kt += kBK) {
      const int kvalid = n_keys - kt;  // keys of this tile at column < kvalid are real
      const __nv_bfloat16* tK = sK + (p.smem_row0[a] + kt) * kLd;
      const __nv_bfloat16* tV = sV + (p.smem_row0[a] + kt) * kLd;
      // S = Q K^T : 16 x 64 per warp; key tiles wholly past the keys are not computed (masked below)
      float s[8][4];
#pragma unroll
      for (int n = 0; n < 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        uint32_t qf[4];
        ldsm_x4(qf, sQw + (lane & 15) * kLd + ks * 16 + (lane >> 4) * 8);
#pragma unroll
        for (int n = 0; n < 8; ++n) {
          if (n * 8 < kvalid) {
            uint32_t b[2];
            ldsm_x2(b, tK + (n * 8 + (lane & 7)) * kLd + ks * 16 + ((lane >> 3) & 1) * 8);
            mma_bf16(s[n], qf, b);
          }
        }
      }
      // mask, online softmax in base 2 with the scale folded in
      float mx0 = m0, mx1 = m1;
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const int c = n * 8 + (lane & 3) * 2;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float x = s[n][e] * p.scale_log2;
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
      uint32_t pf[4][4];  // P rounded to bf16: the A operand of the four 16-key k-steps
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const float p0 = exp2f(s[n][0] - mx0), p1 = exp2f(s[n][1] - mx0);
        const float p2 = exp2f(s[n][2] - mx1), p3 = exp2f(s[n][3] - mx1);
        rs0 += p0 + p1;
        rs1 += p2 + p3;
        pf[n >> 1][(n & 1) * 2 + 0] = pack_bf16x2(p0, p1);
        pf[n >> 1][(n & 1) * 2 + 1] = pack_bf16x2(p2, p3);
      }
      l0 = l0 * c0 + rs0;
      l1 = l1 * c1 + rs1;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        o[j][0] *= c0, o[j][1] *= c0, o[j][2] *= c1, o[j][3] *= c1;
      }
      // O += P V : k = the tile's keys in 16-key steps, n = 128 (16 tiles of 8)
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        if (ks * 16 < kvalid) {
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            uint32_t b[2];
            ldsm_x2_t(b, tV + (ks * 16 + (lane & 15)) * kLd + j * 8);
            mma_bf16(o[j], pf[ks], b);
          }
        }
      }
    }
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      l0 += __shfl_xor_sync(0xffffffffu, l0, off);
      l1 += __shfl_xor_sync(0xffffffffu, l1, off);
    }
    // acc = bf16(acc + bf16(scale * bf16(o / l)))
    const float i0 = 1.f / l0, i1 = 1.f / l1, sc = p.scale[a];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float y0 = round_bf16(o[j][0] * i0), y1 = round_bf16(o[j][1] * i0);
      const float y2 = round_bf16(o[j][2] * i1), y3 = round_bf16(o[j][3] * i1);
      acc[j][0] = pack_bf16x2(__fadd_rn(bf16_lo(acc[j][0]), round_bf16(__fmul_rn(sc, y0))),
                              __fadd_rn(bf16_hi(acc[j][0]), round_bf16(__fmul_rn(sc, y1))));
      acc[j][1] = pack_bf16x2(__fadd_rn(bf16_lo(acc[j][1]), round_bf16(__fmul_rn(sc, y2))),
                              __fadd_rn(bf16_hi(acc[j][1]), round_bf16(__fmul_rn(sc, y3))));
    }
  }

  // out: through the warp's own Q rows (no other warp reads them), then one 16-byte store per (row, lane of the half-warp)
  __syncwarp();
  const int g = lane >> 2, t2 = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    *reinterpret_cast<uint32_t*>(sQw + g * kLd + j * 8 + t2) = acc[j][0];
    *reinterpret_cast<uint32_t*>(sQw + (g + 8) * kLd + j * 8 + t2) = acc[j][1];
  }
  __syncwarp();
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const int rl = 2 * t + half;
    const int64_t r = row0 + warp * 16 + rl;
    if (r < p.rows)
      ptx::st_na_v4(p.out + r * p.ldo + h * 128 + sub * 8, *reinterpret_cast<const uint4*>(sQw + rl * kLd + sub * 8));
  }
}

}  // namespace mc

int32_t mc_ip_attn(const void* q, int64_t ldq, int64_t rows, int32_t heads, const float* w, float eps, const void* kv, int64_t ldkv,
                   const int32_t* n_keys, const float* scales, int32_t n_adapters, void* out, int64_t ldo, void* stream) {
  using namespace mc::ip;
  MC_CHECK_ARG(q && w && kv && n_keys && scales && out, "mc_ip_attn: null pointer");
  MC_CHECK_ARG(rows >= 1 && heads >= 1 && heads <= 65535, "mc_ip_attn: rows=%lld heads=%d", static_cast<long long>(rows), heads);
  MC_CHECK_ARG(ldq % 8 == 0 && ldq >= static_cast<int64_t>(heads) * 128 && ldo % 8 == 0 && ldo >= static_cast<int64_t>(heads) * 128 &&
                   ldkv % 8 == 0 && ldkv >= static_cast<int64_t>(heads) * 256,
               "mc_ip_attn: ldq=%lld ldo=%lld (multiples of 8, >= heads*128) ldkv=%lld (multiple of 8, >= heads*256)",
               static_cast<long long>(ldq), static_cast<long long>(ldo), static_cast<long long>(ldkv));
  MC_CHECK_ARG(mc::aligned16(q) && mc::aligned16(kv) && mc::aligned16(out) && mc::aligned16(w), "mc_ip_attn: q, w, kv, out must be 16-byte aligned");
  MC_CHECK_ARG(n_adapters >= 1 && n_adapters <= kMaxAdapters, "mc_ip_attn: n_adapters=%d outside [1, %d]", n_adapters, kMaxAdapters);
  MC_CHECK_ARG((rows + kBQ - 1) / kBQ <= 0x7fffffff, "mc_ip_attn: rows=%lld exceed one grid dimension", static_cast<long long>(rows));
  Args p{};
  p.q = static_cast<const __nv_bfloat16*>(q);
  p.ldq = ldq, p.rows = rows, p.heads = heads, p.w = w, p.eps = eps;
  p.kv = static_cast<const __nv_bfloat16*>(kv), p.ldkv = ldkv;
  p.out = static_cast<__nv_bfloat16*>(out), p.ldo = ldo;
  p.scale_log2 = 1.4426950408889634f / sqrtf(128.0f);
  p.n_adapters = n_adapters;
  int kv_rows = 0, key_rows = 0;
  for (int a = 0; a < n_adapters; ++a) {
    MC_CHECK_ARG(n_keys[a] >= 1, "mc_ip_attn: adapter %d has %d keys", a, n_keys[a]);
    MC_CHECK_ARG(n_keys[a] <= kMaxKeys && key_rows + pad16(n_keys[a]) <= kMaxKeys,
                 "mc_ip_attn: the keys of adapters 0..%d, each count rounded up to 16, exceed the %d key rows per head that shared "
                 "memory holds", a, kMaxKeys);
    p.n_keys[a] = n_keys[a], p.kv_row0[a] = kv_rows, p.smem_row0[a] = key_rows, p.scale[a] = scales[a];
    kv_rows += n_keys[a];
    key_rows += pad16(n_keys[a]);
  }
  p.key_rows = key_rows;
  static mc::PerDeviceOnce once;
  int32_t rc = mc::set_max_smem_once(mc::ip_attn_kernel, smem_bytes(kMaxKeys), once, "cudaFuncSetAttribute(ip_attn smem)");
  if (rc) return rc;
  const dim3 grid(static_cast<unsigned>((rows + kBQ - 1) / kBQ), heads);
  mc::ip_attn_kernel<<<grid, kThreads, smem_bytes(key_rows), static_cast<cudaStream_t>(stream)>>>(p);
  MC_CHECK_LAUNCH("ip_attn_kernel launch");
  return MC_OK;
}
