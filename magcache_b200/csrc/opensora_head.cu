// Open-Sora 1.2's final layer as ONE streaming pass over the B*N x D bf16 rows — T2IFinalLayer
// (videosys/models/transformers/open_sora_transformer_3d.py:50-86: LayerNorm, t2i_modulate, Linear(D -> 32)) and `unpatchify`
// (:625-647) — optionally with the cache hit in front of it (`x = x0 + residual`, eval/magcache/experiments/opensora.py:344) and
// the sampler's CFG combine + Euler update behind it (videosys/schedulers/scheduling_rflow_open_sora.py:244-251).
//
// Every value is the one the op chain of OpenSoraEngine.head writes (mc_cache_hit_add -> mc_ln_modulate mode 2 -> mc_gemm_bf16
// with MC_EPI_BIAS_BF16 -> permute / crop / .float()): the hit sum is bf16(x0 + res); LayerNorm + t2i_modulate go through the
// same per-row code (rowwise.cuh); the projection issues the GEMM's own instruction, wgmma m64n128k16, over K in the GEMM's order
// with the same zero padding of K, so every output feature sees the same accumulation (for N = 32 mc_gemm_bf16 runs its 128-wide
// tile on a B operand whose rows 32-127 are TMA zero fill; an output column depends only on its own B row, so here rows 32-127
// are whatever follows the weight in shared memory and columns 32-127 of the accumulator are dropped).
//
// One CTA per SM walks 64-row tiles. final_layer.linear.weight stays in shared memory for the whole launch (32 x D bf16, 72 KB at
// D = 1152) next to the bf16 operand tile of the current 64 rows (144 KB): that leaves no room for a staging ring, so the eight
// warps load their rows straight from global memory (one warp per row, like mc_ln_modulate mode 2, two rows' loads in flight per
// warp, one on a hit), normalise and modulate them in registers and write the swizzled operand tile; warpgroup 0 then issues the
// 4 * D / 64 wgmmas and runs the epilogue from its accumulator registers while warpgroup 1 starts on the next tile.
//
// Step mode: rows [0, B/2 N) are the conditional samples and [B/2 N, B N) the unconditional ones (`torch.cat([z, z], 0)`, :238).
// A tile is the same 64 token positions of both halves, the conditional rows first: their prediction stays in the registers of
// the thread that also holds the matching unconditional value, and only the velocity channels (the first C/2 of the C = 8, the
// `chunk(2, dim=1)[0]` of :244) leave the kernel, as z_out = z + (u + g (c - u)) dt with every operation rounded on its own.
#include "common.cuh"
#include "ptx.cuh"
#include "rowwise.cuh"

namespace mc {
namespace osh {
constexpr int kRows = 64;         // rows of a tile: one m64 wgmma
constexpr int kKC = 64;           // K columns per 128-byte swizzled operand row
constexpr int kOut = 32;          // Linear outputs: patch (1, 2, 2) x C = 8 channels
constexpr int kC = 8;
constexpr int kMaxCols = 1152;    // 18 K chunks: W 72 KB + operand tile 144 KB
constexpr int kG = 5;             // 8-element groups per lane: cols <= 32 * 8 * kG
constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kWChunk = kOut * 128;   // 4 KB: W rows of one K chunk
constexpr int kAChunk = kRows * 128;  // 8 KB: operand rows of one K chunk
constexpr int kBSpan = 128 * 128;     // 16 KB: what one n128 B descriptor reads from its chunk on

// Byte offset of 16-byte piece `piece` of row r inside a K-major, 128-byte swizzled tile (8-row groups 1024 B apart).
__device__ __forceinline__ uint32_t sw128(int r, int piece) {
  return static_cast<uint32_t>((r >> 3) * 1024 + (r & 7) * 128 + ((piece ^ (r & 7)) << 4));
}
inline int smem_bytes(int cols) {
  const int nkc = (cols + kKC - 1) / kKC;
  const int a = nkc * kAChunk;
  return nkc * kWChunk + (a > kBSpan - kWChunk ? a : kBSpan - kWChunk);  // the last W chunk's descriptor reads 16 KB on
}
}  // namespace osh

struct OsHeadParams {
  const __nv_bfloat16* x;    // [B N, cols]: the stream, or x0 on a cache hit
  const __nv_bfloat16* res;  // [B N, cols] cached residual (hit)
  const __nv_bfloat16* w;    // [32, cols] final_layer.linear.weight
  const float* bias;         // [32] bf16 values
  const float* mod;          // [B, 2, cols] shift | scale per sample, bf16 values
  int64_t N;                 // rows per sample: T H W
  int B, cols, T, H, W, Hx, Wx;
  int T_out;                 // frames of the output (and z) tensor: T, or more when `out` / `z` point at a frame window of it
  float eps;
  const float* z;            // step mode: [B/2, C/2, T, Hx, Wx]; nullptr: plain mode
  const float* dt;           // step mode: [B/2]
  float g;
  float* out;                // plain: [B, C, T_out, Hx, Wx]; step: [B/2, C/2, T_out, Hx, Wx] (may alias z)
};

template <bool HIT>
__global__ void __launch_bounds__(osh::kThreads, 1) opensora_head_kernel(const OsHeadParams p) {
  using namespace osh;
  constexpr int kRB = HIT ? 1 : 2;  // rows whose loads a warp has in flight at once (a hit loads two inputs per row)
  extern __shared__ __align__(1024) uint8_t smem[];
  const int nkc = (p.cols + kKC - 1) / kKC;
  uint8_t* ws = smem;                  // W, chunk kc at kc * kWChunk
  uint8_t* as = smem + nkc * kWChunk;  // operand tile, chunk kc at kc * kAChunk
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups = p.cols >> 3, groups_pad = nkc * 8;

  // W into shared memory, its K padding zero; the operand tile's K padding is zeroed once (the rows never write it)
  for (int i = threadIdx.x; i < kOut * groups_pad; i += kThreads) {
    const int r = i / groups_pad, g = i - r * groups_pad;
    const uint4 v = g < groups ? *reinterpret_cast<const uint4*>(p.w + static_cast<int64_t>(r) * p.cols + g * 8) : make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4*>(ws + (g >> 3) * kWChunk + sw128(r, g & 7)) = v;
  }
  const int pad = groups_pad - groups;
  for (int i = threadIdx.x; i < kRows * pad; i += kThreads) {
    const int r = i / pad, g = groups + (i - r * pad);
    *reinterpret_cast<uint4*>(as + (g >> 3) * kAChunk + sw128(r, g & 7)) = make_uint4(0, 0, 0, 0);
  }

  const bool step = p.z != nullptr;
  const int64_t span = step ? (p.B / 2) * p.N : p.B * p.N;  // rows of one pass
  const int64_t n_tiles = (span + kRows - 1) / kRows;
  const float inv_n = 1.0f / static_cast<float>(p.cols);
  const int64_t S = static_cast<int64_t>(p.H) * p.W;
  const int64_t plane = static_cast<int64_t>(p.Hx) * p.Wx;
  float keep[16];  // step mode: bf16(acc + bias) of the conditional rows, features < 32 of this thread's fragment
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    for (int pass = 0; pass < (step ? 2 : 1); ++pass) {
      const int64_t r0 = pass * span + tile * kRows, r_end = (pass + 1) * span;
      // ---- LayerNorm + t2i_modulate of the tile's rows into the operand tile (warp per row; each warp issues the loads of kRB
      // rows before it reduces the first, so that enough bytes are in flight with one CTA per SM)
      for (int rt0 = warp; rt0 < kRows; rt0 += kWarps * kRB) {
        uint4 raw[kRB][kG], rawr[HIT ? kRB : 1][kG];
#pragma unroll
        for (int u = 0; u < kRB; ++u) {
          const int64_t row = r0 + rt0 + u * kWarps;
#pragma unroll
          for (int i = 0; i < kG; ++i) {
            const int g = lane + i * 32;
            if (row < r_end && g < groups) {
              raw[u][i] = ptx::ld_nc_v4(p.x + row * p.cols + g * 8);
              if constexpr (HIT) rawr[u][i] = ptx::ld_nc_v4(p.res + row * p.cols + g * 8);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < kRB; ++u) {
          const int rt = rt0 + u * kWarps;
          const int64_t row = r0 + rt;
          if (row >= r_end) break;
          float v[kG][8];
#pragma unroll
          for (int i = 0; i < kG; ++i) {
            if (lane + i * 32 < groups) {
              unpack_bf16x8(raw[u][i], v[i]);
              if constexpr (HIT) {
                float r8[8];
                unpack_bf16x8(rawr[u][i], r8);
#pragma unroll
                for (int j = 0; j < 8; ++j) v[i][j] = round_bf16(v[i][j] + r8[j]);  // `x0 + residual` as a bf16 tensor op
              }
            }
          }
          float mean;
          const float rstd = ln_rstd<kG>(v, lane, 32, groups, inv_n, p.eps, WarpReduce(), mean);
          const float* sh = p.mod + (row / p.N) * 2 * p.cols;
#pragma unroll
          for (int i = 0; i < kG; ++i) {
            const int g = lane + i * 32;
            if (g < groups) {
              float o[8];
              t2i_modulate8(v[i], mean, rstd, sh + p.cols + g * 8, sh + g * 8, o);
              *reinterpret_cast<uint4*>(as + (g >> 3) * kAChunk + sw128(rt, g & 7)) = pack_bf16x8(o);
            }
          }
        }
      }
      ptx::fence_proxy_async_smem();
      __syncthreads();
      float acc[64];  // one per pass: not live while the rows are converted
      // ---- the projection, K in the GEMM's order
      if (warp < 4) {
        const uint64_t da = ptx::gmma_desc_sw128_kmajor(ptx::smem_u32(as)), db = ptx::gmma_desc_sw128_kmajor(ptx::smem_u32(ws));
        ptx::wgmma_fence();
        for (int kc = 0; kc < nkc; ++kc) {
#pragma unroll
          for (int k = 0; k < kKC / 16; ++k)
            ptx::wgmma_m64n128k16_ss(acc, da + (kc * kAChunk >> 4) + 2 * k, db + (kc * kWChunk >> 4) + 2 * k, (kc | k) != 0 ? 1u : 0u);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::fence_regs(acc);
      }
      __syncthreads();  // the operand tile is free for the next pass
      if (warp >= 4) continue;
      // ---- epilogue: bf16(acc + bias) -> unpatchify + crop. Fragment: rows 16 wq + lane / 4 (+ 8), feature 8 i + 2 (lane % 4) (+ 1)
      // = (2 hp + wp) C + c, i.e. i = 2 hp + wp and c = 2 (lane % 4) (+ 1).
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int rr = (warp & 3) * 16 + (lane >> 2) + 8 * h;
        const int64_t row = r0 + rr;
        const bool live = row < r_end;
        const int64_t q = row - pass * span;  // conditional row (step), or the row
        const int64_t b = q / p.N, n = q - b * p.N;
        const int t = static_cast<int>(n / S), s = static_cast<int>(n - t * S);
        const int hh = s / p.W, ww = s - hh * p.W;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int yy = 2 * hh + (i >> 1), xx = 2 * ww + (i & 1);
          const bool in = live && yy < p.Hx && xx < p.Wx;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = 2 * (lane & 3) + e, j = 8 * i + c;
            const float y = round_bf16(acc[4 * i + 2 * h + e] + __ldg(p.bias + j));
            if (!step) {
              if (in) p.out[((b * kC + c) * p.T_out + t) * plane + static_cast<int64_t>(yy) * p.Wx + xx] = y;
            } else if (pass == 0) {
              keep[4 * i + 2 * h + e] = y;
            } else if (in && c < kC / 2) {
              const int64_t o = ((b * (kC / 2) + c) * p.T_out + t) * plane + static_cast<int64_t>(yy) * p.Wx + xx;
              const float vel = __fadd_rn(y, __fmul_rn(p.g, __fsub_rn(keep[4 * i + 2 * h + e], y)));  // uncond + g * (cond - uncond)
              p.out[o] = __fadd_rn(p.z[o], __fmul_rn(vel, __ldg(p.dt + b)));                         // z + v_pred * dt
            }
          }
        }
      }
    }
  }
}

}  // namespace mc

namespace {
int32_t opensora_head_launch(const char* fn, const void* x, const void* res_or_null, int32_t B, int32_t T, int32_t H, int32_t W,
                             int32_t cols, const float* mod, const void* w, const float* bias, int32_t C_out, float eps, int32_t Hx,
                             int32_t Wx, int32_t T_out, const float* z_or_null, const float* dt, float guidance_scale, float* out,
                             void* stream) {
  using namespace mc;
  MC_CHECK_ARG(x && mod && w && bias && out, "%s: null pointer", fn);
  MC_CHECK_ARG(C_out == osh::kC, "%s: built for patch (1, 2, 2) x 8 output channels (32 features), got C_out=%d", fn, C_out);
  MC_CHECK_ARG(cols >= 8 && cols % 8 == 0 && cols <= osh::kMaxCols, "%s: cols=%d must be a multiple of 8 in [8, %d]", fn, cols,
               osh::kMaxCols);
  MC_CHECK_ARG(B >= 1 && T >= 1 && H >= 1 && W >= 1, "%s: bad shape B=%d T=%d H=%d W=%d", fn, B, T, H, W);
  MC_CHECK_ARG(T_out >= T, "%s: the output holds %d frames, fewer than the %d of x", fn, T_out, T);
  MC_CHECK_ARG(Hx >= 2 * H - 1 && Hx <= 2 * H && Wx >= 2 * W - 1 && Wx <= 2 * W,
               "%s: crop %d x %d does not match the %d x %d patch grid", fn, Hx, Wx, H, W);
  MC_CHECK_ARG(aligned16(x) && (res_or_null == nullptr || aligned16(res_or_null)) && aligned16(w) && aligned16(mod),
               "%s: x / res / w / mod must be 16-byte aligned", fn);
  MC_CHECK_ARG(z_or_null == nullptr || (B % 2 == 0 && dt != nullptr), "%s: step mode needs an even B (cond | uncond halves) and dt", fn);
  OsHeadParams p{};
  p.x = static_cast<const __nv_bfloat16*>(x);
  p.res = static_cast<const __nv_bfloat16*>(res_or_null);
  p.w = static_cast<const __nv_bfloat16*>(w);
  p.bias = bias, p.mod = mod;
  p.N = static_cast<int64_t>(T) * H * W;
  p.B = B, p.cols = cols, p.T = T, p.H = H, p.W = W, p.Hx = Hx, p.Wx = Wx;
  p.T_out = T_out;
  p.eps = eps;
  p.z = z_or_null, p.dt = dt, p.g = guidance_scale;
  p.out = out;
  const int64_t span = z_or_null ? (B / 2) * p.N : B * p.N;
  const int64_t tiles = (span + osh::kRows - 1) / osh::kRows;
  const int grid = static_cast<int>(tiles < num_sms() ? tiles : num_sms());
  const int smem = osh::smem_bytes(cols);
  static PerDeviceOnce once_hit, once_stream;
  const int32_t rc = res_or_null ? set_max_smem_once(opensora_head_kernel<true>, osh::smem_bytes(osh::kMaxCols), once_hit, "cudaFuncSetAttribute(opensora_head smem)")
                                 : set_max_smem_once(opensora_head_kernel<false>, osh::smem_bytes(osh::kMaxCols), once_stream, "cudaFuncSetAttribute(opensora_head smem)");
  if (rc) return rc;
  if (res_or_null)
    opensora_head_kernel<true><<<grid, osh::kThreads, smem, static_cast<cudaStream_t>(stream)>>>(p);
  else
    opensora_head_kernel<false><<<grid, osh::kThreads, smem, static_cast<cudaStream_t>(stream)>>>(p);
  MC_CHECK_LAUNCH("opensora_head_kernel launch");
  return MC_OK;
}
}  // namespace

extern "C" int32_t mc_opensora_head(const void* x, const void* res_or_null, int32_t B, int32_t T, int32_t H, int32_t W, int32_t cols,
                                    const float* mod, const void* w, const float* bias, int32_t C_out, float eps, int32_t Hx, int32_t Wx,
                                    const float* z_or_null, const float* dt, float guidance_scale, float* out, void* stream) {
  return opensora_head_launch("mc_opensora_head", x, res_or_null, B, T, H, W, cols, mod, w, bias, C_out, eps, Hx, Wx, T, z_or_null, dt,
                              guidance_scale, out, stream);
}

// The sequence-parallel final layer: x holds one rank's T frames of every sample, out / z point at frame t0 of tensors of T_out
// frames, so each rank writes its own frame window of the full-size prediction (or updated latent) in place.
extern "C" int32_t mc_opensora_head_frames(const void* x, const void* res_or_null, int32_t B, int32_t T, int32_t H, int32_t W,
                                           int32_t cols, const float* mod, const void* w, const float* bias, int32_t C_out, float eps,
                                           int32_t Hx, int32_t Wx, int32_t T_out, const float* z_or_null, const float* dt,
                                           float guidance_scale, float* out, void* stream) {
  return opensora_head_launch("mc_opensora_head_frames", x, res_or_null, B, T, H, W, cols, mod, w, bias, C_out, eps, Hx, Wx, T_out,
                              z_or_null, dt, guidance_scale, out, stream);
}
