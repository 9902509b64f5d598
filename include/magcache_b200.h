/*
 * magcache_b200 — C ABI of the H100-native MagCache hot path (libmagcache_b200.so).
 *
 * Every entry point takes plain pointers and sizes (no torch types). Device pointers are raw CUDA device
 * addresses (tensor.data_ptr()); `stream` is a cudaStream_t passed as void* (torch.cuda.current_stream().cuda_stream).
 * All functions return 0 on success and a negative MC_ERR_* code on failure; mc_last_error() returns a
 * thread-local, human-readable description of the last failure. Nothing here falls back to the CPU:
 * device entry points fail with MC_ERR_CUDA if no sm_90 device/driver is usable.
 *
 * Each declaration cites the reference statement(s) it replaces (paths relative to the Zehong-Ma/MagCache tree).
 */
#ifndef MAGCACHE_B200_H_
#define MAGCACHE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MC_OK 0
#define MC_ERR_INVALID (-1) /* bad argument (null pointer, bad dtype, shape/alignment not supported) */
#define MC_ERR_CUDA (-2)    /* CUDA runtime/driver error (message carries cudaGetErrorString) */
#define MC_ERR_STATE (-3)   /* controller asked to re-use a residual that was never stored, cnt out of range, ... */

/* element types of device buffers */
#define MC_F32 0
#define MC_BF16 1

const char* mc_last_error(void);
int32_t mc_abi_version(void); /* bumped whenever a signature in this header changes */

/* ------------------------------------------------------------------------------------------------------------
 * Host logic (float64 / int, bit-exact with the reference's Python/numpy arithmetic)
 * ---------------------------------------------------------------------------------------------------------- */

/* nearest_interp(src_array, target_length)          MagCache4Wan2.1/magcache_generate.py:27-34
 * (identical copies: MagCache4FLUX/magcache_flux.py:12-19, MagCache4HunyuanVideo/magcache_sample_video.py:20-27).
 * idx = round_half_even(arange(T) * (L-1)/(T-1)); T == 1 -> src[L-1]. `dst` has T entries. */
int32_t mc_nearest_interp(const double* src, int32_t L, double* dst, int32_t T);

/* Qwen-Image's variant (MagCache4QwenImage/magcache_generate.py:14-21): idx = round_half_even(np.linspace(0, L-1, T));
 * L == T returns a copy; T == 1 picks src[0] (the Wan form picks src[L-1]). */
int32_t mc_nearest_interp_linspace(const double* src, int32_t L, double* dst, int32_t T);

/* Per-CFG-branch form used by Wan (magcache_generate.py:915-919): de-interleave [0::2]/[1::2], interpolate each
 * to `steps`, re-interleave. src has 2*L_half entries, dst 2*steps entries. */
int32_t mc_nearest_interp_cfg(const double* src, int32_t L_total, double* dst, int32_t steps);

/* Controller variants (SURVEY Appendix A). */
#define MC_CMP_LT 0            /* err <  thresh : Wan2.1 magcache_generate.py:286 */
#define MC_CMP_LE 1            /* err <= thresh : FLUX magcache_flux.py:332, Hunyuan magcache_sample_video.py:96 */
#define MC_RETAIN_FLOOR 0      /* cnt >= int(num_steps*R)       Wan :279, Hunyuan :90 */
#define MC_RETAIN_HALF_UP 1    /* cnt >= int(R*num_steps + 0.5) FLUX :327 */
#define MC_RETAIN_CEIL 2       /* cnt >= ceil(R*num_steps)      OmniGen2 magcache_utils.py:343 */
/* Wan2.2 two-expert windows, MagCache4Wan2.2/magcache_generate.py:294-303 (split_step = 2*high_noise_steps, cnt spans both experts).
 * The reference keeps cnt in an int64 torch tensor, so its `cnt <= python_float` comparison happens in float32: reproduced. */
#define MC_RETAIN_WAN22_T2V 3  /* skip-disabled if cnt < int(split*R) or (split <= cnt <= (n-split)*R + split) */
#define MC_RETAIN_WAN22_I2V 4  /* skip-disabled if cnt < int(split + (n-split)*R) */
#define MC_RETAIN_EXPLICIT 5   /* cnt >= split_step: Open-Sora `self.t >= self.skip_time`, eval/magcache/experiments/opensora.py:297, :424 */
/* mc_ctrl_config.flags */
#define MC_CTRL_SIGNED_ERR 1     /* err += 1 - ratio (no abs): eval/magcache/experiments/opensora.py:301 */
#define MC_CTRL_RESET_AT_ZERO 2  /* accumulators re-initialised whenever a call sees cnt == 0: MagCache4FramePack/magcache_demo_gradio.py:253-256 */
#define MC_CTRL_RATIO_VETO 4     /* skip only while |1 - mag_ratios[.]| <= ratio_veto: magcache_demo_gradio.py:265 */
#define MC_CTRL_WRAP_KEEPS_ACC 8 /* at cnt >= num_steps only the counter is reset, the accumulators carry over into the next sample:
                                    MagCache4QwenImage/magcache_generate.py:243-244 (Wan2.1 :306-311, FLUX :432-436, ... reset all) */

typedef struct mc_ctrl_config {
  int32_t num_steps;       /* forward calls per video: 2*sample_steps for CFG models (Wan :899), steps otherwise */
  int32_t branches;        /* 1 = scalar state (FLUX/Hunyuan), 2 = state per CFG branch, branch = cnt % 2 (Wan :281-288) */
  int32_t K;               /* max consecutive skips (accumulated_steps <= K) */
  int32_t cmp;             /* MC_CMP_* */
  int32_t retention_mode;  /* MC_RETAIN_* */
  int32_t veto_index;      /* -1 = none. FLUX :332: never skip when round_half_even(cnt*((veto_base-1)/(num_steps-1))) == veto_index */
  int32_t veto_base;       /* 28 for FLUX */
  int32_t split_step;      /* MC_RETAIN_WAN22_*: calls made to the high-noise expert per video (2*high_noise_steps);
                              MC_RETAIN_EXPLICIT: first call allowed to skip; else unused */
  int32_t table_offset;    /* the ratio of call cnt is mag_ratios[cnt - table_offset]: 0 everywhere except the paper-evaluation forwards
                              (`self.ratio[self.t-10]` eval/magcache/experiments/Wan2.1_EVAL/wan_magcache.py:775; `ratio[t-1]` opensora.py:298) */
  int32_t min_cnt;         /* additionally require cnt >= min_cnt (FramePack `and self.cnt>=1`, magcache_demo_gradio.py:259); 0 = off */
  int32_t flags;           /* MC_CTRL_* bits */
  int32_t reserved;        /* must be 0 */
  double thresh;           /* magcache_thresh */
  double retention_ratio;
  double ratio_veto;       /* with MC_CTRL_RATIO_VETO (FramePack: 0.06); a zero-filled tail of this struct means "Wan2.1 behaviour" */
  const double* mag_ratios; /* [num_steps - table_offset], already interpolated; borrowed for the duration of the call / handle */
} mc_ctrl_config;

typedef struct mc_ctrl_state { /* mirrors the reference's class attributes (magcache_generate.py:897-906) */
  int32_t cnt;
  int32_t accumulated_steps[2];
  int32_t pad;
  double accumulated_ratio[2];
  double accumulated_err[2];
} mc_ctrl_state;

/* One controller decision = the `if self.cnt >= int(self.num_steps*self.retention_ratio):` statement,
 * magcache_generate.py:279-292 (FLUX :327-338, Hunyuan :90-102). Updates `st` in place, writes 1/0 to *skip.
 * Does NOT advance cnt (see mc_ctrl_advance). */
int32_t mc_ctrl_decide(const mc_ctrl_config* cfg, mc_ctrl_state* st, int32_t* skip);
/* `self.cnt += 1; if self.cnt >= self.num_steps: reset`   magcache_generate.py:306-311. */
int32_t mc_ctrl_advance(const mc_ctrl_config* cfg, mc_ctrl_state* st);
/* Whole schedule: run `calls` decisions from a fresh state, mask[i] in {0,1}. */
int32_t mc_ctrl_mask(const mc_ctrl_config* cfg, int32_t calls, uint8_t* mask);
/* Reject configurations the reference would crash on (Appendix A quirk 4: cnt 0 eligible with an empty cache). */
int32_t mc_ctrl_validate(const mc_ctrl_config* cfg);

/* Handle form of the same controller (SURVEY §8b: create / step / reset / destroy) for hosts that prefer an opaque object to the
 * two structs: the handle owns a COPY of the config and of the table and the state of one model instance.
 *   mc_ctrl_create  validates (mc_ctrl_validate) and returns NULL + mc_last_error() on a bad configuration;
 *   mc_ctrl_step    = decide + advance for the call the handle's own counter points at (magcache_generate.py:277-292 + :306-311);
 *                     *cnt_out (optional) receives the counter AFTER the call;
 *   mc_ctrl_reset   = what `__class__.cnt = 0` between prompts intends (magcache_flux.py:478): cnt 0, fresh accumulators;
 *   mc_ctrl_state_of exposes the state struct (borrowed pointer, valid until destroy). */
typedef struct mc_ctrl mc_ctrl;
mc_ctrl* mc_ctrl_create(const mc_ctrl_config* cfg, int32_t initial_accumulated_steps);
int32_t mc_ctrl_step(mc_ctrl* h, int32_t* skip, int32_t* cnt_out);
int32_t mc_ctrl_reset(mc_ctrl* h);
const mc_ctrl_state* mc_ctrl_state_of(const mc_ctrl* h);
void mc_ctrl_destroy(mc_ctrl* h);

/* ------------------------------------------------------------------------------------------------------------
 * Residual-cache kernels (HBM-bound)
 * ---------------------------------------------------------------------------------------------------------- */

/* cache-hit branch  `x = x + residual_x`            magcache_generate.py:295 (FLUX :340, Hunyuan :104).
 * out[i] = x[i] + r[i], computed in fp32, rounded to out_dtype (torch type promotion: bf16+fp32->fp32, bf16+bf16->bf16).
 * out must not overlap x or r (inputs are streamed through the non-coherent path). n = element count. */
int32_t mc_cache_hit_add(const void* x, int32_t x_dtype, const void* r, int32_t r_dtype, void* out, int32_t out_dtype,
                         int64_t n, void* stream);

/* cache-miss epilogue `residual_x = x - ori_x`      magcache_generate.py:299 (FLUX :426, Hunyuan :140). */
int32_t mc_residual_sub(const void* x_out, int32_t xo_dtype, const void* x_in, int32_t xi_dtype, void* r, int32_t r_dtype,
                        int64_t n, void* stream);

/* classifier-free-guidance combine of the caller loop (SURVEY §8f rank 1)
 * `noise_pred = noise_pred_uncond + guide_scale * (noise_pred_cond - noise_pred_uncond)`
 * eval/magcache/experiments/Wan2.1_EVAL/wan_magcache.py:301-302 — one pass, fp32, each operation rounded like torch eager. */
int32_t mc_cfg_combine(const float* cond, const float* uncond, float guide_scale, float* out, int64_t n, void* stream);

/* CFG combine + the scheduler's latent update in ONE pass (SURVEY §8f rank 1; caller loop wan_magcache.py:301-310:
 * `noise_pred = ...; temp_x0 = sample_scheduler.step(noise_pred, t, latents)`). The flow-matching solvers the reference uses
 * (FlowUniPC, FlowDPM++ — upstream, not in the reference tree — and plain Euler) all compute
 *     v   = uncond + guide_scale * (cond - uncond)
 *     out = coef_x * x + coef_v * v + sum_{i < n_hist} coef_h[i] * hist[i]        (Euler: coef_x = 1, coef_v = sigma_next - sigma)
 *     x0  = x - sigma * v                         (written when x0_out != NULL: the x0-prediction the multistep solvers store)
 * with scalar coefficients computed on the host. fp32; every product / sum rounded separately in the order written (bit-equal
 * to the torch eager chain). out may alias x (in-place update); hist: device pointers, n_hist <= 4. */
int32_t mc_cfg_step(const float* cond, const float* uncond, float guide_scale, const float* x, float coef_x, float coef_v,
                    const float* const* hist, const float* coef_h, int32_t n_hist, float sigma, float* out, float* x0_out, int64_t n,
                    void* stream);

/* FP8 weight dequantisation (MagCache4HunyuanVideo/README.md:76-96, `--use-fp8 --dit-weight ..._fp8.pt`): upstream's
 * `fp8_linear_forward` [EXT hyvideo/modules/fp8_optimization.py] forms `qdata.to(bf16) * scale.to(bf16)` (fp8_activation_dequant)
 * before every F.linear of a double / single block.
 *   out[r, c] = bf16_rn(float(q[r, c]) * float(scale[r]))   q float8_e4m3fn [rows, cols], scale bf16 [rows], out bf16 [rows, cols]
 * The scale is per row because one matrix may stack the rows of several Linears (the modulation table). Both conversions and the
 * fp32 product are exact, so the result is bit-equal to upstream's; codes 0x7F / 0xFF give NaN. Contiguous operands; 16-byte loads
 * when cols % 16 == 0 and q / out are 16-byte aligned, one element per thread otherwise. HBM-bound (3 bytes per element). */
int32_t mc_dequant_fp8_bf16(const void* q, const void* scale, void* out, int64_t rows, int32_t cols, void* stream);

/* calibration statistics                              magcache_generate.py:167-169 (one pass instead of ~7 + 3 syncs).
 * r_cur, r_prev: [rows, cols]. stats (device, 4 doubles, overwritten): sum(ratio), sum(ratio^2), sum(1-cos), rows
 * with ratio = ||r_cur[i]||2 / (||r_prev[i]||2 + denom_eps)  (denom_eps = 0 Wan :167; 1e-8 eval variant wan_magcache.py:652)
 * and cos with eps 1e-8 as F.cosine_similarity. Host side: mean = s0/n, std = sqrt((s1 - s0^2/n)/(n-1)), cos_dis = s2/n. */
int32_t mc_residual_stats(const void* r_cur, int32_t cur_dtype, const void* r_prev, int32_t prev_dtype, int64_t rows,
                          int32_t cols, double denom_eps, double* stats_dev, void* stream);

/* Fused miss epilogue for calibration runs: r = x_out - x_in, and the statistics of r against r_prev in the same pass. */
int32_t mc_residual_sub_stats(const void* x_out, int32_t xo_dtype, const void* x_in, int32_t xi_dtype, void* r,
                              const void* r_prev, int64_t rows, int32_t cols, double denom_eps, double* stats_dev,
                              void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * TeaCache comparator (SURVEY §8f rank 4: the baseline every published MagCache table is compared against)
 * eval/magcache/experiments/Wan2.1_EVAL/wan_teacache.py:533-564 (controller), :566-582 (same hit / miss branches), :899-928 (setup)
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct mc_tea_config {
  int32_t num_steps;     /* forward calls per video (2*sample_steps) */
  int32_t ret_steps;     /* calls [0, ret_steps) always compute        (:538; 1*2 or 10*2, :919/:927) */
  int32_t cutoff_steps;  /* calls [cutoff_steps, num_steps) always compute (:921/:928) */
  int32_t n_coef;        /* polynomial degree + 1, <= 8 */
  double thresh;         /* teacache_thresh */
  double coef[8];        /* np.poly1d order: highest power first (:915-926) */
} mc_tea_config;

typedef struct mc_tea_state {
  int32_t cnt;
  int32_t pad;
  double accumulated[2]; /* accumulated_rel_l1_distance_even / _odd */
} mc_tea_state;

/* *needs = 1 when the call at st->cnt consults the distance (retention / cutoff calls do not: no reduction, no host sync). */
int32_t mc_tea_needs_distance(const mc_tea_config* cfg, const mc_tea_state* st, int32_t* needs);
/* One decision (:535-564): *calc = 1 -> run the block stack, 0 -> reuse the cached residual. rel_l1 = mean|e - e_prev| / mean|e_prev|
 * of this CFG branch (ignored on retention / cutoff calls). Does not advance cnt. */
int32_t mc_tea_decide(const mc_tea_config* cfg, mc_tea_state* st, double rel_l1, int32_t* calc);
/* cnt += 1, wrapping at num_steps (:587-589; the accumulators are NOT reset at the wrap, as in the reference). */
int32_t mc_tea_advance(const mc_tea_config* cfg, mc_tea_state* st);
/* sums_dev (device, 2 doubles, overwritten) = { sum |cur - prev|, sum |prev| } over n fp32 elements — the two means of :543. */
int32_t mc_rel_l1(const float* cur, const float* prev, int64_t n, double* sums_dev, void* stream);
/* Open-Sora's TeaCache rule (eval/magcache/experiments/opensora.py:96-107), one call:
 *   forced (timestep[0] == all_timesteps[0] or == all_timesteps[-1]) -> *calc = 1, *accumulated_out = 0
 *   else accumulated += np.poly1d(coef)(rel); *calc = !(accumulated < thresh); on a compute the sum is reset to 0
 * rel is the value `.cpu().item()` returns (the bf16 quotient of the two bf16 means), ignored when forced. coef: n_coef (1..8)
 * coefficients, highest power first. float64 throughout, bit-exact with the reference. */
int32_t mc_tea_opensora_decide(int32_t forced, double rel, double accumulated, double thresh, const double* coef, int32_t n_coef,
                               int32_t* calc, double* accumulated_out);

/* ------------------------------------------------------------------------------------------------------------
 * DiT block-stack kernels (cache-miss branch `for block in self.blocks: x = block(x, **kwargs)`,
 * magcache_generate.py:297-298; block arithmetic per upstream Wan2.1 wan/modules/model.py, SURVEY Appendix B.1)
 * ---------------------------------------------------------------------------------------------------------- */

/* patch_embedding input side (magcache_generate.py:237): latent fp32 [C, F, H, W] -> token-major im2col
 * bf16 [F*(H/2)*(W/2), C*4] (column = c*4 + dh*2 + dw, the Conv3d weight's flattened (c, kt=1, kh, kw) order). */
int32_t mc_patchify(const float* latent, int32_t C, int32_t F, int32_t H, int32_t W, void* tokens_bf16, void* stream);

/* AdaLN-modulated LayerNorm: y = LN(x) * a + b, eps inside the LN, no affine in the LN itself; per-row fp32 statistics.
 *   mode 0: a = 1 + p0[scale_idx], b = p0[shift_idx]   p0 = e = modulation + e0, fp32 [k, cols]  (block norm1/norm2:
 *           `norm1(x).float() * (1 + e[1]) + e[0]`, upstream WanAttentionBlock.forward); p1 unused
 *   mode 1: a = p0, b = p1                             (norm3, elementwise affine weight / bias)
 *   mode 2: y = bf16(bf16(bf16(LN(x)) * bf16(1 + p0[scale_idx])) + p0[shift_idx])   p0 fp32 [k, cols] holding bf16 values; p1 and
 *           round_ln_to_bf16 unused. `t2i_modulate(self.norm1(x), shift, scale)` of STDiT3Block.forward
 *           (videosys/models/transformers/open_sora_transformer_3d.py:187, :248) and of T2IFinalLayer (:80), where every step is a
 *           bf16 tensor op. x and out bf16, 16-byte aligned, cols <= 2048.
 * x: [rows, cols] (fp32 or bf16); round_ln_to_bf16 != 0 reproduces `.type_as(x)` for a bf16 stream (block 0).
 * out: [rows, cols] bf16 (GEMM operand) or fp32. x/out 32-byte aligned, cols % 8 == 0, cols <= 8192. */
int32_t mc_ln_modulate(const void* x, int32_t x_dtype, int64_t rows, int32_t cols, float eps, int32_t mode,
                       const float* p0, const float* p1, int32_t scale_idx, int32_t shift_idx,
                       int32_t round_ln_to_bf16, void* out, int32_t out_dtype, void* stream);

/* Mode 2 of mc_ln_modulate (same per-row arithmetic, same output bits) fused with the input distance of Open-Sora's TeaCache
 * (eval/magcache/experiments/opensora.py:95, :102):
 *   out = t2i_modulate(spatial_blocks[0].norm1(x), shift, scale)                    `modulated_inp`
 *   sums_dev[0] += sum float(|bf16(out - prev)|),  sums_dev[1] += sum float(|prev|)  `(modulated_inp - previous_modulated_input).abs()`,
 *                                                                                    `previous_modulated_input.abs()` before `.mean()`
 * prev: the previous call's bf16 output, [rows, cols]; out may not alias x or prev. The sums are added, so per-sample launches into one
 * zeroed sums_dev give the sums over all samples. Deterministic: per-CTA partials (fp64) in partials_dev, at least
 * 2 * MC_LN_REL_L1_MAX_CTAS doubles of device scratch, then one fixed-order sum; the same inputs give the same bits on every launch.
 * x, out, prev, p0, partials_dev 16-byte aligned; cols % 8 == 0, cols <= 2048. */
#define MC_LN_REL_L1_MAX_CTAS 4096
int32_t mc_ln_t2i_modulate_rel_l1(const void* x, int64_t rows, int32_t cols, float eps, const float* p0, int32_t scale_idx,
                                  int32_t shift_idx, const void* prev, void* out, double* partials_dev, double* sums_dev,
                                  void* stream);

/* WanRMSNorm over the full model dim followed by 3-axis RoPE (rope_apply), in place on bf16 [rows, cols]:
 *   y = bf16(rope(float(bf16(x * rsqrt(mean(x^2)+eps))) * w)).  cos_sin == NULL -> no RoPE (cross-attention q/k).
 * cos_sin: fp32 [rows, head_dim] interleaved (cos, sin) per complex pair, i.e. [rows, head_dim/2, 2]; row = token. */
int32_t mc_rmsnorm_rope(void* x_bf16, int64_t ld, int64_t rows, int32_t cols, const float* w, float eps,
                        const float* cos_sin, int32_t head_dim, void* stream);
/* the same over `segs` adjacent column blocks of `cols` columns per row (q | k of the fused q|k|v projection in ONE launch):
 * x [rows, >= segs*cols] with row pitch ld, w [segs, cols]; RoPE (when cos_sin != NULL) is applied to every block. */
int32_t mc_rmsnorm_rope_segs(void* x_bf16, int64_t ld, int64_t rows, int32_t segs, int32_t cols, const float* w, float eps,
                             const float* cos_sin, int32_t head_dim, void* stream);

/* MMDiT (FLUX) attention front end [EXT diffusers FluxAttnProcessor2_0, called from MagCache4FLUX/magcache_flux.py:361-366, :413-418]:
 * per-HEAD RMSNorm (head_dim 128; y = bf16(bf16(x * rsqrt(mean x^2 + eps)) * w), w fp32 copies of the bf16 weights [128]) followed
 * by `apply_rotary_emb` on consecutive (real, imag) pairs, in place on x bf16 [rows, heads*128] (row stride ld).
 * cos_sin: fp32 [rows, 128] interleaved (cos, sin) per pair, or NULL. */
int32_t mc_rmsnorm_head_rope(void* x_bf16, int64_t ld, int64_t rows, int32_t heads, const float* w, float eps, const float* cos_sin,
                             void* stream);
/* Open-Sora 1.2 (STDiT3, head_dim 72; csrc/opensora_kernels.cu) ------------------------------------------------------------
 * q / k normalisation of OpenSoraAttention.forward (videosys/models/modules/attentions.py:71-75, `qk_norm_legacy=False`): per-head
 * LlamaRMSNorm(72) (normalization.py:17-22: y = bf16(w * bf16(x * rsqrt(mean x^2 + eps))), w fp32 copies of the bf16 weight [72]),
 * then, when cos_sin != NULL, RoPE on interleaved pairs in fp32 rounded to bf16 (rotary_embedding_torch
 * `RotaryEmbedding(72).rotate_queries_or_keys` [EXT]), in place on x bf16 [rows, heads*72] (row pitch ld % 8 == 0).
 * cos_sin: fp32 [pos_mod, 72] = (cos, sin) per pair; row r uses position (r / pos_div) % pos_mod — the frame index of a B (T S) C
 * token row with pos_div = S, pos_mod = T. */
int32_t mc_rmsnorm_head72_rope(void* x_bf16, int64_t ld, int64_t rows, int32_t heads, const float* w, float eps, const float* cos_sin,
                               int64_t pos_div, int32_t pos_mod, void* stream);
/* softmax(q k^T * scale) v, head_dim 72, over independent segments in one launch: segs_dev (device) int32 [n_segs, 4] =
 * (q_start, q_len, k_start, k_len); the q rows [q_start, q_start+q_len) attend to the k / v rows [k_start, k_start+k_len) (k_len >= 1).
 * The spatial self-attention (B*T frames of S tokens, `rearrange(x, "B (T S) C -> (B T) S C")` + OpenSoraAttention,
 * open_sora_transformer_3d.py:202-204) and the cross-attention with per-sample caption lengths (`flash_attn_varlen_func` of
 * OpenSoraMultiHeadCrossAttention.flash_attn_impl, attentions.py:136-153). max_q_len >= every q_len. Row-major bf16 views,
 * leading dimensions % 8 == 0, 16-byte aligned pointers. */
int32_t mc_attn_varlen_d72(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out, int64_t ldo,
                           int32_t heads, const int32_t* segs_dev, int32_t n_segs, int32_t max_q_len, float scale, void* stream);
/* The temporal self-attention of STDiT3Block (open_sora_transformer_3d.py:196-198) without the `rearrange` copies: the rows of
 * q / k / v / out are in B (T S) C order, and sequence (b, s) is the T rows b*T*S + t*S + s, t < T. head_dim 72. The kernel and
 * its rounding chain follow from T:
 *   T <= 32 (videos up to 4 s): attn_temporal_d72_kernel, P in fp32: fp32 dot products, e = exp2f(x - m), fp32 online softmax
 *     and accumulation of e * v, out = bf16(acc / l). Only the output is rounded.
 *   T > 32 (8 s and longer: T = 60, 120, 240): attn_temporal_mma_d72_kernel, the chain of mc_attn_varlen_d72: fp32 scores from
 *     mma.sync, e = exp2f(x - m_tile) per 64-key tile, e rounded to bf16 for the PV product (fp32 accumulation), the row sum l
 *     over the unrounded e, out = bf16(acc / l).
 * Past 32 frames B*S*heads*ceil(T/64) must fit one grid dimension (< 2^31) and B*T*S < 2^31; otherwise MC_ERR_INVALID. */
int32_t mc_attn_temporal_d72(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out, int64_t ldo,
                             int32_t B, int32_t T, int32_t S, int32_t heads, float scale, void* stream);

/* out[c] = bf16(bf16(sum_r x[r, c]) / rows): the mean over the valid text tokens that conditions HunyuanVideo's token refiner
 * [EXT hyvideo SingleTokenRefiner.forward, called at MagCache4HunyuanVideo/magcache_sample_video.py:69]. x bf16 [rows, cols] (row stride ld). */
int32_t mc_colmean_bf16(const void* x, int64_t ld, int32_t rows, int32_t cols, void* out, void* stream);
/* y = silu(x), bf16 -> bf16 (fp32 inside): `self.silu(emb)` of AdaLayerNormZero / ...Single / ...Continuous. */
int32_t mc_silu_bf16(const void* x, void* y, int64_t n, void* stream);

/* bf16 GEMM on wgmma, TMA-fed:  acc[m,n] = sum_k A[m,k] * B[n,k]   (A: [M,K] row-major, B: [N,K] row-major).
 * lda/ldb/ldo in elements; K % 8 == 0, lda % 8 == 0, ldb % 8 == 0, 16-byte aligned bases. */
#define MC_EPI_BIAS_BF16 0        /* out_bf16[m,n] = bf16(acc + bias[n])                              nn.Linear under autocast */
#define MC_EPI_BIAS_GELU_BF16 1   /* out_bf16 = bf16(gelu_tanh(float(bf16(acc + bias[n]))))            ffn[0] + GELU(tanh) */
#define MC_EPI_BIAS_GATE_RESID 2  /* resid_f32[m,n] += float(bf16(acc + bias[n])) * gate[n] (gate NULL -> 1) `x = x + y * e[2]` */
#define MC_EPI_ROWBIAS_BF16 3     /* out_bf16[m,n] = bf16(acc + bias[m])                               V^T = Wv * h^T + bv */
#define MC_EPI_BIAS_F32 4         /* out_f32[m,n] = acc + bias[n]                                                           */
#define MC_EPI_BIAS_GELU_ERF_BF16 5 /* out_bf16 = bf16(gelu_erf(float(bf16(acc + bias[n]))))          img_emb Linear + nn.GELU() (i2v) */
#define MC_EPI_BIAS_GATE_RESID_BF16 6 /* x_bf16[m,n] = bf16(x + bf16(gate[n] * bf16(acc + bias[n])))  all-bf16 streams (FLUX MMDiT:
                                         `hidden_states = hidden_states + gate.unsqueeze(1) * attn_output`), in place on `out` */
#define MC_EPI_BIAS_SILU_BF16 7   /* out_bf16 = bf16(silu(float(bf16(acc + bias[n]))))                 TimestepEmbedding linear_1 + SiLU */
int32_t mc_gemm_bf16(const void* A, int64_t lda, const void* B, int64_t ldb, int32_t M, int32_t N, int32_t K,
                     const float* bias, int32_t epilogue, void* out, int64_t ldo, const float* gate, void* stream);

/* Non-causal attention forward on wgmma: out[i, h*128:(h+1)*128] = softmax(q_h k_h^T * scale) v_h, head_dim = 128
 * (WanSelfAttention / WanT2VCrossAttention [EXT] behind MagCache4Wan2.1/magcache_generate.py:297-298; the joint attention of
 * MagCache4FLUX/magcache_flux.py:343-425 and MagCache4HunyuanVideo/magcache_sample_video.py:108-140).
 * q: [Lq, heads*128] bf16 (ldq), k: [Lk, heads*128] bf16 (ldk), v: [Lk, heads*128] bf16 (ldv) — all ROW-MAJOR views, so the three
 * can be column slices of one fused q|k|v projection buffer; out: [Lq, heads*128] bf16 (ldo). Leading dimensions % 8 == 0,
 * pointers 16-byte aligned.
 * workspace: device scratch for the split-KV partials that small grids use (mc_attn_workspace_bytes tells how much a shape
 * needs; 0 = the shape never splits, workspace may be NULL). The caller owns it: one per stream of concurrent use. */
int32_t mc_attn_workspace_bytes(int32_t Lq, int32_t Lk, int32_t heads, int64_t* bytes_out);
int32_t mc_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out,
                    int64_t ldo, int32_t Lq, int32_t Lk, int32_t heads, float scale, void* workspace, int64_t workspace_bytes,
                    void* stream);
/* Token-sharded form (SURVEY §8e; the exchange of videosys/core/comm.py:272-292 overlapped with the attention itself): the key /
 * value rows [first_key_row, ...) are the caller's own and already resident; the other ranks' rows arrive while the kernel runs.
 * KV tiles are consumed in rotated order starting at the caller's own rows, and before a tile that touches source segment s
 * (rows [s*seg_rows, (s+1)*seg_rows)) is loaded the kernel waits until seg_flags[s] (device memory, written by the sender
 * after the segment's data) has reached *seg_epoch (device memory, read when the kernel runs). seg_flags == NULL: no waiting
 * (plain rotation). */
int32_t mc_attn_fwd_ex(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out,
                       int64_t ldo, int32_t Lq, int32_t Lk, int32_t heads, float scale, void* workspace, int64_t workspace_bytes,
                       int32_t first_key_row, const uint32_t* seg_flags, const uint32_t* seg_epoch, int32_t seg_rows, void* stream);

/* ---- peer-to-peer exchange of token-sharded runs (one node, NVLink / NVSwitch; csrc/p2p.cu) ------------------------------------
 * The counterpart of the reference's sequence-parallel gather (videosys/core/comm.py:272-292): every rank owns a window that its
 * peers map through CUDA IPC; K|V segments and flags are moved by the copy engines, consumers poll the flags in device memory.
 * mc_p2p_alloc: cudaMalloc `bytes` (zero-filled) on the current device and return its IPC handle (64 bytes) for the peers.
 * mc_p2p_open / close: map / unmap a peer's window in this process.  mc_p2p_free: release an own window.
 * mc_p2p_bump: on `stream`, *epoch += 1 (and *own_flag = *epoch when given): starts a new exchange round.
 * mc_p2p_push: on `stream`, for every destination i: copy `bytes` from src to dst_ptrs[i], then copy *epoch (4 bytes) to
 *              flag_ptrs[i] — a peer that observes the flag observes the data. bytes == 0: flags only.
 * mc_p2p_wait: on `stream`, a one-block kernel that returns once flags[0..n) have all reached *epoch. */
int32_t mc_p2p_alloc(int64_t bytes, void** ptr_out, void* handle_out);
int32_t mc_p2p_open(const void* handle, void** ptr_out);
int32_t mc_p2p_close(void* ptr);
int32_t mc_p2p_free(void* ptr);
int32_t mc_p2p_bump(uint32_t* epoch, uint32_t* own_flag_or_null, void* stream);
int32_t mc_p2p_push(const void* src, void* const* dst_ptrs, void* const* flag_ptrs, int32_t n_dst, int64_t bytes, const uint32_t* epoch,
                    void* stream);
int32_t mc_p2p_wait(const uint32_t* flags, int32_t n, const uint32_t* epoch, void* stream);
/* mc_p2p_push2d: the 2-D form of mc_p2p_push, for Open-Sora's sequence-parallel layout switch. It replaces the `all_to_all_with_pad`
 * of STDiT3Block.dynamic_switch (videosys/models/transformers/open_sora_transformer_3d.py:275-296, videosys/core/comm.py:297-367)
 * and the `gather_sequence` in front of the final layer (eval/magcache/experiments/opensora.py:356-361). On `stream`: every copy i,
 * cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height) in bytes (any of them may be local or in a peer's window), in list
 * order; then *epoch (4 bytes) to every flag_ptrs[j]: a peer that observes its flag observes every block. Copies with width or
 * height 0 are skipped. All arguments are checked before anything is issued. */
typedef struct mc_copy2d {
  void* dst;
  int64_t dpitch;
  const void* src;
  int64_t spitch;
  int64_t width;
  int64_t height;
} mc_copy2d;
int32_t mc_p2p_push2d(const mc_copy2d* copies, int32_t n_copies, void* const* flag_ptrs, int32_t n_flags, const uint32_t* epoch,
                      void* stream);

/* ---- the collective formulation of the same exchange (SURVEY §8b `mc_nccl_init` / `mc_allgather_kv`; csrc/nccl_gather.cu) ---------
 * `dist.all_gather(tensor_list, input_)` + `torch.cat` of videosys/core/comm.py:272-292 as ONE ncclAllGather on the caller's
 * stream. NCCL is looked up at run time (the copy the process already loaded, else libnccl.so.2): MC_ERR_STATE when it is absent.
 * mc_nccl_unique_id: 128 bytes created by ONE rank and handed to the others by the host (any channel).
 * mc_nccl_init:      collective over the `world` ranks, each on its own current device; NULL + mc_last_error() on failure.
 * mc_allgather_kv:   k_full[r * n : (r+1) * n] = rank r's k_local[0 : n] (n = elems_per_rank bf16 elements, same on every rank), and
 *                    the same for v when v_local / v_full are given (both NULL: one fused K|V buffer, the engines' layout);
 *                    stream-ordered, capturable into a CUDA graph. */
typedef struct mc_nccl mc_nccl;
int32_t mc_nccl_unique_id(void* id_out_128);
mc_nccl* mc_nccl_init(int32_t rank, int32_t world, const void* unique_id_128);
int32_t mc_nccl_destroy(mc_nccl* h);
int32_t mc_allgather_kv(mc_nccl* h, const void* k_local, const void* v_local, void* k_full, void* v_full, int64_t elems_per_rank,
                        void* stream);

/* Small fp32 linear for the time-embedding path (autocast-disabled region, magcache_generate.py:249-254):
 * y[m, n] = act(sum_k x[m,k] * W[n,k] + b[n]), M <= 8. act: 0 none, 1 SiLU applied to the INPUT x first (time_projection),
 * 2 SiLU applied to the output. */
int32_t mc_linear_f32_small(const float* x, int32_t M, int32_t K, const float* W, const float* b, int32_t N, int32_t act,
                            float* y, void* stream);

/* Head + unpatchify (magcache_generate.py:304-305), with the cache-hit sum `x + residual_x` (:295) formed on the fly:
 * out[c, f, 2h+p, 2w+q] = Linear_fp32(LN(x)*(1+e1)+e0)[token, (p,q,c)], one pass over the rows (wgmma, 3-pass bf16 split:
 * fp32-class accuracy; see csrc/head_wgmma.cu).
 * x: [rows, cols] for the tokens row_offset .. row_offset+rows-1 of the F*Hp*Wp grid (rows = F*Hp*Wp, row_offset = 0 unless the
 * token axis is sharded): fp32 with r == NULL (the residual stream), or bf16 together with r fp32 [rows, cols] — the
 * un-materialised hit sum x0_bf16 + r_f32. cols % 64 == 0.
 * head_mod: [2, cols] modulation parameter, e: [cols] time embedding, Wt: head.weight TRANSPOSED [cols, 64] fp32, b: [64];
 * out fp32 [C, F, 2Hp, 2Wp]: only the positions of the given tokens are written.
 * workspace: mc_head_workspace_bytes(cols) bytes of device scratch, 1024-byte aligned (the modulated, split weight of this call).
 * flags bit 0: round the hit sum to bf16 before the head (in-place `x += residual` on a bf16 tensor, wan_teacache.py:569/577). */
int32_t mc_head_workspace_bytes(int32_t cols, int64_t* bytes_out);
int32_t mc_head_unpatchify(const void* x, int32_t x_dtype, const float* r_or_null, int64_t rows, int64_t row_offset, int32_t cols,
                           int32_t F, int32_t Hp, int32_t Wp, int32_t C_out, const float* head_mod, const float* e,
                           const float* Wt, const float* b, float eps, float* out, void* workspace, int64_t workspace_bytes,
                           int32_t flags, void* stream);
/* The two halves of mc_head_unpatchify, for callers that know the time embedding before the rows are ready (the engine prepares
 * right after the time MLP): mc_head_prepare folds the modulation into the weight (W' = (1 + e1) * W as bf16 hi / lo, the two
 * per-output constants) into `workspace`; mc_head_unpatchify_ex streams the rows against a prepared workspace and stores them into
 * n_out <= 8 output tensors (token-sharded runs: every peer's copy, P2P stores). */
int32_t mc_head_prepare(const float* head_mod, const float* e, const float* Wt, const float* b, int32_t cols, void* workspace,
                        int64_t workspace_bytes, void* stream);
int32_t mc_head_unpatchify_ex(const void* x, int32_t x_dtype, const float* r_or_null, int64_t rows, int64_t row_offset, int32_t cols,
                              int32_t F, int32_t Hp, int32_t Wp, int32_t C_out, float eps, float* const* outs, int32_t n_out,
                              const void* prepared, int64_t prepared_bytes, int32_t flags, void* stream);
/* The caller loop's step folded into the head pass (SURVEY §8f-1; eval/magcache/experiments/wan_magcache.py:301-310:
 * `noise_pred = uncond + g * (cond - uncond)`, `scheduler.step`): this launch is the UNCONDITIONAL head of a denoising step, given
 * the conditional prediction `cond` of the same step and the current latent `x_latent` (both fp32 in the output layout
 * [C, F, 2Hp, 2Wp]). Instead of the unconditional prediction y it stores
 *     out = coef_x * x_latent + coef_v * (y + guide_scale * (cond - y))
 * (flow-matching Euler: coef_x = 1, coef_v = sigma_next - sigma), every product and sum rounded separately in that order: bit-equal
 * to mc_head_unpatchify_ex followed by mc_cfg_step. x_latent may alias an output (in-place update of the latent). Positions of
 * tokens outside [row_offset, row_offset + rows) are not touched. */
int32_t mc_head_unpatchify_step(const void* x, int32_t x_dtype, const float* r_or_null, int64_t rows, int64_t row_offset, int32_t cols,
                                int32_t F, int32_t Hp, int32_t Wp, int32_t C_out, float eps, float* const* outs, int32_t n_out,
                                const void* prepared, int64_t prepared_bytes, int32_t flags, const float* cond, const float* x_latent,
                                float guide_scale, float coef_x, float coef_v, void* stream);

/* Open-Sora 1.2's final layer in one pass (csrc/opensora_head.cu): T2IFinalLayer (videosys/models/transformers/
 * open_sora_transformer_3d.py:50-86) and `unpatchify` (:625-647), replacing OpenSoraEngine.head's mc_ln_modulate (mode 2) per
 * sample + mc_gemm_bf16 (MC_EPI_BIAS_BF16, N = 32) + the permute / crop / `.float()` copy, and on a cache hit the mc_cache_hit_add
 * in front of them (eval/magcache/experiments/opensora.py:344 `x = ori_x + residual`). Per row of x bf16 [B*T*H*W, cols] (sample
 * b = row / (T*H*W)):
 *   x   = res_or_null ? bf16(x + res) : x                           (res bf16, same shape; the sum is never written)
 *   h   = bf16(bf16(bf16(LN(x)) * bf16(1 + scale_b)) + shift_b)     (mc_ln_modulate mode 2, eps; mod fp32 [B, 2, cols] = shift | scale)
 *   o_j = bf16(sum_k h_k w_jk + bias_j), j < 32                     (the wgmma instruction and K order of mc_gemm_bf16: same bits)
 *   pred[b, c, t, 2h+p, 2w+q] = o_{(2p+q)*8 + c}, cropped to Hx x Wx (Hx in {2H-1, 2H}, likewise Wx)
 * Plain mode (z_or_null == NULL): out fp32 [B, 8, T, Hx, Wx] = pred, bit-equal to the op chain.
 * Step mode (z_or_null != NULL, B even): samples [0, B/2) are the conditional and [B/2, B) the unconditional halves of the CFG
 * batch; the tail of RFLOW.sample (videosys/schedulers/scheduling_rflow_open_sora.py:244-251) over the 4 velocity channels
 *   v   = u + g * (c - u),  c = pred[b, ch], u = pred[b + B/2, ch], ch < 4   (`output.chunk(2, dim=1)[0]`, `pred.chunk(2, dim=0)`)
 *   out[b, ch] = z[b, ch] + v * dt[b]                               (z, out fp32 [B/2, 4, T, Hx, Wx], dt fp32 [B/2] on the device)
 * each operation rounded on its own in that order (no FMA contraction); out may alias z; pred itself is never written.
 * w: final_layer.linear.weight bf16 [32, cols]; bias fp32 [32] (bf16 values). cols % 8 == 0, cols <= 1152; C_out must be 8.
 * x / res / w / mod 16-byte aligned. No workspace. */
int32_t mc_opensora_head(const void* x, const void* res_or_null, int32_t B, int32_t T, int32_t H, int32_t W, int32_t cols,
                         const float* mod, const void* w, const float* bias, int32_t C_out, float eps, int32_t Hx, int32_t Wx,
                         const float* z_or_null, const float* dt, float guidance_scale, float* out, void* stream);
/* mc_opensora_head_frames: mc_opensora_head on one rank's frames of a sequence-parallel run. It replaces the `gather_sequence` of x
 * in front of the final layer (eval/magcache/experiments/opensora.py:356-361) with a final layer on the rank's own frames. x (and
 * res) hold T frames of every sample; out and z are tensors of T_out >= T frames, passed pre-offset to the rank's first frame t0
 * (out + t0 * Hx * Wx, z + t0 * Hx * Wx), so the launch writes frames [t0, t0 + T) of every (sample, channel) and reads the same
 * frames of z. Every written value has the bits mc_opensora_head writes for that frame of the full tensors. */
int32_t mc_opensora_head_frames(const void* x, const void* res_or_null, int32_t B, int32_t T, int32_t H, int32_t W, int32_t cols,
                                const float* mod, const void* w, const float* bias, int32_t C_out, float eps, int32_t Hx, int32_t Wx,
                                int32_t T_out, const float* z_or_null, const float* dt, float guidance_scale, float* out, void* stream);

/* bf16 transpose dst[c, r] = src[r, c]. */
int32_t mc_transpose_bf16(const void* src, int64_t lds, int32_t rows, int32_t cols, void* dst, int64_t ldd, void* stream);

/* sinusoidal_embedding_1d(freq_dim, t) in float64, cos half first (magcache_generate.py:250-251): pos_dev [n_pos] f64 ->
 * out fp32 [n_pos, dim]. */
int32_t mc_time_sinusoid(const double* pos_dev, int32_t n_pos, int32_t dim, float* out, void* stream);

/* elementwise helpers */
int32_t mc_cast(const void* src, int32_t src_dtype, void* dst, int32_t dst_dtype, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * The whole patched forward in one call (SURVEY §8b `mc_dit_forward`): prologue -> { cache hit | block stack + residual } -> head,
 * MagCache4Wan2.1/magcache_generate.py:229-275 and :293-305 for a text-to-video WanModel; the skip decision (:277-292) is the
 * caller's (mc_ctrl_step). Native host code that issues the launch sequence of the Python engine (magcache_b200/wan.py) through
 * the entry points above, on buffers carved out of ONE caller-owned workspace: same kernels, operands and order, bit-identical
 * results. Built for the plain case (one sample, one timestep, one GPU, head_dim 128, 16 output channels); i2v / VACE /
 * token-sharded / per-token-timestep forwards are sequenced by the Python engine.
 * All weight pointers are DEVICE pointers in the engine's packed layout, borrowed (they must outlive the handle), 16-byte aligned:
 * bf16 `[out, in]` matrices (`const void*`), fp32 vectors / small fp32 matrices (`const float*`); biases are the bf16-rounded values
 * kept as fp32 (nn.Linear under autocast).
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct mc_dit_dims {
  int32_t dim, ffn_dim, num_heads, num_layers; /* dim == num_heads * 128 */
  int32_t in_dim, out_dim;                     /* latent channels in (patch (1,2,2): in_dim*4 columns) and out (16) */
  int32_t freq_dim, text_dim, text_len;
  float eps;
} mc_dit_dims;

typedef struct mc_dit_block {                 /* one WanAttentionBlock [EXT upstream wan/modules/model.py] */
  const float* mod;                           /* modulation               fp32 [6, dim] */
  const void* w_qkv;  const float* b_qkv;     /* self_attn q|k|v fused    bf16 [3 dim, dim], fp32 [3 dim] */
  const void* w_o;    const float* b_o;       /* self_attn.o */
  const float* nqk;                           /* norm_q | norm_k weights  fp32 [2, dim] */
  const float* n3_w;  const float* n3_b;      /* norm3 (affine LayerNorm) */
  const void* c_wq;   const float* c_bq;      /* cross_attn.q */
  const void* c_wkv;  const float* c_bkv;     /* cross_attn k|v fused     bf16 [2 dim, dim] */
  const void* c_wo;   const float* c_bo;      /* cross_attn.o */
  const float* c_nq;  const float* c_nk;      /* cross_attn norm_q / norm_k */
  const void* w_f1;   const float* b_f1;      /* ffn[0]                   bf16 [ffn_dim, dim] */
  const void* w_f2;   const float* b_f2;      /* ffn[2]                   bf16 [dim, ffn_dim] */
} mc_dit_block;

typedef struct mc_dit_weights {
  const void* patch_w;  const float* patch_b; /* patch_embedding          bf16 [dim, in_dim*4] in (c, kt, kh, kw) order */
  const void* text_w1;  const float* text_b1; /* text_embedding[0]        bf16 [dim, text_dim] */
  const void* text_w2;  const float* text_b2; /* text_embedding[2]        bf16 [dim, dim] */
  const float* time_w1; const float* time_b1; /* time_embedding[0]        fp32 [dim, freq_dim] */
  const float* time_w2; const float* time_b2; /* time_embedding[2]        fp32 [dim, dim] */
  const float* tproj_w; const float* tproj_b; /* time_projection[1]       fp32 [6 dim, dim] */
  const float* head_mod;                      /* head.modulation          fp32 [2, dim] */
  const float* head_wt; const float* head_b;  /* head.head weight TRANSPOSED fp32 [dim, 64], bias fp32 [64] */
  const mc_dit_block* blocks;                 /* [num_layers] (copied by mc_dit_create) */
} mc_dit_weights;

typedef struct mc_dit mc_dit;
/* NULL (and mc_last_error) on unsupported dims or null / misaligned pointers. No device work. */
mc_dit* mc_dit_create(const mc_dit_dims* dims, const mc_dit_weights* weights);
void mc_dit_destroy(mc_dit* h);
/* Device scratch one (F, Hp, Wp) token grid needs: every activation of a forward (patch tokens, x0, the fp32 stream, q|k|v, FFN
 * hidden, text embeddings, time embeddings, the head's prepared weight, split-KV partials). Host arithmetic only. */
int32_t mc_dit_workspace_bytes(const mc_dit* h, int32_t F, int32_t Hp, int32_t Wp, int64_t* bytes_out);
/* Bind the handle to a token grid: `workspace` (1024-byte aligned, >= mc_dit_workspace_bytes, caller-owned, one per stream of
 * concurrent use) and the RoPE table fp32 [F*Hp*Wp, 128] (interleaved cos, sin; mc_rmsnorm_rope's layout). No device work. */
int32_t mc_dit_bind(mc_dit* h, int32_t F, int32_t Hp, int32_t Wp, void* workspace, int64_t workspace_bytes, const float* rope_cos_sin);
/* One patched forward on `stream`. latent fp32 [in_dim, F, 2Hp, 2Wp]; t_dev: the timestep as ONE device double; context bf16
 * [text_len, text_dim], zero-padded (may be NULL when skip != 0: a hit does not read it); residual fp32 [F*Hp*Wp, dim]: the slot
 * `residual_cache[cnt % 2]` — READ when skip != 0 (`x + residual_x`, :295), WRITTEN when skip == 0 (`x - ori_x`, :299);
 * out fp32 [16, F, 2Hp, 2Wp]. All device pointers, 16-byte aligned. Returns the first failing entry point's code. */
int32_t mc_dit_forward(mc_dit* h, const float* latent, const double* t_dev, const void* context_bf16, int32_t skip, float* residual,
                       float* out, void* stream);
/* The launch plan of mc_dit_forward(skip) as text, one line per launch, operands printed as name+byte_offset; nothing is launched
 * (inspection / test aid: the CPU suite compares it with the sequence the Python engine issues). *needed = bytes incl. the
 * terminator; the text is written when buf_bytes >= *needed. */
int32_t mc_dit_plan(mc_dit* h, int32_t skip, char* buf, int64_t buf_bytes, int64_t* needed);

#ifdef __cplusplus
}
#endif
#endif /* MAGCACHE_B200_H_ */
