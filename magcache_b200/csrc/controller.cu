// Host-side MagCache logic: error plumbing, nearest_interp, and the skip controller.
// float64 / int arithmetic in exactly the reference's operation order so the skip mask is bit-exact.
//   controller   MagCache4Wan2.1/magcache_generate.py:277-292, :306-311
//                MagCache4FLUX/magcache_flux.py:326-338, :431-436
//                MagCache4HunyuanVideo/magcache_sample_video.py:88-102, :149-154
//                MagCache4FramePack/magcache_demo_gradio.py:252-270 (ratio veto, cnt >= 1, re-initialisation at cnt == 0)
//                eval/magcache/experiments/Wan2.1_EVAL/wan_magcache.py:770-786 (table offset 10), opensora.py:297-308 (signed error)
//   interp       MagCache4Wan2.1/magcache_generate.py:27-34, :915-919
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace mc {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int num_sms() {
  static int cached[kMaxDevices] = {};
  const int dev = current_device();
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached[dev] = n;
    else
      cached[dev] = 148;
  }
  return cached[dev];
}

// first call index that is allowed to skip (single-threshold modes)
static int32_t retention_start(const mc_ctrl_config* c) {
  const double n = static_cast<double>(c->num_steps);
  switch (c->retention_mode) {
    case MC_RETAIN_HALF_UP:
      return static_cast<int32_t>(c->retention_ratio * n + 0.5);  // int(R*n + 0.5)
    case MC_RETAIN_CEIL:
      return static_cast<int32_t>(std::ceil(c->retention_ratio * n));
    default:
      return static_cast<int32_t>(n * c->retention_ratio);  // int(n*R): truncation
  }
}

// `use_magcache` of the reference: may this call consult the controller at all?
static bool eligible(const mc_ctrl_config* c, int32_t cnt) {
  const double n = static_cast<double>(c->num_steps), sp = static_cast<double>(c->split_step), R = c->retention_ratio;
  switch (c->retention_mode) {
    case MC_RETAIN_WAN22_I2V:  // MagCache4Wan2.2/magcache_generate.py:295-297
      return !(cnt < static_cast<int32_t>(sp + (n - sp) * R));
    case MC_RETAIN_WAN22_T2V: {  // :298-300 ; `tensor(int64) <= python float` compares in float32
      const bool early = cnt < static_cast<int32_t>(sp * R);
      const float upper = static_cast<float>((n - sp) * R + sp);
      const bool window = (static_cast<float>(cnt) <= upper) && (cnt >= c->split_step);
      return !(early || window);
    }
    case MC_RETAIN_EXPLICIT:  // opensora.py:297 `self.t >= self.skip_time`
      return cnt >= c->split_step && cnt >= c->min_cnt;
    default:
      return cnt >= retention_start(c) && cnt >= c->min_cnt;
  }
}

static int32_t check_cfg(const mc_ctrl_config* c) {
  MC_CHECK_ARG(c != nullptr, "mc_ctrl: null config");
  MC_CHECK_ARG(c->num_steps >= 1, "mc_ctrl: num_steps=%d must be >= 1", c->num_steps);
  MC_CHECK_ARG(c->branches == 1 || c->branches == 2, "mc_ctrl: branches=%d must be 1 or 2", c->branches);
  MC_CHECK_ARG(c->mag_ratios != nullptr, "mc_ctrl: mag_ratios is null (reference: AttributeError, no table matched ckpt_dir)");
  MC_CHECK_ARG(c->cmp == MC_CMP_LT || c->cmp == MC_CMP_LE, "mc_ctrl: bad cmp %d", c->cmp);
  MC_CHECK_ARG(c->retention_mode >= 0 && c->retention_mode <= 5, "mc_ctrl: bad retention_mode %d", c->retention_mode);
  MC_CHECK_ARG(c->table_offset >= 0 && c->table_offset < c->num_steps, "mc_ctrl: table_offset=%d outside [0, num_steps)", c->table_offset);
  MC_CHECK_ARG(c->min_cnt >= 0, "mc_ctrl: min_cnt=%d must be >= 0", c->min_cnt);
  MC_CHECK_ARG((c->flags & ~(MC_CTRL_SIGNED_ERR | MC_CTRL_RESET_AT_ZERO | MC_CTRL_RATIO_VETO | MC_CTRL_WRAP_KEEPS_ACC)) == 0 && c->reserved == 0, "mc_ctrl: unknown flag bits 0x%x", c->flags);
  MC_CHECK_ARG(!(c->flags & MC_CTRL_RATIO_VETO) || c->ratio_veto >= 0.0, "mc_ctrl: ratio_veto must be >= 0");
  MC_CHECK_ARG(c->retention_mode < MC_RETAIN_WAN22_T2V || (c->split_step >= 0 && c->split_step <= c->num_steps),
               "mc_ctrl: split_step=%d outside [0, num_steps]", c->split_step);
  MC_CHECK_ARG(c->veto_index < 0 || c->num_steps >= 2, "mc_ctrl: step veto needs num_steps >= 2 (reference divides by num_steps-1)");
  return MC_OK;
}

static inline void reset_branch(mc_ctrl_state* st, int i) {
  st->accumulated_err[i] = 0.0;
  st->accumulated_steps[i] = 0;
  st->accumulated_ratio[i] = 1.0;
}

// returns 0/1, or a negative error code
static int32_t decide(const mc_ctrl_config* c, mc_ctrl_state* st) {
  if ((c->flags & MC_CTRL_RESET_AT_ZERO) && st->cnt == 0) {
    reset_branch(st, 0);
    reset_branch(st, 1);
  }
  if (!eligible(c, st->cnt)) return 0;
  if (st->cnt < c->table_offset) {
    // the reference would read ratio[negative] = an entry counted from the END of the table; refuse instead of reproducing that
    set_error("mc_ctrl_decide: call %d is skip-eligible but precedes table_offset=%d (retention window shorter than the table offset)", st->cnt,
              c->table_offset);
    return MC_ERR_STATE;
  }
  const int i = (c->branches == 2) ? (st->cnt % 2) : 0;
  const double cur = c->mag_ratios[st->cnt - c->table_offset];
  st->accumulated_ratio[i] = st->accumulated_ratio[i] * cur;
  st->accumulated_steps[i] += 1;
  const double diff = 1.0 - st->accumulated_ratio[i];
  st->accumulated_err[i] += (c->flags & MC_CTRL_SIGNED_ERR) ? diff : std::fabs(diff);
  bool ok = (c->cmp == MC_CMP_LE) ? (st->accumulated_err[i] <= c->thresh) : (st->accumulated_err[i] < c->thresh);
  ok = ok && (st->accumulated_steps[i] <= c->K);
  if (c->flags & MC_CTRL_RATIO_VETO) ok = ok && (std::fabs(1.0 - cur) <= c->ratio_veto);
  if (c->veto_index >= 0) {
    // np.round(cnt * ((base-1)/(num_steps-1))).astype(int) != veto_index ; nearbyint = round-half-even
    const double scale = static_cast<double>(c->veto_base - 1) / static_cast<double>(c->num_steps - 1);
    const long mapped = static_cast<long>(std::nearbyint(static_cast<double>(st->cnt) * scale));
    ok = ok && (mapped != c->veto_index);
  }
  if (ok) return 1;
  reset_branch(st, i);
  return 0;
}

static void advance(const mc_ctrl_config* c, mc_ctrl_state* st) {
  st->cnt += 1;
  if (st->cnt >= c->num_steps) {
    st->cnt = 0;
    if (!(c->flags & MC_CTRL_WRAP_KEEPS_ACC)) {
      reset_branch(st, 0);
      reset_branch(st, 1);
    }
  }
}

}  // namespace mc

extern "C" {

const char* mc_last_error(void) { return mc::g_err; }
int32_t mc_abi_version(void) { return 7; }

int32_t mc_nearest_interp(const double* src, int32_t L, double* dst, int32_t T) {
  MC_CHECK_ARG(src && dst, "mc_nearest_interp: null pointer");
  MC_CHECK_ARG(L >= 1 && T >= 1, "mc_nearest_interp: L=%d T=%d must be >= 1", L, T);
  if (T == 1) {
    dst[0] = src[L - 1];
    return MC_OK;
  }
  const double scale = static_cast<double>(L - 1) / static_cast<double>(T - 1);
  for (int32_t i = 0; i < T; ++i) {
    const long idx = static_cast<long>(std::nearbyint(static_cast<double>(i) * scale));  // np.round: half to even
    MC_CHECK_ARG(idx >= 0 && idx < L, "mc_nearest_interp: index %ld out of range", idx);
    dst[i] = src[idx];
  }
  return MC_OK;
}

int32_t mc_nearest_interp_linspace(const double* src, int32_t L, double* dst, int32_t T) {
  MC_CHECK_ARG(src && dst, "mc_nearest_interp_linspace: null pointer");
  MC_CHECK_ARG(L >= 1 && T >= 1, "mc_nearest_interp_linspace: L=%d T=%d must be >= 1", L, T);
  if (L == T) {
    for (int32_t i = 0; i < T; ++i) dst[i] = src[i];
    return MC_OK;
  }
  // np.linspace(0, L-1, T): arange(T) * ((L-1)/(T-1)) + 0 with the last sample forced to L-1; T == 1 -> [0.]
  const double step = (T > 1) ? static_cast<double>(L - 1) / static_cast<double>(T - 1) : 0.0;
  for (int32_t i = 0; i < T; ++i) {
    double pos = static_cast<double>(i) * step;
    if (T > 1 && i == T - 1) pos = static_cast<double>(L - 1);
    const long idx = static_cast<long>(std::nearbyint(pos));
    MC_CHECK_ARG(idx >= 0 && idx < L, "mc_nearest_interp_linspace: index %ld out of range", idx);
    dst[i] = src[idx];
  }
  return MC_OK;
}

int32_t mc_nearest_interp_cfg(const double* src, int32_t L_total, double* dst, int32_t steps) {
  MC_CHECK_ARG(src && dst, "mc_nearest_interp_cfg: null pointer");
  MC_CHECK_ARG(L_total >= 2 && L_total % 2 == 0 && steps >= 1, "mc_nearest_interp_cfg: L_total=%d steps=%d", L_total, steps);
  const int32_t L = L_total / 2;
  std::vector<double> a(L), b(L), oa(steps), ob(steps);
  for (int32_t i = 0; i < L; ++i) {
    a[i] = src[2 * i];
    b[i] = src[2 * i + 1];
  }
  int32_t rc = mc_nearest_interp(a.data(), L, oa.data(), steps);
  if (rc) return rc;
  rc = mc_nearest_interp(b.data(), L, ob.data(), steps);
  if (rc) return rc;
  for (int32_t i = 0; i < steps; ++i) {
    dst[2 * i] = oa[i];
    dst[2 * i + 1] = ob[i];
  }
  return MC_OK;
}

int32_t mc_ctrl_decide(const mc_ctrl_config* cfg, mc_ctrl_state* st, int32_t* skip) {
  int32_t rc = mc::check_cfg(cfg);
  if (rc) return rc;
  MC_CHECK_ARG(st && skip, "mc_ctrl_decide: null pointer");
  if (st->cnt < 0 || st->cnt >= cfg->num_steps) {
    mc::set_error("mc_ctrl_decide: cnt=%d outside [0, %d)", st->cnt, cfg->num_steps);
    return MC_ERR_STATE;
  }
  const int32_t d = mc::decide(cfg, st);
  if (d < 0) return d;
  *skip = d;
  return MC_OK;
}

int32_t mc_ctrl_advance(const mc_ctrl_config* cfg, mc_ctrl_state* st) {
  MC_CHECK_ARG(cfg && st, "mc_ctrl_advance: null pointer");
  mc::advance(cfg, st);
  return MC_OK;
}

int32_t mc_ctrl_mask(const mc_ctrl_config* cfg, int32_t calls, uint8_t* mask) {
  int32_t rc = mc::check_cfg(cfg);
  if (rc) return rc;
  MC_CHECK_ARG(mask && calls >= 0, "mc_ctrl_mask: bad arguments");
  mc_ctrl_state st;
  std::memset(&st, 0, sizeof(st));
  st.accumulated_ratio[0] = st.accumulated_ratio[1] = 1.0;
  for (int32_t i = 0; i < calls; ++i) {
    const int32_t d = mc::decide(cfg, &st);
    if (d < 0) return d;
    mask[i] = static_cast<uint8_t>(d);
    mc::advance(cfg, &st);
  }
  return MC_OK;
}

// ---- handle form (SURVEY §8b) -----------------------------------------------------------------------------------------------
struct mc_ctrl {
  mc_ctrl_config cfg;
  std::vector<double> table;
  mc_ctrl_state st;
  int32_t initial_steps;
};

static void ctrl_fresh(mc_ctrl* h) {
  std::memset(&h->st, 0, sizeof(h->st));
  h->st.accumulated_ratio[0] = h->st.accumulated_ratio[1] = 1.0;
  h->st.accumulated_steps[0] = h->st.accumulated_steps[1] = h->initial_steps;  // OmniGen2: 3 (magcache_utils.py:44)
}

mc_ctrl* mc_ctrl_create(const mc_ctrl_config* cfg, int32_t initial_accumulated_steps) {
  if (mc_ctrl_validate(cfg) != MC_OK) return nullptr;
  if (initial_accumulated_steps < 0) {
    mc::set_error("mc_ctrl_create: initial_accumulated_steps=%d must be >= 0", initial_accumulated_steps);
    return nullptr;
  }
  mc_ctrl* h = new mc_ctrl();
  h->cfg = *cfg;
  h->table.assign(cfg->mag_ratios, cfg->mag_ratios + (cfg->num_steps - cfg->table_offset));
  h->cfg.mag_ratios = h->table.data();
  h->initial_steps = initial_accumulated_steps;
  ctrl_fresh(h);
  return h;
}

int32_t mc_ctrl_step(mc_ctrl* h, int32_t* skip, int32_t* cnt_out) {
  MC_CHECK_ARG(h && skip, "mc_ctrl_step: null pointer");
  const int32_t d = mc::decide(&h->cfg, &h->st);
  if (d < 0) return d;
  *skip = d;
  mc::advance(&h->cfg, &h->st);
  if (cnt_out) *cnt_out = h->st.cnt;
  return MC_OK;
}

int32_t mc_ctrl_reset(mc_ctrl* h) {
  MC_CHECK_ARG(h, "mc_ctrl_reset: null handle");
  ctrl_fresh(h);
  return MC_OK;
}

const mc_ctrl_state* mc_ctrl_state_of(const mc_ctrl* h) { return h ? &h->st : nullptr; }

void mc_ctrl_destroy(mc_ctrl* h) { delete h; }

// ---- TeaCache comparator: eval/magcache/experiments/Wan2.1_EVAL/wan_teacache.py:535-564 ------------------------------------
static int32_t tea_check(const mc_tea_config* c, const mc_tea_state* st) {
  MC_CHECK_ARG(c && st, "mc_tea: null pointer");
  MC_CHECK_ARG(c->num_steps >= 1 && c->n_coef >= 1 && c->n_coef <= 8, "mc_tea: num_steps=%d n_coef=%d", c->num_steps, c->n_coef);
  if (st->cnt < 0 || st->cnt >= c->num_steps) {
    mc::set_error("mc_tea: cnt=%d outside [0, %d)", st->cnt, c->num_steps);
    return MC_ERR_STATE;
  }
  return MC_OK;
}

int32_t mc_tea_needs_distance(const mc_tea_config* cfg, const mc_tea_state* st, int32_t* needs) {
  int32_t rc = tea_check(cfg, st);
  if (rc) return rc;
  MC_CHECK_ARG(needs, "mc_tea_needs_distance: null pointer");
  *needs = !(st->cnt < cfg->ret_steps || st->cnt >= cfg->cutoff_steps);
  return MC_OK;
}

int32_t mc_tea_decide(const mc_tea_config* cfg, mc_tea_state* st, double rel_l1, int32_t* calc) {
  int32_t rc = tea_check(cfg, st);
  if (rc) return rc;
  MC_CHECK_ARG(calc, "mc_tea_decide: null pointer");
  const int i = st->cnt % 2;  // even -> condition, odd -> uncondition
  if (st->cnt < cfg->ret_steps || st->cnt >= cfg->cutoff_steps) {
    *calc = 1;
    st->accumulated[i] = 0.0;
    return MC_OK;
  }
  double y = 0.0;  // np.poly1d(coefficients)(x): Horner, highest power first
  for (int k = 0; k < cfg->n_coef; ++k) y = y * rel_l1 + cfg->coef[k];
  st->accumulated[i] += y;
  if (st->accumulated[i] < cfg->thresh) {
    *calc = 0;
  } else {
    *calc = 1;
    st->accumulated[i] = 0.0;
  }
  return MC_OK;
}

// ---- Open-Sora's rule: eval/magcache/experiments/opensora.py:96-107 (forced on the first / last sampler timestep, no counter) ---
int32_t mc_tea_opensora_decide(int32_t forced, double rel, double accumulated, double thresh, const double* coef, int32_t n_coef,
                               int32_t* calc, double* accumulated_out) {
  MC_CHECK_ARG(calc && accumulated_out, "mc_tea_opensora_decide: null pointer");
  if (forced) {
    *calc = 1;
    *accumulated_out = 0.0;
    return MC_OK;
  }
  MC_CHECK_ARG(coef && n_coef >= 1 && n_coef <= 8, "mc_tea_opensora_decide: n_coef=%d outside [1, 8]", n_coef);
  double y = 0.0;  // np.poly1d(coefficients)(rel): Horner, highest power first
  for (int k = 0; k < n_coef; ++k) y = y * rel + coef[k];
  accumulated += y;
  if (accumulated < thresh) {
    *calc = 0;
  } else {
    *calc = 1;
    accumulated = 0.0;
  }
  *accumulated_out = accumulated;
  return MC_OK;
}

int32_t mc_tea_advance(const mc_tea_config* cfg, mc_tea_state* st) {
  MC_CHECK_ARG(cfg && st, "mc_tea_advance: null pointer");
  st->cnt += 1;
  if (st->cnt >= cfg->num_steps) st->cnt = 0;
  return MC_OK;
}

int32_t mc_ctrl_validate(const mc_ctrl_config* cfg) {
  int32_t rc = mc::check_cfg(cfg);
  if (rc) return rc;
  int32_t start = 0;
  while (start < cfg->num_steps && !mc::eligible(cfg, start)) ++start;
  if (start < cfg->num_steps && start < cfg->table_offset) {
    mc::set_error("mc_ctrl_validate: first skip-eligible call %d precedes table_offset=%d (the reference would index the table from its end)", start,
                  cfg->table_offset);
    return MC_ERR_STATE;
  }
  if (start < cfg->branches) {
    mc::set_error(
        "mc_ctrl_validate: first skip-eligible call is %d but %d residual slot(s) must be filled first "
        "(reference: `x + None` TypeError; raise retention_ratio or num_steps)",
        start, cfg->branches);
    return MC_ERR_STATE;
  }
  return MC_OK;
}

}  // extern "C"
