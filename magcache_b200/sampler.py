"""The caller loop's per-step tail — CFG combine + scheduler update — on the fused `mc_cfg_step` kernel (SURVEY §8f rank 1).

Reference call site: eval/magcache/experiments/Wan2.1_EVAL/wan_magcache.py:289-310

    noise_pred = noise_pred_uncond + guide_scale * (noise_pred_cond - noise_pred_uncond)
    temp_x0 = sample_scheduler.step(noise_pred.unsqueeze(0), t, latents[0].unsqueeze(0), return_dict=False, generator=seed_g)[0]

The schedulers (`FlowUniPCMultistepScheduler`, `FlowDPMSolverMultistepScheduler`, :263-279) are upstream Wan code that is not in
the reference tree ("parity unpinned", see oracle/sampler_ref.py). All of them update the latent by a LINEAR combination of the
current sample, the guided flow prediction and a few stored tensors, with scalar coefficients that depend only on the sigma
schedule — so the host computes the scalars in float64 and every tensor operation of a step is one or two launches of
`mc_cfg_step` (instead of ~15 element-wise torch kernels and their temporaries).
"""
import math

import torch

from . import ops


def sampling_sigmas(steps, shift):
    """`shift*s/(1+(shift-1)*s)` over s = linspace(1, 0, steps+1) (float64, terminal 0 included); timestep = 1000*sigma."""
    out = []
    for i in range(steps + 1):
        s = 1.0 - i / steps
        out.append(shift * s / (1.0 + (shift - 1.0) * s))
    return out


def cfg_denoise_step(model, x, t, context, context_null, seq_len, guide_scale, coef_v, coef_x=1.0, forward=None, hist=None, coef_h=0.0,
                     sigma=0.0, x0_out=None, **kw):
    """`x <- coef_x * x + coef_v * (uncond + g * (cond - uncond))` with both predictions from the patched forward of `model`
    (SURVEY §8f rank 1 as written). On the unsharded Wan engine the combine and the update ride in the epilogue of the unconditional
    call's head kernel (`mc_head_unpatchify_step`): the unconditional prediction is never written, no separate pass over the
    latents runs — on a step where both calls hit the cache the whole step is two streaming head launches. Token-sharded engines
    (whose head stores go to every peer) and multistep solvers that keep history terms use `ops.cfg_step` after the two calls.
    Bit-equal either way. `forward(x, t, context) -> prediction` replaces the plain `model([x], t=..., context=[...])` call (a
    caller that wraps its forwards, e.g. with timing events).
    `hist` (one stored tensor of a multistep solver, DPM++ 2M's previous x0-prediction) adds `coef_h * hist` to the update and,
    with `x0_out`, writes the x0-prediction `x - sigma * v` there: in the same head epilogue (`mc_head_unpatchify_step_hist`) on
    the fused path, as `ops.cfg_step(..., hist=[hist], ...)` on the others."""
    from .patch import _engine
    if forward is None:
        def forward(xx, tt, cc):
            return model([xx], t=tt, context=[cc], seq_len=seq_len, **kw)[0]
    cond = forward(x, t, context)
    eng = _engine(model)
    # the fused form is built for one timestep per call and 16 output channels (not Wan2.2 TI2V-5B: per-token t, 48 channels)
    if hist is None and x0_out is not None:
        raise ValueError("magcache_b200: cfg_denoise_step writes x0_out only together with a history term (hist)")
    if getattr(eng, "shard", None) is None and hasattr(eng, "arm_step") and t.numel() == 1 and len(getattr(eng, "head_groups", (0,))) == 1:
        if hist is None:
            eng.arm_step(cond, x, guide_scale, coef_x, coef_v, out=x)
        else:
            eng.arm_step(cond, x, guide_scale, coef_x, coef_v, out=x, hist=hist, coef_h=coef_h, sigma=sigma, x0_out=x0_out)
        return forward(x, t, context_null)
    uncond = forward(x, t, context_null)
    if hist is None:
        return ops.cfg_step(cond, uncond, guide_scale, x, coef_v, coef_x=coef_x, out=x)
    return ops.cfg_step(cond, uncond, guide_scale, x, coef_v, coef_x=coef_x, hist=[hist], coef_h=[coef_h], sigma=sigma, out=x, x0_out=x0_out)


class FlowEulerSampler:
    """x <- x + (sigma_{i+1} - sigma_i) * v : one launch per step, in place."""

    def __init__(self, sigmas):
        self.sigmas = [float(s) for s in sigmas]
        self.i = 0

    @property
    def timestep(self):
        return 1000.0 * self.sigmas[self.i]

    def step(self, cond, uncond, guide_scale, x):
        d = self.sigmas[self.i + 1] - self.sigmas[self.i]
        self.i += 1
        return ops.cfg_step(cond, uncond, guide_scale, x, d, out=x)

    def denoise(self, model, x, t, context, context_null, seq_len, guide_scale, **kw):
        """One whole step of the caller loop (wan_magcache.py:296-310): cond call, uncond call, CFG combine, scheduler update; the
        latent `x` [C, F, H, W] is updated in place and returned. `model` carries the patched forward (`init_magcache`)."""
        d = self.sigmas[self.i + 1] - self.sigmas[self.i]
        self.i += 1
        return cfg_denoise_step(model, x, t, context, context_null, seq_len, guide_scale, coef_v=d, **kw)


def timestep_transform(t, model_kwargs, base_resolution=512 * 512, base_num_frames=1, scale=1.0, num_timesteps=1):
    """Open-Sora's resolution- and length-dependent timestep shift (scheduling_rflow_open_sora.py:47-70), the same torch statements."""
    t = t / num_timesteps
    resolution = model_kwargs["height"] * model_kwargs["width"]
    ratio_space = (resolution / base_resolution).sqrt()
    if model_kwargs["num_frames"][0] == 1:
        num_frames = torch.ones_like(model_kwargs["num_frames"])
    else:
        num_frames = model_kwargs["num_frames"] // 17 * 5  # the VAE's temporal reduction
    ratio_time = (num_frames / base_num_frames).sqrt()
    ratio = ratio_space * ratio_time * scale
    new_t = ratio * t / (1 + (ratio - 1) * t)
    return new_t * num_timesteps


class OpenSoraRFlowSampler:
    """`RFLOW.sample` of Open-Sora 1.2 (videosys/schedulers/scheduling_rflow_open_sora.py:164-256) with the same constructor and
    `sample` signature, so it can stand in for the pipeline's `scheduler`. The timestep schedule, `all_timesteps` and `dt` are the
    reference's statements, evaluated in torch on the host. Each step is one CFG forward of the doubled batch; when `model` carries
    an installed Open-Sora forward (`init_magcache_opensora` / `init_teacache_opensora`), the step's tail — velocity channels,
    cond / uncond split, `uncond + g * (cond - uncond)`, `z + v_pred * dt` — runs inside that forward's final layer
    (`OpenSoraEngine.arm_step`, `mc_opensora_head`), so the prediction is never written. Any other model runs the reference's torch
    statements after its forward. Both give the reference's bits."""

    def __init__(self, num_sampling_steps=30, cfg_scale=7.0, num_timesteps=1000, use_timestep_transform=True, use_discrete_timesteps=False):
        self.num_sampling_steps = num_sampling_steps
        self.num_timesteps = num_timesteps
        self.cfg_scale = cfg_scale
        self.use_discrete_timesteps = use_discrete_timesteps
        self.use_timestep_transform = use_timestep_transform

    def timesteps(self, batch, model_args):
        """The per-step timestep tensors [batch] on the host (:208-213)."""
        timesteps = [(1.0 - i / self.num_sampling_steps) * self.num_timesteps for i in range(self.num_sampling_steps)]
        if self.use_discrete_timesteps:
            timesteps = [int(round(t)) for t in timesteps]
        timesteps = [torch.tensor([t] * batch) for t in timesteps]
        if self.use_timestep_transform:
            host_args = {k: model_args[k].cpu() for k in ("height", "width", "num_frames")}
            timesteps = [timestep_transform(t, host_args, num_timesteps=self.num_timesteps) for t in timesteps]
        return timesteps

    def dt(self, timesteps, i):
        """`dt` of step i (:249-250)."""
        dt = timesteps[i] - timesteps[i + 1] if i < len(timesteps) - 1 else timesteps[i]
        return dt / self.num_timesteps

    def sample(self, model, z, model_args, y_null, device, mask=None, guidance_scale=None, progress=True, verbose=False):
        from .patch import magcache_opensora_forward, opensora_engine, teacache_opensora_forward
        if mask is not None:
            raise NotImplementedError("magcache_b200: Open-Sora sampling with a mask (image / video conditioning with x_mask) is not supported")
        if guidance_scale is None:
            guidance_scale = self.cfg_scale
        model_args["y"] = torch.cat([model_args["y"], y_null], 0)
        host_ts = self.timesteps(z.shape[0], model_args)
        timesteps = [t.to(device) for t in host_ts]
        dtype = model.x_embedder.proj.weight.dtype
        # `int(t.to(dtype).item())` (:222) of the first entry: every entry is the same, and the reference's `.item()` of the whole
        # [B] tensor raises for two or more prompts
        all_timesteps = [int(t[0].to(dtype).item()) for t in host_ts]
        eng = None
        if getattr(type(model), "forward", None) in (magcache_opensora_forward, teacache_opensora_forward):
            if model.__dict__.get("_mc_shard_kw", {}).get("shard_world", 1) > 1:
                raise NotImplementedError("magcache_b200: the Open-Sora sampler has no token-sharded path")
            eng = opensora_engine(model, torch.device(device))
            z = z.to(device=device, dtype=torch.float32, copy=True)  # the sampler's own latent, updated in place (bf16 -> fp32 is exact)
        steps = list(enumerate(timesteps))
        if progress and (not torch.distributed.is_initialized() or torch.distributed.get_rank() == 0):
            from tqdm import tqdm
            steps = tqdm(steps)
        for i, t in steps:
            z_in = torch.cat([z, z], 0)
            t = torch.cat([t, t], 0)
            dt = self.dt(host_ts, i).to(device)
            if eng is not None:
                if dt.dtype != torch.float32:
                    raise NotImplementedError(f"magcache_b200: the fused Open-Sora step takes an fp32 dt (model_args gave {dt.dtype})")
                eng.arm_step(z, guidance_scale, dt, z)
                try:
                    z = model(z_in, t, all_timesteps, **model_args)
                finally:
                    eng._step = None
                continue
            output = model(z_in, t, all_timesteps, **model_args)
            pred = output.chunk(2, dim=1)[0]
            pred_cond, pred_uncond = pred.chunk(2, dim=0)
            v_pred = pred_uncond + guidance_scale * (pred_cond - pred_uncond)
            z = z + v_pred * dt[:, None, None, None, None]
        return z


class FlowUniPCSampler:
    """UniPC (bh2, x0-prediction, order 2, lower order on the first and last step, corrector after the first step) on the
    flow parameterisation alpha = 1 - sigma. Two launches per step: [corrector + x0-prediction] and [predictor]."""

    def __init__(self, sigmas, order=2):
        if order not in (1, 2):
            raise NotImplementedError("FlowUniPCSampler: solver order 1 or 2 (the reference's callers use the default, 2)")
        self.sigmas = [float(s) for s in sigmas]
        self.order = order
        self.i = 0
        self.lower_order_nums = 0
        self.this_order = 1
        self._m = []       # x0 predictions, newest last (device tensors, recycled)
        self._last = None  # corrected sample of the previous step
        self._free = []

    @property
    def timestep(self):
        return 1000.0 * self.sigmas[self.i]

    @staticmethod
    def _lam(sigma):
        return math.log(1.0 - sigma) - math.log(sigma)

    @staticmethod
    def _b(hh, order):
        """b_k = h_phi_{k+1} * k! / B(h) of the UniPC linear system (k = 1..order), B(h) = expm1(hh)."""
        h_phi_1 = math.expm1(hh)
        B_h = h_phi_1
        h_phi_k = h_phi_1 / hh - 1.0
        b, fact = [], 1
        for k in range(1, order + 1):
            b.append(h_phi_k * fact / B_h)
            fact *= k + 1
            h_phi_k = h_phi_k / hh - 1.0 / fact
        return h_phi_1, B_h, b

    def _buf(self, like):
        return self._free.pop() if self._free else torch.empty_like(like)

    def corrector_coeffs(self):
        """Coefficients of x_corr = c_last*last + c_m0*m0 + c_m1*m1 + c_mt*m_t at step i (order = self.this_order)."""
        s_t, s_0 = self.sigmas[self.i], self.sigmas[self.i - 1]
        alpha_t = 1.0 - s_t
        h = self._lam(s_t) - self._lam(s_0)
        h_phi_1, B_h, b = self._b(-h, self.this_order)
        if self.this_order == 1:
            rho_t, c_m1, extra_m0 = 0.5, 0.0, 0.0
        else:
            rk = (self._lam(self.sigmas[self.i - 2]) - self._lam(s_0)) / h
            # [[1, 1], [rk, 1]] @ [rho0, rho_t] = [b1, b2]
            rho0 = (b[0] - b[1]) / (1.0 - rk)
            rho_t = b[0] - rho0
            c_m1 = -alpha_t * B_h * rho0 / rk
            extra_m0 = alpha_t * B_h * rho0 / rk
        c_m0 = -alpha_t * h_phi_1 + alpha_t * B_h * rho_t + extra_m0
        return s_t / s_0, c_m0, c_m1, -alpha_t * B_h * rho_t

    def predictor_coeffs(self, order):
        """Coefficients of x_next = c_x*x_corr + c_mt*m_t + c_mp*m_prev at step i."""
        s_t, s_0 = self.sigmas[self.i + 1], self.sigmas[self.i]
        if s_t == 0.0:  # terminal sigma: lambda = +inf, expm1(-inf) = -1 -> the sample becomes the x0 prediction
            return 0.0, 1.0, 0.0
        alpha_t = 1.0 - s_t
        h = self._lam(s_t) - self._lam(s_0)
        h_phi_1, B_h, _ = self._b(-h, order)
        c_mt, c_mp = -alpha_t * h_phi_1, 0.0
        if order == 2:
            rk = (self._lam(self.sigmas[self.i - 1]) - self._lam(s_0)) / h
            c_mp = -alpha_t * B_h * 0.5 / rk
            c_mt -= c_mp
        return s_t / s_0, c_mt, c_mp

    def step(self, cond, uncond, guide_scale, x):
        """cond / uncond: the two forwards' outputs at (x, sigma_i), fp32, same shape as x. Returns the next sample (a tensor
        owned by the sampler until the next call)."""
        sig = self.sigmas[self.i]
        m_t, x_corr = self._buf(x), self._buf(x)
        if self.i > 0 and self._last is not None:
            c_last, c_m0, c_m1, c_mt = self.corrector_coeffs()
            hist, coef = [self._last, self._m[-1]], [c_last, c_m0]
            if self.this_order == 2:
                hist.append(self._m[-2])
                coef.append(c_m1)
            # m_t = x - sigma*v, so c_mt*m_t = c_mt*x - c_mt*sigma*v
            ops.cfg_step(cond, uncond, guide_scale, x, -c_mt * sig, coef_x=c_mt, hist=hist, coef_h=coef, sigma=sig, out=x_corr, x0_out=m_t)
        else:
            ops.cfg_step(cond, uncond, guide_scale, x, 0.0, coef_x=1.0, sigma=sig, out=x_corr, x0_out=m_t)
        self._m.append(m_t)
        if len(self._m) > self.order:
            self._free.append(self._m.pop(0))
        n_steps = len(self.sigmas) - 1
        self.this_order = min(min(self.order, n_steps - self.i), self.lower_order_nums + 1)
        if self._last is not None:
            self._free.append(self._last)
        self._last = x_corr
        c_x, c_mt, c_mp = self.predictor_coeffs(self.this_order)
        out = self._buf(x)
        hist, coef = ([self._m[-2]], [c_mp]) if self.this_order == 2 else ([], [])
        # second launch: no guidance (cond = uncond = m_t, g = 0 gives v = m_t exactly)
        ops.cfg_step(m_t, m_t, 0.0, x_corr, c_mt, coef_x=c_x, hist=hist, coef_h=coef, out=out)
        if self.lower_order_nums < self.order:
            self.lower_order_nums += 1
        self.i += 1
        return out


class FlowDPMSolverSampler:
    """DPM-Solver++ (Lu et al. 2022, "DPM-Solver++: Fast Solver for Guided Sampling of Diffusion Probabilistic Models"): data
    (x0) prediction, multistep, order 2 with the midpoint update, first order on the first step (no history yet) and on the last
    (lower_order_final: sigma_next = 0), on the flow parameterisation alpha = 1 - sigma, lambda = log(alpha) - log(sigma). It
    stands in for upstream Wan's `FlowDPMSolverMultistepScheduler` (`--sample_solver dpm++`, MagCache4Wan2.1/magcache_generate.py:
    728-731, MagCache4Wan2.2/magcache_generate.py:526-529). PARITY UNPINNED: that scheduler is upstream Wan code which is not in the
    reference tree; what follows restates the published algorithm with the configuration Wan constructs it with, as far as it is
    known without that source (algorithm "dpmsolver++", solver_order 2, "midpoint", lower_order_final, final sigma 0, the
    scheduler's own shift 1 over the caller's `sampling_sigmas(steps, shift)`, timestep = 1000 * sigma); none of it could be checked
    against upstream's code.

    Per step, with s the current and t the next sigma, h = lambda_t - lambda_s, m0 = x - sigma_s * v (v the guided flow
    prediction) and m1 the previous step's m0:
        order 1:  x_t = (sigma_t / sigma_s) x - alpha_t (e^-h - 1) m0
        order 2:  x_t = (sigma_t / sigma_s) x - alpha_t (e^-h - 1) D0 - 1/2 alpha_t (e^-h - 1) D1,   D0 = m0, D1 = (m0 - m1) / r0,
                  r0 = (lambda_s - lambda_{s-1}) / h
    folded on the host into float64 scalars, out = cx * x + cv * v + ch * m1 (`coeffs`), and ONE `mc_cfg_step` launch per step that
    also writes m0 for the next step. The first-order update equals the Euler step x + (sigma_t - sigma_s) v in exact arithmetic
    (alpha_t (e^-h - 1) = sigma_t / sigma_s - 1). `denoise` folds the launch into the unconditional call's head on the unsharded Wan
    engine (`cfg_denoise_step` -> `mc_head_unpatchify_step_hist`), so a step whose two calls hit the cache is two head launches.
    The latent is updated in place; the two x0-prediction buffers are the sampler's own and are recycled."""

    def __init__(self, sigmas, order=2):
        if order not in (1, 2):
            raise NotImplementedError("FlowDPMSolverSampler: solver order 1 or 2 (Wan constructs the scheduler with order 2)")
        self.sigmas = [float(s) for s in sigmas]
        self.order = order
        self.i = 0
        self._m = None  # [previous x0-prediction (zeros before the first step), this step's], device tensors swapped every step

    @property
    def timestep(self):
        return 1000.0 * self.sigmas[self.i]

    @staticmethod
    def _lam(sigma):
        """lambda = log(1 - sigma) - log(sigma), with the two ends of a flow schedule stated: the terminal sigma 0 has lambda = +inf
        (its update returns the x0-prediction), sigma 1 (where `sampling_sigmas` starts) has lambda = -inf (h = +inf: e^-h = 0)."""
        if sigma == 0.0:
            return math.inf
        if sigma == 1.0:
            return -math.inf
        return math.log(1.0 - sigma) - math.log(sigma)

    def step_order(self, i=None):
        """1 on the first and the last step, else the solver order."""
        i = self.i if i is None else i
        return 1 if self.order == 1 or i == 0 or i == len(self.sigmas) - 2 else 2

    def coeffs(self, i=None):
        """(cx, cv, ch) of step i, float64: out = cx * x + cv * v + ch * m1."""
        i = self.i if i is None else i
        s_s, s_t = self.sigmas[i], self.sigmas[i + 1]
        h = self._lam(s_t) - self._lam(s_s)
        a = (1.0 - s_t) * math.expm1(-h)  # alpha_t (e^-h - 1): -alpha_t from sigma_s = 1, -1 into sigma_t = 0
        ratio = s_t / s_s
        if self.step_order(i) == 1:
            # x_t = ratio x - a (x - sigma_s v)
            return ratio - a, a * s_s, 0.0
        r0 = (self._lam(s_s) - self._lam(self.sigmas[i - 1])) / h
        ch = 0.5 * a / r0  # -1/2 a D1 = -(a / (2 r0)) m0 + (a / (2 r0)) m1; 0 after a sigma-1 step (r0 = +inf)
        b = a + ch         # the whole weight of m0 = x - sigma_s v
        return ratio - b, b * s_s, ch

    def _bufs(self, like):
        m = self._m
        if m is None or m[0].shape != like.shape or m[0].device != like.device or m[0].dtype != like.dtype:
            m = self._m = [torch.zeros_like(like), torch.zeros_like(like)]
        return m

    def _advance(self):
        self._m.reverse()  # this step's x0-prediction is the next step's history
        self.i += 1

    def step(self, cond, uncond, guide_scale, x):
        """cond / uncond: the two forwards' outputs at (x, sigma_i), fp32, same shape as x. x is updated in place and returned."""
        cx, cv, ch = self.coeffs()
        m1, m0 = self._bufs(x)
        ops.cfg_step(cond, uncond, guide_scale, x, cv, coef_x=cx, hist=[m1], coef_h=[ch], sigma=self.sigmas[self.i], out=x, x0_out=m0)
        self._advance()
        return x

    def denoise(self, model, x, t, context, context_null, seq_len, guide_scale, **kw):
        """One whole step of the caller loop (wan_magcache.py:296-310), as `FlowEulerSampler.denoise`: cond call, uncond call, CFG
        combine, scheduler update; the latent `x` [C, F, H, W] is updated in place and returned."""
        cx, cv, ch = self.coeffs()
        m1, m0 = self._bufs(x)
        out = cfg_denoise_step(model, x, t, context, context_null, seq_len, guide_scale, coef_v=cv, coef_x=cx, hist=m1, coef_h=ch,
                               sigma=self.sigmas[self.i], x0_out=m0, **kw)
        self._advance()
        return out
