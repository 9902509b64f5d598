"""Test infrastructure: a float64 tensor-form restatement of DPM-Solver++ 2M on the flow parameterisation, the reference for
`magcache_b200.sampler.FlowDPMSolverSampler` (the `sample_solver == 'dpm++'` branch of the caller loop,
eval/magcache/experiments/Wan2.1_EVAL/wan_magcache.py:270-279, 289-310).

PARITY UNPINNED, like oracle/sampler_ref.py's UniPC: the scheduler (`FlowDPMSolverMultistepScheduler`, upstream Wan-Video
`wan/utils/fm_solvers.py`) is not under the reference tree. What follows states the published algorithm (Lu et al. 2022,
DPM-Solver++, data prediction, multistep order 2, the "midpoint" second-order update, first order on the first step and on the
last, whose sigma is 0) with the configuration Wan builds the scheduler with, as far as it is known without its source: alpha = 1 -
sigma, lambda = log(alpha) - log(sigma), the caller's `get_sampling_sigmas` schedule with the terminal 0 appended and no second
shift. The statements are the paper's, evaluated on torch float64 tensors, so the ends of the schedule follow IEEE arithmetic
(log 0 = -inf): sigma 1 gives lambda = -inf, sigma 0 gives +inf, and e^-inf = 0.
"""
import torch

from oracle import sampler_ref


class DPMppRef:
    """DPM-Solver++ 2M, predict-x0, solver_order 2 (1: first order throughout), lower_order_final."""

    def __init__(self, sigmas, order=2):
        self.sigmas = torch.as_tensor(sigmas, dtype=torch.float64)
        self.order = order
        self.i = 0
        self.model_outputs = [None] * order
        self.lower_order_nums = 0
        self.this_order = 1

    @staticmethod
    def _lam(sigma):
        alpha = 1.0 - sigma
        return torch.log(alpha) - torch.log(sigma)

    def step(self, v, x):
        """v: guided flow prediction at (x, sigma_i). Returns the next sample."""
        x, v = x.double(), v.double()
        s_s, s_t = self.sigmas[self.i], self.sigmas[self.i + 1]
        m0 = x - s_s * v  # flow prediction -> data (x0) prediction
        self.model_outputs = self.model_outputs[1:] + [m0]
        n_steps = len(self.sigmas) - 1
        lower_final = self.i == n_steps - 1
        self.this_order = 1 if (self.order == 1 or self.lower_order_nums < 1 or lower_final) else 2
        alpha_t = 1.0 - s_t
        h = self._lam(s_t) - self._lam(s_s)
        if self.this_order == 1:
            x_t = (s_t / s_s) * x - (alpha_t * (torch.exp(-h) - 1.0)) * m0
        else:
            m1 = self.model_outputs[-2]
            h_0 = self._lam(s_s) - self._lam(self.sigmas[self.i - 1])
            r0 = h_0 / h
            D0, D1 = m0, (1.0 / r0) * (m0 - m1)
            x_t = (s_t / s_s) * x - (alpha_t * (torch.exp(-h) - 1.0)) * D0 - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1
        if self.lower_order_nums < self.order:
            self.lower_order_nums += 1
        self.i += 1
        return x_t


def ref_coeffs(sigmas, order=2):
    """(cx, cv, ch) of every step and the order schedule, read out of DPMppRef's own statements: the update is linear in (x, v, m1),
    so on x = e0, v = e1 with the previous x0-prediction m1 = e2 the next sample is exactly (cx, cv, ch)."""
    ref = DPMppRef(sigmas, order)
    e = torch.eye(3, dtype=torch.float64)
    out, orders = [], []
    for i in range(len(ref.sigmas) - 1):
        ref.i, ref.lower_order_nums = i, min(i, order)
        ref.model_outputs = [None] * (order - 1) + [e[2]]
        y = ref.step(e[1], e[0])
        out.append(tuple(float(c) for c in y))
        orders.append(ref.this_order)
    return out, orders


def denoise(model_v, x, sigmas, guide, sampler="dpm++"):
    """oracle.sampler_ref.denoise with DPM++ 2M as well: model_v(x, sigma, branch) -> flow prediction (cond first, then uncond)."""
    if sampler != "dpm++":
        return sampler_ref.denoise(model_v, x, sigmas, guide, sampler)
    s = DPMppRef(sigmas)
    for i in range(len(sigmas) - 1):
        v = sampler_ref.cfg(model_v(x, sigmas[i], 0), model_v(x, sigmas[i], 1), guide)
        x = s.step(v, x)
    return x
