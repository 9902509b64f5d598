"""DPM++ 2M on the H100: `mc_head_unpatchify_step_hist` (the unconditional head with the solver's update in its epilogue: CFG
combine, the one history term, the x0-prediction) bit-equal to `mc_head_unpatchify_ex` followed by `mc_cfg_step(hist, x0_out)`,
and `FlowDPMSolverSampler.denoise` over a Wan2.1 loop.

* Edge shapes: the CTA geometries of test_head_readout_gpu.py (`geometry_rows`: one row, 17, the 16-rows-per-CTA clamp, ragged
  tail boxes, a last CTA with fewer tiles, the bench row count) at cols 64 / 128 / 1536 (and three of them at 5120), as token-range
  launches into fenced outputs (test_kernel_bounds_gpu.py's `fenced` / `check_fence`): the latent is updated in place (out = x),
  x0_out is a fenced window of its own, cond and hist hold NaN at every position the launch does not own. Miss (fp32 stream) and
  hit (bf16 patch embedding + fp32 residual) forms; x0_out given and omitted.
* The benchmarked latent 16 x 21 x 60 x 104 (32 760 tokens, dim 1536), whole token range, in place, fenced.
* A 10-step Wan2.1 loop at the 1.3B width (dim 1536, ffn 8960, 12 heads) and two blocks, MagCache on: `denoise` (fused) bit-equal
  to the two patched calls + `FlowDPMSolverSampler.step` every step, the hit / miss sequence the controller's, and the final
  latent no further from an fp64 evaluation of the same loop than 1.5x the bf16 CPU oracle's distance (+1e-4), the criterion of
  test_wan_forward_gpu.py.
"""
import copy

import pytest
import torch

from test_head_readout_gpu import _grid, _tokens, geometry_rows, make_rows, modulation
from test_kernel_bounds_gpu import _fill_bytes_ok, check_fence, fenced

DEV = "cuda"
BF, F32 = torch.bfloat16, torch.float32


def _ops():
    from magcache_b200 import ops
    return ops


def _coefs():
    """(g, cx, cv, ch, sigma) of a second-order step of a 10-step schedule at shift 5 (ch != 0)."""
    from magcache_b200.sampler import FlowDPMSolverSampler, sampling_sigmas
    smp = FlowDPMSolverSampler(sampling_sigmas(10, 5.0))
    cx, cv, ch = smp.coeffs(3)
    assert smp.step_order(3) == 2 and ch != 0.0
    return 5.0, cx, cv, ch, smp.sigmas[3]


class _HistCase:
    """Head rows for the token range [off, off + rows) of `grid`: x (fp32 stream), x0 / r (hit), each with 128 NaN rows after it;
    the latent window (updated in place) and the x0 window in fenced 1-D buffers; cond and hist with NaN off the range."""

    def __init__(self, rows, cols, grid, off, g):
        self.rows, self.cols, self.grid, self.off = rows, cols, grid, off
        target = make_rows(rows, cols, g)
        self.x, _ = fenced((rows, cols), F32, (0, 128, 0, 0), pitch=cols)
        self.x.copy_(target)
        self.x0, _ = fenced((rows, cols), BF, (0, 128, 0, 0), pitch=cols)
        self.x0.copy_(target.to(BF))
        self.r, _ = fenced((rows, cols), F32, (0, 128, 0, 0), pitch=cols)
        self.r.copy_(target - self.x0.float() + 1e-2 * torch.randn(rows, cols, generator=g, device=DEV))
        F, Hp, Wp = grid
        self.shape = (16, F, 2 * Hp, 2 * Wp)
        self.n = 16 * F * 4 * Hp * Wp
        tok = torch.zeros(F * Hp * Wp, dtype=torch.bool, device=DEV)
        tok[off:off + rows] = True
        self.own = tok
        pos = _tokens(torch.arange(self.n, device=DEV), grid)
        self.own_idx, other = pos[tok].reshape(-1), pos[~tok].reshape(-1)
        self.cond = torch.randn(self.n, generator=g, device=DEV)
        self.hist = torch.randn(self.n, generator=g, device=DEV)
        self.cond[other] = float("nan")
        self.hist[other] = float("nan")
        self.lat = torch.randn(self.n, generator=g, device=DEV)
        self.out, self.obuf = fenced((self.n,), F32, (0, 0, 8, 8), fill="fence")
        self.x0o, self.x0buf = fenced((self.n,), F32, (0, 0, 8, 8), fill="fence")

    def _head(self, form, prep, **kw):
        hm_e_w_b = prep[1]
        if form == "miss":
            return _ops().head_unpatchify(self.x, *hm_e_w_b, self.grid, row_offset=self.off, prep=prep[0], **kw)
        return _ops().head_unpatchify(self.x0, *hm_e_w_b, self.grid, residual=self.r, row_offset=self.off, prep=prep[0], **kw)

    def fused(self, form, prep, coefs, with_x0=True):
        g, cx, cv, ch, sig = coefs
        self.obuf.view(torch.uint8).fill_(0xA5)
        self.x0buf.view(torch.uint8).fill_(0xA5)
        self.out[self.own_idx] = self.lat[self.own_idx]
        out = self.out.view(self.shape)
        x0 = self.x0o.view(self.shape) if with_x0 else None
        self._head(form, prep, out=out, step=(self.cond.view(self.shape), out, g, cx, cv), step_hist=(self.hist.view(self.shape), ch, sig, x0))
        check_fence(self.out, self.obuf)
        check_fence(self.x0o, self.x0buf)
        t_out, t_x0 = _tokens(self.out, self.grid), _tokens(self.x0o, self.grid)
        assert bool(_fill_bytes_ok(t_out[~self.own]).all()), (form, self.rows, self.cols, "a store landed on another token")
        assert bool(_fill_bytes_ok(t_x0[~self.own]).all()), (form, self.rows, self.cols, "an x0 store landed on another token")
        if not with_x0:
            assert bool(_fill_bytes_ok(t_x0).all()), "x0_out omitted, yet written"
        return t_out[self.own], t_x0[self.own]

    def unfused(self, form, prep, coefs):
        """The op chain the fused launch replaces: the plain head (token range), then mc_cfg_step over the whole tensors."""
        g, cx, cv, ch, sig = coefs
        y = torch.zeros(self.shape, device=DEV)
        self._head(form, prep, out=y)
        out, x0 = torch.empty(self.n, device=DEV), torch.empty(self.n, device=DEV)
        _ops().cfg_step(self.cond, y.view(-1), g, self.lat, cv, coef_x=cx, hist=[self.hist], coef_h=[ch], sigma=sig, out=out, x0_out=x0)
        return _tokens(out, self.grid)[self.own], _tokens(x0, self.grid)[self.own]


def _prep(cols, g):
    hm, e, _, _ = modulation(cols, g)
    W = torch.randn(cols, 64, generator=g, device=DEV) * 0.05
    b = torch.randn(64, generator=g, device=DEV) * 0.1
    return _ops().head_prepare(hm, e, W, b), (hm, e, W, b)


def _check(case, g, label, x0_variants=(True,)):
    prep, coefs = _prep(case.cols, g), _coefs()
    for form in ("miss", "hit"):
        want_out, want_x0 = case.unfused(form, prep, coefs)
        assert bool(torch.isfinite(want_out).all()), (label, form)
        for with_x0 in x0_variants:
            got_out, got_x0 = case.fused(form, prep, coefs, with_x0)
            assert torch.equal(got_out, want_out), (label, form, with_x0, "out")
            if with_x0:
                assert torch.equal(got_x0, want_x0), (label, form, "x0")


@pytest.mark.gpu
@pytest.mark.parametrize("cols", [64, 128, 1536, 5120])
def test_step_hist_edge_shapes_fenced(cols):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    geo = geometry_rows(sms)
    names = list(geo) if cols <= 1536 else ["17", "16sm-1", "128sm-5"]
    g = torch.Generator(device=DEV).manual_seed(100 + cols)
    for k, name in enumerate(names):
        rows = geo[name]
        grid, off = _grid(rows)
        _check(_HistCase(rows, cols, grid, off, g), g, f"cols {cols} rows {rows} ({name})", (True, False) if k == 0 else (True,))
        torch.cuda.empty_cache()


@pytest.mark.gpu
def test_step_hist_benchmarked_shape():
    """The bench's latent 16 x 21 x 60 x 104 at dim 1536: the whole token range, the latent updated in place."""
    g = torch.Generator(device=DEV).manual_seed(7)
    grid = (21, 30, 52)
    _check(_HistCase(21 * 30 * 52, 1536, grid, 0, g), g, "bench", (True, False))


@pytest.mark.gpu
def test_wan21_dpm_loop_fused_equals_unfused_and_holds_to_fp64():
    import magcache_b200 as mc
    from magcache_b200 import ops
    from oracle import sampler_ref, wan_ref

    import dpm_solver_ref as R

    steps, guide, kw = 10, 5.0, dict(thresh=0.12, K=2, retention_ratio=0.2)
    table = mc.tables()["wan2.1_t2v_1.3b"]
    dims = dict(wan_ref.CONFIGS["t2v-1.3B"], num_layers=2)
    model = wan_ref.WanModel(**dims, text_dim=4096, text_len=512).init_synthetic(0)

    def ours():
        m = copy.deepcopy(model).to(DEV)
        m.__class__ = type("OurWan", (model.__class__,), {})
        mc.init_magcache(m, steps, mag_ratios=table, **kw)
        return m

    def ref(double):
        m = copy.deepcopy(model)
        if double:
            m = m.double()
        m.__class__ = type("RefWan", (model.__class__,), {})
        wan_ref.install_magcache(m.__class__, table, steps, **kw)
        return m

    a_model, b_model, r_model, r64 = ours(), ours(), ref(False), ref(True)
    gen = torch.Generator().manual_seed(5)
    lat = torch.randn(16, 2, 16, 24, generator=gen)
    ctx, ctx_null = torch.randn(37, 4096, generator=gen), torch.randn(32, 4096, generator=gen)
    n_tok = 2 * 8 * 12
    sig = mc.sampling_sigmas(steps, 5.0)
    sa, sb = mc.FlowDPMSolverSampler(sig), mc.FlowDPMSolverSampler(sig)
    sr, sr64 = R.DPMppRef(torch.tensor(sig, dtype=torch.float64)), R.DPMppRef(torch.tensor(sig, dtype=torch.float64))
    ctx_d, ctxn_d = ctx.to(DEV), ctx_null.to(DEV)
    xa, xb, xr, x64 = lat.to(DEV), lat.to(DEV), lat.clone(), lat.double()
    kinds, launches = [], []
    with torch.no_grad():
        for i in range(steps):
            t = torch.tensor([sa.timestep], dtype=torch.float32)
            td = t.to(DEV)
            cond = a_model([xa], t=td, context=[ctx_d], seq_len=n_tok)[0]
            uncond = a_model([xa], t=td, context=[ctxn_d], seq_len=n_tok)[0]
            xa = sa.step(cond, uncond, guide, xa)
            n0 = ops.LAUNCHES
            out = sb.denoise(b_model, xb, td, ctx_d, ctxn_d, n_tok, guide)
            launches.append(ops.LAUNCHES - n0)
            assert out.data_ptr() == xb.data_ptr()
            assert torch.equal(xa, xb) and torch.equal(sa._m[0], sb._m[0]), i
            for attr in ("cnt", "accumulated_ratio", "accumulated_err", "accumulated_steps"):
                assert getattr(a_model, attr) == getattr(b_model, attr), attr
            c_r = r_model([xr], t=t, context=[ctx], seq_len=n_tok)[0]
            kinds.append(int(r_model.last_skip))
            u_r = r_model([xr], t=t, context=[ctx_null], seq_len=n_tok)[0]
            kinds.append(int(r_model.last_skip))
            xr = sr.step(sampler_ref.cfg(c_r, u_r, guide), xr).float()
            with wan_ref.exact_fp64():
                c64 = r64([x64], t=t.double(), context=[ctx.double()], seq_len=n_tok)[0]
                u64 = r64([x64], t=t.double(), context=[ctx_null.double()], seq_len=n_tok)[0]
            x64 = sr64.step(sampler_ref.cfg(c64, u64, guide), x64)
            assert int(r64.last_skip) == kinds[-1]
            rel = float((xb.cpu().double() - xr.double()).norm() / xr.double().norm())
            assert rel < 3e-2, (i, rel)
    want = mc.MagCacheConfig("wan2.1", 0.12, 2, 0.2, steps, table="wan2.1_t2v_1.3b").schedule().tolist()
    assert kinds == want and any(kinds[2 * i] and kinds[2 * i + 1] for i in range(steps))
    assert b_model._mc_engine._step is None
    e_ours = float((xb.cpu().double() - x64).norm() / x64.norm())
    e_ref = float((xr.double() - x64).norm() / x64.norm())
    print(f"[dpm++ loop] rel-L2: ours vs fp64 {e_ours:.3e} | oracle(bf16) vs fp64 {e_ref:.3e}; launches per step {launches}")
    assert e_ours <= 1.5 * e_ref + 1e-4
