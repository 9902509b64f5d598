"""The head (`head_prep_kernel` + `head_tc_kernel`, csrc/head_wgmma.cu) read back one modulated LayerNorm value per output
element, each checked against fp64 with a bound from the kernel's rounding chain, at the CTA geometries the row split makes.

The readout. With b = 0 and Wt[k, c] = 1 if k == 64 j + c, else 0, launch j of the head returns, for every row and each of its 64
output features c, y = LN(v)_k * s_k + t_k at k = 64 j + c, where s = 1 + (mod[1] + e) and t = mod[0] + e in fp32 (the values
the preparation forms). cols / 64 launches read every element of every row back, so an error in one element's mean, rstd, eps or
split is not averaged over the row as it is by a random 64-wide Linear. mod and e are random fp32 values: s is no bf16 value,
W'_lo = bf16(s - bf16(s)) != 0, and both split passes carry weight. One pass with a random Wt and b checks the real Linear.

The chain the file header states, per element k of a row, u = 2^-24 (fp32 unit roundoff), nkc = cols / 64 chunks:
  * v = fp32(x0 + r), rounded to bf16 with round_sum_to_bf16 (hit form), or the fp32 stream: the exact input of the fp64 reference.
  * x^ = fp32(v - p), p the fp32 mean of the row's first 64 elements (the pilot). The reference takes p in fp64; the kernel's
    (16-term sums, two shuffle adds) is within 18 u mean|v[:64]| of it, which X = |v - p| + 18 u mean|v[:64]| carries.
  * The split: x^ = x^_hi + x^_lo + d_x and s = s_hi + s_lo + d_s with bf16 hi and lo: each rounding is within 2^-8 of its
    operand and lo is within 2^-8 of the value, so |d| <= 2^-16 |.|, and the omitted x^_lo W'_lo is <= 2^-16 |x^ s|. acc =
    x^_hi s_hi + x^_lo s_hi + x^_hi s_lo is x^ s within 3 * 2^-16 |x^ s|, plus 8 u for the subtraction and the three fp32
    accumulations (E_SPLIT). c1 = s_hi + s_lo (exact in fp32) is s within 2^-16 |s| (E_C1, + 2 u).
  * The statistics in fp32. Per thread: 16-element chunk sums (each chunk mean within 15 u S, S the largest mean X over the
    16-element slices a thread takes), Chan's update over nkc chunks (each within 5 u S, damped by the later weights to
    (nkc + 1) / 2 of that), two shuffle merges (2 u S each): the shifted mean is within D = (24 + 3 nkc) u S. The M2 sums and
    updates carry at most 6 u per step relative to the second moment Q = mean X^2 (>= var), so rstd is relative within
    E_r = (12 + 3 nkc) u (var + Q) / (var + eps) + 5 u (rsqrtf's 2 ulp, the scale by 1/cols and the eps add).
  * Epilogue y = fma(rstd, acc - mean^ c1, c0): the subtraction u rstd (|acc| + |mean^ c1|), the fma u |y|; c0 = t in the
    readout (exact), fp32(sum t W + b) otherwise (u |c0|).
  * The random-W pass adds the fp32 accumulation over cols in the tensor cores: 12 accumulations per chunk, at most 2 u each
    relative to sum_k |x^_k W'_kc| (GAMMA).
So |y - y64| <= rstd |s| (E_SPLIT X + E_C1 |mean - p|) + rstd |s| D + E_r |LN s| + the epilogue roundings, summed over k
against |W| for the random pass. The bound is worst-case per term; the printed ratio (`pytest -s`) shows the margin.

Rows (one kind per row, cyclic over the launch): plain; a common offset of 1e3 (the pilot must cancel it); three massive
activation columns past the first 64 (1e3 - 1e4); sigma = 1e-3 (variance near eps, where eps's placement shows); all equal and
all zero (y must be t to within the bound: exact, here); late offset (the first 64 columns 500 sigma away from the rest, so the
pilot does not help: x^ is hundreds of sigma and the split's 2^-16 relative error is scaled by it). Late-offset rows are held to
this chain, which is looser than the north star's rtol 1e-3 / atol 1e-4 by the factor |x^| rstd; their ratio to the north star
is printed (about 1 - 1.6 at cols 1536 - 5120 on an H100). The kernel is left as it is for them unless a row from a real engine
run shows the same error.

Forms: the fp32 stream, the cache hit (bf16 patch embedding + fp32 residual), the hit with the sum rounded to bf16, and the
step form (CFG combine + scheduler update in the epilogue, the latent updated in place), the last checked for fences and for
the step arithmetic on the readout (its bit identity to head + cfg_step is tested in test_kernels_gpu.py).

Geometry: the kernel gives each CTA rows_per_cta = max(16, ceil(rows / SMs)) contiguous rows and its last 128-row tile a tail
box of rows_per_cta % 128 rows; the row counts here are computed from the device's SM count (`head_geometry`).

Fences: the output is a window of a 1-D fenced fp32 buffer; every launch is a token-range call, so the positions of the tokens
before and after the range must keep the fence bytes; x and r are the first rows of buffers with 128 NaN rows after them.

`test_head_readout_checker_rejects_each_modelled_mutant` (CPU) runs a torch model of the chain through the same checker. Only it
runs without a GPU; this module imports without initialising CUDA.
"""
import pytest
import torch

from test_kernel_bounds_gpu import _fill_bytes_ok, check_fence, fenced

DEV = "cuda"
BF, F32 = torch.bfloat16, torch.float32
U = 2.0 ** -24
E_SPLIT = 3 * 2.0 ** -16 + 8 * U
E_C1 = 2.0 ** -16 + 2 * U
EPS = 1e-6
KINDS = ("plain", "offset", "massive", "lowvar", "equal", "zero", "late")
FORMS = ("stream", "hit", "hit_round", "step")


def _ops():
    from magcache_b200 import ops
    return ops


def head_geometry(rows, sms):
    """(rows_per_cta, tail_rows, grid, tiles of the last CTA, tiles of a full range) as mc_head_unpatchify_ex computes them."""
    rpc = max(16, -(-rows // sms))
    grid = -(-rows // rpc)
    last = rows - rpc * (grid - 1)
    return rpc, rpc % 128, grid, -(-last // 128), -(-rpc // 128)


def geometry_rows(sms):
    """The row counts of the CTA geometries: one row; 17; the clamp to 16 rows per CTA; one full tile per CTA (no tail box);
    a last CTA short inside a full box; rows_per_cta = 129 (a 1-row tail box, grid < SMs); two full tiles; the bench shape
    (32 760); and a last CTA with fewer tiles than a full range."""
    short_last = next(r for r in range(200 * (sms - 1) + 1, 200 * sms)
                      if (lambda g: g[3] < g[4] and g[1] != 0)(head_geometry(r, sms)))
    rows = {"1": 1, "17": 17, "16sm-1": 16 * sms - 1, "128sm": 128 * sms, "128sm-5": 128 * sms - 5, "128sm+1": 128 * sms + 1,
            "256sm": 256 * sms, "bench": 32760, "short_last": short_last}
    assert head_geometry(rows["16sm-1"], sms)[0] == 16
    assert head_geometry(rows["128sm"], sms)[1] == 0
    assert head_geometry(rows["128sm+1"], sms)[:2] == (129, 1) and head_geometry(rows["128sm+1"], sms)[2] < sms
    assert head_geometry(rows["256sm"], sms)[:2] == (256, 0)
    return rows


# ------------------------------------------------------------------------------------------- inputs
def row_kinds(rows, device):
    return torch.arange(rows, device=device) % len(KINDS)


def make_rows(rows, cols, g, device=DEV):
    """fp32 [rows, cols]: row i of kind KINDS[i % 7] (module docstring)."""
    n = lambda *s: torch.randn(*s, generator=g, device=device)  # noqa: E731
    kind = row_kinds(rows, device)[:, None]
    x = 2.0 * n(rows, cols) + 0.1
    x = torch.where(kind == 1, n(rows, cols) + 1e3, x)
    massive = n(rows, cols)
    cols_m = [(64 + 5) % cols, (64 + 37) % cols, cols - 1]
    for c, mag in zip(cols_m, (1e3, -5e3, 1e4)):
        massive[:, c] = mag
    x = torch.where(kind == 2, massive, x)
    x = torch.where(kind == 3, 0.5 + 1e-3 * n(rows, cols), x)
    x = torch.where(kind == 4, (3.0 * n(rows, 1)).expand(rows, cols), x)
    x = torch.where(kind == 5, torch.zeros_like(x), x)
    late = n(rows, cols)
    late[:, :64] += 500.0
    x = torch.where(kind == 6, late, x)
    return x


def modulation(cols, g, device=DEV):
    """head_mod [2, cols], e [cols] (random fp32) and the s, t the kernel forms from them."""
    hm = torch.randn(2, cols, generator=g, device=device) * 0.3
    e = torch.randn(cols, generator=g, device=device) * 0.3
    return hm, e, 1.0 + (hm[1] + e), hm[0] + e


# ------------------------------------------------------------------------------------------- reference and bound
def head_chain(v, s, t, Wt=None, b=None, eps=EPS):
    """fp64 reference and per-element bound (module docstring) of the head on fp32 rows v [rows, cols]: the readout
    (Wt None: [rows, cols], element k = LN(v)_k s_k + t_k) or the Linear with Wt [cols, 64], b [64] ([rows, 64])."""
    v, s, t = v.double(), s.double(), t.double()
    rows, cols = v.shape
    nkc = cols // 64
    p = v[:, :64].mean(1, keepdim=True)
    dp = 18 * U * v[:, :64].abs().mean(1, keepdim=True)
    X = (v - p).abs() + dp
    mu = v.mean(1, keepdim=True)
    var = (v - mu).pow(2).mean(1, keepdim=True)
    rstd = (var + eps).rsqrt()
    ln_s = (v - mu) * rstd * s
    Mh = (mu - p).abs() + dp
    S = X.view(rows, nkc, 2, 4, 8).mean((2, 4)).amax((1, 2))[:, None]
    D = (24 + 3 * nkc) * U * S
    Q = X.pow(2).mean(1, keepdim=True)
    E_r = (12 + 3 * nkc) * U * (var + Q) / (var + eps) + 5 * U
    if Wt is None:
        mm = mma = lambda a: a  # noqa: E731
        c0 = t.expand(rows, cols)
        gamma = 0.0
    else:
        W = Wt.double()
        mm, mma = (lambda a: a @ W), (lambda a: a @ W.abs())  # noqa: E731
        c0 = mm(t[None]) + b.double()
        gamma = (12 * nkc + 16) * 2 * U
    c1 = mm(s[None])
    lin = mm(ln_s)
    ref = lin + c0
    acc = mma(X * s.abs())
    bound = (rstd * (E_SPLIT + gamma) * acc + rstd * E_C1 * Mh * mma(s.abs()[None]) + rstd * D * c1.abs() + E_r * lin.abs()
             + U * (rstd * (acc + Mh * c1.abs()) + ref.abs()) + (0.0 if Wt is None else U * (c0.abs() + rstd * Mh * c1.abs())))
    return ref, bound


NORTH_STAR = lambda ref: 1e-3 * ref.abs() + 1e-4  # noqa: E731


class HeadReadout:
    """Every launch: |got - ref| <= bound per element (`check`), the worst ratio kept per (label, row kind); `report` prints
    them with the late-offset rows' ratio to the north star."""

    def __init__(self):
        self.worst, self.north = {}, {}

    def check(self, got, ref, bound, kinds, label, what):
        err = (got.double() - ref).abs()
        assert bool(torch.isfinite(got).all()), (what, "non-finite output")
        r = torch.where(err == 0, 0.0, err / bound)
        for i, k in enumerate(KINDS):
            m = kinds == i
            if bool(m.any()):
                key = (label, k)
                self.worst[key] = max(self.worst.get(key, 0.0), float(r[m].max()))
                if k == "late":
                    self.north[label] = max(self.north.get(label, 0.0), float((err / NORTH_STAR(ref))[m].max()))
        worst = float(r.max())
        if worst > 1.0:
            i = int(r.reshape(-1).argmax())
            row = i // r.shape[1]
            raise AssertionError((what, f"row {row} ({KINDS[int(kinds[row])]}): |err| {float(err.reshape(-1)[i]):.3e} > bound "
                                        f"{float(bound.reshape(-1)[i]):.3e} (x{worst:.2f})"))

    def report(self):
        for (label, k), w in sorted(self.worst.items()):
            extra = f", late offset / north star {self.north[label]:.2f}" if k == "late" and label in self.north else ""
            print(f"\nhead readout {label} {k}: worst error / bound {w:.3f}{extra}", end="")
        print()


# ------------------------------------------------------------------------------------------- CPU model of the chain
def _fma32(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def _seqsum(a):
    acc = torch.zeros(a.shape[:-1])
    for i in range(a.shape[-1]):
        acc = acc + a[..., i]
    return acc


def model_head(v, s, t, eps=EPS, mutant=None):
    """head_tc_kernel on the readout, in torch fp32: v [rows, cols] fp32; the four threads of a row each take columns
    [8 sub, 8 sub + 8) and [32 + 8 sub, 32 + 8 sub + 8) of every 64-column chunk. Mutants: "mean" (the row mean) / "rstd"
    (scaled by 1 + 1e-4), "eps_after" (rsqrt(var) + eps), "chan" (n_a one chunk too many), "no_pilot", "drop_lo" (no x^_lo W'_hi pass)."""
    rows, cols = v.shape
    nkc = cols // 64
    sl = v.view(rows, nkc, 2, 4, 8).permute(0, 1, 3, 2, 4).reshape(rows, nkc, 4, 16)
    ps = _seqsum(sl[:, 0])
    ps = ps + ps[:, [1, 0, 3, 2]]
    ps = ps + ps[:, [2, 3, 0, 1]]
    pilot = ps * (1.0 / 64.0)
    if mutant == "no_pilot":
        pilot = torch.zeros_like(pilot)
    xh = sl - pilot[:, None, :, None]
    cm = _seqsum(xh) * (1.0 / 16.0)
    cq = torch.zeros(rows, nkc, 4)
    for i in range(16):
        d = xh[..., i] - cm
        cq = _fma32(d, d, cq)
    mean, m2 = torch.zeros(rows, 4), torch.zeros(rows, 4)
    for kc in range(nkc):
        na = torch.tensor(16.0 * (kc + 1 if mutant == "chan" else kc))
        rn = 1.0 / (na + 16.0)
        delta = cm[:, kc] - mean
        mean = _fma32(delta, 16.0 * rn, mean)
        m2 = m2 + _fma32(delta * delta, na * 16.0 * rn, cq[:, kc])
    for o, idx in ((1, [1, 0, 3, 2]), (2, [2, 3, 0, 1])):
        om, oq = mean[:, idx], m2[:, idx]
        cnt = cols * (0.25 if o == 1 else 0.5)
        delta = om - mean
        mean = 0.5 * (mean + om)
        m2 = m2 + oq + delta * delta * (cnt * 0.5)
    mh = mean[:, :1]
    var = m2[:, :1] * torch.tensor(1.0 / cols, dtype=F32)
    rstd = var.rsqrt() + eps if mutant == "eps_after" else (var + eps).rsqrt()
    if mutant == "mean":  # the row's mean mean^ + p scaled
        mh = mh + 1e-4 * (mh + pilot[:, :1])
    if mutant == "rstd":
        rstd = rstd * (1 + 1e-4)
    x = xh.reshape(rows, nkc, 4, 2, 8).permute(0, 1, 3, 2, 4).reshape(rows, cols)
    hi = x.to(BF).float()
    lo = torch.zeros_like(x) if mutant == "drop_lo" else (x - hi).to(BF).float()
    s_hi = s.to(BF).float()
    s_lo = (s - s_hi).to(BF).float()
    acc = (hi * s_hi + lo * s_hi) + hi * s_lo
    return _fma32(rstd, acc - mh * (s_hi + s_lo), t)


def _passes(got, v, s, t):
    ref, bound = head_chain(v, s, t)
    try:
        HeadReadout().check(got, ref, bound, row_kinds(v.shape[0], "cpu"), "model", "model")
    except AssertionError:
        return False
    return True


def test_head_readout_checker_rejects_each_modelled_mutant():
    """The checker bites (CPU): the faithful model of the kernel's chain passes at cols 64 and 1536 over every row kind; mean
    or rstd 1e-4 off, eps added after rsqrt, a Chan weight one chunk off, no pilot and a dropped lo pass each fail."""
    g = torch.Generator().manual_seed(0)
    for cols in (64, 1536):
        v = make_rows(4 * len(KINDS), cols, g, device="cpu")
        _, _, s, t = modulation(cols, g, device="cpu")
        assert _passes(model_head(v, s, t), v, s, t), cols
        for mutant in ("mean", "rstd", "eps_after", "chan", "no_pilot", "drop_lo"):
            assert not _passes(model_head(v, s, t, mutant=mutant), v, s, t), (cols, mutant)


# ------------------------------------------------------------------------------------------- GPU readout
def _grid(rows):
    """A 3-D token grid holding the rows at token offset 3 with at least two more tokens after them."""
    F = -(-(rows + 5) // 35)
    return (F, 5, 7), 3


def _tokens(out, grid):
    """The output [16, F, 2 Hp, 2 Wp] back in token order: [F * Hp * Wp, 64], feature (q * 2 + r) * 16 + channel."""
    F, Hp, Wp = grid
    return out.view(16, F, Hp, 2, Wp, 2).permute(1, 2, 4, 3, 5, 0).reshape(F * Hp * Wp, 64)


class _Case:
    """One (rows, cols) input: x (fp32 stream), x0 / r (hit), with 128 NaN rows after each; the output window and the latent /
    cond of the step form in fenced buffers."""

    def __init__(self, rows, cols, g):
        self.rows, self.cols = rows, cols
        self.grid, self.off = _grid(rows)
        target = make_rows(rows, cols, g)
        self.x, _ = fenced((rows, cols), F32, (0, 128, 0, 0), pitch=cols)
        self.x.copy_(target)
        self.x0, _ = fenced((rows, cols), BF, (0, 128, 0, 0), pitch=cols)
        self.x0.copy_(target.to(BF))
        # the residual: what bf16 x0 drops of the row, plus noise of the row's own scale (none on the constant rows)
        noise = torch.tensor([1e-2, 1e-2, 1e-2, 1e-4, 0.0, 0.0, 1e-2], device=DEV)[row_kinds(rows, DEV)][:, None]
        self.r, _ = fenced((rows, cols), F32, (0, 128, 0, 0), pitch=cols)
        self.r.copy_(target - self.x0.float() + noise * torch.randn(rows, cols, generator=g, device=DEV))
        F, Hp, Wp = self.grid
        self.n = 16 * F * 4 * Hp * Wp
        self.out, self.obuf = fenced((self.n,), F32, (0, 0, 8, 8), fill="fence")
        self.v = {"stream": self.x, "hit": self.x0.float() + self.r}
        self.v["hit_round"] = self.v["hit"].to(BF).float()
        tok = torch.zeros(F * Hp * Wp, dtype=torch.bool, device=DEV)
        tok[self.off:self.off + rows] = True
        self.own = tok
        pos = _tokens(torch.arange(self.n, device=DEV), self.grid)  # output index of every (token, feature)
        self.own_idx, other_idx = pos[tok].reshape(-1), pos[~tok].reshape(-1)
        self.cond = torch.randn(self.n, generator=g, device=DEV)
        self.cond[other_idx] = float("nan")  # read only at the launch's own tokens
        self.lat = torch.randn(self.n, generator=g, device=DEV)

    def run(self, form, hm, e, Wt, b, prep, step=None):
        ops = _ops()
        self.obuf.view(torch.uint8).fill_(0xA5)
        kw = dict(row_offset=self.off, out=self.out.view(16, self.grid[0], 2 * self.grid[1], 2 * self.grid[2]), prep=prep)
        if form == "stream":
            ops.head_unpatchify(self.x, hm, e, Wt, b, self.grid, **kw)
        else:
            if form == "step":  # the latent at the own tokens, fence bytes elsewhere: updated in place
                self.out[self.own_idx] = self.lat[self.own_idx]
                kw["step"] = (self.cond.view_as(kw["out"]), kw["out"], *step)
            ops.head_unpatchify(self.x0, hm, e, Wt, b, self.grid, residual=self.r, round_sum_to_bf16=form == "hit_round", **kw)
        check_fence(self.out, self.obuf)
        tok = _tokens(self.out, self.grid)
        assert bool(_fill_bytes_ok(tok[~self.own]).all()), (form, self.rows, self.cols, "a store landed on another token")
        return tok[self.own]


def _readout(case, g, rec, label):
    """Every form over cols / 64 readout launches, then the random-W Linear."""
    ops = _ops()
    rows, cols = case.rows, case.cols
    hm, e, s, t = modulation(cols, g)
    kinds = row_kinds(rows, DEV)
    refs = {f: head_chain(case.v[f], s, t) for f in ("stream", "hit", "hit_round")}
    step = (4.5, 0.93, -0.37)
    b0 = torch.zeros(64, device=DEV)
    for j in range(cols // 64):
        Wt = torch.zeros(cols, 64, device=DEV)
        Wt[64 * j + torch.arange(64, device=DEV), torch.arange(64, device=DEV)] = 1.0
        prep = ops.head_prepare(hm, e, Wt, b0)
        sl = slice(64 * j, 64 * j + 64)
        for form in FORMS:
            got = case.run(form, hm, e, Wt, b0, prep, step)
            what = (label, form, rows, cols, j)
            if form == "step":
                # the hit form's y, then the step in fp32 torch ops (each rounded, the order of cfg_step)
                y = case.run("hit", hm, e, Wt, b0, prep)
                c = _tokens(case.cond, case.grid)[case.own]
                xl = _tokens(case.lat, case.grid)[case.own]
                f = lambda a: torch.tensor(a, dtype=F32, device=DEV)  # noqa: E731
                want = f(step[1]) * xl + f(step[2]) * (y + f(step[0]) * (c - y))
                assert torch.equal(got, want), what
                continue
            ref, bound = refs[form]
            rec.check(got, ref[:, sl], bound[:, sl], kinds, f"{label} {form}", what)
    W = torch.randn(cols, 64, generator=g, device=DEV) * 0.05
    b = torch.randn(64, generator=g, device=DEV) * 0.1
    prep = ops.head_prepare(hm, e, W, b)
    for form in ("stream", "hit", "hit_round"):
        got = case.run(form, hm, e, W, b, prep)
        ref, bound = head_chain(case.v[form], s, t, W, b)
        rec.check(got, ref, bound, kinds, f"{label} {form} random-W", (label, form, rows, cols, "random W"))


@pytest.mark.gpu
@pytest.mark.parametrize("cols", [64, 128, 1536, 3072, 5120])
def test_head_readout_fenced(cols):
    """Every element of every row read back and held to the chain's bound, in every form, at every CTA geometry for cols <=
    1536 (at 64 and 128 columns, one or two chunks per row, a converter warp once overwrote the row statistics of the tile the
    epilogue was still reading) (the CTA geometries at 17, 16 SMs - 1 and 128 SMs - 5 rows for the two wide heads, TI2V-5B's 3072 and Wan2.1-14B's
    5120), into fenced token-range outputs from inputs with NaN rows after them."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    geo = geometry_rows(sms)
    names = list(geo) if cols <= 1536 else ["17", "16sm-1", "128sm-5"]
    g = torch.Generator(device=DEV).manual_seed(cols)
    rec = HeadReadout()
    for name in names:
        rows = geo[name]
        _readout(_Case(rows, cols, g), g, rec, f"cols {cols} rows {rows} ({name})")
        torch.cuda.empty_cache()
    rec.report()
