"""`mc_opensora_head` on the GPU: plain mode, the cache-hit form and step mode, each bit-equal to the op chain it replaces
(ops.cache_hit_add -> ops.ln_t2i_modulate per sample -> ops.gemm -> unpatchify / crop / .float(), then the reference's sampler
statements), with NaN-poisoned margins around every input and fenced outputs; and a 480p x 51-frame, 30-step video under MagCache
0.12 / K3 whose every latent is bit-equal with the fused sampler and with the engine's forward followed by the reference's statements."""
import copy

import pytest
import torch

from magcache_b200 import _lib as L
from magcache_b200 import ops, patch as patch_mod
from magcache_b200.sampler import OpenSoraRFlowSampler

import opensora_ref as R

pytestmark = pytest.mark.gpu
dev = "cuda"
BF = torch.bfloat16
PAD = 4096  # elements of poison / fence on each side


def _poisoned(t):
    """`t` copied into the middle of a buffer whose margins are NaN (bf16 / fp32): a read past either end shows in the output."""
    buf = torch.full((t.numel() + 2 * PAD,), float("nan"), dtype=t.dtype, device=dev)
    mid = buf[PAD:PAD + t.numel()].view(t.shape)
    mid.copy_(t)
    return mid


def _fenced(shape, fill=None):
    buf = torch.full((int(torch.Size(shape).numel()) + 2 * PAD,), -7.25, dtype=torch.float32, device=dev)
    mid = buf[PAD:PAD + torch.Size(shape).numel()].view(shape)
    if fill is not None:
        mid.copy_(fill)
    return buf, mid


def _fence_intact(buf):
    return bool((buf[:PAD] == -7.25).all() and (buf[-PAD:] == -7.25).all())


def _operands(B, T, H, W, D, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    R_ = B * T * H * W
    x = (torch.randn(R_, D, generator=g) * 1.5 + 0.3).to(BF)
    res = (torch.randn(R_, D, generator=g) * 0.7).to(BF)
    mod = (torch.randn(B, 2, D, generator=g) * 0.2).to(BF).float()
    w = (torch.randn(32, D, generator=g) / D ** 0.5).to(BF)
    bias = (0.05 * torch.randn(32, generator=g)).to(BF).float()
    return [t.to(dev) for t in (x, res, mod, w, bias)]


def _chain(x, res, mod, w, bias, B, T, H, W, Hx, Wx):
    """OpenSoraEngine.head's launches (and the hit add in front of it)."""
    N, D = T * H * W, x.shape[1]
    if res is not None:
        x = ops.cache_hit_add(x, res)
    h = torch.empty_like(x)
    for b in range(B):
        ops.ln_t2i_modulate(x[b * N:(b + 1) * N], mod[b], 1, 0, out=h[b * N:(b + 1) * N])
    o = ops.gemm(h, w, bias, L.MC_EPI_BIAS_BF16)
    o = o.view(B, T, H, W, 1, 2, 2, 8).permute(0, 7, 1, 4, 2, 5, 3, 6).reshape(B, 8, T, 2 * H, 2 * W)
    return o[:, :, :T, :Hx, :Wx].float()


SHAPES = [  # B, T, H, W, Hx, Wx, D: odd crops, T = 1 / 15 / 60, B = 2 / 4, row counts on and off the 64-row tile, a K tail (D = 144)
    (2, 1, 3, 5, 5, 9, 1152),
    (2, 15, 6, 10, 12, 19, 1152),
    (4, 60, 3, 4, 6, 8, 1152),
    (4, 15, 5, 7, 9, 13, 144),
    (2, 1, 1, 1, 1, 2, 1152),
]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"B{s[0]}-T{s[1]}-{s[2]}x{s[3]}-crop{s[4]}x{s[5]}-D{s[6]}" for s in SHAPES])
@pytest.mark.parametrize("hit", [False, True], ids=["stream", "hit"])
def test_plain_and_step_bit_equal_to_op_chain(shape, hit):
    B, T, H, W, Hx, Wx, D = shape
    x, res, mod, w, bias = _operands(B, T, H, W, D, seed=sum(shape) + hit)
    r = res if hit else None
    want = _chain(x, r, mod, w, bias, B, T, H, W, Hx, Wx)
    px, pr, pm, pw = _poisoned(x), _poisoned(res) if hit else None, _poisoned(mod), _poisoned(w)
    buf, out = _fenced((B, 8, T, Hx, Wx))
    got = ops.opensora_head(px, pm, pw, bias, (T, H, W), (T, Hx, Wx), res=pr, out=out)
    torch.cuda.synchronize()
    assert _fence_intact(buf)
    assert torch.equal(got, want), (got - want).abs().max().item()
    # step mode: z + (u + g (c - u)) dt over the velocity channels, out aliasing z
    g = 7.0
    dt = torch.tensor([0.0331, 0.0125][:B // 2], device=dev)
    z0 = torch.randn(B // 2, 4, T, Hx, Wx, device=dev)
    pred_cond, pred_uncond = want.chunk(2, dim=1)[0].chunk(2, dim=0)
    v_pred = pred_uncond + g * (pred_cond - pred_uncond)
    z_want = z0 + v_pred * dt[:, None, None, None, None]
    zbuf, z = _fenced(z0.shape, z0)
    got = ops.opensora_head(px, pm, pw, bias, (T, H, W), (T, Hx, Wx), res=pr, step=(z, g, dt), out=z)
    torch.cuda.synchronize()
    assert _fence_intact(zbuf) and got.data_ptr() == z.data_ptr()
    assert torch.equal(got, z_want), (got - z_want).abs().max().item()


def test_bad_arguments_are_refused():
    x, res, mod, w, bias = _operands(2, 1, 2, 2, 1152, 0)
    with pytest.raises(L.MagCacheError, match="crop"):
        ops.opensora_head(x, mod, w, bias, (1, 2, 2), (1, 2, 2))
    assert L.lib.mc_opensora_head(x.data_ptr(), None, 2, 1, 2, 2, 1152, mod.data_ptr(), w.data_ptr(), bias.data_ptr(), 4, 1e-6, 4, 4,
                                  None, None, 0.0, x.data_ptr(), None) == L.MC_ERR_INVALID
    assert L.lib.mc_opensora_head(x.data_ptr(), None, 1, 1, 2, 2, 1152, mod.data_ptr(), w.data_ptr(), bias.data_ptr(), 8, 1e-6, 4, 4,
                                  x.data_ptr(), None, 0.0, x.data_ptr(), None) == L.MC_ERR_INVALID


# ---- a whole 480p x 51-frame video (latent 15 x 60 x 107: odd width, cropped) -------------------------------------------------------
class _Unfused:
    """Hides the installed forward from the sampler: its unfused path runs the engine's forward, then the reference's statements."""

    def __init__(self, m):
        self.m, self.x_embedder = m, m.x_embedder

    def __call__(self, *a, **k):
        return self.m(*a, **k)


def _video(model, wrap, z, args, y_null):
    calls = []
    hook = model.register_forward_hook(lambda mod, a, out: calls.append((a[0][:1].float().clone(), mod.skip_steps, mod.t)))
    try:
        with torch.no_grad():
            out = OpenSoraRFlowSampler().sample(_Unfused(model) if wrap else model, z, copy.copy(args), y_null, dev, progress=False)
    finally:
        hook.remove()
    return calls, out


def test_full_size_video_480p_51_frames():
    model = R.STDiT3(**R.CONFIGS["full"]).init_synthetic(0).to(dev, BF).eval()
    model.__class__ = type("OursOSFull", (R.STDiT3,), {})
    g = torch.Generator(device="cpu").manual_seed(5)
    z = torch.randn(1, 4, 15, 60, 107, generator=g).to(dev, BF)
    y = torch.randn(1, 1, 300, 4096, generator=g).to(dev)
    y_null = torch.randn(1, 1, 300, 4096, generator=g).to(dev)
    cap = torch.zeros(1, 300, dtype=torch.long, device=dev)
    cap[:, :37] = 1
    bf = dict(dtype=BF, device=dev)
    args = dict(y=y, mask=cap, fps=torch.tensor([24], **bf), height=torch.tensor([480], **bf), width=torch.tensor([854], **bf),
                num_frames=torch.tensor([51], **bf))
    runs = []
    for wrap in (False, True):
        patch_mod.init_magcache_opensora(model, thresh=0.12, K=3)
        runs.append(_video(model, wrap, z, args, y_null))
    (fc, fz), (pc, pz) = runs
    assert len(fc) == len(pc) == 30
    for i, (a, b) in enumerate(zip(fc, pc)):
        assert torch.equal(a[0], b[0]), i
        assert a[1:] == b[1:], (i, a[1:], b[1:])
    assert torch.equal(fz, pz) and torch.isfinite(fz).all()
    assert max(c[1] for c in fc) > 0  # some steps hit the cache
