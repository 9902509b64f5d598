"""`mc_dit_forward` (SURVEY §8b; csrc/dit_forward.cu) on the GPU: the natively sequenced forward must produce the SAME BITS as the
Python-sequenced engine — same kernels, operands and order (the launch plans are compared on CPU, tests/test_native_plan_cpu.py) —
for the miss branch (output and the residual it writes) and the hit branch (reading that residual), also through the reference's
own call (`model([x], t=..., context=[...], seq_len=...)` with `native=True`), and against the oracle."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


@pytest.mark.parametrize("dims_kw,grid", [(dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2), (3, 16, 24)),
                                           (dict(dim=1536, ffn_dim=8960, num_heads=12, num_layers=1), (3, 30, 52)),
                                           (dict(dim=1536, ffn_dim=8960, num_heads=12, num_layers=30), (21, 30, 52))])
def test_native_forward_bit_equal_to_python_sequenced(dims_kw, grid):
    import magcache_b200 as mc
    from magcache_b200 import ops
    dims = mc.WanDims(**dims_kw, text_dim=512, text_len=64)
    w = mc.WanWeights.random(dims, torch.device(DEV), seed=3)
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(16, grid[0], 2 * grid[1], 2 * grid[2], generator=g).to(DEV)
    ctx = torch.randn(40, 512, generator=g).to(DEV)
    t = torch.tensor([611.0], device=DEV)
    py, nat = mc.WanEngine(w, native=False), mc.WanEngine(w, native=True)
    outs = {}
    for name, eng in (("py", py), ("nat", nat)):
        eng.stage_inputs(lat, t, ctx)
        n0 = ops.LAUNCHES
        miss = eng.forward("miss", 0).clone()
        n_miss = ops.LAUNCHES - n0
        res = eng.res[0].clone()
        n0 = ops.LAUNCHES
        hit = eng.forward("hit", 0).clone()
        outs[name] = (miss, res, hit, n_miss, ops.LAUNCHES - n0)
    torch.cuda.synchronize()
    assert nat._nat is not None and py._nat is None, "the native engine must really have gone through mc_dit_forward"
    for i, what in enumerate(("miss output", "residual", "hit output")):
        a, b = outs["py"][i], outs["nat"][i]
        assert torch.isfinite(a).all() and torch.equal(a, b), (what, float((a - b).abs().max()))
    assert outs["py"][3] == outs["nat"][3] and outs["py"][4] == outs["nat"][4], "same number of launches"
    # the workspace is the caller's: a second handle on its own workspace gives the same bits again (no hidden state)
    again = mc.NativeWanForward(w)
    again.bind(nat.grid, nat._rope_for(nat.grid))
    res2 = torch.empty_like(outs["nat"][1])
    m2 = again.forward(nat.s_lat, nat.s_t, nat.ctx_in, False, res2)
    h2 = again.forward(nat.s_lat, nat.s_t, None, True, res2)
    assert torch.equal(m2, outs["nat"][0]) and torch.equal(res2, outs["nat"][1]) and torch.equal(h2, outs["nat"][2])
    again.close()


def test_native_patched_forward_follows_the_oracle():
    """The reference's call with the natively sequenced engine underneath: same skip sequence and controller state as the oracle,
    outputs to the bf16-pipeline tolerance of tests/test_wan_forward_gpu.py, and bit-equal to the Python-sequenced engine."""
    import magcache_b200 as mc
    from oracle import wan_ref
    model = wan_ref.WanModel(**wan_ref.CONFIGS["tiny"], text_dim=512, text_len=64).init_synthetic(0)
    g = torch.Generator().manual_seed(2)
    lat, ctx, ctx_null = torch.randn(16, 3, 16, 24, generator=g), torch.randn(37, 512, generator=g), torch.randn(30, 512, generator=g)
    n_tok = 3 * 8 * 12
    table = mc.tables()["wan2.1_t2v_1.3b"]
    ref = copy.deepcopy(model)
    ref.__class__ = type("RefN", (ref.__class__,), {})
    wan_ref.install_magcache(type(ref), table, 6, thresh=0.5, K=2, retention_ratio=0.2)
    ours = {}
    for name, native in (("py", False), ("nat", True)):
        m = copy.deepcopy(model).to(DEV)
        m.__class__ = type("Our" + name, (m.__class__,), {})
        mc.init_magcache(m, 6, table="wan2.1_t2v_1.3b", thresh=0.5, K=2, retention_ratio=0.2)
        object.__setattr__(m, "_mc_engine", mc.WanEngine(mc.WanWeights.from_module(m, torch.device(DEV)), native=native))
        ours[name] = m
    kinds = []
    with torch.no_grad():
        for call in range(12):
            t = torch.tensor([900.0 - 120.0 * (call // 2)])
            c = ctx if call % 2 == 0 else ctx_null
            a = ref([lat], t=t, context=[c], seq_len=n_tok)[0]
            kinds.append(int(ref.last_skip))
            b = {k: m([lat.to(DEV)], t=t.to(DEV), context=[c.to(DEV)], seq_len=n_tok)[0] for k, m in ours.items()}
            assert torch.equal(b["py"], b["nat"]), call
            assert rel_l2(b["nat"].cpu(), a) <= 2e-2, (call, rel_l2(b["nat"].cpu(), a))
            assert type(ours["nat"]).accumulated_err == type(ref).accumulated_err and type(ours["nat"]).cnt == type(ref).cnt
    assert 0 < sum(kinds) < 12 and ours["nat"]._mc_engine._nat is not None


def test_nccl_gather_capi_single_rank_eager_and_captured():
    """`mc_nccl_unique_id` / `mc_nccl_init` / `mc_allgather_kv` / `mc_nccl_destroy` on one GPU (a communicator of one rank: the gather is
    the identity): run-time lookup of libnccl, communicator creation, the fused K|V form and the two-buffer form, eagerly and captured
    into a CUDA graph and replayed. (Two ranks: tests/test_shard_gpu.py, modes collective_capi*.)"""
    import ctypes
    from magcache_b200 import _lib
    lib = _lib.lib
    uid = ctypes.create_string_buffer(128)
    _lib.check(lib.mc_nccl_unique_id(uid))
    h = lib.mc_nccl_init(0, 1, uid)
    assert h, lib.mc_last_error()
    try:
        g = torch.Generator(device=DEV).manual_seed(0)
        k, v = (torch.randn(1024, 512, device=DEV, generator=g).bfloat16() for _ in range(2))
        kf, vf = torch.zeros_like(k), torch.zeros_like(v)
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.mc_allgather_kv(h, k.data_ptr(), None, kf.data_ptr(), None, k.numel(), stream))
        torch.cuda.synchronize()
        assert torch.equal(kf, k)
        kf.zero_()
        _lib.check(lib.mc_allgather_kv(h, k.data_ptr(), v.data_ptr(), kf.data_ptr(), vf.data_ptr(), k.numel(), stream))
        torch.cuda.synchronize()
        assert torch.equal(kf, k) and torch.equal(vf, v)
        assert lib.mc_allgather_kv(h, k.data_ptr(), v.data_ptr(), kf.data_ptr(), None, k.numel(), stream) == _lib.MC_ERR_INVALID
        kf.zero_(), vf.zero_()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            _lib.check(lib.mc_allgather_kv(h, k.data_ptr(), v.data_ptr(), kf.data_ptr(), vf.data_ptr(), k.numel(), torch.cuda.current_stream().cuda_stream))
        k.mul_(2.0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(kf, k) and torch.equal(vf, v)
        del graph
    finally:
        torch.cuda.synchronize()
        assert lib.mc_nccl_destroy(h) == _lib.MC_OK
