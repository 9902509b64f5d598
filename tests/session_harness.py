"""Sessions: several complete generations on ONE patched model in one process, each compared bit for bit with the same generation on a
fresh copy of the model. Shared by tests/test_engine_sessions_cpu.py (emulated kernels) and tests/test_engine_sessions_gpu.py.

Between generations an engine keeps shape-sized workspaces, RoPE tables, text lengths, timestep ranges and captured graphs, residual
caches and the controller's state. A fresh engine is held to the oracle and to fp64 by the other tests; equality with it carries that
guarantee over to every later generation of a long-lived engine.

A cached input is delivered to the next generation in one of three ways (`deliver`):
  inplace   `copy_` into the previous tensor: same address, same object, new content;
  recycled  the previous tensor is dropped and a new one of the same size allocated: the allocator hands out the freed block again,
            unless something (the engine) still holds the old tensor — then no address can repeat, which is what the engine's
            cache keys rely on. When neither happens the case was not exercised and the test skips, saying so;
  new       a separate tensor, the previous one still alive."""
import copy
import gc
import weakref

import pytest
import torch

from magcache_b200 import controller

MODES = ("inplace", "recycled", "new")


@pytest.fixture()
def record_hits(monkeypatch):
    """Every controller decision, appended to the deciding module's `_session_hits` (one bool per call, True = cache hit)."""
    orig = controller.AttrController.decide
    orig_tea = controller.OpenSoraTeaController.decide

    def decide(self, o):
        hit = orig(self, o)
        o.__dict__.setdefault("_session_hits", []).append(hit)
        return hit

    def decide_tea(self, o, forced, rel):
        calc = orig_tea(self, o, forced, rel)
        o.__dict__.setdefault("_session_hits", []).append(not calc)
        return calc

    monkeypatch.setattr(controller.AttrController, "decide", decide)
    monkeypatch.setattr(controller.OpenSoraTeaController, "decide", decide_tea)


def deliver(inputs, key, value, mode):
    """Put `value` into `inputs[key]` (the only reference the test holds to the previous tensor) the way `mode` says."""
    old = inputs[key]
    assert old.shape == value.shape and old.dtype == value.dtype, "deliver() changes content, not shape"
    if mode == "inplace":
        old.copy_(value)
        return
    if mode == "new":
        inputs[key] = value.clone()
        return
    assert mode == "recycled", mode
    ptr, alive = old.data_ptr(), weakref.ref(old)
    del old, inputs[key]
    gc.collect()
    held = alive() is not None
    t, others = torch.empty_like(value), []
    while not held and t.data_ptr() != ptr and len(others) < 64:  # other free blocks of that size may come first
        others.append(t)
        t = torch.empty_like(value)
    del others
    if not held and t.data_ptr() != ptr:
        pytest.skip(f"recycled address not exercised: the allocator did not hand out the freed block of {key!r} again")
    if held:
        assert t.data_ptr() != ptr
    t.copy_(value)
    inputs[key] = t


def _clone(v):
    if torch.is_tensor(v):
        return v.clone()
    if isinstance(v, (list, tuple)):
        return type(v)(_clone(x) for x in v)
    if isinstance(v, dict):
        return {k: _clone(x) for k, x in v.items()}
    return v


def _snap(v):
    if torch.is_tensor(v):
        return v.detach().clone()
    if isinstance(v, (list, tuple)):
        return [_snap(x) for x in v]
    return copy.deepcopy(v)


def _same(a, b, where):
    if torch.is_tensor(a) or torch.is_tensor(b):
        assert torch.is_tensor(a) and torch.is_tensor(b), where
        assert a.shape == b.shape and a.dtype == b.dtype, (where, a.shape, b.shape)
        assert torch.equal(a, b), (where, float((a.double() - b.double()).abs().max()))
    elif isinstance(a, (list, tuple)):
        assert isinstance(b, (list, tuple)) and len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, f"{where}[{i}]")
    elif isinstance(a, dict):
        assert isinstance(b, dict) and a.keys() == b.keys(), where
        for k in a:
            _same(a[k], b[k], f"{where}.{k}")
    else:
        assert a == b, (where, a, b)


def generation(model, calls, residual, state):
    """Run `calls` (a list of `fn(model) -> output`) on `model`; after each, snapshot the output, the cached residual
    (`residual(model)`), the controller state (the attributes in `state`) and whether the call was a cache hit."""
    recs = []
    with torch.no_grad():
        for fn in calls:
            n = len(model.__dict__.get("_session_hits", []))
            out = fn(model)
            hits = model.__dict__.get("_session_hits", [])[n:]
            recs.append({"out": _snap(out), "residual": _snap(residual(model)), "hit": list(hits),
                         "state": {a: _snap(getattr(model, a, None)) for a in state}})
    return recs


class Session:
    """One long-lived patched model (`self.model`) next to a factory of fresh ones. `run(make_calls, inputs)` runs a generation on
    the session model with `inputs` as delivered and the same generation on a fresh model with copies of them (so the fresh
    engine holds none of the session's tensors), and asserts both are identical step by step."""

    def __init__(self, fresh, residual, state):
        self.fresh, self.residual, self.state = fresh, residual, state
        self.model = fresh()
        self.n = 0

    def run(self, make_calls, inputs, before=None):
        """`make_calls(inputs) -> calls`; `before(model)`, if given, runs on both models first (a re-installation, a reset)."""
        self.n += 1
        if before is not None:
            before(self.model)
        got = generation(self.model, make_calls(inputs), self.residual, self.state)
        ref = self.fresh()
        if before is not None:
            before(ref)
        want = generation(ref, make_calls(_clone(inputs)), self.residual, self.state)
        del ref
        gc.collect()
        assert len(got) == len(want)
        for i, (g, w) in enumerate(zip(got, want)):
            for k in ("hit", "state", "out", "residual"):
                _same(g[k], w[k], f"generation {self.n} step {i} {k}")
        return got
