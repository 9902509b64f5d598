"""Unmerged PEFT LoRA adapters on the FLUX and Qwen-Image engines: finding them on the module, the reference's scale / unscale statements, and
packing each adapted Linear's update as a tail of the GEMM that computes its base output (`ops.gemm(tail=(U, T))`).

PEFT and diffusers are not part of this project. The layer layout and the statements below are restated from upstream (parity
unpinned, like oracle/sampler_ref.py's schedulers): PEFT's `lora.Linear.forward` (non-DoRA) is

    result = base_layer(x)
    for a in active_adapters:            # skipped when disable_adapters or merged
        if a not in lora_A: continue
        result = result + lora_B[a](lora_A[a](lora_dropout[a](x))) * scaling[a]

and the FLUX forward wraps itself in diffusers' `scale_lora_layers(self, lora_scale)` / `unscale_lora_layers(self, lora_scale)`
(MagCache4FLUX/magcache_flux.py:274-287, :437-439; calibration :62-75, :224-226; Kontext magcache_flux_kontext.py:279-289,
:439-441); the Qwen-Image forward the same way around its own (MagCache4QwenImage/magcache_generate.py:185-192, :249-250;
calibration :106-113, :168-169).

On the engine every distinct GEMM input x (a block's LN+modulate rows, its attention output, ...) gets one down-projection
U = bf16(x A^T), A the stack of every adapter that reads x, each padded to a multiple of 8 rows. A consumer GEMM then adds
U[:, its columns] T^T inside its own main loop, T = bf16(scaling * lora_B) (block-diagonal for FLUX's concatenated q|k
weights; Qwen-Image's q and k, read in place, are two tailed weights).
Rounding: PEFT computes bf16(bf16(bf16(B bf16(A x)) * s) + bf16(base(x))); the engine sums base and update in fp32 and rounds
once in the epilogue, with the scale folded into T. Only U and T are rounded to bf16 on the way.
"""
import math
import weakref

import torch
from torch import nn


def is_lora_layer(m):
    """A PEFT LoRA layer, by its attribute surface (no `peft` import): `base_layer`, `lora_A` / `lora_B`, `scaling`."""
    d = getattr(m, "_modules", None)
    return d is not None and "base_layer" in d and "lora_A" in d and "lora_B" in d and hasattr(m, "scaling")


def base_linear(m):
    """The nn.Linear whose weight / bias a (possibly LoRA-wrapped) module computes its base output with."""
    return m.base_layer if is_lora_layer(m) else m


def _set_scale(m, a, scale):
    """PEFT `LoraLayer.set_scale`: scaling = scale * alpha / r (alpha / sqrt(r) with rslora)."""
    if a not in m.scaling:
        return
    r = m.r[a]
    m.scaling[a] = scale * m.lora_alpha[a] / (math.sqrt(r) if getattr(m, "use_rslora", {}).get(a, False) else r)


def scale_lora_layers(model, weight):
    """diffusers `scale_lora_layers`: a no-op at weight 1; otherwise every LoRA layer's active adapters with a lora_A get
    scaling *= weight (PEFT `scale_layer`)."""
    if weight == 1.0:
        return
    for m in model.modules():
        if is_lora_layer(m):
            for a in m.active_adapters:
                if a in m.lora_A.keys():
                    m.scaling[a] *= weight


def unscale_lora_layers(model, weight=None):
    """diffusers `unscale_lora_layers`: a no-op for None or 1; scaling /= weight for weight != 0 (PEFT `unscale_layer`); at
    weight 0 every active adapter's scaling is reset to alpha / r (`set_scale(a, 1.0)`), which drops any `set_adapters` weight."""
    if weight is None or weight == 1.0:
        return
    for m in model.modules():
        if is_lora_layer(m):
            for a in m.active_adapters:
                if weight != 0:
                    if a in m.lora_A.keys():
                        m.scaling[a] /= weight
                else:
                    _set_scale(m, a, 1.0)


def _live(m, name):
    """[(lora_A weight, lora_B weight, scaling)] that PEFT's forward adds on `m` now; raises on what the engine does not run."""
    if m.disable_adapters or m.merged:
        return []
    out = []
    for a in m.active_adapters:
        if a not in m.lora_A.keys():
            continue
        if getattr(m, "use_dora", {}).get(a, False):
            raise NotImplementedError(f"magcache_b200: DoRA adapter {a!r} on {name} is not supported")
        if m.lora_B[a].bias is not None:
            raise NotImplementedError(f"magcache_b200: adapter {a!r} on {name} has a lora_B bias (lora_bias), not supported")
        drop = m.lora_dropout[a] if a in m.lora_dropout.keys() else None
        if isinstance(drop, nn.Dropout) and drop.training and drop.p > 0:
            raise NotImplementedError(f"magcache_b200: adapter {a!r} on {name} has an active dropout (training mode, p={drop.p})")
        out.append((m.lora_A[a].weight, m.lora_B[a].weight, float(m.scaling[a])))
    return out


def _layer_key(m):
    """Everything about a LoRA layer that can change what it adds, or its base weight (a merge), between two calls. Read through
    the modules' own dicts: this runs for every adapted layer at every call."""
    mods = m._modules
    la, lb, ld = mods["lora_A"]._modules, mods["lora_B"]._modules, mods["lora_dropout"]._modules
    sc, dora = m.scaling, getattr(m, "use_dora", {})
    ads = []
    for a, A in la.items():
        B = lb[a]
        Aw, Bw, d = A._parameters["weight"], B._parameters["weight"], ld.get(a)
        ads.append((a, id(Aw), Aw._version, id(Bw), Bw._version, sc[a], B._parameters.get("bias") is None, dora.get(a, False),
                    d.training if d is not None else False))
    return (id(m), m.disable_adapters, tuple(getattr(m, "merged_adapters", ())), tuple(m.active_adapters), tuple(ads))


# ------------------------------------------------------------------------------------------------ where adapters may sit
_DOUBLE = (("attn", "to_q"), ("attn", "to_k"), ("attn", "to_v"), ("attn.to_out", "0"), ("attn", "add_q_proj"), ("attn", "add_k_proj"),
           ("attn", "add_v_proj"), ("attn", "to_add_out"), ("ff.net.0", "proj"), ("ff.net", "2"), ("ff_context.net.0", "proj"),
           ("ff_context.net", "2"), ("norm1", "linear"), ("norm1_context", "linear"))
_SINGLE = (("attn", "to_q"), ("attn", "to_k"), ("attn", "to_v"), ("", "proj_mlp"), ("", "proj_out"), ("norm", "linear"))
_TOP = (("", "x_embedder"), ("", "context_embedder"), ("", "proj_out"), ("norm_out", "linear"))
_QWEN_BLOCK = _DOUBLE[:8] + (("img_mlp.net.0", "proj"), ("img_mlp.net", "2"), ("txt_mlp.net.0", "proj"), ("txt_mlp.net", "2"),
                             ("img_mod", "1"), ("txt_mod", "1"))
_QWEN_TOP = (("", "img_in"), ("", "txt_in"), ("norm_out", "linear"), ("", "proj_out"))


def _positions(model, blocks, top):
    """[(target key, the parent module's `_modules` dict, child name, module path)] for every Linear an adapter may sit on (the
    covered targets: per block list `blocks` = [(kind, attribute, (parent, child) pairs)], then the top-level `top`), then the
    time_text_embed Linears, which must carry none. (The dict, not the parent: the model's own would hold the model.)"""
    pos = []

    def add(key, root, prefix, parent, child):
        p = root.get_submodule(parent) if parent else root
        path = ".".join(x for x in (prefix, parent, child) if x)
        pos.append((key, p._modules, child, path))

    for kind, attr, pairs in blocks:
        for i, blk in enumerate(getattr(model, attr)):
            for parent, child in pairs:
                add((kind, i, f"{parent}.{child}".lstrip(".")), blk, f"{attr}.{i}", parent, child)
    for parent, child in top:
        add(("top", 0, f"{parent}.{child}".lstrip(".")), model, "", parent, child)
    tte = model.time_text_embed
    for emb in ("timestep_embedder", "guidance_embedder", "text_embedder"):
        if hasattr(tte, emb):
            for child in ("linear_1", "linear_2"):
                add(None, tte, "time_text_embed", emb, child)
    return pos


def flux_positions(model):
    """`_positions` of a FluxTransformer2DModel: the double and single block Linears with their AdaLayerNorm projections,
    x_embedder, context_embedder, norm_out.linear, proj_out."""
    return _positions(model, (("double", "transformer_blocks", _DOUBLE), ("single", "single_transformer_blocks", _SINGLE)), _TOP)


def qwen_positions(model):
    """`_positions` of a QwenImageTransformer2DModel: per block the attention and MLP Linears and `img_mod.1` / `txt_mod.1`; img_in,
    txt_in, norm_out.linear, proj_out."""
    return _positions(model, (("double", "transformer_blocks", _QWEN_BLOCK),), _QWEN_TOP)


# PEFT's `lora.Linear` surface beyond what `is_lora_layer` recognises a layer by; the scan and the packing read all of it
_SURFACE = ("active_adapters", "disable_adapters", "merged", "lora_dropout", "r", "lora_alpha")


def _check_surface(m, name):
    missing = [a for a in _SURFACE if not hasattr(m, a)]
    if missing:
        raise NotImplementedError(f"magcache_b200: {name} has a LoRA layer's base_layer / lora_A / lora_B / scaling but not PEFT's "
                                  f"{', '.join(missing)}; only PEFT `lora.Linear` layers run on the engine")


class LoraScan:
    """Reads a module's adapters at every call, at the positions `family.positions` lists (FLUX or QWEN below). `scan()` walks the
    recorded positions (a dict lookup per position; LoRA layers also get their state read) and returns (spec, merged, wrappers,
    changed): spec maps each covered target to the adapters PEFT would add there now, `merged` identifies the merged adapters
    (their updates live in the base weights), `wrappers` holds the LoRA layers found, `changed` says whether anything differs from
    the previous scan. On a change the whole module is searched once for LoRA layers outside the covered targets, which raise.

    What a scan cannot see: a write to adapter or base weights through `.data` (it bumps no version counter; adapter hot-swapping
    writes that way), and a merge whose LoRA layers were removed before the scan could see them (`fuse_lora()` then
    `unload_lora_weights()` between two forwards). After either, call `invalidate_engine`.

    The module is held by a weak reference: the engine that owns the scan is an attribute of the module, and a strong reference
    back would leave the module and its weights to the cyclic garbage collector once the caller drops them."""

    def __init__(self, model, family=None):
        self._model, self.family = weakref.ref(model), FLUX if family is None else family
        self.positions = self.family.positions(model)
        self._key = None

    @property
    def model(self):
        return self._model()

    def scan(self):
        layers = []
        for key, mods, child, path in self.positions:
            m = mods[child]
            if is_lora_layer(m):
                layers.append((key, m, path))
        try:
            state = tuple(_layer_key(m) for _, m, _ in layers)
        except (AttributeError, KeyError):
            for _, m, path in layers:
                _check_surface(m, path)
            raise
        if state == self._key:
            return self._spec, self._merged, self._wrappers, False
        covered = {id(m) for key, m, _ in layers if key is not None}
        for name, m in self.model.named_modules():
            if is_lora_layer(m) and id(m) not in covered:
                raise NotImplementedError(f"magcache_b200: a LoRA adapter on {name} is not supported on the {self.family.name} engine "
                                          f"(covered: {self.family.covered})")
        spec = {}
        for key, m, path in layers:
            live = _live(m, path)
            if live:
                spec[key] = live
        self._key, self._spec = state, spec
        self._merged = tuple((id(m), tuple(m.merged_adapters)) for _, m, _ in layers if getattr(m, "merged_adapters", ()))
        self._wrappers = tuple(m for _, m, _ in layers)
        return spec, self._merged, self._wrappers, True


FluxLoraScan = LoraScan  # (its family defaults to FLUX)


# ------------------------------------------------------------------------------------------------ packing
def _pad8(r):
    return (r + 7) // 8 * 8


class Group:
    """One down-projection: A [R, K] bf16, the stacked (8-row padded) lora_A of every adapter that reads the same GEMM input.
    The engine sets `u = bf16(src A^T)` once `src` holds the call's input; consumers read the rows of U matching their A rows."""

    def __init__(self, A):
        self.A, self.u, self.src = A, None, None

    def u_rows(self, a):
        """U rows of the GEMM input `a`, a row range of `src` (the token-sharded path launches row blocks of one input)."""
        src = self.src
        assert a.stride() == src.stride() and a.shape[1] == src.shape[1] and a.dtype == src.dtype
        step = src.stride(0) * src.element_size()
        off = a.data_ptr() - src.data_ptr()
        assert off % step == 0 and 0 <= off // step <= src.shape[0] - a.shape[0], "GEMM input is not a row range of the down-projected one"
        r0 = off // step
        return self.u[r0:r0 + a.shape[0]]


class Tailed:
    """A bf16 weight [N, K] with a LoRA tail: T [N, r] bf16 against columns [c0, c0 + r) of its group's U. Indexing takes a row
    block of both, like Fp8Weight."""

    def __init__(self, w, group, c0, t):
        self.w, self.group, self.c0, self.t = w, group, c0, t

    @property
    def shape(self):
        return self.w.shape

    def __getitem__(self, rows):
        return Tailed(self.w[rows], self.group, self.c0, self.t[rows])

    def tail(self, a):
        """(U, T) for the GEMM input `a`."""
        return self.group.u_rows(a)[:, self.c0:self.c0 + self.t.shape[1]], self.t


# GEMM input (group), packed weight (consumer) and row block of the packed weight (q|k: 0 / 1) of each covered target
_D_MAP = {"attn.to_q": ("h", "qk_w", 0), "attn.to_k": ("h", "qk_w", 1), "attn.to_v": ("h", "v_w", 0), "attn.to_out.0": ("att", "o_w", 0),
          "attn.add_q_proj": ("ch", "cqk_w", 0), "attn.add_k_proj": ("ch", "cqk_w", 1), "attn.add_v_proj": ("ch", "cv_w", 0),
          "attn.to_add_out": ("catt", "co_w", 0), "ff.net.0.proj": ("h2", "ff1_w", 0), "ff.net.2": ("ffh", "ff2_w", 0),
          "ff_context.net.0.proj": ("ch2", "cff1_w", 0), "ff_context.net.2": ("cffh", "cff2_w", 0)}
_S_MAP = {"proj_mlp": ("h", "mlp_w", 0), "attn.to_q": ("h", "qk_w", 0), "attn.to_k": ("h", "qk_w", 1), "attn.to_v": ("h", "v_w", 0),
          "proj_out": ("cat", "out_w", 0)}
_T_MAP = {"x_embedder": ("x", "x_w", 0), "context_embedder": ("ctx", "ctx_w", 0), "proj_out": ("head", "out_w", 0)}
# modulation rows: (the weights' row offset attribute, down-projection group) of each adapted modulation Linear
_ADA = {("double", "norm1.linear"): ("ada", "ada"), ("double", "norm1_context.linear"): ("ada_c", "ada"), ("single", "norm.linear"): ("ada", "ada"),
        ("top", "norm_out.linear"): ("ada_out", "ada")}
_QD_MAP = {**{k: v for k, v in _D_MAP.items() if k.startswith("attn.")}, "img_mlp.net.0.proj": ("h2", "ff1_w", 0),
           "img_mlp.net.2": ("ffh", "ff2_w", 0), "txt_mlp.net.0.proj": ("ch2", "cff1_w", 0), "txt_mlp.net.2": ("cffh", "cff2_w", 0)}
_QT_MAP = {"img_in": ("x", "img_w", 0), "txt_in": ("ctx", "txt_w", 0), "proj_out": ("head", "out_w", 0)}
# a Qwen hit computes only the final layer's modulation rows, so norm_out.linear's adapters get a down-projection of their own
_QADA = {("double", "img_mod.1"): ("ada", "ada"), ("double", "txt_mod.1"): ("ada_c", "ada"), ("top", "norm_out.linear"): ("ada_out", "ada_out")}


class Family:
    """Where one model family's adapters may sit (`positions`) and where each lands in its engine's weights: per block kind the
    target map of `_D_MAP`'s form, the modulation targets of `_ADA`'s form, and the top-level weight names."""

    def __init__(self, name, positions, maps, ada, top, covered):
        self.name, self.positions, self.maps, self.ada, self.top, self.covered = name, positions, maps, ada, top, covered


FLUX = Family("FLUX", flux_positions, {"double": _D_MAP, "single": _S_MAP, "top": _T_MAP}, _ADA, ("x_w", "ctx_w", "out_w"),
              "the block Linears, the AdaLayerNorm projections, x_embedder, context_embedder, proj_out")
QWEN = Family("Qwen-Image", qwen_positions, {"double": _QD_MAP, "top": _QT_MAP}, _QADA, ("img_w", "txt_w", "out_w"),
              "the block attention and MLP Linears, img_mod.1, txt_mod.1, img_in, txt_in, norm_out.linear, proj_out")


class LoraPack:
    """An engine's view of the adapters of one call: per block, the packed weights that carry a tail and the groups whose
    down-projections feed them; the prologue / head weights; the modulation table's parts. Built from a spec
    {(kind, block, target): [(lora_A, lora_B, scaling)]}; T (the scaled lora_B rows) and the A stacks are reused from the
    previous pack wherever their inputs (tensor identity, version, scaling) are unchanged, so a new scale repacks only T.

    A packed weight held as a (q, k) tuple (QwenImageWeights reads them in place) gets one `Tailed` per adapted element, each with
    its own T over its own columns of the group's U. The modulation rows are the engine's parts (`w.ada_parts`, or the one stacked
    `w.ada_w`): an adapted Linear's rows become a `Tailed` part."""

    def __init__(self, w, spec, prev=None, family=None):
        family = FLUX if family is None else family
        self.w = w
        dev = w.device
        cache = prev._cache if prev is not None else {}
        self._cache = {}
        by_block = {}
        for (kind, i, tgt), ads in spec.items():
            by_block.setdefault((kind, i), []).append((tgt, ads))
        self.double = [dict(b) for b in w.double]
        self.single = [dict(b) for b in w.single]
        self.top = {k: getattr(w, k) for k in family.top}
        self.groups = {}
        ada_tails = []  # (row0, rows, adapters, target key, group)
        for (kind, i), items in sorted(by_block.items(), key=lambda kv: (kv[0][0], kv[0][1])):
            dst = self.double[i] if kind == "double" else self.single[i] if kind == "single" else self.top
            cmap = family.maps[kind]
            consumers = {}  # consumer -> (group, [(row block index, adapters)])
            for tgt, ads in items:
                if (kind, tgt) in family.ada:
                    a, g = family.ada[(kind, tgt)]
                    r0 = w.ada_out if a == "ada_out" else w.double[i][a] if kind == "double" else w.single[i][a]
                    ada_tails.append((r0, ads[0][1].shape[0], ads, (kind, i, tgt), g))
                    continue
                g, c, blk = cmap[tgt]
                consumers.setdefault(c, (g, []))[1].append((blk, ads, (kind, i, tgt)))
            groups = {}
            for c in sorted(consumers, key=lambda c: (consumers[c][0], c)):
                groups.setdefault(consumers[c][0], []).append(c)
            gmap = {}
            for g, cs in groups.items():
                parts, offs, c0 = [], {}, 0
                for c in cs:
                    offs[c] = c0
                    for blk, ads, _ in sorted(consumers[c][1], key=lambda x: x[0]):
                        for A, _, _ in ads:
                            parts.append(A)
                            c0 += _pad8(A.shape[0])
                grp = Group(self._a_stack(parts, dev, cache, (kind, i, g)))
                gmap[g] = grp
                for c in cs:
                    base = dst[c]
                    if isinstance(base, tuple):  # one Tailed per adapted element, at its own columns
                        els, c0 = list(base), offs[c]
                        for blk, ads, key in sorted(consumers[c][1], key=lambda x: x[0]):
                            t = self._t_rows([(0, ads, key)], base[blk].shape[0], dev, cache, (kind, i, c, blk))
                            els[blk] = Tailed(base[blk], grp, c0, t)
                            c0 += sum(_pad8(A.shape[0]) for A, _, _ in ads)
                        dst[c] = tuple(els)
                        continue
                    t = self._t_rows(consumers[c][1], base.shape[0], dev, cache, (kind, i, c))
                    dst[c] = Tailed(base, grp, offs[c], t)
            if kind != "top":
                dst["lora"] = gmap
            else:
                self.groups.update(gmap)
        self.ada_parts = None
        if ada_tails:
            ada_tails.sort(key=lambda x: x[0])
            offs = []
            for g in sorted({x[4] for x in ada_tails}):
                grp_parts, c0 = [], 0
                for r0, rows, ads, key, gg in ada_tails:
                    if gg == g:
                        offs.append((r0, c0))
                        for A, _, _ in ads:
                            grp_parts.append(A)
                            c0 += _pad8(A.shape[0])
                self.groups[g] = Group(self._a_stack(grp_parts, dev, cache, (g,)))
            offs = dict(offs)
            parts = []
            tails = iter(ada_tails)
            nxt = next(tails, None)
            for p0, pw in (w.ada_parts if w.ada_parts is not None else [(0, w.ada_w)]):
                row, p1 = p0, p0 + pw.shape[0]
                while nxt is not None and nxt[0] < p1:
                    r0, rows, ads, key, g = nxt
                    assert r0 + rows <= p1, "an adapted modulation Linear spans two weight parts"
                    if r0 > row:
                        parts.append((row, pw[row - p0:r0 - p0]))
                    t = self._t_rows([(0, ads, key)], rows, dev, cache, key)
                    parts.append((r0, Tailed(pw[r0 - p0:r0 - p0 + rows], self.groups[g], offs[r0], t)))
                    row = r0 + rows
                    nxt = next(tails, None)
                if row < p1:
                    parts.append((row, pw[row - p0:] if row > p0 else pw))
            self.ada_parts = parts

    def _a_stack(self, parts, dev, cache, key):
        sig = tuple((id(A), A._version, A.shape) for A in parts)
        hit = cache.get(key)
        if hit is not None and hit[0] == sig:
            self._cache[key] = hit
            return hit[1]
        K = parts[0].shape[1]
        A = torch.zeros(sum(_pad8(p.shape[0]) for p in parts), K, dtype=torch.bfloat16, device=dev)
        r = 0
        for p in parts:
            A[r:r + p.shape[0]] = p.detach().to(device=dev, dtype=torch.bfloat16)
            r += _pad8(p.shape[0])
        self._cache[key] = (sig, A)
        return A

    def _t_rows(self, blocks, N, dev, cache, key):
        """T [N, sum of padded ranks]: an adapter of row block b (lora_B [n, r]) fills rows [b n, b n + n) and its own columns (the
        concatenated q|k weight gets the block-diagonal [[s B_q, 0], [0, s B_k]])."""
        blocks = sorted(blocks, key=lambda x: x[0])
        sig = tuple((b, tuple((id(Bw), Bw._version, s) for _, Bw, s in ads)) for b, ads, _ in blocks)
        hit = cache.get(key)
        if hit is not None and hit[0] == sig:
            self._cache[key] = hit
            return hit[1]
        R = sum(_pad8(A.shape[0]) for _, ads, _ in blocks for A, _, _ in ads)
        T = torch.zeros(N, R, dtype=torch.bfloat16, device=dev)
        c = 0
        for b, ads, _ in blocks:
            for A, Bw, s in ads:
                r = A.shape[0]
                n = Bw.shape[0]
                T[b * n:(b + 1) * n, c:c + r] = (Bw.detach().to(device=dev, dtype=torch.float64) * s).to(torch.bfloat16)
                c += _pad8(r)
        self._cache[key] = (sig, T)
        return T
