"""Token-axis sharding of the Wan forward over the GPUs of one node (SURVEY.md §8e).

Everything in the forward is token-local except self-attention, which needs every key/value. Each rank owns a contiguous
range of tokens (contiguous in (f, h, w) raster order — the "temporal/token shard"), keeps its slice of the residual stream
and of the residual cache (as the reference's only sequence-parallel MagCache does, eval/magcache/experiments/opensora.py:310,347),
and per layer contributes its K|V rows to the other ranks — the counterpart of videosys/core/comm.py:272-292
(`dist.all_gather` + `torch.cat`). The controller is a pure function of `cnt` and the table, so every rank takes the same
hit/miss decision without communicating.

Two exchanges implement the same interface (`KVExchange`):

* `P2PExchange` (CUDA, the product path): no collective library on the data path. Every rank owns a cudaMalloc'ed window mapped by
  its peers through CUDA IPC (`mc_p2p_*`, csrc/p2p.cu). The K|V rows a rank has just projected are pushed into every peer's
  gathered buffer by the copy engines on a side stream, nearest consumer first, each push followed by a 4-byte flag; the attention
  kernel starts on its own keys at once and waits, tile by tile, for the flag of the segment it needs next (`mc_attn_fwd_ex`), so
  the transfer hides behind the attention itself. The head kernel stores its rows straight into every peer's output tensor.
* `CollectiveExchange` (torch.distributed all-gather / all-reduce: gloo on CPU in the test-suite, NCCL with MC_SHARD_P2P=0):
  the plain formulation, kept as the reference point of the partitioning logic.

Token counts that are not a multiple of the world size follow the reference's pad rule (videosys/core/comm.py:373-381: pad the
sequence to the next multiple, split equally, drop the pad after the gather): every rank owns ceil(N / P) row SLOTS, the last
rank's trailing slots are pad — never computed, never attended to (the key count stays N).
"""
import ctypes
import os
from dataclasses import dataclass

import torch
import torch.distributed as dist


@dataclass
class TokenShard:
    rank: int
    world: int
    n_tokens: int
    group: object = None

    def __post_init__(self):
        if self.start >= self.n_tokens:
            raise ValueError(f"token count {self.n_tokens} leaves rank {self.rank} of {self.world} without tokens")

    @property
    def n_slots(self):
        """Row slots per rank = ceil(N / P) (videosys/core/comm.py:373-378: pad = (P - N % P) % P)."""
        return -(-self.n_tokens // self.world)

    @property
    def pad(self):
        return self.n_slots * self.world - self.n_tokens

    @property
    def n_padded(self):
        return self.n_slots * self.world

    @property
    def start(self):
        return self.rank * self.n_slots

    @property
    def stop(self):
        return min(self.start + self.n_slots, self.n_tokens)

    @property
    def n_local(self):
        """Valid (computed) rows of this rank: n_slots, less the pad on the last rank(s)."""
        return self.stop - self.start

    def rows(self, t):
        """This rank's rows of a token-major tensor [N, ...]."""
        return t[self.start:self.stop]


def gather_rows(local, full, group=None, async_op=False):
    """All-gather token rows: full[r*n:(r+1)*n] = rank r's `local` ([n, C], contiguous, same n on every rank)."""
    assert local.is_contiguous() and full.is_contiguous() and full.shape[0] % local.shape[0] == 0
    return dist.all_gather_into_tensor(full, local, group=group, async_op=async_op)


def sum_partial_outputs(out, group=None):
    """Every rank wrote only its tokens' positions of the (zero-initialised) output: the sum over ranks is the full tensor,
    exactly (x + 0 == x), and leaves it replicated for the caller's scheduler step."""
    dist.all_reduce(out, op=dist.ReduceOp.SUM, group=group)
    return out


def allreduce_stats(stats, group=None):
    """Calibration statistics of a sharded run: (sum ratio, sum ratio^2, sum (1-cos), rows) add across ranks."""
    dist.all_reduce(stats, op=dist.ReduceOp.SUM, group=group)
    return stats


# ---------------------------------------------------------------------------------------------------------------------
# K|V exchange + output assembly
# ---------------------------------------------------------------------------------------------------------------------
class CollectiveExchange:
    """all_gather_into_tensor of the K|V rows (issued asynchronously, waited for right before the attention) and an all-reduce
    of the zero-initialised head output."""

    p2p = False

    def __init__(self, shard: TokenShard, width, out_shape, device, extra_rows=0):
        assert extra_rows == 0 or shard.pad == 0, "locally written tail rows follow the token rows directly: no pad slots in between"
        self.sh, self.device, self.out_shape, self.extra = shard, device, tuple(out_shape), extra_rows
        bf = dict(dtype=torch.bfloat16, device=device)
        self.kv_loc = torch.zeros(shard.n_slots, width, **bf)          # pad slots stay zero
        self.kv_all = torch.empty(shard.n_padded + extra_rows, width, **bf)
        self._work = None
        # MC_SHARD_NCCL=capi (CUDA): the gather is `mc_allgather_kv` — ncclAllGather behind the C ABI on a communicator of this
        # exchange's own (csrc/nccl_gather.cu) — instead of torch.distributed's; same buffers, same ordering
        self._nccl = None
        if torch.device(device).type == "cuda" and os.environ.get("MC_SHARD_NCCL", "") == "capi":
            from . import _lib
            uid = ctypes.create_string_buffer(128)
            if shard.rank == 0:
                _lib.check(_lib.lib.mc_nccl_unique_id(uid))
            box = [bytes(uid.raw)]
            dist.broadcast_object_list(box, src=0 if shard.group is None else dist.get_global_rank(shard.group, 0), group=shard.group)
            h = _lib.lib.mc_nccl_init(shard.rank, shard.world, ctypes.create_string_buffer(box[0], 128))
            if not h:
                raise _lib.MagCacheError(_lib.MC_ERR_STATE, _lib.lib.mc_last_error().decode("utf-8", "replace"))
            self._lib, self._nccl = _lib, h
            self.comm = torch.cuda.Stream(device=device)
            self._done = None

    def own_rows(self, i):
        if self._nccl is not None and self._done is not None:
            torch.cuda.current_stream().wait_event(self._done)  # the gather that last read kv_loc has drained
        return self.kv_loc[:self.sh.n_local]

    def tail_rows(self, i):
        """The `extra_rows` key rows behind the token rows that every rank writes for itself (MMDiT: the replicated text tokens)."""
        return self.kv_all[self.sh.n_padded:]

    def begin(self, i):
        if self._nccl is not None:  # on a side stream, so that the q projection overlaps it like the async c10d gather does
            main = torch.cuda.current_stream()
            ev = torch.cuda.Event()
            ev.record(main)
            self.comm.wait_event(ev)
            self._lib.check(self._lib.lib.mc_allgather_kv(self._nccl, self.kv_loc.data_ptr(), None, self.kv_all.data_ptr(), None,
                                                          self.kv_loc.numel(), self.comm.cuda_stream))
            self._done = torch.cuda.Event()
            self._done.record(self.comm)
            return
        self._work = gather_rows(self.kv_loc, self.kv_all[:self.sh.n_padded], self.sh.group, async_op=True)

    def keys_values(self, i):
        """(gathered [N (+ extra), width] view, extra keyword arguments for ops.attention). Blocks the stream until the rows are there."""
        if self._nccl is not None:
            torch.cuda.current_stream().wait_event(self._done)
        else:
            self._work.wait()
        return self.kv_all[:self.sh.n_tokens + self.extra], {}

    def head_output(self, slot):
        return torch.zeros(self.out_shape, dtype=torch.float32, device=self.device), None

    def finish_head(self, out, slot):
        return sum_partial_outputs(out, self.sh.group)

    def join(self):
        if self._nccl is not None and self._done is not None:
            torch.cuda.current_stream().wait_event(self._done)
            self._done = None  # a later forward (possibly captured into a graph of its own) must not wait on this event again

    def close(self):
        if self._nccl is not None:
            torch.cuda.synchronize()
            self._lib.lib.mc_nccl_destroy(self._nccl)
            self._nccl = None


class _RawCuda:
    """Zero-copy view of device memory the library allocated (an IPC window): just enough of __cuda_array_interface__."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


class P2PExchange:
    """The copy-engine / flag exchange described in the module docstring. One per engine (its windows are sized for one token
    count). All ranks must construct it collectively (the IPC handles travel through `all_gather_object`)."""

    p2p = True
    FLAG_BYTES = 4096

    def __init__(self, shard: TokenShard, width, out_shape, device, extra_rows=0):
        from . import _lib
        self._lib = _lib
        lib, check = _lib.lib, _lib.check
        assert extra_rows == 0 or shard.pad == 0, "locally written tail rows follow the token rows directly: no pad slots in between"
        self.sh, self.device, self.out_shape, self.width, self.extra = shard, device, tuple(out_shape), width, extra_rows
        P = shard.world
        out_numel = 1
        for v in out_shape:
            out_numel *= v
        self.out_bytes = (out_numel * 4 + 255) // 256 * 256
        self.kv_bytes = ((shard.n_padded + extra_rows) * width * 2 + 255) // 256 * 256
        self.seg_bytes = shard.n_slots * width * 2
        total = self.FLAG_BYTES + 2 * self.out_bytes + 2 * self.kv_bytes
        ptr = ctypes.c_void_p()
        handle = ctypes.create_string_buffer(64)
        check(lib.mc_p2p_alloc(total, ctypes.byref(ptr), handle))
        self.base = ptr.value
        handles = [None] * P
        dist.all_gather_object(handles, bytes(handle.raw), group=shard.group)
        self.peer_base = []
        for r in range(P):
            if r == shard.rank:
                self.peer_base.append(self.base)
                continue
            pp = ctypes.c_void_p()
            check(lib.mc_p2p_open(ctypes.create_string_buffer(handles[r], 64), ctypes.byref(pp)))
            self.peer_base.append(pp.value)
        self.window = torch.as_tensor(_RawCuda(self.base, total), device=device)
        flags = self.window[:self.FLAG_BYTES].view(torch.int32)
        self.kv_flags = [flags[0:P], flags[64:64 + P]]          # [exchange parity][source rank]
        self.out_flags = [flags[128:128 + P], flags[192:192 + P]]  # [CFG slot][source rank]
        o0 = self.FLAG_BYTES
        self.outs = [self.window[o0 + s * self.out_bytes:o0 + s * self.out_bytes + out_numel * 4].view(torch.float32).view(self.out_shape)
                     for s in range(2)]
        k0 = o0 + 2 * self.out_bytes
        self.kv = [self.window[k0 + i * self.kv_bytes:k0 + i * self.kv_bytes + (shard.n_padded + extra_rows) * width * 2].view(torch.bfloat16)
                   .view(shard.n_padded + extra_rows, width) for i in range(2)]
        if extra_rows:
            # the attention kernel waits on the flag of every segment a KV tile touches; the tail rows are local, their
            # "segments" (indices P ...) are permanently published
            n_tail = (extra_rows + shard.n_slots - 1) // shard.n_slots + 1
            assert P + n_tail <= 64, "flag table: 64 entries per exchange parity"
            flags[P:P + n_tail] = 0x7FFFFFFF
            flags[64 + P:64 + P + n_tail] = 0x7FFFFFFF
        self._kv_off = [k0 + i * self.kv_bytes + shard.start * width * 2 for i in range(2)]
        self.epochs = torch.zeros(4, dtype=torch.int32, device=device)  # [0] K|V exchange rounds, [1] head-output rounds
        self.comm = torch.cuda.Stream(device=device)
        self._done = [None, None]
        # push order: nearest consumer first — rank r-1 reaches this rank's keys first, then r-2, ... (the kernel's rotated key order)
        self.order = [(shard.rank - s) % P for s in range(1, P)]
        dist.barrier(group=shard.group)  # every window is mapped before anyone pushes

    # -- K|V ------------------------------------------------------------------------------------------------------
    def own_rows(self, i):
        """This rank's segment of gathered buffer i: the K|V projection writes here directly. Waits (stream-side) until the pushes that
        last read it have drained."""
        if self._done[i] is not None:
            torch.cuda.current_stream().wait_event(self._done[i])
        sh = self.sh
        return self.kv[i][sh.start:sh.start + sh.n_local]

    def tail_rows(self, i):
        """The `extra_rows` key rows behind the token rows of gathered buffer i, written by every rank for itself (MMDiT: the
        replicated text tokens); call after `own_rows(i)` (which orders the stream behind the pushes that last read the buffer — they
        never touch the tail, but the attention that last read it is ordered the same way)."""
        return self.kv[i][self.sh.n_padded:]

    def begin(self, i):
        lib, check = self._lib.lib, self._lib.check
        sh, P = self.sh, self.sh.world
        main = torch.cuda.current_stream()
        ep = self.epochs[0:1]
        check(lib.mc_p2p_bump(ep.data_ptr(), self.kv_flags[i][sh.rank:sh.rank + 1].data_ptr(), main.cuda_stream))
        ev = torch.cuda.Event()
        ev.record(main)
        self.comm.wait_event(ev)
        n = P - 1
        dst = (ctypes.c_void_p * n)(*[self.peer_base[r] + self._kv_off[i] for r in self.order])
        flg = (ctypes.c_void_p * n)(*[self.peer_base[r] + (0 if i == 0 else 256) + 4 * sh.rank for r in self.order])
        check(lib.mc_p2p_push(self.base + self._kv_off[i], dst, flg, n, self.seg_bytes, ep.data_ptr(), self.comm.cuda_stream))
        done = torch.cuda.Event()
        done.record(self.comm)
        self._done[i] = done

    def keys_values(self, i):
        sh = self.sh
        return self.kv[i][:sh.n_tokens + self.extra], dict(first_key_row=sh.start, seg_flags=self.kv_flags[i], seg_epoch=self.epochs[0:1], seg_rows=sh.n_slots)

    # -- head output ----------------------------------------------------------------------------------------------
    def head_output(self, slot):
        o0 = self.FLAG_BYTES + slot * self.out_bytes
        return self.outs[slot], [self.peer_base[r] + o0 for r in range(self.sh.world) if r != self.sh.rank]

    def finish_head(self, out, slot):
        lib, check = self._lib.lib, self._lib.check
        sh, P = self.sh, self.sh.world
        main = torch.cuda.current_stream()
        ep = self.epochs[1:2]
        check(lib.mc_p2p_bump(ep.data_ptr(), self.out_flags[slot][sh.rank:sh.rank + 1].data_ptr(), main.cuda_stream))
        n = P - 1
        peers = [r for r in range(P) if r != sh.rank]
        nul = (ctypes.c_void_p * n)(*[None] * n)
        flg = (ctypes.c_void_p * n)(*[self.peer_base[r] + 512 + (0 if slot == 0 else 256) + 4 * sh.rank for r in peers])
        check(lib.mc_p2p_push(None, nul, flg, n, 0, ep.data_ptr(), main.cuda_stream))
        check(lib.mc_p2p_wait(self.out_flags[slot].data_ptr(), P, ep.data_ptr(), main.cuda_stream))
        return out.clone()  # the window slot is rewritten two forwards from now; callers keep outputs across calls

    def join(self):
        """Make the calling stream wait for every push issued so far (end of a forward: required before a graph capture ends, and
        before the engine's buffers may be reused by a non-exchanging forward)."""
        main = torch.cuda.current_stream()
        for ev in self._done:
            if ev is not None:
                main.wait_event(ev)
        self._done = [None, None]  # later forwards (possibly captured into a graph of their own) must not wait on these again

    def close(self):
        lib = self._lib.lib
        torch.cuda.synchronize()
        for r, pb in enumerate(self.peer_base):
            if r != self.sh.rank and pb:
                lib.mc_p2p_close(pb)
        self.peer_base = []
        self.window = self.kv = self.outs = None
        if self.base:
            lib.mc_p2p_free(self.base)
            self.base = 0


def make_exchange(shard, width, out_shape, device, extra_rows=0):
    use_p2p = torch.device(device).type == "cuda" and os.environ.get("MC_SHARD_P2P", "1") != "0"
    return (P2PExchange if use_p2p else CollectiveExchange)(shard, width, out_shape, device, extra_rows=extra_rows)


# ---------------------------------------------------------------------------------------------------------------------
# Open-Sora sequence parallelism (VideoSys DSP): frames for the spatial blocks, positions for the temporal blocks
# ---------------------------------------------------------------------------------------------------------------------
def frame_position_shards(world, T, S, group=None):
    """The partition of `split_sequence` / `all_to_all_with_pad` (videosys/core/comm.py:297-381, `set_pad`): T frames (and S positions
    per frame) padded up to a multiple of P and split in equal blocks, so rank r owns frames [r ceil(T/P), min((r+1) ceil(T/P), T))
    and positions likewise. Returns ([TokenShard over T] * P, [TokenShard over S] * P). Pad frames / positions are never stored or
    computed. A world that leaves a rank without a real frame (or position) raises ValueError: the reference would run that rank on
    pad rows only."""
    for what, n in (("T", T), ("S", S)):
        if n < 1 or -(-n // world) * (world - 1) >= n:
            raise ValueError(f"Open-Sora sequence parallelism: {what} = {n} {'latent frames' if what == 'T' else 'positions per frame'} on "
                             f"P = {world} ranks leaves rank {world - 1} without a real {'frame' if what == 'T' else 'position'}")
    return [TokenShard(r, world, T, group) for r in range(world)], [TokenShard(q, world, S, group) for q in range(world)]


def _ceil256(n):
    return (n + 255) // 256 * 256


class _SwitchBase:
    """Rows are `B (T S) D`. The frame-sharded layout of rank r holds, per sample b, frames [t0_r, t1_r) of every position:
    row b T_r S + (t - t0_r) S + s. The position-sharded layout of rank q holds every frame of positions [s0_q, s1_q): row
    b T S_q + t S_q + (s - s0_q) — itself `B (T S_q)`, so the temporal kernels run on it with S_q in place of S. One block of the
    switch is, per (sample, peer), T_r strided runs of S_q rows (pitch S D) on the frame side and one contiguous run of T_r S_q rows
    on the position side."""

    def __init__(self, rank, world, B, T, S, D, Hx, Wx, device, group):
        self.rank, self.world, self.group, self.device = rank, world, group, device
        self.B, self.T, self.S, self.D, self.plane = B, T, S, D, Hx * Wx
        self.frames, self.positions = frame_position_shards(world, T, S, group)
        self.fr, self.ps = self.frames[rank], self.positions[rank]
        self.out_shapes = {False: (B, 8, T, Hx, Wx), True: (B // 2, 4, T, Hx, Wx)}

    def bytes_per_switch(self):
        """bf16 bytes this rank sends to its peers in one switch (forward or backward; the two are equal)."""
        return sum(self.B * self.fr.n_local * q.n_local * self.D * 2 for q in self.positions if q.rank != self.rank)


class CollectiveSwitch(_SwitchBase):
    """`all_to_all_single` over packed per-peer chunks for the switch and `all_gather` of padded frame windows for the output (gloo on
    CPU in the test-suite; NCCL on the GPU with MC_SHARD_P2P=0)."""

    p2p = False

    def __init__(self, rank, world, B, T, S, D, Hx, Wx, device, group=None):
        super().__init__(rank, world, B, T, S, D, Hx, Wx, device, group)
        bf = dict(dtype=torch.bfloat16, device=device)
        self.pos = torch.empty(B * T * self.ps.n_local, D, **bf)
        self.frm = torch.empty(B * self.fr.n_local * S, D, **bf)
        self.out = {k: torch.empty(v, dtype=torch.float32, device=device) for k, v in self.out_shapes.items()}

    def _a2a(self, send, recv_sizes):
        """One all_to_all_single of the bit patterns, as int32 pairs of bf16 (gloo has no 16-bit types; D is even)."""
        send = [c.reshape(-1).view(torch.int32) for c in send]
        recv = torch.empty(sum(recv_sizes) // 2, dtype=torch.int32, device=self.device)
        dist.all_to_all_single(recv, torch.cat(send), output_split_sizes=[n // 2 for n in recv_sizes],
                               input_split_sizes=[c.numel() for c in send], group=self.group)
        return recv.view(torch.bfloat16).split(recv_sizes)

    def to_positions(self, h):
        """Frame-sharded [B T_r S, D] -> position-sharded [B T S_r, D] (dynamic_switch before the temporal attention)."""
        B, S, D, fr, ps = self.B, self.S, self.D, self.fr, self.ps
        hv = h.view(B, fr.n_local, S, D)
        got = self._a2a([hv[:, :, q.start:q.stop] for q in self.positions], [B * p.n_local * ps.n_local * D for p in self.frames])
        pv = self.pos.view(B, self.T, ps.n_local, D)
        for p, c in zip(self.frames, got):
            pv[:, p.start:p.stop].copy_(c.view(B, p.n_local, ps.n_local, D))
        return self.pos

    def to_frames(self, a):
        """Position-sharded [B T S_r, D] -> frame-sharded [B T_r S, D] (dynamic_switch after the temporal attention)."""
        B, S, D, fr, ps = self.B, self.S, self.D, self.fr, self.ps
        av = a.view(B, self.T, ps.n_local, D)
        got = self._a2a([av[:, p.start:p.stop] for p in self.frames], [B * fr.n_local * q.n_local * D for q in self.positions])
        fv = self.frm.view(B, fr.n_local, S, D)
        for q, c in zip(self.positions, got):
            fv[:, :, q.start:q.stop].copy_(c.view(B, fr.n_local, q.n_local, D))
        return self.frm

    def output_buffer(self, step):
        return self.out[step]

    def gather_output(self, buf, out=None):
        """Every rank wrote its frame window of `buf`; return the whole tensor on every rank (into `out` when given)."""
        lead = buf.shape[0] * buf.shape[1]
        n = self.fr.n_slots * self.plane
        v = buf.view(lead, self.T * self.plane)
        mine = torch.zeros(lead, n, dtype=torch.float32, device=self.device)
        mine[:, :self.fr.n_local * self.plane] = v[:, self.fr.start * self.plane:self.fr.stop * self.plane]
        parts = [torch.empty_like(mine) for _ in range(self.world)]
        dist.all_gather(parts, mine, group=self.group)
        res = torch.empty_like(buf) if out is None else out
        rv = res.view(lead, self.T * self.plane)
        for p, c in zip(self.frames, parts):
            rv[:, p.start * self.plane:p.stop * self.plane] = c[:, :p.n_local * self.plane]
        return res

    def close(self):
        pass


class P2PSwitch(_SwitchBase):
    """The switch and the output assembly on the copy engines (`mc_p2p_push2d`). Every rank owns one IPC window: flags, two
    position-sharded receive buffers, two frame-sharded receive buffers and two full-size output slots. Exchange n of a direction
    uses buffer n % 2 (DESIGN §7 argues why two are enough). All pushes run on the calling stream in the order of the forward, so
    the stream that issued them is also the one that may overwrite their source; a one-block kernel (`mc_p2p_wait`) holds the
    stream until every peer's flag has reached the exchange's epoch. No SM moves data. Constructed collectively."""

    p2p = True
    FLAG_BYTES = 4096

    def __init__(self, rank, world, B, T, S, D, Hx, Wx, device, group=None):
        super().__init__(rank, world, B, T, S, D, Hx, Wx, device, group)
        from . import _lib
        self._lib = _lib
        lib, check = _lib.lib, _lib.check
        assert world <= 64, "flag table: 64 entries per buffer"
        s_slots, t_slots = self.positions[0].n_slots, self.frames[0].n_slots
        self.pos_bytes = _ceil256(B * T * s_slots * D * 2)
        self.frm_bytes = _ceil256(B * t_slots * S * D * 2)
        self.out_bytes = _ceil256(B * 8 * T * self.plane * 4)
        self.off_pos = [self.FLAG_BYTES + i * self.pos_bytes for i in range(2)]
        self.off_frm = [self.FLAG_BYTES + 2 * self.pos_bytes + i * self.frm_bytes for i in range(2)]
        self.off_out = [self.FLAG_BYTES + 2 * self.pos_bytes + 2 * self.frm_bytes + i * self.out_bytes for i in range(2)]
        total = self.off_out[1] + self.out_bytes
        ptr, handle = ctypes.c_void_p(), ctypes.create_string_buffer(64)
        check(lib.mc_p2p_alloc(total, ctypes.byref(ptr), handle))
        self.base = ptr.value
        handles = [None] * world
        dist.all_gather_object(handles, bytes(handle.raw), group=group)
        self.peer_base = []
        for r in range(world):
            if r == rank:
                self.peer_base.append(self.base)
                continue
            pp = ctypes.c_void_p()
            check(lib.mc_p2p_open(ctypes.create_string_buffer(handles[r], 64), ctypes.byref(pp)))
            self.peer_base.append(pp.value)
        self.window = torch.as_tensor(_RawCuda(self.base, total), device=device)
        self.flags = self.window[:self.FLAG_BYTES].view(torch.int32)  # [direction 0..2][parity][source rank] at 128 d + 64 parity + r
        w = self.window

        def view(off, rows, cols, dtype, nbytes):
            return w[off:off + nbytes].view(dtype).view(rows, cols)

        self.pos = [view(o, B * T * self.ps.n_local, D, torch.bfloat16, B * T * self.ps.n_local * D * 2) for o in self.off_pos]
        self.frm = [view(o, B * self.fr.n_local * S, D, torch.bfloat16, B * self.fr.n_local * S * D * 2) for o in self.off_frm]
        self.epochs = torch.zeros(4, dtype=torch.int32, device=device)  # [0] forward switch, [1] backward switch, [2] output
        self.count = [0, 0, 0]
        # push order: the nearest peers first (r + 1, r - 1, r + 2, ...), this rank's own block last
        near = sorted((q for q in range(world) if q != rank), key=lambda q: (min((q - rank) % world, (rank - q) % world), (q - rank) % world))
        self.order = near + [rank]
        dist.barrier(group=group)  # every window is mapped before anyone pushes

    def _flag(self, r, d, parity, src):
        return self.peer_base[r] + 4 * (128 * d + 64 * parity + src)

    def _exchange(self, d, copies):
        """Round of direction d: bump its epoch (this rank's own flag with it), issue `copies` [(dst, dpitch, src, spitch, width,
        height)], one flag per peer, then wait on the stream for every rank's flag. Returns the parity used."""
        lib, check = self._lib.lib, self._lib.check
        i = self.count[d] % 2
        self.count[d] += 1
        stream = torch.cuda.current_stream().cuda_stream
        ep = self.epochs[d:d + 1]
        own = self.flags[128 * d + 64 * i:128 * d + 64 * i + self.world]
        check(lib.mc_p2p_bump(ep.data_ptr(), own[self.rank:self.rank + 1].data_ptr(), stream))
        arr = (self._lib.Copy2D * len(copies))(*[self._lib.Copy2D(*c) for c in copies])
        peers = [q for q in self.order if q != self.rank]
        flg = (ctypes.c_void_p * len(peers))(*[self._flag(q, d, i, self.rank) for q in peers])
        check(lib.mc_p2p_push2d(arr, len(copies), flg, len(peers), ep.data_ptr(), stream))
        check(lib.mc_p2p_wait(own.data_ptr(), self.world, ep.data_ptr(), stream))
        return i

    def _blocks(self, parity, forward, src):
        B, T, S, D, fr = self.B, self.T, self.S, self.D, self.fr
        i, copies = parity, []
        for q in self.order:
            pq = self.positions[q]
            for b in range(B):
                frame_side = src if forward else self.peer_base[q] + self.off_frm[i]
                frame_off = (b * fr.n_local * S + pq.start) * D * 2 if forward else (b * self.frames[q].n_local * S + self.ps.start) * D * 2
                if forward:  # this rank's frames, positions of q -> q's position buffer
                    copies.append((self.peer_base[q] + self.off_pos[i] + (b * T * pq.n_local + fr.start * pq.n_local) * D * 2,
                                   pq.n_local * D * 2, frame_side + frame_off, S * D * 2, pq.n_local * D * 2, fr.n_local))
                else:        # every frame of this rank's positions: q's frames -> q's frame buffer
                    fq = self.frames[q]
                    copies.append((frame_side + frame_off, S * D * 2,
                                   src + (b * T * self.ps.n_local + fq.start * self.ps.n_local) * D * 2, self.ps.n_local * D * 2,
                                   self.ps.n_local * D * 2, fq.n_local))
        return copies

    def to_positions(self, h):
        assert h.is_contiguous() and h.shape == (self.B * self.fr.n_local * self.S, self.D)
        i = self.count[0] % 2
        self._exchange(0, self._blocks(i, True, h.data_ptr()))
        return self.pos[i]

    def to_frames(self, a):
        assert a.is_contiguous() and a.shape == (self.B * self.T * self.ps.n_local, self.D)
        i = self.count[1] % 2
        self._exchange(1, self._blocks(i, False, a.data_ptr()))
        return self.frm[i]

    def output_buffer(self, step):
        i = self.count[2] % 2
        shape = self.out_shapes[step]
        n = 1
        for v in shape:
            n *= v
        return self.window[self.off_out[i]:self.off_out[i] + 4 * n].view(torch.float32).view(shape)

    def gather_output(self, buf, out=None):
        """This rank's frame window of `buf` (the current output slot) into the same slot of every peer: height (samples x channels),
        width T_r Hx Wx fp32, pitch T Hx Wx. Then the whole tensor is copied out of the window (it is rewritten two outputs later)."""
        i = self.count[2] % 2
        assert buf.data_ptr() == self.base + self.off_out[i]
        lead, fr, pl = buf.shape[0] * buf.shape[1], self.fr, self.plane
        off = fr.start * pl * 4
        copies = [(self.peer_base[q] + self.off_out[i] + off, self.T * pl * 4, self.base + self.off_out[i] + off, self.T * pl * 4,
                   fr.n_local * pl * 4, lead) for q in self.order if q != self.rank]
        self._exchange(2, copies)
        if out is None:
            return buf.clone()
        return out.copy_(buf)

    def close(self):
        lib = self._lib.lib
        torch.cuda.synchronize()
        for r, pb in enumerate(self.peer_base):
            if r != self.rank and pb:
                lib.mc_p2p_close(pb)
        self.peer_base = []
        self.window = self.pos = self.frm = None
        if self.base:
            lib.mc_p2p_free(self.base)
            self.base = 0


def make_switch(rank, world, B, T, S, D, Hx, Wx, device, group=None):
    use_p2p = torch.device(device).type == "cuda" and os.environ.get("MC_SHARD_P2P", "1") != "0"
    return (P2PSwitch if use_p2p else CollectiveSwitch)(rank, world, B, T, S, D, Hx, Wx, device, group)
