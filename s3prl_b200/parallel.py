"""Utterance sharding across ranks (one process per GPU

Utterances are independent units, so the upstream forward needs no data-path collective: rank r runs the path on
its contiguous slice of the batch. Two pieces of cross-rank state keep the result identical to the un-sharded
batch: the padded length ``Lmax`` (it fixes the padding, the layer-0 GroupNorm statistics and the frame-mask rule)
and, at the end, ONE all-gather of the Featurizer output ``[B/G, T, D]`` (NCCL over NVLink on the GPU box; the
same code runs over gloo on CPU for the tests).
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous, balanced slice [lo, hi) of ``n_items`` for ``rank`` (first ``n_items % world`` ranks get one more)."""
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_batch(items: Sequence, rank: int, world: int) -> List:
    lo, hi = shard_bounds(len(items), rank, world)
    return list(items[lo:hi])


def global_max_len(local_lens: Sequence[int], device=None) -> int:
    """max over all ranks of the utterance lengths (1 scalar all-reduce); local max when not distributed."""
    m = max(local_lens) if len(local_lens) else 0
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        t = torch.tensor([m], dtype=torch.int64, device=device or "cpu")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        m = int(t.item())
    return m


def gather_features(local: torch.Tensor, n_items: int) -> torch.Tensor:
    """All-gather the per-rank feature blocks ``[n_local, T, D]`` into ``[n_items, T, D]`` (rank-major = original
    order, because shards are contiguous). Equal shards use a single ``all_gather_into_tensor``; uneven shards pad
    to the largest shard first (still one collective)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local
    world = dist.get_world_size()
    sizes = [shard_bounds(n_items, r, world) for r in range(world)]
    counts = [hi - lo for lo, hi in sizes]
    biggest = max(counts)
    if local.shape[0] != biggest:
        pad = torch.zeros((biggest - local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        local = torch.cat([local, pad], dim=0)
    out = torch.empty((world * biggest,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local.contiguous())
    if all(c == biggest for c in counts):
        return out
    parts = [out[r * biggest : r * biggest + counts[r]] for r in range(world)]
    return torch.cat(parts, dim=0)


class FeatureGatherer:
    """Weighted layer sum of this rank's utterances, gathered on every rank (the collective of the sharded step).

    mode "push" (default on a GPU box whenever CUDA IPC peer mapping works): ``s3b_peer_push`` — one kernel reads the
    NL+1 local hidden states once and stores the weighted sum directly into every rank's gathered buffer over NVLink
    peer memory, then releases a sequence flag; the stream waits for step s-1's flags at the start of step s, so ranks
    run with one step of slack instead of meeting in a collective every step. mode "nccl": the weighted-sum kernel
    followed by ONE ``all_gather_into_tensor`` (also the path under gloo on CPU-only hosts, without the kernel).

    ``weighted_sum_gather(hidden_states, norm_weights)`` returns the gathered ``[world * B_local, T, D]`` tensor of the
    current step. In push mode it is complete once the NEXT call (or ``finish()``) has been enqueued on the same
    stream and it stays valid for ``slots - 2`` further calls.
    """

    def __init__(self, local_shape: Tuple[int, int, int], device: torch.device, mode: str = "auto", slots: int = 3):
        import ctypes as C

        from . import lib as _lib

        self.local_shape = tuple(int(x) for x in local_shape)
        self.device = device
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.rank = dist.get_rank() if dist.is_initialized() else 0
        self.step = 0
        self.handle = None
        self.mode = "nccl"
        self._out = None
        if mode in ("auto", "push") and device.type == "cuda" and self.world > 1:
            lib = _lib.load()
            block = 1
            for x in self.local_shape:
                block *= x
            handle = C.c_void_p()
            mine = (C.c_ubyte * 64)()
            ok = True
            with torch.cuda.device(device):
                if lib.s3b_peer_create(self.rank, self.world, block, slots, C.byref(handle), mine) != 0:
                    ok, self._why = False, lib.s3b_last_error().decode()
                # exchange the 64-byte IPC handles (and whether everybody got this far) as host objects, which NCCL and
                # gloo both gather (gloo also where several ranks share one device)
                allh = [None] * self.world
                dist.all_gather_object(allh, (ok, bytes(mine) if ok else b""))
                if all(o for o, _ in allh):
                    blob = b"".join(h for _, h in allh)
                    buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
                    if lib.s3b_peer_connect(handle, buf) != 0:
                        ok, self._why = False, lib.s3b_last_error().decode()
                else:
                    ok = False
                status = [None] * self.world
                dist.all_gather_object(status, ok)
            if all(status):
                self.handle, self.lib, self.slots, self.block, self.mode = handle, lib, slots, block, "push"
            else:
                if handle:
                    lib.s3b_peer_destroy(handle)
                if mode == "push":
                    raise _lib.S3BError(f"peer-memory gather unavailable: {getattr(self, '_why', 'a peer failed')}")
        if self.mode == "nccl" and self.world > 1:
            B, T, D = self.local_shape
            self._out = torch.empty((self.world * B, T, D), dtype=torch.float32, device=device)

    def _slot_tensor(self, step: int) -> torch.Tensor:
        import ctypes as C

        ptr = self.lib.s3b_peer_slot(self.handle, C.c_uint32(step))
        B, T, D = self.local_shape

        class _Raw:  # __cuda_array_interface__ view of library-owned device memory
            __cuda_array_interface__ = {"shape": (self.world * B, T, D), "typestr": "<f4", "data": (int(ptr), False),
                                        "version": 2}

        return torch.as_tensor(_Raw(), device=self.device)

    def weighted_sum_gather(self, hidden_states, norm_weights: torch.Tensor) -> torch.Tensor:
        import ctypes as C

        from .upstream.featurizer import _stacked_view, weighted_sum

        if self.world == 1:
            return weighted_sum(hidden_states, norm_weights)
        if self.mode == "nccl":
            local = weighted_sum(hidden_states, norm_weights)
            dist.all_gather_into_tensor(self._out, local.contiguous())
            return self._out
        stacked = _stacked_view(hidden_states)
        assert tuple(stacked.shape[1:]) == self.local_shape, (stacked.shape, self.local_shape)
        w = norm_weights.detach().to(self.device, torch.float32).contiguous()
        st = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        s = self.step
        with torch.cuda.device(self.device):
            if s > 0:
                _check(self.lib, self.lib.s3b_peer_wait(self.handle, C.c_uint32(s - 1), st))
            _check(self.lib, self.lib.s3b_peer_push(self.handle, C.c_void_p(stacked.data_ptr()), stacked.shape[0],
                                                  stacked.stride(0), C.c_void_p(w.data_ptr()), C.c_uint32(s), st))
        self._keep = (stacked, w)  # alive until the kernel has been enqueued behind the next call
        self.step += 1
        return self._slot_tensor(s)

    def finish(self) -> None:
        """Enqueue the wait for the last pushed step: afterwards (stream order) its gathered tensor is complete."""
        import ctypes as C

        if self.mode == "push" and self.step > 0:
            st = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            with torch.cuda.device(self.device):
                _check(self.lib, self.lib.s3b_peer_wait(self.handle, C.c_uint32(self.step - 1), st))

    def close(self) -> None:
        if self.handle is not None:
            torch.cuda.synchronize(self.device)
            if dist.is_initialized():
                dist.barrier()  # nobody unmaps memory a peer may still be writing
            self.lib.s3b_peer_destroy(self.handle)
            self.handle = None


def _check(lib, status: int) -> None:
    if status != 0:
        from .lib import S3BError

        raise S3BError(lib.s3b_last_error().decode())
