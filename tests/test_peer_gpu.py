"""GPU tests of the peer-memory weighted-sum gather (csrc/peer.cu through the C ABI, and parallel.FeatureGatherer in
push mode), the path every sharded step ends in:
- the push kernel at world 1, in process: against the fp64 sum within NL u sum_l |w_l h_l| (the bound of
  test_port_shapes_gpu.py::test_weighted_sum: an fp32 FMA chain in layer order) and bit for bit against
  s3b_weighted_sum, from one float4 to several passes of the capped grid, with layers one block apart or padded further
  apart;
- the slot and flag protocol: step s lands in slot s % slots at this rank's position and nowhere else, the flag of
  (slot, rank) ends at s + 1, the block counter back at 0. Flags and counter are read from the library's buffer BEFORE
  s3b_peer_wait is called: a publication bug fails an assertion here, it never spins the wait kernel into its timeout;
- one process per rank (gloo on 127.0.0.1 for the host side, rank r on device r % device_count: with fewer devices
  than ranks, ranks share a device through CUDA IPC), through the C ABI and through FeatureGatherer's own call order;
- refusal of out-of-range layer counts, strides and misaligned hidden states.
Every arithmetic case prints measured / bound."""
import ctypes as C
import os
import socket
import time
from datetime import timedelta
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0**-24  # fp32 unit roundoff
PUSH_GRID = 132 * 4 * 256 * 4  # peer.cu: floats one pass of launch_weighted_sum_push's capped grid covers
BLOCKS = [4, 1020, PUSH_GRID, PUSH_GRID + 4, 8 * 499 * 768, 4 * 999 * 1280]
BLOCK_IDS = ["one_float4", "1020", "one_pass", "one_pass+4", "8x499x768", "4x999x1280"]


def _lib():
    from s3prl_b200 import lib

    return lib


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _layout(slots, world, block):
    """Byte offsets of the flags ([slots][world] u32) and of the block counter in an s3b_peer buffer, as struct s3b_peer
    in model.cu lays it out: [slots][world][block] floats, the flags from the next 256-byte boundary, the counter from
    the 256-byte boundary after them."""
    flags = -(-(slots * world * block * 4) // 256) * 256
    return flags, flags + -(-(slots * world * 4) // 256) * 256


def _view(ptr, shape, typestr, device):
    class _Raw:  # __cuda_array_interface__ view of library-owned device memory (as FeatureGatherer._slot_tensor)
        __cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 2}

    return torch.as_tensor(_Raw(), device=device)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


class _Peer:
    """An s3b_peer with views of its whole buffer: data [slots][world][block] fp32, flags [slots][world], counter."""

    def __init__(self, rank, world, block, slots, device="cuda"):
        self.L = _lib().load()
        self.world, self.block, self.slots = world, block, slots
        self.h = C.c_void_p()
        self.ipc = (C.c_ubyte * 64)()
        _lib().check(self.L.s3b_peer_create(rank, world, block, slots, C.byref(self.h), self.ipc))
        base = self.L.s3b_peer_slot(self.h, 0)
        flags, counter = _layout(slots, world, block)
        self.data = _view(base, (slots, world, block), "<f4", device)
        self.flags = _view(base + flags, (slots, world), "<i4", device)
        self.counter = _view(base + counter, (1,), "<i4", device)

    def push(self, hs_ptr, num, stride, w, step):
        return self.L.s3b_peer_push(self.h, hs_ptr, num, stride, C.c_void_p(w.data_ptr()), C.c_uint32(step), _stream())

    def wait(self, step):
        _lib().check(self.L.s3b_peer_wait(self.h, C.c_uint32(step), _stream()))

    def destroy(self):
        self.L.s3b_peer_destroy(self.h)


def _inputs(NL, block, stride, seed, device="cuda"):
    """hs [NL][stride] (layers of different scale, NaN between block and stride: read there and it shows) and signed
    weights (cancellation across layers)."""
    g = torch.Generator(device=device).manual_seed(seed)
    hs = torch.randn(NL, stride, device=device, generator=g)
    hs *= torch.linspace(0.5, 4.0, NL, device=device).view(NL, 1)
    hs[:, block:] = float("nan")
    w = torch.randn(NL, device=device, generator=g)
    return hs, w


def _ws(hs, w):
    """s3b_weighted_sum on the first block of every layer of hs (compacted to [NL][block] first)."""
    hs = hs.contiguous()
    out = torch.full(hs.shape[1:], float("nan"), device=hs.device)
    _lib().check(_lib().load().s3b_weighted_sum(C.c_void_p(hs.data_ptr()), hs.shape[0], hs[0].numel(),
                                                C.c_void_p(w.data_ptr()), C.c_void_p(out.data_ptr()), _stream()))
    return out


def _fp64_ratio(out, hs, w):
    """max over elements of |out - sum_l w_l h_l| / (NL u sum_l |w_l h_l|), in fp64."""
    ref = torch.zeros(hs.shape[1], dtype=torch.float64, device=hs.device)
    mag = torch.zeros_like(ref)
    for l in range(hs.shape[0]):
        t = w[l].double() * hs[l].double()
        ref += t
        mag += t.abs()
    assert torch.isfinite(out).all()
    return ((out.double() - ref).abs() / (hs.shape[0] * U * mag).clamp_min(1e-300)).max().item()


# ------------------------------------------------------------------------------------------------
# the push kernel at world 1
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pad", [0, 132], ids=["stride=block", "padded"])
@pytest.mark.parametrize("block", BLOCKS, ids=BLOCK_IDS)
@pytest.mark.parametrize("NL", [1, 13, 25, 49, 64])
def test_push_arithmetic(s3b_lib, NL, block, pad):
    """One push: the fp64 bound, bit for bit s3b_weighted_sum on the compacted layers, flag 1 and counter 0 before the
    wait, the other slot untouched."""
    stride = block + pad
    hs, w = _inputs(NL, block, stride, NL * 1009 + block + pad)
    p = _Peer(0, 1, block, 2)
    try:
        p.data.fill_(float("nan"))
        torch.cuda.synchronize()
        _lib().check(p.push(C.c_void_p(hs.data_ptr()), NL, stride, w, 0))
        torch.cuda.synchronize()
        assert p.flags.cpu().flatten().tolist() == [1, 0] and p.counter.item() == 0
        p.wait(0)
        torch.cuda.synchronize()
        out = p.data[0, 0].clone()
        assert torch.isnan(p.data[1]).all(), "slot 1 was written by step 0"
    finally:
        p.destroy()
    compact = hs[:, :block].contiguous()
    assert _same_bits(out, _ws(compact, w)), "push differs from s3b_weighted_sum"
    r = _fp64_ratio(out, compact, w)
    print(f"push NL={NL} block={block} stride={stride}: measured/bound {r:.3f}")
    assert r <= 1.0, r


@pytest.mark.parametrize("slots", [2, 3, 8])
def test_push_slots_and_flags(s3b_lib, slots):
    """2 slots + 1 steps with new inputs and weights each (stride alternating between the block and a padded one):
    after each push only slot s % slots changed and holds step s's weighted sum, the flags read s + 1 for the slot just
    written and their old values elsewhere, the counter is 0, and hs is unchanged."""
    NL, block = 13, PUSH_GRID + 4  # two passes of the capped grid: 528 CTAs count in
    p = _Peer(0, 1, block, slots)
    try:
        p.data.fill_(float("nan"))
        torch.cuda.synchronize()
        flags = [0] * slots
        for s in range(2 * slots + 1):
            stride = block + (36 if s % 2 else 0)
            hs, w = _inputs(NL, block, stride, 7919 * slots + s)
            hs_before, before = hs.clone(), p.data.clone()
            _lib().check(p.push(C.c_void_p(hs.data_ptr()), NL, stride, w, s))
            torch.cuda.synchronize()
            k = s % slots
            flags[k] = s + 1
            assert p.flags[:, 0].tolist() == flags and p.counter.item() == 0, (s, p.flags[:, 0].tolist())
            p.wait(s)
            torch.cuda.synchronize()
            for j in range(slots):
                if j != k:
                    assert _same_bits(p.data[j], before[j]), f"step {s} wrote slot {j}"
            assert _same_bits(p.data[k, 0], _ws(hs[:, :block], w)), f"step {s}"
            assert _same_bits(hs, hs_before), f"step {s} changed hs"
    finally:
        p.destroy()


def test_push_refusals(s3b_lib):
    """num outside 1..64, layer_stride below the block or not whole float4, hs off 16-byte alignment: refused with the
    argument's name, and nothing launched (slots, flags and counter untouched). A push before s3b_peer_connect at
    world 2 is refused."""
    L = _lib().load()
    NL, block = 13, 1024
    hs = torch.zeros(65, block + 8, device="cuda")
    w = torch.zeros(65, device="cuda")
    at = C.c_void_p(hs.data_ptr())
    p = _Peer(0, 1, block, 2)
    try:
        p.data.fill_(float("nan"))
        torch.cuda.synchronize()
        # first a call that a library without these checks would still run harmlessly (no layers: zeros into slot 0),
        # so that such a library fails here before any of the out-of-bounds launches below
        cases = [(0, block, at, "num"), (-1, block, at, "num"), (65, block, at, "num"), (-(2**31), block, at, "num"),
                 (NL, block - 4, at, "layer_stride"), (NL, -block, at, "layer_stride"), (NL, 0, at, "layer_stride"),
                 (NL, block + 2, at, "layer_stride"), (NL, block, C.c_void_p(hs.data_ptr() + 4), "hs"),
                 (NL, block, C.c_void_p(hs.data_ptr() + 8), "hs")]
        for num, stride, ptr, what in cases:
            rc = p.push(ptr, num, stride, w, 0)
            msg = L.s3b_last_error().decode()
            assert rc != 0 and msg.startswith(what + " = "), (num, stride, msg)
        torch.cuda.synchronize()
        assert torch.isnan(p.data).all() and not p.flags.any() and p.counter.item() == 0
        # the edges run
        _lib().check(p.push(at, 64, block, w, 0))
        _lib().check(p.push(at, 1, block + 4, w, 1))
        torch.cuda.synchronize()
        assert p.flags.flatten().tolist() == [1, 2] and p.counter.item() == 0
        p.wait(1)
        torch.cuda.synchronize()
        assert not p.data.any()
    finally:
        p.destroy()
    q = _Peer(0, 2, block, 2)
    try:
        assert q.push(at, NL, block, w, 0) != 0 and "s3b_peer_connect" in L.s3b_last_error().decode()
        torch.cuda.synchronize()
        assert not q.flags.any()
    finally:
        q.destroy()


# ------------------------------------------------------------------------------------------------
# one process per rank
# ------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _spawn(fn, world, tmp_path, timeout=300):
    """Run fn(rank, world, port, tmpdir) in `world` spawned processes; fail on a worker's exception or after `timeout`
    seconds, and leave no worker alive either way. Skips with the reason a worker recorded in tmpdir/skip."""
    import torch.multiprocessing as mp

    ctx = mp.start_processes(fn, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=False,
                             start_method="spawn")
    deadline = time.monotonic() + timeout
    try:
        while not ctx.join(timeout=5):
            assert time.monotonic() < deadline, f"{world} ranks did not finish in {timeout} s"
    finally:
        for proc in ctx.processes:
            if proc.is_alive():
                proc.kill()
            proc.join(30)
        assert not any(proc.is_alive() for proc in ctx.processes)
    if (tmp_path / "skip").exists():
        pytest.skip((tmp_path / "skip").read_text())


def _init_rank(rank, world, port, tmpdir):
    """A context on device rank % device_count, then gloo. Returns the device, or None when some rank could not create
    a context (a GPU in exclusive-process compute mode, shared by two ranks): rank 0 records why, for the test to skip."""
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    why = ""
    try:
        torch.cuda.set_device(dev)
        torch.zeros(1, device=dev)
        torch.cuda.synchronize(dev)
    except RuntimeError as e:
        why = f"rank {rank} cannot create a CUDA context on {dev} next to the other ranks: {e}"
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timedelta(seconds=120))
    whys = [None] * world
    dist.all_gather_object(whys, why)
    whys = [w for w in whys if w]
    if whys:
        if rank == 0:
            (Path(tmpdir) / "skip").write_text(whys[0])
        return None
    return dev


def _rank_inputs(NL, block, rank, step, dev):
    """Rank `rank`'s hidden states and weights of step `step`, regenerated identically on every rank; odd ranks pad
    their layers."""
    stride = block + 4 * 33 * (rank % 2)
    hs, w = _inputs(NL, block, stride, 100003 * step + 101 * rank + 17, dev)
    return hs, w, stride


def _direct_worker(rank, world, port, tmpdir):
    """The C ABI across ranks: create, exchange the IPC handles over gloo, connect; per step push, synchronize, host
    barrier, then every flag of the slot and the counter read directly, only then s3b_peer_wait; the slot [world][block]
    is every rank's s3b_weighted_sum bit for bit, the other slots are untouched."""
    import torch.distributed as dist

    try:
        dev = _init_rank(rank, world, port, tmpdir)
        if dev is None:
            return
        NL, block = 13, PUSH_GRID + 4
        for slots in (2, 8):
            p = _Peer(rank, world, block, slots, dev)
            hs, w, stride = _rank_inputs(NL, block, rank, 0, dev)
            assert p.push(C.c_void_p(hs.data_ptr()), NL, stride, w, 0) != 0
            assert "s3b_peer_connect" in p.L.s3b_last_error().decode()
            p.data.fill_(float("nan"))
            torch.cuda.synchronize(dev)
            handles = [None] * world
            dist.all_gather_object(handles, bytes(p.ipc))
            blob = b"".join(handles)
            _lib().check(p.L.s3b_peer_connect(p.h, (C.c_ubyte * len(blob)).from_buffer_copy(blob)))
            dist.barrier()  # every buffer is NaN and mapped everywhere before anyone pushes
            flags = torch.zeros(slots, world, dtype=torch.int32)
            for s in range(2 * slots + 1):
                k = s % slots
                hs, w, stride = _rank_inputs(NL, block, rank, s, dev)
                before = p.data.clone()
                _lib().check(p.push(C.c_void_p(hs.data_ptr()), NL, stride, w, s))
                torch.cuda.synchronize(dev)
                dist.barrier()  # step s has landed in every buffer
                flags[k] = s + 1
                got = p.flags.cpu()
                assert torch.equal(got, flags) and p.counter.item() == 0, (rank, s, got.tolist())
                p.wait(s)
                torch.cuda.synchronize(dev)
                for q in range(world):
                    hq, wq, _ = _rank_inputs(NL, block, q, s, dev)
                    assert _same_bits(p.data[k, q], _ws(hq[:, :block], wq)), f"rank {rank} step {s}: block of {q}"
                for j in range(slots):
                    if j != k:
                        assert _same_bits(p.data[j], before[j]), f"rank {rank} step {s} wrote slot {j}"
                dist.barrier()  # nobody pushes step s + 1 while a rank still reads this step's buffers
            p.destroy()
        if rank == 0:
            print(f"peer ABI: world {world} on {torch.cuda.device_count()} device(s), slots 2 and 8, 5 + 17 steps: "
                  f"every block bit for bit s3b_weighted_sum")
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _gather_inputs(NL, shape, rank, step, in_place, dev):
    """Hidden states as slices of one [NL, B, T, D] buffer (read in place) or as separate tensors (stacked first), and
    softmax weights."""
    g = torch.Generator(device=dev).manual_seed(100003 * step + 101 * rank + 29)
    buf = torch.randn(NL, *shape, device=dev, generator=g)
    w = torch.randn(NL, device=dev, generator=g).softmax(-1)
    return ([buf[l] for l in range(NL)] if in_place else [buf[l].clone() for l in range(NL)]), w


def _gatherer_worker(rank, world, port, tmpdir):
    """FeatureGatherer in push mode with its own call order (call s waits for step s - 1, then pushes s; finish() waits
    for the last step). The tensor of step s is copied right after call s + 1, inside the slots - 2 calls it stays valid
    for, and equals torch.cat of every rank's weighted_sum bit for bit. Ranks on distinct devices are skewed by sleeping
    kernels so that waits overlap pushes; ranks sharing a device synchronize and meet at a host barrier between calls,
    where the flags of the step about to be waited for are checked first: contexts of different processes only
    time-slice a GPU, and nothing here may depend on preempting a spinning wait."""
    import torch.distributed as dist

    from s3prl_b200.parallel import FeatureGatherer
    from s3prl_b200.upstream.featurizer import weighted_sum

    try:
        dev = _init_rank(rank, world, port, tmpdir)
        if dev is None:
            return
        shared = world > torch.cuda.device_count()
        for NL, shape in ((13, (2, 37, 768)), (49, (1, 29, 1280))):
            for in_place in (True, False):
                gth = FeatureGatherer(shape, dev, mode="push")
                assert gth.mode == "push" and gth.world == world
                base = gth.lib.s3b_peer_slot(gth.handle, 0)
                flags = _view(base + _layout(gth.slots, world, gth.block)[0], (gth.slots, world), "<i4", dev)
                steps = 2 * gth.slots + 1
                saved, last = [], None
                for s in range(steps):
                    hs, w = _gather_inputs(NL, shape, rank, s, in_place, dev)
                    if shared:
                        torch.cuda.synchronize(dev)
                        dist.barrier()
                        if s > 0:
                            got = flags[(s - 1) % gth.slots].tolist()
                            assert got == [s] * world, (rank, s, got)
                    elif (rank + s) % 3 == 0:
                        torch.cuda._sleep(5_000_000)
                    out = gth.weighted_sum_gather(hs, w)
                    if last is not None:
                        saved.append(last.clone())
                    last = out
                gth.finish()
                saved.append(last.clone())
                torch.cuda.synchronize(dev)
                for s in range(steps):
                    want = torch.cat([weighted_sum(*_gather_inputs(NL, shape, q, s, True, dev)) for q in range(world)])
                    assert _same_bits(saved[s], want), f"rank {rank} NL={NL} in_place={in_place} step {s}"
                gth.close()
        if rank == 0:
            print(f"FeatureGatherer push: world {world} on {torch.cuda.device_count()} device(s) "
                  f"({'synchronized between calls' if shared else 'skewed ranks'}), NL 13 and 49, in place and stacked: "
                  f"every step bit for bit torch.cat of the ranks' weighted_sum")
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_peer_abi_across_ranks(s3b_lib, tmp_path, world):
    _spawn(_direct_worker, world, tmp_path)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_feature_gatherer_push_across_ranks(s3b_lib, tmp_path, world):
    _spawn(_gatherer_worker, world, tmp_path)
