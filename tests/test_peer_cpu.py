"""CPU tests of the argument checks that s3b_peer_create and the weighted-sum entry points make before any CUDA call:
a bad argument is refused with a message that names it, on any host. The same refusals on real device buffers, and
s3b_peer_push's, are in tests/test_peer_gpu.py and tests/test_port_shapes_gpu.py."""
import ctypes as C

import pytest


def _create(L, rank, world, block, slots):
    h = C.c_void_p()
    ipc = (C.c_ubyte * 64)()
    rc = L.s3b_peer_create(rank, world, block, slots, C.byref(h), ipc)
    if rc == 0:
        L.s3b_peer_destroy(h)
    return rc, L.s3b_last_error().decode()


@pytest.mark.parametrize("rank,world,block,slots,what", [
    (0, 0, 1024, 3, "world"),
    (0, 17, 1024, 3, "world"),  # one flag per rank, read by a 32-thread wait; the push holds 16 peer pointers
    (-1, 2, 1024, 3, "rank"),
    (2, 2, 1024, 3, "rank"),
    (5, 4, 1024, 3, "rank"),
    (0, 1, 0, 3, "block_elems"),
    (0, 1, 6, 3, "block_elems"),  # the push stores float4
    (0, 1, -4, 3, "block_elems"),
    (0, 1, 1024, 1, "slots"),  # a writer may run one step ahead of the slowest reader: two slots at least
    (0, 1, 1024, 9, "slots"),
])
def test_peer_create_refuses_bad_arguments(s3b_lib, rank, world, block, slots, what):
    rc, msg = _create(s3b_lib, rank, world, block, slots)
    assert rc != 0 and what in msg, msg


def test_peer_create_checks_before_the_device(s3b_lib):
    """Null outputs are refused; on a host without a device, arguments that pass are refused for the missing device."""
    h = C.c_void_p()
    assert s3b_lib.s3b_peer_create(0, 1, 1024, 3, C.byref(h), None) != 0
    assert s3b_lib.s3b_peer_create(0, 1, 1024, 3, None, (C.c_ubyte * 64)()) != 0
    assert "null" in s3b_lib.s3b_last_error().decode()
    if s3b_lib.s3b_device_count() > 0:
        return
    rc, msg = _create(s3b_lib, 15, 16, 4, 8)
    assert rc != 0 and "no CUDA device" in msg, msg


HS, W, OUT = 0x7F0000100000, 0x7F0000200000, 0x7F0000300000  # never dereferenced: every call below is refused


def test_weighted_sum_refuses_bad_arguments(s3b_lib):
    """num outside 1..64 (the kernels' shared weight table), negative or non-float4 layer sizes, and hs / out / grad_out
    off 16-byte alignment, on addresses that are never dereferenced. Only on a host without a device: where one is
    visible, test_port_shapes_gpu.py::test_weighted_sum_refusals makes the same calls on real buffers."""
    if s3b_lib.s3b_device_count() > 0:
        pytest.skip("a device is visible: the refusals run on real buffers in test_port_shapes_gpu.py")
    fwd, bwd = s3b_lib.s3b_weighted_sum, s3b_lib.s3b_weighted_sum_backward
    cases = [
        ((HS, 0, 0, W, OUT), "num"),
        ((HS, -1, 8, W, OUT), "num"),
        ((HS, 65, 8, W, OUT), "num"),
        ((HS, -(2**31), 8, W, OUT), "num"),
        ((HS, 13, -4, W, OUT), "n_per_layer"),
        ((HS, 13, -(2**62), W, OUT), "n_per_layer"),
        ((HS, 13, 6, W, OUT), "n_per_layer"),
        ((HS + 4, 13, 8, W, OUT), "hs"),
        ((HS + 8, 13, 8, W, OUT), "hs"),
    ]
    for args, what in cases:
        for fn in (fwd, bwd):
            assert fn(*args, None) != 0, (fn, args)
            msg = s3b_lib.s3b_last_error().decode()
            assert msg.startswith(what + " = "), (args, msg)
    assert fwd(HS, 13, 8, W, OUT + 4, None) != 0
    assert s3b_lib.s3b_last_error().decode().startswith("out = ")
    assert bwd(HS, 13, 8, OUT + 12, W, None) != 0
    assert s3b_lib.s3b_last_error().decode().startswith("grad_out = ")
