"""CPU tests of the data-parallel surface above GG_MAX_BATCH pairs: the merge and step scratch sizes, argument errors that
return instead of aborting, and the peer-memory transport refusing large batches before anything is communicated."""
import ctypes as C

import numpy as np
import pytest

MULTI_CTA = 1   # GG_GRAD_MULTI_CTA


def _merge_bytes(lib, world, cap, ld):
    n = C.c_int64(0)
    return lib.gg_grad_merge_scratch_bytes(world, cap, ld, C.byref(n)), n.value


def _dp_bytes(lib, world, n_pairs, ld):
    n = C.c_int64(0)
    return lib.gg_dp_scratch_bytes(world, n_pairs, ld, C.byref(n)), n.value


def _grad_bytes(lib, n_pairs, ld):
    n = C.c_int64(0)
    assert lib.gg_pair_grad_scratch_bytes(n_pairs, ld, C.byref(n)) == 0
    return n.value


def test_merge_scratch_is_linear_in_entries():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    for ld in (32, 64, 128, 256):
        sizes = {}
        for world in (1, 2, 3, 8):
            for cap in (2, 2048, 16384, 131072):
                rc, n = _merge_bytes(lib, world, cap, ld)
                assert rc == 0 and n > 0
                sizes[world, cap] = n
        for cap in (2048, 16384, 131072):      # (tiny sizes round to the same 256-byte-aligned arrays)
            assert sizes[1, cap] < sizes[2, cap] < sizes[3, cap] < sizes[8, cap]
        for world in (1, 2, 3, 8):
            assert sizes[world, 2] < sizes[world, 2048] < sizes[world, 16384] < sizes[world, 131072]
        # the same entry count costs the same whatever its split, and the cost per entry is bounded (no E^2 term):
        # ids, two radix key/value pairs and the offsets are 24 bytes, the per-tile counts and histograms a little more
        assert sizes[8, 16384] == _merge_bytes(lib, 2, 65536, ld)[1]
        for (world, cap), n in sizes.items():
            assert 24 * world * cap <= n <= 32 * world * cap + 8192
    # scratch does not copy rows: independent of ld
    assert _merge_bytes(lib, 8, 16384, 32)[1] == _merge_bytes(lib, 8, 16384, 256)[1]


def test_dp_scratch_is_the_larger_of_slice_gradient_and_merge():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    for world in (1, 2, 3, 8):
        for B in (1, 1024, 1025, 4096, 65536):
            for ld in (32, 128, 256):
                rc, n = _dp_bytes(lib, world, B, ld)
                assert rc == 0
                slice_ = -(-B // world)
                want = max(_grad_bytes(lib, slice_, ld), _merge_bytes(lib, world, 2 * slice_, ld)[1])
                assert n == want, (world, B, ld)
    # grows with n_pairs at a fixed world; with world the slice gradient shrinks
    seq = [_dp_bytes(lib, 4, B, 128)[1] for B in (1025, 4096, 16384, 65536)]
    assert seq == sorted(seq) and len(set(seq)) == 4
    assert _dp_bytes(lib, 8, 65536, 128)[1] < _dp_bytes(lib, 1, 65536, 128)[1]


def test_scratch_queries_reject_bad_arguments():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    for world, cap, ld in ((0, 16, 128), (-1, 16, 128), (2, 0, 128), (2, -4, 128), (2, 16, 48), (2, 16, 0),
                           (2, 1 << 30, 128), (1 << 16, 1 << 16, 128)):
        assert _merge_bytes(lib, world, cap, ld)[0] != 0, (world, cap, ld)
        assert b"gg_grad_merge_scratch_bytes" in lib.gg_last_error()
    assert lib.gg_grad_merge_scratch_bytes(2, 16, 128, None) != 0
    for world, B, ld in ((0, 2048, 128), (-2, 2048, 128), (2, 0, 128), (2, -1, 128), (2, 1 << 30, 128), (2, 2048, 100),
                         (1 << 30, 2048, 128)):
        assert _dp_bytes(lib, world, B, ld)[0] != 0, (world, B, ld)
        assert b"scratch_bytes" in lib.gg_last_error()
    assert lib.gg_dp_scratch_bytes(2, 2048, 128, None) != 0


def test_merge_ex_argument_errors_return():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    fake = 1 << 20       # never dereferenced: every check below fails before a device pointer is used

    def merge(world=2, cap=16384, ld=128, gathered=fake, scratch=fake, scratch_bytes=None, flags=0):
        if scratch_bytes is None:
            scratch_bytes = _merge_bytes(lib, max(world, 1), max(cap, 1), 128)[1]
        rc = lib.gg_grad_merge_ex(world, cap, ld, gathered, fake, fake, fake, fake, fake, scratch, scratch_bytes, flags, None)
        return rc, lib.gg_last_error().decode()

    for kw, what in ((dict(world=0), "world"), (dict(cap=0), "cap"), (dict(cap=1 << 30), "world * cap"),
                     (dict(flags=4), "flags"), (dict(ld=48), "ld"), (dict(scratch_bytes=1000), "scratch"),
                     (dict(scratch=None), "scratch"), (dict(scratch=fake + 16), "aligned"), (dict(gathered=None), "null"),
                     (dict(gathered=fake + 4), "aligned"), (dict(cap=16383), "even"),
                     (dict(world=2, cap=64, flags=MULTI_CTA, scratch_bytes=0), "scratch")):
        rc, msg = merge(**kw)
        assert rc != 0 and "gg_grad_merge_ex" in msg and what in msg, (kw, msg)
    # the one-CTA merge keeps its own limit and message
    assert lib.gg_grad_merge(2, 16384, 128, fake, fake, fake, fake, fake, fake, None) != 0
    assert b"too many entries" in lib.gg_last_error()


def test_dp_step_ex_argument_errors_return():
    """Without a communicator, and with bad flags, the step entry points return an error before anything else."""
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    fake = 1 << 20
    f = C.c_float
    b1, b2 = C.c_float(0.9), C.c_float(0.999)
    starts = np.zeros(1, np.int64)

    def step(comm=None, n_pairs=4096, flags=0):
        return lib.gg_dp_step_ex(comm, 0, n_pairs, fake, fake, fake, 10, 128, fake, fake, fake, fake, fake, fake, f(0), fake, fake,
                                 4096, fake, fake, fake, fake, fake, f(1e-3), f(0.9), f(0.999), f(1e-8), fake, 1 << 30, flags, None)

    def loop(comm=None, batch_size=4096, start_list=starts.ctypes.data_as(C.c_void_p), flags=0):
        return lib.gg_dp_train_steps_ex(comm, 0, 10, start_list, 1, batch_size, fake, fake, fake, 10, 128, fake, fake, fake, fake,
                                        fake, fake, f(0), fake, fake, 4096, fake, fake, fake, fake, fake, f(1e-3), f(0.9),
                                        f(0.999), f(1e-8), C.byref(b1), C.byref(b2), fake, 1 << 30, flags, None)

    for n in (4096, 64, 0):
        assert step(n_pairs=n) != 0 and b"gg_dp_step_ex" in lib.gg_last_error() and b"communicator" in lib.gg_last_error()
    assert loop() != 0 and b"gg_dp_train_steps_ex" in lib.gg_last_error()
    # the checks that need no communicator state: flags, batch size, host pointers (fake communicator never dereferenced)
    assert step(comm=fake, flags=4) != 0 and b"flags" in lib.gg_last_error()
    assert loop(comm=fake, flags=4) != 0 and b"flags" in lib.gg_last_error()
    assert loop(comm=fake, batch_size=0) != 0 and b"batch size" in lib.gg_last_error()
    assert loop(comm=fake, batch_size=1 << 30) != 0 and b"batch size" in lib.gg_last_error()
    assert loop(comm=fake, start_list=None) != 0 and b"null host pointer" in lib.gg_last_error()
    # the old entry points keep their limit
    rc = lib.gg_dp_train_steps(fake, 0, 10, starts.ctypes.data_as(C.c_void_p), 1, 2048, fake, fake, fake, 10, 128, fake, fake,
                               fake, fake, fake, fake, f(0), fake, fake, 4096, fake, fake, fake, fake, fake, f(1e-3), f(0.9),
                               f(0.999), f(1e-8), C.byref(b1), C.byref(b2), None)
    assert rc != 0 and b"batch size" in lib.gg_last_error()


@pytest.mark.parametrize("transport", ["p2p", None])
def test_data_parallel_large_batch_needs_nccl_before_communicating(transport):
    """A DataParallelStep on the peer-memory transport (or none) refuses B = 1025 with ValueError; no process group
    exists here, so any communication would fail differently."""
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.parallel import DataParallelStep
    dp = object.__new__(DataParallelStep)
    dp.model = Discriminator(50, np.zeros((50, 16)), device="cpu")
    if transport is not None:
        dp.transport = transport
    i = np.zeros(1025, np.int32)
    with pytest.raises(ValueError, match="GG_MAX_BATCH"):
        dp.step(i, i, i.astype(np.float32))
    with pytest.raises(ValueError, match="GG_MAX_BATCH"):
        dp.train_steps(i, i, i.astype(np.float32), [0], 1025)
    assert dp.model.step_count == 0
