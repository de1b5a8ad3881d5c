"""CPU tests of the large mini-batch surface: scratch sizing, argument errors that return instead of aborting, and the
Python layers refusing what only the one-CTA gradient supports before anything reaches a device."""
import ctypes as C

import numpy as np
import pytest


def _scratch_bytes(lib, n_pairs, ld):
    n = C.c_int64(0)
    rc = lib.gg_pair_grad_scratch_bytes(n_pairs, ld, C.byref(n))
    return rc, n.value


def test_scratch_bytes_grow_with_pairs_and_width():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    sizes = {}
    for B in (1, 1024, 1025, 65536):
        for ld in (32, 64, 128, 256):
            rc, n = _scratch_bytes(lib, B, ld)
            assert rc == 0 and n > 0
            sizes[B, ld] = n
    for ld in (32, 64, 128, 256):
        assert sizes[1, ld] < sizes[1024, ld] < sizes[1025, ld] < sizes[65536, ld]
    for B in (1, 1024, 1025, 65536):
        assert sizes[B, 32] < sizes[B, 64] < sizes[B, 128] < sizes[B, 256]
    # at least the term vectors: 2B entries of (ld + 1) floats
    assert sizes[65536, 128] >= 2 * 65536 * 129 * 4


def test_bad_arguments_return_errors():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    for B, ld in ((0, 128), (-3, 128), (1 << 30, 128), (64, 48)):
        assert _scratch_bytes(lib, B, ld)[0] != 0
        assert b"gg_pair_grad_scratch_bytes" in lib.gg_last_error()
    assert lib.gg_pair_grad_scratch_bytes(64, 128, None) != 0
    fake = 1 << 20       # never dereferenced: every check below fails before a device pointer is used
    def ex(mode=0, n_pairs=2048, ld=128, scratch=fake, scratch_bytes=None, flags=0):
        if scratch_bytes is None:
            scratch_bytes = _scratch_bytes(lib, max(n_pairs, 1), ld)[1]
        rc = lib.gg_pair_grad_ex(mode, n_pairs, 0, fake, fake, fake, fake, fake, ld, C.c_float(0), fake, fake, fake, fake, fake,
                                 scratch, scratch_bytes, flags, None)
        return rc, lib.gg_last_error().decode()
    for kw, what in ((dict(mode=7), "mode"), (dict(n_pairs=0), "n_pairs"), (dict(n_pairs=1 << 30), "n_pairs"),
                     (dict(flags=4), "flags"), (dict(ld=48), "ld"), (dict(scratch_bytes=1000), "scratch"),
                     (dict(scratch=None), "scratch"), (dict(scratch=fake + 16), "aligned"),
                     (dict(n_pairs=64, flags=1, scratch_bytes=0), "scratch")):
        rc, msg = ex(**kw)
        assert rc != 0 and "gg_pair_grad_ex" in msg and what in msg, (kw, msg)
    b1, b2 = C.c_float(0.9), C.c_float(0.999)
    starts = np.zeros(1, np.int64)
    for bs, st in ((0, starts.ctypes.data_as(C.c_void_p)), (2048, None)):
        rc = lib.gg_train_steps_ex(0, 10, st, 1, bs, fake, fake, fake, 10, 128, fake, fake, fake, fake, fake, fake, C.c_float(0),
                                   fake, fake, fake, fake, fake, C.c_float(1e-3), b1, b2, C.c_float(1e-8), C.byref(b1), C.byref(b2),
                                   None, 0, None)
        assert rc != 0 and b"gg_train_steps_ex" in lib.gg_last_error()
    # the old entry points keep their limit
    rc = lib.gg_train_steps(0, 10, starts.ctypes.data_as(C.c_void_p), 1, 2048, fake, fake, fake, 10, 128, fake, fake, fake, fake,
                            fake, fake, C.c_float(0), fake, fake, fake, fake, fake, C.c_float(1e-3), b1, b2, C.c_float(1e-8),
                            C.byref(b1), C.byref(b2), None)
    assert rc != 0 and b"batch size" in lib.gg_last_error()
    assert lib.gg_pair_grad(0, 2048, 0, fake, fake, fake, fake, fake, 128, C.c_float(0), fake, fake, fake, fake, fake, None) != 0


def test_persistent_loops_refuse_large_batches_before_device_work():
    """train_steps(persistent=True / "two-barrier") above GG_MAX_BATCH raises ValueError at once; the inputs here are
    host arrays on a CPU-placed model, so any device call would fail differently."""
    from graphgan_b200.discriminator import Discriminator
    m = Discriminator(50, np.zeros((50, 16)), device="cpu")
    i = np.zeros(3000, np.int32)
    for how in (True, "two-barrier"):
        with pytest.raises(ValueError, match="GG_MAX_BATCH"):
            m.train_steps(i, i, i.astype(np.float32), [0], 3000, persistent=how)
    assert m.step_count == 0


def test_data_parallel_refuses_large_batches_before_communicating():
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.parallel import DataParallelStep
    dp = object.__new__(DataParallelStep)      # no process group: the check runs before any communication
    dp.model = Discriminator(50, np.zeros((50, 16)), device="cpu")
    i = np.zeros(1025, np.int32)
    with pytest.raises(ValueError, match="GG_MAX_BATCH"):
        dp.step(i, i, i.astype(np.float32))
    with pytest.raises(ValueError, match="GG_MAX_BATCH"):
        dp.train_steps(i, i, i.astype(np.float32), [0], 1025)
