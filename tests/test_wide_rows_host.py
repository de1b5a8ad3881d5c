"""Host-side rules of the ld = 512 row stride (no GPU): pad_embedding picks ld 512 for 256 < n_emb <= 512 and refuses
wider rows; the C entry points refuse strides the kernels are not built for with an error code and a message."""
import ctypes as C

import numpy as np
import pytest


@pytest.mark.parametrize("d", [257, 300, 512])
def test_pad_embedding_512(d):
    from graphgan_b200.sampler import pad_embedding
    e = np.random.RandomState(d).normal(0, 1, size=(5, d))
    out = pad_embedding(e, "cpu")
    assert tuple(out.shape) == (5, 512)
    assert np.array_equal(out[:, :d].numpy(), e.astype(np.float32))
    assert not out[:, d:].numpy().any()


def test_pad_embedding_rule_below_257_unchanged():
    from graphgan_b200.sampler import pad_embedding
    for d, ld in ((1, 32), (32, 32), (33, 64), (128, 128), (200, 256), (256, 256)):
        assert pad_embedding(np.zeros((2, d)), "cpu").shape[1] == ld


def test_pad_embedding_513_raises():
    from graphgan_b200.sampler import pad_embedding
    with pytest.raises(ValueError, match="at most 512"):
        pad_embedding(np.zeros((2, 513)), "cpu")


@pytest.mark.parametrize("ld", [384, 1024, 48])
def test_c_abi_refuses_other_strides(ld):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    n = C.c_int64(0)
    assert lib.gg_pair_grad_scratch_bytes(64, ld, C.byref(n)) != 0
    assert b"512" in lib.gg_last_error()
    assert lib.gg_grad_merge_scratch_bytes(2, 64, ld, C.byref(n)) != 0
    assert b"512" in lib.gg_last_error()
    d = _cabi.WalkDesc()
    d.ld, d.n_walks, d.n_roots = ld, 1, 1
    assert lib.gg_walk_sample(C.byref(d), None) != 0
    assert b"512" in lib.gg_last_error()


@pytest.mark.parametrize("ld", [32, 256, 512])
def test_c_abi_accepts_supported_strides(ld):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    n = C.c_int64(0)
    assert lib.gg_pair_grad_scratch_bytes(64, ld, C.byref(n)) == 0 and n.value > 0
    assert lib.gg_grad_merge_scratch_bytes(2, 64, ld, C.byref(n)) == 0 and n.value > 0
