"""Training on the exact game (DESIGN.md section 5.5), without a GPU: the ABI version, the argument checks of
gg_adam_apply_dense, the numpy statement of its step (tests/exact_steps_oracle.py) and the single-process rule of
config.exact_roots.
"""
import ctypes as C
import math
import types

import numpy as np
import pytest

from tests import exact_steps_oracle as eso
from tests import update_bits_oracle as ubo

F = np.float32


def test_abi_version():
    from graphgan_b200 import _cabi
    assert _cabi.ABI_VERSION == 11 and _cabi.lib().gg_abi_version() == 11


def _call(lib, n_node=100, ld=64, scale=1.0, null=()):
    p = {k: (None if k in null else C.c_void_p(0x1000)) for k in
         ("emb", "m_emb", "v_emb", "bias", "m_bias", "v_bias", "acc_emb", "acc_bias")}
    return lib.gg_adam_apply_dense(n_node, ld, p["emb"], p["m_emb"], p["v_emb"], p["bias"], p["m_bias"], p["v_bias"],
                                   p["acc_emb"], p["acc_bias"], scale, 1e-5, 0.0, 1e-3, 0.9, 0.999, 1e-8, None)


@pytest.mark.parametrize("bad", [
    dict(ld=48), dict(ld=1024), dict(ld=0), dict(ld=16), dict(n_node=0), dict(n_node=-5),
    dict(scale=math.nan), dict(scale=math.inf), dict(scale=-math.inf),
    dict(null=("emb",)), dict(null=("m_emb",)), dict(null=("v_emb",)), dict(null=("bias",)), dict(null=("m_bias",)),
    dict(null=("v_bias",)), dict(null=("acc_emb",)), dict(null=("acc_bias",)),
])
def test_entry_point_refuses_bad_arguments(bad):
    """A refused call returns non-zero with a message and launches nothing (the pointers are not device memory: a launch
    would fail, and there is no device here)."""
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rc = _call(lib, **bad)
    assert rc != 0
    with pytest.raises(_cabi.GGError):
        _cabi.check(rc, "gg_adam_apply_dense")


@pytest.mark.parametrize("lam_bias", [0.0, 0.03])
@pytest.mark.parametrize("scale", [1.0, -1.0 / 3, 1.0 / 7])
def test_numpy_step_is_the_literal_statement(scale, lam_bias):
    rs = np.random.RandomState(11)
    n, n_emb, ld = 9, 5, 32
    a = eso.random_state(n, n_emb, ld, rs)
    b = {k: v.copy() for k, v in a.items()}
    acc = np.zeros((n, ld))
    acc[:, :n_emb] = rs.normal(0, 1, (n, n_emb))
    acc_b = rs.normal(0, 1, n)
    lt = ubo.lr_t(1e-3, F(0.9) ** 3, F(0.999) ** 3)
    eso.dense_step(a, acc, acc_b, scale, 0.05, lam_bias, lt)
    eso.dense_step_literal(b, acc, acc_b, scale, 0.05, lam_bias, lt)
    for k in a:
        assert ubo.same(a[k], b[k]), k
    assert not a["emb"][:, n_emb:].any() and not a["m_emb"][:, n_emb:].any() and not a["v_emb"][:, n_emb:].any()


def test_numpy_step_reduces_to_the_sparse_step():
    """scale 1, lam 0 and acc = (double) g32: the dense step is adam1 fed g32 (the fp64 products and sum are exact)."""
    rs = np.random.RandomState(3)
    n, n_emb, ld = 20, 12, 32
    a = eso.random_state(n, n_emb, ld, rs)
    b = {k: v.copy() for k, v in a.items()}
    g = np.zeros((n, ld), F)
    g[::3, :n_emb] = rs.normal(0, 0.1, (len(range(0, n, 3)), n_emb)).astype(F)
    gb = np.zeros(n, F)
    gb[::3] = rs.normal(0, 0.1, len(range(0, n, 3))).astype(F)
    lt = ubo.lr_t(1e-3, F(0.9), F(0.999))
    eso.dense_step(a, g.astype(np.float64), gb.astype(np.float64), 1.0, 0.0, 0.0, lt)
    ubo.adam1(b["emb"], b["m_emb"], b["v_emb"], g, lt, F(0.9), F(0.999), F(1e-8))
    ubo.adam1(b["bias_t"], b["m_bias"], b["v_bias"], gb, lt, F(0.9), F(0.999), F(1e-8))
    for k in a:
        assert ubo.same(a[k], b[k]), k


def test_exact_roots_is_single_process():
    from graphgan_b200 import config
    from graphgan_b200.graph_gan import check_exact_mode
    assert config.exact_roots == 0
    check_exact_mode(config, 4)                                      # the default: sampled training, any world size
    cfg = types.SimpleNamespace(exact_roots=64)
    check_exact_mode(cfg, 1)
    for world in (2, 8):
        with pytest.raises(ValueError):
            check_exact_mode(cfg, world)
