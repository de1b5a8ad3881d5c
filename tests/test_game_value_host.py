"""The game value's host reference (tests/game_value_oracle.py) against scipy and the C oracle, and the argument checks of
gg_game_value.  No GPU."""
import ctypes as C

import numpy as np
import pytest

from tests import game_value_oracle as vo


def test_bce_is_minus_log_sigmoid():
    from scipy.special import log_expit
    s = np.array([100, -100, 20, -20, 1e-8, -1e-8, 0.0], np.float32)
    x = s.astype(np.float64)
    for y, want in ((1, -log_expit(x)), (0, -log_expit(-x))):
        got = vo.bce(s, y)
        assert np.all(np.abs(got - want) <= 2 * np.spacing(np.abs(want))), (y, got, want)
    assert vo.bce(np.float32(-100), 1) == 100.0 and vo.bce(np.float32(100), 0) == 100.0


@pytest.mark.parametrize("ld", [32, 64, 128, 256, 512])
def test_scores_are_the_c_oracles_dot_plus_bias(ld):
    from oracle import canonical as can
    rs = np.random.RandomState(ld)
    E = (rs.normal(0, 1, (50, ld)) * rs.choice([1e-3, 1.0, 30.0], (50, 1))).astype(np.float32)
    b = rs.normal(0, 2, 50).astype(np.float32)
    for c in (0, 7, 49):
        vs = rs.randint(0, 50, 80)
        got = vo.scores(E, b, c, vs)
        want = np.array([np.float32(can.dot_c(E[c], E[v]) + b[v]) for v in vs], np.float32)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def _call(lib, n_node=100, ld=64, n_roots=2, null=(), scratch_bytes=1 << 20):
    p = {k: (None if k in null else C.c_void_p(0x1000)) for k in
         ("emb", "bias", "indptr", "adj", "roots", "dist", "root_ok", "pos", "neg", "ok", "scratch")}
    return lib.gg_game_value(n_node, ld, p["emb"], p["bias"], p["indptr"], p["adj"], n_roots, p["roots"], p["dist"],
                             p["root_ok"], p["pos"], p["neg"], p["ok"], p["scratch"], scratch_bytes, None)


@pytest.mark.parametrize("bad", [
    dict(ld=48), dict(ld=1024), dict(ld=0), dict(n_node=0), dict(n_node=-5), dict(n_roots=-1), dict(scratch_bytes=8),
    dict(null=("emb",)), dict(null=("bias",)), dict(null=("indptr",)), dict(null=("adj",)), dict(null=("roots",)),
    dict(null=("dist",)), dict(null=("root_ok",)), dict(null=("pos",)), dict(null=("neg",)), dict(null=("ok",)),
    dict(null=("scratch",)),
])
def test_entry_point_refuses_bad_arguments(bad):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rc = _call(lib, **bad)
    assert rc != 0
    with pytest.raises(_cabi.GGError):
        _cabi.check(rc, "gg_game_value")


def test_scratch_size_and_empty_batch():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    n = C.c_int64(-1)
    assert lib.gg_game_value_scratch_bytes(1000, 3, C.byref(n)) == 0 and n.value == 3 * 2 * 8   # 512 nodes per tile
    assert lib.gg_game_value_scratch_bytes(0, 0, C.byref(n)) == 0 and n.value == 0
    assert lib.gg_game_value_scratch_bytes(-1, 3, C.byref(n)) != 0
    assert lib.gg_game_value_scratch_bytes(10, -3, C.byref(n)) != 0
    assert lib.gg_game_value_scratch_bytes(10, 3, None) != 0
    # no roots: nothing to do, no pointer is looked at
    assert _call(lib, n_roots=0, null=("emb", "dist", "pos", "scratch")) == 0
