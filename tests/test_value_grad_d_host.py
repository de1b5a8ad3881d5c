"""The discriminator gradient's host reference (tests/value_grad_d_oracle.py) and the argument checks of
gg_game_value_grad_d.  No GPU.

- The "smooth" law's gradient is the derivative of its own V: central finite differences along random directions in
  (E_D, b_D), on the fixtures and on a small graph with duplicate raw entries and self-loops (the multiplicities n_kv
  and the factor 2 of d(E_c . E_c) / dE_c).
- The entry point refuses bad arguments, and its scratch size is the documented one.
"""
import ctypes as C

import numpy as np
import pytest

from tests import value_grad_d_oracle as dgo
from tests.golden import loader


def _fixture(name, removal, k=6, seed=1):
    from graphgan_b200 import graph as G
    from oracle import canonical as can
    case = loader.load(name)
    hg = G.HostGraph(case["train_edges"], case["test_edges"], n_node=case.n)
    rs = np.random.RandomState(seed)
    roots = np.sort(rs.choice(np.flatnonzero(hg.degrees() > 0), k, replace=False)).astype(np.int32)
    E_g, b_g = can.pad_rows(case.emb_g), rs.normal(0, 0.2, hg.n_node).astype(np.float32)
    E_d, b_d = can.pad_rows(case.emb_d), rs.normal(0, 0.3, hg.n_node).astype(np.float32)
    return hg, roots, E_g, b_g, E_d, b_d, case.emb_d.shape[1], removal


def _laws(hg, roots, E_g, b_g, removal):
    from oracle import canonical as can
    par = can.bfs_parents(hg.indptr, hg.adj, roots)
    bits = np.zeros((len(hg.adj) + 31) // 32 + 1, np.uint32)
    if removal:
        can.walk_pass(E_g, b_g, hg.indptr, hg.adj, roots, par, hg.degrees()[roots], True, bits, seed=5, pass_tag=1)
        assert bits.any()
    return dgo.laws(E_g, b_g, hg, roots, par, bits)


def _check_fd(hg, roots, dists, oks, E_d, b_d, d, seed=3):
    E, b = E_d.astype(np.float64), b_d.astype(np.float64)
    gE, gb, _, _ = dgo.grad(E, b, hg, roots, dists, oks, "smooth")
    assert np.abs(gE).sum() > 0 and not gE[:, d:].any()
    rs = np.random.RandomState(seed)
    eps = 1e-5
    for _ in range(4):
        dE = np.zeros_like(E)
        dE[:, :d] = rs.normal(0, 1, (hg.n_node, d))
        db = rs.normal(0, 1, hg.n_node)
        fd = (dgo.value_smooth(E + eps * dE, b + eps * db, hg, roots, dists, oks)
              - dgo.value_smooth(E - eps * dE, b - eps * db, hg, roots, dists, oks)) / (2 * eps)
        an = float((gE * dE).sum() + (gb * db).sum())
        scale = float(np.abs(gE * dE).sum() + np.abs(gb * db).sum())
        assert abs(fd - an) <= 1e-6 * scale, (fd, an, scale)


@pytest.mark.parametrize("removal", [False, True])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_smooth_gradient_matches_finite_differences(name, removal):
    hg, roots, E_g, b_g, E_d, b_d, d, _ = _fixture(name, removal)
    dists, oks = _laws(hg, roots, E_g, b_g, removal)
    assert oks.any()
    _check_fd(hg, roots, dists, oks, E_d, b_d, d)


def test_duplicates_and_self_loops():
    """graph[0] = [1, 1, 0, 0, 3] (a duplicate edge and a self-loop), graph[2] holds a self-loop too: the positives count
    every raw entry, and s(c, c) = E_c . E_c + b_c takes both the node side and the centre side."""
    from graphgan_b200 import graph as G
    from oracle import canonical as can
    edges = [(0, 1), (0, 1), (0, 0), (1, 2), (2, 3), (0, 3), (3, 4), (4, 5), (2, 2), (5, 1)]
    hg = G.HostGraph(edges, None, n_node=6)
    assert list(hg.neighbors(0)) == [1, 1, 0, 0, 3]
    rs = np.random.RandomState(7)
    d = 8
    E_g, b_g = can.pad_rows(rs.normal(0, 0.5, (6, d))), rs.normal(0, 0.3, 6).astype(np.float32)
    E_d, b_d = can.pad_rows(rs.normal(0, 0.5, (6, d))), rs.normal(0, 0.3, 6).astype(np.float32)
    roots = np.arange(6, dtype=np.int32)
    dists, oks = _laws(hg, roots, E_g, b_g, False)
    assert oks.all()
    W, _ = dgo.root_w(E_d, b_d, hg, 0, dists[0], oks[0], "smooth")
    assert W[0] > 0 and W[1] > 0                             # the self-loop and the duplicate are positives
    _check_fd(hg, roots, dists, oks, E_d, b_d, d)
    # the positive part alone: n_kv / deg_c weights, the self-loop counted twice in graph[0]
    zero = np.zeros_like(dists)
    _check_fd(hg, roots, zero, oks, E_d, b_d, d, seed=4)


def _call(lib, ld=64, n_node=100, n_roots=2, null=(), scratch_bytes=1 << 40):
    p = {k: (None if k in null else C.c_void_p(0x1000)) for k in
         ("emb", "bias", "raw_indptr", "raw_adj", "roots", "dist", "root_ok", "grad_emb", "grad_bias", "scratch")}
    return lib.gg_game_value_grad_d(n_node, ld, p["emb"], p["bias"], p["raw_indptr"], p["raw_adj"], n_roots, p["roots"],
                                    p["dist"], p["root_ok"], p["grad_emb"], p["grad_bias"], p["scratch"], scratch_bytes,
                                    None)


@pytest.mark.parametrize("bad", [
    dict(ld=48), dict(ld=1024), dict(ld=0), dict(n_node=0), dict(n_node=1 << 31), dict(n_roots=-1), dict(scratch_bytes=8),
    dict(null=("emb",)), dict(null=("bias",)), dict(null=("raw_indptr",)), dict(null=("raw_adj",)), dict(null=("roots",)),
    dict(null=("dist",)), dict(null=("root_ok",)), dict(null=("grad_emb",)), dict(null=("grad_bias",)),
    dict(null=("scratch",)),
])
def test_entry_point_refuses_bad_arguments(bad):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rc = _call(lib, **bad)
    assert rc != 0
    with pytest.raises(_cabi.GGError):
        _cabi.check(rc, "gg_game_value_grad_d")


@pytest.mark.parametrize("ld", [32, 128, 512])
def test_scratch_size_and_empty_batch(ld):
    """12 bytes per (root, node): the multiplicity plane (int32) and W (fp64); per root, ld fp64 partials per 2048-node
    tile of the centre pass and the ld sums C_k; each part 256-byte aligned."""
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    n = 100_000
    tiles = (n + 2047) // 2048
    for R in (0, 1, 2, 7, 64):
        got = C.c_int64(-1)
        assert lib.gg_game_value_grad_d_scratch_bytes(n, ld, R, C.byref(got)) == 0
        want = 12 * R * n + 8 * R * ld * (tiles + 1)
        assert want <= got.value <= want + 4 * 255, (R, got.value, want)
    x = C.c_int64(0)
    assert lib.gg_game_value_grad_d_scratch_bytes(-1, ld, 3, C.byref(x)) != 0
    assert lib.gg_game_value_grad_d_scratch_bytes(10, ld, -3, C.byref(x)) != 0
    assert lib.gg_game_value_grad_d_scratch_bytes(10, 48, 3, C.byref(x)) != 0
    assert lib.gg_game_value_grad_d_scratch_bytes(10, ld, 3, None) != 0
    # no roots: nothing to do, no pointer is looked at
    assert _call(lib, n_roots=0, null=("emb", "dist", "grad_emb", "scratch"), scratch_bytes=0) == 0
