"""The value gradient's host reference (tests/value_grad_oracle.py) and the argument checks of gg_game_value_grad.  No GPU.

- The "smooth" law's gradient is the derivative of its own V: central finite differences along random directions.
- The "pi" law's gradient (the kernel's definition) differs from the smooth one by no more than the step-law bound of
  DESIGN.md section 5.3.
- Sum_y grad_b[y] = 0 and T(root) = -neg_c, to within fp64 rounding.
"""
import ctypes as C

import numpy as np
import pytest

from tests import value_grad_oracle as gro
from tests.golden import loader


def _setup(name, removal, k=6, seed=1):
    from graphgan_b200 import graph as G
    from oracle import canonical as can
    case = loader.load(name)
    hg = G.HostGraph(case["train_edges"], case["test_edges"], n_node=case.n)
    rs = np.random.RandomState(seed)
    cand = np.flatnonzero(hg.degrees() > 0)
    roots = np.sort(rs.choice(cand, min(k, len(cand)), replace=False)).astype(np.int32)
    par = can.bfs_parents(hg.indptr, hg.adj, roots)
    E_g = can.pad_rows(case.emb_g)
    b_g = rs.normal(0, 0.2, hg.n_node).astype(np.float32)
    E_d = can.pad_rows(case.emb_d)
    b_d = rs.normal(0, 0.3, hg.n_node).astype(np.float32)
    bits = np.zeros((len(hg.adj) + 31) // 32 + 1, np.uint32)
    if removal:
        can.walk_pass(E_g, b_g, hg.indptr, hg.adj, roots, par, hg.degrees()[roots], True, bits, seed=5, pass_tag=1)
        assert bits.any()
    return hg, roots, par, bits, E_g, b_g, E_d, b_d


def _neg_smooth(E, b, E_d, b_d, hg, roots, par, bits):
    return sum(gro.root_grad(E, b, E_d, b_d, hg, int(r), par[k], bits, "smooth")["neg"] for k, r in enumerate(roots))


@pytest.mark.parametrize("removal", [False, True])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_smooth_gradient_matches_finite_differences(name, removal):
    hg, roots, par, bits, E_g, b_g, E_d, b_d = _setup(name, removal)
    E, b = E_g.astype(np.float64), b_g.astype(np.float64)
    gE, gb, _, _, per = gro.grad(E, b, E_d, b_d, hg, roots, par, bits, "smooth")
    assert any(o["ok"] for o in per)
    d = _dim(E_g)
    rs = np.random.RandomState(3)
    eps = 1e-5
    for _ in range(4):
        dE = np.zeros_like(E)
        dE[:, :d] = rs.normal(0, 1, (hg.n_node, d))
        db = rs.normal(0, 1, hg.n_node)
        fd = (_neg_smooth(E + eps * dE, b + eps * db, E_d, b_d, hg, roots, par, bits)
              - _neg_smooth(E - eps * dE, b - eps * db, E_d, b_d, hg, roots, par, bits)) / (2 * eps)
        an = float((gE * dE).sum() + (gb * db).sum())
        scale = float(np.abs(gE * dE).sum() + np.abs(gb * db).sum())
        assert abs(fd - an) <= 1e-6 * scale, (fd, an, scale)


def _dim(E):
    """the embedding columns that are not padding"""
    nz = np.flatnonzero(np.abs(E).sum(axis=0))
    return int(nz[-1]) + 1 if len(nz) else E.shape[1]


@pytest.mark.parametrize("removal", [False, True])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_pi_gradient_is_within_the_step_law_bound_of_the_smooth_one(name, removal):
    """|grad_pi - grad_smooth| <= 4 (D + 2) delta A per coordinate: delta the largest relative difference between pi and the
    smooth law over the records of reached lists, D the depth of the tree, A the coordinate's sum of |F E| + |pi T E|."""
    hg, roots, par, bits, E_g, b_g, E_d, b_d = _setup(name, removal)
    for k, r in enumerate(roots):
        a = gro.root_grad(E_g, b_g, E_d, b_d, hg, int(r), par[k], bits, "pi")
        s = gro.root_grad(E_g, b_g, E_d, b_d, hg, int(r), par[k], bits, "smooth")
        assert a["ok"] == s["ok"]
        if not a["ok"]:
            continue
        live = a["T"][a["owner"]] > 0
        delta = float(np.max(np.abs(a["pi"] - s["pi"])[live] / s["pi"][live]))
        assert delta < 1e-5, delta                             # fp32 scores and softmax: a few fp32 ulp
        bound = 4 * (max(a["depth"], s["depth"]) + 2) * delta
        assert np.all(np.abs(a["gE"] - s["gE"]) <= bound * (a["abs_E"] + s["abs_E"])), int(r)
        assert np.all(np.abs(a["gb"] - s["gb"]) <= bound * (a["abs_b"] + s["abs_b"])), int(r)


@pytest.mark.parametrize("name", ["tiny", "rand300", "rand1200"])
def test_bias_gradient_sums_to_zero_and_T_root_is_minus_neg(name):
    hg, roots, par, bits, E_g, b_g, E_d, b_d = _setup(name, True, k=10)
    for k, r in enumerate(roots):
        o = gro.root_grad(E_g, b_g, E_d, b_d, hg, int(r), par[k], bits, "pi")
        if not o["ok"]:
            continue
        assert abs(o["gb"].sum()) <= 1e-13 * o["abs_b"].sum()
        assert abs(o["T_root"] + o["neg"]) <= 1e-14 * abs(o["neg"])
        assert o["T_root"] > 0


def _call(lib, desc=True, ld=64, n_node=100, n_roots=2, null=(), scratch_bytes=1 << 40, tree_words=8, n_roots_big=False):
    from graphgan_b200 import _cabi
    d = _cabi.WalkDesc()
    d.n_node, d.ld, d.n_roots, d.tree_words = n_node, ld, n_roots, tree_words
    for f in ("emb", "bias", "indptr", "adj", "roots", "tree_bits"):
        setattr(d, f, None if f in null else 0x1000)
    if n_roots_big:
        d.n_node, d.n_roots = 1 << 20, 1 << 11
    p = {k: (None if k in null else C.c_void_p(0x1000)) for k in
         ("d_emb", "d_bias", "raw_indptr", "raw_adj", "pos", "neg", "ok", "grad_emb", "grad_bias", "scratch")}
    return lib.gg_game_value_grad(C.byref(d) if desc else None, p["d_emb"], p["d_bias"], p["raw_indptr"], p["raw_adj"],
                                  p["pos"], p["neg"], p["ok"], p["grad_emb"], p["grad_bias"], p["scratch"], scratch_bytes,
                                  None)


@pytest.mark.parametrize("bad", [
    dict(desc=False), dict(ld=48), dict(ld=1024), dict(ld=0), dict(n_node=0), dict(n_roots=-1), dict(tree_words=0),
    dict(scratch_bytes=8), dict(n_roots_big=True),
    dict(null=("emb",)), dict(null=("bias",)), dict(null=("indptr",)), dict(null=("adj",)), dict(null=("roots",)),
    dict(null=("tree_bits",)), dict(null=("d_emb",)), dict(null=("d_bias",)), dict(null=("raw_indptr",)),
    dict(null=("raw_adj",)), dict(null=("pos",)), dict(null=("neg",)), dict(null=("ok",)), dict(null=("grad_emb",)),
    dict(null=("grad_bias",)), dict(null=("scratch",)),
])
def test_entry_point_refuses_bad_arguments(bad):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rc = _call(lib, **bad)
    assert rc != 0
    with pytest.raises(_cabi.GGError):
        _cabi.check(rc, "gg_game_value_grad")


def test_scratch_size_and_empty_batch():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    n, base, one, two = C.c_int64(-1), C.c_int64(-1), C.c_int64(-1), C.c_int64(-1)
    assert lib.gg_game_value_grad_scratch_bytes(1000, 20000, 0, C.byref(base)) == 0
    assert lib.gg_game_value_grad_scratch_bytes(1000, 20000, 1, C.byref(one)) == 0
    assert lib.gg_game_value_grad_scratch_bytes(1000, 20000, 2, C.byref(two)) == 0
    per_root = two.value - one.value
    gd = C.c_int64(-1)
    assert lib.gg_generator_dist_scratch_bytes(1000, 20000, 1, C.byref(gd)) == 0 and lib.gg_generator_dist_scratch_bytes(
        1000, 20000, 2, C.byref(n)) == 0
    # per root: the section 5.1 scratch (less one of its two item lists), dist, h, T, pi_in, pi_stop and father
    # (the section 5.1 scratch + 28 bytes per node), and the value kernel's tile partials
    assert abs(per_root - ((n.value - gd.value) + 28 * 1000)) <= 4 * 256 + 16
    assert base.value > 0                                       # the level offsets and the big-node list do not scale with roots
    assert lib.gg_game_value_grad_scratch_bytes(-1, 3, 3, C.byref(n)) != 0
    assert lib.gg_game_value_grad_scratch_bytes(10, -3, 3, C.byref(n)) != 0
    assert lib.gg_game_value_grad_scratch_bytes(10, 3, -3, C.byref(n)) != 0
    assert lib.gg_game_value_grad_scratch_bytes(10, 3, 3, None) != 0
    # no roots: nothing to do, no pointer is looked at
    assert _call(lib, n_roots=0, null=("emb", "d_emb", "pos", "grad_emb", "scratch"), scratch_bytes=0) == 0
