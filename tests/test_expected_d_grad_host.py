"""The host reference of the D-mode walk law and the expected reference D step (tests/expected_d_grad_oracle.py), and the
argument checks of gg_generator_dist_d and gg_expected_d_grad.  No GPU.

- Exact enumeration: every D walk of a root under the reference's own rules (graph_gan.py:243-268, for_d=True) on tree
  lists that already carry a D pass's root removals or not, with the kernel's step law as exact rationals.  Its stop
  mass is P_D and its void mass p_void, whatever the removal bits.
- P_acc is the square-and-multiply of DESIGN.md section 5.7.
- The expected step is minus the gradient of the expected pass loss with the law held fixed: central finite differences.
"""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

from tests import expected_d_grad_oracle as eo
from tests import gdist_oracle as go
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


def _tree_lists(hg, root, parent, bits):
    """the reference's tree dict for one root (graph_gan.py:96-107): tree[root] = [root] + children, tree[v] = [father] +
    children, children in walk-CSR entry order; a set removal bit of entry (root -> a) drops root from tree[a]"""
    tree = {}
    for v in np.flatnonzero(parent >= 0).tolist() + [root]:
        nb = hg.adj[hg.indptr[v]:hg.indptr[v + 1]].tolist()
        kids = [int(x) for x in nb if x != root and parent[x] == v]
        tree[v] = [root if v == root else int(parent[v])] + kids
    for e in range(hg.indptr[root], hg.indptr[root + 1]):
        a = int(hg.adj[e])
        if parent[a] == root and (bits[e >> 5] >> (e & 31)) & 1:
            tree[a].remove(root)
    return tree


def _pi_exact(E, b, node, cands):
    """the kernel's step law of the list ``cands`` owned by ``node``, as exact rationals"""
    cands = np.asarray(cands, np.int64)
    sc = (go.dots(E, np.full(len(cands), node, np.int64), cands) + b[cands]).astype(np.float32)
    q = go.list_q(sc, np.array([0, len(cands)], np.int64))
    return [Fraction(k, 2 ** 53) for k in go.step_pi_exact(q)]


def _enumerate_d_walks(E, b, tree, root):
    """({v: stop mass}, void mass) of one D walk from ``root`` under the reference's rules, exactly"""
    stops, void = {}, Fraction(0)
    stack = [(root, -1, True, Fraction(1))]
    while stack:
        cur, prev, is_root, mass = stack.pop()
        nb = list(tree[cur][1:] if is_root else tree[cur])
        if len(nb) == 0 or nb == [root]:                       # graph_gan.py:252-257: the pass returns None
            void += mass
            continue
        if root in nb:                                          # graph_gan.py:258-259
            nb.remove(root)
        for x, p in zip(nb, _pi_exact(E, b, cur, nb)):
            if p == 0:
                continue
            if x == prev:                                       # graph_gan.py:264-266
                stops[cur] = stops.get(cur, Fraction(0)) + mass * p
            else:
                stack.append((x, cur, False, mass * p))
    return stops, void


@pytest.mark.parametrize("removal", [False, True])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_law_matches_enumerated_d_walks(name, removal):
    hg, roots, par, bits, E_g, b_g, E_d, b_d = _setup(name, removal, k=20)
    n_void = 0
    for k, r in enumerate(roots):
        r = int(r)
        P, p_void, ok = eo.d_law(E_g, b_g, hg, r, par[k])
        tree = _tree_lists(hg, r, par[k], bits)
        if len(tree[r]) == 1:
            assert ok == 0 and p_void == 0.0 and not P.any()
            continue
        assert ok == 1
        stops, void = _enumerate_d_walks(E_g, b_g, tree, r)
        assert sum(stops.values()) + void == 1
        assert Fraction(p_void) == void                         # multiples of 2^-53: exact
        n_void += void > 0
        assert set(v for v, m in stops.items() if m > 0) == set(np.flatnonzero(P).tolist())
        for v, m in stops.items():
            assert abs(Fraction(float(P[v])) - m) <= m * Fraction(1, 2 ** 48), (v, float(m), P[v])
        assert abs(P.sum() - (1.0 - p_void)) <= 1e-13
    assert n_void > 0


def test_law_does_not_depend_on_removal_bits():
    """the enumeration under a D pass's removals gives the same masses as without them"""
    hg, roots, par, bits, E_g, b_g, _, _ = _setup("rand300", True, k=10)
    for k, r in enumerate(roots):
        r = int(r)
        clean = _tree_lists(hg, r, par[k], np.zeros_like(bits))
        if len(clean[r]) == 1:
            continue
        a = _enumerate_d_walks(E_g, b_g, clean, r)
        b = _enumerate_d_walks(E_g, b_g, _tree_lists(hg, r, par[k], bits), r)
        assert a == b


def test_without_leaves_and_with_every_bit_set_the_d_law_is_the_g_law():
    hg, roots, par, bits, E_g, b_g, _, _ = _setup("rand300", False, k=20)
    n = 0
    for k, r in enumerate(roots):
        r = int(r)
        P, p_void, ok = eo.d_law(E_g, b_g, hg, r, par[k])
        if not ok or p_void > 0:
            continue
        G, g_ok = go.distribution(E_g, b_g, hg.indptr, hg.adj, r, par[k], eo.all_bits(hg))
        assert g_ok == 1 and np.array_equal(P, G)
        n += 1
    assert n


def _literal_pow(base, e):
    bits = bin(e)[2:][::-1]
    p, sq = 1.0, base
    for i, bit in enumerate(bits):
        if bit == "1":
            p = p * sq
        if i + 1 < len(bits):
            sq = sq * sq
    return p


def test_accept_is_square_and_multiply():
    rs = np.random.RandomState(3)
    degs = [0, 1, 2, 3, 4, 5, 7, 8, 31, 32, 33, 1000, 13828, 2 ** 20 + 3]
    for _ in range(200):
        pv = float(rs.randint(0, 2 ** 53) if rs.rand() < 0.3 else rs.randint(0, 2 ** 20)) / 2.0 ** 53
        for d in degs:
            got = eo.accept(pv, d)
            assert got == _literal_pow(1.0 - pv, d)
            want = float(Fraction(1) - Fraction(pv)) ** d
            assert abs(got - want) <= 1e-13 * max(1, d) * want + 1e-300
    assert eo.accept(0.0, 13828) == 1.0 and eo.accept(1.0, 5) == 0.0 and eo.accept(0.25, 0) == 1.0


def _hand_graph():
    """a root with duplicate raw entries, a self-loop, depth-1 leaves and a deeper subtree"""
    from graphgan_b200 import graph as G
    edges = [(0, 1), (0, 2), (0, 3), (0, 1), (0, 0), (1, 4), (1, 5), (4, 6), (2, 7), (7, 8), (5, 8), (3, 0), (8, 9),
             (10, 10), (11, 12)]
    return G.HostGraph(np.asarray(edges), None, n_node=13)


def _fd_check(hg, roots, par, E_g, b_g, E_d, b_d, seed=7):
    P, pv, ok = eo.d_laws(E_g, b_g, hg, roots, par)
    E, b = E_d.astype(np.float64), b_d.astype(np.float64)
    gE, gb, _, _, acc, okr = eo.grad(E, b, hg, roots, P, pv, ok, law="smooth")
    assert okr.any()
    rs = np.random.RandomState(seed)
    d = int(np.flatnonzero(np.abs(E).sum(axis=0))[-1]) + 1
    eps = 1e-6
    for _ in range(4):
        dE = np.zeros_like(E)
        dE[:, :d] = rs.normal(0, 1, (hg.n_node, d))
        db = rs.normal(0, 1, hg.n_node)
        fd = (eo.pass_loss_smooth(E + eps * dE, b + eps * db, hg, roots, P, pv, ok)
              - eo.pass_loss_smooth(E - eps * dE, b - eps * db, hg, roots, P, pv, ok)) / (2 * eps)
        an = float((gE * dE).sum() + (gb * db).sum())
        scale = float(np.abs(gE * dE).sum() + np.abs(gb * db).sum())
        assert abs(-fd - an) <= 1e-6 * scale, (fd, an, scale)
    return acc, okr, pv


@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_expected_step_matches_finite_differences(name):
    hg, roots, par, bits, E_g, b_g, E_d, b_d = _setup(name, True)
    _fd_check(hg, roots, par, E_g, b_g, E_d, b_d)


def test_expected_step_on_a_hand_built_graph():
    from oracle import canonical as can
    hg = _hand_graph()
    roots = np.array([0, 1, 10, 11], np.int32)
    par = can.bfs_parents(hg.indptr, hg.adj, roots)
    rs = np.random.RandomState(2)
    E_g = can.pad_rows(rs.normal(0, 0.5, (13, 20)).astype(np.float32))
    E_d = can.pad_rows(rs.normal(0, 0.5, (13, 20)).astype(np.float32))
    b_g, b_d = rs.normal(0, 0.2, 13).astype(np.float32), rs.normal(0, 0.3, 13).astype(np.float32)
    assert list(hg.raw_adj[hg.raw_indptr[0]:hg.raw_indptr[1]]) == [1, 2, 3, 1, 0, 0, 3]
    acc, okr, pv = _fd_check(hg, roots, par, E_g, b_g, E_d, b_d)
    assert pv[0] > 0 and okr[0] == 1 and 0 < acc[0] < 1     # node 3 is a depth-1 leaf of root 0
    assert acc[0] == eo.accept(pv[0], 7)                    # deg counts the duplicate and both self-loop entries
    assert okr[2] == 0 and acc[2] == 0.0                    # self-loop only: no children
    assert okr[3] == 0                                      # 11 - 12: every walk lands on a depth-1 leaf


def test_entry_points_are_an_addition_to_abi_11():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    assert _cabi.ABI_VERSION == 11 and lib.gg_abi_version() == 11
    for name in ("gg_generator_dist_d", "gg_expected_d_grad_scratch_bytes", "gg_expected_d_grad"):
        assert name in _cabi.SIGNATURES and getattr(lib, name).argtypes == _cabi.SIGNATURES[name][1]


def _call_law(lib, desc=True, ld=64, n_node=100, n_roots=2, null=(), scratch_bytes=1 << 40, tree_words=8,
              n_roots_big=False, edge_score=False, hub_threshold=128):
    from graphgan_b200 import _cabi
    d = _cabi.WalkDesc()
    d.n_node, d.ld, d.n_roots, d.tree_words = n_node, ld, n_roots, tree_words
    for f in ("emb", "bias", "indptr", "adj", "roots", "tree_bits"):
        setattr(d, f, None if f in null else 0x1000)
    if edge_score:
        d.edge_score, d.hub_threshold = 0x1000, hub_threshold
    if n_roots_big:
        d.n_node, d.n_roots = 1 << 20, 1 << 11
    p = {k: (None if k in null else C.c_void_p(0x1000)) for k in ("dist", "p_void", "root_ok", "scratch")}
    return lib.gg_generator_dist_d(C.byref(d) if desc else None, p["dist"], p["p_void"], p["root_ok"], p["scratch"],
                                   scratch_bytes, None)


@pytest.mark.parametrize("bad", [
    dict(desc=False), dict(ld=48), dict(ld=1024), dict(ld=0), dict(n_node=0), dict(tree_words=0), dict(scratch_bytes=8),
    dict(n_roots_big=True), dict(edge_score=True, hub_threshold=0), dict(edge_score=True, hub_threshold=1 << 20),
    dict(null=("emb",)), dict(null=("bias",)), dict(null=("indptr",)), dict(null=("adj",)), dict(null=("roots",)),
    dict(null=("tree_bits",)), dict(null=("dist",)), dict(null=("p_void",)), dict(null=("root_ok",)),
    dict(null=("scratch",)),
])
def test_law_entry_point_refuses_bad_arguments(bad):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rc = _call_law(lib, **bad)
    assert rc != 0
    with pytest.raises(_cabi.GGError):
        _cabi.check(rc, "gg_generator_dist_d")


def _call_grad(lib, ld=64, n_node=100, n_roots=2, null=(), scratch_bytes=1 << 40):
    names = ("emb", "bias", "raw_indptr", "raw_adj", "roots", "dist", "p_void", "root_ok", "accept", "grad_emb",
             "grad_bias", "scratch")
    p = {k: (None if k in null else C.c_void_p(0x1000)) for k in names}
    return lib.gg_expected_d_grad(n_node, ld, p["emb"], p["bias"], p["raw_indptr"], p["raw_adj"], n_roots, p["roots"],
                                  p["dist"], p["p_void"], p["root_ok"], p["accept"], p["grad_emb"], p["grad_bias"],
                                  p["scratch"], scratch_bytes, None)


@pytest.mark.parametrize("bad", [
    dict(ld=48), dict(ld=1024), dict(ld=0), dict(n_node=0), dict(n_node=1 << 31), dict(n_roots=-1), dict(scratch_bytes=8),
    dict(null=("emb",)), dict(null=("bias",)), dict(null=("raw_indptr",)), dict(null=("raw_adj",)), dict(null=("roots",)),
    dict(null=("dist",)), dict(null=("p_void",)), dict(null=("root_ok",)), dict(null=("accept",)),
    dict(null=("grad_emb",)), dict(null=("grad_bias",)), dict(null=("scratch",)),
])
def test_step_entry_point_refuses_bad_arguments(bad):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rc = _call_grad(lib, **bad)
    assert rc != 0
    with pytest.raises(_cabi.GGError):
        _cabi.check(rc, "gg_expected_d_grad")


@pytest.mark.parametrize("ld", [32, 128, 512])
def test_scratch_size_and_empty_batch(ld):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    n, one, two, g1, g2 = (C.c_int64(-1) for _ in range(5))
    assert lib.gg_expected_d_grad_scratch_bytes(5000, ld, 1, C.byref(one)) == 0
    assert lib.gg_expected_d_grad_scratch_bytes(5000, ld, 2, C.byref(two)) == 0
    assert lib.gg_game_value_grad_d_scratch_bytes(5000, ld, 1, C.byref(g1)) == 0
    assert lib.gg_game_value_grad_d_scratch_bytes(5000, ld, 2, C.byref(g2)) == 0
    # section 5.4's layout plus ok_ref, 4 bytes per root (each region rounded up to 256 bytes)
    assert 0 < two.value - g2.value <= 256 and 0 < one.value - g1.value <= 256
    assert abs((two.value - one.value) - (g2.value - g1.value)) <= 256
    assert lib.gg_expected_d_grad_scratch_bytes(-1, ld, 3, C.byref(n)) != 0
    assert lib.gg_expected_d_grad_scratch_bytes(10, ld, -3, C.byref(n)) != 0
    assert lib.gg_expected_d_grad_scratch_bytes(10, 48, 3, C.byref(n)) != 0
    assert lib.gg_expected_d_grad_scratch_bytes(10, ld, 3, None) != 0
    # no roots: nothing to do, no pointer is looked at
    assert _call_grad(lib, n_roots=0, null=("emb", "dist", "accept", "grad_emb", "scratch"), scratch_bytes=0) == 0
    assert _call_law(lib, n_roots=0, null=("emb", "dist", "p_void", "scratch"), scratch_bytes=0) == 0
