"""The host reference of the second moment of one G walk's step (tests/expected_g_moments_oracle.py) and the argument
checks of gg_expected_g_moments.  No GPU.

- The literal oracle's m_c is root_expect's expected step; its sq_c is the walk-by-walk sum over every G walk of the
  root (prob * |s(walk)|^2, s built from the walk's own body pairs); an exactly enumerated two-walk pass has
  E|S|^2 = 2 sq_c + 2 mn_c.
- The Pf + tail decomposition (the device's order of work) gives the literal |s(y)|^2 per node.
- var_c = sq_c - mn_c is >= 0 up to rounding, and 0 for a root whose walk law is a point mass.
"""
import ctypes as C

import numpy as np
import pytest

from tests import expected_g_grad_oracle as eo
from tests import expected_g_moments_oracle as mo
from tests import update_bits_oracle as ub
from tests.test_expected_g_grad_host import _setup


def _roots(name, removal, window):
    hg, roots, par, bits, E_g, b_g, E_d, b_d = _setup(name, removal)
    reward = eo.numpy_reward(E_d, b_d)
    for k, r in enumerate(roots):
        o = mo.root_pairs(E_g, b_g, hg, int(r), par[k], bits, window, reward)
        if o["ok"]:
            yield hg, int(r), par[k], E_g, b_g, reward, o


def _walks(hg, root, parent, dist):
    """every G walk of an ok root by brute force: (probability, recorded path root -> v -> father(v))"""
    for v in np.flatnonzero(dist > 0):
        path = [int(v)]
        while path[-1] != root:
            path.append(int(parent[path[-1]]))
        yield dist[v], path[::-1] + [int(parent[v])]


def _walk_step(E_g, b_g, reward, path, window):
    """s(walk) with each pair's kappa computed on its own (pair_delta mode 1, batch_total 1): dense (rows, bias)"""
    Eg, bg = np.ascontiguousarray(E_g, np.float32), np.asarray(b_g, np.float32)
    pairs = eo.body_pairs(path, window)
    n1 = np.array([p[0] for p in pairs], np.int64)
    n2 = np.array([p[1] for p in pairs], np.int64)
    k, _ = ub.delta(1, ub.score(Eg, bg, n1, n2), reward(n1, n2), 1)
    E = Eg.astype(np.float64)
    rows, bias = np.zeros_like(E), np.zeros(E.shape[0])
    for a, b, kk in zip(n1.tolist(), n2.tolist(), k.astype(np.float64).tolist()):
        rows[a] += kk * E[b]
        rows[b] += kk * E[a]
        bias[b] += kk
    return rows, bias


@pytest.mark.parametrize("window", [1, 2, 3])
@pytest.mark.parametrize("removal", [False, True])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_literal_oracle_against_enumerated_walks(name, removal, window):
    n_ok = 0
    for hg, r, parent, E_g, b_g, reward, o in _roots(name, removal, window):
        n_ok += 1
        lit = mo.literal_root(E_g, o, window)
        # m_c is the section 5.6 expectation of this root
        assert np.all(np.abs(lit["mE"] - o["gE"]) <= 1e-13 * o["abs_E"])
        assert np.all(np.abs(lit["mb"] - o["gb"]) <= 1e-13 * o["abs_b"])
        # walk by walk
        walks = list(_walks(hg, r, parent, o["dist"]))
        steps = [_walk_step(E_g, b_g, reward, path, window) for _, path in walks]
        prob = np.array([p for p, _ in walks])
        sq_w = np.array([float((R * R).sum() + (B * B).sum()) for R, B in steps])
        assert abs(float((prob * sq_w).sum()) - lit["sq"]) <= 1e-12 * lit["sq"]
        # an exactly enumerated pass of two walks
        S = np.stack([np.concatenate([R.ravel(), B]) for R, B in steps])
        G = S @ S.T
        d = np.diag(G)
        e2 = float(prob @ (d[:, None] + d[None, :] + 2 * G) @ prob)
        want = 2 * lit["sq"] + 2 * lit["mn"]
        assert abs(e2 - want) <= 1e-12 * want, (e2, want)
        # and the variance is a variance
        assert lit["sq"] - lit["mn"] >= -1e-12 * lit["sq"]
    assert n_ok


@pytest.mark.parametrize("window", [1, 2, 3])
@pytest.mark.parametrize("removal", [False, True])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_pf_tail_is_the_literal_norm(name, removal, window):
    for hg, r, parent, E_g, b_g, reward, o in _roots(name, removal, window):
        lit = mo.literal_root(E_g, o, window)
        pt = mo.pf_tail(E_g, o, window)
        want = lit["sq_node"]
        assert np.all(np.abs(pt["sq_node"] - want) <= 1e-13 * want), np.max(np.abs(pt["sq_node"] - want) / np.maximum(want, 1e-300))
        assert np.all(pt["abs_sq"] >= pt["sq_node"] * (1 - 1e-12))
        assert not pt["sq_node"][o["depth"] == 0].any()
        # a node at depth < w has no complete row; below that Pf only grows
        assert not pt["pf"][(o["depth"] > 0) & (o["depth"] < window)].any()
        ys = np.flatnonzero(o["depth"] > 1)
        assert np.all(pt["pf"][ys] >= pt["pf"][o["father"][ys]])
        # the same norms from the paths alone
        ys = np.flatnonzero(o["depth"] > 0)
        sq, ab, _ = mo.path_sq(E_g, b_g, parent, ys, window, reward)
        assert np.all(np.abs(sq - want[ys]) <= 1e-13 * ab) and np.all(ab >= sq * (1 - 1e-12))


def test_point_mass_root_has_no_variance():
    """root 0 with the one neighbour 1, itself a leaf: every walk goes 0 -> 1 and stops; var_c is rounding only"""
    from graphgan_b200 import graph as G
    from oracle import canonical as can
    edges = np.array([[0, 1], [2, 3], [3, 4], [2, 4]])
    hg = G.HostGraph(edges, None, n_node=5)
    rs = np.random.RandomState(3)
    E_g = can.pad_rows(rs.normal(0, 0.3, (5, 12)).astype(np.float32))
    b_g = rs.normal(0, 0.2, 5).astype(np.float32)
    E_d = can.pad_rows(rs.normal(0, 0.3, (5, 12)).astype(np.float32))
    b_d = rs.normal(0, 0.3, 5).astype(np.float32)
    par = can.bfs_parents(hg.indptr, hg.adj, np.array([0], np.int32))
    bits = np.zeros((len(hg.adj) + 31) // 32 + 1, np.uint32)
    for w in (1, 2):
        o = mo.root_pairs(E_g, b_g, hg, 0, par[0], bits, w, eo.numpy_reward(E_d, b_d))
        assert o["ok"] and o["dist"][1] == 1.0
        lit = mo.literal_root(E_g, o, w)
        assert lit["sq"] > 0 and abs(lit["sq"] - lit["mn"]) <= 1e-13 * lit["sq"]


def test_entry_points_are_an_addition_to_abi_11():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    assert _cabi.ABI_VERSION == 11 and lib.gg_abi_version() == 11
    for name in ("gg_expected_g_moments_scratch_bytes", "gg_expected_g_moments"):
        assert name in _cabi.SIGNATURES and getattr(lib, name).argtypes == _cabi.SIGNATURES[name][1]


def _call(lib, desc=True, ld=64, n_node=100, n_roots=2, null=(), scratch_bytes=1 << 40, tree_words=8, n_roots_big=False,
          window=2, edge_score=False, hub_threshold=128):
    from graphgan_b200 import _cabi
    d = _cabi.WalkDesc()
    d.n_node, d.ld, d.n_roots, d.tree_words = n_node, ld, n_roots, tree_words
    for f in ("emb", "bias", "indptr", "adj", "roots", "tree_bits"):
        setattr(d, f, None if f in null else 0x1000)
    if edge_score:
        d.edge_score, d.hub_threshold = 0x1000, hub_threshold
    if n_roots_big:
        d.n_node, d.n_roots = 1 << 20, 1 << 11
    p = {k: (None if k in null else C.c_void_p(0x1000)) for k in
         ("d_emb", "d_bias", "n_pairs", "ok", "sq", "mn", "sq_node", "grad_emb", "grad_bias", "scratch")}
    return lib.gg_expected_g_moments(C.byref(d) if desc else None, p["d_emb"], p["d_bias"], window, p["n_pairs"], p["ok"],
                                     p["sq"], p["mn"], p["sq_node"], p["grad_emb"], p["grad_bias"], p["scratch"],
                                     scratch_bytes, None)


@pytest.mark.parametrize("bad", [
    dict(desc=False), dict(ld=48), dict(ld=1024), dict(ld=0), dict(n_node=0), dict(n_roots=-1), dict(tree_words=0),
    dict(scratch_bytes=8), dict(n_roots_big=True), dict(window=0), dict(window=9), dict(window=-2),
    dict(edge_score=True, hub_threshold=0), dict(edge_score=True, hub_threshold=1 << 20),
    dict(null=("emb",)), dict(null=("bias",)), dict(null=("indptr",)), dict(null=("adj",)), dict(null=("roots",)),
    dict(null=("tree_bits",)), dict(null=("d_emb",)), dict(null=("d_bias",)), dict(null=("n_pairs",)), dict(null=("ok",)),
    dict(null=("sq",)), dict(null=("mn",)), dict(null=("grad_emb",)), dict(null=("grad_bias",)), dict(null=("scratch",)),
])
def test_entry_point_refuses_bad_arguments(bad):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rc = _call(lib, **bad)
    assert rc != 0
    with pytest.raises(_cabi.GGError):
        _cabi.check(rc, "gg_expected_g_moments")


def test_scratch_bytes_short_of_the_moments_planes_are_refused():
    """gg_expected_g_grad's scratch is not enough: the moments need their two planes"""
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    nb = C.c_int64(-1)
    assert lib.gg_expected_g_grad_scratch_bytes(100, 64 * 32, 2, 2, C.byref(nb)) == 0
    assert _call(lib, scratch_bytes=nb.value) != 0


@pytest.mark.parametrize("window", [1, 2, 8])
def test_scratch_size_and_empty_batch(window):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    n = C.c_int64(-1)
    got, ref = {}, {}
    for k in (0, 1, 2):
        a, b = C.c_int64(-1), C.c_int64(-1)
        assert lib.gg_expected_g_moments_scratch_bytes(1000, 20000, k, window, C.byref(a)) == 0
        assert lib.gg_expected_g_grad_scratch_bytes(1000, 20000, k, window, C.byref(b)) == 0
        got[k], ref[k] = a.value, b.value
    # gg_expected_g_grad's scratch and two fp64 planes per (root, node)
    assert ref[0] <= got[0] <= ref[0] + 2 * 256
    for k in (1, 2):
        assert abs(got[k] - ref[k] - 16 * 1000 * k) <= 2 * 256
    assert lib.gg_expected_g_moments_scratch_bytes(-1, 3, 3, window, C.byref(n)) != 0
    assert lib.gg_expected_g_moments_scratch_bytes(10, -3, 3, window, C.byref(n)) != 0
    assert lib.gg_expected_g_moments_scratch_bytes(10, 3, -3, window, C.byref(n)) != 0
    assert lib.gg_expected_g_moments_scratch_bytes(10, 3, 3, window, None) != 0
    assert lib.gg_expected_g_moments_scratch_bytes(10, 3, 3, 0, C.byref(n)) != 0
    assert lib.gg_expected_g_moments_scratch_bytes(10, 3, 3, 9, C.byref(n)) != 0
    # no roots: nothing to do, no pointer is looked at
    assert _call(lib, n_roots=0, null=("emb", "d_emb", "n_pairs", "sq", "mn", "grad_emb", "scratch"), scratch_bytes=0) == 0


def test_sampler_refuses_windows_outside_1_to_8():
    from graphgan_b200.sampler import WalkSampler
    for w in (0, 9):
        with pytest.raises(ValueError):
            WalkSampler.expected_g_moments(None, None, None, None, None, None, window=w)
