"""The host reference of the expected reference G step (tests/expected_g_grad_oracle.py) and the argument checks of
gg_expected_g_grad.  No GPU.

- Brute force: every G walk of a root with its probability, its body's window pairs counted as get_node_pairs_from_path
  does; the expected count of each ordered pair is the reach-weight formula of DESIGN.md section 5.6, and their sum n_pairs.
- The row and bias assembly is the derivative of sum rho l(pair), l = -r log sigmoid(s_G), with the weights and rewards
  held fixed: central finite differences.
- The oracle's reach is the section 5.1 chain: dist == reach * pi_stop bit for bit at every reached node that can stop.
"""
import ctypes as C

import numpy as np
import pytest

from tests import expected_g_grad_oracle as eo
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


@pytest.mark.parametrize("window", [1, 2, 3])
@pytest.mark.parametrize("removal", [False, True])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_pair_counts_match_brute_force_walks(name, removal, window):
    hg, roots, par, bits, E_g, b_g, E_d, b_d = _setup(name, removal)
    n_ok = 0
    for k, r in enumerate(roots):
        ok, reach, father, depth, dist, _ = eo.tree_reach(E_g, b_g, hg, int(r), par[k], bits)
        if not ok:
            continue
        n_ok += 1
        counts, total = eo.enumerate_walks(hg, int(r), par[k], dist, window)
        X, Y, rho = eo.window_pairs(reach, father, depth, window)
        want = {}
        for x, y, p in zip(X.tolist(), Y.tolist(), rho.tolist()):
            for key in ((x, y), (y, x)):
                want[key] = want.get(key, 0.0) + p
        assert set(k_ for k_, v in counts.items() if v > 0) == set(want)
        for key, v in want.items():
            assert abs(counts[key] - v) <= 1e-12 * v, (key, counts[key], v)
        n_pairs = float((reach * 2 * np.minimum(depth, window)).sum())
        assert abs(total - n_pairs) <= 1e-12 * n_pairs
        assert abs(sum(want.values()) - n_pairs) <= 1e-12 * n_pairs
        o = eo.root_expect(E_g, b_g, hg, int(r), par[k], bits, window, eo.numpy_reward(E_d, b_d))
        assert o["n_pairs"] == n_pairs
    assert n_ok


@pytest.mark.parametrize("removal", [False, True])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_reach_is_the_law_chain(name, removal):
    hg, roots, par, bits, E_g, b_g, E_d, b_d = _setup(name, removal)
    for k, r in enumerate(roots):
        ok, reach, father, depth, dist, rec = eo.tree_reach(E_g, b_g, hg, int(r), par[k], bits)
        if not ok:
            continue
        fr = np.flatnonzero(rec["is_father"])
        a = rec["owner"][fr]
        live = reach[a] > 0
        assert np.array_equal(dist[a[live]], reach[a[live]] * rec["pi"][fr][live])      # fp64 products, bit for bit
        assert np.all((dist > 0) <= (reach > 0))


def _loss(E, b, X, Y, rho, r_up, r_dn):
    """sum rho l(pair) in fp64, l(n1, n2) = -r log sigmoid(E[n1] . E[n2] + b[n2])"""
    tot = 0.0
    for n1, n2, r in ((X, Y, r_up), (Y, X, r_dn)):
        s = np.einsum("ij,ij->i", E[n1], E[n2]) + b[n2]
        tot += float((rho * r * np.logaddexp(0.0, -s)).sum())
    return tot


@pytest.mark.parametrize("window", [1, 2, 3])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_assembly_matches_finite_differences(name, window):
    hg, roots, par, bits, E_g, b_g, E_d, b_d = _setup(name, True)
    reward = eo.numpy_reward(E_d, b_d)
    E, b = E_g.astype(np.float64), b_g.astype(np.float64)
    rs = np.random.RandomState(7)
    d = int(np.flatnonzero(np.abs(E).sum(axis=0))[-1]) + 1
    for k, r in enumerate(roots):
        ok, reach, father, depth, _, _ = eo.tree_reach(E_g, b_g, hg, int(r), par[k], bits)
        if not ok:
            continue
        X, Y, rho = eo.window_pairs(reach, father, depth, window)
        r_up, r_dn = reward(X, Y).astype(np.float64), reward(Y, X).astype(np.float64)
        sig = lambda s: 1.0 / (1.0 + np.exp(-s))
        k_up = -r_up * (1 - sig(np.einsum("ij,ij->i", E[X], E[Y]) + b[Y]))      # fp64 kappa: the clip inactive
        k_dn = -r_dn * (1 - sig(np.einsum("ij,ij->i", E[Y], E[X]) + b[X]))
        gE, gb, _, _ = eo.assemble(E, X, Y, rho, k_up, k_dn)
        eps = 1e-6
        for _ in range(3):
            dE = np.zeros_like(E)
            dE[:, :d] = rs.normal(0, 1, (hg.n_node, d))
            db = rs.normal(0, 1, hg.n_node)
            fd = (_loss(E + eps * dE, b + eps * db, X, Y, rho, r_up, r_dn)
                  - _loss(E - eps * dE, b - eps * db, X, Y, rho, r_up, r_dn)) / (2 * eps)
            an = float((gE * dE).sum() + (gb * db).sum())
            scale = float(np.abs(gE * dE).sum() + np.abs(gb * db).sum())
            assert abs(fd - an) <= 1e-6 * scale, (fd, an, scale)


def test_void_roots_add_nothing_in_the_oracle():
    hg, roots, par, bits, E_g, b_g, E_d, b_d = _setup("rand300", True, k=20)
    for k, r in enumerate(roots):
        o = eo.root_expect(E_g, b_g, hg, int(r), par[k], bits, 2, eo.numpy_reward(E_d, b_d))
        if not o["ok"]:
            assert o["n_pairs"] == 0.0 and not o["gE"].any() and not o["gb"].any()


def test_entry_points_are_an_addition_to_abi_11():
    """The new entry points extend ABI 11 without changing any existing one: the version stays, and the loader binds the
    new symbols (it refuses a library that does not export every declared symbol)."""
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    assert _cabi.ABI_VERSION == 11 and lib.gg_abi_version() == 11
    for name in ("gg_expected_g_grad_scratch_bytes", "gg_expected_g_grad"):
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
         ("d_emb", "d_bias", "n_pairs", "ok", "grad_emb", "grad_bias", "scratch")}
    return lib.gg_expected_g_grad(C.byref(d) if desc else None, p["d_emb"], p["d_bias"], window, p["n_pairs"], p["ok"],
                                  p["grad_emb"], p["grad_bias"], p["scratch"], scratch_bytes, None)


@pytest.mark.parametrize("bad", [
    dict(desc=False), dict(ld=48), dict(ld=1024), dict(ld=0), dict(n_node=0), dict(n_roots=-1), dict(tree_words=0),
    dict(scratch_bytes=8), dict(n_roots_big=True), dict(window=0), dict(window=9), dict(window=-2),
    dict(edge_score=True, hub_threshold=0), dict(edge_score=True, hub_threshold=1 << 20),
    dict(null=("emb",)), dict(null=("bias",)), dict(null=("indptr",)), dict(null=("adj",)), dict(null=("roots",)),
    dict(null=("tree_bits",)), dict(null=("d_emb",)), dict(null=("d_bias",)), dict(null=("n_pairs",)), dict(null=("ok",)),
    dict(null=("grad_emb",)), dict(null=("grad_bias",)), dict(null=("scratch",)),
])
def test_entry_point_refuses_bad_arguments(bad):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rc = _call(lib, **bad)
    assert rc != 0
    with pytest.raises(_cabi.GGError):
        _cabi.check(rc, "gg_expected_g_grad")


@pytest.mark.parametrize("window", [1, 2, 8])
def test_scratch_size_and_empty_batch(window):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    n, base, one, two = C.c_int64(-1), C.c_int64(-1), C.c_int64(-1), C.c_int64(-1)
    assert lib.gg_expected_g_grad_scratch_bytes(1000, 20000, 0, window, C.byref(base)) == 0
    assert lib.gg_expected_g_grad_scratch_bytes(1000, 20000, 1, window, C.byref(one)) == 0
    assert lib.gg_expected_g_grad_scratch_bytes(1000, 20000, 2, window, C.byref(two)) == 0
    per_root = two.value - one.value
    gd = C.c_int64(-1)
    assert lib.gg_generator_dist_scratch_bytes(1000, 20000, 1, C.byref(gd)) == 0 and lib.gg_generator_dist_scratch_bytes(
        1000, 20000, 2, C.byref(n)) == 0
    # per root: the section 5.1 scratch less one of its two item lists (16 bytes per node), then dist, reach, pi_in,
    # pi_stop, father and the two fp32 kappa planes per window distance
    assert abs(per_root - ((n.value - gd.value) - 16 * 1000 + (36 + 8 * window) * 1000)) <= 9 * 256 + 16
    assert base.value > 0
    assert lib.gg_expected_g_grad_scratch_bytes(-1, 3, 3, window, C.byref(n)) != 0
    assert lib.gg_expected_g_grad_scratch_bytes(10, -3, 3, window, C.byref(n)) != 0
    assert lib.gg_expected_g_grad_scratch_bytes(10, 3, -3, window, C.byref(n)) != 0
    assert lib.gg_expected_g_grad_scratch_bytes(10, 3, 3, window, None) != 0
    assert lib.gg_expected_g_grad_scratch_bytes(10, 3, 3, 0, C.byref(n)) != 0
    assert lib.gg_expected_g_grad_scratch_bytes(10, 3, 3, 9, C.byref(n)) != 0
    # no roots: nothing to do, no pointer is looked at
    assert _call(lib, n_roots=0, null=("emb", "d_emb", "n_pairs", "grad_emb", "scratch"), scratch_bytes=0) == 0


def test_sampler_refuses_windows_outside_1_to_8():
    from graphgan_b200.sampler import WalkSampler
    for w in (0, 9):
        with pytest.raises(ValueError):
            WalkSampler.expected_g_grad(None, None, None, None, None, None, window=w)
