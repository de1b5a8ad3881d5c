"""The best-response value's host reference (tests/best_response_oracle.py) and the argument checks of gg_best_response /
gg_best_response_grad / gg_best_response_spmm.  No GPU.

- At the depth-1 nodes the oracle's G is gdist_oracle.distribution's, bit for bit.
- vstar_c = max_D V_c(G, D): it equals V_c at D* = p / (p + G), exceeds V_c at random D, and lies in [-log 4, 0].
- The "smooth" law's gradient is the derivative of its own vstar with D* recomputed at every point (envelope theorem and
  assembly): central finite differences along random directions, on the fixtures and on a hand-built graph.
- The "pi" law's gradient is within the step-law bound of DESIGN.md section 5.3 of the smooth one.
"""
import ctypes as C

import numpy as np
import pytest

from tests import best_response_oracle as bro
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
    bits = np.zeros((len(hg.adj) + 31) // 32 + 1, np.uint32)
    if removal:
        can.walk_pass(E_g, b_g, hg.indptr, hg.adj, roots, par, hg.degrees()[roots], True, bits, seed=5, pass_tag=1)
        assert bits.any()
    return hg, roots, par, bits, E_g, b_g


def _hand_graph():
    """a root with duplicate raw entries, a self-loop, depth-1 leaves and a deeper subtree"""
    from graphgan_b200 import graph as G
    edges = [(0, 1), (0, 2), (0, 3), (0, 1), (0, 0), (1, 4), (1, 5), (4, 6), (2, 7), (7, 8), (5, 8), (3, 0), (8, 9),
             (10, 10), (11, 12), (0, 13), (13, 14)]
    return G.HostGraph(np.asarray(edges), None, n_node=15)


def _dim(E):
    nz = np.flatnonzero(np.abs(E).sum(axis=0))
    return int(nz[-1]) + 1 if len(nz) else E.shape[1]


@pytest.mark.parametrize("removal", [False, True])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_depth1_law_is_the_distribution_and_vstar_is_the_max_over_d(name, removal):
    hg, roots, par, bits, E_g, b_g = _setup(name, removal)
    rs = np.random.RandomState(11)
    n_ok = 0
    for k, r in enumerate(roots):
        o = bro.root_value(E_g, b_g, hg, int(r), par[k], bits)
        dist, ok = go.distribution(E_g, b_g, hg.indptr, hg.adj, int(r), par[k], bits)
        assert o["ok"] == ok
        if not o["ok"]:
            continue
        n_ok += 1
        for a, g in o["G"].items():
            assert g == dist[a]                                # bit for bit
        assert -np.log(4.0) - 1e-15 <= o["vstar"] <= 1e-15
        assert abs(o["hit"] - sum(o["G"].values())) <= 1e-15
        p_raw = bro.raw_law(hg, int(r))
        nodes = set(p_raw) | set(o["G"])
        dstar = {v: (p_raw.get(v, 0.0) / (p_raw.get(v, 0.0) + o["G"].get(v, 0.0))) for v in nodes}
        dstar = {v: min(max(x, 1e-300), 1.0 - 1e-16) if p_raw.get(v, 0.0) and o["G"].get(v, 0.0) else x
                 for v, x in dstar.items()}
        v_star = sum(m * np.log(dstar[v]) for v, m in p_raw.items() if dstar[v] > 0) + sum(
            g * np.log1p(-dstar[v]) for v, g in o["G"].items() if g > 0)
        assert abs(v_star - o["vstar"]) <= 1e-13
        for _ in range(20):
            Dv = {v: rs.uniform(0.01, 0.99) for v in nodes}
            assert bro.value_at(o["G"], p_raw, Dv) <= o["vstar"] + 1e-14
    assert n_ok


def _vstar_smooth(E, b, hg, roots, par, bits):
    mult = bro.entry_mult(hg)
    return sum(bro.root_value(E, b, hg, int(r), par[k], bits, "smooth", mult)["vstar"] for k, r in enumerate(roots))


def _fd_check(hg, roots, par, bits, E_g, b_g, seed=3):
    E, b = E_g.astype(np.float64), b_g.astype(np.float64)
    gE, gb, _, _, per = bro.grad(E, b, hg, roots, par, bits, "smooth")
    assert any(o["ok"] for o in per)
    d = _dim(E_g)
    rs = np.random.RandomState(seed)
    eps = 1e-6
    for _ in range(4):
        dE = np.zeros_like(E)
        dE[:, :d] = rs.normal(0, 1, (hg.n_node, d))
        db = rs.normal(0, 1, hg.n_node)
        fd = (_vstar_smooth(E + eps * dE, b + eps * db, hg, roots, par, bits)
              - _vstar_smooth(E - eps * dE, b - eps * db, hg, roots, par, bits)) / (2 * eps)
        an = float((gE * dE).sum() + (gb * db).sum())
        scale = float(np.abs(gE * dE).sum() + np.abs(gb * db).sum())
        assert abs(fd - an) <= 1e-6 * scale, (fd, an, scale)
    return per


@pytest.mark.parametrize("removal", [False, True])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_smooth_gradient_matches_finite_differences(name, removal):
    hg, roots, par, bits, E_g, b_g = _setup(name, removal)
    _fd_check(hg, roots, par, bits, E_g, b_g)


def test_smooth_gradient_on_a_hand_built_graph():
    """duplicate raw entries (0 -> 1 twice), a self-loop (0, 0), depth-1 leaves (3, 13 has a child), a removed depth-1 leaf"""
    from oracle import canonical as can
    hg = _hand_graph()
    roots = np.array([0, 1, 10, 11], np.int32)
    par = can.bfs_parents(hg.indptr, hg.adj, roots)
    rs = np.random.RandomState(5)
    E_g = can.pad_rows(rs.normal(0, 0.4, (hg.n_node, 8)).astype(np.float32))
    b_g = rs.normal(0, 0.2, hg.n_node).astype(np.float32)
    bits = np.zeros((len(hg.adj) + 31) // 32 + 1, np.uint32)
    e = next(e for e in range(hg.indptr[0], hg.indptr[1]) if hg.adj[e] == 13)   # 13 keeps its child 14: no void
    bits[e >> 5] |= np.uint32(1 << (e & 31))
    per = _fd_check(hg, roots, par, bits, E_g, b_g)
    assert per[0]["ok"] == 1 and per[0]["G"][13] == 0.0        # removed father: no stop at 13
    assert per[2]["ok"] == 0                                    # self-loop only
    o = bro.root_value(E_g, b_g, hg, 0, par[0], bits)
    assert o["p"][1] == 2 / 8 and o["p"][3] == 2 / 8 and o["p"][2] == 1 / 8   # graph[0] = [1, 2, 3, 1, 0, 0, 3, 13]
    # a removed depth-1 leaf voids the root (section 5.1): 3 is a leaf of 0's tree
    e3 = next(e for e in range(hg.indptr[0], hg.indptr[1]) if hg.adj[e] == 3)
    bits2 = bits.copy()
    bits2[e3 >> 5] |= np.uint32(1 << (e3 & 31))
    o2 = bro.root_value(E_g, b_g, hg, 0, par[0], bits2)
    assert o2["ok"] == 0 and o2["vstar"] == 0.0


@pytest.mark.parametrize("removal", [False, True])
@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_pi_gradient_is_within_the_step_law_bound_of_the_smooth_one(name, removal):
    """|grad_pi - grad_smooth| <= 4 (D + 2) delta A per coordinate (DESIGN.md section 5.3) with D = 1: every term is a
    product of at most three step probabilities and one log."""
    hg, roots, par, bits, E_g, b_g = _setup(name, removal)
    mult = bro.entry_mult(hg)
    for k, r in enumerate(roots):
        a = bro.root_value(E_g, b_g, hg, int(r), par[k], bits, "pi", mult)
        s = bro.root_value(E_g, b_g, hg, int(r), par[k], bits, "smooth", mult)
        assert a["ok"] == s["ok"]
        if not a["ok"]:
            continue
        live = (a["w"] != 0) & (s["pi"] > 0)
        delta = float(np.max(np.abs(a["pi"] - s["pi"])[live] / s["pi"][live])) if live.any() else 0.0
        assert delta < 1e-5, delta
        bound = 4 * 3 * delta + 1e-12
        assert np.all(np.abs(a["gE"] - s["gE"]) <= bound * (a["abs_E"] + s["abs_E"]) + 1e-300), int(r)
        assert np.all(np.abs(a["gb"] - s["gb"]) <= bound * (a["abs_b"] + s["abs_b"]) + 1e-300), int(r)


# ---------------------------------------------------------------------------------------------- C ABI (no device work)
def _call(lib, which="value", desc=True, ld=64, n_node=100, n_roots=2, null=(), scratch_bytes=1 << 40, tree_words=8,
          n_roots_big=False, hub=None):
    from graphgan_b200 import _cabi
    d = _cabi.WalkDesc()
    d.n_node, d.ld, d.n_roots, d.tree_words = n_node, ld, n_roots, tree_words
    for f in ("emb", "bias", "indptr", "adj", "roots", "tree_bits"):
        setattr(d, f, None if f in null else 0x1000)
    if hub is not None:
        d.edge_score, d.hub_threshold = 0x1000, hub
    if n_roots_big:
        d.n_node, d.n_roots = 1 << 20, 1 << 11
    p = {k: (None if k in null else C.c_void_p(0x1000)) for k in
         ("raw_indptr", "mult", "rev", "vstar", "hit", "ok", "acc_coef", "acc_bias", "scratch")}
    dp = C.byref(d) if desc else None
    if which == "value":
        return lib.gg_best_response(dp, p["raw_indptr"], p["mult"], p["vstar"], p["hit"], p["ok"], p["scratch"],
                                    scratch_bytes, None)
    return lib.gg_best_response_grad(dp, p["raw_indptr"], p["mult"], p["rev"], p["vstar"], p["hit"], p["ok"], p["acc_coef"],
                                     p["acc_bias"], p["scratch"], scratch_bytes, None)


_BAD = [
    dict(desc=False), dict(ld=48), dict(ld=1024), dict(ld=0), dict(n_node=0), dict(n_roots=-1), dict(tree_words=0),
    dict(scratch_bytes=8), dict(n_roots_big=True), dict(hub=0), dict(hub=4096),
    dict(null=("emb",)), dict(null=("bias",)), dict(null=("indptr",)), dict(null=("adj",)), dict(null=("roots",)),
    dict(null=("tree_bits",)), dict(null=("raw_indptr",)), dict(null=("mult",)), dict(null=("vstar",)),
    dict(null=("hit",)), dict(null=("ok",)), dict(null=("scratch",)),
]


@pytest.mark.parametrize("bad", _BAD)
def test_value_entry_point_refuses_bad_arguments(bad):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rc = _call(lib, "value", **bad)
    assert rc != 0
    with pytest.raises(_cabi.GGError):
        _cabi.check(rc, "gg_best_response")


@pytest.mark.parametrize("bad", _BAD + [dict(null=("rev",)), dict(null=("acc_coef",)), dict(null=("acc_bias",))])
def test_grad_entry_point_refuses_bad_arguments(bad):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rc = _call(lib, "grad", **bad)
    assert rc != 0
    with pytest.raises(_cabi.GGError):
        _cabi.check(rc, "gg_best_response_grad")


@pytest.mark.parametrize("bad", [dict(ld=48), dict(n_node=-1), dict(null="indptr"), dict(null="adj"), dict(null="emb"),
                                 dict(null="acc_coef"), dict(null="acc_bias"), dict(null="grad_emb"),
                                 dict(null="grad_bias")])
def test_spmm_refuses_bad_arguments(bad):
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    args = {k: C.c_void_p(0x1000) for k in ("indptr", "adj", "emb", "acc_coef", "acc_bias", "grad_emb", "grad_bias")}
    if "null" in bad:
        args[bad["null"]] = None
    rc = lib.gg_best_response_spmm(bad.get("n_node", 10), bad.get("ld", 64), args["indptr"], args["adj"], args["emb"],
                                   args["acc_coef"], args["acc_bias"], args["grad_emb"], args["grad_bias"], None)
    assert rc != 0


def test_scratch_sizes_and_empty_batch():
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    assert _cabi.ABI_VERSION == 11 and lib.gg_abi_version() == 11
    sz = {}
    for fn in ("gg_best_response_scratch_bytes", "gg_best_response_grad_scratch_bytes", "gg_generator_dist_scratch_bytes"):
        for k in (1, 2):
            n = C.c_int64(-1)
            assert getattr(lib, fn)(1000, 20000, k, C.byref(n)) == 0
            sz[fn, k] = n.value
        n = C.c_int64(-1)
        assert getattr(lib, fn)(-1, 3, 3, C.byref(n)) != 0
        assert getattr(lib, fn)(10, -3, 3, C.byref(n)) != 0
        assert getattr(lib, fn)(10, 3, -3, C.byref(n)) != 0
        assert getattr(lib, fn)(10, 3, 3, None) != 0
    per = {fn: sz[fn, 2] - sz[fn, 1] for fn in ("gg_best_response_scratch_bytes", "gg_best_response_grad_scratch_bytes",
                                                "gg_generator_dist_scratch_bytes")}
    # value: the section 5.1 list pools, one item list (16 bytes per node) and pi_c, G, h*, p log1p(G / p) (32 bytes per node)
    assert abs(per["gg_best_response_scratch_bytes"] - (per["gg_generator_dist_scratch_bytes"] + 16 * 1000)) <= 6 * 256
    # gradient: w_a(c), pi_a(x) and the unit offsets, 20 bytes per node more
    assert abs(per["gg_best_response_grad_scratch_bytes"] - per["gg_best_response_scratch_bytes"] - 20 * 1000) <= 6 * 256
    # no roots: nothing to do, no pointer is looked at
    assert _call(lib, "value", n_roots=0, null=("emb", "vstar", "scratch", "mult"), scratch_bytes=0) == 0
    assert _call(lib, "grad", n_roots=0, null=("emb", "vstar", "scratch", "rev", "acc_coef"), scratch_bytes=0) == 0
    assert lib.gg_best_response_spmm(0, 64, None, None, None, None, None, None, None, None) == 0


def test_library_without_the_new_symbols_is_refused():
    from graphgan_b200 import _cabi
    for name in ("gg_best_response_scratch_bytes", "gg_best_response", "gg_best_response_grad_scratch_bytes",
                 "gg_best_response_grad", "gg_best_response_spmm"):
        assert name in _cabi.SIGNATURES
