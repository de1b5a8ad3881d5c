"""The exact generator distribution's host reference (tests/gdist_oracle.py) against the C oracle and a brute-force
enumeration of the reference's walk.  No GPU.

G(v | root) (DESIGN.md section 5.1) is built from the canonical q array of every candidate list; the step law
pi_j = (ceil(q_j 2^53) - ceil(q_{j-1} 2^53)) / 2^53 is exactly the set of 53-bit uniforms for which ggo_choose returns
j, which is checked here at both ends of every interval.
"""
import sys
from fractions import Fraction

import numpy as np
import pytest

from tests import gdist_oracle as go
from tests.golden import loader

FIXTURES = ["tiny", "rand300", "rand1200", "cagrqc"]


@pytest.mark.parametrize("ld", [32, 64, 128, 256, 512])
def test_vectorised_dot_is_the_canonical_dot(ld):
    from oracle import canonical as can
    rs = np.random.RandomState(ld)
    E = (rs.normal(0, 1, (64, ld)) * rs.choice([1e-3, 1.0, 30.0], (64, 1))).astype(np.float32)
    u, v = rs.randint(0, 64, 400), rs.randint(0, 64, 400)
    got = go.dots(E, u, v)
    want = np.array([can.dot_c(E[a], E[b]) for a, b in zip(u, v)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_vectorised_exp_is_the_canonical_exp():
    from oracle import canonical as can
    rs = np.random.RandomState(1)
    x = np.concatenate([-rs.exponential(3.0, 3000), -rs.uniform(0, 90, 2000), [0.0, -0.0, -86.0, -86.5, -1e-30, -85.99]])
    x = x.astype(np.float32)
    assert np.array_equal(go.exp_c(x).view(np.uint32), can.exp_c(x).view(np.uint32))


@pytest.mark.parametrize("n", [1, 2, 3, 31, 32, 33, 64, 97, 2100])
def test_step_law_is_the_set_of_uniforms_ggo_choose_maps_to_each_candidate(n):
    from oracle import canonical as can
    rs = np.random.RandomState(n)
    sc = (rs.normal(0, 3, n) + np.where(rs.rand(n) < 0.1, -120.0, 0.0)).astype(np.float32)   # some exp_c underflows
    q = go.list_q(sc, np.array([0, n]))
    k = go.step_pi_exact(q)
    pi = go.step_pi(q, np.array([0, n]))
    assert np.array_equal(pi, np.array(k, np.float64) / 2.0 ** 53)
    assert sum(k) == 2 ** 53
    js = range(n) if n <= 128 else rs.choice(n, 128, replace=False)
    lo = np.concatenate([[0], np.cumsum(k)[:-1]])
    for j in js:
        if k[j] == 0:
            continue
        for kk in (int(lo[j]), int(lo[j]) + k[j] - 1):      # first and last uniform of candidate j's interval
            assert can.choose(sc, kk / 2.0 ** 53) == j


def _case_graph(name):
    from graphgan_b200 import graph as G
    case = loader.load(name)
    hg = G.HostGraph(case["train_edges"], case["test_edges"], n_node=case.n)
    return case, hg


def _roots(hg, k, seed):
    n = hg.n_node
    return np.arange(n) if n <= k else np.sort(np.random.RandomState(seed).choice(n, k, replace=False))


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_distribution_sums_to_one(name):
    from oracle import canonical as can
    case, hg = _case_graph(name)
    roots = _roots(hg, 40, 2)
    par = can.bfs_parents(hg.indptr, hg.adj, roots)
    E = can.pad_rows(case.emb_g)
    bits = np.zeros((len(hg.adj) + 31) // 32 + 1, np.uint32)
    # a D pass sets father-removal bits; the G law reads them
    can.walk_pass(E, case.bias_g, hg.indptr, hg.adj, roots, par, hg.degrees()[roots], True, bits, seed=5, pass_tag=1)
    assert bits.any()
    for d1 in (np.zeros_like(bits), bits):
        n_ok = 0
        for k, r in enumerate(roots):
            dist, ok = go.distribution(E, case.bias_g, hg.indptr, hg.adj, int(r), par[k], d1)
            assert dist[r] == 0.0 and np.all(dist[par[k] < 0] == 0.0)
            if ok:
                n_ok += 1
                assert abs(dist.sum() - 1.0) <= 1e-12
            else:
                assert not dist.any()
        assert n_ok > 0


def _brute_force(E, bias, indptr, adj, root, parent, d1_bits):
    """Walk every tree path of GraphGAN.sample (graph_gan.py:225-270, for_d = False) from the root; per step the law of
    one draw from the canonical CDF, as exact rationals.  Returns {node: Fraction} or None when a walk can void."""
    from oracle import canonical as can
    bits = np.asarray(d1_bits).view(np.uint32)
    out = {}

    def children(a):
        return [(int(adj[e]), e) for e in range(indptr[a], indptr[a + 1]) if parent[adj[e]] == a]

    def law(cur, cands):
        sc = np.array([np.float32(can.dot_c(E[cur], E[c]) + np.float32(bias[c])) for c in cands], np.float32)
        return [Fraction(k, 2 ** 53) for k in go.step_pi_exact(go.list_q(sc, np.array([0, len(cands)])))]

    def visit(cur, prev, first_edge, p):
        if p == 0:
            return True
        ch = children(cur)
        inc_father = prev >= 0 and not (parent[cur] == root and (bits[first_edge >> 5] >> (first_edge & 31)) & 1)
        cands = ([prev] if inc_father else []) + [c for c, _ in ch]
        if not cands:
            return False                                       # graph_gan.py:252-257: the walk voids
        pis = law(cur, cands)
        if inc_father:
            out[cur] = out.get(cur, Fraction(0)) + p * pis[0]
            pis = pis[1:]
        for (c, e), pi in zip(ch, pis):
            if not visit(c, cur, e if prev < 0 else first_edge, p * pi):
                return False
        return True

    sys.setrecursionlimit(max(sys.getrecursionlimit(), 20000))
    return out if visit(root, -1, -1, Fraction(1)) else None


@pytest.mark.parametrize("name", ["tiny", "rand300"])
def test_oracle_distribution_equals_brute_force_enumeration(name):
    from oracle import canonical as can
    case, hg = _case_graph(name)
    roots = _roots(hg, 12, 3)
    par = can.bfs_parents(hg.indptr, hg.adj, roots)
    E = can.pad_rows(case.emb_g)
    bits = np.zeros((len(hg.adj) + 31) // 32 + 1, np.uint32)
    can.walk_pass(E, case.bias_g, hg.indptr, hg.adj, roots, par, hg.degrees()[roots], True, bits, seed=9, pass_tag=2)
    for d1 in (np.zeros_like(bits), bits):
        for k, r in enumerate(roots):
            dist, ok = go.distribution(E, case.bias_g, hg.indptr, hg.adj, int(r), par[k], d1)
            want = _brute_force(E, case.bias_g, hg.indptr, hg.adj, int(r), par[k], d1)
            assert ok == (want is not None and len(want) > 0)
            if not ok:
                continue
            exact = np.zeros(hg.n_node, np.float64)
            for v, p in want.items():
                exact[v] = float(p)
            assert np.array_equal(exact == 0, dist == 0)
            # each fp64 product rounds once: a depth-h chain is within (h + 1) 2^-53 of the exact rational
            assert np.all(np.abs(dist - exact) <= 64 * 2.0 ** -53 * exact)
            assert sum(want.values()) == 1
