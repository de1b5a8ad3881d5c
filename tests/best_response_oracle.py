"""TEST INFRASTRUCTURE ONLY: the game value against the best discriminator and its generator gradient on the host (DESIGN.md
section 5.8).

Per root c, over the lists of tests/gdist_oracle.candidate_lists with a step law pi, at the depth-1 nodes a (the
walk-CSR children of c, in entry order):
    G(a) = pi_c(a) pi_a(c) (0 when a's father entry is removed),  p(a) = n_ca / |graph[c]|
    h*(a) = G log1p(p / G),  vstar_c = -sum_a (p log1p(G / p) + h*(a)),  hit_c = sum_a G(a),  H_c = sum_a h*(a)
    w_c(a) = h*(a) - pi_c(a) H_c,  w_a(c) = h*(a) (1 - pi_a(c)),  w_a(x) = -pi_a(x) h*(a),  d vstar_c / d s(u, v) = -w_u(v)
Two laws, as tests/value_grad_oracle.py: "pi" (the kernel's; G is gdist_oracle.distribution's bits) and "smooth" (fp64
scores and softmax, differentiable, for finite differences).  vstar and hit follow the kernel's summation order (lane
chains over the root's entries, then a xor butterfly); the gradient is numpy's sums, compared relative to ``abs_*``.
"""
import numpy as np

from tests import gdist_oracle as go
from tests import value_grad_oracle as gro


def entry_mult(hg):
    """n_ca per walk-CSR entry (duplicates in the raw list counted)"""
    n = hg.n_node
    key_raw = np.repeat(np.arange(n, dtype=np.int64), np.diff(hg.raw_indptr)) * n + hg.raw_adj
    key = np.repeat(np.arange(n, dtype=np.int64), np.diff(hg.indptr)) * n + hg.adj
    u, cnt = np.unique(key_raw, return_counts=True)
    return cnt[np.searchsorted(u, key)].astype(np.int64)


def _lane_sum(vals, pos):
    """the kernel's order: lane l chains the values at positions l, l + 32, ... from +0, then the xor butterfly"""
    lanes = np.zeros(32)
    for v, j in zip(vals, pos):
        lanes[j % 32] = lanes[j % 32] + v
    for off in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[np.arange(32) ^ off]
    return float(lanes[0])


def root_value(E, b, hg, root, parent, d1_bits, law="pi", mult=None, rows=None):
    """dict(ok, vstar, hit, H, gE [M, ld], gb [M], abs_E, abs_b, G {a: G(a)}, p, pi, ...) for one root"""
    N, ld = hg.n_node, E.shape[1]
    M = N if rows is None else len(rows)
    out = dict(ok=0, vstar=0.0, hit=0.0, H=0.0, gE=np.zeros((M, ld)), gb=np.zeros(M), abs_E=np.zeros((M, ld)),
               abs_b=np.zeros(M), G={})
    dist, root_ok = go.distribution(np.asarray(E, np.float32), np.asarray(b, np.float32), hg.indptr, hg.adj, root, parent,
                                    d1_bits)
    if not root_ok or hg.raw_indptr[root + 1] == hg.raw_indptr[root]:
        return out
    mult = entry_mult(hg) if mult is None else mult
    owner, cand, is_father, ptr, owners, removed = go.candidate_lists(hg.indptr, hg.adj, root, parent, d1_bits)
    pi = gro._lists(E, b, owner, cand, ptr, law)
    a0, a1 = hg.indptr[root], hg.indptr[root + 1]
    ents = [e for e in range(a0, a1) if parent[hg.adj[e]] == root]
    deg = float(hg.raw_indptr[root + 1] - hg.raw_indptr[root])
    rec_of = {}                                                # (owner, cand) -> record
    for r in np.flatnonzero(np.isin(owner, np.concatenate([[root], hg.adj[ents]]))):
        rec_of[(int(owner[r]), int(cand[r]))] = r
    G, hs, pt, p, pca, pac = {}, {}, {}, {}, {}, {}
    for e in ents:
        a = int(hg.adj[e])
        pca[a] = pi[rec_of[(root, a)]]
        fr = rec_of.get((a, root)) if not removed[a] else None
        pac[a] = pi[fr] if fr is not None and is_father[fr] else 0.0
        g = dist[a] if law == "pi" else pca[a] * pac[a]
        if law == "pi":
            assert g == (pca[a] * pac[a] if fr is not None else 0.0)
        G[a] = g
        p[a] = mult[e] / deg
        hs[a] = g * np.log1p(p[a] / g) if g > 0 else 0.0
        pt[a] = p[a] * np.log1p(g / p[a]) if g > 0 else 0.0
    pos = [e - a0 for e in ents]
    A = [int(hg.adj[e]) for e in ents]
    hit = _lane_sum([G[a] for a in A], pos)
    H = _lane_sum([hs[a] for a in A], pos)
    vstar = 0.0 - _lane_sum([pt[a] + hs[a] for a in A], pos)
    # gradient: w per record of the root's and the depth-1 lists; piece = the sizes the rounding is relative to
    w = np.zeros(len(owner))
    piece = np.zeros(len(owner))
    for a in A:
        r = rec_of[(root, a)]
        w[r] = hs[a] - pca[a] * H
        piece[r] = abs(hs[a]) + abs(pca[a] * H)
        if hs[a] == 0.0:
            continue
        for r2 in range(ptr[np.searchsorted(owners, a)], ptr[np.searchsorted(owners, a) + 1]):
            if is_father[r2]:
                w[r2] = hs[a] * (1.0 - pi[r2])
                piece[r2] = abs(hs[a]) + abs(hs[a] * pi[r2])
            else:
                w[r2] = -pi[r2] * hs[a]
                piece[r2] = abs(pi[r2] * hs[a])
    Ef = np.asarray(E, np.float64)
    slot = np.arange(N) if rows is None else np.full(N, -1, np.int64)
    if rows is not None:
        slot[rows] = np.arange(len(rows))
    gE, aE = np.zeros((M, ld)), np.zeros((M, ld))
    for u, v in ((owner, cand), (cand, owner)):
        r = np.flatnonzero((slot[u] >= 0) & (w != 0))
        np.add.at(gE, slot[u[r]], -w[r, None] * Ef[v[r]])
        np.add.at(aE, slot[u[r]], piece[r, None] * np.abs(Ef[v[r]]))
    gb, ab = np.zeros(M), np.zeros(M)
    r = np.flatnonzero((slot[cand] >= 0) & (w != 0))
    np.add.at(gb, slot[cand[r]], -w[r])
    np.add.at(ab, slot[cand[r]], piece[r])
    out.update(ok=1, vstar=vstar, hit=hit, H=H, gE=gE, gb=gb, abs_E=aE, abs_b=ab, G=G, p=p, hs=hs, pi=pi, pca=pca, pac=pac,
               owner=owner, cand=cand, w=w)
    return out


def value_at(G, p_raw, Dv):
    """V_c(G, D) for a discriminator given by its values D(v) in (0, 1): sum_v p(v) log D(v) + sum_v G(v) log(1 - D(v));
    G, p_raw: {node: mass}, Dv: {node: D}"""
    return (sum(m * np.log(Dv[v]) for v, m in p_raw.items()) + sum(g * np.log1p(-Dv[v]) for v, g in G.items() if g > 0))


def raw_law(hg, root):
    """p_true(. | root) over the raw list, self-loops and duplicates included: {node: mass}"""
    nb = hg.raw_adj[hg.raw_indptr[root]:hg.raw_indptr[root + 1]]
    u, cnt = np.unique(nb, return_counts=True)
    return {int(v): c / len(nb) for v, c in zip(u, cnt)}


def grad(E, b, hg, roots, parents, d1_bits, law="pi", rows=None):
    """sums over ``roots`` -> (gE, gb, abs_E, abs_b, per-root dicts)"""
    M, ld = hg.n_node if rows is None else len(rows), E.shape[1]
    mult = entry_mult(hg)
    gE, gb, aE, ab, per = np.zeros((M, ld)), np.zeros(M), np.zeros((M, ld)), np.zeros(M), []
    for k, r in enumerate(roots):
        o = root_value(E, b, hg, int(r), parents[k], d1_bits, law, mult, rows)
        gE += o["gE"]
        gb += o["gb"]
        aE += o["abs_E"]
        ab += o["abs_b"]
        per.append(o)
    return gE, gb, aE, ab, per
