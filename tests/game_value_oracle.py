"""TEST INFRASTRUCTURE ONLY: the GraphGAN game value V_c(G, D) on the host (DESIGN.md section 5.2).

    pos_c = -(1 / |graph[c]|) sum_k bce(s(c, graph[c][k]), 1)       raw adjacency, entry order
    neg_c = -sum_v G(v | c) bce(s(c, v), 0)                           G(. | c): tests/gdist_oracle.distribution
    s(c, v) = fp32 canonical dot(E_D[c], E_D[v]) + b_D[v]             tests/gdist_oracle.dots, then an fp32 add
    bce(s, y) = (max(s, 0) - s y) + log1p(exp(-|s|))                  fp64 from the fp32 s

The sums here are plain numpy sums, not the kernel's order: comparisons are relative to the sum of |terms|.
"""
import numpy as np

from tests import gdist_oracle as go


def bce(s, y):
    """TF's sigmoid_cross_entropy_with_logits (discriminator.py:26-30) in fp64 from fp32 logits."""
    x = np.asarray(s, np.float32).astype(np.float64)
    return (np.maximum(x, 0.0) - x * float(y)) + np.log1p(np.exp(-np.abs(x)))


def scores(E, bias, c, vs):
    """s(c, v) for every v of ``vs`` (E: padded fp32 [N, ld]) -> float32."""
    vs = np.asarray(vs, np.int64)
    return (go.dots(E, np.full(vs.shape[0], c, np.int64), vs) + np.asarray(bias, np.float32)[vs]).astype(np.float32)


def pos_term(E, bias, raw_indptr, raw_adj, c):
    """(pos_c, sum of |terms|) over graph[c] (duplicates and self-loops count)."""
    nb = np.asarray(raw_adj[raw_indptr[c]:raw_indptr[c + 1]], np.int64)
    if nb.shape[0] == 0:
        return 0.0, 0.0
    t = bce(scores(E, bias, c, nb), 1) / nb.shape[0]
    return -float(t.sum()), float(t.sum())


def neg_term(E, bias, c, dist_row):
    """(neg_c, sum of |terms|) for G(. | c) = dist_row; nodes of probability 0 contribute nothing."""
    v = np.flatnonzero(dist_row)
    t = dist_row[v] * bce(scores(E, bias, c, v), 0)
    return -float(t.sum()), float(t.sum())


def game_value(E_d, b_d, E_g, b_g, hg, root, parent, d1_bits):
    """(pos, neg, ok, |pos terms|, |neg terms|) of one root: hg a graph.HostGraph, parent the root's BFS parent array,
    d1_bits the father-removal bits the G law reads."""
    dist, root_ok = go.distribution(E_g, b_g, hg.indptr, hg.adj, root, parent, d1_bits)
    if not root_ok or hg.raw_indptr[root + 1] == hg.raw_indptr[root]:
        return 0.0, 0.0, 0, 0.0, 0.0
    p, pa = pos_term(E_d, b_d, hg.raw_indptr, hg.raw_adj, root)
    n, na = neg_term(E_d, b_d, root, dist)
    return p, n, 1, pa, na
