"""TEST INFRASTRUCTURE ONLY: the exact discriminator gradient of the game value on the host (DESIGN.md section 5.4).

Per root c (ok_c = 1), G(. | c) the generator's law (tests/gdist_oracle.distribution, or rows passed in):
    W(v) = dV_c / ds(c, v) = n_v sigma(-s) / deg_c - G(v | c) sigma(s)       n_v: v's count in the raw list graph[c]
    grad_b[v] += W(v),  grad_E[v] += W(v) E_D[c],  grad_E[c] += sum_v W(v) E_D[v]
with sigma(|s|) = 1 / (1 + e), sigma(-|s|) = e sigma(|s|), e = exp(-|s|), in fp64.  Two laws for s:
    "fp32"   -- the kernel's: the canonical fp32 score of tests/game_value_oracle.scores;
    "smooth" -- fp64 scores E_D[c] . E_D[v] + b_D[v]: an ordinary differentiable function of (E_D, b_D), so its gradient
                can be checked against finite differences of ``value_smooth``.
Sums here are numpy's, not the kernel's order: comparisons are relative to sums of |terms| (``abs_*``), where W(v) is
counted as its two pieces |n_v sigma(-s) / deg_c| + |G sigma(s)|.
"""
import numpy as np

from tests import game_value_oracle as vo
from tests import gdist_oracle as go


def sigmoids(s):
    """(sigma(s), sigma(-s)) in fp64, the kernel's formulas"""
    x = np.asarray(s, np.float64)
    e = np.exp(-np.abs(x))
    big = 1.0 / (1.0 + e)
    small = e * big
    return np.where(x >= 0, big, small), np.where(x >= 0, small, big)


def bce64(x, y):
    """sigmoid cross-entropy in fp64 from fp64 logits (the smooth law's)"""
    x = np.asarray(x, np.float64)
    return (np.maximum(x, 0.0) - x * float(y)) + np.log1p(np.exp(-np.abs(x)))


def _scores(E, b, c, v, law):
    if law == "fp32":
        return vo.scores(np.asarray(E, np.float32), np.asarray(b, np.float32), c, v).astype(np.float64)
    assert law == "smooth"
    E = np.asarray(E, np.float64)
    return E[v] @ E[c] + np.asarray(b, np.float64)[v]


def laws(E_g, b_g, hg, roots, parents, d1_bits):
    """the generator's G-mode law of every root -> (dist [R, N], root_ok [R])"""
    out = [go.distribution(np.asarray(E_g, np.float32), np.asarray(b_g, np.float32), hg.indptr, hg.adj, int(r), parents[k],
                           d1_bits) for k, r in enumerate(roots)]
    return np.stack([d for d, _ in out]), np.asarray([o for _, o in out], np.int32)


def root_ok(hg, root, law_ok):
    return int(bool(law_ok) and hg.raw_indptr[root + 1] > hg.raw_indptr[root])


def root_w(E_d, b_d, hg, root, dist_row, law_ok, law="fp32"):
    """(W [N], |W pieces| [N]) of one root; both zero when ok_c = 0"""
    N = hg.n_node
    W, P = np.zeros(N), np.zeros(N)
    if not root_ok(hg, root, law_ok):
        return W, P
    lo, hi = hg.raw_indptr[root], hg.raw_indptr[root + 1]
    m = np.bincount(hg.raw_adj[lo:hi], minlength=N)
    v = np.flatnonzero((m > 0) | (np.asarray(dist_row) != 0))
    sp, sn = sigmoids(_scores(E_d, b_d, root, v, law))
    wp, wn = m[v] * sn / float(hi - lo), dist_row[v] * sp
    W[v], P[v] = wp - wn, np.abs(wp) + np.abs(wn)
    return W, P


def grad(E_d, b_d, hg, roots, dists, oks, law="fp32", rows=None):
    """The sums over ``roots`` (dists[k], oks[k]: the law of roots[k]) -> (gE [M, ld], gb [M], abs_E [M, ld], abs_b [M]);
    M = N, or only the nodes ``rows`` (distinct ids) in that order."""
    N, ld = hg.n_node, E_d.shape[1]
    E = np.asarray(E_d, np.float32 if law == "fp32" else np.float64)
    rows = np.arange(N) if rows is None else np.asarray(rows, np.int64)
    slot = np.full(N, -1, np.int64)
    slot[rows] = np.arange(len(rows))
    gE, aE, gb, ab = np.zeros((len(rows), ld)), np.zeros((len(rows), ld)), np.zeros(len(rows)), np.zeros(len(rows))
    for k, c in enumerate(roots):
        c = int(c)
        W, P = root_w(E_d, b_d, hg, c, dists[k], oks[k], law)
        ec = E[c].astype(np.float64)
        gb += W[rows]
        ab += P[rows]
        gE += W[rows, None] * ec[None, :]                  # node side
        aE += P[rows, None] * np.abs(ec)[None, :]
        if slot[c] >= 0:                                    # centre side
            nz = np.flatnonzero(P)
            for i in range(0, len(nz), 1 << 16):
                b = nz[i:i + (1 << 16)]
                Ev = E[b].astype(np.float64)
                gE[slot[c]] += W[b] @ Ev
                aE[slot[c]] += P[b] @ np.abs(Ev)
    return gE, gb, aE, ab


def value_smooth(E_d, b_d, hg, roots, dists, oks):
    """sum over the ok roots of V_c with fp64 scores (the function the "smooth" gradient differentiates)"""
    total = 0.0
    for k, c in enumerate(roots):
        c = int(c)
        if not root_ok(hg, c, oks[k]):
            continue
        lo, hi = hg.raw_indptr[c], hg.raw_indptr[c + 1]
        nb = np.asarray(hg.raw_adj[lo:hi], np.int64)
        total -= bce64(_scores(E_d, b_d, c, nb, "smooth"), 1).sum() / float(hi - lo)
        v = np.flatnonzero(dists[k])
        total -= (dists[k][v] * bce64(_scores(E_d, b_d, c, v, "smooth"), 0)).sum()
    return float(total)
