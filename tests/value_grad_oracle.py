"""TEST INFRASTRUCTURE ONLY: the exact generator gradient of the game value on the host (DESIGN.md section 5.3).

Per root c (ok_c = 1), over the lists of tests/gdist_oracle.candidate_lists with a step law pi:
    G(v) = reach(v) pi_v(father(v)),  h(v) = G(v) bce(s_D(c, v), 0),  neg_c = -sum_v h(v)
    T(a) = h(a) + sum_{children x} T(x),  F_a(x) = T(x) (child) or h(a) (father),  w_a(x) = F_a(x) - pi_a(x) T(a)
    d neg_c / d s(a, x) = -w_a(x),  s(a, x) = E_G[a] . E_G[x] + b_G[x]
Two laws:
    "pi"     -- the kernel's: pi from the canonical fp32 scores and CDF (tests/gdist_oracle.step_pi);
    "smooth" -- fp64 scores and an fp64 softmax of the same lists: an ordinary differentiable function of (E_G, b_G),
                so its gradient can be checked against finite differences.
Sums here are numpy's, not the kernel's order: comparisons are relative to sums of |terms| (``abs_*``), where a term
w_a(x) E[x] is counted as its two pieces |F_a(x) E[x]| + |pi_a(x) T(a) E[x]|, the sizes the rounding is relative to.
"""
import numpy as np

from tests import game_value_oracle as vo
from tests import gdist_oracle as go


def _lists(E, bias, owner, cand, ptr, law):
    """the step law of every record"""
    if law == "pi":
        sc = (go.dots(np.ascontiguousarray(E, np.float32), owner, cand) + np.asarray(bias, np.float32)[cand]).astype(np.float32)
        return go.step_pi(go.list_q(sc, ptr), ptr)
    assert law == "smooth"
    E, bias = np.asarray(E, np.float64), np.asarray(bias, np.float64)
    s = np.einsum("ij,ij->i", E[owner], E[cand]) + bias[cand]
    li = np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))
    e = np.exp(s - np.maximum.reduceat(s, ptr[:-1])[li])
    return e / np.add.reduceat(e, ptr[:-1])[li]


def root_grad(E_g, b_g, E_d, b_d, hg, root, parent, d1_bits, law="pi", rows=None):
    """dict(ok, pos, neg, T_root, gE [M, ld], gb [M], abs_E, abs_b, pi, owner, cand, is_father, ...) for one root; E_g /
    E_d: [N, ld] rows (fp32 for "pi"; any float for "smooth"), the gradient is of V_c = pos_c + neg_c (zero for
    ok_c = 0); M = N, or only the nodes ``rows`` (distinct ids) in that order."""
    N, ld = hg.n_node, E_g.shape[1]
    M = N if rows is None else len(rows)
    out = dict(ok=0, pos=0.0, neg=0.0, T_root=0.0, gE=np.zeros((M, ld)), gb=np.zeros(M), abs_E=np.zeros((M, ld)),
               abs_b=np.zeros(M))
    _, root_ok = go.distribution(np.asarray(E_g, np.float32), np.asarray(b_g, np.float32), hg.indptr, hg.adj, root, parent,
                                 d1_bits)
    if not root_ok or hg.raw_indptr[root + 1] == hg.raw_indptr[root]:
        return out
    owner, cand, is_father, ptr, owners, _ = go.candidate_lists(hg.indptr, hg.adj, root, parent, d1_bits)
    pi = _lists(E_g, b_g, owner, cand, ptr, law)
    reach = np.zeros(N)
    reach[root] = 1.0
    child = np.flatnonzero(~is_father)
    frontier = np.zeros(N, bool)
    frontier[root] = True
    levels = []
    while True:
        sel = child[frontier[owner[child]]]
        sel = sel[reach[owner[sel]] * pi[sel] > 0]
        if len(sel) == 0:
            break
        reach[cand[sel]] = reach[owner[sel]] * pi[sel]
        levels.append(sel)
        frontier = np.zeros(N, bool)
        frontier[cand[sel]] = True
    G = np.zeros(N)
    fr = np.flatnonzero(is_father)
    G[owner[fr]] = reach[owner[fr]] * pi[fr]
    v = np.flatnonzero(G)
    h = np.zeros(N)
    h[v] = G[v] * vo.bce(vo.scores(np.asarray(E_d, np.float32), b_d, root, v), 0)
    T = h.copy()
    for sel in reversed(levels):
        np.add.at(T, owner[sel], T[cand[sel]])
    F = np.where(is_father, h[owner], T[cand])
    F[is_father & (reach[owner] == 0)] = 0.0
    w = F - pi * T[owner]
    E = np.asarray(E_g, np.float64)
    piece = np.abs(F) + np.abs(pi * T[owner])
    slot = np.arange(N) if rows is None else np.full(N, -1, np.int64)
    if rows is not None:
        slot[rows] = np.arange(len(rows))
    gE, aE = np.zeros((M, ld)), np.zeros((M, ld))
    for u, v in ((owner, cand), (cand, owner)):              # d s(a, x) / d E[a] = E[x], d s(a, x) / d E[x] = E[a]
        r = np.flatnonzero(slot[u] >= 0)
        np.add.at(gE, slot[u[r]], -w[r, None] * E[v[r]])
        np.add.at(aE, slot[u[r]], piece[r, None] * np.abs(E[v[r]]))
    gb, ab = np.zeros(M), np.zeros(M)
    r = np.flatnonzero(slot[cand] >= 0)
    np.add.at(gb, slot[cand[r]], -w[r])
    np.add.at(ab, slot[cand[r]], piece[r])
    pos, _ = vo.pos_term(np.asarray(E_d, np.float32), b_d, hg.raw_indptr, hg.raw_adj, root)
    out.update(ok=1, pos=pos, neg=-float(h.sum()), T_root=float(T[root]), gE=gE, gb=gb, abs_E=aE, abs_b=ab, pi=pi,
               owner=owner, cand=cand, is_father=is_father, w=w, F=F, T=T, depth=len(levels))
    return out


def grad(E_g, b_g, E_d, b_d, hg, roots, parents, d1_bits, law="pi", rows=None):
    """the sums over ``roots`` (parents[k]: the BFS parent array of roots[k]) -> (gE, gb, abs_E, abs_b, per-root dicts)"""
    M, ld = hg.n_node if rows is None else len(rows), E_g.shape[1]
    gE, gb, aE, ab, per = np.zeros((M, ld)), np.zeros(M), np.zeros((M, ld)), np.zeros(M), []
    for k, r in enumerate(roots):
        o = root_grad(E_g, b_g, E_d, b_d, hg, int(r), parents[k], d1_bits, law, rows)
        gE += o["gE"]
        gb += o["gb"]
        aE += o["abs_E"]
        ab += o["abs_b"]
        per.append(o)
    return gE, gb, aE, ab, per
