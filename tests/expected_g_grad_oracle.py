"""TEST INFRASTRUCTURE ONLY: the exact expectation of the reference's generator step on the host (DESIGN.md section 5.6).

Per root c (ok_c = 1), over the lists of tests/gdist_oracle.candidate_lists with the kernel's step law pi:
    reach(root) = 1,  reach(x) = reach(a) pi_a(x)          (the section 5.1 chain: the probability that a walk passes x)
    pairs: every reached y != c, d = 1 .. min(w, depth(y)), x = anc_d(y): (x, y) and (y, x), each with weight rho = reach(y)
    kappa(n1, n2) = the pair_delta mode 1 value (tests/update_bits_oracle.delta, batch_total 1) with a_k = r(n1, n2)
    grad_E[n1] += rho kappa E_G[n2],  grad_E[n2] += rho kappa E_G[n1],  grad_b[n2] += rho kappa
The reward r is the fp32 reward of gg_pair_reward: ``reward(n1, n2)`` gives it (on a GPU, the production kernel's bits);
the default is a numpy float32 statement of the same formula, which may differ from the device's logf / expf by an ulp.
Sums here are numpy's, not the kernel's order: comparisons are relative to sums of |terms| (``abs_*``).  A pair whose
fp64 sigmoid lies next to an fp32 rounding boundary (update_bits_oracle.sigmoid's ``ambiguous``) may get a kappa one ulp
away on the device; its terms widen ``abs_*`` by |term| 2^-20 / 1e-12 so that a 1e-12 bar admits that ulp.
"""
import numpy as np

from tests import gdist_oracle as go
from tests import update_bits_oracle as ub
from tests import value_grad_oracle as gro

F = np.float32
AMB_WIDEN = 2.0 ** -20 / 1e-12


def numpy_reward(E_d, b_d):
    """r(n1, n2) = log(1 + exp(clip(s_D, -10, 10))) in float32, s_D the canonical score (discriminator.py:33-34)"""
    E_d, b_d = np.ascontiguousarray(E_d, F), np.asarray(b_d, F)

    def reward(n1, n2):
        s = np.clip(ub.score(E_d, b_d, n1, n2), F(-10), F(10)).astype(F)
        return np.log(F(1) + np.exp(s)).astype(F)
    return reward


def tree_reach(E_g, b_g, hg, root, parent, d1_bits):
    """(ok, reach fp64 [N], father int64 [N] (-1: the root or not reached), depth int64 [N], dist fp64 [N], records)"""
    N = hg.n_node
    dist, ok = go.distribution(np.asarray(E_g, F), np.asarray(b_g, F), hg.indptr, hg.adj, root, parent, d1_bits)
    reach, father, depth = np.zeros(N), np.full(N, -1, np.int64), np.zeros(N, np.int64)
    owner, cand, is_father, ptr, owners, _ = go.candidate_lists(hg.indptr, hg.adj, root, parent, d1_bits)
    if not ok:
        return 0, reach, father, depth, dist, None
    pi = gro._lists(E_g, b_g, owner, cand, ptr, "pi")
    reach[root] = 1.0
    child = np.flatnonzero(~is_father)
    frontier = np.zeros(N, bool)
    frontier[root] = True
    lev = 0
    while True:
        sel = child[frontier[owner[child]]]
        sel = sel[reach[owner[sel]] * pi[sel] > 0]
        if len(sel) == 0:
            break
        lev += 1
        reach[cand[sel]] = reach[owner[sel]] * pi[sel]
        father[cand[sel]] = owner[sel]
        depth[cand[sel]] = lev
        frontier = np.zeros(N, bool)
        frontier[cand[sel]] = True
    return 1, reach, father, depth, dist, dict(owner=owner, cand=cand, is_father=is_father, pi=pi)


def window_pairs(reach, father, depth, window):
    """(x, y, rho): x = anc_d(y) for every reached y and d = 1 .. min(window, depth(y)), rho = reach(y)"""
    ys = np.flatnonzero(depth > 0)
    xs_all, ys_all = [], []
    x = father[ys].copy()
    for d in range(1, window + 1):
        keep = x >= 0
        xs_all.append(x[keep])
        ys_all.append(ys[keep])
        x = np.where(keep, father[np.maximum(x, 0)], -1)
    X, Y = np.concatenate(xs_all), np.concatenate(ys_all)
    return X, Y, reach[Y]


def assemble(E_g, X, Y, rho, k_up, k_dn, rows=None, amb=None):
    """grad_E, grad_b and the sums of |terms| of the pairs (X, Y) with weights rho and coefficients k_up = kappa(X, Y),
    k_dn = kappa(Y, X) (fp64 values); ``rows``: only these node ids, in that order; ``amb``: pairs whose |terms| widen
    the bars"""
    E = np.asarray(E_g, np.float64)
    N, ld = E.shape
    M = N if rows is None else len(rows)
    slot = np.arange(N) if rows is None else np.full(N, -1, np.int64)
    if rows is not None:
        slot[rows] = np.arange(len(rows))
    gE, aE, gb, ab = np.zeros((M, ld)), np.zeros((M, ld)), np.zeros(M), np.zeros(M)
    widen = np.where(amb, AMB_WIDEN, 0.0) if amb is not None else np.zeros(len(X))
    for n1, n2, k in ((X, Y, k_up), (Y, X, k_dn)):
        c = rho * k
        for u, v in ((n1, n2), (n2, n1)):
            r = np.flatnonzero(slot[u] >= 0)
            np.add.at(gE, slot[u[r]], c[r, None] * E[v[r]])
            np.add.at(aE, slot[u[r]], (np.abs(c[r]) * (1.0 + widen[r]))[:, None] * np.abs(E[v[r]]))
        r = np.flatnonzero(slot[n2] >= 0)
        np.add.at(gb, slot[n2[r]], c[r])
        np.add.at(ab, slot[n2[r]], np.abs(c[r]) * (1.0 + widen[r]))
    return gE, gb, aE, ab


def root_expect(E_g, b_g, hg, root, parent, d1_bits, window, reward, rows=None):
    """dict(ok, n_pairs, gE, gb, abs_E, abs_b, n_amb, ...) of one root; E_g fp32 [N, ld]"""
    N, ld = hg.n_node, E_g.shape[1]
    M = N if rows is None else len(rows)
    ok, reach, father, depth, dist, rec = tree_reach(E_g, b_g, hg, root, parent, d1_bits)
    out = dict(ok=ok, n_pairs=0.0, gE=np.zeros((M, ld)), gb=np.zeros(M), abs_E=np.zeros((M, ld)), abs_b=np.zeros(M),
               n_amb=0, reach=reach, father=father, depth=depth, dist=dist)
    if not ok:
        return out
    X, Y, rho = window_pairs(reach, father, depth, window)
    Eg, bg = np.ascontiguousarray(E_g, F), np.asarray(b_g, F)
    k_up, amb_up = ub.delta(1, ub.score(Eg, bg, X, Y), reward(X, Y), 1)
    k_dn, amb_dn = ub.delta(1, ub.score(Eg, bg, Y, X), reward(Y, X), 1)
    amb = amb_up | amb_dn
    gE, gb, aE, ab = assemble(Eg, X, Y, rho, k_up.astype(np.float64), k_dn.astype(np.float64), rows, amb)
    m = np.minimum(depth, window)
    out.update(n_pairs=float((reach * 2 * m).sum()), gE=gE, gb=gb, abs_E=aE, abs_b=ab, n_amb=int(amb.sum()), X=X, Y=Y,
               rho=rho, k_up=k_up, k_dn=k_dn)
    return out


def expect(E_g, b_g, hg, roots, parents, d1_bits, window, reward, rows=None):
    """the sums over ``roots`` -> (gE, gb, abs_E, abs_b, per-root dicts)"""
    M, ld = hg.n_node if rows is None else len(rows), E_g.shape[1]
    gE, gb, aE, ab, per = np.zeros((M, ld)), np.zeros(M), np.zeros((M, ld)), np.zeros(M), []
    for k, r in enumerate(roots):
        o = root_expect(E_g, b_g, hg, int(r), parents[k], d1_bits, window, reward, rows)
        gE += o["gE"]
        gb += o["gb"]
        aE += o["abs_E"]
        ab += o["abs_b"]
        per.append(o)
    return gE, gb, aE, ab, per


def body_pairs(path, window):
    """get_node_pairs_from_path (graph_gan.py:272-291) of one recorded path, as (center, node) pairs"""
    path = path[:-1]
    pairs = []
    for i in range(len(path)):
        for j in range(max(i - window, 0), min(i + window + 1, len(path))):
            if i != j:
                pairs.append((path[i], path[j]))
    return pairs


def enumerate_walks(hg, root, parent, dist, window):
    """every G walk of an ok root by brute force: the walk stopping at v (probability dist[v]) has the tree path root -> v
    followed by father(v).  Returns ({(n1, n2): expected count per walk}, expected pairs per walk)."""
    counts, total = {}, 0.0
    for v in np.flatnonzero(dist > 0):
        path = [int(v)]
        while path[-1] != root:
            path.append(int(parent[path[-1]]))
        path = path[::-1] + [int(parent[v])]
        ps = body_pairs(path, window)
        total += dist[v] * len(ps)
        for p in ps:
            counts[p] = counts.get(p, 0.0) + dist[v]
    return counts, total
