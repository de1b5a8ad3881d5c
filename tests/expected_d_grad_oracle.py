"""TEST INFRASTRUCTURE ONLY: the D-mode walk law and the exact expectation of the reference's discriminator step of one
pass on the host (DESIGN.md section 5.7).

Per root c, over the lists of tests/gdist_oracle.candidate_lists with every father-removal bit of the root's entries set
(a D walk removes the root from every depth-1 list, graph_gan.py:258-259, so the bits it finds do not matter):
    reach(root) = 1,  reach(x) = reach(a) pi_a(x)                         (the section 5.1 chain)
    P_D(v) = reach(v) pi_v(father(v)) for depth(v) >= 2,  0 at the root and at depth 1
    p_void = sum of reach(a) over the depth-1 leaves a                     (graph_gan.py:255-257)
    P_acc = (1 - p_void)^deg_c, square-and-multiply from the least significant bit (``accept``)
    Q = P_D / (1 - p_void),  W_ref(v) = fl(fl(deg_c P_acc) W(v)),  W = section 5.4's per-pair weight with the law Q
The assembly of W_ref is tests/value_grad_d_oracle.grad's, root by root, scaled by a_k = fl(deg_c P_acc).
"""
import numpy as np

from tests import gdist_oracle as go
from tests import value_grad_d_oracle as vd
from tests import value_grad_oracle as gro


def all_bits(hg):
    """father-removal bits with every entry set"""
    return np.full((len(hg.adj) + 31) // 32 + 1, 0xFFFFFFFF, np.uint32)


def d_law(E_g, b_g, hg, root, parent):
    """(P_D fp64 [N], p_void, root_ok) of one root"""
    N = hg.n_node
    owner, cand, is_father, ptr, owners, _ = go.candidate_lists(hg.indptr, hg.adj, root, parent, all_bits(hg))
    P = np.zeros(N, np.float64)
    if not np.any(owner == root):
        return P, 0.0, 0
    pi = gro._lists(E_g, b_g, owner, cand, ptr, "pi")
    reach = np.zeros(N, np.float64)
    reach[root] = 1.0
    child = np.flatnonzero(~is_father)
    frontier = np.zeros(N, bool)
    frontier[root] = True
    while True:
        sel = child[frontier[owner[child]]]
        if len(sel) == 0:
            break
        reach[cand[sel]] = reach[owner[sel]] * pi[sel]
        frontier = np.zeros(N, bool)
        frontier[cand[sel]] = True
    fr = np.flatnonzero(is_father)
    P[owner[fr]] = reach[owner[fr]] * pi[fr]
    has_list = np.zeros(N, bool)
    has_list[owners] = True
    d1 = np.flatnonzero(parent == root)
    d1 = d1[d1 != root]
    leaves = d1[~has_list[d1]]
    p_void = float(np.sort(reach[leaves]).sum()) if len(leaves) else 0.0
    return P, p_void, 1


def d_laws(E_g, b_g, hg, roots, parents):
    """(P_D [R, N], p_void [R], root_ok [R])"""
    out = [d_law(E_g, b_g, hg, int(r), parents[k]) for k, r in enumerate(roots)]
    return (np.stack([o[0] for o in out]), np.asarray([o[1] for o in out], np.float64),
            np.asarray([o[2] for o in out], np.int32))


def accept(p_void, deg):
    """P_acc = (1 - p_void)^deg: square-and-multiply from the least significant bit, one fp64 product per step"""
    base, p, e = 1.0 - float(p_void), 1.0, int(deg)
    while e > 0:
        if e & 1:
            p = p * base
        base = base * base
        e >>= 1
    return p


def root_accept(hg, root, p_void, law_ok):
    """(P_acc, ok_ref) of one root: 0, 0 unless deg_c > 0 and the root has children"""
    deg = int(hg.raw_indptr[root + 1] - hg.raw_indptr[root])
    if deg == 0 or not law_ok:
        return 0.0, 0
    p = accept(p_void, deg)
    return p, int(p > 0.0)


def law_q(P_row, p_void):
    """Q = P_D / (1 - p_void), one fp64 division per node"""
    return np.asarray(P_row, np.float64) / (1.0 - float(p_void))


def grad(E_d, b_d, hg, roots, P_D, p_void, root_ok, law="fp32", rows=None):
    """The expected D step summed over ``roots`` -> (gE [M, ld], gb [M], abs_E, abs_b, accept [R], ok_ref [R])"""
    M = hg.n_node if rows is None else len(rows)
    ld = E_d.shape[1]
    gE, gb, aE, ab = np.zeros((M, ld)), np.zeros(M), np.zeros((M, ld)), np.zeros(M)
    acc, okr = np.zeros(len(roots)), np.zeros(len(roots), np.int32)
    for k, c in enumerate(roots):
        c = int(c)
        acc[k], okr[k] = root_accept(hg, c, p_void[k], root_ok[k])
        if not okr[k]:
            continue
        a = float(hg.raw_indptr[c + 1] - hg.raw_indptr[c]) * acc[k]
        e, b, ae, abb = vd.grad(E_d, b_d, hg, [c], [law_q(P_D[k], p_void[k])], [1], law, rows)
        gE += a * e
        gb += a * b
        aE += a * ae
        ab += a * abb
    return gE, gb, aE, ab, acc, okr


def pass_loss_smooth(E_d, b_d, hg, roots, P_D, p_void, root_ok):
    """the expected loss of one pass with fp64 scores and the law held fixed:
    sum_c P_acc (sum_k bce(s_ck, 1) + deg_c sum_v Q(v) bce(s_cv, 0)) over the roots with ok_ref = 1"""
    total = 0.0
    for k, c in enumerate(roots):
        c = int(c)
        p, ok = root_accept(hg, c, p_void[k], root_ok[k])
        if not ok:
            continue
        lo, hi = hg.raw_indptr[c], hg.raw_indptr[c + 1]
        nb = np.asarray(hg.raw_adj[lo:hi], np.int64)
        q = law_q(P_D[k], p_void[k])
        v = np.flatnonzero(q)
        pos = vd.bce64(vd._scores(E_d, b_d, c, nb, "smooth"), 1).sum()
        neg = (q[v] * vd.bce64(vd._scores(E_d, b_d, c, v, "smooth"), 0)).sum()
        total += p * (pos + float(hi - lo) * neg)
    return float(total)
