"""TEST INFRASTRUCTURE ONLY: the second moment of one G walk's step on the host (DESIGN.md section 5.9).

A G walk that stops at y has the body root = a_0, ..., a_L = y and adds the fixed vector s(y): for every pair
(a_i, a_j), 0 < |i - j| <= w, row a_i gets kappa(a_i, a_j) E_G[a_j], row a_j gets kappa(a_i, a_j) E_G[a_i] and b[a_j]
gets kappa(a_i, a_j), with the kappas of tests/expected_g_grad_oracle.root_expect (including its ambiguous-sigmoid flags).

- ``literal_root`` builds s(y) from body_pairs of the path root -> y -> father(y) for every reached y, then |s(y)|^2,
  sq_c = sum_y P(y) |s(y)|^2, m_c = sum_y P(y) s(y) and mn_c = |m_c|^2 directly.
- ``path_sq`` builds the same |s(y)|^2 for chosen nodes from their tree paths alone (no law, no whole-tree pass).
- ``pf_tail`` restates the device's decomposition in numpy over every reached node: full(y) (the row depth(y) - w of
  y's path), tail(y) (the rows below it), Pf(y) = Pf(father(y)) + full(y) and |s(y)|^2 = Pf(y) + tail(y), with the sums
  of |terms| that bound the device's rounding (an ambiguous pair's |kappa| widened as root_expect widens it).
"""
import numpy as np

from tests import expected_g_grad_oracle as eo


def kappa_planes(o, N, window):
    """kup[d - 1, y] = kappa(anc_d(y), y), kdn[d - 1, y] = kappa(y, anc_d(y)) (fp64 of the fp32 values) and the
    ambiguous flags, from root_expect's pairs"""
    kup, kdn, amb = np.zeros((window, N)), np.zeros((window, N)), np.zeros((window, N), bool)
    if not o["ok"]:
        return kup, kdn, amb
    father, X, Y = o["father"], o["X"], o["Y"]
    d = np.zeros(len(X), np.int64)                              # X = anc_d(Y): walk up from Y
    x = Y.copy()
    for k in range(1, window + 1):
        x = np.where(x >= 0, father[np.maximum(x, 0)], -1)
        d[(x == X) & (d == 0)] = k
    kup[d - 1, Y], kdn[d - 1, Y] = np.asarray(o["k_up"], np.float64), np.asarray(o["k_dn"], np.float64)
    amb[d - 1, Y] = o.get("amb_pairs", False)
    return kup, kdn, amb


def root_pairs(E_g, b_g, hg, root, parent, d1_bits, window, reward):
    """root_expect with the ambiguous flag of every pair kept (``amb_pairs``)"""
    from tests import update_bits_oracle as ub
    o = eo.root_expect(E_g, b_g, hg, root, parent, d1_bits, window, reward)
    if o["ok"]:
        Eg, bg = np.ascontiguousarray(E_g, np.float32), np.asarray(b_g, np.float32)
        _, amb_up = ub.delta(1, ub.score(Eg, bg, o["X"], o["Y"]), reward(o["X"], o["Y"]), 1)
        _, amb_dn = ub.delta(1, ub.score(Eg, bg, o["Y"], o["X"]), reward(o["Y"], o["X"]), 1)
        o["amb_pairs"] = amb_up | amb_dn
    return o


def tree_path(father, y):
    path = [int(y)]
    while father[path[-1]] >= 0:
        path.append(int(father[path[-1]]))
    return path[::-1]


def step_of(E, path, window, kap):
    """s(y) of the walk with the recorded path root -> y -> father(y): ({row: vector}, {node: bias})"""
    rows, bias = {}, {}
    for n1, n2 in eo.body_pairs(path, window):
        k = kap[(n1, n2)]
        rows[n1] = rows.get(n1, 0.0) + k * E[n2]
        rows[n2] = rows.get(n2, 0.0) + k * E[n1]
        bias[n2] = bias.get(n2, 0.0) + k
    return rows, bias


def sq_of(rows, bias):
    return float(sum(float(v @ v) for v in rows.values()) + sum(b * b for b in bias.values()))


def path_sq(E_g, b_g, parent, ys, window, reward):
    """the literal |s(y)|^2 of the nodes ``ys`` from their tree paths alone (``parent``: the tree's parent array, -1 at
    the root), each path pair's kappa computed on its own, and its sum of |terms| (|kappa| and |E_G| throughout).
    Returns (sq, abs_sq, ambiguous): a node with an ambiguous sigmoid on its path may be a kappa ulp off the device."""
    from tests import update_bits_oracle as ub
    Eg, bg = np.ascontiguousarray(E_g, np.float32), np.asarray(b_g, np.float32)
    sq, ab, amb = np.zeros(len(ys)), np.zeros(len(ys)), np.zeros(len(ys), bool)
    for t, y in enumerate(ys):
        path = tree_path(parent, y) + [int(parent[y])]
        pairs = eo.body_pairs(path, window)
        n1 = np.array([q[0] for q in pairs], np.int64)
        n2 = np.array([q[1] for q in pairs], np.int64)
        k, a = ub.delta(1, ub.score(Eg, bg, n1, n2), reward(n1, n2), 1)
        ids = sorted(set(path))                                  # the path's rows only, relabelled 0 .. m - 1
        loc = {v: i for i, v in enumerate(ids)}
        E = Eg[ids].astype(np.float64)
        lpath = [loc[v] for v in path]
        kap = {(loc[q[0]], loc[q[1]]): v for q, v in zip(pairs, k.astype(np.float64).tolist())}
        sq[t] = sq_of(*step_of(E, lpath, window, kap))
        ab[t] = sq_of(*step_of(np.abs(E), lpath, window, {q: abs(v) for q, v in kap.items()}))
        amb[t] = bool(np.any(a))
    return sq, ab, amb


def literal_root(E_g, o, window):
    """dict(ok, sq_node [N], sq, mE [N, ld], mb [N], mn) of one root from root_pairs' output"""
    E = np.asarray(E_g, np.float64)
    N, ld = E.shape
    out = dict(ok=o["ok"], sq_node=np.zeros(N), sq=0.0, mE=np.zeros((N, ld)), mb=np.zeros(N), mn=0.0)
    if not o["ok"]:
        return out
    kap = {}
    for x, y, ku, kd in zip(o["X"].tolist(), o["Y"].tolist(), o["k_up"].tolist(), o["k_dn"].tolist()):
        kap[(x, y)], kap[(y, x)] = float(ku), float(kd)
    father, dist = o["father"], o["dist"]
    for y in np.flatnonzero(o["depth"] > 0):
        rows, bias = step_of(E, tree_path(father, y) + [int(father[y])], window, kap)
        out["sq_node"][y] = sq_of(rows, bias)
        p = dist[y]
        if p > 0:
            for n, v in rows.items():
                out["mE"][n] += p * v
            for n, b in bias.items():
                out["mb"][n] += p * b
    out["sq"] = float((dist * out["sq_node"]).sum())
    out["mn"] = float((out["mE"] ** 2).sum() + (out["mb"] ** 2).sum())
    return out


def pf_tail(E_g, o, window, chunk=1 << 15):
    """dict(full, tail, pf, sq_node, abs_sq [N]) of one ok root (root_pairs' output): section 5.9's decomposition"""
    E = np.asarray(E_g, np.float64)
    N = E.shape[0]
    father, depth = o["father"], o["depth"]
    kup, kdn, amb = kappa_planes(o, N, window)
    wid = np.where(amb, eo.AMB_WIDEN, 0.0)
    full, tail, a_full, a_tail = np.zeros(N), np.zeros(N), np.zeros(N), np.zeros(N)
    ys_all = np.flatnonzero(depth > 0)
    P = 2 * window + 1
    for c0 in range(0, len(ys_all), chunk):
        ys = ys_all[c0:c0 + chunk]
        anc = np.full((P, len(ys)), -1, np.int64)
        anc[0] = ys
        for v in range(1, P):
            prev = anc[v - 1]
            anc[v] = np.where(prev >= 0, father[np.maximum(prev, 0)], -1)
        lc = np.minimum(depth[ys], 2 * window)

        def row(u):
            R, A = np.zeros((len(ys), E.shape[1])), np.zeros((len(ys), E.shape[1]))
            B, AB = np.zeros(len(ys)), np.zeros(len(ys))
            for v in range(P - 1, -1, -1):                       # path order: j ascending
                if v == u or abs(v - u) > window:
                    continue
                live = v <= lc
                if not live.any():
                    continue
                deep = anc[min(u, v)][live]
                dd = abs(v - u) - 1
                ku, kd, wv = kup[dd, deep], kdn[dd, deep], wid[dd, deep]
                cf = ku + kd
                nb = np.maximum(anc[v][live], 0)
                R[live] += cf[:, None] * E[nb]
                A[live] += (np.abs(cf) * (1 + wv))[:, None] * np.abs(E[nb])
                kb = kd if v < u else ku
                B[live] += kb
                AB[live] += np.abs(kb) * (1 + wv)
            return (R * R).sum(axis=1) + B * B, (A * A).sum(axis=1) + AB * AB
        r, a = row(window)
        has = lc >= window
        full[ys[has]], a_full[ys[has]] = r[has], a[has]
        for u in range(window - 1, -1, -1):
            r, a = row(u)
            has = lc >= u
            tail[ys[has]] += r[has]
            a_tail[ys[has]] += a[has]
    pf, a_pf = full.copy(), a_full.copy()
    for lev in range(2, int(depth.max(initial=0)) + 1):
        ys = np.flatnonzero(depth == lev)
        pf[ys] += pf[father[ys]]
        a_pf[ys] += a_pf[father[ys]]
    return dict(full=full, tail=tail, pf=pf, sq_node=pf + tail, abs_sq=a_pf + a_tail)
