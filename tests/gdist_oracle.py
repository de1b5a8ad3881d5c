"""TEST INFRASTRUCTURE ONLY: the exact generator distribution G(v | root) on the host (DESIGN.md section 5.1).

The canonical arithmetic of oracle/gg_oracle.h, vectorised over every candidate list of a tree with numpy so that a
million-node tree takes seconds: fp32 fmaf through fp64 with round-to-odd (the fp64 sum of an exact product and an fp32
addend, rounded to odd, then to fp32, is fmaf's single rounding: 53 >= 2 * 24 + 2), fp32 adds / divisions and fp64
scans as IEEE numpy operations.  test_generator_dist_host.py checks dot, exp and the CDF against the C oracle
(ggo_dot, ggo_exp, ggo_choose at the CDF boundaries) before anything relies on them.
"""
import math

import numpy as np

TWO53 = float(2 ** 53)


def fmaf(a, b, c):
    """fp32 fused multiply-add, elementwise (a, b, c: float32 arrays) -> float32."""
    p = a.astype(np.float64) * b.astype(np.float64)          # exact: 24 + 24 bits
    c = c.astype(np.float64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)                            # s + err == p + c exactly (TwoSum)
    even = (s.view(np.int64) & 1) == 0
    fix = (err != 0) & even
    if fix.any():                                              # round to odd: the odd neighbour towards the exact sum
        s = s.copy()
        s[fix] = np.nextafter(s[fix], np.where(err[fix] > 0, np.inf, -np.inf))
    return s.astype(np.float32)


def exp_c(x):
    """ggo_exp, elementwise (x <= 0, float32)."""
    x = np.asarray(x, np.float32)
    f = lambda v: np.full(x.shape, v, np.float32)
    t = fmaf(x, f(1.44269504088896341), f(12582912.0))
    n = (t - np.float32(12582912.0)).astype(np.float32)
    r = fmaf(n, f(-0.693359375), x)
    r = fmaf(n, f(2.12194440e-4), r)
    p = f(1.9875691500e-4)
    for c in (1.3981999507e-3, 8.3334519073e-3, 4.1665795894e-2, 1.6666665459e-1, 5.0000001201e-1):
        p = fmaf(p, r, f(c))
    r2 = (r * r).astype(np.float32)
    e = fmaf(p, r2, r)
    e = (e + np.float32(1.0)).astype(np.float32)
    ni = np.where(x < -86.0, 0, n).astype(np.int32)
    out = (e.view(np.uint32) + (ni.astype(np.uint32) << np.uint32(23))).view(np.float32)
    return np.where(x < np.float32(-86.0), np.float32(0.0), out).astype(np.float32)


def dots(E, u, v, block=1 << 16):
    """ggo_dot(E[u], E[v]) for index arrays u, v (E: float32 [N, ld])."""
    if len(u) > block:
        return np.concatenate([dots(E, u[i:i + block], v[i:i + block], block) for i in range(0, len(u), block)])
    ld = E.shape[1]
    A = E[u].reshape(len(u), ld // 32, 8, 4)                   # [pair, chunk // 8, lane g, component]
    B = E[v].reshape(len(v), ld // 32, 8, 4)
    s = np.zeros((len(u), 8), np.float32)
    for c in range(ld // 32):
        for k in range(4):
            s = fmaf(A[:, c, :, k], B[:, c, :, k], s)
    for off in (4, 2, 1):
        s = (s + s[:, np.arange(8) ^ off]).astype(np.float32)
    return s[:, 0]


def _butterfly32(v):
    for off in (16, 8, 4, 2, 1):
        v = (v + v[:, np.arange(32) ^ off]).astype(v.dtype)
    return v[:, 0]


def _ks_scan32(x):
    for off in (1, 2, 4, 8, 16):
        y = np.zeros_like(x)
        y[:, off:] = x[:, :-off]
        x = x + y
    return x


def list_q(sc, ptr):
    """Canonical q = cdf / total (fp64) of every list: list i is sc[ptr[i]:ptr[i + 1]] (float32 scores, lists non-empty)."""
    sc = np.asarray(sc, np.float32)
    n = np.diff(ptr)
    L = len(n)
    owner = np.repeat(np.arange(L), n)
    pos = np.arange(len(sc)) - ptr[:-1][owner]
    m = np.maximum.reduceat(sc, ptr[:-1]) if L else np.zeros(0, np.float32)
    e = exp_c((sc - m[owner]).astype(np.float32))
    ntile = (n + 31) // 32
    tptr = np.concatenate([[0], np.cumsum(ntile)])
    tile = tptr[:-1][owner] + pos // 32                       # global tile index of every entry
    grid = np.zeros((int(tptr[-1]), 32), np.float32)
    grid[tile, pos % 32] = e
    T = _butterfly32(grid)                                     # tile sums
    tile_owner = np.repeat(np.arange(L), ntile)
    tpos = np.arange(int(tptr[-1])) - tptr[:-1][tile_owner]
    S = np.zeros(L, np.float32)
    for t in range(int(ntile.max()) if L else 0):              # S = T_0 + T_1 + ... in tile order
        sel = tpos == t
        S[tile_owner[sel]] = (S[tile_owner[sel]] + T[sel]).astype(np.float32)
    x = np.zeros((int(tptr[-1]), 32), np.float64)
    x[tile, pos % 32] = (e / S[owner]).astype(np.float32).astype(np.float64)
    x = _ks_scan32(x)
    carry_t = np.zeros(int(tptr[-1]), np.float64)             # CDF before each tile
    total = np.zeros(L, np.float64)
    for t in range(int(ntile.max()) if L else 0):
        sel = tpos == t
        carry_t[sel] = total[tile_owner[sel]]
        total[tile_owner[sel]] = total[tile_owner[sel]] + x[sel, 31]
    cdf = carry_t[tile] + x[tile, pos % 32]
    return cdf / total[owner]


def step_pi(q, ptr):
    """pi_j = (ceil(q_j 2^53) - ceil(q_{j-1} 2^53)) / 2^53 per list (exact integers; q * 2^53 is exact in fp64)."""
    k = np.ceil(q * TWO53).astype(np.int64)
    prev = np.zeros_like(k)
    prev[1:] = k[:-1]
    prev[ptr[:-1][np.diff(ptr) > 0]] = 0
    return (k - prev).astype(np.float64) / TWO53


def step_pi_exact(q):
    """The same for ONE list as integers: k_j - k_{j-1} (pi_j = that / 2^53), with math.ceil on exact fp64 products."""
    ks = [math.ceil(float(v) * TWO53) for v in q]
    return [ks[0]] + [ks[j] - ks[j - 1] for j in range(1, len(ks))]


def candidate_lists(indptr, adj, root, parent, d1_bits):
    """The G walk's lists over one tree (graph_gan.py:250-259): owner node, candidate id, is-father flag per record,
    grouped by owner (father first, then children in entry order).  Returns (owner, cand, is_father, ptr, owners)."""
    N = len(indptr) - 1
    deg = np.diff(indptr)
    src = np.repeat(np.arange(N, dtype=np.int64), deg)
    in_tree = parent >= 0
    in_tree[root] = True
    child = parent[adj] == src                                 # entry e = (src -> adj[e]) is a tree edge
    ce = np.flatnonzero(child)
    removed = np.zeros(N, bool)
    bits = np.asarray(d1_bits).view(np.uint32)
    re = np.arange(indptr[root], indptr[root + 1])
    re = re[child[re]]
    removed[adj[re]] = ((bits[re >> 5] >> (re & 31).astype(np.uint32)) & 1) == 1
    fa = np.flatnonzero(in_tree & (np.arange(N) != root) & ~removed)
    owner = np.concatenate([fa, src[ce]])
    cand = np.concatenate([parent[fa], adj[ce]]).astype(np.int64)
    key = np.concatenate([np.full(len(fa), -1, np.int64), ce])
    o = np.lexsort((key, owner))
    owner, cand, is_father = owner[o], cand[o], np.concatenate([np.ones(len(fa), bool), np.zeros(len(ce), bool)])[o]
    owners, start = np.unique(owner, return_index=True)
    ptr = np.concatenate([start, [len(owner)]]).astype(np.int64)
    return owner, cand, is_father, ptr, owners, removed


def distribution(E, bias, indptr, adj, root, parent, d1_bits):
    """(dist fp64 [N], root_ok) of one root: the kernel's definition, evaluated level by level in fp64."""
    N = len(indptr) - 1
    E = np.ascontiguousarray(E, np.float32)
    bias = np.asarray(bias, np.float32)
    owner, cand, is_father, ptr, owners, removed = candidate_lists(indptr, adj, root, parent, d1_bits)
    dist = np.zeros(N, np.float64)
    if not np.any(owner == root):
        return dist, 0
    sc = (dots(E, owner, cand) + bias[cand]).astype(np.float32)
    pi = step_pi(list_q(sc, ptr), ptr)
    # reach, top-down by depth
    reach = np.zeros(N, np.float64)
    reach[root] = 1.0
    child_rec = np.flatnonzero(~is_father)
    frontier = np.zeros(N, bool)
    frontier[root] = True
    while True:
        sel = child_rec[frontier[owner[child_rec]]]
        if len(sel) == 0:
            break
        reach[cand[sel]] = reach[owner[sel]] * pi[sel]
        frontier = np.zeros(N, bool)
        frontier[cand[sel]] = True
    fr = np.flatnonzero(is_father)
    dist[owner[fr]] = reach[owner[fr]] * pi[fr]
    # a reachable node with an empty list (father removed, no children) voids the root
    in_tree = parent >= 0
    has_list = np.zeros(N, bool)
    has_list[owners] = True
    if np.any(in_tree & ~has_list & removed & (reach > 0)):
        return np.zeros(N, np.float64), 0
    return dist, 1
