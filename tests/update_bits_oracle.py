"""TEST INFRASTRUCTURE ONLY: the training updates (K2 sparse gradient, K3 Adam, the step loops) on the host, with the
kernels' own fp32 operation order, so that the device must match it bit for bit.

It restates oracle/updates.py (the TF 1.8 semantics) with one change: the pair score is the canonical 8-lane fma dot
(tests/gdist_oracle.dots, pinned to ggo_dot) instead of np.sum.  After the score every step is an explicit fp32 op
sequence on the device, and the same sequence here:

    s      = f32(dot(E[i], E[j]) + b[j])                       one rounding, as __fadd_rn
    p      = f32(1 / (1 + exp(-f64(s))))                        the sigmoid in fp64, rounded once
    delta  = p - label                                          D mode (discriminator.py:26-27)
           = -(r / f32(batch_total)) * (1 - p)  if p >= 1e-5f   G mode (generator.py:26-28), else 0
    term   = f32(f32(delta * other[c]) + f32(lam * own[c]))    GG_ACC: mul, mul, add, no contraction
    g[u,c] = (((+0 + term_0) + term_1) + ...)                   one chain per coordinate over the slot's entries:
                                                                i-side entries in pair order, then j-side ones
    gb[u]  = the same chain over the j-side entries of delta (+ f32(lam * b[row]) in D mode)
    Adam   = GG_ADAM1 (m, v, then the variable), for every row; rows without a gradient take g = 0
    lr_t   = f32(f32(lr * sqrt(f32(1 - b2^t))) / f32(1 - b1^t));  b^t <- f32(b^t * b)

Slots are numbered in first-occurrence order over the entries (i-side first).  The fp64 exp of CUDA and of glibc can
differ by an ulp; ``sigmoid`` flags the pairs whose p64 lies so close to an fp32 rounding boundary that such a
difference could move p, and every test asserts that its inputs have none.

Values are compared by value (-0 == +0) with no NaN: the kernel's m * b1 + (1 - b1) * 0 turns -0 into +0 where an
in-place m *= b1 keeps -0, the one place where a correct implementation may differ in the bits.
"""
import numpy as np

from graphgan_b200.parallel import block_range
from tests import gdist_oracle as go

F = np.float32
AMBIG = 8.0 * 2.0 ** -53          # relative width of the fp64 sigmoid's uncertainty (a 1-ulp exp gap, with room)
CLIP = F(1e-5)


def pad(emb, ld):
    """[N, n_emb] -> zero-padded float32 [N, ld] (the device layout)."""
    emb = np.asarray(emb, np.float64).astype(F)
    out = np.zeros((emb.shape[0], ld), F)
    out[:, :emb.shape[1]] = emb
    return out


def score(E, b, i, j):
    """Canonical fp32 score of the pairs (i, j): E padded float32 [N, ld], b float32 [N]."""
    i, j = np.asarray(i, np.int64), np.asarray(j, np.int64)
    return (go.dots(E, i, j) + np.asarray(b, F)[j]).astype(F)


def ambiguous(p64):
    """True where p64 (1 - 8 * 2^-53) and p64 (1 + 8 * 2^-53) round to different fp32 values: an fp32 rounding boundary
    lies so close to p64 that a 1-ulp difference in exp could move the rounded p."""
    p64 = np.asarray(p64, np.float64)
    return (p64 * (1.0 - AMBIG)).astype(F) != (p64 * (1.0 + AMBIG)).astype(F)


def sigmoid(s):
    """(p, ambiguous): p = f32(1 / (1 + exp(-s))) from fp64, and the pairs where that rounding is not certain."""
    with np.errstate(over="ignore"):                       # exp(-s) = inf below s = -709.78: p = 0, as on the device
        p64 = 1.0 / (1.0 + np.exp(-np.asarray(s, F).astype(np.float64)))
    return p64.astype(F), ambiguous(p64)


def avoid_ambiguous(E, b, i, j):
    """j with every pair whose sigmoid is ambiguous moved to the next row (mod N), until none is.  Scores near 0 hit
    this often: sigma(s) = 1/2 + s/4 - s^3/48, and s/4 of a small fp32 s is often a midpoint between fp32 values near
    1/2, so the rounding of p is decided by the s^3 term, below the error of an fp64 exp."""
    j = np.array(j, copy=True)
    while True:
        amb = sigmoid(score(E, b, i, j))[1]
        if not amb.any():
            return j
        j[amb] = (j[amb] + 1) % E.shape[0]


def delta(mode, s, aux, batch_total):
    """dL/dscore (fp32) and the ambiguity mask of the sigmoid."""
    p, amb = sigmoid(s)
    a = np.asarray(aux, F)
    if mode == 0:
        return (p - a).astype(F), amb
    d = (-(a / F(batch_total)) * (F(1) - p)).astype(F)
    return np.where(p >= CLIP, d, F(0)).astype(F), amb


def slots(ids):
    """(uniq_ids in first-occurrence order, slot of every entry, rank of every entry within its slot)."""
    ids = np.asarray(ids, np.int64)
    u, first, inv = np.unique(ids, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    slot_of = np.empty(len(u), np.int64)
    slot_of[order] = np.arange(len(u))
    slot = slot_of[inv.reshape(-1)]
    srt = np.argsort(slot, kind="stable")                # entries grouped by slot, entry order inside a slot
    start = np.zeros(len(u) + 1, np.int64)
    np.cumsum(np.bincount(slot, minlength=len(u)), out=start[1:])
    rank = np.empty(len(ids), np.int64)
    rank[srt] = np.arange(len(ids)) - start[slot[srt]]
    return ids[np.sort(first)], slot, rank


def grad(mode, i, j, aux, E, b, lam, batch_total=None):
    """The mini-batch gradient -> (uniq_ids, row_slot [N], grad_rows [U, ld], grad_bias [U], ambiguous [B]).

    One fp32 chain per (slot, coordinate) in entry order, vectorised by rank: a slot holds at most one entry of a given
    rank, so one vector add per rank advances every chain by one step."""
    i, j = np.asarray(i, np.int64), np.asarray(j, np.int64)
    B = len(i)
    E, b, lam = np.asarray(E, F), np.asarray(b, F), F(lam)
    d, amb = delta(mode, score(E, b, i, j), aux, B if not batch_total else batch_total)
    ids = np.concatenate([i, j])
    other = np.concatenate([j, i])
    dd = np.concatenate([d, d])
    uniq, slot, rank = slots(ids)
    U = len(uniq)
    rows = np.zeros((U, E.shape[1]), F)
    gb = np.zeros(U, F)
    by_rank = np.argsort(rank, kind="stable")
    cut = np.searchsorted(rank[by_rank], np.arange(int(rank.max()) + 2))
    for r in range(int(rank.max()) + 1):
        t = by_rank[cut[r]:cut[r + 1]]
        term = ((dd[t, None] * E[other[t]]).astype(F) + (lam * E[ids[t]]).astype(F)).astype(F)
        rows[slot[t]] = (rows[slot[t]] + term).astype(F)
        t = t[t >= B]
        bt = dd[t] if mode == 1 else (dd[t] + (lam * b[ids[t]]).astype(F)).astype(F)
        gb[slot[t]] = (gb[slot[t]] + bt).astype(F)
    row_slot = np.full(E.shape[0], -1, np.int32)
    row_slot[uniq] = np.arange(U, dtype=np.int32)
    return uniq.astype(np.int32), row_slot, rows, gb, amb


def grad_literal(mode, i, j, aux, E, b, lam, batch_total=None):
    """The same gradient as a literal per-entry loop of np.float32 scalars (the statement ``grad`` must equal)."""
    i, j = [int(x) for x in i], [int(x) for x in j]
    B = len(i)
    E, b, lam = np.asarray(E, F), np.asarray(b, F), F(lam)
    d, _ = delta(mode, score(E, b, i, j), aux, B if not batch_total else batch_total)
    uniq, pos = [], {}
    for r in i + j:
        if r not in pos:
            pos[r] = len(uniq)
            uniq.append(r)
    rows = np.zeros((len(uniq), E.shape[1]), F)
    gb = np.zeros(len(uniq), F)
    for t in range(2 * B):
        k, side_j = t % B, t >= B
        me, ot = (j[k], i[k]) if side_j else (i[k], j[k])
        u = pos[me]
        for c in range(E.shape[1]):
            rows[u, c] = F(rows[u, c] + F(F(d[k] * E[ot, c]) + F(lam * E[me, c])))
        if side_j:
            gb[u] = F(gb[u] + (d[k] if mode == 1 else F(d[k] + F(lam * b[me]))))
    return np.asarray(uniq, np.int32), rows, gb


def lr_t(lr, b1p, b2p):
    one = F(1)
    return F(F(F(lr) * np.sqrt(F(one - F(b2p)))) / F(one - F(b1p)))


class Adam:
    """Dense TF 1.8 Adam over (E, b) in the GG_ADAM1 order, with fp32 beta powers."""

    def __init__(self, n, ld, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8):
        self.lr, self.b1, self.b2, self.eps = F(lr), F(beta1), F(beta2), F(eps)
        self.m_e, self.v_e = np.zeros((n, ld), F), np.zeros((n, ld), F)
        self.m_b, self.v_b = np.zeros(n, F), np.zeros(n, F)
        self.b1p, self.b2p = F(beta1), F(beta2)

    def lr_t(self):
        return lr_t(self.lr, self.b1p, self.b2p)

    def apply(self, E, b, uniq, g_rows, g_bias, lr=None):
        """One step in place; rows outside ``uniq`` take g = 0.  lr: the lr_t to use (default: from the beta powers)."""
        lt = self.lr_t() if lr is None else F(lr)
        G = np.zeros_like(E)
        G[uniq] = g_rows
        gb = np.zeros_like(b)
        gb[uniq] = g_bias
        for x, m, v, g in ((E, self.m_e, self.v_e, G), (b, self.m_b, self.v_b, gb)):
            adam1(x, m, v, g, lt, self.b1, self.b2, self.eps)
        self.b1p, self.b2p = F(self.b1p * self.b1), F(self.b2p * self.b2)


def adam1(x, m, v, g, lt, b1, b2, eps):
    """GG_ADAM1 elementwise, in place: m = m b1 + (1 - b1) g; v = v b2 + (g g)(1 - b2); x -= lt m / (sqrt(v) + eps)."""
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        m[...] = ((m * b1).astype(F) + (F(F(1) - b1) * g).astype(F)).astype(F)
        v[...] = ((v * b2).astype(F) + ((g * g).astype(F) * F(F(1) - b2)).astype(F)).astype(F)
        x[...] = (x - ((F(lt) * m).astype(F) / (np.sqrt(v).astype(F) + F(eps)).astype(F)).astype(F)).astype(F)


class Model:
    """Parameters + Adam of one pair model (the device PairModel's state, padded to ld)."""

    def __init__(self, emb, ld, bias=None, lr=1e-3, lam=1e-5):
        self.E = pad(emb, ld)
        self.b = np.zeros(self.E.shape[0], F) if bias is None else np.asarray(bias, F).copy()
        self.lam = F(lam)
        self.adam = Adam(self.E.shape[0], ld, lr)

    def state(self):
        a = self.adam
        return {"emb": self.E, "bias_t": self.b, "m_emb": a.m_e, "v_emb": a.v_e, "m_bias": a.m_b, "v_bias": a.v_b}

    def step(self, mode, i, j, aux, batch_total=None):
        """One optimizer step; returns the ambiguity mask of the batch."""
        uniq, _, rows, gb, amb = grad(mode, i, j, aux, self.E, self.b, self.lam, batch_total)
        self.adam.apply(self.E, self.b, uniq, rows, gb)
        return amb

    def steps(self, mode, i, j, aux, starts, batch_size):
        """The step loop over a start list (a short last batch where a start is within batch_size of the end)."""
        amb = np.zeros(0, bool)
        for s0 in starts:
            amb = np.concatenate([amb, self.step(mode, i[s0:s0 + batch_size], j[s0:s0 + batch_size], aux[s0:s0 + batch_size])])
        return amb

    def world_step(self, mode, i, j, aux, world):
        """A data-parallel step of `world` ranks: each rank's block_range slice with batch_total = B, the rank-major
        merge (one fp32 add chain per slot over the ranks in order, from +0), then Adam."""
        B = len(i)
        blocks, amb = [], np.zeros(0, bool)
        for r in range(world):
            lo, hi = block_range(B, r, world)
            if hi == lo:
                continue
            u, _, rows, gb, a = grad(mode, i[lo:hi], j[lo:hi], aux[lo:hi], self.E, self.b, self.lam, batch_total=B)
            blocks.append((u, rows, gb))
            amb = np.concatenate([amb, a])
        uniq, rows, gb = merge(blocks, self.E.shape[0], self.E.shape[1])
        self.adam.apply(self.E, self.b, uniq, rows, gb)
        return amb


def merge(blocks, n, ld):
    """The rank-major merge: slots by first occurrence over the blocks in order, fp32 adds from +0 in rank order (a rank
    holds an id at most once, so one vector add per rank is one step of every chain)."""
    ids = np.concatenate([bl[0] for bl in blocks]) if blocks else np.zeros(0, np.int32)
    _, first = np.unique(ids, return_index=True)
    uniq = ids[np.sort(first)]
    slot = np.full(n, -1, np.int64)
    slot[uniq] = np.arange(len(uniq))
    rows = np.zeros((len(uniq), ld), F)
    gb = np.zeros(len(uniq), F)
    for u, r, g in blocks:
        s = slot[u]
        rows[s] = (rows[s] + r).astype(F)
        gb[s] = (gb[s] + g).astype(F)
    return uniq.astype(np.int32), rows, gb


def same(got, want):
    """Equal by value (-0 == +0) and no NaN on either side."""
    got, want = np.asarray(got), np.asarray(want)
    return got.shape == want.shape and not np.isnan(got).any() and not np.isnan(want).any() and np.array_equal(got, want)
