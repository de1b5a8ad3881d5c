"""Host tests of tests/update_bits_oracle.py, the canonical-score statement of the training updates that
tests/test_update_bits_gpu.py holds the kernels to bit for bit.  No GPU needed."""
import math

import numpy as np
import pytest

from oracle import updates
from tests import update_bits_oracle as ub

F = np.float32
U32 = 2.0 ** -24          # unit roundoff of fp32


def gamma(k):
    return k * U32 / (1.0 - k * U32)


def _batch(rs, n, B):
    """Random pairs with a duplicate pair, a self pair, a row on both sides and a row repeated through the batch."""
    i, j = rs.randint(0, n, B), rs.randint(0, n, B)
    if B >= 6:
        i[3], j[3] = i[0], j[0]
        j[5] = i[5]
        i[1] = j[2]
        i[B // 2:] = i[B // 2]
    return i.astype(np.int64), j.astype(np.int64)


def _model(rs, n, d, ld):
    E = ub.pad(rs.normal(0, 0.5, size=(n, d)), ld)
    b = rs.normal(0, 0.3, size=n).astype(F)
    return E, b


@pytest.mark.parametrize("ld", [32, 64, 128, 256, 512])
def test_score_is_the_c_oracles_dot_plus_bias(ld):
    from oracle import canonical as can
    rs = np.random.RandomState(ld)
    E, b = _model(rs, 64, ld - 3, ld)
    E[:8] *= F(1e3)
    i, j = rs.randint(0, 64, 300), rs.randint(0, 64, 300)
    got = ub.score(E, b, i, j)
    want = np.array([F(can.dot_c(E[p], E[q]) + b[q]) for p, q in zip(i, j)], F)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("ld,B", [(32, 1), (32, 7), (64, 33), (128, 16), (512, 9)])
def test_vectorised_gradient_equals_a_literal_loop(mode, ld, B):
    rs = np.random.RandomState(10 * ld + B + mode)
    n = 12
    E, b = _model(rs, n, ld - 5, ld)
    i, j = _batch(rs, n, B)
    aux = ((rs.random_sample(B) < 0.5) if mode == 0 else rs.random_sample(B) * 3).astype(F)
    if B > 2:
        aux[2] = 0                                             # a reward (or label) of 0
    for bt in (None, 3 * B):
        uniq, row_slot, rows, gb, amb = ub.grad(mode, i, j, aux, E, b, 1e-5, bt)
        lu, lrows, lgb = ub.grad_literal(mode, i, j, aux, E, b, 1e-5, bt)
        assert not amb.any()
        assert np.array_equal(uniq, lu)
        assert np.array_equal(row_slot[uniq], np.arange(len(uniq))) and (row_slot >= 0).sum() == len(uniq)
        assert np.array_equal(rows.view(np.int32), lrows.view(np.int32))
        assert np.array_equal(gb.view(np.int32), lgb.view(np.int32))


def _anchor(mode, i, j, aux, E, b, lam, ld):
    """(g32 rows, g32 bias, bound rows, bound bias, fp64 rows, fp64 bias, number of straddling pairs)."""
    uniq, _, rows, gb, amb = ub.grad(mode, i, j, aux, E, b, lam)
    assert not amb.any()
    B = len(i)
    E64, b64, lam64 = E.astype(np.float64), b.astype(np.float64), float(F(lam))
    prod = E64[i] * E64[j]
    s64 = prod.sum(1) + b64[j]
    mag = np.abs(prod).sum(1) + np.abs(b64[j])
    ds = gamma(ld // 8 + 4) * mag * (1 + 2.0 ** -40)          # |s32 - s| (ld / 8 fmas, 3 butterfly adds, the bias add)
    lo, hi = s64 - ds, s64 + ds
    sig = lambda x: 1.0 / (1.0 + np.exp(-x))
    near = np.where((lo <= 0) & (hi >= 0), 0.0, np.where(np.abs(lo) < np.abs(hi), lo, hi))
    dmax = sig(near) * (1 - sig(near))                         # max sigma' on [lo, hi]
    p64 = sig(s64)
    a = aux.astype(np.float64)
    straddle = np.zeros(B, bool)
    if mode == 0:
        d64 = p64 - a
        dd = dmax * ds + 2 * U32                               # + the roundings of p and of p - label
    else:
        scale = np.abs(a) / B
        logit = math.log(1e-5 / (1 - 1e-5))
        straddle = (lo <= logit) & (hi >= logit)
        d64 = np.where(p64 >= 1e-5, -(a / B) * (1 - p64), 0.0)
        dd = scale * (dmax * ds + 4 * U32)                     # p, 1 - p, r / B and the product
        d32 = ub.delta(mode, ub.score(E, b, i, j), aux, B)[0].astype(np.float64)
        dd = np.where(straddle, np.abs(d32) + np.abs(d64) + dd, dd)   # either side of the clip is right
    N = E.shape[0]
    g64, tabs, dsum = np.zeros((N, ld)), np.zeros((N, ld)), np.zeros((N, ld))
    gb64, babs, bdsum = np.zeros(N), np.zeros(N), np.zeros(N)
    cnt = np.zeros(N, np.int64)
    for k in range(B):
        for me, ot in ((i[k], j[k]), (j[k], i[k])):
            t1, t2 = d64[k] * E64[ot], lam64 * E64[me]
            g64[me] += t1 + t2
            tabs[me] += np.abs(t1) + np.abs(t2)
            dsum[me] += dd[k] * np.abs(E64[ot])
            cnt[me] += 1
        bt = d64[k] + (lam64 * b64[j[k]] if mode == 0 else 0.0)
        gb64[j[k]] += bt
        babs[j[k]] += abs(d64[k]) + (abs(lam64 * b64[j[k]]) if mode == 0 else 0.0)
        bdsum[j[k]] += dd[k]
    gam = np.array([gamma(c + 3) for c in cnt])
    slack = 2.0 ** -45
    bound = gam[:, None] * tabs + dsum + slack * (tabs + dsum)
    bbound = gam * babs + bdsum + slack * (babs + bdsum)
    return uniq, rows, gb, bound[uniq], bbound[uniq], g64[uniq], gb64[uniq], int(straddle.sum())


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("ld", [32, 128, 512])
def test_gradient_within_the_fp64_bound(mode, ld):
    """Each coordinate of the fp32 gradient against the same gradient in fp64 from the same fp32 parameters:
        |g32 - g64| <= gamma_{n+3} sum|terms| + sum_k |d delta_k| |other_k|.
    The chain of a slot with n entries is n adds of terms that are each rounded three times (two products, one add), so
    the arithmetic error is at most gamma_{n+3} times the sum of the terms' magnitudes (Higham, Lemma 3.1 / 3.3).  delta
    itself comes from the fp32 score: the canonical dot is ld / 8 fma roundings per lane, three butterfly adds and the
    bias add, so |s32 - s| <= gamma_{ld/8+4} (sum |e_i e_j| + |b_j|); through the sigmoid that moves delta by at most
    max sigma' on the interval times that, plus the roundings of p and of the D or G formula.  In G mode a pair whose score
    interval holds logit(1e-5) may land on either side of the clip; the test builds exactly four such pairs (a zero
    row i and a bias b_j at logit(1e-5) and its neighbours) and checks that no other pair straddles."""
    rs = np.random.RandomState(ld + mode)
    n, B = 40, 200
    E, b = _model(rs, n, ld - 1, ld)
    i, j = _batch(rs, n, B)
    aux = ((rs.random_sample(B) < 0.5) if mode == 0 else rs.random_sample(B) * 3).astype(F)
    built = 0
    if mode == 1:
        E[0] = 0
        c = F(math.log(1e-5 / (1 - 1e-5)))
        for k, v in enumerate((c, np.nextafter(c, F(0)), np.nextafter(c, F(-20)), np.nextafter(np.nextafter(c, F(0)), F(0)))):
            b[30 + k] = v
            i[100 + k], j[100 + k] = 0, 30 + k
            built += 1
        i[i == 0] = np.where(np.arange(B)[i == 0] >= 100, 0, 1)   # row 0 only in the built pairs
        j[(j >= 30) & (j < 34) & ((np.arange(B) < 100) | (np.arange(B) >= 104))] = 5
    uniq, rows, gb, bound, bbound, g64, gb64, straddle = _anchor(mode, i, j, aux, E, b, 1e-5, ld)
    assert straddle == built
    assert np.all(np.abs(rows - g64) <= bound)
    assert np.all(np.abs(gb - gb64) <= bbound)


@pytest.mark.parametrize("mode", [0, 1])
def test_canonical_and_np_sum_oracles_agree_within_the_score_bound(mode):
    """The new oracle differs from oracle/updates.py only in the score: both gradients sit within the fp64 bound of
    the same exact gradient, with the np.sum score's own bound (pairwise fp32 sum: at most ld roundings) in place of the
    canonical dot's.  Ties the bit-exact oracle to the TF-semantics one the close() tests keep using."""
    ld, n, B = 64, 50, 128
    rs = np.random.RandomState(5 + mode)
    E, b = _model(rs, n, ld, ld)
    i, j = _batch(rs, n, B)
    aux = ((rs.random_sample(B) < 0.5) if mode == 0 else rs.random_sample(B) * 3).astype(F)
    uniq, rows, gb, bound, bbound, g64, gb64, _ = _anchor(mode, i, j, aux, E, b, 1e-5, ld)
    cls = updates.Discriminator if mode == 0 else updates.Generator
    o = cls(n, E, 1e-3, 1e-5, bias_init=b)
    urows, grows, gbias = o.grads(i, j, aux)
    assert np.array_equal(np.asarray(urows, np.int32), uniq)
    # the np.sum score is within gamma_{ld+1} (sum |e_i e_j| + |b_j|): widen the delta part of the bound accordingly
    widen = gamma(ld + 1) / gamma(ld // 8 + 4)
    assert np.all(np.abs(grows - g64) <= bound * widen)
    assert np.all(np.abs(gbias - gb64) <= bbound * widen)
    assert np.all(np.abs(grows - rows) <= bound * (1 + widen))


def test_sigmoid_ambiguity_detector():
    """Flags p64 values within 8 * 2^-53 (relative) of an fp32 rounding boundary, on both sides, and nothing else: the
    midpoints between consecutive fp32 values near 1e-5, 0.5, 1 - 2^-25 (the last step to p = 1.0f) and 1e-30."""
    for p in (F(1e-5), F(0.3), F(1) - F(2.0 ** -24), F(1e-30)):
        mid = (float(p) + float(np.nextafter(p, F(2)))) / 2.0          # exact in fp64
        k = np.arange(-40, 41)
        x = mid * (1.0 + k * 2.0 ** -53)
        flags = ub.ambiguous(x)
        assert flags[np.abs(k) <= 6].all(), p
        assert not flags[np.abs(k) >= 10].any(), p
    rs = np.random.RandomState(1)
    p32 = rs.random_sample(100000).astype(F).astype(np.float64)       # fp32 values: the farthest from a boundary
    assert not ub.ambiguous(p32).any()
    assert not ub.ambiguous(np.array([0.0, 1.0, 1e-300])).any()


def test_no_fp32_score_lands_exactly_on_the_generator_clip():
    """p = f32(sigma(s)) never equals 1e-5f for an fp32 s: near logit(1e-5) one ulp of s moves p by about ten ulps of p,
    and the one crossing skips 1e-5f.  So the clip's `p >= 1e-5f` and `p > 1e-5f` give the same gradient on every input;
    the GPU tests pin the crossing itself."""
    c = F(math.log(1e-5 / (1 - 1e-5)))
    s = [c]
    for _ in range(4096):
        s.append(np.nextafter(s[-1], F(0)))
        s.insert(0, np.nextafter(s[0], F(-20)))
    s = np.array(s, F)
    p, amb = ub.sigmoid(s)
    assert not amb.any()
    assert not (p == ub.CLIP).any()
    assert (p < ub.CLIP).sum() > 1000 and (p > ub.CLIP).sum() > 1000
    assert np.all(np.diff(p) >= 0)


def test_adam_order_and_edges():
    """adam1 is the GG_ADAM1 sequence: against a scalar restatement, at |g| where g^2 is subnormal, rounds to 0 or
    overflows, v = 0 with g = 0 and a subnormal m; the fp32 lr_t and beta powers run into the subnormals."""
    g = np.array([0, 1e-20, -1e-23, 3e19, -1e19, 0.25, 0, 0], F)
    m = np.array([0, 0, 0, 0, 0, 1e-3, 1e-40, -0.0], F)
    v = np.array([0, 0, 0, 0, 0, 1e-6, 0, 0], F)
    x = np.full(8, 0.5, F)
    b1, b2, eps, lt = F(0.9), F(0.999), F(1e-8), F(3e-4)
    want = []
    for k in range(8):
        mm = F(F(m[k] * b1) + F(F(F(1) - b1) * g[k]))
        with np.errstate(over="ignore", under="ignore"):
            vv = F(F(v[k] * b2) + F(F(g[k] * g[k]) * F(F(1) - b2)))
        want.append((mm, vv, F(x[k] - F(F(lt * mm) / F(np.sqrt(vv) + eps)))))
    ub.adam1(x, m, v, g, lt, b1, b2, eps)
    assert ub.same(m, [w[0] for w in want]) and ub.same(v, [w[1] for w in want]) and ub.same(x, [w[2] for w in want])
    assert v[1] > 0 and v[1] < np.finfo(F).tiny                  # g^2 (1 - b2) subnormal, kept
    assert v[2] == 0 and v[3] == np.inf and x[3] == F(0.5)       # rounds to 0; overflows, the update is 0
    assert 0 < m[6] < np.finfo(F).tiny
    a = ub.Adam(1, 32)
    for _ in range(1100):
        a.b1p, a.b2p = F(a.b1p * a.b1), F(a.b2p * a.b2)
    # 0.9 * 4 * 2^-149 = 3.6 * 2^-149 rounds back to 4 * 2^-149: beta1^t stops there, it never reaches 0
    assert a.b1p == F(4 * 2.0 ** -149) and F(a.b1p * a.b1) == a.b1p and a.b2p > 0
    assert a.lr_t() == F(a.lr * np.sqrt(F(1) - a.b2p))


def test_world_step_of_one_rank_is_the_single_step():
    """world_step(world = 1) adds every row to +0 once: the single step's state by value."""
    rs = np.random.RandomState(3)
    n, ld, B = 30, 64, 50
    emb = rs.normal(0, 0.5, size=(n, 60))
    i, j = _batch(rs, n, B)
    aux = (rs.random_sample(B) * 3).astype(F)
    a, w = ub.Model(emb, ld), ub.Model(emb, ld)
    a.step(1, i, j, aux)
    w.world_step(1, i, j, aux, 1)
    for k, v in a.state().items():
        assert ub.same(w.state()[k], v), k
