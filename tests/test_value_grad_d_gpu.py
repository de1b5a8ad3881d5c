"""The exact discriminator gradient of the game value on the device (csrc/value_dgrad.cu, DESIGN.md section 5.4).

Bars: the gradient agrees with the "fp32" law of the host reference (tests/value_grad_d_oracle.py) per coordinate within
1e-12 of that coordinate's sum of |terms|; one-hot laws give the canonical fp32 score's bits; the positive part is the
training kernel's D gradient (gg_pair_grad_ex mode 0) over the raw pairs; the negative part agrees with the training
kernel fed with 2^20 production G-mode walks; pos / neg / ok are the bits of game_value; the gradient's bits do not depend
on the chunking, the root order, the call or a split into two calls; roots that are void, isolated or self-loop-only add
exactly 0; the trainer's dnorm field.
"""
import ctypes as C
import re

import numpy as np
import pytest

from tests import value_grad_d_oracle as dgo
from tests.golden import loader

pytestmark = pytest.mark.gpu


def _graph(name, cuda_device, hub):
    from graphgan_b200 import graph as G, sampler as S
    case = loader.load(name)
    hg = G.HostGraph(case["train_edges"], case["test_edges"], n_node=case.n)
    dg = G.DeviceGraph(hg, cuda_device)
    return case, hg, dg, S.WalkSampler(dg, hub_threshold=hub)


def _params(emb_h, bias_h, cuda_device):
    import torch
    from graphgan_b200 import sampler as S
    from oracle import canonical as can
    emb, bias_h = S.pad_embedding(emb_h, cuda_device), np.asarray(bias_h, np.float32)
    return emb, torch.as_tensor(bias_h).to(cuda_device), can.pad_rows(emb_h, int(emb.shape[1])), bias_h


def _d_pass(smp, hg, trees, emb, bias, roots, cuda_device, seed):
    import torch
    deg = torch.as_tensor(hg.degrees()[roots].astype(np.int64)).to(cuda_device)
    smp.run(emb, bias, trees, deg, True, seed=seed, pass_tag=1)


def _bits(out):
    return [x.cpu().numpy().view(np.uint8).tobytes() for x in out]


def _abi(smp, d_emb, d_bias, roots_d, dist, root_ok, grad_emb, grad_bias):
    """gg_game_value_grad_d straight through the C ABI (adds into grad_emb / grad_bias)"""
    import torch
    from graphgan_b200 import _cabi
    from graphgan_b200._cabi import ptr
    g, R, ld = smp.g, int(roots_d.shape[0]), int(d_emb.shape[1])
    nb = C.c_int64(0)
    _cabi.check(smp.lib.gg_game_value_grad_d_scratch_bytes(g.n_node, ld, R, C.byref(nb)))
    scratch = torch.empty(max(nb.value, 16), dtype=torch.uint8, device=d_emb.device)
    _cabi.check(smp.lib.gg_game_value_grad_d(g.n_node, ld, ptr(d_emb), ptr(d_bias), ptr(g.raw_indptr), ptr(g.raw_adj), R,
                                             ptr(roots_d), ptr(dist), ptr(root_ok), ptr(grad_emb), ptr(grad_bias),
                                             ptr(scratch), nb.value, None), "gg_game_value_grad_d")
    torch.cuda.synchronize()


def _check_oracle(hg, dg, smp, trees, roots, G_, D_, rows=None, device_law=False):
    """the gradient against the "fp32" oracle (on ``rows`` only, when given), and pos / neg / ok against game_value.  The
    law comes from tests/gdist_oracle, or with ``device_law`` from gg_generator_dist (bit-equal to it, DESIGN.md 5.1)."""
    (g_emb, g_bias, Eg, bg), (d_emb, d_bias, Ed, bd) = G_, D_
    out = smp.game_value_grad_d(g_emb, g_bias, d_emb, d_bias, trees)
    assert _bits(out[:3]) == _bits(smp.game_value(g_emb, g_bias, d_emb, d_bias, trees))
    gE, gb = out[3].cpu().numpy(), out[4].cpu().numpy()
    if rows is not None:
        gE, gb = gE[rows], gb[rows]
    if device_law:
        dists, oks = (x.cpu().numpy() for x in smp.distribution(g_emb, g_bias, trees))
    else:
        par = trees.parent_arrays().cpu().numpy()
        dists, oks = dgo.laws(Eg, bg, hg, roots, par, dg.d1_bits.cpu().numpy().view(np.uint32))
    wE, wb, aE, ab = dgo.grad(Ed, bd, hg, roots, dists, oks, "fp32", rows)
    assert np.all(np.abs(gE - wE) <= 1e-12 * aE) and np.all(np.abs(gb - wb) <= 1e-12 * ab), (
        np.max(np.abs(gE - wE) - 1e-12 * aE), np.max(np.abs(gb - wb) - 1e-12 * ab))
    n_emb = int(np.flatnonzero(np.abs(Ed).sum(axis=0))[-1]) + 1
    assert not gE[:, n_emb:].any()                                        # pad columns exactly 0
    assert [dgo.root_ok(hg, int(r), o) for r, o in zip(roots, oks)] == list(out[2].cpu().numpy())
    return out


def _fixture_roots(hg, k, seed):
    n = hg.n_node
    if n <= k:
        return np.arange(n, dtype=np.int32)
    top = np.argsort(-hg.degrees(), kind="stable")[:4]
    return np.unique(np.concatenate([top, np.random.RandomState(seed).choice(n, k, replace=False)])).astype(np.int32)


@pytest.mark.parametrize("hub", [0, 128])
@pytest.mark.parametrize("name", ["tiny", "rand300", "rand1200", "cagrqc"])
def test_matches_oracle(name, hub, cuda_device):
    case, hg, dg, smp = _graph(name, cuda_device, hub)
    roots = _fixture_roots(hg, 40, 1)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, np.random.RandomState(3).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(2).normal(0, 0.3, hg.n_node), cuda_device)
    out0 = _check_oracle(hg, dg, smp, trees, roots, G_, D_)               # no father entry removed
    assert out0[2].cpu().numpy().any() and out0[3].abs().sum().item() > 0
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=3)
    assert dg.d1_bits.any()
    out1 = _check_oracle(hg, dg, smp, trees, roots, G_, D_)
    assert not np.array_equal(out0[3].cpu().numpy(), out1[3].cpu().numpy())


@pytest.mark.parametrize("d", [20, 50, 100, 200, 300, 512])
def test_every_row_stride(d, cuda_device):
    from graphgan_b200 import synth
    _, hg, dg, smp = _graph("rand300", cuda_device, 0)
    n = hg.n_node
    rs = np.random.RandomState(d)
    roots = np.sort(rs.choice(np.flatnonzero(hg.degrees() > 0), 12, replace=False)).astype(np.int32)
    G_ = _params(synth.embeddings(n, d, seed=d, sigma=0.3), rs.normal(0, 0.3, n), cuda_device)
    D_ = _params(synth.embeddings(n, d, seed=d + 1, sigma=0.3), rs.normal(0, 0.3, n), cuda_device)
    out = _check_oracle(hg, dg, smp, smp.build_trees(roots), roots, G_, D_)
    assert int(out[3].shape[1]) == int(D_[0].shape[1])


def test_c3_roots_with_the_largest_hub(cuda_device):
    """C3 (power-law N = 1M, avg-deg 20, n_emb 128): the 13 828-neighbour hub (its C_k sums 1M nodes and its raw list is
    the longest), three of its neighbours and two ordinary roots, after a D pass."""
    from graphgan_b200 import graph as G, sampler as S, synth
    n, d = 1_000_000, 128
    hg = G.HostGraph(synth.power_law(n, 20, seed=0), None, n_node=n)
    deg = np.diff(hg.indptr)
    top = int(np.argmax(deg))
    assert deg[top] > 10000
    nb = hg.adj[hg.indptr[top]:hg.indptr[top + 1]]
    ordinary = np.random.RandomState(3).choice(np.flatnonzero(hg.degrees() > 0), 2, replace=False)
    roots = np.unique(np.concatenate([[top], nb[[0, len(nb) // 2, len(nb) - 1]], ordinary])).astype(np.int32)
    dg = G.DeviceGraph(hg, cuda_device)
    smp = S.WalkSampler(dg, hub_threshold=128)
    trees = smp.build_trees(roots)
    G_ = _params(synth.embeddings(n, d, seed=1), np.random.RandomState(5).normal(0, 0.1, n), cuda_device)
    D_ = _params(synth.embeddings(n, d, seed=2, sigma=0.2), np.random.RandomState(6).normal(0, 0.5, n), cuda_device)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=11)
    rows = np.unique(np.concatenate([roots, nb[:2000], np.random.RandomState(4).choice(n, 2000, replace=False)]))
    out = _check_oracle(hg, dg, smp, trees, roots, G_, D_, rows, device_law=True)
    assert out[2].cpu().numpy().all()


@pytest.mark.parametrize("d", [20, 50, 100, 200, 300, 512])
def test_one_hot_laws_give_the_canonical_score_bits(d, cuda_device):
    """One-hot dist rows fed straight to the ABI (70 roots: several root tiles at every row stride), against the gradient
    built from the C oracle's fp32 score (ggo_dot + bias) within 1e-12 relative per coordinate.  An fp32 ulp of s moves
    sigma by about 1e-7 of itself, so a score with other bits fails."""
    import torch
    from graphgan_b200 import synth
    from oracle import canonical as can
    _, hg, dg, smp = _graph("rand300", cuda_device, 0)
    n = hg.n_node
    rs = np.random.RandomState(d)
    emb, bias, E, b = _params(synth.embeddings(n, d, seed=d), rs.normal(0, 1.0, n), cuda_device)
    roots = rs.choice(np.flatnonzero(hg.degrees() > 0), 70, replace=False).astype(np.int32)
    v1 = rs.randint(0, n, roots.shape[0])
    R = roots.shape[0]
    dist = torch.zeros((R, n), dtype=torch.float64, device=cuda_device)
    dist[torch.arange(R), torch.as_tensor(v1)] = 1.0
    gE = torch.zeros(tuple(emb.shape), dtype=torch.float64, device=cuda_device)
    gb = torch.zeros(n, dtype=torch.float64, device=cuda_device)
    _abi(smp, emb, bias, torch.as_tensor(roots).to(cuda_device), dist, torch.ones(R, dtype=torch.int32, device=cuda_device),
         gE, gb)
    wE, wb, aE, ab = np.zeros(E.shape), np.zeros(n), np.zeros(E.shape), np.zeros(n)
    E64 = E.astype(np.float64)
    for k, c in enumerate(roots):
        lo, hi = hg.raw_indptr[c], hg.raw_indptr[c + 1]
        m = np.bincount(hg.raw_adj[lo:hi], minlength=n).astype(np.float64)
        G = np.zeros(n)
        G[v1[k]] = 1.0
        for v in np.flatnonzero((m > 0) | (G > 0)):
            s = float(np.float32(can.dot_c(E[c], E[v]) + np.float32(b[v])))
            sp, sn = (float(x) for x in dgo.sigmoids(s))
            wp, wn = m[v] * sn / float(hi - lo), G[v] * sp
            w, p = wp - wn, abs(wp) + abs(wn)
            wb[v] += w
            ab[v] += p
            wE[v] += w * E64[c]
            aE[v] += p * np.abs(E64[c])
            wE[c] += w * E64[v]
            aE[c] += p * np.abs(E64[v])
    gE, gb = gE.cpu().numpy(), gb.cpu().numpy()
    assert np.all(np.abs(gE - wE) <= 1e-12 * aE) and np.all(np.abs(gb - wb) <= 1e-12 * ab), d
    assert not gE[:, d:].any()


def _pair_grad(lib, dev, ci, vi, label, emb, bias):
    """gg_pair_grad_ex(mode 0, lambda 0) of the pairs (ci, vi, label) -> dense fp64 (grad_rows [N, ld], grad_bias [N])"""
    import torch
    from graphgan_b200 import _cabi
    from graphgan_b200._cabi import ptr
    B, (n, ld) = len(ci), emb.shape
    i = torch.as_tensor(np.asarray(ci, np.int32)).to(dev)
    j = torch.as_tensor(np.asarray(vi, np.int32)).to(dev)
    aux = torch.full((B,), float(label), dtype=torch.float32, device=dev)
    nu = torch.zeros(1, dtype=torch.int32, device=dev)
    ids = torch.empty(2 * B, dtype=torch.int32, device=dev)
    rows = torch.empty((2 * B, ld), dtype=torch.float32, device=dev)
    gb = torch.empty(2 * B, dtype=torch.float32, device=dev)
    slot = torch.full((n,), -1, dtype=torch.int32, device=dev)
    nb = C.c_int64(0)
    _cabi.check(lib.gg_pair_grad_scratch_bytes(B, ld, C.byref(nb)))
    scratch = torch.empty(max(nb.value, 256), dtype=torch.uint8, device=dev)
    _cabi.check(lib.gg_pair_grad_ex(0, B, 0, ptr(i), ptr(j), ptr(aux), ptr(emb), ptr(bias), ld, 0.0, ptr(nu), ptr(ids),
                                    ptr(rows), ptr(gb), ptr(slot), ptr(scratch), nb.value, 0, None), "gg_pair_grad_ex")
    U = int(nu.item())
    dE = torch.zeros((n, ld), dtype=torch.float64, device=dev)
    db = torch.zeros(n, dtype=torch.float64, device=dev)
    dE[ids[:U].long()] = rows[:U].double()
    db[ids[:U].long()] = gb[:U].double()
    return dE, db


def test_positive_part_is_the_training_kernels_gradient(cuda_device):
    """Zero dist rows with root_ok = 1: the gradient is -1 / deg_c times the D step's gradient (gg_pair_grad_ex, mode 0,
    lambda 0) over the root's raw pairs with label 1, to within that kernel's fp32 rounding.  The scores are moderate
    (s around -1), so its fp32 sigma(s) - 1 does not cancel."""
    import torch
    from graphgan_b200 import synth
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 0)
    n = hg.n_node
    emb, bias, E, b = _params(synth.embeddings(n, 50, seed=9, sigma=0.15), np.random.RandomState(9).normal(-1.0, 0.3, n),
                              cuda_device)
    deg = hg.degrees()
    roots = np.concatenate([np.argsort(-deg, kind="stable")[:2],
                            np.random.RandomState(8).choice(np.flatnonzero(deg > 0), 4, replace=False)]).astype(np.int32)
    for c in roots:
        one = torch.as_tensor([c], dtype=torch.int32).to(cuda_device)
        gE = torch.zeros(tuple(emb.shape), dtype=torch.float64, device=cuda_device)
        gb = torch.zeros(n, dtype=torch.float64, device=cuda_device)
        _abi(smp, emb, bias, one, torch.zeros((1, n), dtype=torch.float64, device=cuda_device),
             torch.ones(1, dtype=torch.int32, device=cuda_device), gE, gb)
        nb = hg.neighbors(int(c))
        pE, pb = _pair_grad(smp.lib, cuda_device, np.full(len(nb), c), nb, 1, emb, bias)
        want_E, want_b = (-pE / len(nb)).cpu().numpy(), (-pb / len(nb)).cpu().numpy()
        _, _, aE, ab = dgo.grad(E, b, hg, [c], np.zeros((1, n)), [1], "fp32")
        assert np.abs(gb.cpu().numpy()).sum() > 0
        assert np.all(np.abs(gE.cpu().numpy() - want_E) <= 1e-5 * aE + 1e-30), int(c)
        assert np.all(np.abs(gb.cpu().numpy() - want_b) <= 1e-5 * ab + 1e-30), int(c)


def test_negative_part_against_the_training_step_over_production_walks(cuda_device):
    """2^20 G-mode walks of four CA-GrQc roots from the production sampler (after a D pass): their stop nodes as label-0
    pairs through gg_pair_grad_ex (mode 0, lambda 0) in 64 batches per root.  The batch means, projected on 8 random
    directions, estimate minus the exact negative part (the gradient with the law less the gradient without it):
    |z| < 5 with z from the batch means' spread."""
    import torch
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    roots = np.argsort(-hg.degrees(), kind="stable")[[0, 5, 40, 200]].astype(np.int32)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, np.random.RandomState(12).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(10).normal(0, 0.3, hg.n_node), cuda_device)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=21)
    per_root, n_batch = 1 << 18, 64
    out = smp.run(G_[0], G_[1], trees, per_root, False, seed=23, pass_tag=5)
    samples = out.samples.cpu().numpy()
    dist, root_ok = smp.distribution(G_[0], G_[1], trees)
    n, ld = hg.n_node, int(D_[0].shape[1])
    n_emb = case.emb_d.shape[1]
    rs = np.random.RandomState(31)
    dirs = []
    for _ in range(8):
        dE = np.zeros((n, ld))
        dE[:, :n_emb] = rs.normal(0, 1, (n, n_emb))
        dirs.append((torch.as_tensor(dE).to(cuda_device), torch.as_tensor(rs.normal(0, 1, n)).to(cuda_device)))
    for k, c in enumerate(roots):
        assert int(root_ok[k].item()) == 1
        one = torch.as_tensor([c], dtype=torch.int32).to(cuda_device)
        grads = []
        for law in (dist[k:k + 1].contiguous(), torch.zeros((1, n), dtype=torch.float64, device=cuda_device)):
            gE = torch.zeros((n, ld), dtype=torch.float64, device=cuda_device)
            gb = torch.zeros(n, dtype=torch.float64, device=cuda_device)
            _abi(smp, D_[0], D_[1], one, law, root_ok[k:k + 1].contiguous(), gE, gb)
            grads.append((gE, gb))
        negE, negb = grads[0][0] - grads[1][0], grads[0][1] - grads[1][1]
        v = samples[k * per_root:(k + 1) * per_root]
        assert np.all(v >= 0)
        means = np.zeros((n_batch, len(dirs)))
        bs = per_root // n_batch
        for t in range(n_batch):
            pE, pb = _pair_grad(smp.lib, cuda_device, np.full(bs, c), v[t * bs:(t + 1) * bs], 0, D_[0], D_[1])
            for q, (dE, db) in enumerate(dirs):
                means[t, q] = float((pE * dE).sum() + (pb * db).sum()) / bs
        for q, (dE, db) in enumerate(dirs):
            exact = -float((negE * dE).sum() + (negb * db).sum())
            z = (means[:, q].mean() - exact) / (means[:, q].std(ddof=1) / np.sqrt(n_batch))
            print("root %d: exact %.6g, estimate %.6g, z = %.2f" % (c, exact, means[:, q].mean(), z))
            assert abs(z) < 5


def test_bits_do_not_depend_on_chunks_order_call_or_split(cuda_device):
    import torch
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    roots = _fixture_roots(hg, 60, 4)
    roots = np.concatenate([roots, roots[:3]])                          # duplicates count twice
    G_ = _params(case.emb_g, case.bias_g, cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(7).normal(0, 0.3, hg.n_node), cuda_device)
    trees = smp.build_trees(roots)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=8)
    args = (G_[0], G_[1], D_[0], D_[1])
    base = _bits(smp.game_value_grad_d(*args, trees))
    assert _bits(smp.game_value_grad_d(*args, trees)) == base                             # repeated call
    assert _bits(smp.game_value_grad_d(*args, trees, max_scratch_bytes=1)) == base        # one root per chunk
    N, nnz, ld = hg.n_node, len(hg.adj), int(D_[0].shape[1])
    per = []
    for fn, a in ((smp.lib.gg_generator_dist_scratch_bytes, (N, nnz, 1)), (smp.lib.gg_game_value_scratch_bytes, (N, 1)),
                  (smp.lib.gg_game_value_grad_d_scratch_bytes, (N, ld, 1))):
        nb = C.c_int64(0)
        fn(*a, C.byref(nb))
        per.append(nb.value)
    assert _bits(smp.game_value_grad_d(*args, trees, max_scratch_bytes=7 * sum(per))) == base     # 7 roots per chunk
    perm = np.random.RandomState(9).permutation(len(roots))
    out = smp.game_value_grad_d(*args, smp.build_trees(roots[perm]))
    inv = torch.as_tensor(np.argsort(perm)).to(cuda_device)
    assert _bits([x[inv] for x in out[:3]]) + _bits(out[3:]) == base                   # roots in another order
    # two ABI calls, the second continuing the first's accumulators, are one call on the concatenated sorted roots
    srt = np.sort(roots)
    st = smp.build_trees(srt)
    dist, root_ok = smp.distribution(G_[0], G_[1], st)
    roots_d = torch.as_tensor(srt).to(cuda_device)
    gE = torch.zeros(tuple(D_[0].shape), dtype=torch.float64, device=cuda_device)
    gb = torch.zeros(hg.n_node, dtype=torch.float64, device=cuda_device)
    for lo, hi in ((0, 25), (25, len(srt))):
        _abi(smp, D_[0], D_[1], roots_d[lo:hi], dist[lo:hi], root_ok[lo:hi], gE, gb)
    assert _bits([gE, gb]) == base[3:]


def test_void_isolated_and_self_loop_roots_add_nothing(cuda_device):
    """An isolated root, a root with only a self-loop and a void root (a depth-1 leaf whose father entry is removed) have
    ok = 0 and leave nonzero accumulators exactly as the other roots make them."""
    import torch
    from graphgan_b200 import graph as G, sampler as S, synth
    n0 = 3000
    edges = np.concatenate([synth.power_law(n0, 10, seed=1), [[n0 + 1, n0 + 1]]])
    n = n0 + 2
    hg = G.HostGraph(edges, None, n_node=n)
    dg = G.DeviceGraph(hg, cuda_device)
    smp = S.WalkSampler(dg, hub_threshold=128)
    good = np.sort(synth.pick_roots(hg.degrees(), 40, seed=2)).astype(np.int32)
    trees = smp.build_trees(good)
    par = trees.parent_arrays().cpu().numpy()
    void = None
    for k, r in enumerate(good):
        for e in range(hg.indptr[r], hg.indptr[r + 1]):
            a = hg.adj[e]
            if par[k][a] == r and not np.any(par[k] == a):
                void = (k, e)
                break
        if void:
            break
    assert void is not None
    bits = dg.d1_bits.cpu().numpy().view(np.uint32).copy()
    bits[void[1] >> 5] |= np.uint32(1) << np.uint32(void[1] & 31)
    dg.d1_bits.copy_(torch.as_tensor(bits.view(np.int32)).to(cuda_device))
    G_ = _params(synth.embeddings(n, 64, seed=3), np.zeros(n), cuda_device)
    D_ = _params(synth.embeddings(n, 64, seed=4), np.random.RandomState(5).normal(0, 0.3, n), cuda_device)
    args = (G_[0], G_[1], D_[0], D_[1])
    rest = np.delete(good, void[0])
    want = smp.game_value_grad_d(*args, smp.build_trees(rest))
    roots = np.concatenate([good, [n0, n0 + 1]]).astype(np.int32)
    out = smp.game_value_grad_d(*args, smp.build_trees(roots))
    ok = out[2].cpu().numpy()
    bad = np.zeros(len(roots), bool)
    bad[[void[0], len(roots) - 2, len(roots) - 1]] = True
    assert not ok[bad].any() and ok[~bad].all()
    assert _bits(out[3:]) == _bits(want[3:])
    alone = smp.game_value_grad_d(*args, smp.build_trees(roots[bad]))
    assert not alone[3].any() and not alone[4].any()
    # the bad roots on top of a previous result change no bit of it, even where the law or a raw list is not zero
    bad_t = smp.build_trees(roots[bad])
    dist, root_ok = smp.distribution(G_[0], G_[1], bad_t)
    gE, gb = want[3].clone(), want[4].clone()
    _abi(smp, D_[0], D_[1], bad_t.roots, dist, root_ok, gE, gb)
    assert _bits([gE, gb]) == _bits(want[3:])


def _train(monkeypatch, tmp_path, cuda_device, flags, tag):
    from graphgan_b200 import config, graph as G
    from graphgan_b200.graph_gan import GraphGAN
    c = loader.load("cagrqc")
    for k, v in dict(n_emb=50, n_epochs=1, n_epochs_dis=1, dis_interval=1, n_epochs_gen=1, gen_interval=1,
                     n_sample_gen=2, device=str(cuda_device), seed=5, value_roots=16, value_grad=flags[0],
                     value_grad_d=flags[1], text_embeddings=False).items():
        monkeypatch.setattr(config, k, v)

    def wr(name, e):
        p = tmp_path / name
        p.write_text("".join("%d\t%d\n" % (a, b) for a, b in e))
        return str(p)
    monkeypatch.setattr(config, "test_filename", wr("test.txt", c.test_edges))
    monkeypatch.setattr(config, "test_neg_filename", wr("test_neg.txt", c.test_neg_edges))
    monkeypatch.setattr(config, "emb_filenames", [str(tmp_path / ("gen%s.emb" % tag)), str(tmp_path / ("dis%s.emb" % tag))])
    monkeypatch.setattr(config, "result_filename", str(tmp_path / ("res%s.txt" % tag)))
    monkeypatch.setattr(config, "model_log", str(tmp_path / "log") + "/")
    hg = G.HostGraph(c.train_edges, c.test_edges)
    gan = GraphGAN(host_graph=hg, node_embed_init_d=c.emb_d, node_embed_init_g=c.emb_g)
    gan.train()
    return gan, (tmp_path / ("res%s.txt" % tag)).read_text().splitlines()


def test_trainer_dnorm(cuda_device, tmp_path, monkeypatch):
    """One short CA-GrQc epoch with value_roots = 16: with value_grad_d the value line ends in dnorm, after gnorm when both
    flags are on, and the earlier fields are the bits of the line without it; everything else in the result file is the
    same."""
    import torch
    gan, lines_d = _train(monkeypatch, tmp_path, cuda_device, (False, True), "d")
    _, lines_gd = _train(monkeypatch, tmp_path, cuda_device, (True, True), "gd")
    _, lines_g = _train(monkeypatch, tmp_path, cuda_device, (True, False), "g")
    _, lines0 = _train(monkeypatch, tmp_path, cuda_device, (False, False), "0")
    assert [ln.split(":")[0] for ln in lines_d] == ["gen", "dis", "value"] * 2
    pat = re.compile(r"^(value:\S+ pos:\S+ neg:\S+ roots:\d+(?: gnorm:\S+)?) dnorm:(\S+)$")
    for ln_d, ln_gd, ln_g, ln0 in zip(lines_d, lines_gd, lines_g, lines0):
        if not ln0.startswith("value:"):
            assert ln_d == ln_gd == ln_g == ln0
            continue
        m, mg = pat.match(ln_d), pat.match(ln_gd)
        assert m and mg, (ln_d, ln_gd)
        assert m.group(1) == ln0 and mg.group(1) == ln_g and mg.group(2) == m.group(2)
        assert np.isfinite(float(m.group(2))) and float(m.group(2)) > 0
    pos, neg, ok, gE, gb = gan.game_value_grad_d(gan.value_roots())
    n = int(ok.sum().item())
    want = float(torch.sqrt((gE[:, :gan.discriminator.n_emb] ** 2).sum() + (gb ** 2).sum()).item()) / n
    assert abs(float(pat.match(lines_d[5]).group(2)) - want) <= 1e-12 * want
