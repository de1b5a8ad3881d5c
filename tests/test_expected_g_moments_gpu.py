"""The second moment of one G walk's step on the device (csrc/value_gref.cu, DESIGN.md section 5.9).

Bars: n_pairs, root_ok, grad_emb and grad_bias are the bits of expected_g_grad; sq_node, sq and mn within 1e-12 of their
sums of |terms| of the host reference (tests/expected_g_moments_oracle.py, whose decomposition the host tests tie to the
literal walk-by-walk norms, with gg_pair_reward's rewards); mn_c of a root alone is the squared norm of that root's
expected_g_grad to 1e-13; the bits do not depend on the chunking, the root order or the call; void, isolated and
self-loop-only roots add 0; the production G pass (sampler, gg_window_pairs, gg_pair_reward, gg_pair_grad_ex mode 1)
agrees per stop node and over 2^18 walks per root; the trainer's gsnr.
"""
import ctypes as C
import re

import numpy as np
import pytest

from tests import expected_g_moments_oracle as mo
from tests.test_expected_g_grad_gpu import (_bits, _d_pass, _device_reward, _fixture_roots, _graph, _pair_grad_g, _params,
                                            _train)

pytestmark = pytest.mark.gpu


def _check(hg, dg, smp, trees, roots, G_, D_, window):
    """moments against expected_g_grad's bits and the oracle; returns the moments' output"""
    (g_emb, g_bias, Eg, bg), (d_emb, d_bias, _, _) = G_, D_
    args = (g_emb, g_bias, d_emb, d_bias, trees)
    out = smp.expected_g_moments(*args, window=window, per_node=True)
    ref = smp.expected_g_grad(*args, window=window)
    assert _bits(out[:2]) + _bits(out[4:6]) == _bits(ref)
    ok, sq, mn, sq_node = (x.cpu().numpy() for x in (out[1], out[2], out[3], out[6]))
    par = trees.parent_arrays().cpu().numpy()
    bits = dg.d1_bits.cpu().numpy().view(np.uint32)
    reward = _device_reward(smp.lib, d_emb, d_bias)
    for k, r in enumerate(roots):
        o = mo.root_pairs(Eg, bg, hg, int(r), par[k], bits, window, reward)
        assert o["ok"] == ok[k]
        if not o["ok"]:
            assert sq[k] == 0 and mn[k] == 0 and not sq_node[k].any()
            continue
        pt = mo.pf_tail(Eg, o, window)
        assert np.all(np.abs(sq_node[k] - pt["sq_node"]) <= 1e-12 * pt["abs_sq"]), np.max(
            np.abs(sq_node[k] - pt["sq_node"]) - 1e-12 * pt["abs_sq"])
        assert abs(sq[k] - float((o["dist"] * pt["sq_node"]).sum())) <= 1e-12 * float((o["dist"] * pt["abs_sq"]).sum())
        want = float((o["gE"] ** 2).sum() + (o["gb"] ** 2).sum())
        assert abs(mn[k] - want) <= 1e-12 * float((o["abs_E"] ** 2).sum() + (o["abs_b"] ** 2).sum()), (mn[k], want)
        assert sq[k] - mn[k] >= -1e-12 * sq[k]
    return out


@pytest.mark.parametrize("name", ["tiny", "rand300", "rand1200", "cagrqc"])
def test_matches_grad_bits_and_oracle(name, cuda_device):
    """against the oracle with the hub cache off; with it at 128 (the same law, bit for bit) the same bits"""
    from graphgan_b200 import sampler as S
    case, hg, dg, smp = _graph(name, cuda_device, 0)
    hub = S.WalkSampler(dg, hub_threshold=128)
    roots = _fixture_roots(hg, 30, 1)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, np.random.RandomState(3).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(2).normal(0, 0.3, hg.n_node), cuda_device)
    args = (G_[0], G_[1], D_[0], D_[1], trees)
    for w in (1, 2, 3):
        out = _check(hg, dg, smp, trees, roots, G_, D_, w)
        assert out[2].abs().sum().item() > 0
        assert _bits(hub.expected_g_moments(*args, window=w, per_node=True)) == _bits(out)
    _d_pass(hub, hg, trees, G_[0], G_[1], roots, cuda_device, seed=3)
    assert dg.d1_bits.any()
    for w in (1, 2, 3) + ((8,) if name == "rand300" else ()):
        out = _check(hg, dg, smp, trees, roots, G_, D_, w)
        assert _bits(hub.expected_g_moments(*args, window=w, per_node=True)) == _bits(out)


@pytest.mark.parametrize("d", [20, 50, 100, 200, 300, 512])
def test_every_row_stride(d, cuda_device):
    from graphgan_b200 import synth
    _, hg, dg, smp = _graph("rand300", cuda_device, 0)
    n = hg.n_node
    rs = np.random.RandomState(d)
    roots = np.sort(rs.choice(np.flatnonzero(hg.degrees() > 0), 12, replace=False)).astype(np.int32)
    G_ = _params(synth.embeddings(n, d, seed=d, sigma=0.3), rs.normal(0, 0.3, n), cuda_device)
    D_ = _params(synth.embeddings(n, d, seed=d + 1, sigma=0.3), rs.normal(0, 0.3, n), cuda_device)
    _check(hg, dg, smp, smp.build_trees(roots), roots, G_, D_, 2)


def _alone(smp, args, trees, window, cuda_device):
    """mn_c of each root called alone against |that call's expected_g_grad|^2"""
    import torch
    for k in range(int(trees.roots.shape[0])):
        t = trees.select(torch.tensor([k], device=cuda_device))
        out = smp.expected_g_moments(*args, t, window=window)
        gE, gb = smp.expected_g_grad(*args, t, window=window)[2:]
        want = float((gE ** 2).sum().item() + (gb ** 2).sum().item())
        assert abs(float(out[3].item()) - want) <= 1e-13 * want, (k, float(out[3].item()), want)


def test_c3_roots_with_the_largest_hub(cuda_device):
    """C3 (power-law N = 1M, avg-deg 20, n_emb 128) at w = 2: the 13 828-neighbour hub, three of its neighbours and two
    ordinary roots, after a D pass.  The hub's row takes the big-node CTA path in every root's tree, so mn_c of each root
    alone against its step's squared norm checks that path's squared contributions; sq_node is checked at the hub, its
    tree children and 400 random reached nodes per root against the literal norm of their paths (path_sq; a whole-tree
    reference at N = 1M would take minutes per root)."""
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
    args = (G_[0], G_[1], D_[0], D_[1])
    out = smp.expected_g_moments(*args, trees, window=2, per_node=True)
    assert _bits(out[:2]) + _bits(out[4:6]) == _bits(smp.expected_g_grad(*args, trees, window=2))
    ok, sq, mn = (x.cpu().numpy() for x in out[1:4])
    assert ok.all() and np.all(sq - mn >= -1e-12 * sq)
    par = trees.parent_arrays().cpu().numpy()
    reward = _device_reward(smp.lib, D_[0], D_[1])
    rs = np.random.RandomState(8)
    for k, r in enumerate(roots):
        row = out[6][k].cpu().numpy()
        reached = np.flatnonzero(row > 0)
        ys = np.unique(np.concatenate([np.flatnonzero(par[k] == top)[:200], rs.choice(reached, 400, replace=False),
                                       [top] if top != r else []])).astype(np.int64)
        ys = ys[row[ys] > 0]
        want, ab, amb = mo.path_sq(G_[2], G_[3], par[k], ys, 2, reward)
        keep = ~amb
        assert keep.sum() > 0.9 * len(ys)
        assert np.all(np.abs(row[ys][keep] - want[keep]) <= 1e-12 * ab[keep])
        print("root %d: sq %.6g, mn %.6g, %d nodes checked" % (r, sq[k], mn[k], int(keep.sum())))
    _alone(smp, args, trees, 2, cuda_device)


def test_mn_of_a_root_alone_is_its_step_squared(cuda_device):
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    roots = _fixture_roots(hg, 12, 6)
    G_ = _params(case.emb_g, case.bias_g, cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(7).normal(0, 0.3, hg.n_node), cuda_device)
    trees = smp.build_trees(roots)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=8)
    for w in (1, 2, 3):
        _alone(smp, (G_[0], G_[1], D_[0], D_[1]), trees, w, cuda_device)


def test_bits_do_not_depend_on_chunks_order_or_call(cuda_device):
    import torch
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    roots = _fixture_roots(hg, 60, 4)
    roots = np.concatenate([roots, roots[:3]])                          # duplicates count twice
    G_ = _params(case.emb_g, case.bias_g, cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(7).normal(0, 0.3, hg.n_node), cuda_device)
    trees = smp.build_trees(roots)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=8)
    args = (G_[0], G_[1], D_[0], D_[1])
    for w in (1, 2):
        base = _bits(smp.expected_g_moments(*args, trees, window=w, per_node=True))
        assert _bits(smp.expected_g_moments(*args, trees, window=w, per_node=True)) == base
        assert _bits(smp.expected_g_moments(*args, trees, window=w, per_node=True, max_scratch_bytes=1)) == base
        nb = C.c_int64(0)
        smp.lib.gg_expected_g_moments_scratch_bytes(hg.n_node, len(hg.adj), 7, w, C.byref(nb))
        assert _bits(smp.expected_g_moments(*args, trees, window=w, per_node=True, max_scratch_bytes=nb.value)) == base
        perm = np.random.RandomState(9).permutation(len(roots))
        out = smp.expected_g_moments(*args, smp.build_trees(roots[perm]), window=w, per_node=True)
        inv = torch.as_tensor(np.argsort(perm)).to(cuda_device)
        got = _bits([x[inv] for x in out[:4]]) + _bits(out[4:6]) + _bits([out[6][inv]])
        assert got == base
        assert _bits(smp.expected_g_moments(*args, trees, window=w)) == base[:6]              # without sq_node


def test_void_isolated_and_self_loop_roots_add_nothing(cuda_device):
    """An isolated root, a root with only a self-loop and a void root (a depth-1 leaf whose father entry is removed):
    sq = mn = 0, sq_node 0, and the accumulators are the bits the other roots make"""
    import torch
    from graphgan_b200 import graph as G, sampler as S, synth
    n0 = 3000
    edges = np.concatenate([synth.power_law(n0, 10, seed=1), [[n0 + 1, n0 + 1]]])
    n = n0 + 2
    hg = G.HostGraph(edges, None, n_node=n)
    dg = G.DeviceGraph(hg, cuda_device)
    smp = S.WalkSampler(dg, hub_threshold=128)
    good = np.sort(synth.pick_roots(hg.degrees(), 40, seed=2)).astype(np.int32)
    par = smp.build_trees(good).parent_arrays().cpu().numpy()
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
    want = smp.expected_g_moments(*args, smp.build_trees(rest), window=2)
    roots = np.concatenate([good, [n0, n0 + 1]]).astype(np.int32)
    out = smp.expected_g_moments(*args, smp.build_trees(roots), window=2, per_node=True)
    ok, sq, mn, sq_node = (x.cpu().numpy() for x in (out[1], out[2], out[3], out[6]))
    bad = np.zeros(len(roots), bool)
    bad[[void[0], len(roots) - 2, len(roots) - 1]] = True
    assert not ok[bad].any() and ok[~bad].all()
    assert not sq[bad].any() and not mn[bad].any() and not sq_node[bad].any()
    assert np.all(sq[~bad] > 0) and np.all(mn[~bad] > 0)
    assert _bits(out[4:6]) == _bits(want[4:6])
    assert _bits([out[2][~torch.as_tensor(bad).to(cuda_device)]]) == _bits([want[2]])


def test_production_g_pass_per_stop_node_and_pass(cuda_device):
    """2^18 G-mode walks of each of four CA-GrQc roots from the production sampler (after a D pass), w = 2.  Every
    recorded path is the tree path root -> stop -> father.  For every distinct stop y, the production step of one walk
    (gg_window_pairs -> gg_pair_reward -> gg_pair_grad_ex mode 1, batch_total 1, lambda 0; fp32) has |s(y)|^2 within
    1e-5 of sq_node.  The walks' mean |s|^2 estimates sq_c, and passes of n = 20 walks estimate n sq_c + n (n - 1) mn_c
    through |S_pass|^2: |z| < 5 from the spread."""
    import scipy.sparse as sp
    import torch
    from graphgan_b200 import _cabi
    from graphgan_b200._cabi import ptr
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    window, n_pass = 2, 20
    roots = np.argsort(-hg.degrees(), kind="stable")[[0, 5, 40, 150]].astype(np.int32)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, np.random.RandomState(12).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(10).normal(0, 0.3, hg.n_node), cuda_device)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=21)
    per_root, max_path = 1 << 18, 64
    out = smp.run(G_[0], G_[1], trees, per_root, False, seed=23, pass_tag=5, max_path=max_path)
    assert np.all(out.status.cpu().numpy() == 1)
    n, ld = hg.n_node, int(G_[0].shape[1])
    par = trees.parent_arrays().cpu().numpy()
    mom = smp.expected_g_moments(G_[0], G_[1], D_[0], D_[1], trees, window=window, per_node=True)
    sq, mn, sq_node = mom[2].cpu().numpy(), mom[3].cpu().numpy(), mom[6].cpu().numpy()
    pair_ptr = torch.empty(2, dtype=torch.int64, device=cuda_device)
    n_out = torch.zeros(1, dtype=torch.int64, device=cuda_device)
    for k, c in enumerate(roots):
        paths = out.paths[k * per_root:(k + 1) * per_root].cpu().numpy()
        plen = out.path_len[k * per_root:(k + 1) * per_root].cpu().numpy().astype(np.int64)
        stop = paths[np.arange(per_root), plen - 2]
        assert np.all(paths[:, 0] == c) and np.all(paths[np.arange(per_root), plen - 1] == par[k][stop])
        for i in range(1, int(plen.max()) - 1):                        # body: the tree path root -> stop
            sel = plen - 2 >= i
            assert np.all(par[k][paths[sel, i]] == paths[sel, i - 1])
        ys, first, inv = np.unique(stop, return_index=True, return_inverse=True)
        rows, cols, vals, prod_sq = [], [], [], np.zeros(len(ys))
        for t, w0 in enumerate(first):
            w = k * per_root + int(w0)
            p, pl = out.paths[w:w + 1].contiguous(), out.path_len[w:w + 1].contiguous()
            _cabi.check(smp.lib.gg_window_pairs(1, ptr(p), ptr(pl), max_path, window, ptr(pair_ptr), None, None, ptr(n_out),
                                                0, None), "gg_window_pairs")
            P = int(n_out.item())
            n1 = torch.empty(P, dtype=torch.int32, device=cuda_device)
            n2 = torch.empty(P, dtype=torch.int32, device=cuda_device)
            _cabi.check(smp.lib.gg_window_pairs(1, ptr(p), ptr(pl), max_path, window, ptr(pair_ptr), ptr(n1), ptr(n2),
                                                ptr(n_out), P, None), "gg_window_pairs")
            r = torch.empty(P, dtype=torch.float32, device=cuda_device)
            _cabi.check(smp.lib.gg_pair_reward(P, ptr(n1), ptr(n2), ptr(D_[0]), ptr(D_[1]), ld, ptr(r), None),
                        "gg_pair_reward")
            pE, pb = _pair_grad_g(smp.lib, cuda_device, n1, n2, r, G_[0], G_[1])
            v = torch.cat([pE.reshape(-1), pb])
            nz = torch.nonzero(v).squeeze(1)
            rows.append(np.full(int(nz.shape[0]), t))
            cols.append(nz.cpu().numpy())
            vals.append(v[nz].cpu().numpy())
            prod_sq[t] = float((v * v).sum().item())
        want = sq_node[k][ys]
        assert np.all(np.abs(prod_sq - want) <= 1e-5 * want), np.max(np.abs(prod_sq - want) / want)
        per_walk = prod_sq[inv]
        z = (per_walk.mean() - sq[k]) / (per_walk.std(ddof=1) / np.sqrt(per_root))
        print("root %d: %d stops, sq %.6g, estimate %.6g, z = %.2f" % (c, len(ys), sq[k], per_walk.mean(), z))
        assert abs(z) < 5
        S = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(len(ys), n * (ld + 1)))
        n_p = per_root // n_pass
        cnt = sp.csr_matrix((np.ones(n_p * n_pass), (np.repeat(np.arange(n_p), n_pass), inv[:n_p * n_pass])),
                            shape=(n_p, len(ys)))
        Sp = cnt @ S
        e2 = np.asarray(Sp.multiply(Sp).sum(axis=1)).ravel()
        want = n_pass * sq[k] + n_pass * (n_pass - 1) * mn[k]
        z = (e2.mean() - want) / (e2.std(ddof=1) / np.sqrt(n_p))
        print("root %d: E|S_pass|^2 %.6g, estimate %.6g, z = %.2f" % (c, want, e2.mean(), z))
        assert abs(z) < 5


@pytest.mark.parametrize("flags", [(), ("value_grad", "value_grad_d", "value_gcos", "value_dcos", "value_jsd")])
def test_trainer_gsnr(flags, cuda_device, tmp_path, monkeypatch):
    """One short CA-GrQc epoch with value_roots = 16: with value_gsnr the value line ends in gsnr > 0, and the line
    before it is the bits of the line without the flag, alone and after every other field"""
    from graphgan_b200 import config
    for k in ("value_dcos", "value_jsd", "value_gsnr"):
        monkeypatch.setattr(config, k, k in flags + ("value_gsnr",))
    gan, lines = _train(monkeypatch, tmp_path, cuda_device, flags, "s")
    monkeypatch.setattr(config, "value_gsnr", False)
    _, lines0 = _train(monkeypatch, tmp_path, cuda_device, flags, "0")
    assert [ln.split(":")[0] for ln in lines] == ["gen", "dis", "value"] * 2
    pat = re.compile(r"^(value:.*) gsnr:(\S+)$")
    for ln, ln0 in zip(lines, lines0):
        if not ln.startswith("value:"):
            assert ln == ln0
            continue
        m = pat.match(ln)
        assert m, ln
        assert m.group(1) == ln0 and float(m.group(2)) > 0
    _, ok, sq, mn, gE, gb = gan.expected_g_moments(gan.value_roots())
    k = gan.generator.n_emb
    sel = ok == 1
    snr = config.n_sample_gen * float((gE[:, :k] ** 2).sum() + (gb ** 2).sum()) / float((sq - mn)[sel].sum())
    assert abs(float(pat.match(lines[5]).group(2)) - snr) <= 1e-12 * snr
