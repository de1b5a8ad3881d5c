"""The exact expectation of the reference's generator step on the device (csrc/value_gref.cu, DESIGN.md section 5.6).

Bars: per coordinate within 1e-12 of the coordinate's sum of |terms| of the host reference (tests/expected_g_grad_oracle.py,
with gg_pair_reward's rewards), n_pairs within 1e-14 relative; pad columns exactly 0; the bits do not depend on the
chunking, the root order or the call; void, isolated and self-loop-only roots add exactly 0; the production G pass
(sampler, gg_window_pairs, gg_pair_reward, gg_pair_grad_ex mode 1) agrees with it over 2^20 walks; the trainer's gcos.
"""
import ctypes as C
import re

import numpy as np
import pytest

from tests import expected_g_grad_oracle as eo
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


def _device_reward(lib, d_emb, d_bias):
    """r(n1, n2) with the bits of gg_pair_reward (the production reward kernel)"""
    import torch
    from graphgan_b200 import _cabi
    from graphgan_b200._cabi import ptr
    dev, ld = d_emb.device, int(d_emb.shape[1])

    def reward(n1, n2):
        if len(n1) == 0:
            return np.zeros(0, np.float32)
        i = torch.as_tensor(np.asarray(n1, np.int32)).to(dev)
        j = torch.as_tensor(np.asarray(n2, np.int32)).to(dev)
        out = torch.empty(len(n1), dtype=torch.float32, device=dev)
        _cabi.check(lib.gg_pair_reward(len(n1), ptr(i), ptr(j), ptr(d_emb), ptr(d_bias), ld, ptr(out), None), "gg_pair_reward")
        return out.cpu().numpy()
    return reward


def _check_oracle(hg, dg, smp, trees, roots, G_, D_, window, rows=None):
    (g_emb, g_bias, Eg, bg), (d_emb, d_bias, _, _) = G_, D_
    out = smp.expected_g_grad(g_emb, g_bias, d_emb, d_bias, trees, window=window)
    n_pairs, ok = out[0].cpu().numpy(), out[1].cpu().numpy()
    gE, gb = out[2].cpu().numpy(), out[3].cpu().numpy()
    if rows is not None:
        gE, gb = gE[rows], gb[rows]
    par = trees.parent_arrays().cpu().numpy()
    bits = dg.d1_bits.cpu().numpy().view(np.uint32)
    wE, wb, aE, ab, per = eo.expect(Eg, bg, hg, roots, par, bits, window, _device_reward(smp.lib, d_emb, d_bias), rows)
    assert [o["ok"] for o in per] == list(ok)
    want_n = np.array([o["n_pairs"] for o in per])
    assert np.all(np.abs(n_pairs - want_n) <= 1e-14 * want_n), np.max(np.abs(n_pairs - want_n) / np.maximum(want_n, 1e-300))
    assert np.all(np.abs(gE - wE) <= 1e-12 * aE) and np.all(np.abs(gb - wb) <= 1e-12 * ab), (
        np.max(np.abs(gE - wE) - 1e-12 * aE), np.max(np.abs(gb - wb) - 1e-12 * ab))
    n_emb = int(np.flatnonzero(np.abs(Eg).sum(axis=0))[-1]) + 1
    assert not gE[:, n_emb:].any()                                      # pad columns exactly 0
    print("window %d: %d ok roots, %d ambiguous sigmoids" % (window, int(ok.sum()), sum(o["n_amb"] for o in per)))
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
    roots = _fixture_roots(hg, 30, 1)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, np.random.RandomState(3).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(2).normal(0, 0.3, hg.n_node), cuda_device)
    before = {}
    for w in (1, 2, 3):
        before[w] = _check_oracle(hg, dg, smp, trees, roots, G_, D_, w)
        assert before[w][1].cpu().numpy().any() and before[w][2].abs().sum().item() > 0
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=3)
    assert dg.d1_bits.any()
    for w in (1, 2, 3):
        out = _check_oracle(hg, dg, smp, trees, roots, G_, D_, w)
        assert not np.array_equal(out[2].cpu().numpy(), before[w][2].cpu().numpy())


@pytest.mark.parametrize("d", [20, 50, 100, 200, 300, 512])
def test_every_row_stride(d, cuda_device):
    from graphgan_b200 import synth
    _, hg, dg, smp = _graph("rand300", cuda_device, 0)
    n = hg.n_node
    rs = np.random.RandomState(d)
    roots = np.sort(rs.choice(np.flatnonzero(hg.degrees() > 0), 12, replace=False)).astype(np.int32)
    G_ = _params(synth.embeddings(n, d, seed=d, sigma=0.3), rs.normal(0, 0.3, n), cuda_device)
    D_ = _params(synth.embeddings(n, d, seed=d + 1, sigma=0.3), rs.normal(0, 0.3, n), cuda_device)
    out = _check_oracle(hg, dg, smp, smp.build_trees(roots), roots, G_, D_, 2)
    assert int(out[2].shape[1]) == int(G_[0].shape[1])


def test_c3_roots_with_the_largest_hub(cuda_device):
    """C3 (power-law N = 1M, avg-deg 20, n_emb 128) at w = 2: the 13 828-neighbour hub, three of its neighbours and two
    ordinary roots, after a D pass.  The hub's down part is split over eight chains; the test prints how many window
    pairs have the hub as their ancestor (its children and grandchildren) per root."""
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
    out = _check_oracle(hg, dg, smp, trees, roots, G_, D_, 2, rows)
    assert out[1].cpu().numpy().all()
    par = trees.parent_arrays().cpu().numpy()
    for k, r in enumerate(roots):
        ch = np.flatnonzero(par[k] == top)
        print("root %d: %d tree children and %d tree grandchildren of the hub" % (r, len(ch), int(np.isin(par[k], ch).sum())))


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
        base = _bits(smp.expected_g_grad(*args, trees, window=w))
        assert _bits(smp.expected_g_grad(*args, trees, window=w)) == base                             # repeated call
        assert _bits(smp.expected_g_grad(*args, trees, window=w, max_scratch_bytes=1)) == base        # one root per chunk
        nb = C.c_int64(0)
        smp.lib.gg_expected_g_grad_scratch_bytes(hg.n_node, len(hg.adj), 7, w, C.byref(nb))
        assert _bits(smp.expected_g_grad(*args, trees, window=w, max_scratch_bytes=nb.value)) == base  # 7 roots per chunk
        perm = np.random.RandomState(9).permutation(len(roots))
        out = smp.expected_g_grad(*args, smp.build_trees(roots[perm]), window=w)
        inv = torch.as_tensor(np.argsort(perm)).to(cuda_device)
        assert _bits([x[inv] for x in out[:2]]) + _bits(out[2:]) == base                             # roots in another order


def test_void_isolated_and_self_loop_roots_add_nothing(cuda_device):
    """An isolated root, a root with only a self-loop and a void root (a depth-1 leaf whose father entry is removed) have
    root_ok = 0 and n_pairs = 0, and leave the gradient exactly as the other roots make it."""
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
    want = smp.expected_g_grad(*args, smp.build_trees(rest), window=2)
    roots = np.concatenate([good, [n0, n0 + 1]]).astype(np.int32)
    out = smp.expected_g_grad(*args, smp.build_trees(roots), window=2)
    ok, n_pairs = out[1].cpu().numpy(), out[0].cpu().numpy()
    bad = np.zeros(len(roots), bool)
    bad[[void[0], len(roots) - 2, len(roots) - 1]] = True
    assert not ok[bad].any() and ok[~bad].all()
    assert not n_pairs[bad].any() and np.all(n_pairs[~bad] > 0)
    assert _bits(out[2:]) == _bits(want[2:])
    alone = smp.expected_g_grad(*args, smp.build_trees(roots[bad]), window=2)
    assert not alone[0].any() and not alone[2].any() and not alone[3].any()


def _pair_grad_g(lib, dev, n1, n2, reward, emb, bias):
    """gg_pair_grad_ex(mode 1, batch_total 1, lambda 0) of the pairs (n1, n2) with rewards -> dense fp64 (rows, bias)"""
    import torch
    from graphgan_b200 import _cabi
    from graphgan_b200._cabi import ptr
    B, (n, ld) = int(n1.shape[0]), emb.shape
    nu = torch.zeros(1, dtype=torch.int32, device=dev)
    ids = torch.empty(2 * B, dtype=torch.int32, device=dev)
    rows = torch.empty((2 * B, ld), dtype=torch.float32, device=dev)
    gb = torch.empty(2 * B, dtype=torch.float32, device=dev)
    slot = torch.full((n,), -1, dtype=torch.int32, device=dev)
    nb = C.c_int64(0)
    _cabi.check(lib.gg_pair_grad_scratch_bytes(B, ld, C.byref(nb)))
    scratch = torch.empty(max(nb.value, 256), dtype=torch.uint8, device=dev)
    _cabi.check(lib.gg_pair_grad_ex(1, B, 1, ptr(n1), ptr(n2), ptr(reward), ptr(emb), ptr(bias), ld, 0.0, ptr(nu), ptr(ids),
                                    ptr(rows), ptr(gb), ptr(slot), ptr(scratch), nb.value, 0, None), "gg_pair_grad_ex")
    U = int(nu.item())
    dE = torch.zeros((n, ld), dtype=torch.float64, device=dev)
    db = torch.zeros(n, dtype=torch.float64, device=dev)
    dE[ids[:U].long()] = rows[:U].double()
    db[ids[:U].long()] = gb[:U].double()
    return dE, db


def test_production_g_pass_over_2_20_walks(cuda_device):
    """2^20 G-mode walks of four CA-GrQc roots from the production sampler (after a D pass), their window pairs
    (gg_window_pairs, w = 2), rewards (gg_pair_reward) and G gradient (gg_pair_grad_ex mode 1, batch_total 1, lambda 0) in
    64 batches per root.  The batch means per walk, projected on 8 random directions, estimate the exact expectation, and
    the batches' pairs per walk estimate n_pairs: |z| < 5 with z from the batch means' spread.  The roots avoid those
    whose G sigmoids sit at fp32 1 along the walks (the 200th by degree has an expectation of 3e-8): there kappa is a
    multiple of 2^-24 r that few pairs reach, and 64 batch means are far from normal."""
    import torch
    from graphgan_b200 import _cabi
    from graphgan_b200._cabi import ptr
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    window = 2
    roots = np.argsort(-hg.degrees(), kind="stable")[[0, 5, 40, 150]].astype(np.int32)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, np.random.RandomState(12).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(10).normal(0, 0.3, hg.n_node), cuda_device)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=21)
    per_root, n_batch, max_path = 1 << 18, 64, 64
    out = smp.run(G_[0], G_[1], trees, per_root, False, seed=23, pass_tag=5, max_path=max_path)
    assert np.all(out.status.cpu().numpy() == 1)
    n, ld = hg.n_node, int(G_[0].shape[1])
    n_emb = case.emb_g.shape[1]
    rs = np.random.RandomState(31)
    dirs = []
    for _ in range(8):
        dE = np.zeros((n, ld))
        dE[:, :n_emb] = rs.normal(0, 1, (n, n_emb))
        dirs.append((torch.as_tensor(dE).to(cuda_device), torch.as_tensor(rs.normal(0, 1, n)).to(cuda_device)))
    bs = per_root // n_batch
    pair_ptr = torch.empty(bs + 1, dtype=torch.int64, device=cuda_device)
    n_out = torch.zeros(1, dtype=torch.int64, device=cuda_device)
    for k, c in enumerate(roots):
        one = smp.expected_g_grad(G_[0], G_[1], D_[0], D_[1], trees.select(torch.tensor([k], device=cuda_device)),
                                  window=window)
        assert int(one[1].item()) == 1
        nbar, gE, gb = float(one[0].item()), one[2], one[3]
        means, pairs = np.zeros((n_batch, len(dirs))), np.zeros(n_batch)
        for t in range(n_batch):
            w0 = k * per_root + t * bs
            paths, plen = out.paths[w0:w0 + bs].contiguous(), out.path_len[w0:w0 + bs].contiguous()
            _cabi.check(smp.lib.gg_window_pairs(bs, ptr(paths), ptr(plen), max_path, window, ptr(pair_ptr), None, None,
                                                ptr(n_out), 0, None), "gg_window_pairs")
            P = int(n_out.item())
            n1 = torch.empty(P, dtype=torch.int32, device=cuda_device)
            n2 = torch.empty(P, dtype=torch.int32, device=cuda_device)
            _cabi.check(smp.lib.gg_window_pairs(bs, ptr(paths), ptr(plen), max_path, window, ptr(pair_ptr), ptr(n1), ptr(n2),
                                                ptr(n_out), P, None), "gg_window_pairs")
            r = torch.empty(P, dtype=torch.float32, device=cuda_device)
            _cabi.check(smp.lib.gg_pair_reward(P, ptr(n1), ptr(n2), ptr(D_[0]), ptr(D_[1]), ld, ptr(r), None), "gg_pair_reward")
            pE, pb = _pair_grad_g(smp.lib, cuda_device, n1, n2, r, G_[0], G_[1])
            pairs[t] = P / bs
            for q, (dE, db) in enumerate(dirs):
                means[t, q] = float((pE * dE).sum() + (pb * db).sum()) / bs
        z = (pairs.mean() - nbar) / (pairs.std(ddof=1) / np.sqrt(n_batch))
        print("root %d: n_pairs %.6g, estimate %.6g, z = %.2f" % (c, nbar, pairs.mean(), z))
        assert abs(z) < 5
        for q, (dE, db) in enumerate(dirs):
            exact = float((gE * dE).sum() + (gb * db).sum())
            z = (means[:, q].mean() - exact) / (means[:, q].std(ddof=1) / np.sqrt(n_batch))
            print("root %d: exact %.6g, estimate %.6g, z = %.2f" % (c, exact, means[:, q].mean(), z))
            assert abs(z) < 5


def _train(monkeypatch, tmp_path, cuda_device, flags, tag):
    from graphgan_b200 import config, graph as G
    from graphgan_b200.graph_gan import GraphGAN
    c = loader.load("cagrqc")
    for k, v in dict(n_emb=50, n_epochs=1, n_epochs_dis=1, dis_interval=1, n_epochs_gen=1, gen_interval=1,
                     n_sample_gen=2, device=str(cuda_device), seed=5, value_roots=16, text_embeddings=False).items():
        monkeypatch.setattr(config, k, v)
    for k in ("value_grad", "value_grad_d", "value_gcos"):
        monkeypatch.setattr(config, k, k in flags)

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


@pytest.mark.parametrize("flags", [(), ("value_grad",)])
def test_trainer_gcos(flags, cuda_device, tmp_path, monkeypatch):
    """One short CA-GrQc epoch with value_roots = 16: with value_gcos the value line ends in gcos in [-1, 1], and the line
    before it is the bits of the line without the flag, alone and after gnorm."""
    import torch
    gan, lines = _train(monkeypatch, tmp_path, cuda_device, flags + ("value_gcos",), "c")
    _, lines0 = _train(monkeypatch, tmp_path, cuda_device, flags, "0")
    assert [ln.split(":")[0] for ln in lines] == ["gen", "dis", "value"] * 2
    pat = re.compile(r"^(value:.*) gcos:(\S+)$")
    for ln, ln0 in zip(lines, lines0):
        if not ln.startswith("value:"):
            assert ln == ln0
            continue
        m = pat.match(ln)
        assert m, ln
        assert m.group(1) == ln0 and -1.0 <= float(m.group(2)) <= 1.0
    rE, rb = gan.expected_g_grad(gan.value_roots())[2:]
    gE, gb = gan.game_value_grad(gan.value_roots())[3:]
    k = gan.generator.n_emb
    cos = float(((rE[:, :k] * gE[:, :k]).sum() + (rb * gb).sum()) / torch.sqrt(
        ((rE[:, :k] ** 2).sum() + (rb ** 2).sum()) * ((gE[:, :k] ** 2).sum() + (gb ** 2).sum())))
    assert abs(float(pat.match(lines[5]).group(2)) - cos) <= 1e-12
