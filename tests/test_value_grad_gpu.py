"""The exact generator gradient of the game value on the device (csrc/value_grad.cu, DESIGN.md section 5.3).

Bars: the gradient agrees with the "pi" law of the host reference (tests/value_grad_oracle.py) per coordinate within 1e-12
of that coordinate's sum of |terms|; pos / neg / ok are the bits of game_value; the gradient's bits do not depend on the
chunking, the root order or the call; roots that are void, isolated or self-loop-only add exactly 0; a score-function
estimate over 2^20 production walks agrees with it; the trainer's gnorm field.
"""
import ctypes as C
import re

import numpy as np
import pytest

from tests import value_grad_oracle as gro
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


def _check_oracle(hg, dg, smp, trees, roots, G_, D_, rows=None):
    """the gradient against the "pi" oracle (on ``rows`` only, when given), and pos / neg / ok against game_value"""
    (g_emb, g_bias, Eg, bg), (d_emb, d_bias, Ed, bd) = G_, D_
    out = smp.game_value_grad(g_emb, g_bias, d_emb, d_bias, trees)
    assert _bits(out[:3]) == _bits(smp.game_value(g_emb, g_bias, d_emb, d_bias, trees))
    gE, gb = out[3].cpu().numpy(), out[4].cpu().numpy()
    if rows is not None:
        gE, gb = gE[rows], gb[rows]
    par = trees.parent_arrays().cpu().numpy()
    bits = dg.d1_bits.cpu().numpy().view(np.uint32)
    wE, wb, aE, ab, per = gro.grad(Eg, bg, Ed, bd, hg, roots, par, bits, "pi", rows)
    assert np.all(np.abs(gE - wE) <= 1e-12 * aE) and np.all(np.abs(gb - wb) <= 1e-12 * ab), (
        np.max(np.abs(gE - wE) - 1e-12 * aE), np.max(np.abs(gb - wb) - 1e-12 * ab))
    d = Eg.shape[1]
    n_emb = int(np.flatnonzero(np.abs(Eg).sum(axis=0))[-1]) + 1
    assert not gE[:, n_emb:d].any()                                     # pad columns exactly 0
    assert [o["ok"] for o in per] == list(out[2].cpu().numpy())
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
    assert int(out[3].shape[1]) == int(G_[0].shape[1])


def test_c3_roots_with_the_largest_hub(cuda_device):
    """C3 (power-law N = 1M, avg-deg 20, n_emb 128): the 13 828-neighbour hub, three of its neighbours and two ordinary
    roots, after a D pass.  The hub's child-edge sum is split over eight chains (DESIGN.md section 5.3)."""
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
    out = _check_oracle(hg, dg, smp, trees, roots, G_, D_, rows)
    assert out[2].cpu().numpy().all()


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
    base = _bits(smp.game_value_grad(*args, trees))
    assert _bits(smp.game_value_grad(*args, trees)) == base                             # repeated call
    assert _bits(smp.game_value_grad(*args, trees, max_scratch_bytes=1)) == base        # one root per chunk
    nb = C.c_int64(0)
    smp.lib.gg_game_value_grad_scratch_bytes(hg.n_node, len(hg.adj), 7, C.byref(nb))
    assert _bits(smp.game_value_grad(*args, trees, max_scratch_bytes=nb.value)) == base  # 7 roots per chunk
    perm = np.random.RandomState(9).permutation(len(roots))
    out = smp.game_value_grad(*args, smp.build_trees(roots[perm]))
    inv = torch.as_tensor(np.argsort(perm)).to(cuda_device)
    assert _bits([x[inv] for x in out[:3]]) + _bits(out[3:]) == base                   # roots in another order


def test_void_isolated_and_self_loop_roots_add_nothing(cuda_device):
    """An isolated root, a root with only a self-loop and a void root (a depth-1 leaf whose father entry is removed) have
    ok = 0 and leave the gradient exactly as the other roots make it."""
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
    want = smp.game_value_grad(*args, smp.build_trees(rest))
    roots = np.concatenate([good, [n0, n0 + 1]]).astype(np.int32)
    out = smp.game_value_grad(*args, smp.build_trees(roots))
    ok = out[2].cpu().numpy()
    bad = np.zeros(len(roots), bool)
    bad[[void[0], len(roots) - 2, len(roots) - 1]] = True
    assert not ok[bad].any() and ok[~bad].all()
    assert _bits(out[3:]) == _bits(want[3:])
    alone = smp.game_value_grad(*args, smp.build_trees(roots[bad]))
    assert not alone[3].any() and not alone[4].any()


def test_score_function_estimate_over_production_walks(cuda_device):
    """2^20 G-mode walks of four CA-GrQc roots through the production sampler (after a D pass), paths recorded: the mean of
    log(1 - D(v, c)) * sum over the path's steps of (ds(a, x) - E_pi[ds(a, .)]) is the exact gradient's projection on a
    random direction d, |z| < 5 for 8 directions per root.  This checks the law of every step of the path."""
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    roots = np.argsort(-hg.degrees(), kind="stable")[[0, 5, 40, 200]].astype(np.int32)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, np.random.RandomState(12).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(10).normal(0, 0.3, hg.n_node), cuda_device)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=21)
    par = trees.parent_arrays().cpu().numpy()
    bits = dg.d1_bits.cpu().numpy().view(np.uint32)
    per_root, max_path = 1 << 18, 64
    out = smp.run(G_[0], G_[1], trees, per_root, False, seed=23, pass_tag=5, max_path=max_path)
    paths, plen, samples = out.paths.cpu().numpy(), out.path_len.cpu().numpy(), out.samples.cpu().numpy()
    E = G_[2].astype(np.float64)
    from tests import game_value_oracle as vo
    rs = np.random.RandomState(31)
    dirs = []
    for _ in range(8):
        dE = np.zeros_like(E)
        n_emb = int(np.flatnonzero(np.abs(E).sum(axis=0))[-1]) + 1
        dE[:, :n_emb] = rs.normal(0, 1, (hg.n_node, n_emb))
        dirs.append((dE, rs.normal(0, 1, hg.n_node)))
    for k, c in enumerate(roots):
        one = smp.game_value_grad(G_[0], G_[1], D_[0], D_[1], trees.select(smp.torch.tensor([k], device=cuda_device)))
        assert int(one[2].item()) == 1
        gE, gb = one[3].cpu().numpy(), one[4].cpu().numpy()
        o = gro.root_grad(G_[2], G_[3], D_[2], D_[3], hg, int(c), par[k], bits, "pi")
        owner, cand, is_f, pi = o["owner"], o["cand"], o["is_father"], o["pi"]
        rec_of = np.full(hg.n_node, -1, np.int64)                      # the record of the step into x (child) ...
        rec_of[cand[~is_f]] = np.flatnonzero(~is_f)
        stop_of = np.full(hg.n_node, -1, np.int64)                     # ... and of the stop step of a
        stop_of[owner[is_f]] = np.flatnonzero(is_f)
        w = slice(k * per_root, (k + 1) * per_root)
        P, L = paths[w], plen[w]
        assert np.all((L >= 2) & (L <= max_path))
        v = samples[w]
        f = -vo.bce(vo.scores(D_[2], D_[3], int(c), v), 0)             # log(1 - D(v, c))
        steps = np.arange(max_path - 1)[None, :] < (L - 1)[:, None]
        a, x = np.where(steps, P[:, :-1], 0), np.where(steps, P[:, 1:], 0)     # (entries past path_len are not written)
        is_stop = steps & (x == par[k][a]) & (a != c)
        rec = np.where(is_stop, stop_of[a], rec_of[x])
        assert np.all(rec[steps] >= 0)
        for dE, db in dirs:
            ds = np.einsum("ij,ij->i", dE[owner], E[cand]) + np.einsum("ij,ij->i", E[owner], dE[cand]) + db[cand]
            mu = np.zeros(hg.n_node)
            np.add.at(mu, owner, pi * ds)
            term = ds - mu[owner]
            score = np.where(steps, term[np.maximum(rec, 0)], 0.0).sum(axis=1)
            est = f * score
            exact = float((gE * dE).sum() + (gb * db).sum())
            z = (est.mean() - exact) / (est.std() / np.sqrt(per_root))
            print("root %d: exact %.6g, estimate %.6g, z = %.2f" % (c, exact, est.mean(), z))
            assert abs(z) < 5


def _train(monkeypatch, tmp_path, cuda_device, value_grad, tag):
    from graphgan_b200 import config, graph as G
    from graphgan_b200.graph_gan import GraphGAN
    c = loader.load("cagrqc")
    for k, v in dict(n_emb=50, n_epochs=1, n_epochs_dis=1, dis_interval=1, n_epochs_gen=1, gen_interval=1,
                     n_sample_gen=2, device=str(cuda_device), seed=5, value_roots=16, value_grad=value_grad,
                     text_embeddings=False).items():
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


def test_trainer_gnorm(cuda_device, tmp_path, monkeypatch):
    """One short CA-GrQc epoch with value_roots = 16: with value_grad the value line ends in gnorm and its first four
    fields are the bits of the line without it; everything else in the result file is the same."""
    import torch
    gan, lines = _train(monkeypatch, tmp_path, cuda_device, True, "g")
    _, lines0 = _train(monkeypatch, tmp_path, cuda_device, False, "0")
    assert [ln.split(":")[0] for ln in lines] == ["gen", "dis", "value"] * 2
    pat = re.compile(r"^(value:\S+ pos:\S+ neg:\S+ roots:\d+) gnorm:(\S+)$")
    for ln, ln0 in zip(lines, lines0):
        if not ln.startswith("value:"):
            assert ln == ln0
            continue
        m = pat.match(ln)
        assert m, ln
        assert m.group(1) == ln0 and float(m.group(2)) > 0
    pos, neg, ok, gE, gb = gan.game_value_grad(gan.value_roots())
    n = int(ok.sum().item())
    want = float(torch.sqrt((gE[:, :gan.generator.n_emb] ** 2).sum() + (gb ** 2).sum()).item()) / n
    assert abs(float(pat.match(lines[5]).group(2)) - want) <= 1e-12 * want
