"""The GraphGAN game value V_c(G, D) on the device (csrc/value.cu, DESIGN.md section 5.2).

Bars: pos and neg agree with the host reference (tests/game_value_oracle.py on top of tests/gdist_oracle.py) within
1e-12 of the sum of |terms|; with one-hot G rows, neg is -bce of the C oracle's fp32 score to 4 fp64 ulp (so every score
has the canonical fp32 bits); the bits do not depend on the chunking, the root order or the call; neg agrees with the
production sampler's walks; the ok flags and the trainer's value line.
"""
import ctypes as C
import re

import numpy as np
import pytest

from tests import game_value_oracle as vo
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


def _check_oracle(hg, dg, smp, trees, roots, G_, D_):
    (g_emb, g_bias, Eg, bg), (d_emb, d_bias, Ed, bd) = G_, D_
    pos, neg, ok = (x.cpu().numpy() for x in smp.game_value(g_emb, g_bias, d_emb, d_bias, trees))
    par = trees.parent_arrays().cpu().numpy()
    bits = dg.d1_bits.cpu().numpy().view(np.uint32)
    for k, r in enumerate(roots):
        wp, wn, wok, pa, na = vo.game_value(Ed, bd, Eg, bg, hg, int(r), par[k], bits)
        assert ok[k] == wok, int(r)
        assert abs(pos[k] - wp) <= 1e-12 * pa and abs(neg[k] - wn) <= 1e-12 * na, (int(r), pos[k], wp, neg[k], wn)
    return pos, neg, ok


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
    roots = _fixture_roots(hg, 100, 1)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, case.bias_g, cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(2).normal(0, 0.3, hg.n_node), cuda_device)
    pos0, neg0, ok0 = _check_oracle(hg, dg, smp, trees, roots, G_, D_)       # no father entry removed
    assert ok0.any() and np.all(pos0[ok0 == 1] < 0) and np.all(neg0[ok0 == 1] < 0)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=3)
    assert dg.d1_bits.any()
    _, neg1, _ = _check_oracle(hg, dg, smp, trees, roots, G_, D_)
    assert not np.array_equal(neg0, neg1)


@pytest.mark.parametrize("d", [20, 50, 100, 200, 300, 512])
def test_one_hot_rows_give_the_canonical_score_bits(d, cuda_device):
    """dist rows set to one-hot vectors and fed straight to gg_game_value: neg = -bce(s) with s the C oracle's fp32 score,
    to 4 fp64 ulp.  70 roots span several root tiles at every row stride."""
    import torch
    from graphgan_b200 import _cabi, synth
    from graphgan_b200._cabi import ptr
    from oracle import canonical as can
    _, hg, dg, _ = _graph("rand300", cuda_device, 0)
    n = hg.n_node
    rs = np.random.RandomState(d)
    emb, bias, E, bias_h = _params(synth.embeddings(n, d, seed=d), rs.normal(0, 1.0, n), cuda_device)
    roots = rs.choice(np.flatnonzero(hg.degrees() > 0), 70, replace=False).astype(np.int32)
    v = rs.randint(0, n, roots.shape[0])
    dist = torch.zeros((roots.shape[0], n), dtype=torch.float64, device=cuda_device)
    dist[torch.arange(roots.shape[0]), torch.as_tensor(v)] = 1.0
    R = roots.shape[0]
    roots_d = torch.as_tensor(roots).to(cuda_device)
    root_ok = torch.ones(R, dtype=torch.int32, device=cuda_device)
    pos = torch.empty(R, dtype=torch.float64, device=cuda_device)
    neg, ok = torch.empty_like(pos), torch.empty(R, dtype=torch.int32, device=cuda_device)
    lib = _cabi.lib()
    nb = C.c_int64(0)
    _cabi.check(lib.gg_game_value_scratch_bytes(n, R, C.byref(nb)))
    scratch = torch.empty(nb.value, dtype=torch.uint8, device=cuda_device)
    _cabi.check(lib.gg_game_value(n, int(emb.shape[1]), ptr(emb), ptr(bias), ptr(dg.raw_indptr), ptr(dg.raw_adj), R,
                                  ptr(roots_d), ptr(dist), ptr(root_ok), ptr(pos), ptr(neg), ptr(ok), ptr(scratch),
                                  nb.value, None), "gg_game_value")
    torch.cuda.synchronize()
    neg, pos, ok = neg.cpu().numpy(), pos.cpu().numpy(), ok.cpu().numpy()
    assert ok.all()
    for k, c in enumerate(roots):
        s = np.float32(can.dot_c(E[c], E[v[k]]) + np.float32(bias_h[v[k]]))
        want = -vo.bce(s, 0)
        assert abs(neg[k] - want) <= 4 * np.spacing(abs(want)), (d, int(c), int(v[k]), neg[k], want)
        wp, pa = vo.pos_term(E, bias_h, hg.raw_indptr, hg.raw_adj, int(c))
        assert abs(pos[k] - wp) <= 1e-12 * pa


def test_c3_roots_with_the_largest_hub(cuda_device):
    """C3 (power-law N = 1M, avg-deg 20, n_emb 128): the 13 828-neighbour hub, three of its neighbours and two ordinary
    roots, after a D pass; the host reference evaluates only these rows."""
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
    pos, neg, ok = _check_oracle(hg, dg, smp, trees, roots, G_, D_)
    assert ok.all()


def test_bits_do_not_depend_on_chunks_order_or_call(cuda_device):
    import torch
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    roots = _fixture_roots(hg, 150, 4)
    G_ = _params(case.emb_g, case.bias_g, cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(7).normal(0, 0.3, hg.n_node), cuda_device)
    trees = smp.build_trees(roots)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=8)
    args = (G_[0], G_[1], D_[0], D_[1])
    bits = lambda out: [x.cpu().numpy().view(np.uint8).tobytes() for x in out]
    base = bits(smp.game_value(*args, trees))
    assert bits(smp.game_value(*args, trees)) == base                                 # repeated call
    assert bits(smp.game_value(*args, trees, max_scratch_bytes=1)) == base            # one root per chunk
    nb = C.c_int64(0)
    smp.lib.gg_generator_dist_scratch_bytes(hg.n_node, len(hg.adj), 7, C.byref(nb))
    assert bits(smp.game_value(*args, trees, max_scratch_bytes=nb.value)) == base     # 7 roots per chunk
    perm = np.random.RandomState(9).permutation(len(roots))
    out = smp.game_value(*args, smp.build_trees(roots[perm]))
    inv = torch.as_tensor(np.argsort(perm)).to(cuda_device)
    assert bits([x[inv] for x in out]) == base                                        # roots in another order


def test_neg_agrees_with_sampled_walks(cuda_device):
    """2^20 G-mode walks of four CA-GrQc roots through the production sampler (after a D pass): the mean of
    -bce(s(c, v), 0) over the sampled v is neg_c within |z| < 5."""
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    roots = np.argsort(-hg.degrees(), kind="stable")[[0, 5, 40, 200]].astype(np.int32)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, case.bias_g, cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(10).normal(0, 0.3, hg.n_node), cuda_device)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=21)
    pos, neg, ok = (x.cpu().numpy() for x in smp.game_value(G_[0], G_[1], D_[0], D_[1], trees))
    per_root = 1 << 18
    out = smp.run(G_[0], G_[1], trees, per_root, False, seed=23, pass_tag=5)
    samples = out.samples.cpu().numpy()
    for k, c in enumerate(roots):
        assert ok[k] == 1
        sm = samples[k * per_root:(k + 1) * per_root]
        uniq, inv = np.unique(sm, return_inverse=True)
        t = -vo.bce(vo.scores(D_[2], D_[3], int(c), uniq), 0)[inv]
        z = (t.mean() - neg[k]) / (t.std() / np.sqrt(per_root))
        print("root %d: neg %.6f, sampled %.6f, z = %.2f" % (c, neg[k], t.mean(), z))
        assert abs(z) < 5


def test_ok_flags(cuda_device):
    """An isolated root, a root with only a self-loop and a void root (a depth-1 leaf whose father entry is removed)
    have ok = 0 and pos = neg = 0; the other roots ok = 1."""
    import torch
    from graphgan_b200 import graph as G, sampler as S, synth
    n0 = 3000
    edges = np.concatenate([synth.power_law(n0, 10, seed=1), [[n0 + 1, n0 + 1]]])
    n = n0 + 2                                                # node n0: isolated; node n0 + 1: a self-loop only
    hg = G.HostGraph(edges, None, n_node=n)
    dg = G.DeviceGraph(hg, cuda_device)
    smp = S.WalkSampler(dg, hub_threshold=128)
    roots = np.concatenate([synth.pick_roots(hg.degrees(), 40, seed=2), [n0, n0 + 1]]).astype(np.int32)
    trees = smp.build_trees(roots)
    par = trees.parent_arrays().cpu().numpy()
    # the void root: a root with a depth-1 child that has no children in its tree; remove that child's father entry
    void = None
    for k, r in enumerate(roots[:-2]):
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
    pos, neg, ok = (x.cpu().numpy() for x in smp.game_value(G_[0], G_[1], D_[0], D_[1], trees))
    bad = np.zeros(len(roots), bool)
    bad[[void[0], len(roots) - 2, len(roots) - 1]] = True
    assert not ok[bad].any() and ok[~bad].all()
    assert not pos[bad].any() and not neg[bad].any()
    assert np.all(pos[~bad] < 0) and np.all(neg[~bad] < 0)


def _train(monkeypatch, tmp_path, cuda_device, value_roots, tag):
    from graphgan_b200 import config, graph as G
    from graphgan_b200.graph_gan import GraphGAN
    c = loader.load("cagrqc")
    for k, v in dict(n_emb=50, n_epochs=1, n_epochs_dis=1, dis_interval=1, n_epochs_gen=1, gen_interval=1,
                     n_sample_gen=2, device=str(cuda_device), seed=5, value_roots=value_roots, text_embeddings=False).items():
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


def test_trainer_value_line(cuda_device, tmp_path, monkeypatch):
    """One short CA-GrQc epoch: with value_roots = 16 the evaluation appends the value line after the link-prediction
    lines (before training and after the epoch); with 0 the result file holds exactly the link-prediction lines, and
    they are the same in both runs (the value changes nothing in training)."""
    gan, lines = _train(monkeypatch, tmp_path, cuda_device, 16, "16")
    assert [ln.split(":")[0] for ln in lines] == ["gen", "dis", "value"] * 2
    pat = re.compile(r"^value:(\S+) pos:(\S+) neg:(\S+) roots:(\d+)$")
    for ln in lines[2::3]:
        m = pat.match(ln)
        assert m, ln
        v, p, q, n = float(m.group(1)), float(m.group(2)), float(m.group(3)), int(m.group(4))
        assert n == 16 and p < 0 and q < 0 and abs(v - (p + q)) <= 1e-12 * abs(v)
    assert lines[5] != lines[2]                                      # the epoch moved the value
    roots = gan.value_roots()
    assert len(roots) == 16 and np.array_equal(roots, np.sort(roots))
    assert gan.value_line().strip() == lines[5]                       # the same roots and bits on a second evaluation
    pos, neg, ok = (x.cpu().numpy() for x in gan.game_value(roots))
    assert ok.all() and float(lines[5].split()[0].split(":")[1]) == float((pos + neg).mean())
    _, lines0 = _train(monkeypatch, tmp_path, cuda_device, 0, "0")
    assert [ln.split(":")[0] for ln in lines0] == ["gen", "dis"] * 2
    assert lines0 == [ln for ln in lines if not ln.startswith("value:")]
