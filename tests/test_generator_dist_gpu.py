"""The exact generator distribution G(v | root) on the device (csrc/gdist.cu, DESIGN.md section 5.1).

Bars: dist and root_ok equal the host reference (tests/gdist_oracle.py, itself checked against the C oracle and a
brute-force enumeration in test_generator_dist_host.py) bit for bit -- at every row stride, with and without
father-removal bits, with the hub score cache on and off -- and the production sampler's empirical frequencies follow
the law (G-test).
"""
import numpy as np
import pytest

from tests import gdist_oracle as go
from tests.golden import loader

pytestmark = pytest.mark.gpu


def _sampler(hg, cuda_device, hub_threshold):
    from graphgan_b200 import graph as G, sampler as S
    dg = G.DeviceGraph(hg, cuda_device)
    return dg, S.WalkSampler(dg, hub_threshold=hub_threshold)


def _check_exact(hg, smp, dg, trees, emb, bias, E, bias_h, roots):
    dist, ok = smp.distribution(emb, bias, trees)
    dist, ok = dist.cpu().numpy(), ok.cpu().numpy()
    par = trees.parent_arrays().cpu().numpy()
    bits = dg.d1_bits.cpu().numpy().view(np.uint32)
    for k, r in enumerate(roots):
        want, want_ok = go.distribution(E, bias_h, hg.indptr, hg.adj, int(r), par[k], bits)
        assert ok[k] == want_ok, (int(r), ok[k], want_ok)
        assert np.array_equal(dist[k].view(np.uint64), want.view(np.uint64)), int(r)
    return dist, ok


def _d_pass(smp, hg, trees, emb, bias, roots, cuda_device, seed):
    import torch
    deg = torch.as_tensor(hg.degrees()[roots].astype(np.int64)).to(cuda_device)
    smp.run(emb, bias, trees, deg, True, seed=seed, pass_tag=1)


def _fixture_roots(hg, k, seed):
    n = hg.n_node
    if n <= k:
        return np.arange(n, dtype=np.int32)
    top = np.argsort(-hg.degrees(), kind="stable")[:4]
    rs = np.random.RandomState(seed)
    return np.unique(np.concatenate([top, rs.choice(n, k, replace=False)])).astype(np.int32)


@pytest.mark.parametrize("hub", [0, 64, 128, 300])
@pytest.mark.parametrize("name", ["tiny", "rand300", "rand1200", "cagrqc"])
def test_matches_oracle_bit_for_bit(name, hub, cuda_device):
    import torch
    from graphgan_b200 import graph as G, sampler as S
    from oracle import canonical as can
    case = loader.load(name)
    hg = G.HostGraph(case["train_edges"], case["test_edges"], n_node=case.n)
    dg, smp = _sampler(hg, cuda_device, hub)
    roots = _fixture_roots(hg, 120, 1)
    trees = smp.build_trees(roots)
    emb = S.pad_embedding(case.emb_g, cuda_device)
    bias = torch.as_tensor(case.bias_g).to(cuda_device)
    E = can.pad_rows(case.emb_g)
    dist0, ok0 = _check_exact(hg, smp, dg, trees, emb, bias, E, case.bias_g, roots)   # no father entry removed
    _d_pass(smp, hg, trees, emb, bias, roots, cuda_device, seed=3)
    assert dg.d1_bits.any()
    dist1, ok1 = _check_exact(hg, smp, dg, trees, emb, bias, E, case.bias_g, roots)
    assert not np.array_equal(dist0, dist1)
    # the hub cache never changes a bit: the same law without it
    if hub:
        d_off, ok_off = smp.distribution(emb, bias, trees, reuse=False)
        assert np.array_equal(d_off.cpu().numpy().view(np.uint64), dist1.view(np.uint64))
        assert np.array_equal(ok_off.cpu().numpy(), ok1)


@pytest.mark.parametrize("d", [20, 50, 100, 200, 300, 512])
@pytest.mark.parametrize("hub", [0, 8])
def test_every_row_stride(d, hub, cuda_device):
    import torch
    from graphgan_b200 import graph as G, sampler as S, synth
    from oracle import canonical as can
    case = loader.load("rand300")
    hg = G.HostGraph(case["train_edges"], case["test_edges"], n_node=case.n)
    dg, smp = _sampler(hg, cuda_device, hub)
    roots = np.arange(0, hg.n_node, 3, dtype=np.int32)
    trees = smp.build_trees(roots)
    emb_h = synth.embeddings(hg.n_node, d, seed=d)
    bias_h = np.random.RandomState(d).normal(0, 0.3, hg.n_node).astype(np.float32)
    emb = S.pad_embedding(emb_h, cuda_device)
    bias = torch.as_tensor(bias_h).to(cuda_device)
    E = can.pad_rows(emb_h, int(emb.shape[1]))
    _d_pass(smp, hg, trees, emb, bias, roots, cuda_device, seed=d)
    _check_exact(hg, smp, dg, trees, emb, bias, E, bias_h, roots)


def test_c3_roots_with_the_largest_hub(cuda_device):
    """C3 (power-law N = 1M, avg-deg 20, n_emb 128): the 13 828-neighbour hub, three of its neighbours and ordinary roots;
    the host reference evaluates only these rows."""
    import torch
    from graphgan_b200 import graph as G, sampler as S, synth
    from oracle import canonical as can
    n, d = 1_000_000, 128
    hg = G.HostGraph(synth.power_law(n, 20, seed=0), None, n_node=n)
    deg = np.diff(hg.indptr)
    top = int(np.argmax(deg))
    assert deg[top] > 10000
    nb = hg.adj[hg.indptr[top]:hg.indptr[top + 1]]
    ordinary = np.random.RandomState(3).choice(np.flatnonzero(hg.degrees() > 0), 2, replace=False)
    roots = np.unique(np.concatenate([[top], nb[[0, len(nb) // 2, len(nb) - 1]], ordinary])).astype(np.int32)
    dg, smp = _sampler(hg, cuda_device, 128)
    trees = smp.build_trees(roots)
    emb_h = synth.embeddings(n, d, seed=1)
    bias_h = np.random.RandomState(5).normal(0, 0.1, n).astype(np.float32)
    emb = S.pad_embedding(emb_h, cuda_device)
    bias = torch.as_tensor(bias_h).to(cuda_device)
    _d_pass(smp, hg, trees, emb, bias, roots, cuda_device, seed=11)
    dist, ok = _check_exact(hg, smp, dg, trees, emb, bias, can.pad_rows(emb_h, int(emb.shape[1])), bias_h, roots)
    assert ok.all()
    assert np.all(np.abs(dist.sum(1) - 1.0) <= 1e-12)


def _g_statistic(counts, p, total):
    from scipy import stats
    expect = p * total
    big = expect >= 5
    obs = np.concatenate([counts[big], [counts[~big].sum()]]).astype(np.float64)
    exp = np.concatenate([expect[big], [expect[~big].sum()]])
    keep = exp > 0
    obs, exp = obs[keep], exp[keep]
    nz = obs > 0
    g = 2.0 * np.sum(obs[nz] * np.log(obs[nz] / exp[nz]))
    return g, int(keep.sum()) - 1, float(stats.chi2.sf(g, int(keep.sum()) - 1))


@pytest.mark.parametrize("flat_steps", [None, 0])
def test_sampler_frequencies_follow_the_law(flat_steps, cuda_device):
    """2^20 G-mode walks of four CA-GrQc roots through the production sampler (after a D pass has removed fathers):
    nodes of probability 0 are never sampled, no walk of an accepted root voids, and a G-test over the nodes with an
    expected count >= 5 (the rest pooled) does not reject the law."""
    import torch
    from graphgan_b200 import graph as G, sampler as S
    case = loader.load("cagrqc")
    hg = G.HostGraph(case["train_edges"], case["test_edges"], n_node=case.n)
    dg, smp = _sampler(hg, cuda_device, 128)
    if flat_steps is not None:
        smp.flat_steps = flat_steps
    roots = np.argsort(-hg.degrees(), kind="stable")[[0, 5, 40, 200]].astype(np.int32)
    trees = smp.build_trees(roots)
    emb = S.pad_embedding(case.emb_g, cuda_device)
    bias = torch.as_tensor(case.bias_g).to(cuda_device)
    _d_pass(smp, hg, trees, emb, bias, roots, cuda_device, seed=21)
    dist, ok = smp.distribution(emb, bias, trees)
    dist, ok = dist.cpu().numpy(), ok.cpu().numpy()
    per_root = 1 << 18
    out = smp.run(emb, bias, trees, per_root, False, seed=23, pass_tag=5)
    status, samples = out.status.cpu().numpy(), out.samples.cpu().numpy()
    for k in range(len(roots)):
        assert ok[k] == 1
        st, sm = status[k * per_root:(k + 1) * per_root], samples[k * per_root:(k + 1) * per_root]
        assert np.all(st == S.DONE)
        counts = np.bincount(sm, minlength=hg.n_node)
        assert not counts[dist[k] == 0].any()
        g, df, p = _g_statistic(counts, dist[k], per_root)
        print("root %d: G = %.1f, df = %d, p = %.4g (flat_steps %s)" % (roots[k], g, df, p, flat_steps))
        assert p > 1e-4


def test_totals_and_roots_without_a_law(cuda_device):
    """Rows sum to 1 within 1e-12; an isolated root and a root with only a self-loop have root_ok = 0 and all-zero rows."""
    import torch
    from graphgan_b200 import graph as G, sampler as S, synth
    n0 = 3000
    edges = np.concatenate([synth.power_law(n0, 10, seed=1), [[n0 + 1, n0 + 1]]])
    n = n0 + 2                                                # node n0: isolated; node n0 + 1: a self-loop only
    hg = G.HostGraph(edges, None, n_node=n)
    dg, smp = _sampler(hg, cuda_device, 128)
    roots = np.concatenate([synth.pick_roots(hg.degrees(), 200, seed=2), [n0, n0 + 1]]).astype(np.int32)
    trees = smp.build_trees(roots)
    emb = S.pad_embedding(synth.embeddings(n, 64, seed=3), cuda_device)
    bias = torch.zeros(n, dtype=torch.float32, device=cuda_device)
    _d_pass(smp, hg, trees, emb, bias, roots, cuda_device, seed=4)
    dist, ok = smp.distribution(emb, bias, trees)
    dist, ok = dist.cpu().numpy(), ok.cpu().numpy()
    assert ok[-1] == 0 and ok[-2] == 0
    assert not dist[ok == 0].any()
    assert ok[:-2].all()
    assert np.all(np.abs(dist[ok == 1].sum(1) - 1.0) <= 1e-12)
    assert np.all(dist[np.arange(len(roots)), roots] == 0.0)
    # chunked evaluation (a small scratch budget) gives the same bits
    d2, ok2 = smp.distribution(emb, bias, trees, max_scratch_bytes=1)
    assert np.array_equal(d2.cpu().numpy().view(np.uint64), dist.view(np.uint64)) and np.array_equal(ok2.cpu().numpy(), ok)


def test_generator_relevance(cuda_device):
    import torch
    from graphgan_b200 import graph as G, sampler as S, synth
    from graphgan_b200.generator import Generator
    n = 2000
    hg = G.HostGraph(synth.power_law(n, 8, seed=5), None, n_node=n)
    dg, smp = _sampler(hg, cuda_device, 128)
    gen = Generator(n, synth.embeddings(n, 50, seed=6), device=cuda_device)
    gen.sampler = smp
    roots = synth.pick_roots(hg.degrees(), 32, seed=7).astype(np.int32)
    rows = gen.relevance(roots)
    dist, _ = smp.distribution(gen.emb, gen.bias_t, smp.build_trees(roots))
    assert torch.equal(rows, dist)
    rs = np.random.RandomState(8)
    pr = rs.choice(roots, 500)
    pv = rs.randint(0, n, 500)
    pv[:32] = hg.adj[hg.indptr[pr[:32]]]                      # some pairs with a sizeable probability
    got = gen.relevance(pr, pv).cpu().numpy()
    slot = {int(r): k for k, r in enumerate(roots)}
    want = dist.cpu().numpy()[[slot[int(r)] for r in pr], pv]
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    assert (got > 0).any()
