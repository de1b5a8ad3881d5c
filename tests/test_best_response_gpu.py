"""The game value against the best discriminator and its generator gradient on the device (csrc/best_response.cu, DESIGN.md
section 5.8).

Bars: ok is game_value's; hit is the bits of the documented order applied to gg_generator_dist's dist at the depth-1 nodes
(so G(a) is checked through it); vstar within 1e-13 of the host reference (tests/best_response_oracle.py) and above
V_c(G, D) of game_value; the gradient within 1e-12 of each coordinate's sum of |terms| of the reference, pad columns
exactly 0; bits independent of the chunking, the root order and the call; void, isolated and self-loop-only roots add
nothing; exact_jsd_step lowers the mean JSD to first order; the value line's jsd / hit fields.
"""
import ctypes as C

import numpy as np
import pytest

from tests import best_response_oracle as bro
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


def _fixture_roots(hg, k, seed):
    n = hg.n_node
    if n <= k:
        return np.arange(n, dtype=np.int32)
    top = np.argsort(-hg.degrees(), kind="stable")[:4]
    return np.unique(np.concatenate([top, np.random.RandomState(seed).choice(n, k, replace=False)])).astype(np.int32)


def _hit_from_dist(hg, roots, par, dist, ok):
    """the documented order of hit (lane chains over the root's entries, xor butterfly) on gg_generator_dist's rows"""
    out = np.zeros(len(roots))
    for k, c in enumerate(roots):
        if not ok[k]:
            continue
        a0, a1 = hg.indptr[c], hg.indptr[c + 1]
        ents = [e for e in range(a0, a1) if par[k][hg.adj[e]] == c]
        out[k] = bro._lane_sum([dist[k, hg.adj[e]] for e in ents], [e - a0 for e in ents])
    return out


def _check(hg, dg, smp, trees, roots, G_, D_=None, rows=None, grad=True):
    """value bits against gg_generator_dist / game_value, vstar and the gradient against the "pi" oracle"""
    g_emb, g_bias, Eg, bg = G_
    out = smp.best_response_grad(g_emb, g_bias, trees) if grad else smp.best_response(g_emb, g_bias, trees)
    if grad:
        assert _bits(out[:3]) == _bits(smp.best_response(g_emb, g_bias, trees))
    vs, ht, ok = (x.cpu().numpy() for x in out[:3])
    dist, root_ok = smp.distribution(g_emb, g_bias, trees)
    dist = dist.cpu().numpy()
    par = trees.parent_arrays().cpu().numpy()
    deg = hg.degrees()[roots]
    assert np.array_equal(ok, ((root_ok.cpu().numpy() == 1) & (deg > 0)).astype(np.int32))
    assert _hit_from_dist(hg, roots, par, dist, ok).tobytes() == ht.tobytes()
    bits = dg.d1_bits.cpu().numpy().view(np.uint32)
    wE, wb, aE, ab, per = bro.grad(Eg, bg, hg, roots, par, bits, "pi", rows)
    assert [o["ok"] for o in per] == list(ok)
    assert np.all(np.abs(vs - np.array([o["vstar"] for o in per])) <= 1e-13)
    assert np.all((vs >= -np.log(4.0) - 1e-13) & (vs <= 0))
    if D_ is not None:
        pos, neg, okv = (x.cpu().numpy() for x in smp.game_value(g_emb, g_bias, D_[0], D_[1], trees))
        assert np.array_equal(okv, ok) and np.all(vs[ok == 1] >= (pos + neg)[ok == 1] - 1e-12)
    if grad:
        gE, gb = out[3].cpu().numpy(), out[4].cpu().numpy()
        if rows is not None:
            gE, gb = gE[rows], gb[rows]
        assert np.all(np.abs(gE - wE) <= 1e-12 * aE) and np.all(np.abs(gb - wb) <= 1e-12 * ab), (
            np.max(np.abs(gE - wE) - 1e-12 * aE), np.max(np.abs(gb - wb) - 1e-12 * ab))
        n_emb = int(np.flatnonzero(np.abs(Eg).sum(axis=0))[-1]) + 1
        assert not gE[:, n_emb:].any()                                  # pad columns exactly 0
    return out


@pytest.mark.parametrize("hub", [0, 64, 128, 300])
@pytest.mark.parametrize("name", ["tiny", "rand300", "rand1200", "cagrqc"])
def test_matches_oracle_and_generator_dist(name, hub, cuda_device):
    case, hg, dg, smp = _graph(name, cuda_device, hub)
    roots = _fixture_roots(hg, 40, 1)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, np.random.RandomState(3).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(2).normal(0, 0.3, hg.n_node), cuda_device)
    grad = hub in (0, 128)
    out0 = _check(hg, dg, smp, trees, roots, G_, D_, grad=grad)      # no father entry removed
    assert out0[2].cpu().numpy().any()
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=3)
    assert dg.d1_bits.any()
    out1 = _check(hg, dg, smp, trees, roots, G_, D_, grad=grad)
    if grad:
        assert out0[3].abs().sum().item() > 0


def test_vstar_bounds_v_with_a_trained_discriminator(cuda_device):
    """CA-GrQc with the pretrained D and with a D moved towards D* by exact steps: vstar >= V everywhere"""
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    roots = _fixture_roots(hg, 64, 5)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, case.bias_g, cuda_device)
    D_ = _params(case.emb_d, case.bias_d, cuda_device)
    vs = smp.best_response(G_[0], G_[1], trees)[0].cpu().numpy()
    d_emb, d_bias = D_[0].clone(), D_[1].clone()
    for _ in range(20):                                                 # plain ascent on V: D gets better
        pos, neg, ok, gE, gb = smp.game_value_grad_d(G_[0], G_[1], d_emb, d_bias, trees)
        n = max(int(ok.sum().item()), 1)
        d_emb += (0.1 / n) * gE.float()
        d_bias += (0.1 / n) * gb.float()
    v_before = smp.game_value(G_[0], G_[1], D_[0], D_[1], trees)
    v_after = smp.game_value(G_[0], G_[1], d_emb, d_bias, trees)
    for pos, neg, ok in (v_before, v_after):
        sel = ok.cpu().numpy() == 1
        v = (pos + neg).cpu().numpy()
        assert np.all(vs[sel] >= v[sel] - 1e-12)
    mean = lambda t: float(((t[0] + t[1]).cpu().numpy()[t[2].cpu().numpy() == 1]).mean())
    assert mean(v_after) > mean(v_before)                               # the trained D is closer to D*


@pytest.mark.parametrize("d", [20, 50, 100, 200, 300, 512])
def test_every_row_stride(d, cuda_device):
    from graphgan_b200 import synth
    _, hg, dg, smp = _graph("rand300", cuda_device, 0)
    n = hg.n_node
    rs = np.random.RandomState(d)
    roots = np.sort(rs.choice(np.flatnonzero(hg.degrees() > 0), 12, replace=False)).astype(np.int32)
    G_ = _params(synth.embeddings(n, d, seed=d, sigma=0.3), rs.normal(0, 0.3, n), cuda_device)
    trees = smp.build_trees(roots)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=d)
    out = _check(hg, dg, smp, trees, roots, G_)
    assert int(out[3].shape[1]) == int(G_[0].shape[1])


def test_c3_roots_with_the_largest_hub(cuda_device):
    """C3 (power-law N = 1M, avg-deg 20, n_emb 128): the 13 828-neighbour hub, three of its neighbours and two ordinary
    roots, after a D pass, hub cache on."""
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
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=11)
    rows = np.unique(np.concatenate([roots, nb[:2000], np.random.RandomState(4).choice(n, 2000, replace=False)]))
    out = _check(hg, dg, smp, trees, roots, G_, rows=rows)
    assert out[2].cpu().numpy().all()


def test_bits_do_not_depend_on_chunks_order_or_call(cuda_device):
    import torch
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    roots = _fixture_roots(hg, 60, 4)
    roots = np.concatenate([roots, roots[:3]])                          # duplicates count twice
    G_ = _params(case.emb_g, case.bias_g, cuda_device)
    trees = smp.build_trees(roots)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=8)
    args = (G_[0], G_[1])
    base = _bits(smp.best_response_grad(*args, trees))
    assert _bits(smp.best_response_grad(*args, trees)) == base                             # repeated call
    assert _bits(smp.best_response_grad(*args, trees, max_scratch_bytes=1)) == base        # one root per chunk
    nb = C.c_int64(0)
    smp.lib.gg_best_response_grad_scratch_bytes(hg.n_node, len(hg.adj), 7, C.byref(nb))
    assert _bits(smp.best_response_grad(*args, trees, max_scratch_bytes=nb.value)) == base  # 7 roots per chunk
    assert _bits(smp.best_response(*args, trees, max_scratch_bytes=1)) == base[:3]
    perm = np.random.RandomState(9).permutation(len(roots))
    out = smp.best_response_grad(*args, smp.build_trees(roots[perm]))
    inv = torch.as_tensor(np.argsort(perm)).to(cuda_device)
    assert _bits([x[inv] for x in out[:3]]) + _bits(out[3:]) == base                      # roots in another order


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
    args = (G_[0], G_[1])
    rest = np.delete(good, void[0])
    want = smp.best_response_grad(*args, smp.build_trees(rest))
    roots = np.concatenate([good, [n0, n0 + 1]]).astype(np.int32)
    out = smp.best_response_grad(*args, smp.build_trees(roots))
    ok = out[2].cpu().numpy()
    bad = np.zeros(len(roots), bool)
    bad[[void[0], len(roots) - 2, len(roots) - 1]] = True
    assert not ok[bad].any() and ok[~bad].all()
    assert not out[0].cpu().numpy()[bad].any() and not out[1].cpu().numpy()[bad].any()
    assert _bits(out[3:]) == _bits(want[3:])
    alone = smp.best_response_grad(*args, smp.build_trees(roots[bad]))
    assert not alone[3].any() and not alone[4].any()


def _gan(monkeypatch, tmp_path, cuda_device, name, tag="", **cfg):
    import torch
    from graphgan_b200 import config, graph as G
    from graphgan_b200.graph_gan import GraphGAN
    c = loader.load(name)
    base = dict(n_emb=int(c.emb_g.shape[1]), device=str(cuda_device), seed=5, text_embeddings=False, app="none",
                value_roots=0, exact_roots=64, emb_filenames=[str(tmp_path / ("gen%s.emb" % tag)),
                                                              str(tmp_path / ("dis%s.emb" % tag))],
                result_filename=str(tmp_path / ("res%s.txt" % tag)), model_log=str(tmp_path / "log") + "/")
    base.update(cfg)
    for k, v in base.items():
        monkeypatch.setattr(config, k, v)
    hg = G.HostGraph(c.train_edges, c.test_edges, n_node=c.n)
    gan = GraphGAN(host_graph=hg, node_embed_init_d=c.emb_d, node_embed_init_g=c.emb_g)
    rs = np.random.RandomState(17)
    gan.generator.bias_t.copy_(torch.as_tensor(rs.normal(0, 0.2, hg.n_node).astype(np.float32)))
    return gan


def _mean_jsd(vstar, ok):
    sel = ok.bool()
    return float((vstar[sel] / 2 + np.log(2.0)).sum().item()) / int(sel.sum().item())


@pytest.mark.parametrize("name", ["tiny", "rand300", "cagrqc"])
def test_exact_jsd_step_is_first_order(name, cuda_device, tmp_path, monkeypatch):
    """at lr 1e-4 one exact_jsd_step lowers the mean JSD, and the change is <grad mean JSD, theta_new - theta_old> (fp64,
    actual parameter deltas) within 10 %"""
    gan = _gan(monkeypatch, tmp_path, cuda_device, name)
    roots = gan.exact_roots()
    g = gan.generator
    g.lr = np.float32(1e-4)
    vstar, hit, ok, gE, gb = gan.best_response_grad(roots)
    n = int(ok.sum().item())
    assert n > 0
    e0, b0 = g.emb.double().clone(), g.bias_t.double().clone()
    pre = gan.exact_jsd_step(roots)
    assert _bits(pre) == _bits((vstar, hit, ok))
    pred = float(((gE * (g.emb.double() - e0)).sum() + (gb * (g.bias_t.double() - b0)).sum()).item()) / (2 * n)
    post = gan.best_response(roots)
    actual = _mean_jsd(post[0], post[2]) - _mean_jsd(vstar, ok)
    print("jsd first-order ratio %s: %.4f (change %.3g)" % (name, actual / pred, actual))
    assert actual < 0
    assert abs(actual / pred - 1) <= 0.1, (actual, pred)


def test_value_line_jsd_fields(cuda_device, tmp_path, monkeypatch):
    """jsd / hit end the value line, alone and after gnorm / dnorm / gcos / dcos; the earlier fields keep their bits"""
    import re
    gan = _gan(monkeypatch, tmp_path, cuda_device, "cagrqc", value_roots=16, exact_roots=0)
    from graphgan_b200 import config
    plain = gan.value_line().strip()
    monkeypatch.setattr(config, "value_jsd", True)
    line = gan.value_line().strip()
    m = re.match(r"^(.*) jsd:(\S+) hit:(\S+)$", line)
    assert m and m.group(1) == plain
    vs, ht, ok = (x.cpu().numpy() for x in gan.best_response(gan.value_roots()))
    sel = ok == 1
    assert float(m.group(2)) == float((vs[sel] / 2 + np.log(2.0)).mean())
    assert float(m.group(3)) == float(ht[sel].mean())
    assert 0 <= float(m.group(2)) <= np.log(2.0) and 0 <= float(m.group(3)) <= 1
    for k in ("value_grad", "value_grad_d", "value_gcos", "value_dcos"):
        monkeypatch.setattr(config, k, True)
    full = gan.value_line().strip()
    monkeypatch.setattr(config, "value_jsd", False)
    full0 = gan.value_line().strip()
    assert full == full0 + " jsd:%s hit:%s" % (m.group(2), m.group(3))
