"""The D-mode walk law and the exact expectation of the reference's discriminator step on the device (csrc/gdist.cu,
csrc/value.cu, csrc/value_dgrad.cu; DESIGN.md section 5.7).

Bars: the law (P_D, p_void, root_ok) bit for bit against tests/expected_d_grad_oracle.py, the same bits before and after
a D pass; the expected step per coordinate within 1e-12 of the coordinate's sum of |terms|, pad columns exactly 0; the
bits do not depend on the chunking, the root order or the call; roots that cannot emit rows add exactly 0; the production
D pass (sampler, gg_emit_d_rows, gg_pair_grad_ex mode 0) agrees with the law, the acceptance and the step; dcos.
"""
import ctypes as C
import re

import numpy as np
import pytest
from scipy import stats

from tests import expected_d_grad_oracle as eo
from tests import gdist_oracle as go
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


def _fixture_roots(hg, k, seed):
    n = hg.n_node
    if n <= k:
        return np.arange(n, dtype=np.int32)
    top = np.argsort(-hg.degrees(), kind="stable")[:4]
    return np.unique(np.concatenate([top, np.random.RandomState(seed).choice(n, k, replace=False)])).astype(np.int32)


def _check_law(hg, smp, trees, roots, G_):
    g_emb, g_bias, Eg, bg = G_
    P, pv, ok = (x.cpu().numpy() for x in smp.d_distribution(g_emb, g_bias, trees))
    par = trees.parent_arrays().cpu().numpy()
    wP, wpv, wok = eo.d_laws(Eg, bg, hg, roots, par)
    assert np.array_equal(ok, wok) and np.array_equal(pv, wpv) and np.array_equal(P, wP)
    return P, pv, ok


def _check_step(hg, smp, trees, roots, G_, D_, rows=None):
    (g_emb, g_bias, _, _), (d_emb, d_bias, Ed, bd) = G_, D_
    acc, pv, okr, gE, gb = smp.expected_d_grad(g_emb, g_bias, d_emb, d_bias, trees)
    P, pv2, ok = (x.cpu().numpy() for x in smp.d_distribution(g_emb, g_bias, trees))
    acc, pv, okr, gE, gb = (x.cpu().numpy() for x in (acc, pv, okr, gE, gb))
    assert np.array_equal(pv, pv2)
    wE, wb, aE, ab, wacc, wok = eo.grad(Ed, bd, hg, roots, P, pv, ok, "fp32", rows)
    assert np.array_equal(acc, wacc) and np.array_equal(okr, wok)          # square-and-multiply, bit for bit
    if rows is not None:
        gE, gb = gE[rows], gb[rows]
    assert np.all(np.abs(gE - wE) <= 1e-12 * aE) and np.all(np.abs(gb - wb) <= 1e-12 * ab), (
        np.max(np.abs(gE - wE) - 1e-12 * aE), np.max(np.abs(gb - wb) - 1e-12 * ab))
    n_emb = int(np.flatnonzero(np.abs(Ed).sum(axis=0))[-1]) + 1
    assert not gE[:, n_emb:].any()                                          # pad columns exactly 0
    print("%d ok_ref roots of %d, p_void > 0 at %d" % (int(okr.sum()), len(roots), int((pv > 0).sum())))
    return acc, okr, gE, gb


@pytest.mark.parametrize("hub", [0, 64, 128, 300])
@pytest.mark.parametrize("name", ["tiny", "rand300", "rand1200", "cagrqc"])
def test_law_matches_oracle_before_and_after_a_d_pass(name, hub, cuda_device):
    case, hg, dg, smp = _graph(name, cuda_device, hub)
    roots = _fixture_roots(hg, 30, 1)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, np.random.RandomState(3).normal(0, 0.2, hg.n_node), cuda_device)
    before = _bits(smp.d_distribution(G_[0], G_[1], trees))
    _check_law(hg, smp, trees, roots, G_)
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=3)
    assert dg.d1_bits.any()
    _check_law(hg, smp, trees, roots, G_)
    assert _bits(smp.d_distribution(G_[0], G_[1], trees)) == before


@pytest.mark.parametrize("name", ["tiny", "rand300", "rand1200", "cagrqc"])
def test_step_matches_oracle(name, cuda_device):
    case, hg, dg, smp = _graph(name, cuda_device, 128)
    roots = _fixture_roots(hg, 30, 1)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, np.random.RandomState(3).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(2).normal(0, 0.3, hg.n_node), cuda_device)
    acc, okr, gE, _ = _check_step(hg, smp, trees, roots, G_, D_)
    assert okr.any() and np.abs(gE).sum() > 0


@pytest.mark.parametrize("d", [20, 50, 100, 200, 300, 512])
def test_every_row_stride(d, cuda_device):
    from graphgan_b200 import synth
    _, hg, dg, smp = _graph("rand300", cuda_device, 0)
    n = hg.n_node
    rs = np.random.RandomState(d)
    roots = np.sort(rs.choice(np.flatnonzero(hg.degrees() > 0), 12, replace=False)).astype(np.int32)
    G_ = _params(synth.embeddings(n, d, seed=d, sigma=0.3), rs.normal(0, 0.3, n), cuda_device)
    D_ = _params(synth.embeddings(n, d, seed=d + 1, sigma=0.3), rs.normal(0, 0.3, n), cuda_device)
    trees = smp.build_trees(roots)
    _check_law(hg, smp, trees, roots, G_)
    _check_step(hg, smp, trees, roots, G_, D_)


def test_c3_roots_with_the_largest_hub(cuda_device):
    """C3 (power-law N = 1M, avg-deg 20, n_emb 128): the 13 828-neighbour hub, three of its neighbours and two ordinary
    roots, after a D pass, with the hub score cache on."""
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
    before = _bits(smp.d_distribution(G_[0], G_[1], trees))
    _d_pass(smp, hg, trees, G_[0], G_[1], roots, cuda_device, seed=11)
    _, pv, ok = _check_law(hg, smp, trees, roots, G_)
    assert _bits(smp.d_distribution(G_[0], G_[1], trees)) == before
    assert ok.all()
    print("C3 p_void per root:", dict(zip(roots.tolist(), pv.tolist())))
    rows = np.unique(np.concatenate([roots, nb[:2000], np.random.RandomState(4).choice(n, 2000, replace=False)]))
    _check_step(hg, smp, trees, roots, G_, D_, rows)


def test_d_law_is_the_g_law_without_leaves_and_with_every_bit_set(cuda_device):
    import torch
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    roots = _fixture_roots(hg, 60, 5)
    trees = smp.build_trees(roots)
    G_ = _params(case.emb_g, case.bias_g, cuda_device)
    P, pv, ok = smp.d_distribution(G_[0], G_[1], trees)
    dg.d1_bits.fill_(-1)
    dist, g_ok = smp.distribution(G_[0], G_[1], trees)
    sel = ((pv == 0) & (ok == 1)).cpu().numpy()
    assert sel.sum() >= 5
    assert torch.equal(g_ok[torch.as_tensor(sel).to(cuda_device)], ok[torch.as_tensor(sel).to(cuda_device)])
    assert _bits([P[torch.as_tensor(sel).to(cuda_device)]]) == _bits([dist[torch.as_tensor(sel).to(cuda_device)]])


def test_one_root_is_a_k_times_the_game_gradient_with_law_q(cuda_device):
    """For one root, the expected step is a_k = deg_c P_acc times game_value_grad_d fed law = (Q, root_ok): the same
    passes, W scaled by a_k before the sums, so the two agree to fp64 rounding (1e-13 of the sums of |terms|)."""
    import torch
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    G_ = _params(case.emb_g, np.random.RandomState(3).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(2).normal(0, 0.3, hg.n_node), cuda_device)
    roots = _fixture_roots(hg, 40, 2)
    trees = smp.build_trees(roots)
    P, pv, ok = smp.d_distribution(G_[0], G_[1], trees)
    acc_all = smp.expected_d_grad(G_[0], G_[1], D_[0], D_[1], trees)[0].cpu().numpy()
    n_checked = 0
    for k in np.flatnonzero(acc_all > 0)[:6]:
        one = trees.select(torch.tensor([k], device=cuda_device))
        acc, _, okr, gE, gb = smp.expected_d_grad(G_[0], G_[1], D_[0], D_[1], one)
        q = (P[k:k + 1] / (1.0 - pv[k])).contiguous()
        yE, yb = smp.game_value_grad_d(G_[0], G_[1], D_[0], D_[1], one, law=(q, ok[k:k + 1].contiguous()))[3:]
        a = float(hg.degrees()[roots[k]]) * float(acc.item())
        _, _, aE, ab = dgo.grad(D_[2], D_[3], hg, [int(roots[k])], [q[0].cpu().numpy()], [1], "fp32")
        assert np.all(np.abs(gE.cpu().numpy() - a * yE.cpu().numpy()) <= 1e-13 * a * aE + 1e-300)
        assert np.all(np.abs(gb.cpu().numpy() - a * yb.cpu().numpy()) <= 1e-13 * a * ab + 1e-300)
        n_checked += 1
    assert n_checked >= 3


def test_bits_do_not_depend_on_chunks_order_or_call(cuda_device):
    import torch
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    roots = _fixture_roots(hg, 60, 4)
    roots = np.concatenate([roots, roots[:3]])                              # duplicates count twice
    G_ = _params(case.emb_g, case.bias_g, cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(7).normal(0, 0.3, hg.n_node), cuda_device)
    trees = smp.build_trees(roots)
    args = (G_[0], G_[1], D_[0], D_[1])
    base = _bits(smp.expected_d_grad(*args, trees))
    law = _bits(smp.d_distribution(G_[0], G_[1], trees))
    assert _bits(smp.expected_d_grad(*args, trees)) == base                                     # repeated call
    assert _bits(smp.expected_d_grad(*args, trees, max_scratch_bytes=1)) == base                # one root per chunk
    assert _bits(smp.d_distribution(G_[0], G_[1], trees, max_scratch_bytes=1)) == law
    nb, ng = C.c_int64(0), C.c_int64(0)
    smp.lib.gg_generator_dist_scratch_bytes(hg.n_node, len(hg.adj), 7, C.byref(ng))
    smp.lib.gg_expected_d_grad_scratch_bytes(hg.n_node, int(D_[0].shape[1]), 7, C.byref(nb))
    assert _bits(smp.expected_d_grad(*args, trees, max_scratch_bytes=nb.value + ng.value)) == base  # 7 roots per chunk
    perm = np.random.RandomState(9).permutation(len(roots))
    out = smp.expected_d_grad(*args, smp.build_trees(roots[perm]))
    inv = torch.as_tensor(np.argsort(perm)).to(cuda_device)
    assert _bits([x[inv] for x in out[:3]]) + _bits(out[3:]) == base                          # roots in another order


def test_roots_that_emit_nothing_add_nothing(cuda_device):
    """An isolated root, a self-loop-only root and a root whose every walk voids (a single depth-1 leaf) have ok_ref = 0
    and leave the gradient exactly as the other roots make it."""
    from graphgan_b200 import graph as G, sampler as S, synth
    n0 = 3000
    edges = np.concatenate([synth.power_law(n0, 10, seed=1), [[n0 + 1, n0 + 1], [n0 + 2, n0 + 3]]])
    n = n0 + 4
    hg = G.HostGraph(edges, None, n_node=n)
    dg = G.DeviceGraph(hg, cuda_device)
    smp = S.WalkSampler(dg, hub_threshold=128)
    good = np.sort(synth.pick_roots(hg.degrees()[:n0], 40, seed=2)).astype(np.int32)
    G_ = _params(synth.embeddings(n, 64, seed=3), np.zeros(n), cuda_device)
    D_ = _params(synth.embeddings(n, 64, seed=4), np.random.RandomState(5).normal(0, 0.3, n), cuda_device)
    args = (G_[0], G_[1], D_[0], D_[1])
    want = smp.expected_d_grad(*args, smp.build_trees(good))
    assert want[2].cpu().numpy().any()
    bad = np.array([n0, n0 + 1, n0 + 2], np.int32)
    roots = np.concatenate([good, bad])
    out = smp.expected_d_grad(*args, smp.build_trees(roots))
    acc, pv, okr = (x.cpu().numpy() for x in out[:3])
    assert not okr[-3:].any() and not acc[-3:].any() and np.array_equal(okr[:-3], want[2].cpu().numpy())
    assert pv[-1] == 1.0 and pv[-3] == 0.0 and pv[-2] == 0.0
    assert _bits(out[3:]) == _bits(want[3:])
    alone = smp.expected_d_grad(*args, smp.build_trees(bad))
    assert not alone[0].any() and not alone[3].any() and not alone[4].any()


def _pair_grad_rows(lib, dev, ci, vi, label, emb, bias):
    """gg_pair_grad_ex(mode 0, batch_total 1, lambda 0) of the rows (ci, vi, label): the sum of the per-row gradients of
    bce -> dense fp64 (grad_rows [N, ld], grad_bias [N])"""
    import torch
    from graphgan_b200 import _cabi
    from graphgan_b200._cabi import ptr
    B, (n, ld) = int(ci.shape[0]), emb.shape
    aux = label.to(torch.float32).contiguous()
    nu = torch.zeros(1, dtype=torch.int32, device=dev)
    ids = torch.empty(2 * B, dtype=torch.int32, device=dev)
    rows = torch.empty((2 * B, ld), dtype=torch.float32, device=dev)
    gb = torch.empty(2 * B, dtype=torch.float32, device=dev)
    slot = torch.full((n,), -1, dtype=torch.int32, device=dev)
    nb = C.c_int64(0)
    _cabi.check(lib.gg_pair_grad_scratch_bytes(B, ld, C.byref(nb)))
    scratch = torch.empty(max(nb.value, 256), dtype=torch.uint8, device=dev)
    _cabi.check(lib.gg_pair_grad_ex(0, B, 1, ptr(ci), ptr(vi), ptr(aux), ptr(emb), ptr(bias), ld, 0.0, ptr(nu), ptr(ids),
                                    ptr(rows), ptr(gb), ptr(slot), ptr(scratch), nb.value, 0, None), "gg_pair_grad_ex")
    U = int(nu.item())
    dE = torch.zeros((n, ld), dtype=torch.float64, device=dev)
    db = torch.zeros(n, dtype=torch.float64, device=dev)
    dE[ids[:U].long()] = rows[:U].double()
    db[ids[:U].long()] = gb[:U].double()
    return dE, db


def _production_roots(hg, smp, G_, D_, cuda_device):
    """four CA-GrQc roots with 0.1 < P_acc < 0.9, spread over the degrees"""
    cand = np.flatnonzero(hg.degrees() > 1).astype(np.int32)
    acc = smp.expected_d_grad(G_[0], G_[1], D_[0], D_[1], smp.build_trees(cand))[0].cpu().numpy()
    mid = cand[(acc > 0.1) & (acc < 0.9)]
    assert len(mid) >= 4
    mid = mid[np.argsort(-hg.degrees()[mid], kind="stable")]
    return np.sort(mid[np.linspace(0, len(mid) - 1, 4).astype(int)]).astype(np.int32)


def test_production_d_walks_follow_the_law(cuda_device):
    """2^20 D walks of four CA-GrQc roots from the production sampler (sample_num 2^18 per root, not finalized): the
    per-walk void rate against p_void, and a G-test of the stop nodes against Q (cells with expected count < 5 pooled)."""
    import torch
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    G_ = _params(case.emb_g, np.random.RandomState(12).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(10).normal(0, 0.3, hg.n_node), cuda_device)
    roots = _production_roots(hg, smp, G_, D_, cuda_device)
    trees = smp.build_trees(roots)
    P, pv, ok = (x.cpu().numpy() for x in smp.d_distribution(G_[0], G_[1], trees))
    per_root = 1 << 18
    out = smp.run(G_[0], G_[1], trees, torch.full((4,), per_root, dtype=torch.int64, device=cuda_device), True, seed=41,
                  pass_tag=9, finalize=False)
    status, samples = out.status.cpu().numpy(), out.samples.cpu().numpy()
    for k, c in enumerate(roots):
        st, sm = status[k * per_root:(k + 1) * per_root], samples[k * per_root:(k + 1) * per_root]
        assert np.all((st == 1) | (st == 2))
        rate = float((st == 2).mean())
        z = (rate - pv[k]) / np.sqrt(pv[k] * (1 - pv[k]) / per_root)
        q = P[k] / (1.0 - pv[k])
        cnt = np.bincount(sm[st == 1], minlength=hg.n_node)
        assert not cnt[q == 0].any()
        e = q * cnt.sum()
        big = e >= 5
        O = np.concatenate([cnt[big], [cnt[~big].sum()]])
        E = np.concatenate([e[big], [e[~big].sum()]])
        keep = E > 0
        O, E = O[keep], E[keep]
        g = 2.0 * float(np.sum(np.where(O > 0, O * np.log(np.maximum(O, 1) / E), 0.0)))
        p = float(stats.chi2.sf(g, len(O) - 1)) if len(O) > 1 else 1.0
        print("root %d: p_void %.6f, void rate %.6f, z = %.2f; G = %.1f on %d cells, p = %.3g" % (c, pv[k], rate, z, g,
                                                                                                  len(O), p))
        assert abs(z) < 5 and p > 1e-4


def test_production_d_passes_match_acceptance_and_step(cuda_device):
    """2^12 finalized D passes (sample_num = deg, distinct pass_tags) of the same four roots: the acceptance frequency of
    each root against P_acc, and the mean over passes of gg_emit_d_rows -> gg_pair_grad_ex (mode 0, lambda 0, the sum
    over the rows: the batch mean undone), negated, against the expected step on 8 random directions: |z| < 5."""
    import torch
    case, hg, dg, smp = _graph("cagrqc", cuda_device, 128)
    G_ = _params(case.emb_g, np.random.RandomState(12).normal(0, 0.2, hg.n_node), cuda_device)
    D_ = _params(case.emb_d, np.random.RandomState(10).normal(0, 0.3, hg.n_node), cuda_device)
    roots = _production_roots(hg, smp, G_, D_, cuda_device)
    trees = smp.build_trees(roots)
    acc, _, okr, gE, gb = smp.expected_d_grad(G_[0], G_[1], D_[0], D_[1], trees)
    acc = acc.cpu().numpy()
    n, ld = hg.n_node, int(D_[0].shape[1])
    n_emb = case.emb_d.shape[1]
    rs = np.random.RandomState(31)
    dirE = np.zeros((8, n, ld))
    dirE[:, :, :n_emb] = rs.normal(0, 1, (8, n, n_emb))
    dirs = torch.as_tensor(np.concatenate([dirE.reshape(8, -1), rs.normal(0, 1, (8, n))], axis=1)).to(cuda_device)
    exact = (dirs @ torch.cat([gE.reshape(-1), gb])).cpu().numpy()
    deg = torch.as_tensor(hg.degrees()[roots].astype(np.int64)).to(cuda_device)
    n_pass = 1 << 12
    accepted = np.zeros((n_pass, 4))
    proj = np.zeros((n_pass, 8))
    for t in range(n_pass):
        out = smp.run(G_[0], G_[1], trees, deg, True, seed=77, pass_tag=1000 + t)
        accepted[t] = out.root_ok.cpu().numpy()
        c, nb_, lb, n_rows = smp.emit_d_rows(out)
        k = int(n_rows.item())
        if k == 0:
            continue
        pE, pb = _pair_grad_rows(smp.lib, cuda_device, c[:k].contiguous(), nb_[:k].contiguous(), lb[:k], D_[0], D_[1])
        proj[t] = -(dirs @ torch.cat([pE.reshape(-1), pb])).cpu().numpy()
    for j, c in enumerate(roots):
        f = accepted[:, j].mean()
        z = (f - acc[j]) / np.sqrt(acc[j] * (1 - acc[j]) / n_pass)
        print("root %d: P_acc %.5f, accepted %.5f, z = %.2f" % (c, acc[j], f, z))
        assert abs(z) < 5
    for q in range(8):
        z = (proj[:, q].mean() - exact[q]) / (proj[:, q].std(ddof=1) / np.sqrt(n_pass))
        print("direction %d: exact %.6g, estimate %.6g, z = %.2f" % (q, exact[q], proj[:, q].mean(), z))
        assert abs(z) < 5


def _train(monkeypatch, tmp_path, cuda_device, flags, tag):
    from graphgan_b200 import config, graph as G
    from graphgan_b200.graph_gan import GraphGAN
    c = loader.load("cagrqc")
    for k, v in dict(n_emb=50, n_epochs=1, n_epochs_dis=1, dis_interval=1, n_epochs_gen=1, gen_interval=1,
                     n_sample_gen=2, device=str(cuda_device), seed=5, value_roots=16, text_embeddings=False).items():
        monkeypatch.setattr(config, k, v)
    for k in ("value_grad", "value_grad_d", "value_gcos", "value_dcos"):
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


@pytest.mark.parametrize("flags", [(), ("value_grad", "value_grad_d", "value_gcos")])
def test_trainer_dcos(flags, cuda_device, tmp_path, monkeypatch):
    """One short CA-GrQc epoch with value_roots = 16: with value_dcos the value line ends in dcos in [-1, 1], and the line
    before it is the bits of the line without the flag, alone and after gnorm, dnorm and gcos."""
    import torch
    gan, lines = _train(monkeypatch, tmp_path, cuda_device, flags + ("value_dcos",), "c")
    _, lines0 = _train(monkeypatch, tmp_path, cuda_device, flags, "0")
    assert [ln.split(":")[0] for ln in lines] == ["gen", "dis", "value"] * 2
    pat = re.compile(r"^(value:.*) dcos:(\S+)$")
    for ln, ln0 in zip(lines, lines0):
        if not ln.startswith("value:"):
            assert ln == ln0
            continue
        m = pat.match(ln)
        assert m, ln
        assert m.group(1) == ln0 and -1.0 <= float(m.group(2)) <= 1.0
    rE, rb = gan.expected_d_grad(gan.value_roots())[3:]
    gE, gb = gan.game_value_grad_d(gan.value_roots())[3:]
    k = gan.discriminator.n_emb
    cos = float(((rE[:, :k] * gE[:, :k]).sum() + (rb * gb).sum()) / torch.sqrt(
        ((rE[:, :k] ** 2).sum() + (rb ** 2).sum()) * ((gE[:, :k] ** 2).sum() + (gb ** 2).sum())))
    assert abs(float(pat.match(lines[5]).group(2)) - cos) <= 1e-12
