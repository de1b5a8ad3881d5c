"""Shared level-synchronous steps (csrc/walk.cu: flat_dedupe_kernel / flat_draw_kernel): from step 2 on, the walks of a
root that stand on the same node draw from ONE candidate list and CDF.  Bit-exact against the T1 oracle on the C3 graph
with the FULL sample_num of each root -- the C3 parity test caps a root at 40 walks, which hides most repeats.

Roots: a hub with thousands of walks (repeats at step 2 certainly occur), neighbours of the 13 828-neighbour node and a
spread of ordinary roots; D mode and G mode (many walks per root, paths recorded).  hub_threshold 300 makes nodes of up
to 299 neighbours on-demand items, so their shared CDFs span several 32-entry tiles.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FLAT_CTR_WORDS = 1 + 4 * 16          # csrc/walk.cu: FLAT_CTR_WORDS


@pytest.fixture(scope="module")
def c3():
    from graphgan_b200 import graph as G, synth
    n = 1_000_000
    hg = G.HostGraph(synth.power_law(n, 20, seed=0), None, n_node=n)
    deg = np.diff(hg.indptr)
    top = int(np.argmax(deg))
    assert deg[top] > 10000
    nb = hg.adj[hg.indptr[top]:hg.indptr[top + 1]]
    hub = int(np.flatnonzero((deg >= 2000) & (deg <= 4000))[0])      # a root with 2 000 - 4 000 walks
    rs = np.random.RandomState(7)
    ordinary = rs.choice(np.flatnonzero(hg.degrees() > 0), 24, replace=False)
    roots = np.unique(np.concatenate([[hub], nb[[0, len(nb) // 3, len(nb) - 1]], ordinary])).astype(np.int32)
    return hg, synth.embeddings(n, 128, seed=1), roots


def _level_counters(plan):
    import torch
    c = plan._flat[:4 * FLAT_CTR_WORDS].view(torch.int32).cpu().numpy()
    return {s: (int(c[1 + 4 * s]), int(c[1 + 4 * s + 1]), int(c[1 + 4 * s + 2])) for s in range(1, 5)}


@pytest.mark.parametrize("hub_threshold", [128, 300])
def test_shared_levels_full_sample_num_c3(c3, hub_threshold, cuda_device):
    import torch
    from graphgan_b200 import graph as G, sampler as S
    from oracle import canonical as can
    hg, emb_h, roots = c3
    dg = G.DeviceGraph(hg, cuda_device)
    smp = S.WalkSampler(dg, hub_threshold=hub_threshold)
    smp.flat_steps = 4
    trees = smp.build_trees(roots)
    par = trees.parent_arrays().cpu().numpy()
    assert np.array_equal(par, can.bfs_parents(hg.indptr, hg.adj, roots))
    emb = S.pad_embedding(emb_h, cuda_device)
    bias_h = np.random.RandomState(5).normal(0, 0.1, hg.n_node).astype(np.float32)
    bias = torch.as_tensor(bias_h).to(cuda_device)
    E = can.pad_rows(emb_h, int(emb.shape[1]))
    bits = np.zeros(dg.n_bit_words, np.uint32)
    n_gen = 400
    for for_d, tag in ((True, 31), (False, 32)):
        num = hg.degrees()[roots].astype(np.int64) if for_d else np.full(len(roots), n_gen, np.int64)
        ref = can.walk_pass(E, bias_h, hg.indptr, hg.adj, roots, par, num, for_d, bits, seed=13, pass_tag=tag,
                            max_path=0 if for_d else 64)
        plan = smp.plan(trees, torch.as_tensor(num).to(cuda_device) if for_d else n_gen, for_d, 0 if for_d else 64)
        out = smp.run(emb, bias, trees, None, for_d, seed=13, pass_tag=tag, plan=plan)
        W = ref.samples.shape[0]
        assert W == plan.n_walks and (not for_d or W > 2000)
        assert np.array_equal(out.status.cpu().numpy()[:W], ref.status)
        assert np.array_equal(out.samples.cpu().numpy()[:W], ref.samples)
        assert np.array_equal(out.wsteps.cpu().numpy()[:W], ref.wsteps)
        assert np.array_equal(out.wsuml.cpu().numpy()[:W], ref.wsuml)
        assert np.array_equal(out.root_ok.cpu().numpy()[:len(roots)], ref.root_ok)
        assert np.array_equal(dg.d1_bits.cpu().numpy().view(np.uint32), bits)
        cnt = out.counters_host()
        assert (cnt["steps"], cnt["sum_l"], cnt["path_overflow"]) == (ref.steps, ref.sum_l, ref.path_overflow)
        if not for_d:
            assert np.array_equal(out.path_len.cpu().numpy()[:W], ref.path_len)
            gp = out.paths.cpu().numpy()
            for w in np.flatnonzero(ref.status == can.DONE):
                assert np.array_equal(gp[w, :ref.path_len[w]], ref.paths[w, :ref.path_len[w]])
        # the shared path really shared: level 2 has fewer distinct (root, node) items than walks on non-cached nodes
        records, hubs, distinct = _level_counters(plan)[2]
        assert 0 < distinct < records - hubs, (records, hubs, distinct)
