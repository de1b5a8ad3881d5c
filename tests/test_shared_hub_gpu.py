"""Hub groups of a shared level (csrc/walk.cu: flat_dedupe_kernel, flat_hub_reserve_kernel, flat_hub_fill_kernel and the
group branch of flat_choose_kernel): the walks of a root that stand on the same score-cached node at level 2 are drawn
by one warp from ONE build of the node's list.  Bit-exact against the T1 oracle on the C3 graph with the FULL sample_num
of each root, so that groups of many walks occur.

Roots: a hub with 2 000 - 4 000 walks, neighbours of the 13 828-neighbour node and a spread of ordinary roots; D mode
and G mode (400 walks per root, paths recorded).  hub_threshold 64 / 128 / 300: hub lists of a few tiles, and lists
longer than the warp's 2048-entry score buffer (global scratch, per-tile totals in the idle buffer).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FLAT_CTR_WORDS = 1 + 4 * 16          # csrc/walk.cu: FLAT_CTR_WORDS (the hub group words follow them)
FLAT_CTR_ALL = FLAT_CTR_WORDS + 3 * 16


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
    rs = np.random.RandomState(11)
    ordinary = rs.choice(np.flatnonzero(hg.degrees() > 0), 24, replace=False)
    roots = np.unique(np.concatenate([[hub], nb[[1, len(nb) // 2, len(nb) - 2]], ordinary])).astype(np.int32)
    return hg, synth.embeddings(n, 128, seed=1), roots


def _hub_counters(plan, s=2):
    """(hub records, hub owners, hub work items) of level s"""
    import torch
    c = plan._flat[:4 * FLAT_CTR_ALL].view(torch.int32).cpu().numpy()
    return int(c[1 + 4 * s + 1]), int(c[FLAT_CTR_WORDS + 3 * s]), int(c[FLAT_CTR_WORDS + 3 * s + 1])


@pytest.mark.parametrize("hub_threshold", [64, 128, 300])
def test_shared_hub_groups_full_sample_num_c3(c3, hub_threshold, cuda_device):
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
    bias_h = np.random.RandomState(9).normal(0, 0.1, hg.n_node).astype(np.float32)
    bias = torch.as_tensor(bias_h).to(cuda_device)
    E = can.pad_rows(emb_h, int(emb.shape[1]))
    bits = np.zeros(dg.n_bit_words, np.uint32)
    n_gen = 400
    hub_records = hub_owners = 0
    for for_d, tag in ((True, 41), (False, 42)):
        num = hg.degrees()[roots].astype(np.int64) if for_d else np.full(len(roots), n_gen, np.int64)
        ref = can.walk_pass(E, bias_h, hg.indptr, hg.adj, roots, par, num, for_d, bits, seed=17, pass_tag=tag,
                            max_path=0 if for_d else 64)
        plan = smp.plan(trees, torch.as_tensor(num).to(cuda_device) if for_d else n_gen, for_d, 0 if for_d else 64)
        out = smp.run(emb, bias, trees, None, for_d, seed=17, pass_tag=tag, plan=plan)
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
        records, owners, work = _hub_counters(plan)
        assert 0 < owners <= records and owners <= work <= records, (records, owners, work)
        hub_records += records
        hub_owners += owners
    # the hub walks really were grouped: level 2 built fewer hub lists than it drew hub walks
    assert hub_owners < hub_records, (hub_owners, hub_records)
