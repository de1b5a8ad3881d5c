"""The walk sampler (csrc/walk.cu) at the batch size bench.py runs, where it takes paths that small root batches never do:

  depth-1 chunk queue   step1_cdf_kernel hands out the first S1_SINGLES (root, neighbour) pairs one per queue item and the
                        rest in chunks of S1_CHUNK; only a batch whose roots have more than S1_SINGLES neighbours in all
                        (plan.nq) reaches the chunks;
  split hub groups      on the shared level 2, a group of more than HUB_GROUP_MAX walks of one root on one score-cached
                        node is cut into several work items (flat_hub_reserve_kernel, the group branch of
                        flat_choose_kernel);
  large flat buffers    the level-2 table and CDF slab are sized from the walk count: ~312 k D walks here, a 2^20-slot
                        table, like bench.py's 322 k.

Workload: C3 (power-law N = 1M, avg-deg 20, n_emb = 128), the 32 highest-degree nodes plus a 2 500-root pick_roots spread,
a D pass with sample_num = deg(root) and a G pass (20 walks, max_path 64) that reads the D pass's father-removal bits,
hub_threshold 128 and flat_steps 4 (the bench defaults).  The biases are random, plus +4 on one neighbour p of the
top-degree node and +6 on its score-cached tree children x that have children of their own, +4 on those: many of the top root's 13 828
walks go to p at step 0 and on to the x, so level 2 holds hub groups of several hundred walks, each walk drawing
between the father p and the x's children (whose bias matches p's, so the draw decides).

Checks: the thresholds were crossed (read back from the sampler's buffers); a stratified root sample is bit-exact against
the T1 oracle (oracle/gg_oracle.c), every walk of the roots with at most CAP walks and the first CAP walks of the larger
ones (the Philox draw of walk k does not depend on the walk count); the D rows of every root equal prepare_data_for_d's
rows built from the sampled nodes; and every root's outputs are the same bits however the roots are batched and whichever
sampler options are on.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FLAT_CTR_WORDS = 1 + 4 * 16          # csrc/walk.cu: FLAT_CTR_WORDS (the hub group words follow them)
FLAT_CTR_ALL = FLAT_CTR_WORDS + 3 * 16
S1_SINGLES = 65536                   # csrc/walk.cu: S1_SINGLES (queue items after it are chunks of pairs)
HUB_GROUP_MAX = 128                  # csrc/walk.cu: HUB_GROUP_MAX (a larger hub group is split into work items)
N_TOP, N_SPREAD = 32, 2500
HUB_THRESHOLD, FLAT_STEPS, N_GEN, MAX_PATH = 128, 4, 20, 64
SEED, TAG_D, TAG_G = 23, 51, 52
CAP = 64                             # walks per root that the oracle runs
SLICE_ROOTS = 64


def _sampler(dg, flat_steps=FLAT_STEPS, hub_threshold=HUB_THRESHOLD, **kw):
    from graphgan_b200 import sampler as S
    smp = S.WalkSampler(dg, hub_threshold=hub_threshold, **kw)
    smp.flat_steps = flat_steps
    return smp


def _flat_table(plan, hub_threshold=HUB_THRESHOLD):
    """(keys, gcnt) of the shared level's hash table in the flat-step scratch: the offsets mirror csrc/walk.cu
    flat_layout, and the total must equal the size the library asked for.  Only level 2 shares, so the table still
    holds level 2 after the pass: key = root slot * n_node + node, gcnt = walks of the key's hub group."""
    W = max(plan.n_walks, 1)
    stride = (hub_threshold + 31) // 32 * 32
    cap = 1
    while cap < 2 * W:
        cap <<= 1
    off = 0
    offs = []
    for nbytes in (4 * FLAT_CTR_ALL, 16 * W, 16 * W, 16 * W, 4 * W, 4 * W, 4 * W * stride,
                   8 * cap, 4 * cap, 4 * W, 4 * W, 8 * W * (stride + 1), 4 * cap, 4 * cap, 4 * W, 16 * W):
        offs.append(off)
        off += (nbytes + 255) // 256 * 256
    buf = plan._flat
    assert off == buf.numel(), "csrc/walk.cu flat_layout changed: update _flat_table"
    import torch
    keys = buf[offs[7]:offs[7] + 8 * cap].view(torch.int64).cpu().numpy()
    gcnt = buf[offs[12]:offs[12] + 4 * cap].view(torch.int32).cpu().numpy()
    return keys, gcnt


def _hub_counters(plan, s=2):
    """(hub records, hub owners, hub work items) of level s"""
    import torch
    c = plan._flat[:4 * FLAT_CTR_ALL].view(torch.int32).cpu().numpy()
    return int(c[1 + 4 * s + 1]), int(c[FLAT_CTR_WORDS + 3 * s]), int(c[FLAT_CTR_WORDS + 3 * s + 1])


def _host(out, dg):
    """one pass's outputs on the host; paths past path_len (never written) read -1"""
    W, R = out.n_walks, out.n_roots
    res = dict(samples=out.samples[:W].cpu().numpy(), status=out.status[:W].cpu().numpy(),
               wsteps=out.wsteps[:W].cpu().numpy(), wsuml=out.wsuml[:W].cpu().numpy(),
               root_ok=out.root_ok[:R].cpu().numpy(), bits=dg.d1_bits.cpu().numpy().view(np.uint32).copy(),
               counters=out.counters_host())
    if out.paths is not None:
        pl = out.path_len[:W].cpu().numpy()
        keep = np.arange(out.max_path)[None, :] < np.minimum(pl, out.max_path)[:, None]
        res["path_len"] = pl
        res["paths"] = np.where(keep, out.paths[:W].cpu().numpy(), -1)
    return res


def _passes(smp, dg, trees, ranges, deg, emb, bias, keep=False):
    """The D pass (bits zeroed first) over every range [lo, hi) of the roots of `trees`, then the G pass over every
    range; the outputs of each pass concatenated in range order, the counters summed.  keep: also return the last
    range's (plan, output) per pass."""
    import torch
    dg.d1_bits.zero_()
    res, kept = {}, {}
    R = int(trees.roots.shape[0])
    for for_d, tag in ((True, TAG_D), (False, TAG_G)):
        parts = []
        for lo, hi in ranges:
            tb = trees if (lo, hi) == (0, R) else trees.slice(lo, hi)      # (a slice copies its tree rows)
            num = torch.as_tensor(deg[tb.roots.cpu().numpy()].astype(np.int64)).to(smp.device) if for_d else N_GEN
            plan = smp.plan(tb, num, for_d, 0 if for_d else MAX_PATH)
            out = smp.run(emb, bias, tb, None, for_d, seed=SEED, pass_tag=tag, plan=plan)
            parts.append(_host(out, dg))
            if keep:
                kept[for_d] = (plan, out)
        r = {k: np.concatenate([p[k] for p in parts]) for k in parts[0] if k not in ("bits", "counters")}
        r["bits"] = parts[-1]["bits"]
        r["counters"] = {k: sum(p["counters"][k] for p in parts) for k in parts[0]["counters"]}
        res[for_d] = r
    return (res, kept) if keep else res


@pytest.fixture(scope="module")
def c3(cuda_device):
    import torch
    from graphgan_b200 import graph as G, sampler as S, synth
    from oracle import canonical as can
    n = 1_000_000
    hg = G.HostGraph(synth.power_law(n, 20, seed=0), None, n_node=n)
    dw = np.diff(hg.indptr)
    deg = hg.degrees()
    top = int(np.argmax(dw))
    assert dw[top] > 10000
    emb_h = synth.embeddings(n, 128, seed=1)
    bias_h = np.random.RandomState(9).normal(0, 0.1, n).astype(np.float32)
    # d2: score-cached depth-2 nodes of the top's tree with children of their own (a group on a one-candidate list draws
    # nothing); p: the neighbour of the top node with the highest score among their parents
    par = can.bfs_parents(hg.indptr, hg.adj, [top])[0]
    n_child = np.bincount(par[par >= 0], minlength=n)
    d2 = np.flatnonzero((dw >= HUB_THRESHOLD) & (par >= 0) & (n_child >= 2))
    d2 = d2[(par[d2] != top) & (par[par[d2]] == top)]
    ps = np.unique(par[d2])
    p = int(ps[np.argmax(emb_h[ps] @ emb_h[top] + bias_h[ps])])
    xs = d2[par[d2] == p]
    bias_h[p] += 4.0
    bias_h[xs] += 6.0
    bias_h[np.flatnonzero(np.isin(par, xs))] += 4.0     # level 2 draws between p and these, not p alone
    order = np.argsort(-dw, kind="stable")
    roots = np.unique(np.concatenate([order[:N_TOP], synth.pick_roots(deg, N_SPREAD, seed=0)])).astype(np.int32)
    dg = G.DeviceGraph(hg, cuda_device)
    smp = _sampler(dg)
    trees = smp.build_trees(roots)
    emb = S.pad_embedding(emb_h, cuda_device)
    bias = torch.as_tensor(bias_h).to(cuda_device)
    res, kept = _passes(smp, dg, trees, [(0, len(roots))], deg, emb, bias, keep=True)
    plan_d, out_d = kept[True]
    plan_g = kept[False][0]
    # what the thresholds saw, read before the buffers go
    b = plan_d.depth1_buffers(smp)
    cnt, s1_order, s1_slot = (b[k].cpu().numpy() for k in ("cnt", "order", "slot"))
    keys, gcnt = _flat_table(plan_d)
    center, neighbor, label, n_rows = smp.emit_d_rows(out_d)
    k = int(n_rows.item())
    info = dict(nq=plan_d.nq, n_walks_d=plan_d.n_walks, n_walks_g=plan_g.n_walks, hub_d=_hub_counters(plan_d),
                hub_g=_hub_counters(plan_g), cnt=cnt, s1_order=s1_order, s1_slot=s1_slot, keys=keys, gcnt=gcnt,
                walk_ptr=plan_d.walk_ptr.cpu().numpy(), row_ptr=plan_d.row_ptr.cpu().numpy(),
                rows=(center[:k].cpu().numpy(), neighbor[:k].cpu().numpy(), label[:k].cpu().numpy()))
    del kept, plan_d, plan_g, out_d, b, center, neighbor, label
    yield dict(hg=hg, deg=deg, top=top, roots=roots, dg=dg, trees=trees, emb=emb, bias=bias, emb_h=emb_h, bias_h=bias_h,
               res=res, info=info)
    del dg, trees, emb, bias
    torch.cuda.empty_cache()


def test_thresholds_crossed(c3):
    info, roots, n = c3["info"], c3["roots"], c3["hg"].n_node
    cnt, order = info["cnt"], info["s1_order"]
    chunked = int((cnt[order[S1_SINGLES:]] > 0).sum())
    records, owners, work = info["hub_d"]
    hub = info["gcnt"] > 0
    sizes = info["gcnt"][hub]
    print("\nR %d  nq %d  D walks %d  G walks %d  chunk-region pairs built %d  level 2 (D): hub records %d, owners %d, "
          "work items %d, largest group %d, groups > %d: %d  level 2 (G): %s"
          % (len(roots), info["nq"], info["n_walks_d"], info["n_walks_g"], chunked, records, owners, work, sizes.max(),
             HUB_GROUP_MAX, int((sizes > HUB_GROUP_MAX).sum()), info["hub_g"]))
    assert info["nq"] > 2 * S1_SINGLES                         # the depth-1 queue reaches its chunks
    assert chunked > 0                                         # ... and pairs there were built
    assert info["n_walks_d"] > 100_000
    assert work > owners, (records, owners, work)              # a hub group was split
    # the table read back through _flat_table agrees with the counters
    assert int(sizes.sum()) == records and int(hub.sum()) == owners
    assert int(((sizes + HUB_GROUP_MAX - 1) // HUB_GROUP_MAX).sum()) == work
    slot, node = info["keys"][hub] // n, info["keys"][hub] % n
    assert (slot < len(roots)).all() and (np.diff(c3["hg"].indptr)[node] >= HUB_THRESHOLD).all()
    assert c3["top"] in roots[slot[sizes > HUB_GROUP_MAX]]


def _oracle_sample(c3):
    """slots: the top-degree root, roots owning built chunk-region pairs, roots with a split hub group, a spread over
    the degree range and roots whose D walks voided"""
    info, roots, deg = c3["info"], c3["roots"], c3["deg"]
    rs = np.random.RandomState(5)
    R = len(roots)
    top = int(np.flatnonzero(roots == c3["top"])[0])
    pairs = info["s1_order"][S1_SINGLES:]
    owners = np.unique(info["s1_slot"][pairs[info["cnt"][pairs] > 0]])
    small = owners[deg[roots[owners]] <= CAP]
    chunk = rs.choice(small, min(12, len(small)), replace=False)
    big = np.setdiff1d(owners, small)
    chunk = np.concatenate([chunk, rs.choice(big, min(4, len(big)), replace=False)])
    hub = info["gcnt"] > HUB_GROUP_MAX
    split = np.unique(info["keys"][hub] // c3["hg"].n_node)
    by_deg = np.argsort(deg[roots], kind="stable")
    spread = by_deg[np.linspace(0, R - 1, 40).astype(np.int64)]
    void = np.flatnonzero(c3["res"][True]["root_ok"] == 0)
    void = rs.choice(void, min(8, len(void)), replace=False)
    return np.unique(np.concatenate([[top], chunk, split, spread, void]).astype(np.int64)), len(chunk), len(split), len(void)


def test_oracle_stratified_sample(c3):
    import torch
    from oracle import canonical as can
    hg, roots, deg, res, info = c3["hg"], c3["roots"], c3["deg"], c3["res"], c3["info"]
    E = can.pad_rows(c3["emb_h"], int(c3["emb"].shape[1]))
    wp = info["walk_ptr"]
    sample, n_chunk, n_split, n_void = _oracle_sample(c3)
    print("\noracle sample: %d roots (%d chunk-pair owners, %d with split groups, %d voided), %d of them capped at %d walks"
          % (len(sample), n_chunk, n_split, n_void, int((deg[roots[sample]] > CAP).sum()), CAP))
    assert n_chunk > 0 and n_split > 0
    gd, gg = res[True], res[False]
    bits_gpu = gd["bits"]
    center, neighbor, label = info["rows"]
    unpack = lambda b: np.unpackbits(b.view(np.uint8), bitorder="little")
    ub_gpu = unpack(bits_gpu)
    for lo in range(0, len(sample), 8):                        # bfs_parents: 4 MB per root
        sl = sample[lo:lo + 8]
        sroots = roots[sl]
        par = c3["trees"].parent_arrays(rows=torch.as_tensor(sl).to(c3["dg"].device)).cpu().numpy()
        assert np.array_equal(par, can.bfs_parents(hg.indptr, hg.adj, sroots)), "BFS trees differ from the oracle"
        full = deg[sroots] <= CAP
        num = np.minimum(deg[sroots], CAP).astype(np.int64)
        bits_ref = np.zeros_like(bits_gpu)
        ref = can.walk_pass(E, c3["bias_h"], hg.indptr, hg.adj, sroots, par, num, True, bits_ref, seed=SEED,
                            pass_tag=TAG_D)
        ub_ref = unpack(bits_ref)
        for j, (s, r) in enumerate(zip(sl, sroots)):
            g = slice(wp[s], wp[s] + num[j])
            o = slice(ref.walk_ptr[j], ref.walk_ptr[j + 1])
            for k in ("samples", "status", "wsteps", "wsuml"):
                assert np.array_equal(gd[k][g], ref[k][o]), ("D", k, int(r))
            e = slice(hg.indptr[r], hg.indptr[r + 1])
            if full[j]:
                assert gd["root_ok"][s] == ref.root_ok[j], ("D root_ok", int(r))
                assert np.array_equal(ub_gpu[e], ub_ref[e]), ("D bits", int(r))
            else:                                              # the oracle ran a prefix of the walks
                assert gd["root_ok"][s] <= ref.root_ok[j], ("D root_ok", int(r))
                assert not (ub_ref[e] & ~ub_gpu[e]).any(), ("D bits", int(r))
            if full[j]:                                        # the root's D rows (none unless ok)
                one = can.WalkResult(root_ok=ref.root_ok[j:j + 1], samples=ref.samples[o],
                                     walk_ptr=np.array([0, num[j]], np.int64))
                want = can.d_rows(one, [r], hg.raw_indptr, hg.raw_adj)
                a, m = info["row_ptr"][s], len(want[0])
                assert m == (2 * deg[r] if ref.root_ok[j] else 0)
                for got, w in zip((center, neighbor, label), want):
                    assert np.array_equal(got[a:a + m], w), ("D rows", int(r))
        # G: every walk (N_GEN <= CAP), under the GPU's D-pass bits
        ref = can.walk_pass(E, c3["bias_h"], hg.indptr, hg.adj, sroots, par, np.full(len(sl), N_GEN, np.int64), False,
                            bits_gpu.copy(), seed=SEED, pass_tag=TAG_G, max_path=MAX_PATH)
        keep = np.arange(MAX_PATH)[None, :] < np.minimum(ref.path_len, MAX_PATH)[:, None]
        rpaths = np.where(keep, ref.paths[:, :MAX_PATH], -1)
        for j, (s, r) in enumerate(zip(sl, sroots)):
            g = slice(s * N_GEN, (s + 1) * N_GEN)
            o = slice(j * N_GEN, (j + 1) * N_GEN)
            for k in ("samples", "status", "wsteps", "wsuml", "path_len"):
                assert np.array_equal(gg[k][g], ref[k][o]), ("G", k, int(r))
            assert np.array_equal(gg["paths"][g], rpaths[o]), ("G paths", int(r))
            assert gg["root_ok"][s] == ref.root_ok[j], ("G root_ok", int(r))


def test_d_rows_every_root(c3):
    """gg_emit_d_rows at scale: prepare_data_for_d's rows (graph_gan.py:192-201) from the sampled nodes, for every root"""
    hg, roots, res, info = c3["hg"], c3["roots"], c3["res"][True], c3["info"]
    wp = info["walk_ptr"]
    ok = np.flatnonzero(res["root_ok"])
    want_c, want_n, want_l = [], [], []
    for s in ok:
        r = roots[s]
        pos = hg.raw_adj[hg.raw_indptr[r]:hg.raw_indptr[r + 1]]
        neg = res["samples"][wp[s]:wp[s + 1]]
        want_c.append(np.full(len(pos) + len(neg), r, np.int32))
        want_n += [pos, neg]
        want_l += [np.ones(len(pos), np.int32), np.zeros(len(neg), np.int32)]
    got_c, got_n, got_l = info["rows"]
    assert np.array_equal(got_c, np.concatenate(want_c))
    assert np.array_equal(got_n, np.concatenate(want_n))
    assert np.array_equal(got_l, np.concatenate(want_l))


CONFIGS = {
    "slices": {},
    "flat_steps0": dict(flat_steps=0),
    "flat_steps14": dict(flat_steps=14),
    "hub_first_off": dict(hub_first=False),
    "depth1_off": dict(depth1=False),
    "tma_off": dict(tma=False),
    "hub_threshold300": dict(hub_threshold=300),
}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_batch_independence(c3, name):
    """A root's outputs depend on the root alone: the full batch, slices of at most 64 roots (each below the chunk
    queue: nq <= S1_SINGLES) and every sampler option give the same bits, root by root, in both passes"""
    dg, trees, deg = c3["dg"], c3["trees"], c3["deg"]
    smp = _sampler(dg, **CONFIGS[name])
    if name == "slices":
        ranges, lo = [], 0
        nq = np.diff(c3["hg"].indptr)[c3["roots"]]
        while lo < len(nq):
            hi = lo + 1
            while hi < len(nq) and hi - lo < SLICE_ROOTS and nq[lo:hi + 1].sum() <= S1_SINGLES:
                hi += 1
            ranges.append((lo, hi))
            lo = hi
        assert len(ranges) > 1
    else:
        ranges = [(0, len(c3["roots"]))]
    got = _passes(smp, dg, trees, ranges, deg, c3["emb"], c3["bias"])
    for for_d in (True, False):
        want, have = c3["res"][for_d], got[for_d]
        assert set(want) == set(have)
        for k in want:
            if k == "counters":
                for c in ("steps", "sum_l", "accepted", "ok_roots", "path_overflow"):
                    assert have[k][c] == want[k][c], (name, for_d, c)
            elif not np.array_equal(have[k], want[k]):
                bad = np.flatnonzero((have[k] != want[k]).reshape(len(want[k]), -1).any(1))
                raise AssertionError("%s, %s pass: %s differs at %d entries, first %d" % (name, "D" if for_d else "G", k,
                                                                                         len(bad), bad[0]))
