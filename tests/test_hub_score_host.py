"""Host tests of the target-major hub score work list (DeviceGraph.hub_tiles) and of the numpy statement of the
canonical dot that tests/test_hub_score_gpu.py checks the hub scores against.

The list is built with torch; on a machine without a GPU it is built on the CPU, the same code."""
import numpy as np
import pytest

from tests.golden import loader

GOLDEN = ["tiny", "rand300", "rand1200", "cagrqc"]


# ---------------------------------------------------------------- the canonical dot in numpy
def fma32(a, b, s):
    """float32 fmaf(a, b, s) elementwise, rounded once: a * b is exact in float64, the float64 sum is turned into its
    round-to-odd value (53 >= 24 + 2 bits, so the final rounding to float32 is the single rounding of the fma)."""
    p = a.astype(np.float64) * b.astype(np.float64)
    s64 = s.astype(np.float64)
    t = p + s64
    bp = t - p
    err = (p - (t - bp)) + (s64 - bp)                  # exact: p + s64 == t + err
    fix = (err != 0) & ((t.view(np.int64) & 1) == 0)
    t = np.where(fix, np.nextafter(t, np.where(err > 0, np.inf, -np.inf)), t)
    return t.astype(np.float32)


def canonical_dot(A, B):
    """dot(A[k], B[k]) for every k as the kernels compute it (oracle/gg_oracle.c: ggo_dot): lane g = 0..7 runs one fma
    chain over the float4 chunks g, g + 8, ... of the row, then the butterfly over the eight lanes."""
    A, B = np.asarray(A, np.float32), np.asarray(B, np.float32)
    ld = A.shape[1]
    s = np.zeros((8, A.shape[0]), np.float32)
    for g in range(8):
        for c in range(g, ld // 4, 8):
            for k in range(4):
                s[g] = fma32(A[:, 4 * c + k], B[:, 4 * c + k], s[g])
    t = [s[g] + s[g ^ 4] for g in range(8)]
    a = [t[g] + t[g ^ 2] for g in range(8)]
    return a[0] + a[1]


@pytest.mark.parametrize("ld", [32, 64, 128, 256, 512])
def test_canonical_dot_matches_oracle(ld):
    from oracle import canonical as can
    rs = np.random.RandomState(ld)
    A = (rs.normal(0, 0.5, (300, ld)) * rs.choice([1e-3, 1, 1e3], (300, 1))).astype(np.float32)
    B = rs.normal(0, 0.5, (300, ld)).astype(np.float32)
    got = canonical_dot(A, B)
    want = np.array([can.dot_c(A[k], B[k]) for k in range(A.shape[0])], np.float32)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


# ---------------------------------------------------------------- the work list
def _graphs():
    from graphgan_b200 import graph as G, synth
    out = {}
    for name in GOLDEN:
        case = loader.load(name)
        out[name] = G.HostGraph(case["train_edges"], case["test_edges"], n_node=case.n)
    out["powerlaw_20k"] = G.HostGraph(synth.power_law(20000, 20, seed=0), None, n_node=20000)
    return out


@pytest.fixture(scope="module")
def graphs():
    return _graphs()


def check_hub_list(hg, items, pairs, n_items, n_entries, threshold, cap):
    """items / pairs (numpy) hold exactly the hub entries, each once, grouped by target, items within the cap"""
    deg = np.diff(hg.indptr)
    src_of = np.repeat(np.arange(hg.n_node), deg)
    want = np.flatnonzero(deg[src_of] >= threshold)             # hub entries, hub-major
    assert n_entries == want.shape[0] == pairs.shape[0]
    assert n_items == items.shape[0]
    if n_entries == 0:
        assert n_items == 0
        return
    u, e = pairs[:, 0].astype(np.int64), pairs[:, 1].astype(np.int64)
    assert np.array_equal(np.sort(e), want)                     # every hub entry, once
    assert np.array_equal(u, src_of[e])                         # (u, e): u is the source of e
    tgt = hg.adj[e]
    assert np.all(np.diff(tgt) >= 0)                             # grouped by target ...
    same = np.diff(tgt) == 0
    assert np.all(np.diff(e)[same] > 0)                          # ... hub-major within a target (stable)
    v, first, count = items[:, 0], items[:, 1].astype(np.int64), items[:, 2].astype(np.int64)
    assert np.all(items[:, 3] == 0)
    assert np.all((count >= 1) & (count <= cap))
    assert first[0] == 0 and np.array_equal(first[1:], (first + count)[:-1]) and first[-1] + count[-1] == n_entries
    assert np.array_equal(np.repeat(v, count), tgt)             # an item's pairs all point into its target
    cont = v[1:] == v[:-1]                                       # a target is cut only after a full item
    assert np.all(count[:-1][cont] == cap)


@pytest.mark.parametrize("threshold", [1, 64, 300, 10 ** 9])
@pytest.mark.parametrize("name", GOLDEN + ["powerlaw_20k"])
def test_hub_list(graphs, name, threshold):
    from graphgan_b200 import graph as G
    hg = graphs[name]
    dg = G.DeviceGraph(hg, "cpu")
    items, pairs, n_items, n_entries = dg.hub_tiles(threshold)
    check_hub_list(hg, items.numpy(), pairs.numpy(), n_items, n_entries, threshold, G.HUB_ITEM_CAP)
    assert dg.edge_score.shape[0] == max(hg.adj.shape[0], 1)
    assert dg.hub_tiles(threshold) is dg._hub                    # cached


def test_hub_list_cuts_long_runs(graphs):
    """a small cap cuts the runs of the high in-degree targets into several items"""
    from graphgan_b200 import graph as G
    hg = graphs["powerlaw_20k"]
    dg = G.DeviceGraph(hg, "cpu")
    items, pairs, n_items, n_entries = dg.hub_tiles(64, item_cap=3)
    check_hub_list(hg, items.numpy(), pairs.numpy(), n_items, n_entries, 64, 3)
    assert np.any(items.numpy()[1:, 0] == items.numpy()[:-1, 0])


def test_hub_list_asymmetric_csr():
    """the list needs no reverse entries: a directed walk CSR works as well"""
    from graphgan_b200 import graph as G
    hg = G.HostGraph.from_arrays(6, np.zeros(7, np.int64), np.zeros(0, np.int32),       # 0 -> 2, 3, 4, 5; 1 -> 2
                                 np.array([0, 4, 5, 5, 5, 5, 5], np.int64), np.array([2, 3, 4, 5, 2], np.int32))
    dg = G.DeviceGraph(hg, "cpu")
    items, pairs, n_items, n_entries = dg.hub_tiles(1)
    check_hub_list(hg, items.numpy(), pairs.numpy(), n_items, n_entries, 1, G.HUB_ITEM_CAP)
    assert items.numpy()[:, 0].tolist() == [2, 3, 4, 5] and items.numpy()[:, 2].tolist() == [2, 1, 1, 1]
