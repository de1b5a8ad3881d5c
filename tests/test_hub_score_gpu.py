"""GPU tests of the target-major hub scores (csrc/hub.cu: hub_score_tm_kernel): every listed hub entry e = (u -> v)
must hold dot(E[u], E[v]) + b[v] bit for bit as the canonical dot computes it (tests/test_hub_score_host.py restates
it in numpy and checks that restatement against the C oracle), at every row width, on the golden graphs (every hub
entry) and on the benchmarked power law (a sample of the entries plus every entry of the longest target runs)."""
import numpy as np
import pytest

from tests.golden import loader
from tests.test_hub_score_host import GOLDEN, canonical_dot, check_hub_list

pytestmark = pytest.mark.gpu
N_EMB = [20, 50, 128, 200, 512]          # -> ld 32, 64, 128, 256, 512 (zero padded columns included)


def _scores(dg, smp_threshold, emb, bias):
    from graphgan_b200 import _cabi
    import torch
    items, pairs, n_items, n_entries = dg.hub_tiles(smp_threshold)
    dg.edge_score.fill_(float("nan"))
    st = torch.cuda.current_stream(dg.device).cuda_stream
    _cabi.check(_cabi.lib().gg_hub_scores(n_items, items.data_ptr(), pairs.data_ptr(), emb.data_ptr(), bias.data_ptr(),
                                          int(emb.shape[1]), dg.edge_score.data_ptr(), st), "gg_hub_scores")
    torch.cuda.synchronize()
    return items.cpu().numpy(), pairs.cpu().numpy(), n_items, n_entries


def _expect(E, b, u, v):
    return (canonical_dot(E[u], E[v]) + b[v]).astype(np.float32)


def _device_emb(n, n_emb, seed, dev):
    import torch
    from graphgan_b200 import sampler as S
    g = torch.Generator(device=dev).manual_seed(seed)
    return S.pad_embedding(torch.randn(n, n_emb, generator=g, device=dev).mul_(0.4), dev)


@pytest.mark.parametrize("n_emb", N_EMB)
@pytest.mark.parametrize("name", GOLDEN)
def test_golden_hub_scores(name, n_emb, cuda_device):
    import torch
    from graphgan_b200 import graph as G
    case = loader.load(name)
    hg = G.HostGraph(case["train_edges"], case["test_edges"], n_node=case.n)
    dg = G.DeviceGraph(hg, cuda_device)
    emb = _device_emb(hg.n_node, n_emb, n_emb, cuda_device)
    E = emb.cpu().numpy()
    b = np.random.RandomState(n_emb).normal(0, 0.3, hg.n_node).astype(np.float32)
    bias = torch.as_tensor(b).to(cuda_device)
    for threshold in (1, 64, 128, 300):
        items, pairs, n_items, n_entries = _scores(dg, threshold, emb, bias)
        check_hub_list(hg, items, pairs, n_items, n_entries, threshold, G.HUB_ITEM_CAP)
        if n_entries == 0:
            continue
        u, e = pairs[:, 0].astype(np.int64), pairs[:, 1].astype(np.int64)
        got = dg.edge_score.cpu().numpy()[e]
        assert np.array_equal(got.view(np.int32), _expect(E, b, u, hg.adj[e]).view(np.int32)), (name, n_emb, threshold)


@pytest.fixture(scope="module")
def c3_graph():
    from graphgan_b200 import graph as G, synth
    return G.HostGraph(synth.power_law(1_000_000, 20, seed=0), None, n_node=1_000_000)


@pytest.mark.parametrize("n_emb", N_EMB)
def test_c3_hub_scores(c3_graph, n_emb, cuda_device):
    import torch
    from graphgan_b200 import graph as G
    hg = c3_graph
    dg = G.DeviceGraph(hg, cuda_device)
    emb = _device_emb(hg.n_node, n_emb, 7 + n_emb, cuda_device)
    bias = torch.randn(hg.n_node, generator=torch.Generator(device="cpu").manual_seed(n_emb)).mul_(0.3).to(cuda_device)
    b = bias.cpu().numpy()
    rs = np.random.RandomState(n_emb)
    for threshold in (64, 128, 300):
        items, pairs, n_items, n_entries = _scores(dg, threshold, emb, bias)
        check_hub_list(hg, items, pairs, n_items, n_entries, threshold, G.HUB_ITEM_CAP)
        score = dg.edge_score.cpu().numpy()
        long_runs = np.argsort(-items[:, 2].astype(np.int64), kind="stable")[:64]            # the cut runs, whole
        sel = np.concatenate([rs.choice(n_entries, 20000, replace=False)] +
                             [np.arange(items[t, 1], items[t, 1] + items[t, 2]) for t in long_runs])
        u, e = pairs[sel, 0].astype(np.int64), pairs[sel, 1].astype(np.int64)
        v = hg.adj[e].astype(np.int64)
        Eu, Ev = (emb[torch.as_tensor(x).to(cuda_device)].cpu().numpy() for x in (u, v))
        want = (canonical_dot(Eu, Ev) + b[v]).astype(np.float32)
        assert np.array_equal(score[e].view(np.int32), want.view(np.int32)), (n_emb, threshold)
        assert not np.isnan(score[pairs[:, 1]]).any()                                         # every hub entry written
