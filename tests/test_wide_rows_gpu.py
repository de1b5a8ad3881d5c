"""GPU tests of embeddings wider than 256 columns (ld = 512, n_emb 257 .. 512).

The walk kernels keep the current row in shared memory at ld = 512 and stream one candidate row per 8-lane group
(csrc/walk_common.cuh: score_list_wide); the Adam sweep and the two-barrier step loop give a warp a whole row; the
multi-CTA gradient sums the bias of its long slots in a kernel of its own.  Bars: bit-exact walks against the canonical
oracle (T1), bit-identical kernels where two paths compute the same thing, the oracle tolerance of
tests/test_updates_gpu.py for the optimizer steps."""
import numpy as np
import pytest

from tests.golden import loader
from tests.test_large_batch_gpu import Grad, _batch, _long_batch, _setup as grad_setup, close

pytestmark = pytest.mark.gpu
MULTI_CTA = 1   # GG_GRAD_MULTI_CTA


def _bits(t):
    return t.view(__import__("torch").int32)


# ---------------------------------------------------------------- walks
def _walk_compare(hg, emb_h, bias_h, roots, dev, *, hub, flat_steps=0, tma=True, rng="philox", n_sample_gen=8, max_path=48,
                  seed=77, cap=1 << 30):
    """D pass then G pass (with paths) on the mutated trees, against oracle/canonical.walk_pass; returns the counters."""
    import torch
    from graphgan_b200 import graph as G, sampler as S
    from oracle import canonical as can
    roots = np.asarray(roots, np.int32)
    dg = G.DeviceGraph(hg, dev)
    smp = S.WalkSampler(dg, hub_threshold=hub, tma=tma)
    smp.flat_steps = flat_steps
    trees = smp.build_trees(roots)
    par = trees.parent_arrays().cpu().numpy()
    assert np.array_equal(par, can.bfs_parents(hg.indptr, hg.adj, roots))
    emb = S.pad_embedding(emb_h, dev)
    assert emb.shape[1] == 512
    bias = torch.as_tensor(bias_h).to(dev)
    E = can.pad_rows(emb_h, 512)
    bits = np.zeros(dg.n_bit_words, np.uint32)
    sn = np.minimum(hg.degrees()[roots], cap).astype(np.int64)
    out_cnt = {}
    for for_d, tag, num in ((True, 5, sn), (False, 6, np.full(len(roots), n_sample_gen, np.int64))):
        mp = 0 if for_d else max_path
        if rng == "stream":
            u = np.random.RandomState(tag).random_sample(400000)
            ref = can.walk_pass(E, bias_h, hg.indptr, hg.adj, roots, par, num, for_d, bits, rng_mode=can.RNG_STREAM, stream=u,
                                max_path=mp)
            out = smp.run(emb, bias, trees, torch.as_tensor(num).to(dev) if for_d else int(n_sample_gen), for_d,
                          rng_mode=S.RNG_STREAM, stream=torch.as_tensor(u).to(dev), max_path=mp)
        else:
            ref = can.walk_pass(E, bias_h, hg.indptr, hg.adj, roots, par, num, for_d, bits, seed=seed, pass_tag=tag,
                                max_path=mp)
            out = smp.run(emb, bias, trees, torch.as_tensor(num).to(dev) if for_d else int(n_sample_gen), for_d,
                          seed=seed, pass_tag=tag, max_path=mp)
        W = ref.samples.shape[0]
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
            gp, rp = out.paths.cpu().numpy(), ref.paths
            for w in np.flatnonzero(ref.status == can.DONE):
                assert np.array_equal(gp[w, :ref.path_len[w]], rp[w, :ref.path_len[w]])
        cnt["max_l"], cnt["max_path"], cnt["walks"] = ref.max_l, int(ref.path_len.max()) if not for_d else 0, W
        out_cnt["d" if for_d else "g"] = cnt
    return out_cnt


def _golden(name, d):
    from graphgan_b200 import graph as G, synth
    case = loader.load(name)
    hg = G.HostGraph(case["train_edges"], case["test_edges"], n_node=case.n)
    emb = synth.embeddings(case.n, d, seed=d, sigma=0.3)
    bias = np.random.RandomState(d + 1).normal(0, 0.3, case.n).astype(np.float32)
    rs = np.random.RandomState(2)
    roots = np.arange(case.n) if case.n <= 1200 else np.sort(rs.choice(np.flatnonzero(hg.degrees() > 0), 300, replace=False))
    return hg, emb, bias, roots


@pytest.mark.parametrize("d", [300, 512])
@pytest.mark.parametrize("name", ["tiny", "rand300", "rand1200", "cagrqc"])
def test_golden_walks_match_oracle(name, d, cuda_device):
    """Every walk path at ld = 512: scores on demand (hub 0) and from the per-pass hub scores / root CDFs (8, 128), the
    persistent kernel alone and behind four level-synchronous steps, hub lists TMA-staged or not, both RNG modes."""
    hg, emb, bias, roots = _golden(name, d)
    for hub, flat, tma in ((0, 0, True), (8, 0, True), (8, 4, True), (8, 4, False), (128, 0, False), (128, 4, True)):
        _walk_compare(hg, emb, bias, roots, cuda_device, hub=hub, flat_steps=flat, tma=tma)
    for hub in (0, 8):
        _walk_compare(hg, emb, bias, roots, cuda_device, hub=hub, rng="stream")


@pytest.mark.parametrize("flat_steps", [0, 4])
def test_c3_powerlaw_1m_at_n_emb_512(flat_steps, cuda_device):
    """The bench graph (power-law 1M, avg-deg 20) with the hub roots of tests/test_config_parity_gpu.py at n_emb = 512:
    lists beyond the shared score buffer, TMA-staged hub lists, the depth-1 CDF sharing."""
    from graphgan_b200 import graph as G, synth
    n = 1_000_000
    hg = G.HostGraph(synth.power_law(n, 20, seed=0), None, n_node=n)
    deg = np.diff(hg.indptr)
    top = int(np.argmax(deg))
    nb = hg.adj[hg.indptr[top]:hg.indptr[top + 1]]
    rs = np.random.RandomState(3)
    ordinary = rs.choice(np.flatnonzero(hg.degrees() > 0), 56, replace=False)
    roots = np.unique(np.concatenate([[top, 1, 7, 300], nb[[0, len(nb) // 2, len(nb) - 1]], ordinary]))
    emb = synth.embeddings(n, 512, seed=1)
    bias = np.random.RandomState(5).normal(0, 0.1, n).astype(np.float32)
    st = _walk_compare(hg, emb, bias, roots, cuda_device, hub=128, flat_steps=flat_steps, cap=40, n_sample_gen=20, max_path=64,
                       seed=11)
    assert st["d"]["max_l"] > 2048
    assert st["g"]["path_overflow"] == 0
    assert st["d"]["rows_gathered"] > 0


def test_deep_trees_at_n_emb_300(cuda_device):
    """A path tail of 44 nodes behind a power-law graph, biases that pull the generator down the path: long walks."""
    from graphgan_b200 import graph as G, synth
    n0, tail = 100_000, 44
    base = synth.power_law(n0, 8, seed=2)
    n = n0 + tail
    anchor = n0 - 5
    chain = np.stack([np.concatenate([[anchor], np.arange(n0, n - 1)]), np.arange(n0, n)], 1)
    hg = G.HostGraph(np.concatenate([base, chain]), None, n_node=n)
    ordinary = np.random.RandomState(4).choice(np.flatnonzero(hg.degrees()[:n0] > 0), 20, replace=False)
    roots = np.unique(np.concatenate([[0, anchor, n - 1, n - 2, n0 + 3], ordinary]))
    bias = np.random.RandomState(5).normal(0, 0.1, n).astype(np.float32)
    bias[n0:] = 8.0 * (tail - 1 - np.arange(tail))
    for flat in (0, 14):
        st = _walk_compare(hg, synth.embeddings(n, 300, seed=6, sigma=0.35), bias, roots, cuda_device, hub=128, flat_steps=flat,
                           cap=48, n_sample_gen=20, max_path=64)
        assert 40 < st["g"]["max_path"] <= 64


# ---------------------------------------------------------------- updates
@pytest.mark.parametrize("d", [300, 512])
def test_steps_match_oracle(d, cuda_device):
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.generator import Generator
    from oracle import updates
    rs = np.random.RandomState(d)
    n, B, steps = 2000, 256, 4
    emb = rs.normal(0, 0.5, size=(n, d))
    dis, gen = Discriminator(n, emb, device=cuda_device), Generator(n, emb, device=cuda_device)
    assert dis.ld == 512
    od, og = updates.Discriminator(n, emb, 1e-3, 1e-5), updates.Generator(n, emb, 1e-3, 1e-5)
    for _ in range(steps):
        i, j = _batch(rs, n, B)
        lab = (rs.random_sample(B) < 0.5).astype(np.float32)
        rew = (rs.random_sample(B) * 3).astype(np.float32)
        dis.d_step(i, j, lab); od.d_updates(i, j, lab)
        gen.g_step(i, j, rew); og.g_updates(i, j, rew)
        assert int((dis.row_slot != -1).sum()) == 0 and int((gen.row_slot != -1).sum()) == 0
    for m, o in ((dis, od), (gen, og)):
        assert close(m.embedding_numpy(), o.E, steps=steps) and close(m.bias_t.cpu().numpy(), o.b, steps=steps)
        assert close(m.m_emb[:, :d].cpu().numpy(), o.adam.m_e, steps=steps)
        assert close(m.v_emb[:, :d].cpu().numpy(), o.adam.v_e, steps=steps)
        if d < m.ld:
            assert float(m.emb[:, d:].abs().max()) == 0.0      # the padding columns stay zero


@pytest.mark.parametrize("B", [7, 333, 1024])
@pytest.mark.parametrize("mode", [0, 1])
def test_multi_cta_gradient_equals_one_cta(B, mode, cuda_device):
    import torch
    from graphgan_b200 import _cabi
    lib, ld = _cabi.lib(), 512
    rs = np.random.RandomState(B + mode)
    n = max(40, B // 3)
    emb, bias, i, j, a = grad_setup(cuda_device, rs, n, 300, B, mode)
    bt = 0 if mode == 0 else 3 * B + 1
    ref = Grad(cuda_device, n, ld, B).run(lib, mode, i, j, a, emb, bias, ld, 1e-5, bt)
    got = Grad(cuda_device, n, ld, B).run(lib, mode, i, j, a, emb, bias, ld, 1e-5, bt, ex_flags=MULTI_CTA)
    U = ref.U
    assert got.U == U
    assert torch.equal(got.uniq[:U], ref.uniq[:U])
    assert torch.equal(_bits(got.rows[:U]), _bits(ref.rows[:U]))
    assert torch.equal(_bits(got.bias[:U]), _bits(ref.bias[:U]))
    assert torch.equal(got.row_slot, ref.row_slot)


@pytest.mark.parametrize("mode", [0, 1])
def test_long_slot_bias_above_1024_pairs(mode, cuda_device):
    """B = 4096 with one centre row in > 16 entries: its slot goes to the one-CTA-per-slot sums, whose 512 threads are all
    columns at ld = 512.  The bias of that slot must be the entry-order sum of its terms (numpy float32, from +0)."""
    import torch
    from graphgan_b200 import _cabi
    lib, ld, B, n = _cabi.lib(), 512, 4096, 3000
    rs = np.random.RandomState(40 + mode)
    emb, bias, _, _, _ = grad_setup(cuda_device, rs, n, 512, 8, mode)
    i, j = _long_batch(rs, n, B, 600)                     # row 3 is the centre of 600 pairs
    aux = (rs.random_sample(B) < 0.5).astype(np.float32) if mode == 0 else (rs.random_sample(B) * 3).astype(np.float32)
    to = lambda x: torch.as_tensor(np.ascontiguousarray(x)).to(cuda_device)
    g = Grad(cuda_device, n, ld, B).run(lib, mode, to(i), to(j), to(aux), emb, bias, ld, 1e-5, ex_flags=0)
    # numpy float64: per row, the sum over its j-side entries of delta (+ lambda * b in D mode); the float32 entry-order
    # chain may differ from it by rounding only (bounded by the sum of magnitudes)
    E = emb.cpu().numpy().astype(np.float64)
    b = bias.cpu().numpy().astype(np.float64)
    s = np.einsum("kd,kd->k", E[i], E[j]) + b[j]
    p = 1.0 / (1.0 + np.exp(-s))
    delta = (p - aux) if mode == 0 else np.where(p >= 1e-5, -(aux / B) * (1.0 - p), 0.0)
    term = delta + (1e-5 * b[j] if mode == 0 else 0.0)
    want, mag = np.zeros(n), np.zeros(n)
    np.add.at(want, j, term)
    np.add.at(mag, j, np.abs(term))
    uniq = g.uniq[:g.U].cpu().numpy()
    got = g.bias[:g.U].cpu().numpy().astype(np.float64)
    assert np.bincount(np.concatenate([i, j]), minlength=n)[3] > 16 and 3 in set(uniq.tolist())
    err = np.abs(got - want[uniq])
    assert bool((err <= 1e-4 * mag[uniq] + 1e-6).all()), float(err.max())


def test_merge_ex_equals_one_cta_merge(cuda_device):
    import torch
    from graphgan_b200 import _cabi
    from tests.dist_large_batch_worker import gathered_blocks, merge_ex
    from tests.test_dp_large_batch_gpu import Out, _setup as dp_setup
    lib, ld = _cabi.lib(), 512
    for world, mode in ((1, 0), (3, 1), (8, 0)):
        rs = np.random.RandomState(world + 10 * mode)
        n, B = 500, 1000
        emb, bias, i, j, a = dp_setup(cuda_device, rs, n, 400, B, mode)
        scratch_slot = torch.full((n,), -1, dtype=torch.int32, device=cuda_device)
        gathered, cap = gathered_blocks(lib, mode, i, j, a, emb, bias, ld, 1e-5, world, scratch_slot)
        E = world * cap
        ref, got = Out(cuda_device, n, ld, E, gathered, cap), Out(cuda_device, n, ld, E, gathered, cap)
        _cabi.check(lib.gg_grad_merge(world, cap, ld, gathered.data_ptr(), *(t.data_ptr() for t in ref.args()), None),
                    "gg_grad_merge")
        merge_ex(lib, world, cap, ld, gathered, *got.args(), flags=MULTI_CTA)
        torch.cuda.synchronize()
        U = int(ref.n_unique.item())
        assert int(got.n_unique.item()) == U >= 1
        assert torch.equal(got.uniq[:U], ref.uniq[:U])
        assert torch.equal(_bits(got.rows[:U]), _bits(ref.rows[:U]))
        assert torch.equal(_bits(got.bias[:U]), _bits(ref.bias[:U]))
        assert torch.equal(got.row_slot, ref.row_slot)


def test_adam_sweeps_bit_identical(cuda_device):
    """gg_adam_apply's sweeps (per-thread loads, the CTA-barrier and warp-specialised TMA pipelines) on a gradient whose
    rows touch all four 128-column quarters of a row; row_slot is cleared by each."""
    import ctypes as C
    import torch
    from graphgan_b200 import _cabi
    lib, ld, n = _cabi.lib(), 512, 5003
    rs = np.random.RandomState(9)
    base = {k: torch.as_tensor(rs.normal(0, s, size=shape).astype(np.float32)).to(cuda_device)
            for k, s, shape in (("emb", 0.5, (n, ld)), ("m", 0.01, (n, ld)), ("v", 1e-4, (n, ld)), ("bias", 0.1, (n,)),
                                ("mb", 0.01, (n,)), ("vb", 1e-4, (n,)))}
    base["v"] = base["v"].abs(); base["vb"] = base["vb"].abs()
    U = 700
    rows = torch.as_tensor(rs.choice(n, U, replace=False).astype(np.int32)).to(cuda_device)
    grad = torch.as_tensor(rs.normal(0, 1, size=(U, ld)).astype(np.float32)).to(cuda_device)
    gb = torch.as_tensor(rs.normal(0, 1, size=U).astype(np.float32)).to(cuda_device)
    results = []
    for path in ("ldg", "tma", "tma256x2", "tma512x3", "ws16", "ws8"):
        _cabi.check(lib.gg_set_adam_path(path.encode()), "gg_set_adam_path")
        t = {k: v.clone() for k, v in base.items()}
        slot = torch.full((n,), -1, dtype=torch.int32, device=cuda_device)
        slot[rows.long()] = torch.arange(U, dtype=torch.int32, device=cuda_device)
        _cabi.check(lib.gg_adam_apply(n, ld, t["emb"].data_ptr(), t["m"].data_ptr(), t["v"].data_ptr(), t["bias"].data_ptr(),
                                      t["mb"].data_ptr(), t["vb"].data_ptr(), None, rows.data_ptr(), grad.data_ptr(), gb.data_ptr(),
                                      slot.data_ptr(), C.c_float(1e-3), C.c_float(0.9), C.c_float(0.999), C.c_float(1e-8), None),
                    "gg_adam_apply")
        torch.cuda.synchronize()
        assert int((slot != -1).sum()) == 0, path
        results.append((path, t))
    _cabi.check(lib.gg_set_adam_path(b"ldg"), "gg_set_adam_path")
    ref = results[0][1]
    for q in range(4):      # the gradient really moved every quarter of the rows that have one
        cols = slice(128 * q, 128 * (q + 1))
        moved = (ref["m"][rows.long(), cols] - base["m"][rows.long(), cols] * 0.9).abs().max()
        assert float(moved) > 0.0
    for path, t in results[1:]:
        for k in base:
            assert torch.equal(_bits(t[k]), _bits(ref[k])), (path, k)


@pytest.mark.parametrize("cls_name", ["Discriminator", "Generator"])
def test_persistent_loops_equal_step_loop(cls_name, cuda_device):
    """gg_train_loop (two-barrier: CTA 0 publishes the gradient, every CTA sweeps and clears row_slot) and gg_train_fused
    against gg_train_steps, bit for bit, on a graph small enough for both.  A row is four sweep segments at ld = 512: a
    slot cleared before every segment has read it would drop part of the gradient."""
    import torch
    from graphgan_b200 import discriminator, generator
    cls = getattr(discriminator if cls_name == "Discriminator" else generator, cls_name)
    rs = np.random.RandomState(21)
    n, d, M, B = 1500, 480, 6000, 200
    emb = rs.normal(0, 0.5, size=(n, d))
    i = np.repeat(rs.randint(0, n, M // 10 + 1), 10)[:M].astype(np.int32)
    j = rs.randint(0, n, M).astype(np.int32)
    aux = (rs.random_sample(M) < 0.5).astype(np.float32) if cls_name == "Discriminator" else (rs.random_sample(M) * 3).astype(np.float32)
    starts = list(range(0, M, B))
    rs.shuffle(starts)
    ref = cls(n, emb, device=cuda_device)
    ref.train_steps(i, j, aux, starts, B, persistent=False)
    for how in ("two-barrier", True):
        m = cls(n, emb, device=cuda_device)
        m.train_steps(i, j, aux, starts, B, persistent=how)
        torch.cuda.synchronize()
        for name in ("emb", "bias_t", "m_emb", "v_emb", "m_bias", "v_bias"):
            assert torch.equal(_bits(getattr(m, name)), _bits(getattr(ref, name))), (how, name)
        assert int((m.row_slot != -1).sum()) == 0


# ---------------------------------------------------------------- evaluation and I/O
def test_reward_and_pair_dot_against_float64(cuda_device):
    import ctypes as C
    import torch
    from graphgan_b200 import _cabi
    from graphgan_b200.discriminator import Discriminator
    rs = np.random.RandomState(31)
    n, d, B = 900, 300, 4000
    emb = rs.normal(0, 0.3, size=(n, d))
    dis = Discriminator(n, emb, device=cuda_device)
    i, j = rs.randint(0, n, B).astype(np.int32), rs.randint(0, n, B).astype(np.int32)
    E = dis.emb.cpu().numpy().astype(np.float64)
    b = dis.bias_t.cpu().numpy().astype(np.float64)
    s = np.einsum("kd,kd->k", E[i], E[j]) + b[j]
    want = np.log1p(np.exp(np.clip(s, -10.0, 10.0)))       # discriminator.py:33-34
    got = dis.reward_pairs(torch.as_tensor(i).to(cuda_device), torch.as_tensor(j).to(cuda_device)).cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5)
    lib = _cabi.lib()
    out = torch.empty(B, dtype=torch.float64, device=cuda_device)
    ti, tj = torch.as_tensor(i).to(cuda_device), torch.as_tensor(j).to(cuda_device)
    _cabi.check(lib.gg_pair_dot_f64(B, ti.data_ptr(), tj.data_ptr(), dis.emb.data_ptr(), 512, out.data_ptr(), None),
                "gg_pair_dot_f64")
    np.testing.assert_allclose(out.cpu().numpy(), np.einsum("kd,kd->k", E[i], E[j]), rtol=1e-12, atol=1e-12)


def test_binary_dump_round_trip_at_n_emb_300(cuda_device, tmp_path):
    """write_embeddings_binary unpads the 512-float rows to the 300 columns (gg_unpad_rows); reading it back gives the
    model's embedding and the fp32 input, exactly."""
    from graphgan_b200 import io
    from graphgan_b200.generator import Generator
    n, d = 2000, 300
    e = np.random.RandomState(3).normal(0, 0.5, size=(n, d)).astype(np.float32)
    gen = Generator(n, e, device=cuda_device)
    assert gen.ld == 512
    io.write_embeddings_binary(str(tmp_path / "g.f32"), gen)
    back = io.read_embeddings_binary(str(tmp_path / "g.f32"))
    assert back.shape == (n, d) and back.dtype == np.float32
    assert np.array_equal(back, gen.embedding_numpy()) and np.array_equal(back, e)


def test_graphgan_checkpoint_resume_at_n_emb_300(cuda_device, tmp_path, monkeypatch):
    """GraphGAN on CA-GrQc with 300-wide initial embeddings (ld 512): save -> load -> one more epoch equals two
    uninterrupted epochs, bit for bit (parameters, Adam slots and powers, father-removal bits, pass counter)."""
    import torch
    from graphgan_b200 import graph as G, synth
    from graphgan_b200.graph_gan import GraphGAN
    from tests.test_updates_gpu import _small_gan_config
    c = loader.load("cagrqc")
    hg = G.HostGraph(c.train_edges, c.test_edges)
    n, d = hg.n_node, 300
    emb_d, emb_g = synth.embeddings(n, d, seed=41, sigma=0.3), synth.embeddings(n, d, seed=42, sigma=0.3)
    config = _small_gan_config(monkeypatch, tmp_path, cuda_device, c)
    monkeypatch.setattr(config, "n_emb", d)
    monkeypatch.setattr(config, "n_epochs", 2)
    a = GraphGAN(host_graph=hg, node_embed_init_d=emb_d, node_embed_init_g=emb_g)
    assert a.generator.ld == 512 and a.discriminator.ld == 512
    a.train()                                           # saves at the start of epoch 1 (save_steps = 1)
    monkeypatch.setattr(config, "n_epochs", 1)
    monkeypatch.setattr(config, "load_model", True)
    b = GraphGAN(host_graph=hg, node_embed_init_d=emb_d, node_embed_init_g=emb_g)
    b.train()                                           # loads the epoch-0 state, runs one more epoch
    for ma, mb in ((a.generator, b.generator), (a.discriminator, b.discriminator)):
        assert ma.step_count > 0
        for name in ("emb", "bias_t", "m_emb", "v_emb", "m_bias", "v_bias"):
            assert torch.equal(getattr(ma, name), getattr(mb, name)), name
        assert ma.beta1_power == mb.beta1_power and ma.beta2_power == mb.beta2_power and ma.step_count == mb.step_count
        assert float(ma.emb[:, d:].abs().max()) == 0.0
    assert torch.equal(a.device_graph.d1_bits, b.device_graph.d1_bits)
    assert a.pass_counter == b.pass_counter


def test_world1_data_parallel_at_ld_512(cuda_device):
    """torch.distributed.run with one rank (tests/dist_wide_rows_worker.py): DataParallelStep equals PairModel at ld 512
    over NCCL (one-CTA and multi-CTA batches) and over the peer-memory transport."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1", "--master-addr", "127.0.0.1",
           "--master-port", "29657", os.path.join(root, "tests", "dist_wide_rows_worker.py")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=root)
    assert r.returncode == 0 and "DP_WIDE_WORLD1_OK" in r.stdout, r.stdout[-3000:]
