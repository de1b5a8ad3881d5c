"""GPU tests of mini-batches above GG_MAX_BATCH: the multi-CTA sparse gradient (gg_pair_grad_ex) against the one-CTA
kernel bit for bit, against the numpy oracle (oracle/updates.py) above 1024 pairs, and the layers above it (the C step
loop, Session.run feeds, GraphGAN.train)."""
import ctypes as C

import numpy as np
import pytest

from tests.golden import loader

pytestmark = pytest.mark.gpu
RTOL = 1e-5
MULTI_CTA = 1   # GG_GRAD_MULTI_CTA


def close(got, want, rtol=RTOL, lr=1e-3, steps=8):
    """The bar of tests/test_updates_gpu.py (see the reasoning there): relative Frobenius error <= 1e-5, >= 99.99 % of
    the coordinates within rtol 1e-5 (+ 1e-6 abs), no coordinate off by more than 2 * lr per step taken."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    diff = np.abs(got - want)
    fro = np.linalg.norm(diff) / max(np.linalg.norm(want), 1e-30)
    ok_frac = float(np.mean(diff <= rtol * np.abs(want) + 1e-6))
    return fro <= rtol and ok_frac >= 0.9999 and float(diff.max()) <= 2 * lr * steps


def _batch(rs, n, B, centre_every=3):
    """Random pairs with a duplicate pair, a self pair, a row on both sides and one centre repeated through the batch."""
    i, j = rs.randint(0, n, B), rs.randint(0, n, B)
    i[::centre_every] = n // 2
    if B >= 6:
        i[3], j[3] = i[0], j[0]
        j[5] = i[5]
        i[1] = j[2]
    else:
        j[0] = i[0]
    return i.astype(np.int32), j.astype(np.int32)


class Grad:
    """One raw call of gg_pair_grad or gg_pair_grad_ex on fresh output buffers."""

    def __init__(self, dev, n, ld, B):
        import torch
        self.torch = torch
        self.n_unique = torch.zeros(1, dtype=torch.int32, device=dev)
        self.uniq = torch.full((2 * B,), -7, dtype=torch.int32, device=dev)
        self.rows = torch.full((2 * B, ld), 7.0, dtype=torch.float32, device=dev)
        self.bias = torch.full((2 * B,), 7.0, dtype=torch.float32, device=dev)
        self.row_slot = torch.full((n,), -1, dtype=torch.int32, device=dev)

    def run(self, lib, mode, i, j, a, emb, bias, ld, lam, batch_total=0, ex_flags=None):
        from graphgan_b200 import _cabi
        B = int(i.shape[0])
        args = (mode, B, batch_total, i.data_ptr(), j.data_ptr(), a.data_ptr(), emb.data_ptr(), bias.data_ptr(), ld, C.c_float(lam),
                self.n_unique.data_ptr(), self.uniq.data_ptr(), self.rows.data_ptr(), self.bias.data_ptr(), self.row_slot.data_ptr())
        if ex_flags is None:
            _cabi.check(lib.gg_pair_grad(*args, None), "gg_pair_grad")
        else:
            n = C.c_int64(0)
            _cabi.check(lib.gg_pair_grad_scratch_bytes(B, ld, C.byref(n)), "gg_pair_grad_scratch_bytes")
            scratch = self.torch.empty(n.value, dtype=self.torch.uint8, device=emb.device)
            _cabi.check(lib.gg_pair_grad_ex(*args, scratch.data_ptr(), n.value, ex_flags, None), "gg_pair_grad_ex")
        self.torch.cuda.synchronize()
        self.U = int(self.n_unique.item())
        return self


def _bits(t):
    return t.view(__import__("torch").int32)


def _setup(dev, rs, n, d, B, mode):
    import torch
    from graphgan_b200.sampler import pad_embedding
    emb = pad_embedding(rs.normal(0, 0.5, size=(n, d)), dev)
    bias = torch.as_tensor(rs.normal(0, 0.1, size=n).astype(np.float32)).to(dev)
    i, j = _batch(rs, n, B)
    aux = (rs.random_sample(B) < 0.5).astype(np.float32) if mode == 0 else (rs.random_sample(B) * 3).astype(np.float32)
    to = lambda x: torch.as_tensor(x).to(dev)
    return emb, bias, to(i), to(j), to(aux)


@pytest.mark.parametrize("B", [1, 7, 64, 333, 1024])
@pytest.mark.parametrize("ld", [32, 64, 128, 256])
@pytest.mark.parametrize("mode", [0, 1])
def test_multi_cta_equals_one_cta_kernel(B, ld, mode, cuda_device):
    """The multi-CTA path (forced with GG_GRAD_MULTI_CTA) and pair_grad_kernel give the same bits: slot count and
    order, per-row sums, bias sums and the row -> slot map.  G mode with batch_total != n_pairs (a rank's slice)."""
    import torch
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rs = np.random.RandomState(B * 7 + ld + mode)
    n = max(40, B // 3)
    emb, bias, i, j, a = _setup(cuda_device, rs, n, ld - 5, B, mode)
    bt = 0 if mode == 0 else 3 * B + 1
    ref = Grad(cuda_device, n, ld, B).run(lib, mode, i, j, a, emb, bias, ld, 1e-5, bt)
    got = Grad(cuda_device, n, ld, B).run(lib, mode, i, j, a, emb, bias, ld, 1e-5, bt, ex_flags=MULTI_CTA)
    U = ref.U
    assert got.U == U and 1 <= U <= 2 * B
    assert torch.equal(got.uniq[:U], ref.uniq[:U])
    assert torch.equal(_bits(got.rows[:U]), _bits(ref.rows[:U]))
    assert torch.equal(_bits(got.bias[:U]), _bits(ref.bias[:U]))
    assert torch.equal(got.row_slot, ref.row_slot)
    # without the flag, gg_pair_grad_ex runs the one-CTA kernel itself
    same = Grad(cuda_device, n, ld, B).run(lib, mode, i, j, a, emb, bias, ld, 1e-5, bt, ex_flags=0)
    assert same.U == U and torch.equal(_bits(same.rows[:U]), _bits(ref.rows[:U])) and torch.equal(same.row_slot, ref.row_slot)


@pytest.mark.parametrize("mode", [0, 1])
def test_large_batch_equals_disjoint_slices(mode, cuda_device):
    """B = 8192 made of eight 1024-pair slices on disjoint row sets: a row confined to one slice keeps the relative
    order of its entries, so its gradient must equal gg_pair_grad on its slice (with batch_total = 8192) bit for bit."""
    import torch
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rs = np.random.RandomState(11 + mode)
    per, S, ld = 300, 1024, 128
    n = 8 * per
    emb, bias, _, _, _ = _setup(cuda_device, rs, n, 100, 8, mode)
    ii, jj = [], []
    for k in range(8):
        i, j = _batch(rs, per, S)
        ii.append(i + k * per); jj.append(j + k * per)
    i_all, j_all = np.concatenate(ii), np.concatenate(jj)
    aux = (rs.random_sample(8 * S) < 0.5).astype(np.float32) if mode == 0 else (rs.random_sample(8 * S) * 3).astype(np.float32)
    to = lambda x: torch.as_tensor(np.ascontiguousarray(x)).to(cuda_device)
    big = Grad(cuda_device, n, ld, 8 * S).run(lib, mode, to(i_all), to(j_all), to(aux), emb, bias, ld, 1e-5, ex_flags=0)
    slot_big = big.row_slot.cpu().numpy()
    for k in range(8):
        sl = slice(k * S, (k + 1) * S)
        one = Grad(cuda_device, n, ld, S).run(lib, mode, to(i_all[sl]), to(j_all[sl]), to(aux[sl]), emb, bias, ld, 1e-5, 8 * S)
        rows = one.uniq[:one.U].long()
        at = torch.as_tensor(slot_big[rows.cpu().numpy()]).long().to(cuda_device)
        assert bool((at >= 0).all())
        assert torch.equal(big.uniq[at], one.uniq[:one.U])
        assert torch.equal(_bits(big.rows[at]), _bits(one.rows[:one.U]))
        assert torch.equal(_bits(big.bias[at]), _bits(one.bias[:one.U]))


def _long_batch(rs, n, B, long_len):
    i, j = _batch(rs, n, B, centre_every=7)
    if long_len:
        i[:long_len] = 3                                # one row with more than long_len entries
    return i, j


@pytest.mark.parametrize("B,long_len", [(1025, 0), (4096, 0), (50000, 30500)])
def test_large_batch_steps_match_oracle(B, long_len, cuda_device):
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.generator import Generator
    from oracle import updates
    rs = np.random.RandomState(B)
    n, d, steps = 3000, 64, 3
    emb = rs.normal(0, 0.5, size=(n, d))
    dis, gen = Discriminator(n, emb, device=cuda_device), Generator(n, emb, device=cuda_device)
    od, og = updates.Discriminator(n, emb, 1e-3, 1e-5), updates.Generator(n, emb, 1e-3, 1e-5)
    for _ in range(steps):
        i, j = _long_batch(rs, n, B, long_len)
        lab = (rs.random_sample(B) < 0.5).astype(np.float32)
        rew = (rs.random_sample(B) * 3).astype(np.float32)
        dis.d_step(i, j, lab); od.d_updates(i, j, lab)
        gen.g_step(i, j, rew); og.g_updates(i, j, rew)
        assert int((dis.row_slot != -1).sum()) == 0 and int((gen.row_slot != -1).sum()) == 0
    for m, o in ((dis, od), (gen, og)):
        assert close(m.embedding_numpy(), o.E, steps=steps) and close(m.bias_t.cpu().numpy(), o.b, steps=steps)
        assert close(m.m_emb[:, :d].cpu().numpy(), o.adam.m_e, steps=steps)
        assert close(m.v_emb[:, :d].cpu().numpy(), o.adam.v_e, steps=steps)
        assert m.step_count == steps


def test_large_batch_step_is_deterministic(cuda_device):
    import torch
    from graphgan_b200.discriminator import Discriminator
    rs = np.random.RandomState(5)
    n, d, B = 4000, 128, 50000
    emb = rs.normal(0, 0.5, size=(n, d))
    i, j = _long_batch(rs, n, B, 30500)
    lab = (rs.random_sample(B) < 0.5).astype(np.float32)
    runs = []
    for _ in range(2):
        m = Discriminator(n, emb, device=cuda_device)
        m.d_step(i, j, lab)
        torch.cuda.synchronize()
        runs.append(m)
    for name in ("emb", "bias_t", "m_emb", "v_emb", "m_bias", "v_bias"):
        assert torch.equal(getattr(runs[0], name), getattr(runs[1], name)), name


def test_c_loop_equals_step_by_step(cuda_device):
    """train_steps above GG_MAX_BATCH (gg_train_steps_ex) equals a per-batch step() loop bit for bit, with shuffled
    starts and a short last batch; the persistent loops refuse such batches."""
    import torch
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.generator import Generator
    rs = np.random.RandomState(8)
    n, d, M, B = 6000, 50, 20000, 3000
    emb = rs.normal(0, 0.5, size=(n, d))
    i = np.repeat(rs.randint(0, n, M // 40 + 1), 40)[:M].astype(np.int32)    # centres repeated: long slots
    j = rs.randint(0, n, M).astype(np.int32)
    starts = list(range(0, M, B))
    rs.shuffle(starts)
    for cls, aux in ((Discriminator, (rs.random_sample(M) < 0.5).astype(np.float32)),
                     (Generator, (rs.random_sample(M) * 3).astype(np.float32))):
        a = cls(n, emb, device=cuda_device)
        for s0 in starts:
            a.step(i[s0:s0 + B], j[s0:s0 + B], aux[s0:s0 + B])
        b = cls(n, emb, device=cuda_device)
        b.train_steps(i, j, aux, starts, B, persistent=None)
        for name in ("emb", "bias_t", "m_emb", "v_emb", "m_bias", "v_bias"):
            assert torch.equal(getattr(a, name), getattr(b, name)), name
        assert a.beta1_power == b.beta1_power and a.beta2_power == b.beta2_power and a.step_count == b.step_count == len(starts)
        assert int((b.row_slot != -1).sum()) == 0
        for how in (True, "two-barrier"):
            with pytest.raises(ValueError):
                b.train_steps(i, j, aux, starts, B, persistent=how)


def test_session_feed_and_trainer_epoch(cuda_device, tmp_path, monkeypatch):
    """A Session.run(d_updates) feed of 3000 pairs matches the oracle; one epoch of GraphGAN.train() with
    batch_size_dis = batch_size_gen = 2048 completes with one optimizer step per batch."""
    from graphgan_b200 import config, graph as G
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.graph_gan import GraphGAN
    from graphgan_b200.session import Session
    from oracle import updates
    rs = np.random.RandomState(4)
    n, d, B = 700, 50, 3000
    emb = rs.normal(0, 0.5, size=(n, d))
    dis, od, sess = Discriminator(n, emb, device=cuda_device), updates.Discriminator(n, emb, 1e-3, 1e-5), Session()
    i, j = _batch(rs, n, B)
    lab = (rs.random_sample(B) < 0.5).astype(int)
    sess.run(dis.d_updates, feed_dict={dis.node_id: i, dis.node_neighbor_id: j, dis.label: lab})
    od.d_updates(i, j, lab.astype(np.float32))
    assert close(sess.run(dis.embedding_matrix), od.E, steps=1)

    c = loader.load("rand1200")
    for k, v in dict(n_emb=int(c.emb_g.shape[1]), n_epochs=1, n_epochs_dis=1, dis_interval=1, n_epochs_gen=1, gen_interval=1,
                     n_sample_gen=2, device=str(cuda_device), seed=13, app="none", batch_size_dis=2048, batch_size_gen=2048,
                     emb_filenames=[str(tmp_path / "gen.emb"), str(tmp_path / "dis.emb")],
                     result_filename=str(tmp_path / "res.txt"), model_log=str(tmp_path / "log") + "/").items():
        monkeypatch.setattr(config, k, v)
    gan = GraphGAN(host_graph=G.HostGraph(c.train_edges, c.test_edges), node_embed_init_d=c.emb_d, node_embed_init_g=c.emb_g)
    sizes = {}
    for kind in ("d", "g"):
        orig = getattr(gan, "prepare_data_for_" + kind)
        def wrapped(orig=orig, kind=kind):
            out = orig()
            sizes[kind] = len(out[0])
            return out
        setattr(gan, "prepare_data_for_" + kind, wrapped)
    gan.train()
    assert sizes["d"] > 2048
    assert gan.discriminator.step_count == -(-sizes["d"] // 2048)
    assert gan.generator.step_count == -(-sizes["g"] // 2048)
    for m in (gan.discriminator, gan.generator):
        assert bool(np.isfinite(m.embedding_numpy()).all()) and int((m.row_slot != -1).sum()) == 0
