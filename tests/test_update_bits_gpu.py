"""GPU tests of the training updates against tests/update_bits_oracle.py: equality, not a tolerance.

The sparse gradient (gg_pair_grad, gg_pair_grad_ex one-CTA and multi-CTA), the Adam sweep (every gg_adam_apply path,
teacher-forced), the step loops (step, gg_train_steps[_ex], gg_train_loop, gg_train_fused), the simulated data-parallel
step and one epoch of GraphGAN.train() must give the oracle's values exactly (-0 == +0, no NaN).  Every batch is checked
on the host to hold no pair whose fp64 sigmoid could round differently with a 1-ulp different exp."""
import ctypes as C
import math

import numpy as np
import pytest

from tests import update_bits_oracle as ub
from tests.golden import loader
from tests.test_large_batch_gpu import Grad, _batch as centre_batch

pytestmark = pytest.mark.gpu
F = np.float32
MULTI_CTA = 1   # GG_GRAD_MULTI_CTA
STATE = ("emb", "bias_t", "m_emb", "v_emb", "m_bias", "v_bias")
ADAM_PATHS = ("ldg", "tma", "tma256x2", "tma512x3", "ws16", "ws8")


def _to(x, dev):
    import torch
    return torch.as_tensor(np.ascontiguousarray(x)).to(dev)


def _paths(B):
    """gg_pair_grad (up to 1024 pairs), gg_pair_grad_ex without flags, gg_pair_grad_ex forced multi-CTA."""
    return ([None] if B <= 1024 else []) + [0, MULTI_CTA]


def _check_grad(lib, dev, mode, i, j, aux, E, b, lam, batch_total=0):
    """Every gradient path on (i, j, aux) against the oracle: n_unique, uniq_ids, grad_rows (pad columns included),
    grad_bias, row_slot."""
    n, ld = E.shape
    uniq, row_slot, rows, gb, amb = ub.grad(mode, i, j, aux, E, b, lam, batch_total or None)
    assert not amb.any()
    U = len(uniq)
    args = (_to(i.astype(np.int32), dev), _to(j.astype(np.int32), dev), _to(aux.astype(F), dev), _to(E, dev), _to(b, dev))
    for flags in _paths(len(i)):
        g = Grad(dev, n, ld, len(i)).run(lib, mode, *args, ld, float(lam), batch_total=batch_total, ex_flags=flags)
        assert g.U == U, flags
        assert np.array_equal(g.uniq[:U].cpu().numpy(), uniq), flags
        got = g.rows[:U].cpu().numpy()
        assert ub.same(got, rows), (flags, np.argwhere(got != rows)[:5])
        assert ub.same(g.bias[:U].cpu().numpy(), gb), flags
        assert np.array_equal(g.row_slot.cpu().numpy(), row_slot), flags


def _pairs(rs, n, B):
    i, j = centre_batch(rs, n, B, centre_every=5)
    return i.astype(np.int64), j.astype(np.int64)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("ld,d,B", [(32, 29, 1), (32, 32, 2), (64, 61, 7), (128, 127, 64), (256, 250, 333), (512, 509, 1023),
                                    (128, 100, 1024), (64, 63, 1025), (32, 31, 4096)])
def test_gradient_equals_oracle(mode, ld, d, B, cuda_device):
    from graphgan_b200 import _cabi
    rs = np.random.RandomState(ld * 7 + B + mode)
    n = max(64, B // 3)
    E = ub.pad(rs.normal(0, 0.5, size=(n, d)), ld)
    b = rs.normal(0, 0.5, size=n).astype(F)
    i, j = _pairs(rs, n, B)
    aux = ((rs.random_sample(B) < 0.5) if mode == 0 else rs.random_sample(B) * 3).astype(F)
    _check_grad(_cabi.lib(), cuda_device, mode, i, j, aux, E, b, 1e-5)
    if mode == 1:                      # one rank's slice of a larger batch: the mean is over batch_total pairs
        _check_grad(_cabi.lib(), cuda_device, mode, i, j, aux, E, b, 1e-5, batch_total=3 * B + 1)


@pytest.mark.parametrize("mode", [0, 1])
def test_gradient_of_a_50000_pair_batch_with_a_30500_entry_row(mode, cuda_device):
    from graphgan_b200 import _cabi
    rs = np.random.RandomState(50 + mode)
    n, ld, B = 40000, 128, 50000
    E = ub.pad(rs.normal(0, 0.3, size=(n, 120)), ld)
    b = rs.normal(0, 0.5, size=n).astype(F)
    i, j = rs.randint(0, n, B), rs.randint(0, n, B)
    i[:30500] = 17                     # one row with 30 500 i-side entries (and some j-side ones)
    j = ub.avoid_ambiguous(E, b, i, j)
    aux = ((rs.random_sample(B) < 0.5) if mode == 0 else rs.random_sample(B) * 3).astype(F)
    _check_grad(_cabi.lib(), cuda_device, mode, i.astype(np.int64), j.astype(np.int64), aux, E, b, 1e-5)


def _edge_scores():
    """fp32 scores at the edges of the sigmoid and the generator clip: the 129 fp32 values around the point where
    f32(sigma(s)) crosses 1e-5f, scores where p rounds to 1.0f, and scores near -20, -100 and -800."""
    s = np.float32(math.log(1e-5 / (1 - 1e-5)))
    while ub.sigmoid(np.array([s], F))[0][0] >= ub.CLIP:
        s = np.nextafter(s, F(-20))
    while ub.sigmoid(np.array([s], F))[0][0] < ub.CLIP:
        s = np.nextafter(s, F(0))      # s: the smallest fp32 score whose p passes the clip
    around = [s]
    for _ in range(64):
        around.append(np.nextafter(around[-1], F(0)))
        around.insert(0, np.nextafter(around[0], F(-20)))
    far = [17.5, 18.0, 25.0, 88.0, 100.0, -20.0, np.nextafter(F(-20), F(0)), -100.0, -103.5, -745.0, -800.0, 0.0, 3.0, -3.0]
    return np.array(around + far, F), 64


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("ld", [32, 256])
def test_gradient_at_score_edges(mode, ld, cuda_device):
    """Row 0 is all zeros, so s(0, j) = b_j exactly and the bias places every score.  Labels 0 and 1, rewards of 0."""
    from graphgan_b200 import _cabi
    s, at = _edge_scores()
    p, amb = ub.sigmoid(s)
    assert not amb.any()
    assert p[at] >= ub.CLIP and p[at - 1] < ub.CLIP and (p == 1).sum() >= 3 and (p == 0).sum() >= 2
    B = len(s)
    rs = np.random.RandomState(ld + mode)
    n = B + 1
    E = ub.pad(rs.normal(0, 0.5, size=(n, ld - 3)), ld)
    E[0] = 0
    b = np.zeros(n, F)
    b[1:] = s
    i, j = np.zeros(B, np.int64), np.arange(1, n, dtype=np.int64)
    aux = ((np.arange(B) % 2) if mode == 0 else rs.random_sample(B) * 3).astype(F)
    if mode == 1:
        aux[::7] = 0
    _check_grad(_cabi.lib(), cuda_device, mode, i, j, aux, E, b, 1e-5)
    # the clip itself: below the crossing the generator's delta is exactly 0, at it and above it is not
    d, _ = ub.delta(1, s, np.ones(B, F), B)
    assert (d[:at] == 0).all() and (d[at:at + 65] != 0).all()


@pytest.mark.parametrize("ld,n", [(32, 257), (128, 3000), (256, 700), (512, 300)])
def test_adam_teacher_forced_every_path(ld, n, cuda_device):
    """Gradient buffers, m, v and row_slot written by hand, then gg_adam_apply on every path: all six state tensors equal
    the GG_ADAM1 oracle over all rows, and row_slot is reset.  Includes |g| where g^2 is subnormal (1e-20) or rounds to
    0 (1e-23), |g| where g^2 overflows (the update is 0), v = 0 with g = 0, and subnormal m."""
    import torch
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rs = np.random.RandomState(ld + n)
    U = n // 3
    uniq = rs.choice(n, U, replace=False).astype(np.int32)
    g_rows = (rs.normal(0, 1, size=(U, ld)) * 10.0 ** rs.randint(-8, 2, size=(U, 1))).astype(F)
    g_bias = rs.normal(0, 1, size=U).astype(F)
    specials = np.array([1e-20, -1e-20, 1e-23, -1e-23, 1e19, 2e19, -3e19, 0.0], F)
    g_rows[:len(specials), :8] = specials
    g_rows[0, 8:16] = specials[::-1]
    g_bias[:len(specials)] = specials
    m = (rs.normal(0, 1e-3, size=(n, ld))).astype(F)
    v = (rs.random_sample((n, ld)) * 1e-6).astype(F)
    m_b, v_b = rs.normal(0, 1e-3, size=n).astype(F), (rs.random_sample(n) * 1e-6).astype(F)
    m[uniq[:3], :8] = F(3e-39)                    # subnormal m
    m[uniq[3], :8] = F(-1e-45)
    v[uniq[:8], :8] = 0                           # v = 0 (and g = 0 in the last special)
    untouched = np.setdiff1d(np.arange(n), uniq)[:4]
    v[untouched] = 0
    m[untouched[0]] = F(-0.0)
    m_b[uniq[:8]], v_b[uniq[:8]] = F(1e-40), 0
    x = (rs.normal(0, 0.5, size=(n, ld))).astype(F)
    xb = rs.normal(0, 0.5, size=n).astype(F)
    lr_t = ub.lr_t(1e-3, F(0.9) ** 3, F(0.999) ** 3)
    b1, b2, eps = F(0.9), F(0.999), F(1e-8)
    want = [a.copy() for a in (x, m, v, xb, m_b, v_b)]
    G = np.zeros_like(x)
    G[uniq] = g_rows
    Gb = np.zeros_like(xb)
    Gb[uniq] = g_bias
    ub.adam1(want[0], want[1], want[2], G, lr_t, b1, b2, eps)
    ub.adam1(want[3], want[4], want[5], Gb, lr_t, b1, b2, eps)
    assert (want[2] == np.inf).any() and ((want[2] > 0) & (want[2] < np.finfo(F).tiny)).any()
    row_slot = np.full(n, -1, np.int32)
    row_slot[uniq] = np.arange(U, dtype=np.int32)
    cap = 2 * U
    rows_buf = np.full((cap, ld), 5.0, F)
    rows_buf[:U] = g_rows
    bias_buf = np.full(cap, 5.0, F)
    bias_buf[:U] = g_bias
    try:
        for path in ADAM_PATHS:
            _cabi.check(lib.gg_set_adam_path(path.encode()), path)
            st = [_to(a, cuda_device) for a in (x, m, v, xb, m_b, v_b)]
            slot_d = _to(row_slot, cuda_device)
            nu = torch.tensor([U], dtype=torch.int32, device=cuda_device)
            ids = _to(np.concatenate([uniq, np.zeros(cap - U, np.int32)]), cuda_device)
            gr, gbb = _to(rows_buf, cuda_device), _to(bias_buf, cuda_device)
            _cabi.check(lib.gg_adam_apply(n, ld, *(t.data_ptr() for t in st), nu.data_ptr(), ids.data_ptr(), gr.data_ptr(),
                                          gbb.data_ptr(), slot_d.data_ptr(), C.c_float(lr_t), C.c_float(b1), C.c_float(b2), C.c_float(eps), None),
                        "gg_adam_apply")
            torch.cuda.synchronize()
            for name, got, w in zip(("emb", "m", "v", "bias", "m_bias", "v_bias"), st, want):
                got = got.cpu().numpy()
                assert ub.same(got, w), (path, name, np.argwhere(got != w)[:5])
            assert int((slot_d != -1).sum()) == 0, path
    finally:
        lib.gg_set_adam_path(b"ldg")


def _compare(model, ora, what):
    import torch
    torch.cuda.synchronize()
    for name, w in ora.state().items():
        got = getattr(model, name).cpu().numpy()
        assert ub.same(got, w), (what, name, np.argwhere(got != w)[:5])
    assert model.beta1_power == ora.adam.b1p and model.beta2_power == ora.adam.b2p, what
    assert model.lr_t() == ora.adam.lr_t(), what
    assert int((model.row_slot != -1).sum()) == 0, what


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("n,d,M,B", [(700, 50, 1000, 64), (300, 200, 1100, 64), (3000, 100, 2 * 2048 + 500, 2048)])
def test_step_loops_equal_oracle(mode, n, d, M, B, cuda_device):
    """step() per batch, gg_train_steps[_ex] and, up to 1024 pairs, gg_train_loop and gg_train_fused, each against the
    oracle's loop over the same shuffled starts (short last batch)."""
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.generator import Generator
    cls = Discriminator if mode == 0 else Generator
    rs = np.random.RandomState(n + d + mode)
    emb = rs.normal(0, 0.5, size=(n, d))
    i = np.repeat(rs.randint(0, n, M // 3 + 1), 3)[:M].astype(np.int32)
    j = rs.randint(0, n, M).astype(np.int32)
    aux = ((rs.random_sample(M) < 0.5) if mode == 0 else rs.random_sample(M) * 3).astype(F)
    starts = list(range(0, M, B))
    rs.shuffle(starts)
    a = cls(n, emb, device=cuda_device)
    ora = ub.Model(a.emb.cpu().numpy(), a.ld, lr=float(a.lr), lam=float(a.lam))
    assert not ora.steps(mode, i, j, aux, starts, B).any()
    for s0 in starts:
        a.step(i[s0:s0 + B], j[s0:s0 + B], aux[s0:s0 + B])
    _compare(a, ora, "step")
    for how in ((False, "two-barrier", True) if B <= 1024 else (None,)):
        m = cls(n, emb, device=cuda_device)
        m.train_steps(i, j, aux, starts, B, persistent=how)
        _compare(m, ora, how)


def test_long_step_loop_through_subnormal_beta_powers(cuda_device):
    """1 100 steps at tiny n: beta1^t runs into the fp32 subnormals and stops at 4 * 2^-149 (0.9 times it rounds back);
    lr_t and both beta powers, and every state tensor, stay equal to the oracle on every loop."""
    from graphgan_b200.generator import Generator
    rs = np.random.RandomState(1100)
    n, d, B, steps = 16, 20, 8, 1100
    emb = rs.normal(0, 0.5, size=(n, d))
    M = B * steps - 3
    i, j = rs.randint(0, n, M).astype(np.int32), rs.randint(0, n, M).astype(np.int32)
    aux = (rs.random_sample(M) * 3).astype(F)
    starts = list(range(0, M, B))
    rs.shuffle(starts)
    ref = Generator(n, emb, device=cuda_device)
    ora = ub.Model(ref.emb.cpu().numpy(), ref.ld, lr=float(ref.lr), lam=float(ref.lam))
    assert not ora.steps(1, i, j, aux, starts, B).any()
    assert ora.adam.b1p == F(4 * 2.0 ** -149)
    for how in (False, "two-barrier", True):
        m = Generator(n, emb, device=cuda_device)
        m.train_steps(i, j, aux, starts, B, persistent=how)
        _compare(m, ora, how)
    for s0 in starts:
        ref.step(i[s0:s0 + B], j[s0:s0 + B], aux[s0:s0 + B])
    _compare(ref, ora, "step")


@pytest.mark.parametrize("B", [1025, 65536])
@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("mode", [0, 1])
def test_simulated_world_step_equals_oracle(B, world, mode, cuda_device):
    """Slices -> gg_grad_merge_ex -> gg_adam_apply, two steps, against the oracle's world-W step."""
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.generator import Generator
    from tests.dist_large_batch_worker import simulated_merge
    cls = Discriminator if mode == 0 else Generator
    rs = np.random.RandomState(B + world + 10 * mode)
    n, d = 3000, 64
    sim = cls(n, rs.normal(0, 0.5, size=(n, d)), device=cuda_device)
    ora = ub.Model(sim.emb.cpu().numpy(), sim.ld, lr=float(sim.lr), lam=float(sim.lam))
    for _ in range(2):
        i, j = centre_batch(rs, n, B, centre_every=7)
        j = ub.avoid_ambiguous(ora.E, ora.b, i, j)       # the oracle's parameters are the device's (checked below)
        aux = ((rs.random_sample(B) < 0.5) if mode == 0 else rs.random_sample(B) * 3).astype(F)
        assert not ora.world_step(mode, i.astype(np.int64), j.astype(np.int64), aux, world).any()
        simulated_merge(sim, _to(i, cuda_device), _to(j, cuda_device), _to(aux, cuda_device), world)
        sim.apply_adam()
    _compare(sim, ora, "world %d" % world)


def test_trainer_epoch_replays_through_oracle(cuda_device, tmp_path, monkeypatch):
    """One epoch of GraphGAN.train() on rand1200.  The batches each model's train_steps receives are recorded and replayed
    through the oracle (the fed rewards taken as given): the final parameters and Adam state are the oracle's."""
    from graphgan_b200 import graph as G, model as M
    from graphgan_b200.graph_gan import GraphGAN
    from tests.test_updates_gpu import _small_gan_config
    c = loader.load("rand1200")
    config = _small_gan_config(monkeypatch, tmp_path, cuda_device, c)
    monkeypatch.setattr(config, "n_epochs", 1)
    calls = []
    orig = M.PairModel.train_steps

    def record(self, node_id, node_neighbor_id, aux, start_list, batch_size, persistent=None):
        host = lambda x: x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)
        calls.append((self, host(node_id).astype(np.int64), host(node_neighbor_id).astype(np.int64), host(aux).astype(F),
                      list(start_list), int(batch_size)))
        return orig(self, node_id, node_neighbor_id, aux, start_list, batch_size, persistent)

    monkeypatch.setattr(M.PairModel, "train_steps", record)
    gan = GraphGAN(host_graph=G.HostGraph(c.train_edges, c.test_edges), node_embed_init_d=c.emb_d, node_embed_init_g=c.emb_g)
    oras = {id(mm): ub.Model(mm.emb.cpu().numpy(), mm.ld, bias=mm.bias_t.cpu().numpy(), lr=float(mm.lr), lam=float(mm.lam))
            for mm in (gan.generator, gan.discriminator)}
    gan.train()
    assert {id(cl[0]) for cl in calls} == set(oras) and len(calls) >= 4
    for mm, i, j, aux, starts, B in calls:
        assert not oras[id(mm)].steps(mm._step_mode, i, j, aux, starts, B).any()
    for mm in (gan.generator, gan.discriminator):
        _compare(mm, oras[id(mm)], type(mm).__name__)


@pytest.mark.parametrize("ld", [64, 512])
def test_all_score_is_canonical_dot_plus_bias(ld, cuda_device):
    from graphgan_b200.generator import Generator
    rs = np.random.RandomState(ld)
    n = 200
    g = Generator(n, rs.normal(0, 0.5, size=(n, ld - 7)), device=cuda_device)
    g.bias_t.copy_(_to(rs.normal(0, 0.5, size=n).astype(F), cuda_device))
    E, b = g.emb.cpu().numpy(), g.bias_t.cpu().numpy()
    got = g.all_score_matrix().cpu().numpy()
    u, v = np.repeat(np.arange(n), n), np.tile(np.arange(n), n)
    assert np.array_equal(got.reshape(-1).view(np.int32), ub.score(E, b, u, v).view(np.int32))


def test_pair_reward_within_the_documented_error(cuda_device):
    """reward = logf(1 + expf(clip(s, -10, 10))) (discriminator.py:33-34) against fp64 softplus of the clipped fp32 s.
    CUDA documents expf to 2 ulp and logf to 1 ulp; with the rounding of 1 + e the bound is
        |r - log(1 + exp(c))| <= (2 ulp(e) + ulp(1 + e) / 2) / (1 + e) + ulp(r)
    (a relative error x of the argument of log moves log by at most x / (1 - x)).  The scores are exact: row 0 is zero."""
    from graphgan_b200.discriminator import Discriminator
    s = np.array([10, -10, np.nextafter(F(10), F(11)), np.nextafter(F(10), F(9)), np.nextafter(F(-10), F(-11)),
                  np.nextafter(F(-10), F(-9)), 0, -0.0, 20, -20, 1e-7, 5.5, -5.5, 88, -88], F)
    n = len(s) + 1
    rs = np.random.RandomState(4)
    emb = rs.normal(0, 0.5, size=(n, 40))
    emb[0] = 0
    m = Discriminator(n, emb, device=cuda_device)
    b = np.zeros(n, F)
    b[1:] = s
    m.bias_t.copy_(_to(b, cuda_device))
    got = m.reward_pairs(np.zeros(len(s), np.int32), np.arange(1, n, dtype=np.int32)).cpu().numpy().astype(np.float64)
    c = np.clip(s, F(-10), F(10)).astype(np.float64)
    assert np.array_equal(c, np.clip(s.astype(np.float64), -10, 10))
    e = np.exp(c)
    ulp = lambda x: np.spacing(np.abs(x).astype(F)).astype(np.float64)
    want = np.log1p(e)
    x = (2 * ulp(e) + ulp(1 + e) / 2) / (1 + e)
    bound = x / (1 - x) + ulp(want)
    assert np.all(np.abs(got - want) <= bound), np.abs(got - want) / bound
    assert got[0] == got[2] == got[8] and got[1] == got[4] == got[9]      # the clip
