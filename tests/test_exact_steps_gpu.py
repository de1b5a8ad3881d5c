"""Training on the exact game on the device (csrc/adam.cu: gg_adam_apply_dense; GraphGAN.exact_d_step / exact_g_step /
exact_d_phase; DESIGN.md section 5.5).

Bars: with scale 1, lambda 0 and acc = (double) g32 the dense step gives the bits of gg_adam_apply fed the same fp32 rows,
at every row stride; with lambda != 0 and scale = +-1/n it gives the bits of the numpy statement
(tests/exact_steps_oracle.py) for both models' bias rules, pad columns exactly 0; a D phase with the law computed once
gives the bits of one that recomputes it every step; one G step lowers the mean value and one D step raises it, by the
first-order amount within 10 %; steps do not depend on the root order, a repeat or the scratch budget; and train() with
config.exact_roots keeps its result file, touches no sampling state and resumes from a checkpoint bit for bit.
"""
import numpy as np
import pytest

from tests import exact_steps_oracle as eso
from tests import update_bits_oracle as ubo
from tests.golden import loader

pytestmark = pytest.mark.gpu

F = np.float32
NAMES = ("emb", "bias_t", "m_emb", "v_emb", "m_bias", "v_bias")


def _bits(t):
    return t.detach().cpu().numpy().view(np.uint8).tobytes()


def _model_bits(m):
    return [_bits(getattr(m, k)) for k in NAMES] + [float(m.beta1_power), float(m.beta2_power), m.step_count]


def _load(model, st):
    import torch
    for k, v in st.items():
        getattr(model, k).copy_(torch.as_tensor(v))


# ------------------------------------------------------------------ the device step
@pytest.mark.parametrize("n_emb", [20, 50, 100, 200, 300, 512])
def test_dense_step_is_the_sparse_step(n_emb, cuda_device):
    """scale 1, lambda 0, acc = (double) g32 on a row subset and 0 elsewhere: the bits of gg_adam_apply fed the same rows"""
    import torch
    from graphgan_b200.model import PairModel
    n = 700
    rs = np.random.RandomState(n_emb)
    init = rs.normal(0, 0.5, (n, n_emb)).astype(F)
    a, b = (PairModel(n, init, lr=1e-3, lam=0.0, device=cuda_device) for _ in range(2))
    st = eso.random_state(n, n_emb, a.ld, rs)
    st["emb"][:, :n_emb] = init
    for m in (a, b):
        _load(m, st)
        m.beta1_power, m.beta2_power = F(0.9) ** 4, F(0.999) ** 4
    rows = np.sort(rs.choice(n, 150, replace=False))
    g = np.zeros((len(rows), a.ld), F)
    g[:, :n_emb] = rs.normal(0, 0.1, (len(rows), n_emb)).astype(F)
    gb = rs.normal(0, 0.1, len(rows)).astype(F)
    a.row_slot[torch.as_tensor(rows).to(cuda_device)] = torch.arange(len(rows), dtype=torch.int32, device=cuda_device)
    a.grad_rows[:len(rows)] = torch.as_tensor(g).to(cuda_device)
    a.grad_bias[:len(rows)] = torch.as_tensor(gb).to(cuda_device)
    a.apply_adam()
    acc = torch.zeros((n, a.ld), dtype=torch.float64, device=cuda_device)
    acc_b = torch.zeros(n, dtype=torch.float64, device=cuda_device)
    acc[torch.as_tensor(rows).to(cuda_device)] = torch.as_tensor(g).double().to(cuda_device)
    acc_b[torch.as_tensor(rows).to(cuda_device)] = torch.as_tensor(gb).double().to(cuda_device)
    b.apply_dense_grad(acc, acc_b, 1.0)
    torch.cuda.synchronize()
    assert _model_bits(a) == _model_bits(b)
    assert not b.emb[:, n_emb:].any() and int((a.row_slot != -1).sum()) == 0


@pytest.mark.parametrize("n_emb", [20, 300])
@pytest.mark.parametrize("which", ["generator", "discriminator"])
def test_dense_step_matches_numpy(which, n_emb, cuda_device):
    """three steps with lambda != 0 and scale = +-1/n against the numpy statement, bit for bit; the generator's biases
    take no L2 (generator.py:28-29), the discriminator's do; pad columns of E, m and v stay exactly 0"""
    import torch
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.generator import Generator
    n = 500
    rs = np.random.RandomState(n_emb + 7)
    init = rs.normal(0, 0.5, (n, n_emb)).astype(F)
    m = (Generator if which == "generator" else Discriminator)(n, init, device=cuda_device)
    m.lam = F(0.05)
    st = eso.random_state(n, n_emb, m.ld, rs)
    st["emb"][:, :n_emb] = init
    _load(m, st)
    lam_b = 0.0 if which == "generator" else 0.05
    b1p, b2p = F(0.9), F(0.999)
    for scale in (1.0 / 7, -1.0 / 5, 1.0 / 3):
        acc = np.zeros((n, m.ld))
        acc[:, :n_emb] = rs.normal(0, 2.0, (n, n_emb))
        acc_b = rs.normal(0, 2.0, n)
        lt = ubo.lr_t(m.lr, b1p, b2p)
        assert float(m.lr_t()) == float(lt)
        m.apply_dense_grad(torch.as_tensor(acc).to(cuda_device), torch.as_tensor(acc_b).to(cuda_device), scale)
        eso.dense_step(st, acc, acc_b, scale, 0.05, lam_b, lt)
        b1p, b2p = F(b1p * F(0.9)), F(b2p * F(0.999))
        for k in NAMES:
            assert ubo.same(getattr(m, k).cpu().numpy(), st[k]), (scale, k)
        assert m.beta1_power == b1p and m.beta2_power == b2p
    for k in ("emb", "m_emb", "v_emb"):
        assert not getattr(m, k)[:, n_emb:].any(), k
    assert m.step_count == 3


def test_dense_step_refuses_wrong_gradients(cuda_device):
    import torch
    from graphgan_b200.generator import Generator
    m = Generator(40, np.zeros((40, 8), F), device=cuda_device)
    ok_e = torch.zeros((40, m.ld), dtype=torch.float64, device=cuda_device)
    ok_b = torch.zeros(40, dtype=torch.float64, device=cuda_device)
    for e, b in ((ok_e.float(), ok_b), (ok_e, ok_b[:39]), (ok_e[:, :8], ok_b), (ok_e.cpu(), ok_b)):
        with pytest.raises(ValueError):
            m.apply_dense_grad(e, b, 1.0)
    assert m.step_count == 0


# ------------------------------------------------------------------ the steps of the game
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
    for m, s in ((gan.generator, 0.2), (gan.discriminator, 0.3)):
        m.bias_t.copy_(torch.as_tensor(rs.normal(0, s, hg.n_node).astype(F)))
    return gan, c


def _snap(gan):
    return gan.generator.state_dict(), gan.discriminator.state_dict()


def _restore(gan, s):
    gan.generator.load_state_dict(s[0])
    gan.discriminator.load_state_dict(s[1])


def test_d_phase_law_reuse_is_bit_identical(cuda_device, tmp_path, monkeypatch):
    """three D steps with G's law computed once give the bits of three steps that recompute it (a budget below R N 8)"""
    gan, _ = _gan(monkeypatch, tmp_path, cuda_device, "cagrqc")
    gan.prepare_data_for_d()                                  # father-removal bits: the law of a trained run
    assert gan.device_graph.d1_bits.any()
    roots = gan.exact_roots()
    calls = []
    dist_fn = gan.sampler.distribution
    gan.sampler.distribution = lambda *a, **k: (calls.append(1), dist_fn(*a, **k))[1]
    s0 = _snap(gan)
    outs_a = gan.exact_d_phase(roots, 3)
    assert len(calls) == 1
    bits_a = _model_bits(gan.discriminator), _model_bits(gan.generator)
    _restore(gan, s0)
    outs_b = gan.exact_d_phase(roots, 3, max_scratch_bytes=len(roots) * gan.n_node * 8 - 1)
    assert len(calls) == 1                                    # recomputed inside every step instead
    assert bits_a == (_model_bits(gan.discriminator), _model_bits(gan.generator))
    assert [[_bits(x) for x in o] for o in outs_a] == [[_bits(x) for x in o] for o in outs_b]
    assert gan.discriminator.step_count == 3


def _mean_v(pos, neg, ok):
    sel = ok.bool()
    return float((pos + neg)[sel].sum().item()) / int(sel.sum().item())


@pytest.mark.parametrize("name", ["tiny", "rand300", "cagrqc"])
def test_first_order(name, cuda_device, tmp_path, monkeypatch):
    """at lr 1e-4 one G step lowers the mean V and one D step raises it, and the change is <grad V, theta_new - theta_old>
    (fp64, actual parameter deltas) within 10 %"""
    gan, _ = _gan(monkeypatch, tmp_path, cuda_device, name)
    roots = gan.exact_roots()
    ratios = {}
    for phase, model, grad_fn, step_fn in (("G", gan.generator, gan.game_value_grad, gan.exact_g_step),
                                           ("D", gan.discriminator, gan.game_value_grad_d, gan.exact_d_step)):
        model.lr = F(1e-4)
        pos, neg, ok, gE, gb = grad_fn(roots)
        n = int(ok.sum().item())
        assert n > 0
        e0, b0 = model.emb.double().clone(), model.bias_t.double().clone()
        pre = step_fn(roots)
        assert [_bits(x) for x in pre] == [_bits(x) for x in (pos, neg, ok)]
        pred = float(((gE * (model.emb.double() - e0)).sum() + (gb * (model.bias_t.double() - b0)).sum()).item()) / n
        actual = _mean_v(*gan.game_value(roots)) - _mean_v(pos, neg, ok)
        ratios[phase] = actual / pred
        assert (actual < 0) if phase == "G" else (actual > 0), (phase, actual)
        assert abs(actual / pred - 1) <= 0.1, (phase, actual, pred)
    print("first-order ratio %s: G %.4f D %.4f" % (name, ratios["G"], ratios["D"]))


def test_steps_are_deterministic(cuda_device, tmp_path, monkeypatch):
    """a D step then a G step: the same bits for a permuted root list, a repeat and a budget of one root per chunk"""
    gan, _ = _gan(monkeypatch, tmp_path, cuda_device, "cagrqc")
    gan.prepare_data_for_d()
    roots = gan.exact_roots()
    perm = np.random.RandomState(2).permutation(len(roots))
    s0 = _snap(gan)
    got = []
    for rr, budget in ((roots, None), (roots, None), (roots[perm], None), (roots, 1)):
        _restore(gan, s0)
        inv = np.argsort(perm) if rr is not roots else np.arange(len(roots))
        d = gan.exact_d_step(rr, max_scratch_bytes=budget)
        g = gan.exact_g_step(rr, max_scratch_bytes=budget)
        vals = [_bits(x.cpu()[inv]) for x in d + g]
        got.append((vals, _model_bits(gan.discriminator), _model_bits(gan.generator)))
    assert all(x == got[0] for x in got[1:])
    assert got[0][1][-1] == 1 and got[0][2][-1] == 1


def test_trainer(cuda_device, tmp_path, monkeypatch):
    """train() with exact_roots = 64 on CA-GrQc, 2 epochs of 2 D + 2 G steps: the usual result lines plus the value line,
    the sampling state untouched, eight trace entries; save -> load -> continue equals the uninterrupted run"""
    import torch
    c = loader.load("cagrqc")

    def wr(name, e):
        p = tmp_path / name
        p.write_text("".join("%d\t%d\n" % (a, b) for a, b in e))
        return str(p)
    cfg = dict(app="link_prediction", test_filename=wr("test.txt", c.test_edges),
               test_neg_filename=wr("test_neg.txt", c.test_neg_edges), n_epochs=2, n_epochs_dis=2, n_epochs_gen=2,
               dis_interval=1, gen_interval=1, value_roots=16, save_steps=1)
    a, _ = _gan(monkeypatch, tmp_path, cuda_device, "cagrqc", tag="a", **cfg)
    bits0, rng0 = a.device_graph.d1_bits.clone(), a.shuffle_rng.get_state()
    a.train()
    lines = (tmp_path / "resa.txt").read_text().splitlines()
    assert [ln.split(":")[0] for ln in lines] == ["gen", "dis", "value"] * 3
    assert torch.equal(a.device_graph.d1_bits, bits0) and a.pass_counter == 0
    rng1 = a.shuffle_rng.get_state()
    assert rng1[0] == rng0[0] and np.array_equal(rng1[1], rng0[1]) and rng1[2:] == rng0[2:]
    assert [(p, s) for p, s, _, _ in a.exact_trace] == [("D", 0), ("D", 1), ("G", 0), ("G", 1)] * 2
    assert all(n > 0 and np.isfinite(v) for _, _, v, n in a.exact_trace)
    assert a.generator.step_count == 4 and a.discriminator.step_count == 4
    # the run was saved at the start of epoch 1: load it and run that epoch again
    from graphgan_b200 import config
    monkeypatch.setattr(config, "n_epochs", 1)
    monkeypatch.setattr(config, "load_model", True)
    b, _ = _gan(monkeypatch, tmp_path, cuda_device, "cagrqc", tag="b", **dict(cfg, n_epochs=1))
    b.train()
    for ma, mb in ((a.generator, b.generator), (a.discriminator, b.discriminator)):
        assert _model_bits(ma) == _model_bits(mb)
    assert b.exact_trace == a.exact_trace[4:]
