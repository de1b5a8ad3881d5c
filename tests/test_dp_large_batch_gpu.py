"""GPU tests of the data-parallel step above GG_MAX_BATCH pairs on one H100.  Ranks are simulated on one device: each
rank's block of the all-gathered buffer is gg_pair_grad_ex on its slice (tests/dist_large_batch_worker.py).
  - the forced multi-CTA merge equals the one-CTA gg_grad_merge bit for bit;
  - above the one-CTA limit the merge equals a numpy emulation of its contract exactly;
  - a simulated world-W step (slices -> merge -> Adam) agrees with the single-GPU PairModel.step;
  - world 1 end to end under torch.distributed: DataParallelStep equals PairModel bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.dist_large_batch_worker import batch, gathered_blocks, merge_ex, simulated_merge
from tests.test_large_batch_gpu import _batch as one_gpu_batch, close

pytestmark = pytest.mark.gpu
MULTI_CTA = 1   # GG_GRAD_MULTI_CTA
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Out:
    """Fresh merge outputs (poisoned) and a row_slot that holds rank 0's local slots, as the slice gradient leaves it."""

    def __init__(self, dev, n, ld, E, gathered, cap):
        import torch
        self.n_unique = torch.zeros(1, dtype=torch.int32, device=dev)
        self.uniq = torch.full((E,), -7, dtype=torch.int32, device=dev)
        self.rows = torch.full((E, ld), 7.0, dtype=torch.float32, device=dev)
        self.bias = torch.full((E,), 7.0, dtype=torch.float32, device=dev)
        self.row_slot = torch.full((n,), -1, dtype=torch.int32, device=dev)
        g = gathered.view(torch.int32)
        nu0 = int(g[cap * ld + 2 * cap].item())
        self.row_slot[g[cap * ld + cap:cap * ld + cap + nu0].long()] = torch.arange(nu0, dtype=torch.int32, device=dev)

    def args(self):
        return self.n_unique, self.uniq, self.rows, self.bias, self.row_slot


def _bits(t):
    return t.view(__import__("torch").int32)


def _setup(dev, rs, n, d, B, mode):
    import torch
    from graphgan_b200.sampler import pad_embedding
    emb = pad_embedding(rs.normal(0, 0.5, size=(n, d)), dev)
    bias = torch.as_tensor(rs.normal(0, 0.1, size=n).astype(np.float32)).to(dev)
    i, j, aux = batch(rs, n, B, mode)
    to = lambda x: torch.as_tensor(x).to(dev)
    return emb, bias, to(i), to(j), to(aux)


def _block_ids(gathered, world, cap, ld):
    g = gathered.view(__import__("torch").int32).cpu().numpy().reshape(world, -1)
    return [g[r, cap * ld + cap:cap * ld + cap + g[r, cap * ld + 2 * cap]] for r in range(world)]


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("ld", [32, 64, 128, 256])
@pytest.mark.parametrize("mode", [0, 1])
def test_multi_cta_merge_equals_one_cta_merge(world, ld, mode, cuda_device):
    """n_unique, uniq_ids order, rows, bias and row_slot, bit for bit.  At world >= 3 the last rank sends nothing (nu = 0);
    the batch's centre row is in every rank's block."""
    import torch
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rs = np.random.RandomState(world * 100 + ld + mode)
    n, B = 500, 1000
    emb, bias, i, j, a = _setup(cuda_device, rs, n, ld - 3, B, mode)
    scratch_slot = torch.full((n,), -1, dtype=torch.int32, device=cuda_device)
    empty = (world - 1,) if world >= 3 else ()
    gathered, cap = gathered_blocks(lib, mode, i, j, a, emb, bias, ld, 1e-5, world, scratch_slot, empty_ranks=empty)
    ids = _block_ids(gathered, world, cap, ld)
    assert all(n // 2 in ids[r] for r in range(world) if r not in empty)
    assert all(len(ids[r]) == 0 for r in empty)
    E = world * cap
    assert E <= 16384
    ref, got, dflt = (Out(cuda_device, n, ld, E, gathered, cap) for _ in range(3))
    _cabi.check(lib.gg_grad_merge(world, cap, ld, gathered.data_ptr(), *(t.data_ptr() for t in ref.args()), None), "gg_grad_merge")
    merge_ex(lib, world, cap, ld, gathered, *got.args(), flags=MULTI_CTA)
    merge_ex(lib, world, cap, ld, gathered, *dflt.args(), flags=0)      # without the flag: the one-CTA kernel
    torch.cuda.synchronize()
    U = int(ref.n_unique.item())
    assert U == len(np.unique(np.concatenate(ids))) and U >= 1
    for out in (got, dflt):
        assert int(out.n_unique.item()) == U
        assert torch.equal(out.uniq[:U], ref.uniq[:U])
        assert torch.equal(_bits(out.rows[:U]), _bits(ref.rows[:U]))
        assert torch.equal(_bits(out.bias[:U]), _bits(ref.bias[:U]))
        assert torch.equal(out.row_slot, ref.row_slot)


def emulate_merge(gathered, world, cap, ld, n):
    """The merge contract in numpy: entries in t = r * cap + s order, slots by first occurrence, float32 adds from +0 in
    rank order (a rank holds an id at most once, so one vectorised add per rank is one step of every chain)."""
    g = gathered.cpu().numpy().reshape(world, -1)
    gi = g.view(np.int32)
    blocks = []
    for r in range(world):
        nu = int(gi[r, cap * ld + 2 * cap])
        blocks.append((gi[r, cap * ld + cap:cap * ld + cap + nu], g[r, :cap * ld].reshape(cap, ld)[:nu], g[r, cap * ld:cap * ld + nu]))
    ids = np.concatenate([b[0] for b in blocks])
    _, first = np.unique(ids, return_index=True)
    uniq = ids[np.sort(first)]
    slot = np.full(n, -1, np.int32)
    slot[uniq] = np.arange(uniq.shape[0], dtype=np.int32)
    rows = np.zeros((uniq.shape[0], ld), np.float32)
    bias = np.zeros(uniq.shape[0], np.float32)
    for bid, brows, bbias in blocks:
        s = slot[bid]
        rows[s] = rows[s] + brows
        bias[s] = bias[s] + bbias
    return uniq, rows, bias, slot


def _check_against_emulation(lib, dev, gathered, world, cap, ld, n):
    import torch
    E = world * cap
    assert E > 16384          # beyond gg_grad_merge: the default path is the multi-CTA one
    out = Out(dev, n, ld, E, gathered, cap)
    merge_ex(lib, world, cap, ld, gathered, *out.args(), flags=0)
    uniq, rows, bias, slot = emulate_merge(gathered, world, cap, ld, n)
    U = uniq.shape[0]
    assert int(out.n_unique.item()) == U
    assert np.array_equal(out.uniq[:U].cpu().numpy(), uniq)
    assert np.array_equal(out.rows[:U].cpu().numpy().view(np.int32), rows.view(np.int32))
    assert np.array_equal(out.bias[:U].cpu().numpy().view(np.int32), bias.view(np.int32))
    assert np.array_equal(out.row_slot.cpu().numpy(), slot)
    torch.cuda.synchronize()
    return U


def test_merge_of_c3_hub_batch_equals_emulation(cuda_device):
    """World 8 over slice 0 of the C3-shaped D rows at B = 65 536 (the batch that holds the 13 828-neighbour hub)."""
    import torch
    from graphgan_b200 import _cabi
    from graphgan_b200.discriminator import Discriminator
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from bench_large_batch import d_rows
    lib = _cabi.lib()
    n, d, B, world = 1_000_000, 128, 65536, 8
    centre, neigh, label, _ = d_rows(n)
    m = Discriminator(n, torch.empty((n, d), device=cuda_device).normal_(0, 0.1), device=cuda_device)
    to = lambda x: torch.as_tensor(np.ascontiguousarray(x)).to(cuda_device)
    gathered, cap = gathered_blocks(lib, 0, to(centre[:B]), to(neigh[:B]), to(label[:B]), m.emb, m.bias_t, d, m.lam, world,
                                    m.row_slot)
    ids = _block_ids(gathered, world, cap, d)
    assert np.bincount(np.concatenate(ids)).max() >= 4          # the hub's 27 656 rows span four slices: one slot, four ranks
    U = _check_against_emulation(lib, cuda_device, gathered, world, cap, d, n)
    assert U == len(np.unique(np.concatenate([centre[:B], neigh[:B]])))


@pytest.mark.parametrize("mode", [0, 1])
def test_merge_of_uneven_slices_equals_emulation(mode, cuda_device):
    """World 3, B = 20 001 (slices of 6 667 pairs: multi-CTA slice gradients), long and shared rows."""
    from graphgan_b200 import _cabi
    lib = _cabi.lib()
    rs = np.random.RandomState(3 + mode)
    n, ld, B, world = 3000, 64, 20001, 3
    emb, bias, i, j, a = _setup(cuda_device, rs, n, 60, B, mode)
    import torch
    slot = torch.full((n,), -1, dtype=torch.int32, device=cuda_device)
    gathered, cap = gathered_blocks(lib, mode, i, j, a, emb, bias, ld, 1e-5, world, slot)
    _check_against_emulation(lib, cuda_device, gathered, world, cap, ld, n)


@pytest.mark.parametrize("B", [1025, 4096, 65536])
@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("mode", [0, 1])
def test_simulated_world_step_matches_single_gpu_step(B, world, mode, cuda_device):
    """Two steps of slices -> gg_grad_merge_ex -> gg_adam_apply against PairModel.step, with the bar and the batch shape
    of tests/test_large_batch_gpu.py (the sums differ only in their grouping: per-rank partials, then rank order)."""
    import torch
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.generator import Generator
    cls = Discriminator if mode == 0 else Generator
    rs = np.random.RandomState(B + world + 10 * mode)
    n, d, steps = 3000, 64, 2
    e0 = rs.normal(0, 0.5, size=(n, d))
    single, sim = cls(n, e0, device=cuda_device), cls(n, e0, device=cuda_device)
    to = lambda x: torch.as_tensor(x).to(cuda_device)
    for _ in range(steps):
        i, j = one_gpu_batch(rs, n, B, centre_every=7)
        aux = ((rs.random_sample(B) < 0.5) if mode == 0 else rs.random_sample(B) * 3).astype(np.float32)
        single.step(i, j, aux)
        simulated_merge(sim, to(i), to(j), to(aux), world)
        sim.apply_adam()
        torch.cuda.synchronize()
        assert int((sim.row_slot != -1).sum()) == 0
    for name in ("emb", "bias_t", "m_emb", "v_emb"):
        assert close(getattr(sim, name).cpu().numpy(), getattr(single, name).cpu().numpy(), steps=steps), name
    assert sim.beta1_power == single.beta1_power and sim.step_count == single.step_count == steps


def test_world1_data_parallel_equals_single_gpu(cuda_device):
    """torch.distributed.run with one rank: DataParallelStep.step / .train_steps at B = 4096 and 65 536 against
    PairModel bit for bit, row_slot cleared, one collective per step (tests/dist_large_batch_worker.py, mode world1)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "1", "--master-addr", "127.0.0.1",
           "--master-port", "29653", os.path.join(ROOT, "tests", "dist_large_batch_worker.py"), "world1"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and "DP_WORLD1_OK" in r.stdout, r.stdout[-3000:]
