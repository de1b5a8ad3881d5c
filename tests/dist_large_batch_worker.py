"""Worker for the data-parallel tests above GG_MAX_BATCH pairs (launched through torch.distributed.run by
tests/test_dp_large_batch_gpu.py and tests/test_dist_large_batch.py), plus the one-GPU simulation of a world-W step that
both the worker and the single-GPU tests use.

  mode "world1": one rank.  DataParallelStep.step / .train_steps at B = 4096 and 65 536 equal PairModel.step /
                 .train_steps bit for bit (with one rank the merge adds every row to +0, which changes no bits).
  mode "multi":  one rank per GPU (world = min(GPUs, 4)).  Replicas stay bit-identical, the merged gradient equals the
                 one-GPU simulation of the same world bit for bit, train_steps equals the step loop, GraphGAN.train()
                 runs with batch 4096, and the peer-memory transport still refuses batches above 1024 pairs.
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STATE = ("emb", "bias_t", "m_emb", "v_emb", "m_bias", "v_bias")


def gathered_blocks(lib, mode, i, j, a, emb, bias, ld, lam, world, row_slot, empty_ranks=()):
    """The all-gathered buffer of a world-`world` step, built on one device: rank r's block is gg_pair_grad_ex on its
    block_range slice with batch_total = B (row_slot reset between slices; left as the last rank's slice leaves it).
    Ranks in `empty_ranks` get n_unique = 0, as a rank without rows sends.  Returns (gathered, cap)."""
    import torch
    from graphgan_b200 import _cabi
    from graphgan_b200.parallel import block_range
    B = int(i.shape[0])
    cap = 2 * (-(-B // world))
    nf = int(lib.gg_grad_buf_floats(cap, ld))
    gathered = torch.zeros(world * nf, dtype=torch.float32, device=emb.device)
    n = C.c_int64(0)
    _cabi.check(lib.gg_pair_grad_scratch_bytes(max(-(-B // world), 1), ld, C.byref(n)), "gg_pair_grad_scratch_bytes")
    scratch = torch.empty(n.value, dtype=torch.uint8, device=emb.device)
    at = lambda r, off: gathered.data_ptr() + 4 * (r * nf + off)
    for r in range(world):
        lo, hi = block_range(B, r, world)
        row_slot.fill_(-1)
        if hi == lo or r in empty_ranks:
            continue
        _cabi.check(lib.gg_pair_grad_ex(mode, hi - lo, B, i.data_ptr() + 4 * lo, j.data_ptr() + 4 * lo, a.data_ptr() + 4 * lo,
                                        emb.data_ptr(), bias.data_ptr(), ld, C.c_float(float(lam)), at(r, cap * ld + 2 * cap),
                                        at(r, cap * ld + cap), at(r, 0), at(r, cap * ld), row_slot.data_ptr(), scratch.data_ptr(),
                                        n.value, 0, None), "gg_pair_grad_ex")
    torch.cuda.synchronize()
    return gathered, cap


def merge_ex(lib, world, cap, ld, gathered, n_unique, uniq_ids, grad_rows, grad_bias, row_slot, flags=0):
    import torch
    from graphgan_b200 import _cabi
    n = C.c_int64(0)
    _cabi.check(lib.gg_grad_merge_scratch_bytes(world, cap, ld, C.byref(n)), "gg_grad_merge_scratch_bytes")
    scratch = torch.empty(n.value, dtype=torch.uint8, device=gathered.device)
    _cabi.check(lib.gg_grad_merge_ex(world, cap, ld, gathered.data_ptr(), n_unique.data_ptr(), uniq_ids.data_ptr(),
                                     grad_rows.data_ptr(), grad_bias.data_ptr(), row_slot.data_ptr(), scratch.data_ptr(), n.value,
                                     flags, None), "gg_grad_merge_ex")
    torch.cuda.synchronize()


def simulated_merge(model, i, j, a, world):
    """Slices -> gathered blocks -> gg_grad_merge_ex into the model's gradient buffers (grown to 2B entries), as the step
    of a world-`world` run computes it on every rank.  The model's parameters are not changed."""
    B = int(i.shape[0])
    model._large_batch_buffers(B)
    gathered, cap = gathered_blocks(model.lib, model._step_mode, i, j, a, model.emb, model.bias_t, model.ld, model.lam, world,
                                    model.row_slot)
    merge_ex(model.lib, world, cap, model.ld, gathered, model.n_unique, model.uniq_ids, model.grad_rows, model.grad_bias,
             model.row_slot)


def batch(rs, n, B, mode):
    """Random pairs with one centre repeated through the batch (present in every slice) and a long run of one row."""
    i, j = rs.randint(0, n, B).astype(np.int32), rs.randint(0, n, B).astype(np.int32)
    i[::3] = n // 2
    i[1:B // 4:2] = 7
    aux = ((rs.random_sample(B) < 0.5) if mode == 0 else rs.random_sample(B) * 3).astype(np.float32)
    return i, j, aux


def _world1(dev):
    import torch
    from graphgan_b200 import parallel
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.generator import Generator
    rs = np.random.RandomState(21)
    n, d = 20000, 100
    e0 = rs.normal(0, 0.5, size=(n, d))
    for cls, mode in ((Discriminator, 0), (Generator, 1)):
        for B in (4096, 65536):
            single, repl = cls(n, e0, device=dev), cls(n, e0, device=dev)
            dp = parallel.DataParallelStep(repl)
            for step in range(3):
                i, j, aux = batch(rs, n, B, mode)
                before = dp.stats()["collectives_issued"]
                single.step(i, j, aux)
                dp.step(i, j, aux)
                torch.cuda.synchronize()
                assert dp.stats()["collectives_issued"] == before + 1, (cls.__name__, B, step)
                for name in STATE:
                    assert torch.equal(getattr(single, name), getattr(repl, name)), (cls.__name__, B, step, name)
                assert single.beta1_power == repl.beta1_power and single.beta2_power == repl.beta2_power
                assert int((repl.row_slot != -1).sum()) == 0
            # the C loop: shuffled starts and a short last batch (1000 pairs: the one-CTA step)
            M = 3 * B + 1000
            ii, jj, ax = batch(rs, n, M, mode)
            starts = list(range(0, M, B))
            rs.shuffle(starts)
            sa, ra = cls(n, e0, device=dev), cls(n, e0, device=dev)
            da = parallel.DataParallelStep(ra)
            before = da.stats()["collectives_issued"]
            sa.train_steps(ii, jj, ax, starts, B)
            da.train_steps(ii, jj, ax, starts, B)
            torch.cuda.synchronize()
            for name in STATE:
                assert torch.equal(getattr(sa, name), getattr(ra, name)), (cls.__name__, B, "train_steps", name)
            assert sa.beta1_power == ra.beta1_power and sa.beta2_power == ra.beta2_power and sa.step_count == ra.step_count
            assert da.stats()["collectives_issued"] - before == len(starts)
            assert int((ra.row_slot != -1).sum()) == 0
    print("DP_WORLD1_OK")


def _multi(dev, rank, world):
    import torch
    import torch.distributed as dist
    from graphgan_b200 import parallel
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.generator import Generator
    rs = np.random.RandomState(31)          # same seed on every rank: every rank holds the same batches
    n, d = 20000, 128
    e0 = rs.normal(0, 0.5, size=(n, d))
    for cls, mode in ((Discriminator, 0), (Generator, 1)):
        for B in (1025, 4096, 65536):
            repl = cls(n, e0, device=dev)
            dp = parallel.DataParallelStep(repl)
            for step in range(2):
                i, j, aux = batch(rs, n, B, mode)
                if rank == 0:          # the one-GPU simulation of this world, on the same parameters
                    sim = cls(n, e0, device=dev)
                    sim.load_state_dict(repl.state_dict())
                    to = lambda x: torch.as_tensor(x).to(dev)
                    simulated_merge(sim, to(i), to(j), to(aux), world)
                dp.step(i, j, aux)
                torch.cuda.synchronize()
                if rank == 0:
                    U = int(sim.n_unique.item())
                    assert int(repl.n_unique.item()) == U, (cls.__name__, B, step)
                    assert torch.equal(repl.uniq_ids[:U], sim.uniq_ids[:U])
                    assert torch.equal(repl.grad_rows[:U].view(torch.int32), sim.grad_rows[:U].view(torch.int32))
                    assert torch.equal(repl.grad_bias[:U].view(torch.int32), sim.grad_bias[:U].view(torch.int32))
                assert int((repl.row_slot != -1).sum()) == 0
            for name in STATE:
                rows = [torch.empty_like(getattr(repl, name)) for _ in range(world)]
                dist.all_gather(rows, getattr(repl, name))
                assert all(torch.equal(rows[0], r) for r in rows[1:]), (cls.__name__, B, name)
            # the C loop == the step loop
            M = 2 * B + 777
            ii, jj, ax = batch(rs, n, M, mode)
            starts = list(range(0, M, B))
            rs.shuffle(starts)
            ra, rb = cls(n, e0, device=dev), cls(n, e0, device=dev)
            da, db = parallel.DataParallelStep(ra), parallel.DataParallelStep(rb)
            for s0 in starts:
                da.step(ii[s0:s0 + B], jj[s0:s0 + B], ax[s0:s0 + B])
            db.train_steps(ii, jj, ax, starts, B)
            torch.cuda.synchronize()
            for name in STATE:
                assert torch.equal(getattr(ra, name), getattr(rb, name)), (cls.__name__, B, "train_steps", name)
            assert ra.beta1_power == rb.beta1_power and ra.step_count == rb.step_count
    # the peer-memory transport keeps its 1024-pair limit
    pm = Discriminator(n, e0, device=dev)
    dpp = parallel.DataParallelStep(pm, transport="p2p")
    i, j, aux = batch(rs, n, 1025, 0)
    for call in (lambda: dpp.step(i, j, aux), lambda: dpp.train_steps(i, j, aux, [0], 1025)):
        try:
            call()
        except ValueError as e:
            assert "GG_MAX_BATCH" in str(e)
        else:
            raise AssertionError("p2p accepted a batch above GG_MAX_BATCH")
    assert pm.step_count == 0
    dpp.use("nccl")
    # the trainer under torch.distributed with batches above GG_MAX_BATCH
    import tempfile
    from graphgan_b200 import config, graph as G
    from graphgan_b200.graph_gan import GraphGAN
    from tests.golden import loader
    c = loader.load("rand1200")
    tmp = tempfile.mkdtemp()
    config.n_emb, config.n_epochs, config.n_epochs_dis, config.dis_interval = int(c.emb_g.shape[1]), 1, 1, 1
    config.n_epochs_gen, config.gen_interval, config.n_sample_gen, config.seed = 1, 1, 2, 9
    config.app, config.batch_size_dis, config.batch_size_gen = "none", 4096, 4096
    config.emb_filenames = [os.path.join(tmp, "g.emb"), os.path.join(tmp, "d.emb")]
    config.result_filename, config.model_log = os.path.join(tmp, "r.txt"), tmp + "/"
    gan = GraphGAN(host_graph=G.HostGraph(c.train_edges, c.test_edges), node_embed_init_d=c.emb_d, node_embed_init_g=c.emb_g)
    assert gan.world == world
    gan.train()
    torch.cuda.synchronize()
    assert gan.discriminator.step_count > 0 and gan.generator.step_count > 0
    for m in (gan.generator, gan.discriminator):
        for name in STATE:
            rows = [torch.empty_like(getattr(m, name)) for _ in range(world)]
            dist.all_gather(rows, getattr(m, name))
            assert all(torch.equal(rows[0], r) for r in rows[1:]), ("train", name)
    dist.barrier()
    if rank == 0:
        print("DP_MULTI_OK")


def main(mode):
    import torch
    import torch.distributed as dist
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    try:
        if mode == "world1":
            assert world == 1
            _world1(dev)
        else:
            _multi(dev, rank, world)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1])
