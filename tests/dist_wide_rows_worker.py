"""Worker of tests/test_wide_rows_gpu.py::test_world1_data_parallel_at_ld_512 (launched through torch.distributed.run
with one rank): at n_emb = 300 (ld 512), DataParallelStep.step / .train_steps equal PairModel.step / .train_steps bit for
bit, with the NCCL transport at B = 512 (one-CTA slice gradient and merge) and B = 4096 (multi-CTA), and with the
peer-memory transport at B = 256 (the gradient kernel pushes into the exchange buffer, the merge kernel waits on flags).
With one rank the merge adds every row to +0, which changes no values.  Prints DP_WIDE_WORLD1_OK."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.dist_large_batch_worker import STATE, batch   # noqa: E402


def _world1(dev):
    import torch
    from graphgan_b200 import parallel
    from graphgan_b200.discriminator import Discriminator
    from graphgan_b200.generator import Generator
    rs = np.random.RandomState(31)
    n, d = 6000, 300
    e0 = rs.normal(0, 0.5, size=(n, d))
    for cls, mode in ((Discriminator, 0), (Generator, 1)):
        for transport, B in (("nccl", 512), ("nccl", 4096), ("p2p", 256)):   # (the p2p exchange buffer holds 256-pair batches)
            single, repl = cls(n, e0, device=dev), cls(n, e0, device=dev)
            assert single.ld == 512
            dp = parallel.DataParallelStep(repl, transport=transport)
            for step in range(3):
                i, j, aux = batch(rs, n, B, mode)
                single.step(i, j, aux)
                dp.step(i, j, aux)
                torch.cuda.synchronize()
                for name in STATE:
                    assert torch.equal(getattr(single, name), getattr(repl, name)), (cls.__name__, transport, B, step, name)
                assert single.beta1_power == repl.beta1_power and single.beta2_power == repl.beta2_power
                assert int((repl.row_slot != -1).sum()) == 0
            M = 3 * B + 100
            ii, jj, ax = batch(rs, n, M, mode)
            starts = list(range(0, M, B))
            rs.shuffle(starts)
            sa, ra = cls(n, e0, device=dev), cls(n, e0, device=dev)
            da = parallel.DataParallelStep(ra, transport=transport)
            sa.train_steps(ii, jj, ax, starts, B, persistent=False)
            da.train_steps(ii, jj, ax, starts, B)
            torch.cuda.synchronize()
            for name in STATE:
                assert torch.equal(getattr(sa, name), getattr(ra, name)), (cls.__name__, transport, B, "train_steps", name)
            assert sa.step_count == ra.step_count == len(starts)
            assert int((ra.row_slot != -1).sum()) == 0
    print("DP_WIDE_WORLD1_OK")


def main():
    import torch
    import torch.distributed as dist
    assert int(os.environ["WORLD_SIZE"]) == 1
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    dist.init_process_group("nccl", device_id=dev)
    try:
        _world1(dev)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
