"""Data-parallel steps above GG_MAX_BATCH pairs at the C3 shape: slices + multi-CTA merge against the redundant whole-batch
gradient, and the cost of the exchange path at world 1.

usage: python tools/bench_dp_large_batch.py [--out FILE.jsonl] [--n 1000000] [--seconds 1.0] [--batches 4096,16384,65536]
       torchrun --nproc-per-node W tools/bench_dp_large_batch.py ...      (adds the multi-GPU figures (d))

Workload: the D-shaped rows of tools/bench_large_batch.py (N = 1M, ld 128, ~40 M rows grouped by centre); batches at
random slice starts, always including slice 0 (the 13 828-neighbour hub).  With CUDA events over >= --seconds of work:
  (a) whole     gg_pair_grad_ex(B): the gradient every rank would compute if it skipped the exchange
  (b) slices    per W in {2, 4, 8}, on one GPU: gg_pair_grad_ex(B / W) on one rank's slice (every rank of the batch in
                turn) and gg_grad_merge_ex over W simulated blocks -- what one rank computes per step, without the all-gather
  (c) world 1   whole steps of gg_dp_train_steps_ex (slice = batch, all-gather of one block, merge, sweep) against
                gg_train_steps_ex, alternating; the difference is the exchange copy and the merge
  (d) torchrun  per-step time of gg_dp_train_steps_ex and of an all-gather of the same size, on W GPUs
The row_slot reset that a stand-alone gradient or merge needs is timed separately and subtracted.  Every line carries the
card's name, power limit and SM clock; lines are printed and appended to --out (rank 0 only).
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_large_batch import card, d_rows, events_us, reps_for   # noqa: E402
from graphgan_b200 import _cabi, parallel                         # noqa: E402
from graphgan_b200._cabi import ptr                               # noqa: E402
from graphgan_b200.discriminator import Discriminator             # noqa: E402
from tests.dist_large_batch_worker import gathered_blocks         # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--batches", default="4096,16384,65536")
    ap.add_argument("--worlds", default="2,4,8")
    args = ap.parse_args()

    import torch.distributed as dist
    under_run = "RANK" in os.environ
    for k, v in (("MASTER_ADDR", "127.0.0.1"), ("MASTER_PORT", "29671"), ("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0")):
        os.environ.setdefault(k, v)
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    info = card()

    def emit(d):
        if rank:
            return
        d = dict(d, gpu=info["gpu"], power_limit=info["power_limit"], sm_clock=info["sm_clock"])
        print(json.dumps(d), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(d) + "\n")

    n, d = args.n, 128
    centre, neigh, label, max_deg = d_rows(n)
    M = int(centre.shape[0])
    emit({"kind": "workload", "n": n, "n_emb": d, "rows": M, "max_degree": max_deg, "world": world,
          "launched_by_torchrun": under_run})
    ci, ni, li = (torch.as_tensor(x).to(dev) for x in (centre, neigh, label))
    m = Discriminator(n, torch.empty((n, d), device=dev).normal_(0, 0.1), device=dev)
    lib, st = m.lib, m._stream()
    rs = np.random.RandomState(1)
    f = lambda x: C.c_float(float(x))
    reset = lambda: m.row_slot.fill_(-1)

    def timed(fn, with_reset):
        reps = reps_for(fn, args.seconds)
        us = events_us(fn, reps)
        return (us - events_us(reset, reps) if with_reset else us), reps

    for B in (int(x) for x in args.batches.split(",")):
        starts = (rs.randint(0, M // B, 4096) * B).astype(np.int64)
        starts[0] = 0
        if world == 1:
            # ---- (a) the redundant whole-batch gradient
            scratch = m._large_batch_buffers(B)
            pos = [0]

            def whole():
                s0 = int(starts[pos[0] % 64]); pos[0] += 1
                _cabi.check(lib.gg_pair_grad_ex(0, B, 0, ptr(ci) + 4 * s0, ptr(ni) + 4 * s0, ptr(li) + 4 * s0, ptr(m.emb),
                                                ptr(m.bias_t), d, f(m.lam), ptr(m.n_unique), ptr(m.uniq_ids), ptr(m.grad_rows),
                                                ptr(m.grad_bias), ptr(m.row_slot), ptr(scratch), scratch.numel(), 0, st), "gg_pair_grad_ex")
                reset()
            us, reps = timed(whole, True)
            emit({"kind": "a_whole_batch_grad", "B": B, "us": round(us, 2), "reps": reps})
            # ---- (b) one rank's slice gradient + the merge of W blocks
            for W in (int(x) for x in args.worlds.split(",")):
                cap = 2 * (-(-B // W))
                nf = int(lib.gg_grad_buf_floats(cap, d))
                block = torch.zeros(nf, dtype=torch.float32, device=dev)
                nb = C.c_int64(0)
                _cabi.check(lib.gg_dp_scratch_bytes(W, B, d, C.byref(nb)), "gg_dp_scratch_bytes")
                dscratch = torch.empty(nb.value, dtype=torch.uint8, device=dev)
                at = lambda off: block.data_ptr() + 4 * off
                pos = [0]

                def slice_grad():
                    k = pos[0]; pos[0] += 1
                    s0, r = int(starts[(k // W) % 64]), k % W
                    lo, hi = parallel.block_range(B, r, W)
                    _cabi.check(lib.gg_pair_grad_ex(0, hi - lo, B, ptr(ci) + 4 * (s0 + lo), ptr(ni) + 4 * (s0 + lo),
                                                    ptr(li) + 4 * (s0 + lo), ptr(m.emb), ptr(m.bias_t), d, f(m.lam),
                                                    at(cap * d + 2 * cap), at(cap * d + cap), at(0), at(cap * d), ptr(m.row_slot),
                                                    ptr(dscratch), dscratch.numel(), 0, st), "gg_pair_grad_ex")
                    reset()
                us_slice, reps_slice = timed(slice_grad, True)
                blocks = []
                for s0 in starts[:4]:
                    s0 = int(s0)
                    g, _ = gathered_blocks(lib, 0, ci[s0:s0 + B], ni[s0:s0 + B], li[s0:s0 + B], m.emb, m.bias_t, d, m.lam, W, m.row_slot)
                    blocks.append(g)
                reset()
                pos = [0]

                def merge():
                    g = blocks[pos[0] % len(blocks)]; pos[0] += 1
                    _cabi.check(lib.gg_grad_merge_ex(W, cap, d, g.data_ptr(), ptr(m.n_unique), ptr(m.uniq_ids), ptr(m.grad_rows),
                                                     ptr(m.grad_bias), ptr(m.row_slot), ptr(dscratch), dscratch.numel(), 1, st),
                                "gg_grad_merge_ex")
                    reset()
                us_merge, reps_merge = timed(merge, True)
                emit({"kind": "b_slice_grad_plus_merge", "B": B, "W": W, "us_slice_grad": round(us_slice, 2),
                      "us_merge": round(us_merge, 2), "us_per_rank": round(us_slice + us_merge, 2),
                      "allgather_bytes_per_rank": 4 * W * nf, "reps_slice": reps_slice, "reps_merge": reps_merge})
                del blocks
        # ---- (c) world-1 steps / (d) W-GPU steps: gg_dp_train_steps_ex
        dp = parallel.DataParallelStep(m)
        cap = 2 * (-(-B // world))
        local, gathered = dp._buffers(cap)
        scratch = dp._large_batch_scratch(B)
        dp._select()

        def steps(name, k):
            sl = np.ascontiguousarray(starts[:k])

            def run():
                b1, b2 = C.c_float(float(m.beta1_power)), C.c_float(float(m.beta2_power))
                common = (0, M, sl.ctypes.data_as(C.c_void_p), k, B, ptr(ci), ptr(ni), ptr(li), n, d, ptr(m.emb), ptr(m.m_emb),
                          ptr(m.v_emb), ptr(m.bias_t), ptr(m.m_bias), ptr(m.v_bias), f(m.lam))
                tail = (ptr(m.n_unique), ptr(m.uniq_ids), ptr(m.grad_rows), ptr(m.grad_bias), ptr(m.row_slot), f(m.lr), f(m.beta1),
                        f(m.beta2), f(m.eps), C.byref(b1), C.byref(b2), ptr(scratch), scratch.numel())
                if name == "gg_train_steps_ex":
                    _cabi.check(lib.gg_train_steps_ex(*common, *tail, st), name)
                else:
                    _cabi.check(lib.gg_dp_train_steps_ex(dp.comm, *common, ptr(local), ptr(gathered), cap, *tail, 0, st), name)
            return run

        probe = steps("gg_dp_train_steps_ex", 4)
        probe()
        torch.cuda.synchronize()
        k = max(8, min(len(starts), int(args.seconds * 1e6 / (events_us(probe, 1) / 4))))
        dp_run = steps("gg_dp_train_steps_ex", k)
        if world == 1:
            one = steps("gg_train_steps_ex", k)
            one()
            ab = []
            for _ in range(3):
                ab.append(("gg_train_steps_ex", round(events_us(one, 1) / k, 2)))
                ab.append(("gg_dp_train_steps_ex", round(events_us(dp_run, 1) / k, 2)))
            emit({"kind": "c_world1_step", "B": B, "steps": k, "us_step_alternating": ab})
        else:
            dist.barrier()
            us_step = events_us(dp_run, 1) / k
            buf = torch.zeros(int(lib.gg_grad_buf_floats(cap, d)), dtype=torch.float32, device=dev)
            out = torch.empty(world * buf.numel(), dtype=torch.float32, device=dev)
            dist.barrier()
            us_ag = events_us(lambda: dist.all_gather_into_tensor(out, buf), k)
            emit({"kind": "d_multi_gpu_step", "B": B, "world": world, "steps": k, "us_step": round(us_step, 2),
                  "us_allgather": round(us_ag, 2), "allgather_share": round(us_ag / us_step, 3),
                  "allgather_bytes_per_rank": 4 * world * buf.numel()})
    if world == 1:
        emit({"kind": "d_multi_gpu_step", "status": "not measured: one GPU (run under torchrun on a box with several GPUs)"})
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
