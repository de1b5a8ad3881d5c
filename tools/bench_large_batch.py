"""Large mini-batch benchmark of one optimizer step (K2 gradient + K3 dense Adam sweep) at the C3 shape.

usage: python tools/bench_large_batch.py [--out FILE.jsonl] [--n 1000000] [--n-emb 128] [--seconds 1.0] [--profile]

Workload: N = 1M nodes, n_emb = 128 (ld 128; --n-emb takes another row stride: 32, 64, 128, 256 or 512),
D-shaped rows -- the centres of synth.power_law(N, 20), each repeated
2 * deg times, with its adjacency twice as neighbours and labels 1 then 0 (~40 M rows, grouped by centre like the rows a
D pass emits).  For every B it times, with CUDA events over >= --seconds of work after a warm-up, on batches at random
slice starts (always including slice 0, which holds the largest hub):
  grad   gg_pair_grad_ex alone (the row_slot reset it needs is timed separately and subtracted)
  sweep  gg_adam_apply alone
  step   whole steps through gg_train_steps_ex
At B <= 1024 it also alternates gg_train_steps and gg_train_steps_ex (the same kernels) to show the spread.
--profile adds per-kernel times of the multi-CTA gradient at the largest B (torch.profiler, a run of its own).
Prints one JSON line per measurement (and the card's name, power limit and SM clock) and appends them to --out.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from graphgan_b200 import _cabi, synth                # noqa: E402
from graphgan_b200._cabi import ptr                   # noqa: E402
from graphgan_b200.discriminator import Discriminator  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, sm, sm_max = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def d_rows(n, seed=0):
    e = synth.power_law(n, 20, seed=seed)
    src = np.concatenate([e[:, 0], e[:, 1]]).astype(np.int64)
    dst = np.concatenate([e[:, 1], e[:, 0]]).astype(np.int32)
    order = np.argsort(src, kind="stable")
    src, dst = src[order], dst[order]
    deg = np.bincount(src, minlength=n)
    ptr_ = np.concatenate([[0], np.cumsum(deg)])
    # per centre c: [c] * 2deg | adj[c] + adj[c] | [1] * deg + [0] * deg
    centre = np.repeat(np.arange(n, dtype=np.int32), 2 * deg)
    rows_of = np.repeat(ptr_[:-1], 2 * deg)
    k = np.arange(centre.shape[0], dtype=np.int64) - np.repeat(2 * ptr_[:-1], 2 * deg)
    d_c = np.repeat(deg, 2 * deg)
    neigh = dst[rows_of + (k % d_c)]
    label = (k < d_c).astype(np.float32)
    return centre, neigh, label, int(deg.max())


def events_us(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def reps_for(fn, seconds):
    """Calls of fn that take about `seconds` (one calibration call after the warm-up)."""
    fn(); torch.cuda.synchronize()
    t0 = time.perf_counter(); fn(); torch.cuda.synchronize()
    return max(20, int(seconds / max(time.perf_counter() - t0, 1e-6)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--n-emb", type=int, default=128, choices=[32, 64, 128, 256, 512], help="embedding width (= the row stride)")
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--batches", default="64,1024,4096,16384,65536")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    lines = []

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(d) + "\n")

    dev = torch.device("cuda:0")
    info = card()
    emit(dict(info, kind="card"))
    n, d = args.n, args.n_emb
    centre, neigh, label, max_deg = d_rows(n)
    M = int(centre.shape[0])
    emit({"kind": "workload", "n": n, "n_emb": d, "rows": M, "max_degree": max_deg})
    ci, ni, li = (torch.as_tensor(x).to(dev) for x in (centre, neigh, label))
    m = Discriminator(n, torch.empty((n, d), device=dev).normal_(0, 0.1), device=dev)
    lib, st = m.lib, m._stream()
    rs = np.random.RandomState(1)
    f = lambda x: C.c_float(float(x))

    for B in (int(x) for x in args.batches.split(",")):
        scratch = m._large_batch_buffers(B)
        n_slices = M // B
        starts = (rs.randint(0, n_slices, 4096) * B).astype(np.int64)
        starts[0] = 0
        longest = 0
        for s0 in starts[:64]:
            ids = np.concatenate([centre[s0:s0 + B], neigh[s0:s0 + B]])
            longest = max(longest, int(np.bincount(ids).max()))
        pos = [0]

        def grad():
            s0 = int(starts[pos[0] % len(starts)]); pos[0] += 1
            _cabi.check(lib.gg_pair_grad_ex(0, B, 0, ptr(ci) + 4 * s0, ptr(ni) + 4 * s0, ptr(li) + 4 * s0, ptr(m.emb), ptr(m.bias_t), d,
                                            f(m.lam), ptr(m.n_unique), ptr(m.uniq_ids), ptr(m.grad_rows), ptr(m.grad_bias),
                                            ptr(m.row_slot), ptr(scratch), scratch.numel(), 0, st), "gg_pair_grad_ex")
            m.row_slot.fill_(-1)

        def reset():
            m.row_slot.fill_(-1)

        def sweep():
            _cabi.check(lib.gg_adam_apply(n, d, ptr(m.emb), ptr(m.m_emb), ptr(m.v_emb), ptr(m.bias_t), ptr(m.m_bias), ptr(m.v_bias),
                                          ptr(m.n_unique), ptr(m.uniq_ids), ptr(m.grad_rows), ptr(m.grad_bias), ptr(m.row_slot),
                                          f(1e-4), f(m.beta1), f(m.beta2), f(m.eps), st), "gg_adam_apply")

        def steps(fn_name, k):
            def run():
                b1, b2 = C.c_float(float(m.beta1_power)), C.c_float(float(m.beta2_power))
                sl = np.ascontiguousarray(starts[:k])
                common = (0, M, sl.ctypes.data_as(C.c_void_p), k, B, ptr(ci), ptr(ni), ptr(li), n, d, ptr(m.emb), ptr(m.m_emb),
                          ptr(m.v_emb), ptr(m.bias_t), ptr(m.m_bias), ptr(m.v_bias), f(m.lam), ptr(m.n_unique), ptr(m.uniq_ids),
                          ptr(m.grad_rows), ptr(m.grad_bias), ptr(m.row_slot), f(m.lr), f(m.beta1), f(m.beta2), f(m.eps),
                          C.byref(b1), C.byref(b2))
                if fn_name == "gg_train_steps":
                    _cabi.check(lib.gg_train_steps(*common, st), fn_name)
                else:
                    _cabi.check(lib.gg_train_steps_ex(*common, ptr(scratch), scratch.numel(), st), fn_name)
            return run

        g_reps = reps_for(grad, args.seconds)
        us_grad_reset = events_us(grad, g_reps)
        us_reset = events_us(reset, g_reps)
        s_reps = reps_for(sweep, args.seconds)
        us_sweep = events_us(sweep, s_reps)
        k = max(8, min(len(starts), int(args.seconds * 1e6 / (us_grad_reset + us_sweep))))
        step_ex = steps("gg_train_steps_ex", k)
        step_ex()
        us_step = events_us(step_ex, 1) / k
        rec = {"kind": "large_batch", "B": B, "us_grad": round(us_grad_reset - us_reset, 2), "us_sweep": round(us_sweep, 2),
               "us_step": round(us_step, 2), "pairs_per_s": round(B / us_step * 1e6), "longest_slot": longest,
               "grad_path": "one-CTA" if B <= 1024 else "multi-CTA", "reps_grad": g_reps, "reps_sweep": s_reps, "steps": k,
               "power_limit": info["power_limit"], "gpu": info["gpu"]}
        emit(rec)
        if B <= 1024:
            old = steps("gg_train_steps", k)
            old()
            ab = []
            for _ in range(3):
                ab.append(("gg_train_steps", round(events_us(old, 1) / k, 2)))
                ab.append(("gg_train_steps_ex", round(events_us(step_ex, 1) / k, 2)))
            emit({"kind": "small_batch_ab", "B": B, "steps": k, "us_step_alternating": ab, "power_limit": info["power_limit"]})

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        B = max(int(x) for x in args.batches.split(","))
        scratch = m._large_batch_buffers(B)
        for s0 in (0, B * 37):
            def g1():
                _cabi.check(lib.gg_pair_grad_ex(0, B, 0, ptr(ci) + 4 * s0, ptr(ni) + 4 * s0, ptr(li) + 4 * s0, ptr(m.emb), ptr(m.bias_t),
                                                d, f(m.lam), ptr(m.n_unique), ptr(m.uniq_ids), ptr(m.grad_rows), ptr(m.grad_bias),
                                                ptr(m.row_slot), ptr(scratch), scratch.numel(), 0, st), "gg_pair_grad_ex")
                m.row_slot.fill_(-1)
            g1(); torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(20):
                    g1()
                torch.cuda.synchronize()
            per = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" or getattr(e, "device_time_total", 0) > 0:
                    t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    name = e.key
                    for tag in ("mc_forward", "mc_count", "mc_number", "mc_keys", "mc_hist", "mc_scatter", "mc_terms",
                                "mc_short_sums", "mc_long_sums", "mc_long_bias", "exclusive_scan", "fill", "elementwise", "Memset"):
                        if tag in name:
                            name = tag
                            break
                    per[name] = per.get(name, 0.0) + t / 20.0
            ids = np.concatenate([centre[s0:s0 + B], neigh[s0:s0 + B]])
            emit({"kind": "grad_stage_profile", "B": B, "start": s0, "longest_slot": int(np.bincount(ids).max()),
                  "us_per_call": {k: round(v, 2) for k, v in sorted(per.items(), key=lambda kv: -kv[1])},
                  "power_limit": info["power_limit"]})


if __name__ == "__main__":
    main()
