"""Cost of the exact generator gradient of the game value (csrc/value_grad.cu, DESIGN.md section 5.3) on the bench graph.

C3 = synth.power_law(1M, 20, seed 0), n_emb 128, hub threshold 128; the 64 roots of tools/bench_generator_dist.py (the
top-degree node, three of its neighbours, the 12 highest-degree bench roots and 48 random bench roots), in one chunk
(scratch budget 16 GiB).  Per timed step, each between its own CUDA events: the tree build, WalkSampler.distribution,
gg_game_value on its rows (the section 5.2 figures of the same run) and WalkSampler.game_value_grad.  One further step
runs under torch.profiler, which splits game_value_grad into its kernels:
  - gdist_rec   the recording section 5.1 kernel (dist + pi_in, pi_stop, father, every level's items);
  - value       gg_game_value on that dist (value_kernel + value_reduce_kernel);
  - h           value_h_kernel (h = dist * bce);
  - tsum        the bottom-up pass (T, then w_in / w_stop);
  - gather      big_nodes_kernel + gather_kernel (the rows of the gradient);
  - memset      the scratch clears.
Bytes per stage are what the algorithm has to move, from shapes (R roots, N nodes, nnz walk entries, ld floats per row):
  gdist_rec  the section 5.1 rows it gathers (counter) * 4 ld + R N (16 + 8 + 8 + 8 + 4) written;
  value      N (4 ld + 4) + 8 R N;   h  N (4 ld + 4) + 16 R N;
  tsum       R (nnz / 8 + 4 nnz) tree bits and entries, twice, + R N (8 T + 8 h + 16 w + 4 father) read + 24 R N written;
  gather     per root 2 (N - 1) rows of 4 ld bytes (child and father rows) + R nnz (4 + 4 father) + 2 N (8 ld + 8) once.
Also checks that the outputs are identical over the steps and that pos / neg / ok equal gg_game_value's.  Card name,
power limit and SM clock come from a read-only nvidia-smi query.  Writes one JSON object to
measurements/h100/value_grad.json (or --out).

    python tools/bench_value_grad.py [--steps 5] [--warmup 1] [--scratch-gb 16] [--out PATH]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_BYTES_PER_S = 3.35e12    # H100 SXM5 80 GB data sheet
STAGES = (("gdist_rec", ("gdist_rec_kernel",)), ("value", ("value_kernel", "value_reduce_kernel")),
          ("h", ("value_h_kernel",)), ("tsum", ("tsum_kernel",)), ("gather", ("big_nodes_kernel", "gather_kernel")),
          ("memset", ("Memset", "memset")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--scratch-gb", type=float, default=16.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "measurements", "h100", "value_grad.json"))
    args = ap.parse_args()
    import torch
    from bench_generator_dist import gpu_info
    from graphgan_b200 import graph as G, sampler as S, synth
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    dev = torch.device("cuda:0")
    n, d = 1_000_000, 128
    hg = G.HostGraph(synth.power_law(n, 20, seed=0), None, n_node=n)
    deg = hg.degrees()
    top = int(np.argmax(np.diff(hg.indptr)))
    nb = hg.adj[hg.indptr[top]:hg.indptr[top + 1]]
    bench_roots = synth.pick_roots(deg, 16384, seed=0)
    hubs = bench_roots[np.argsort(-deg[bench_roots], kind="stable")[:12]]
    rand = np.random.RandomState(1).choice(bench_roots, 48, replace=False)
    roots = np.unique(np.concatenate([[top], nb[[0, len(nb) // 2, len(nb) - 1]], hubs, rand])).astype(np.int32)
    R, nnz = len(roots), int(len(hg.adj))
    dg = G.DeviceGraph(hg, dev)
    smp = S.WalkSampler(dg, hub_threshold=128)
    g_emb = S.pad_embedding(synth.embeddings(n, d, seed=1), dev)
    g_bias = torch.as_tensor(np.random.RandomState(5).normal(0, 0.1, n).astype(np.float32)).to(dev)
    d_emb = S.pad_embedding(synth.embeddings(n, d, seed=2, sigma=0.2), dev)
    d_bias = torch.as_tensor(np.random.RandomState(6).normal(0, 0.5, n).astype(np.float32)).to(dev)
    ld = int(g_emb.shape[1])
    budget = int(args.scratch_gb * (1 << 30))
    counters = torch.zeros(16, dtype=torch.int64, device=dev)

    ev = lambda: torch.cuda.Event(enable_timing=True)
    t = {k: [] for k in ("tree_build", "distribution", "value", "value_grad")}
    outs = []
    trees = None
    for step in range(args.warmup + args.steps):
        e = [ev() for _ in range(5)]
        e[0].record()
        trees = smp.build_trees(roots)
        e[1].record()
        counters.zero_()
        dist, root_ok = smp.distribution(g_emb, g_bias, trees, max_scratch_bytes=budget, counters=counters)
        e[2].record()
        val = smp.game_value(g_emb, g_bias, d_emb, d_bias, trees, max_scratch_bytes=budget)
        e[3].record()
        out = smp.game_value_grad(g_emb, g_bias, d_emb, d_bias, trees, max_scratch_bytes=budget)
        e[4].record()
        torch.cuda.synchronize()
        if step >= args.warmup:
            for i, k in enumerate(t):
                t[k].append(e[i].elapsed_time(e[i + 1]))
            outs.append([x.cpu().numpy().tobytes() for x in out])
    # game_value includes its own distribution: the value kernel alone is the difference
    same = all(o == outs[0] for o in outs) and outs[0][:3] == [x.cpu().numpy().tobytes() for x in val]
    rows_gathered = int(counters[8].item())
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        smp.game_value_grad(g_emb, g_bias, d_emb, d_bias, trees, max_scratch_bytes=budget)
        torch.cuda.synchronize()
    stage_ms = {k: 0.0 for k, _ in STAGES}
    for evt in prof.key_averages():
        for k, names in STAGES:
            if any(s in evt.key for s in names) and not (k == "value" and "value_h_kernel" in evt.key):
                stage_ms[k] += evt.device_time_total / 1e3     # microseconds -> ms
                break
    bytes_ = {
        "gdist_rec": rows_gathered * 4 * ld + R * n * 44,
        "value": n * (4 * ld + 4) + 8 * R * n,
        "h": n * (4 * ld + 4) + 16 * R * n,
        "tsum": 2 * R * (nnz // 8 + 4 * nnz) + R * n * 44 + 24 * R * n,
        "gather": 2 * R * (n - 1) * 4 * ld + R * nnz * 8 + 2 * n * (8 * ld + 8),
        "memset": R * n * (8 + 8 + 8 + 4),
    }
    med = lambda xs: float(np.median(xs))
    okh = np.frombuffer(outs[0][2], np.int32)
    line = {
        "workload": "generator gradient of the game value, power_law N=1M avg_deg=20 (C3), n_emb %d (ld %d), hub_threshold "
                    "128, %d roots in one chunk" % (d, ld, R),
        "roots": R, "root_ok": int(okh.sum()),
        "ms_per_root": {"tree_build": med(t["tree_build"]) / R, "distribution": med(t["distribution"]) / R,
                        "value_kernel": (med(t["value"]) - med(t["distribution"])) / R,
                        "game_value_grad": med(t["value_grad"]) / R},
        "ms_per_call_median": {k: med(v) for k, v in t.items()},
        "game_value_grad_over_distribution": med(t["value_grad"]) / med(t["distribution"]),
        "profiled_stage_ms_per_root": {k: v / R for k, v in stage_ms.items()},
        "profiled_stage_bytes": bytes_,
        "profiled_stage_bytes_per_s": {k: (bytes_[k] / (stage_ms[k] * 1e-3) if stage_ms[k] > 0 else None) for k in bytes_},
        "profiled_stage_fraction_of_hbm_bound": {k: (bytes_[k] / HBM_BYTES_PER_S / (stage_ms[k] * 1e-3) if stage_ms[k] > 0
                                                     else None) for k in bytes_},
        "distribution_rows_gathered": rows_gathered,
        "grad_norm": float(np.sqrt((np.frombuffer(outs[0][3], np.float64) ** 2).sum()
                                   + (np.frombuffer(outs[0][4], np.float64) ** 2).sum())),
        "identical_over_steps_and_value_bits_equal_game_value": bool(same),
        "scratch_budget_bytes": budget, "steps": args.steps, "warmup": args.warmup, "gpu": gpu_info(),
    }
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(line, indent=1) + "\n")
    print(json.dumps(line))


if __name__ == "__main__":
    main()
