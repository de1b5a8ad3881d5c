"""Throughput of the exact generator distribution G(v | root) (csrc/gdist.cu, DESIGN.md section 5.1) on the bench graph.

C3 = synth.power_law(1M, 20, seed 0), n_emb 128, hub threshold 128.  Roots: the top-degree node (13 828 neighbours), three
of its neighbours, the 12 highest-degree roots of the bench's root set (synth.pick_roots, 16 384 roots, seed 0) and 48
random roots of that set.  Per timed step: one WalkSampler.distribution call over all of them (hub scores + the
level-synchronous pass, roots in chunks of the scratch budget), between CUDA events.  Reports:
  - roots/s (median over steps) and ms per call;
  - candidate rows gathered per root (the call's rows_gathered counter: every on-demand score fetches one row, every
    list with >= 2 candidates its owner's row) and the bytes/s they make, (4 * ld + 8) bytes per row, against the
    H100's 3.35 TB/s data-sheet HBM bandwidth;
  - sum-to-one error and root_ok count of the last call;
  - card name, power limit and SM clock (nvidia-smi query, read only).
Writes one JSON object to measurements/h100/generator_dist.json (or --out).

    python tools/bench_generator_dist.py [--steps 10] [--warmup 2] [--scratch-gb 8] [--out PATH]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12    # H100 SXM5 80 GB data sheet


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=20).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smax}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        import torch
        return {"name": torch.cuda.get_device_name(0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--scratch-gb", type=float, default=8.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "measurements", "h100", "generator_dist.json"))
    args = ap.parse_args()
    import torch
    from graphgan_b200 import graph as G, sampler as S, synth
    from graphgan_b200.sampler import CNT
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
    dg = G.DeviceGraph(hg, dev)
    smp = S.WalkSampler(dg, hub_threshold=128)
    trees = smp.build_trees(roots)
    emb = S.pad_embedding(synth.embeddings(n, d, seed=1), dev)
    bias = torch.as_tensor(np.random.RandomState(5).normal(0, 0.1, n).astype(np.float32)).to(dev)
    ld = int(emb.shape[1])
    budget = int(args.scratch_gb * (1 << 30))
    counters = torch.zeros(16, dtype=torch.int64, device=dev)
    for _ in range(args.warmup):
        smp.distribution(emb, bias, trees, max_scratch_bytes=budget)
    torch.cuda.synchronize()
    ms, rows = [], []
    for _ in range(args.steps):
        counters.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dist, ok = smp.distribution(emb, bias, trees, max_scratch_bytes=budget, counters=counters)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
        rows.append(int(counters[CNT["rows_gathered"]].item()))
    R = len(roots)
    med = float(np.median(ms))
    rows_per_root = float(np.median(rows)) / R
    sums = dist.sum(1).cpu().numpy()
    okh = ok.cpu().numpy()
    bps = rows_per_root * R * (4 * ld + 8) / (med * 1e-3)
    line = {
        "workload": "generator distribution, power_law N=1M avg_deg=20 (C3), n_emb %d (ld %d), hub_threshold 128" % (d, ld),
        "roots": R, "tree_nodes_mean": float(np.mean([(trees.parent_arrays([k]).cpu().numpy() >= 0).sum() + 1
                                                      for k in range(R)])),
        "roots_per_s": R / (med * 1e-3), "ms_per_call_median": med, "ms_per_call_min": float(np.min(ms)),
        "ms_per_root": med / R, "rows_gathered_per_root": rows_per_root, "bytes_per_s": bps,
        "fraction_of_3_35_TBps": bps / HBM_BYTES_PER_S, "root_ok": int(okh.sum()),
        "max_sum_error": float(np.max(np.abs(sums[okh == 1] - 1.0))) if okh.any() else None,
        "scratch_budget_bytes": budget, "steps": args.steps, "warmup": args.warmup, "gpu": gpu_info(),
    }
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(line, indent=1) + "\n")
    print(json.dumps(line))


if __name__ == "__main__":
    main()
