"""Cost of the exact discriminator gradient of the game value (csrc/value_dgrad.cu, DESIGN.md section 5.4) on the bench
graph.

C3 = synth.power_law(1M, 20, seed 0), n_emb 128, hub threshold 128; the 64 roots of tools/bench_generator_dist.py (the
top-degree node, three of its neighbours, the 12 highest-degree bench roots and 48 random bench roots), in one chunk
(scratch budget 16 GiB).  Per timed step, each between its own CUDA events: the tree build, WalkSampler.distribution,
WalkSampler.game_value (distribution + the value kernel) and WalkSampler.game_value_grad_d (distribution + the value
kernel + the gradient passes).  One further step runs under torch.profiler, which splits game_value_grad_d into kernels:
  - law      gdist_kernel (the section 5.1 law);
  - value    value_kernel + value_reduce_kernel;
  - mult     the multiplicity plane: its memset + mult_kernel;
  - W        value_w_kernel;
  - centre   cen_kernel + cen_reduce_kernel (C_k);
  - node     node_kernel (the rows).
Bytes and fp64 FMAs per pass are what the algorithm has to move and compute, from shapes (R roots, N nodes, ld floats per
row, the roots' raw degrees D, root tiles of 64 roots in the W pass and 32 in the centre pass at ld 128):
  mult    4 R N cleared + 12 D (entry read, count read and written);
  W       N (4 ld + 4) (rows and biases, once per 64-root tile) + R N (8 dist + 4 count + 8 W written); fp64: none counted
          (R N ld fp32 FMAs for the scores, one exp and one reciprocal per pair);
  centre  8 R N (W) + 4 N ld per 32-root tile + 8 R ld (N / 2048) partials written and read; R N ld fp64 FMAs;
  node    8 R N (W) + 2 N (8 ld + 8) (the accumulator rows read and written); R N ld fp64 FMAs.
Bounds: 3.35 TB/s of HBM3 and 34 TFLOP/s of FP64 (17 T FMA/s) on CUDA cores, the data sheet of an H100 SXM at 700 W.
Also checks that the outputs are identical over the steps and that pos / neg / ok equal game_value's.  Card name, power
limit and SM clock come from a read-only nvidia-smi query.  Writes one JSON object to
measurements/h100/value_grad_d.json (or --out).

    python tools/bench_value_grad_d.py [--steps 10] [--warmup 2] [--scratch-gb 16] [--out PATH]
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
FP64_FMA_PER_S = 17e12       # 34 TFLOP/s FP64 on CUDA cores, same data sheet
STAGES = (("law", ("gdist_kernel",)), ("value", ("value_kernel", "value_reduce_kernel")), ("mult", ("mult_kernel",)),
          ("W", ("value_w_kernel",)), ("centre", ("cen_kernel", "cen_reduce_kernel")), ("node", ("node_kernel",)),
          ("memset", ("Memset", "memset")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--scratch-gb", type=float, default=16.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "measurements", "h100", "value_grad_d.json"))
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
    R, D = len(roots), int(deg[roots].sum())
    dg = G.DeviceGraph(hg, dev)
    smp = S.WalkSampler(dg, hub_threshold=128)
    g_emb = S.pad_embedding(synth.embeddings(n, d, seed=1), dev)
    g_bias = torch.as_tensor(np.random.RandomState(5).normal(0, 0.1, n).astype(np.float32)).to(dev)
    d_emb = S.pad_embedding(synth.embeddings(n, d, seed=2, sigma=0.2), dev)
    d_bias = torch.as_tensor(np.random.RandomState(6).normal(0, 0.5, n).astype(np.float32)).to(dev)
    ld = int(d_emb.shape[1])
    budget = int(args.scratch_gb * (1 << 30))

    ev = lambda: torch.cuda.Event(enable_timing=True)
    t = {k: [] for k in ("tree_build", "distribution", "game_value", "game_value_grad_d")}
    outs = []
    trees = val = None
    for step in range(args.warmup + args.steps):
        e = [ev() for _ in range(5)]
        e[0].record()
        trees = smp.build_trees(roots)
        e[1].record()
        smp.distribution(g_emb, g_bias, trees, max_scratch_bytes=budget)
        e[2].record()
        val = smp.game_value(g_emb, g_bias, d_emb, d_bias, trees, max_scratch_bytes=budget)
        e[3].record()
        out = smp.game_value_grad_d(g_emb, g_bias, d_emb, d_bias, trees, max_scratch_bytes=budget)
        e[4].record()
        torch.cuda.synchronize()
        if step >= args.warmup:
            for i, k in enumerate(t):
                t[k].append(e[i].elapsed_time(e[i + 1]))
            outs.append([x.cpu().numpy().tobytes() for x in out])
    same = all(o == outs[0] for o in outs) and outs[0][:3] == [x.cpu().numpy().tobytes() for x in val]
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        smp.game_value_grad_d(g_emb, g_bias, d_emb, d_bias, trees, max_scratch_bytes=budget)
        torch.cuda.synchronize()
    stage_ms = {k: 0.0 for k, _ in STAGES}
    for evt in prof.key_averages():
        for k, names in STAGES:
            if any(s in evt.key for s in names) and not (k == "value" and "value_w_kernel" in evt.key):
                stage_ms[k] += evt.device_time_total / 1e3     # microseconds -> ms
                break
    stage_ms["mult"] += stage_ms.pop("memset")                 # the multiplicity plane's clear is the call's only memset
    n_ct = (n + 2047) // 2048
    bytes_ = {
        "mult": 4 * R * n + 12 * D,
        "W": n * (4 * ld + 4) * ((R + 63) // 64) + 20 * R * n,
        "centre": 8 * R * n + 4 * n * ld * ((R + 31) // 32) + 2 * 8 * R * ld * n_ct,
        "node": 8 * R * n + 2 * n * (8 * ld + 8),
    }
    fma64 = {"mult": 0, "W": 0, "centre": R * n * ld, "node": R * n * ld}
    med = lambda xs: float(np.median(xs))
    okh = np.frombuffer(outs[0][2], np.int32)
    sec = lambda k: stage_ms[k] * 1e-3
    bound = {k: max(bytes_[k] / HBM_BYTES_PER_S, fma64[k] / FP64_FMA_PER_S) for k in bytes_}
    line = {
        "workload": "discriminator gradient of the game value, power_law N=1M avg_deg=20 (C3), n_emb %d (ld %d), "
                    "hub_threshold 128, %d roots in one chunk" % (d, ld, R),
        "roots": R, "root_ok": int(okh.sum()), "raw_degree_sum": D,
        "ms_per_root": {"tree_build": med(t["tree_build"]) / R, "distribution": med(t["distribution"]) / R,
                        "value_kernel": (med(t["game_value"]) - med(t["distribution"])) / R,
                        "gradient_passes": (med(t["game_value_grad_d"]) - med(t["game_value"])) / R,
                        "game_value_grad_d": med(t["game_value_grad_d"]) / R},
        "ms_per_call_median": {k: med(v) for k, v in t.items()},
        "gradient_passes_over_distribution": (med(t["game_value_grad_d"]) - med(t["game_value"])) / med(t["distribution"]),
        "profiled_stage_ms_per_root": {k: v / R for k, v in stage_ms.items()},
        "profiled_stage_bytes": bytes_,
        "profiled_stage_fp64_fma": fma64,
        "profiled_stage_bytes_per_s": {k: (bytes_[k] / sec(k) if stage_ms[k] > 0 else None) for k in bytes_},
        "profiled_stage_fp64_fma_per_s": {k: (fma64[k] / sec(k) if stage_ms[k] > 0 else None) for k in bytes_},
        "profiled_stage_bound": {k: ("fp64" if fma64[k] / FP64_FMA_PER_S > bytes_[k] / HBM_BYTES_PER_S else "hbm")
                                 for k in bytes_},
        "profiled_stage_fraction_of_bound": {k: (bound[k] / sec(k) if stage_ms[k] > 0 else None) for k in bytes_},
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
