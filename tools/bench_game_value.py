"""Cost of the exact game value V_c(G, D) (csrc/value.cu, DESIGN.md section 5.2) on the bench graph.

C3 = synth.power_law(1M, 20, seed 0), n_emb 128, hub threshold 128; the 64 roots of tools/bench_generator_dist.py (the
top-degree node, three of its neighbours, the 12 highest-degree bench roots and 48 random bench roots), in one chunk
(scratch budget 16 GiB).  Per timed step, each between its own CUDA events:
  - tree build (WalkSampler.build_trees of the 64 roots);
  - the generator distribution (WalkSampler.distribution: hub scores + gg_generator_dist), dist [64, N];
  - the value kernel (gg_game_value on those rows: the pos and neg items, then the tile reduction).
Reports medians per root, the value kernel's share of the gdist time, and for the value kernel the bytes and FMAs its
algorithm needs, from shapes (per chunk of R roots: N (4 ld + 4) bytes of discriminator rows and biases + 8 R N bytes of
dist; R N ld FMAs), the achieved rates and its share of whichever data-sheet bound is larger (3.35 TB/s HBM3, 67 TFLOP/s
FP32 = 33.5 T FMA/s; figures for a 700 W H100 SXM).  Also checks that the kernel's output is identical over the steps and
equal to WalkSampler.game_value's.  Card name, power limit and SM clock come from a read-only nvidia-smi query.
Writes one JSON object to measurements/h100/game_value.json (or --out).

    python tools/bench_game_value.py [--steps 10] [--warmup 2] [--scratch-gb 16] [--out PATH]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_BYTES_PER_S = 3.35e12    # H100 SXM5 80 GB data sheet
FP32_FMA_PER_S = 67e12 / 2   # 67 TFLOP/s FP32, two flops per FMA


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--scratch-gb", type=float, default=16.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "measurements", "h100", "game_value.json"))
    args = ap.parse_args()
    import torch
    from bench_generator_dist import gpu_info
    from graphgan_b200 import _cabi, graph as G, sampler as S, synth
    from graphgan_b200._cabi import ptr
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
    R = len(roots)
    dg = G.DeviceGraph(hg, dev)
    smp = S.WalkSampler(dg, hub_threshold=128)
    g_emb = S.pad_embedding(synth.embeddings(n, d, seed=1), dev)
    g_bias = torch.as_tensor(np.random.RandomState(5).normal(0, 0.1, n).astype(np.float32)).to(dev)
    d_emb = S.pad_embedding(synth.embeddings(n, d, seed=2, sigma=0.2), dev)
    d_bias = torch.as_tensor(np.random.RandomState(6).normal(0, 0.5, n).astype(np.float32)).to(dev)
    ld = int(d_emb.shape[1])
    budget = int(args.scratch_gb * (1 << 30))
    lib = _cabi.lib()
    nbytes = C.c_int64(0)
    _cabi.check(lib.gg_game_value_scratch_bytes(n, R, C.byref(nbytes)))
    scratch = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    pos = torch.empty(R, dtype=torch.float64, device=dev)
    neg, ok = torch.empty_like(pos), torch.empty(R, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream

    def value(trees, dist, root_ok):
        _cabi.check(lib.gg_game_value(n, ld, ptr(d_emb), ptr(d_bias), ptr(dg.raw_indptr), ptr(dg.raw_adj), R, ptr(trees.roots),
                                      ptr(dist), ptr(root_ok), ptr(pos), ptr(neg), ptr(ok), ptr(scratch), scratch.numel(), st),
                    "gg_game_value")

    ev = lambda: torch.cuda.Event(enable_timing=True)
    t_tree, t_dist, t_val, outs = [], [], [], []
    for step in range(args.warmup + args.steps):
        e = [ev() for _ in range(4)]
        e[0].record()
        trees = smp.build_trees(roots)
        e[1].record()
        dist, root_ok = smp.distribution(g_emb, g_bias, trees, max_scratch_bytes=budget)
        e[2].record()
        value(trees, dist, root_ok)
        e[3].record()
        torch.cuda.synchronize()
        if step >= args.warmup:
            t_tree.append(e[0].elapsed_time(e[1]))
            t_dist.append(e[1].elapsed_time(e[2]))
            t_val.append(e[2].elapsed_time(e[3]))
            outs.append(b"".join(x.cpu().numpy().tobytes() for x in (pos, neg, ok)))
    whole = smp.game_value(g_emb, g_bias, d_emb, d_bias, trees, max_scratch_bytes=budget)
    same = all(o == outs[0] for o in outs) and outs[0] == b"".join(x.cpu().numpy().tobytes() for x in whole)
    med = lambda xs: float(np.median(xs))
    tv = med(t_val) * 1e-3
    bytes_ = n * (4 * ld + 4) + 8 * R * n
    fmas = R * n * ld
    t_bytes, t_fma = bytes_ / HBM_BYTES_PER_S, fmas / FP32_FMA_PER_S
    okh, posh, negh = ok.cpu().numpy(), pos.cpu().numpy(), neg.cpu().numpy()
    line = {
        "workload": "game value, power_law N=1M avg_deg=20 (C3), n_emb %d (ld %d), hub_threshold 128, %d roots in one chunk"
                    % (d, ld, R),
        "roots": R, "root_ok": int(okh.sum()),
        "ms_per_root": {"tree_build": med(t_tree) / R, "distribution": med(t_dist) / R, "value_kernel": med(t_val) / R},
        "ms_per_call_median": {"tree_build": med(t_tree), "distribution": med(t_dist), "value_kernel": med(t_val)},
        "value_kernel_ms_min": float(np.min(t_val)),
        "value_over_distribution": med(t_val) / med(t_dist),
        "value_kernel": {
            "bytes_per_chunk": bytes_, "fma_per_chunk": fmas,
            "bytes_per_s": bytes_ / tv, "fma_per_s": fmas / tv,
            "bound": "HBM bandwidth" if t_bytes >= t_fma else "FP32 FMA",
            "bound_ms": max(t_bytes, t_fma) * 1e3,
            "fraction_of_bound": max(t_bytes, t_fma) / tv,
        },
        "mean_value": float((posh + negh)[okh == 1].mean()), "mean_pos": float(posh[okh == 1].mean()),
        "mean_neg": float(negh[okh == 1].mean()),
        "identical_over_steps_and_to_game_value": bool(same),
        "scratch_budget_bytes": budget, "steps": args.steps, "warmup": args.warmup, "gpu": gpu_info(),
    }
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(line, indent=1) + "\n")
    print(json.dumps(line))


if __name__ == "__main__":
    main()
