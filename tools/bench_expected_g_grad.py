"""Cost of the exact expectation of the reference's G step (csrc/value_gref.cu, DESIGN.md section 5.6), and its cosine with
grad_G V on CA-GrQc during reference training.

Cost: C3 = synth.power_law(1M, 20, seed 0), n_emb 128, hub threshold 128, window 2; the 64 roots of
tools/bench_value_grad.py, in one chunk (scratch budget 16 GiB).  Per timed step, between CUDA events:
WalkSampler.distribution and WalkSampler.expected_g_grad.  One further call runs under torch.profiler, which splits
expected_g_grad into its kernels:
  - gdist_rec   the recording section 5.1 kernel;
  - reach       reach_kernel (top-down over the recorded levels);
  - score       score_kernel (kappa_up / kappa_dn of every (reached y, d));
  - npairs      npairs_kernel;
  - gather      big_nodes_kernel + gather_kernel;
  - memset      the scratch clears.
Bytes per stage are what the algorithm has to move, from shapes and counts (R roots, N nodes, nnz walk entries, ld floats
per row, M reached nodes, P = sum over reached y of min(w, depth(y)) window pairs, S = entries scanned by the down walks):
  gdist_rec  rows gathered (counter) * 4 ld + R N 44;  reach  M (16 + 8 + 8 + 8);
  score      P (4 rows of 4 ld + 8 kappa) + M w 4 father reads;  npairs  R N (4 w + 8);
  gather     2 P (4 ld + 16) row and coefficient reads + S (4 + 4 + 4) + 2 N (8 ld + 8) accumulators.
The figures count every row read once per use; rows repeated across siblings come from L2, so the HBM share is a floor.
gcos: CA-GrQc (the test fixture: training edges, pretrained embeddings), reference training with the defaults of
config.py except n_epochs = 2, text files off, value_roots = 512 with value_grad and value_gcos: the value lines at the
pretrained embeddings and after one and after two epochs.
Card name, power limit and SM clock come from a read-only nvidia-smi query.  Writes one JSON object to
measurements/h100/expected_g_grad.json (or --out).

    python tools/bench_expected_g_grad.py [--steps 5] [--warmup 1] [--scratch-gb 16] [--epochs 2] [--out PATH]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_BYTES_PER_S = 3.35e12    # H100 SXM5 80 GB data sheet
WINDOW = 2
STAGES = (("gdist_rec", ("gdist_rec_kernel",)), ("reach", ("reach_kernel",)), ("score", ("score_kernel",)),
          ("npairs", ("npairs_kernel",)), ("gather", ("big_nodes_kernel", "gather_kernel")), ("memset", ("Memset", "memset")))


def c3_cost(args):
    import torch
    from bench_generator_dist import gpu_info
    from graphgan_b200 import graph as G, sampler as S, synth
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
    ld = int(g_emb.shape[1])
    budget = int(args.scratch_gb * (1 << 30))
    counters = torch.zeros(16, dtype=torch.int64, device=dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    t = {k: [] for k in ("distribution", "expected_g_grad")}
    outs, trees = [], smp.build_trees(roots)
    for step in range(args.warmup + args.steps):
        e = [ev() for _ in range(3)]
        e[0].record()
        counters.zero_()
        smp.distribution(g_emb, g_bias, trees, max_scratch_bytes=budget, counters=counters)
        e[1].record()
        out = smp.expected_g_grad(g_emb, g_bias, d_emb, d_bias, trees, window=WINDOW, max_scratch_bytes=budget)
        e[2].record()
        torch.cuda.synchronize()
        if step >= args.warmup:
            for i, k in enumerate(t):
                t[k].append(e[i].elapsed_time(e[i + 1]))
            outs.append([x.cpu().numpy().tobytes() for x in out])
    same = all(o == outs[0] for o in outs)
    rows_gathered = int(counters[8].item())
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        smp.expected_g_grad(g_emb, g_bias, d_emb, d_bias, trees, window=WINDOW, max_scratch_bytes=budget)
        torch.cuda.synchronize()
    stage_ms = {k: 0.0 for k, _ in STAGES}
    for evt in prof.key_averages():
        for k, names in STAGES:
            if any(s in evt.key for s in names):
                stage_ms[k] += evt.device_time_total / 1e3     # microseconds -> ms
                break
    # counts from the trees (host): reached nodes, window pairs, entries the down walks scan, pairs under the top hub
    par = trees.parent_arrays().cpu().numpy()
    M = P = S_ = hub_pairs = 0
    degw = np.diff(hg.indptr)
    for k in range(R):
        fa = par[k].astype(np.int64)                     # -1 for the root and nodes outside the tree
        tree = fa >= 0
        tree[roots[k]] = True
        m, x = np.zeros(n, np.int64), fa.copy()
        for _ in range(WINDOW):                          # m = min(w, depth)
            live = x >= 0
            m += live
            x = np.where(live, fa[np.maximum(x, 0)], -1)
        M += int(tree.sum())
        P += int(m.sum())
        # node u's list is scanned by the down walks of itself and of its ancestors up to w - 1 levels above it
        S_ += int((degw[tree] * (1 + np.minimum(m[tree], WINDOW - 1))).sum())
        ch = np.flatnonzero(fa == top)
        hub_pairs += len(ch) + int(np.isin(fa, ch).sum())
    bytes_ = {
        "gdist_rec": rows_gathered * 4 * ld + R * n * 44,
        "reach": M * 40,
        "score": P * (16 * ld + 8) + M * WINDOW * 4,
        "npairs": R * n * (4 * WINDOW + 8),
        "gather": 2 * P * (4 * ld + 16) + S_ * 12 + 2 * n * (8 * ld + 8),
        "memset": R * n * (8 + 4),
    }
    med = lambda xs: float(np.median(xs))
    okh = np.frombuffer(outs[0][1], np.int32)
    return {
        "workload": "expected reference G step, power_law N=1M avg_deg=20 (C3), n_emb %d (ld %d), hub_threshold 128, window "
                    "%d, %d roots in one chunk" % (d, ld, WINDOW, R),
        "roots": R, "root_ok": int(okh.sum()),
        "ms_per_root": {k: med(v) / R for k, v in t.items()},
        "ms_per_call_median": {k: med(v) for k, v in t.items()},
        "expected_g_grad_over_distribution": med(t["expected_g_grad"]) / med(t["distribution"]),
        "profiled_stage_ms_per_root": {k: v / R for k, v in stage_ms.items()},
        "profiled_stage_bytes": bytes_,
        "profiled_stage_bytes_per_s": {k: (bytes_[k] / (stage_ms[k] * 1e-3) if stage_ms[k] > 0 else None) for k in bytes_},
        "profiled_stage_fraction_of_hbm_bound": {k: (bytes_[k] / HBM_BYTES_PER_S / (stage_ms[k] * 1e-3) if stage_ms[k] > 0
                                                     else None) for k in bytes_},
        "reached_nodes": M, "window_pairs_per_orientation": P, "down_walk_entries_scanned": S_,
        "pairs_below_the_top_hub_children_plus_grandchildren": hub_pairs,
        "n_pairs_mean": float(np.frombuffer(outs[0][0], np.float64)[okh == 1].mean()),
        "identical_over_steps": bool(same),
        "scratch_budget_bytes": budget, "steps": args.steps, "warmup": args.warmup, "gpu": gpu_info(),
    }


def cagrqc_gcos(args):
    from graphgan_b200 import config, graph as G
    from graphgan_b200.graph_gan import GraphGAN
    from tests.golden import loader
    c = loader.load("cagrqc")
    tmp = tempfile.mkdtemp()

    def wr(name, e):
        p = os.path.join(tmp, name)
        with open(p, "w") as f:
            f.write("".join("%d\t%d\n" % (a, b) for a, b in e))
        return p
    for k, v in dict(n_epochs=args.epochs, value_roots=512, value_grad=True, value_gcos=True, text_embeddings=False,
                     device="cuda:0", test_filename=wr("test.txt", c.test_edges),
                     test_neg_filename=wr("test_neg.txt", c.test_neg_edges),
                     emb_filenames=[os.path.join(tmp, "gen.emb"), os.path.join(tmp, "dis.emb")],
                     result_filename=os.path.join(tmp, "res.txt"), model_log=os.path.join(tmp, "log") + "/").items():
        setattr(config, k, v)
    gan = GraphGAN(host_graph=G.HostGraph(c.train_edges, c.test_edges), node_embed_init_d=c.emb_d, node_embed_init_g=c.emb_g)
    gan.train()
    with open(config.result_filename) as f:
        lines = [ln.strip() for ln in f if ln.startswith("value:")]
    rows = []
    for ep, ln in enumerate(lines):
        kv = dict(x.split(":", 1) for x in ln.split())
        rows.append({"after_epochs": ep, "gcos": float(kv["gcos"]), "gnorm": float(kv["gnorm"]), "value": float(kv["value"]),
                     "roots": int(kv["roots"])})
    return {"dataset": "CA-GrQc (pretrained embeddings, reference config defaults, window %d)" % config.window_size,
            "value_roots": 512, "per_evaluation": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--scratch-gb", type=float, default=16.0)
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "measurements", "h100", "expected_g_grad.json"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    line = {"c3_cost": c3_cost(args), "cagrqc_gcos": cagrqc_gcos(args)}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(line, indent=1) + "\n")
    print(json.dumps(line))


if __name__ == "__main__":
    main()
