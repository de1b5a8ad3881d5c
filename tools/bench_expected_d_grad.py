"""Cost of the D-mode walk law and of the exact expectation of the reference's D step (csrc/gdist.cu, csrc/value.cu,
csrc/value_dgrad.cu; DESIGN.md section 5.7), and the step's cosine with grad_D V on CA-GrQc during reference training.

Cost: C3 = synth.power_law(1M, 20, seed 0), n_emb 128, hub threshold 128; the 64 roots of tools/bench_value_grad.py, in
one chunk (scratch budget 16 GiB).  Per timed step, between CUDA events: WalkSampler.distribution (the G law),
WalkSampler.d_distribution (the D law) and WalkSampler.expected_d_grad (D law + passes).  One further expected_d_grad
call runs under torch.profiler, which splits it into its kernels:
  - d_law    gdist_d_kernel;
  - accept   accept_kernel;
  - mult     mult_kernel;
  - W        value_wref_kernel;
  - centre   cen_kernel + cen_reduce_kernel;
  - node     node_kernel;
  - memset   the clears.
Bytes per pass are what the algorithm has to move (R roots, N nodes, ld floats per row, T = ceil(R / 64) root tiles of
the W pass, U = ceil(R / 32) root tiles of the centre pass):
  W       T N 4 ld rows + R N (8 P_D + 4 mult + 8 W);  centre  U N 4 ld rows + R N 8 W + R N/2048 8 ld partials;
  node    R N 8 W + 2 N (8 ld + 8) accumulators (read and written).
dcos: CA-GrQc (the test fixture: training edges, pretrained embeddings), reference training with the defaults of
config.py except n_epochs = 2, text files off, value_roots = 512 with value_grad_d and value_dcos: the value lines at the
pretrained embeddings and after one and after two epochs.
Card name, power limit and SM clock come from a read-only nvidia-smi query.  Writes one JSON object to
measurements/h100/expected_d_grad.json (or --out).

    python tools/bench_expected_d_grad.py [--steps 5] [--warmup 1] [--scratch-gb 16] [--epochs 2] [--out PATH]
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
STAGES = (("d_law", ("gdist_d_kernel",)), ("accept", ("accept_kernel",)), ("mult", ("mult_kernel",)),
          ("W", ("value_wref_kernel",)), ("centre", ("cen_kernel", "cen_reduce_kernel")), ("node", ("node_kernel",)),
          ("memset", ("Memset", "memset")))


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
    ev = lambda: torch.cuda.Event(enable_timing=True)
    t = {k: [] for k in ("g_law", "d_law", "expected_d_grad")}
    outs, trees = [], smp.build_trees(roots)
    for step in range(args.warmup + args.steps):
        e = [ev() for _ in range(4)]
        e[0].record()
        smp.distribution(g_emb, g_bias, trees, max_scratch_bytes=budget)
        e[1].record()
        smp.d_distribution(g_emb, g_bias, trees, max_scratch_bytes=budget)
        e[2].record()
        out = smp.expected_d_grad(g_emb, g_bias, d_emb, d_bias, trees, max_scratch_bytes=budget)
        e[3].record()
        torch.cuda.synchronize()
        if step >= args.warmup:
            for i, k in enumerate(t):
                t[k].append(e[i].elapsed_time(e[i + 1]))
            outs.append([x.cpu().numpy().tobytes() for x in out])
    same = all(o == outs[0] for o in outs)
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        smp.expected_d_grad(g_emb, g_bias, d_emb, d_bias, trees, max_scratch_bytes=budget)
        torch.cuda.synchronize()
    stage_ms = {k: 0.0 for k, _ in STAGES}
    for evt in prof.key_averages():
        for k, names in STAGES:
            if any(s in evt.key for s in names):
                stage_ms[k] += evt.device_time_total / 1e3     # microseconds -> ms
                break
    T, U, ct = -(-R // 64), -(-R // 32), -(-n // 2048)
    bytes_ = {
        "W": T * n * 4 * ld + R * n * 20,
        "centre": U * n * 4 * ld + R * n * 8 + R * ct * 8 * ld * 2,
        "node": R * n * 8 + 2 * n * (8 * ld + 8),
    }
    med = lambda xs: float(np.median(xs))
    acc = np.frombuffer(outs[0][0], np.float64)
    pv = np.frombuffer(outs[0][1], np.float64)
    okr = np.frombuffer(outs[0][2], np.int32)
    passes = sum(stage_ms[k] for k in ("accept", "mult", "W", "centre", "node"))
    return {
        "workload": "D-mode law and expected reference D step, power_law N=1M avg_deg=20 (C3), n_emb %d (ld %d), "
                    "hub_threshold 128, %d roots in one chunk" % (d, ld, R),
        "roots": R, "ok_ref": int(okr.sum()), "roots_with_p_void": int((pv > 0).sum()),
        "p_void_max": float(pv.max()), "accept_min_over_ok_ref": float(acc[okr == 1].min()) if okr.any() else None,
        "ms_per_root": {k: med(v) / R for k, v in t.items()},
        "ms_per_call_median": {k: med(v) for k, v in t.items()},
        "d_law_over_g_law": med(t["d_law"]) / med(t["g_law"]),
        "profiled_stage_ms_per_root": {k: v / R for k, v in stage_ms.items()},
        "profiled_passes_ms_per_root": passes / R,
        "profiled_stage_bytes": bytes_,
        "profiled_stage_bytes_per_s": {k: (bytes_[k] / (stage_ms[k] * 1e-3) if stage_ms[k] > 0 else None) for k in bytes_},
        "profiled_stage_fraction_of_hbm_bound": {k: (bytes_[k] / HBM_BYTES_PER_S / (stage_ms[k] * 1e-3) if stage_ms[k] > 0
                                                     else None) for k in bytes_},
        "identical_over_steps": bool(same),
        "scratch_budget_bytes": budget, "steps": args.steps, "warmup": args.warmup, "gpu": gpu_info(),
    }


def cagrqc_dcos(args):
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
    for k, v in dict(n_epochs=args.epochs, value_roots=512, value_grad_d=True, value_dcos=True, text_embeddings=False,
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
        rows.append({"after_epochs": ep, "dcos": float(kv["dcos"]), "dnorm": float(kv["dnorm"]), "value": float(kv["value"]),
                     "roots": int(kv["roots"])})
    acc, pv, okr = (x.cpu().numpy() for x in gan.expected_d_grad(gan.value_roots())[:3])
    return {"dataset": "CA-GrQc (pretrained embeddings, reference config defaults)", "value_roots": 512,
            "per_evaluation": rows,
            "after_training": {"ok_ref": int(okr.sum()), "mean_accept_over_ok_ref": float(acc[okr == 1].mean()),
                               "roots_with_p_void": int((pv > 0).sum())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--scratch-gb", type=float, default=16.0)
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "measurements", "h100", "expected_d_grad.json"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    line = {"c3_cost": c3_cost(args), "cagrqc_dcos": cagrqc_dcos(args)}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(line, indent=1) + "\n")
    print(json.dumps(line))


if __name__ == "__main__":
    main()
