"""Cost of the second moment of one G walk's step (csrc/value_gref.cu, DESIGN.md section 5.9), and the signal-to-noise
ratio of the reference's G pass on CA-GrQc during reference training.

Cost: C3 = synth.power_law(1M, 20, seed 0), n_emb 128, hub threshold 128, window 2; the 64 roots of
tools/bench_expected_g_grad.py, in one chunk (scratch budget 24 GiB).  Per timed step, between CUDA events and alternating
in the same run: WalkSampler.expected_g_grad and WalkSampler.expected_g_moments.  One further call of
expected_g_moments runs under torch.profiler, which splits off the new stages:
  - moment      moment_kernel (full(y) and tail(y) of every reached y);
  - prefix      moment_prefix_kernel (top-down Pf and |s(y)|^2);
  - root_sum    root_sum_kernel, twice (sq_c and mn_c);
  - gather_sq   gather_sq_kernel (gather_kernel's work and the squared-contribution plane);
  - rest        every other kernel and memset (section 5.6's stages and the clears).
Bytes per stage are what the algorithm has to move (R roots, N nodes, M reached nodes, ld floats per row):
  moment     M (2w + 1) 4 ld path rows + M 2w 4 father reads + M (2w + 1) w 8 kappa reads + M 16 stores;
  prefix     M (16 item + 3 * 8 + 2 * 8);  root_sum  R N (8 + 8 + 8);
  gather_sq  the section 5.6 gather's bytes (tools/bench_expected_g_grad.py) + R N 8 plane stores.
The moment and gather figures count every row read once per use; repeated rows come from L2, so the HBM share is a floor.
gsnr: CA-GrQc (the test fixture: training edges, pretrained embeddings), reference training with the defaults of config.py
except n_epochs = 2, text files off, value_roots = 512 with value_gcos and value_gsnr: the value lines at the pretrained
embeddings and after one and two epochs, with the median of var_c / mn_c over the ok value roots with mn_c > 0 at each.
Card name, power limit and SM clock come from a read-only nvidia-smi query.  Writes one JSON object to
measurements/h100/expected_g_moments.json (or --out).

    python tools/bench_expected_g_moments.py [--steps 5] [--warmup 1] [--scratch-gb 24] [--epochs 2] [--out PATH]
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
STAGES = (("moment", ("moment_kernel",)), ("prefix", ("moment_prefix_kernel",)), ("root_sum", ("root_sum_kernel",)),
          ("gather_sq", ("gather_sq_kernel",)))


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
    t = {k: [] for k in ("expected_g_grad", "expected_g_moments")}
    trees = smp.build_trees(roots)
    a = (g_emb, g_bias, d_emb, d_bias, trees)
    same, first = True, None
    for step in range(args.warmup + args.steps):
        e = [ev() for _ in range(3)]
        e[0].record()
        ref = smp.expected_g_grad(*a, window=WINDOW, max_scratch_bytes=budget)
        e[1].record()
        out = smp.expected_g_moments(*a, window=WINDOW, max_scratch_bytes=budget)
        e[2].record()
        torch.cuda.synchronize()
        if step >= args.warmup:
            for i, k in enumerate(t):
                t[k].append(e[i].elapsed_time(e[i + 1]))
        bits = [x.cpu().numpy().tobytes() for x in out]
        same = same and bits[:2] + bits[4:] == [x.cpu().numpy().tobytes() for x in ref] and bits == (first or bits)
        first = first or bits
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        smp.expected_g_moments(*a, window=WINDOW, max_scratch_bytes=budget)
        torch.cuda.synchronize()
    stage_ms = {k: 0.0 for k, _ in STAGES}
    stage_ms["rest"] = 0.0
    for evt in prof.key_averages():
        for k, names in STAGES:
            if any(s in evt.key for s in names):
                stage_ms[k] += evt.device_time_total / 1e3     # microseconds -> ms
                break
        else:
            stage_ms["rest"] += evt.device_time_total / 1e3
    par = trees.parent_arrays().cpu().numpy()
    M = P = S_ = 0
    degw = np.diff(hg.indptr)
    for k in range(R):
        fa = par[k].astype(np.int64)
        tree = fa >= 0
        tree[roots[k]] = True
        m, x = np.zeros(n, np.int64), fa.copy()
        for _ in range(WINDOW):
            live = x >= 0
            m += live
            x = np.where(live, fa[np.maximum(x, 0)], -1)
        M += int(tree.sum())
        P += int(m.sum())
        S_ += int((degw[tree] * (1 + np.minimum(m[tree], WINDOW - 1))).sum())
    w = WINDOW
    bytes_ = {
        "moment": M * ((2 * w + 1) * 4 * ld + 2 * w * 4 + (2 * w + 1) * w * 8 + 16),
        "prefix": M * (16 + 24 + 16),
        "root_sum": R * n * 24,
        "gather_sq": 2 * P * (4 * ld + 16) + S_ * 12 + 2 * n * (8 * ld + 8) + R * n * 8,
    }
    med = lambda xs: float(np.median(xs))
    ok = np.frombuffer(first[1], np.int32) == 1
    sq, mn = np.frombuffer(first[2], np.float64), np.frombuffer(first[3], np.float64)
    return {
        "workload": "second moment of the expected reference G step, power_law N=1M avg_deg=20 (C3), n_emb %d (ld %d), "
                    "hub_threshold 128, window %d, %d roots in one chunk" % (d, ld, WINDOW, R),
        "roots": R, "root_ok": int(ok.sum()),
        "ms_per_root": {k: med(v) / R for k, v in t.items()},
        "ms_per_call_median": {k: med(v) for k, v in t.items()},
        "moments_over_grad": med(t["expected_g_moments"]) / med(t["expected_g_grad"]),
        "profiled_stage_ms_per_root": {k: v / R for k, v in stage_ms.items()},
        "profiled_stage_bytes": bytes_,
        "profiled_stage_fraction_of_hbm_bound": {k: (bytes_[k] / HBM_BYTES_PER_S / (stage_ms[k] * 1e-3) if stage_ms[k] > 0
                                                     else None) for k in bytes_},
        "reached_nodes": M, "window_pairs_per_orientation": P,
        "var_over_mn_median": float(np.median((sq - mn)[ok & (mn > 0)] / mn[ok & (mn > 0)])),
        "grad_bits_equal_and_identical_over_steps": bool(same),
        "scratch_budget_bytes": budget, "steps": args.steps, "warmup": args.warmup, "gpu": gpu_info(),
    }


def cagrqc_gsnr(args):
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
    for k, v in dict(n_epochs=args.epochs, value_roots=512, value_gcos=True, value_gsnr=True, text_embeddings=False,
                     device="cuda:0", test_filename=wr("test.txt", c.test_edges),
                     test_neg_filename=wr("test_neg.txt", c.test_neg_edges),
                     emb_filenames=[os.path.join(tmp, "gen.emb"), os.path.join(tmp, "dis.emb")],
                     result_filename=os.path.join(tmp, "res.txt"), model_log=os.path.join(tmp, "log") + "/").items():
        setattr(config, k, v)
    gan = GraphGAN(host_graph=G.HostGraph(c.train_edges, c.test_edges), node_embed_init_d=c.emb_d, node_embed_init_g=c.emb_g)
    ratios, line_of = [], gan.value_line

    def value_line():
        _, ok, sq, mn = (x.cpu().numpy() for x in gan.expected_g_moments(gan.value_roots())[:4])
        sel = (ok == 1) & (mn > 0)
        ratios.append(float(np.median((sq - mn)[sel] / mn[sel])))
        return line_of()
    gan.value_line = value_line
    gan.train()
    with open(config.result_filename) as f:
        lines = [ln.strip() for ln in f if ln.startswith("value:")]
    rows = []
    for ep, ln in enumerate(lines):
        kv = dict(x.split(":", 1) for x in ln.split())
        rows.append({"after_epochs": ep, "gsnr": float(kv["gsnr"]), "gcos": float(kv["gcos"]), "value": float(kv["value"]),
                     "roots": int(kv["roots"]), "var_over_mn_median": ratios[ep]})
    return {"dataset": "CA-GrQc (pretrained embeddings, reference config defaults, window %d, n_sample_gen %d)"
                       % (config.window_size, config.n_sample_gen),
            "value_roots": 512, "per_evaluation": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--scratch-gb", type=float, default=24.0)
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "measurements", "h100", "expected_g_moments.json"))
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    line = {"c3_cost": c3_cost(args), "cagrqc_gsnr": cagrqc_gsnr(args)}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(line, indent=1) + "\n")
    print(json.dumps(line))


if __name__ == "__main__":
    main()
