"""Cost and figures of the game value against the best discriminator (csrc/best_response.cu, DESIGN.md section 5.8).

1. C3 = synth.power_law(1M, 20, seed 0), n_emb 128, hub threshold 128, the 64 roots of tools/bench_game_value.py in one
   chunk (scratch budget --scratch-gb).  Per timed step, each between its own CUDA events: tree build, distribution
   (section 5.1), best_response (value), best_response_grad (value + gradient + the final SpMM).  Medians per root, and
   for the value path the algorithmic bytes of the rows it scores (an upper bound: every depth-1 list scored on demand,
   (n_a + 1) rows of 4 ld + 4 bytes per depth-1 node a, plus the root's list) over its time, against the 3.35 TB/s HBM3
   data-sheet figure (a 700 W H100 SXM figure).
2. C3, all 16 384 bench roots (synth.pick_roots(deg, 16384, seed 0)) in one call each of best_response and
   best_response_grad under the default 2 GiB budget (their trees alone take 40 GB).
3. CA-GrQc (tests/golden/cagrqc.npz, pretrained embeddings) with every root: mean JSD and hit over the ok roots at the
   pretrained generator; after one production D pass over every root (its father removals): the share of true-neighbour
   entries (c -> a, a reached) whose father entry is removed, so G(a | c) = 0, and mean JSD and hit; then a G-only fit of
   --fit-steps Adam steps on the mean JSD (lr --fit-lr, no L2 term), mean JSD and hit along the way.
Card name, power limit and SM clock come from a read-only nvidia-smi query.  Writes one JSON object to
measurements/h100/best_response.json (or --out).

    python tools/bench_best_response.py [--steps 5] [--warmup 1] [--scratch-gb 16] [--fit-steps 20] [--out PATH]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_BYTES_PER_S = 3.35e12    # H100 SXM5 80 GB data sheet


def _jsd_hit(vs, ht, ok):
    sel = ok.cpu().numpy() == 1
    v, h = vs.cpu().numpy()[sel], ht.cpu().numpy()[sel]
    return {"mean_jsd": float((v / 2 + np.log(2.0)).mean()), "mean_hit": float(h.mean()), "ok_roots": int(sel.sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--scratch-gb", type=float, default=16.0)
    ap.add_argument("--fit-steps", type=int, default=20)
    ap.add_argument("--fit-lr", type=float, default=1e-3)
    ap.add_argument("--out", default=os.path.join(ROOT, "measurements", "h100", "best_response.json"))
    args = ap.parse_args()
    import torch
    from bench_generator_dist import gpu_info
    from graphgan_b200 import graph as G, sampler as S, synth
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    dev = torch.device("cuda:0")
    budget = int(args.scratch_gb * (1 << 30))
    out = {"gpu": gpu_info(), "scratch_budget_bytes": budget, "steps": args.steps, "warmup": args.warmup}

    # ---- 1. C3, 64 roots
    n, d = 1_000_000, 128
    hg = G.HostGraph(synth.power_law(n, 20, seed=0), None, n_node=n)
    deg = hg.degrees()
    wdeg = np.diff(hg.indptr)
    top = int(np.argmax(wdeg))
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
    ld = int(g_emb.shape[1])
    ev = lambda: torch.cuda.Event(enable_timing=True)
    t = {k: [] for k in ("tree_build", "distribution", "best_response", "best_response_grad")}
    outs = []
    for step in range(args.warmup + args.steps):
        e = [ev() for _ in range(5)]
        e[0].record()
        trees = smp.build_trees(roots)
        e[1].record()
        smp.distribution(g_emb, g_bias, trees, max_scratch_bytes=budget)
        e[2].record()
        v = smp.best_response(g_emb, g_bias, trees, max_scratch_bytes=budget)
        e[3].record()
        gr = smp.best_response_grad(g_emb, g_bias, trees, max_scratch_bytes=budget)
        e[4].record()
        torch.cuda.synchronize()
        if step >= args.warmup:
            for i, k in enumerate(t):
                t[k].append(e[i].elapsed_time(e[i + 1]))
            outs.append(b"".join(x.cpu().numpy().tobytes() for x in v + gr))
    med = {k: float(np.median(x)) for k, x in t.items()}
    rows = sum(int(wdeg[a]) + 1 for c in roots for a in hg.adj[hg.indptr[c]:hg.indptr[c + 1]]) + int(wdeg[roots].sum())
    vbytes = rows * (4 * ld + 4)
    out["c3_64_roots"] = {
        "workload": "power_law N=1M avg_deg=20 (C3), n_emb %d (ld %d), hub_threshold 128, %d roots in one chunk" % (d, ld, R),
        "ms_per_root": {k: x / R for k, x in med.items()},
        "ms_per_call_median": med,
        "value_over_distribution": med["best_response"] / med["distribution"],
        "grad_over_distribution": med["best_response_grad"] / med["distribution"],
        "value_row_bytes_upper_bound": vbytes,
        "value_fraction_of_hbm_bound_upper": vbytes / HBM_BYTES_PER_S / (med["best_response"] * 1e-3),
        "identical_over_steps": all(o == outs[0] for o in outs),
        **_jsd_hit(*v),
    }
    print(json.dumps(out["c3_64_roots"]), flush=True)
    # ---- 2. C3, all bench roots in one call (ascending ids: the trees, 2.5 MB per root, are not copied), 2 GiB budget
    del v, gr, trees
    torch.cuda.empty_cache()
    all_roots = np.sort(np.asarray(bench_roots, np.int32))
    trees = smp.build_trees(all_roots)
    res = {}
    for name, fn in (("best_response", smp.best_response), ("best_response_grad", smp.best_response_grad)):
        fn(g_emb, g_bias, trees.select(torch.arange(64, device=dev)))   # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        o = fn(g_emb, g_bias, trees)
        torch.cuda.synchronize()
        res[name + "_s"] = time.perf_counter() - t0
        if name == "best_response":
            res.update(_jsd_hit(*o))
    res["roots"] = len(all_roots)
    res["ms_per_root"] = {k[:-2]: res[k] * 1e3 / len(all_roots) for k in ("best_response_s", "best_response_grad_s")}
    out["c3_all_bench_roots"] = res
    print(json.dumps(res), flush=True)
    del trees, dg, smp, g_emb, hg
    torch.cuda.empty_cache()

    # ---- 3. CA-GrQc
    from tests.golden import loader
    c = loader.load("cagrqc")
    hg = G.HostGraph(c["train_edges"], c["test_edges"], n_node=c.n)
    dg = G.DeviceGraph(hg, dev)
    smp = S.WalkSampler(dg, hub_threshold=128)
    roots = np.flatnonzero(hg.degrees() > 0).astype(np.int32)
    trees = smp.build_trees(roots)
    emb = S.pad_embedding(c.emb_g, dev)
    bias = torch.zeros(hg.n_node, dtype=torch.float32, device=dev)
    q = {"roots": len(roots), "pretrained": _jsd_hit(*smp.best_response(emb, bias, trees))}
    smp.run(emb, bias, trees, torch.as_tensor(hg.degrees()[roots].astype(np.int64)).to(dev), True, seed=1, pass_tag=1)
    bits = dg.d1_bits.cpu().numpy().view(np.uint32)
    par = trees.parent_arrays().cpu().numpy()
    n_ent = n_rm = 0
    for k, r in enumerate(roots):
        for e in range(hg.indptr[r], hg.indptr[r + 1]):
            if par[k][hg.adj[e]] != r:
                continue
            n_ent += 1
            n_rm += int((bits[e >> 5] >> (e & 31)) & 1)
    q["after_one_d_pass"] = _jsd_hit(*smp.best_response(emb, bias, trees))
    q["after_one_d_pass"]["share_of_true_neighbour_entries_removed"] = n_rm / max(n_ent, 1)
    # G-only fit: Adam on the mean JSD (the fp64 gradient scaled by 1/(2 n_ok))
    from graphgan_b200.generator import Generator
    gen = Generator(hg.n_node, c.emb_g, device=dev)
    gen.lr = np.float32(args.fit_lr)
    gen.lam = np.float32(0.0)
    fit = []
    for step in range(args.fit_steps + 1):
        vs, ht, ok, gE, gb = smp.best_response_grad(gen.emb, gen.bias_t, trees)
        fit.append(dict(step=step, **_jsd_hit(vs, ht, ok)))
        if step < args.fit_steps:
            gen.apply_dense_grad(gE, gb, 1.0 / (2 * int(ok.sum().item())))
    q["g_only_fit"] = {"lr": args.fit_lr, "trace": fit}
    out["cagrqc"] = q
    print(json.dumps(q), flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
