"""Cost of training on the exact game (DESIGN.md section 5.5): the dense Adam sweep, one exact D / G step on the bench
graph and whole-graph steps on CA-GrQc.

  sweep     gg_adam_apply_dense against gg_adam_apply (the ldg sweep, no gradient rows) at C3 shape, N = 1M, ld 128, the two
            alternating, each timed between CUDA events over --reps launches.  Bytes: the dense step reads acc (8) and reads
            and writes E, m, v (24) per element, and 32 per bias (acc_bias 8, b / m_b / v_b 24); the sparse sweep moves 24 per
            element and 28 per row (biases and the row -> slot map).  Against 3.35 TB/s, the HBM3 bandwidth of the H100 SXM
            data sheet.
  C3 step   C3 = synth.power_law(1M, 20, seed 0), n_emb 128, hub threshold 128, the 64 roots of
            tools/bench_generator_dist.py, one chunk (scratch budget --scratch-gb).  One exact D step with G's law
            computed beforehand (GraphGAN.exact_d_step with law=...), one exact G step (exact_g_step), the law itself, each
            between CUDA events.  One further D step and G step run under torch.profiler, which gives the device time per
            kernel; the sweep is adam_dense_kernel.
  CA-GrQc   the tests/golden/cagrqc fixture (N = 5242, n_emb 50), every non-isolated root: one D phase of
            config.n_epochs_dis steps (GraphGAN.exact_d_phase) and one G step, after one untimed warm-up of each.
Card name, power limit and SM clock come from a read-only nvidia-smi query in the same run.  Writes one JSON object to
measurements/h100/exact_steps.json (or --out).

    python tools/bench_exact_steps.py [--steps 5] [--warmup 1] [--reps 20] [--scratch-gb 16] [--out PATH]
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


def sweep(torch, dev, reps):
    from graphgan_b200 import _cabi
    from graphgan_b200._cabi import ptr
    lib = _cabi.lib()
    n, ld = 1_000_000, 128
    g = torch.Generator(device=dev).manual_seed(0)
    emb = torch.randn((n, ld), device=dev, generator=g) * 0.3
    m, v = torch.zeros_like(emb), torch.full_like(emb, 1e-6)
    b, mb, vb = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.full((n,), 1e-6, device=dev)
    acc = torch.randn((n, ld), device=dev, dtype=torch.float64, generator=g)
    acc_b = torch.randn(n, device=dev, dtype=torch.float64, generator=g)
    slot = torch.full((n,), -1, dtype=torch.int32, device=dev)
    rows, rb = torch.zeros((16, ld), device=dev), torch.zeros(16, device=dev)
    nu, uq = torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(16, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    f = C.c_float

    def dense():
        _cabi.check(lib.gg_adam_apply_dense(n, ld, ptr(emb), ptr(m), ptr(v), ptr(b), ptr(mb), ptr(vb), ptr(acc), ptr(acc_b),
                                            C.c_double(1e-3), f(1e-5), f(1e-5), f(1e-6), f(0.9), f(0.999), f(1e-8), st))

    def sparse():
        _cabi.check(lib.gg_adam_apply(n, ld, ptr(emb), ptr(m), ptr(v), ptr(b), ptr(mb), ptr(vb), ptr(nu), ptr(uq), ptr(rows),
                                      ptr(rb), ptr(slot), f(1e-6), f(0.9), f(0.999), f(1e-8), st))
    arms = {"dense": dense, "sparse": sparse}
    times = {k: [] for k in arms}
    for k in arms:                     # warm-up
        arms[k]()
    torch.cuda.synchronize()
    for rnd in range(4):               # alternating rounds of `reps` launches each
        for k in (("dense", "sparse") if rnd % 2 == 0 else ("sparse", "dense")):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                arms[k]()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / reps)
    bytes_ = {"dense": 32 * n * ld + 32 * n, "sparse": 24 * n * ld + 28 * n}
    out = {}
    for k in arms:
        ms = float(np.median(times[k]))
        out[k] = {"ms_median": ms, "ms_rounds": times[k], "bytes": bytes_[k], "bytes_per_s": bytes_[k] / (ms * 1e-3),
                  "fraction_of_hbm": bytes_[k] / (ms * 1e-3) / HBM_BYTES_PER_S}
    out["dense_fraction_over_sparse_fraction"] = out["dense"]["fraction_of_hbm"] / out["sparse"]["fraction_of_hbm"]
    del emb, m, v, acc, acc_b
    torch.cuda.empty_cache()
    return out


def c3_steps(torch, dev, steps, warmup, budget):
    from graphgan_b200 import graph as G, synth
    from graphgan_b200.graph_gan import GraphGAN
    n, d = 1_000_000, 128
    hg = G.HostGraph(synth.power_law(n, 20, seed=0), None, n_node=n)
    deg = hg.degrees()
    top = int(np.argmax(np.diff(hg.indptr)))
    nb = hg.adj[hg.indptr[top]:hg.indptr[top + 1]]
    bench_roots = synth.pick_roots(deg, 16384, seed=0)
    hubs = bench_roots[np.argsort(-deg[bench_roots], kind="stable")[:12]]
    rand = np.random.RandomState(1).choice(bench_roots, 48, replace=False)
    roots = np.unique(np.concatenate([[top], nb[[0, len(nb) // 2, len(nb) - 1]], hubs, rand])).astype(np.int32)
    gan = GraphGAN(host_graph=hg, node_embed_init_d=synth.embeddings(n, d, seed=2, sigma=0.2),
                   node_embed_init_g=synth.embeddings(n, d, seed=1))
    gan.generator.bias_t.copy_(torch.as_tensor(np.random.RandomState(5).normal(0, 0.1, n).astype(np.float32)))
    gan.discriminator.bias_t.copy_(torch.as_tensor(np.random.RandomState(6).normal(0, 0.5, n).astype(np.float32)))
    g = gan.generator
    ev = lambda: torch.cuda.Event(enable_timing=True)
    t = {"law": [], "d_step_cached_law": [], "g_step": []}
    for step in range(warmup + steps):
        e = [ev() for _ in range(4)]
        e[0].record()
        law = gan.sampler.distribution(g.emb, g.bias_t, gan._exact_trees(roots), max_scratch_bytes=budget)
        e[1].record()
        gan.exact_d_step(roots, law=law, max_scratch_bytes=budget)
        e[2].record()
        gan.exact_g_step(roots, max_scratch_bytes=budget)
        e[3].record()
        torch.cuda.synchronize()
        if step >= warmup:
            for i, k in enumerate(t):
                t[k].append(e[i].elapsed_time(e[i + 1]))
    from torch.profiler import ProfilerActivity, profile
    prof_ms = {}
    for name, fn in (("d_step_cached_law", lambda: gan.exact_d_step(roots, law=law, max_scratch_bytes=budget)),
                     ("g_step", lambda: gan.exact_g_step(roots, max_scratch_bytes=budget))):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        per = {}
        for evt in prof.key_averages():
            if evt.device_time_total > 0:
                per[evt.key] = per.get(evt.key, 0.0) + evt.device_time_total / 1e3
        prof_ms[name] = dict(sorted(per.items(), key=lambda kv: -kv[1]))
    med = lambda xs: float(np.median(xs))
    R = len(roots)
    sweep_ms = {k: sum(v for kk, v in p.items() if "adam_dense" in kk) for k, p in prof_ms.items()}
    return {
        "workload": "power_law N=1M avg_deg=20 (C3), n_emb %d (ld 128), hub_threshold 128, %d roots in one chunk" % (d, R),
        "roots": R, "ms_median": {k: med(v) for k, v in t.items()}, "ms_all": t,
        "ms_per_root": {k: med(v) / R for k, v in t.items()},
        "profiled_sweep_ms": sweep_ms,
        "profiled_ms_per_root_without_sweep": {k: (sum(p.values()) - sweep_ms[k]) / R for k, p in prof_ms.items()},
        "profiled_kernel_ms": prof_ms,
    }


def cagrqc_steps(torch, dev):
    from graphgan_b200 import config, graph as G
    from graphgan_b200.graph_gan import GraphGAN
    from tests.golden import loader
    c = loader.load("cagrqc")
    hg = G.HostGraph(c.train_edges, c.test_edges, n_node=c.n)
    config.exact_roots = hg.n_node
    gan = GraphGAN(host_graph=hg, node_embed_init_d=c.emb_d, node_embed_init_g=c.emb_g)
    roots = gan.exact_roots()
    gan.exact_d_phase(roots, 1)
    gan.exact_g_step(roots)
    torch.cuda.synchronize()
    ev = lambda: torch.cuda.Event(enable_timing=True)
    e = [ev() for _ in range(3)]
    e[0].record()
    outs = gan.exact_d_phase(roots, int(config.n_epochs_dis))
    e[1].record()
    gan.exact_g_step(roots)
    e[2].record()
    torch.cuda.synchronize()
    return {"workload": "CA-GrQc (tests/golden/cagrqc), N = %d, n_emb %d, every non-isolated root" % (c.n, c.emb_g.shape[1]),
            "roots": len(roots), "root_ok": int(outs[0][2].sum().item()), "d_phase_steps": int(config.n_epochs_dis),
            "d_phase_ms": e[0].elapsed_time(e[1]), "g_step_ms": e[1].elapsed_time(e[2])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--scratch-gb", type=float, default=16.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "measurements", "h100", "exact_steps.json"))
    args = ap.parse_args()
    import torch
    from bench_generator_dist import gpu_info
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    dev = torch.device("cuda:0")
    from graphgan_b200 import config
    config.device = "cuda:0"
    line = {"gpu": gpu_info(), "sweep_c3_shape": sweep(torch, dev, args.reps)}
    line["c3_step"] = c3_steps(torch, dev, args.steps, args.warmup, int(args.scratch_gb * (1 << 30)))
    torch.cuda.empty_cache()
    line["cagrqc"] = cagrqc_steps(torch, dev)
    line["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(line, indent=1) + "\n")
    print(json.dumps(line))


if __name__ == "__main__":
    main()
