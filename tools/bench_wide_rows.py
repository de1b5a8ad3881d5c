"""Walk-stage throughput and the dense Adam sweep at n_emb 128, 256 and 512 on the bench graph (C3).

C3 = synth.power_law(1M, 20, seed 0), the bench's roots (synth.pick_roots, R = 16 384 resident, seed 0), hub threshold 128,
the default walk path (depth-1 reuse, level-synchronous steps, TMA-staged hub lists).  The widths alternate within one
process (rounds x widths), so clock drift hits all of them alike.  Per width:
  - D-pass negative edges/s (accepted walks / pass time) and the walk-stage ms (device events around gg_walk_sample's
    walk phase, the stage whose row gathers change with the width);
  - rows_gathered (the pass's counter: the depth-1 stage's rows and the walk stage's, as bench.py reports it) and
    achieved bytes/s = rows_gathered * (4 * ld + 8) / walk-stage time -- an upper bound, since the depth-1 stage's rows
    are in the numerator and not its time in the denominator; and the same for the walk stage's own rows
    (rows_gathered_walk_stage, the counter's growth during the walk stage);
  - the dense Adam sweep (gg_adam_apply, per-thread loads) over E, m, v of the 1M rows;
  - T1 parity: the last pass's walks of 12 roots against the canonical C oracle;
  - card name, power limit and SM clock (nvidia-smi query, read only).
Writes one JSON line per width to measurements/h100/wide_rows.jsonl (or --out).

    python tools/bench_wide_rows.py [--rounds 3] [--steps 10] [--out PATH]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=20).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smax}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        import torch
        return {"name": torch.cuda.get_device_name(0)}


def parity(hg, emb_h, ld, roots, trees, out, seed, tag, k=12):
    """Walks of the first k roots of the pass against oracle/canonical.walk_pass (T1)."""
    from oracle import canonical as can
    sel = np.arange(min(k, len(roots)))
    par = trees.parent_arrays(sel).cpu().numpy()
    wp = out.walk_ptr.cpu().numpy()
    num = np.diff(wp)[sel]
    bits = np.zeros((hg.adj.shape[0] + 31) // 32, np.uint32)
    ref = can.walk_pass(can.pad_rows(emb_h, ld), np.zeros(hg.n_node, np.float32), hg.indptr, hg.adj,
                        roots[sel], par, num, True, bits, seed=seed, pass_tag=tag)
    W = int(num.sum())
    ok = (np.array_equal(out.samples.cpu().numpy()[:W], ref.samples) and np.array_equal(out.status.cpu().numpy()[:W], ref.status))
    return {"roots": int(len(sel)), "walks": W, "bit_exact": bool(ok)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--roots", type=int, default=16384)
    ap.add_argument("--widths", default="128,256,512")
    ap.add_argument("--out", default=os.path.join(ROOT, "measurements", "h100", "wide_rows.jsonl"))
    args = ap.parse_args()
    import torch
    from graphgan_b200 import _cabi, graph as G, sampler as S, synth
    from graphgan_b200.sampler import CNT
    dev = torch.device("cuda:0")
    lib = _cabi.lib()
    n = 1_000_000
    hg = G.HostGraph(synth.power_law(n, 20, seed=0), None, n_node=n)
    roots = synth.pick_roots(hg.degrees(), args.roots, seed=0)
    dg = G.DeviceGraph(hg, dev)
    smp = S.WalkSampler(dg, hub_threshold=128)
    trees = smp.build_trees(roots)
    sample_num = dg.raw_deg[trees.roots.long()]
    bias = torch.zeros(n, dtype=torch.float32, device=dev)
    widths = [int(w) for w in args.widths.split(",")]
    embs = {d: synth.embeddings(n, d, seed=1) for d in widths}
    ev = lambda: torch.cuda.Event(enable_timing=True)
    res = {d: {"pass_ms": [], "walk_ms": [], "rows": [], "rows_walk": [], "accepted": [], "adam_ms": []} for d in widths}
    last = {}
    for r in range(args.rounds):
        for d in widths:
            emb = S.pad_embedding(embs[d], dev)
            ld = int(emb.shape[1])
            plan = smp.plan(trees, sample_num, True)
            for s in range(2):                                   # warm-up
                smp.run(emb, bias, trees, sample_num, True, seed=0, pass_tag=900 + s, plan=plan)
            torch.cuda.synchronize()
            for s in range(args.steps):
                e = [ev() for _ in range(4)]
                tag = 1000 * (r + 1) + s
                e[0].record()
                smp.precompute(emb, bias, plan)
                smp.run(emb, bias, trees, sample_num, True, seed=0, pass_tag=tag, finalize=False, plan=plan, precompute=False,
                        phase_mask=1)
                c1 = plan.counters.clone()                       # the depth-1 stage's counts (device copy)
                e[1].record()
                out = smp.run(emb, bias, trees, sample_num, True, seed=0, pass_tag=tag, finalize=False, plan=plan,
                              precompute=False, phase_mask=2, zero_counters=False)
                e[2].record()
                smp.finalize(out)
                smp.emit_d_rows(out)
                e[3].record()
                torch.cuda.synchronize()
                cnt = out.counters_host()
                res[d]["pass_ms"].append(e[0].elapsed_time(e[3]))
                res[d]["walk_ms"].append(e[1].elapsed_time(e[2]))
                res[d]["rows"].append(cnt["rows_gathered"])
                res[d]["rows_walk"].append(cnt["rows_gathered"] - int(c1[CNT["rows_gathered"]].item()))
                res[d]["accepted"].append(cnt["accepted"])
                last[d] = (out, tag)
            # dense Adam sweep over the 1M rows (no gradient rows: every row decays and moves, the timed work)
            m, v = torch.zeros_like(emb), torch.zeros_like(emb)
            mb, vb, b = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
            slot = torch.full((n,), -1, dtype=torch.int32, device=dev)
            g = torch.zeros((1, ld), device=dev)
            gb = torch.zeros(1, device=dev)
            for s in range(args.steps + 2):
                e0, e1 = ev(), ev()
                e0.record()
                _cabi.check(lib.gg_adam_apply(n, ld, emb.data_ptr(), m.data_ptr(), v.data_ptr(), b.data_ptr(), mb.data_ptr(),
                                              vb.data_ptr(), None, None, g.data_ptr(), gb.data_ptr(), slot.data_ptr(),
                                              C.c_float(1e-3), C.c_float(0.9), C.c_float(0.999), C.c_float(1e-8), None),
                            "gg_adam_apply")
                e1.record()
                torch.cuda.synchronize()
                if s >= 2:
                    res[d]["adam_ms"].append(e0.elapsed_time(e1))
            if r == args.rounds - 1:
                out, tag = last[d]
                res[d]["parity"] = parity(hg, embs[d], ld, roots, trees, out, 0, tag)
            del emb, m, v
            torch.cuda.empty_cache()
    info = gpu_info()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for d in widths:
            x = res[d]
            ld = S.pad_embedding(np.zeros((1, d)), "cpu").shape[1]
            walk_ms = float(np.median(x["walk_ms"]))
            rows = float(np.median(x["rows"]))
            rows_walk = float(np.median(x["rows_walk"]))
            line = {
                "n_emb": d, "ld": int(ld), "graph": "power_law N=1M avg_deg=20 (C3), R=%d resident roots, hub_threshold 128" % len(roots),
                "neg_edges_per_s": float(np.median(np.asarray(x["accepted"]) / (np.asarray(x["pass_ms"]) * 1e-3))),
                "pass_ms_median": float(np.median(x["pass_ms"])), "walk_stage_ms_median": walk_ms,
                "walk_stage_ms_min": float(np.min(x["walk_ms"])), "rows_gathered": rows,
                "walk_stage_bytes_per_s": rows * (4 * ld + 8) / (walk_ms * 1e-3),
                "rows_gathered_walk_stage": rows_walk,
                "walk_stage_own_rows_bytes_per_s": rows_walk * (4 * ld + 8) / (walk_ms * 1e-3),
                "adam_sweep_ms_median": float(np.median(x["adam_ms"])),
                "adam_sweep_bytes_per_s": 24.0 * n * ld / (float(np.median(x["adam_ms"])) * 1e-3),
                "t1_parity": x.get("parity"), "samples": len(x["walk_ms"]), "rounds": args.rounds, "gpu": info,
            }
            f.write(json.dumps(line) + "\n")
            print(json.dumps(line))


if __name__ == "__main__":
    main()
