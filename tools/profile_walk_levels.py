#!/usr/bin/env python
"""tools/profile_walk_levels.py -- device time of the walk stage per kernel and per level, with the level sizes.

Runs the D-sampling pass of bench.py's workload (default C3: power-law N = 1M, n_emb 128, R = 16 384 roots) under
torch.profiler (CUDA activities only) for --passes passes and writes ONE JSON record:

  levels[s]   device microseconds per pass of each kernel of level-synchronous step s (flat_dedupe / flat_enum /
              flat_choose / flat_draw and the table clear of a shared level), and the level's sizes read back from the
              flat counters: records (walks that take step s), hub items (walks on a score-cached node), distinct
              keys (distinct (root slot, node) items of a shared level that are not score-cached; 0 on a level that
              does not share) and hub owners / hub work items (distinct score-cached (root slot, node) groups of a
              shared level and the work items they were split into; 0 where hub walks run per walk);
  stage       flat_start_kernel, the walk_kernel tail, and the whole walk stage (first to last of its kernels);
  precompute  device microseconds per pass of the per-pass precompute kernels (the hub score kernel and root_cdf_kernel),
              from a second profiled region of --passes whole passes of its own.
  depth1      the same for the depth-1 stage (root_step_kernel, step1_cdf_kernel), from the same region.

The levels reuse kernel names, so a kernel is given to a level by launch order within the pass.  Load an A/B library
with GG_LIB=<path> (tools/variants.py) to profile another build.

    python tools/profile_walk_levels.py [--passes 20] [--out FILE]
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FLAT_CTR_WORDS = 1 + 4 * 16          # csrc/walk.cu: FLAT_CTR_WORDS
FLAT_CTR_ALL = FLAT_CTR_WORDS + 3 * 16   # csrc/walk.cu: FLAT_CTR_ALL (the hub group words follow the level words)


def short_name(name):
    m = re.search(r"(\w+_kernel)(<[^()]*>)?\(", name)
    if m:
        return m.group(1) + (m.group(2) or "")
    return "memset" if "memset" in name.lower() else name


def kernel_events(prof):
    """(start_ns, duration_ns, short name) of every device activity, in launch order"""
    out = []
    for e in prof.profiler.kineto_results.events():
        if str(e.device_type()).endswith("CUDA"):
            out.append((e.start_ns(), e.duration_ns(), short_name(e.name())))
    out.sort()
    return out


def split_levels(events, n_passes):
    """per pass: {level key: {kernel: ns}}; level keys 1..S, 'start', 'tail'; plus the stage's first-to-last span"""
    passes, cur, span = [], None, None
    level, after_choose = 0, False
    for t, dur, name in events:
        base = name.split("<")[0]
        if base == "flat_start_kernel":
            cur, level, after_choose = {"start": {name: dur}}, 0, False
            span = [t, t + dur]
            passes.append((cur, span))
            continue
        if cur is None:
            continue
        if base == "walk_kernel":
            cur.setdefault("tail", {})[name] = dur
            span[1] = t + dur
            cur = None
            continue
        if base in ("memset", "flat_dedupe_kernel", "flat_enum_kernel") and (after_choose or level == 0):
            level, after_choose = level + 1, False
        if base == "flat_choose_kernel":
            after_choose = True
        if level > 0:
            d = cur.setdefault(level, {})
            d[name] = d.get(name, 0) + dur
        span[1] = t + dur
    if len(passes) != n_passes:
        raise RuntimeError("found %d walk stages in the trace, expected %d" % (len(passes), n_passes))
    return passes


DEPTH1_KERNELS = ("root_step_kernel", "step1_cdf_kernel")


def precompute_kernels(events, n_passes, depth1=False):
    """{kernel: microseconds per pass} of the precompute kernels (hub_score*_kernel, root_cdf_kernel), or with depth1 of
    the depth-1 stage (root_step_kernel, step1_cdf_kernel)"""
    tot, cnt = {}, {}
    for _, dur, name in events:
        base = name.split("<")[0]
        if (base in DEPTH1_KERNELS) if depth1 else (base.startswith("hub_score") or base == "root_cdf_kernel"):
            tot[name] = tot.get(name, 0) + dur
            cnt[name] = cnt.get(name, 0) + 1
    for k, c in cnt.items():
        if c != n_passes:
            raise RuntimeError("found %d launches of %s in the trace, expected %d" % (c, k, n_passes))
    return {k: round(v / n_passes / 1e3, 2) for k, v in sorted(tot.items())}


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=30)
        name, plim, clk = (x.strip() for x in r.stdout.strip().splitlines()[0].split(","))
        return {"name": name, "power_limit": plim, "max_sm_clock": clk}
    except Exception as e:      # noqa: BLE001
        return {"error": str(e)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--passes", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--workload", default="powerlaw_1m")
    p.add_argument("--roots", type=int, default=16384)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--label", default=None, help="free text stored in the record (which library, which setting)")
    p.add_argument("--out", default=None, help="append the record to this file (it is always printed)")
    args = p.parse_args()
    if args.passes < 20:
        raise SystemExit("--passes must be >= 20")

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from graphgan_b200 import _cabi, graph as G, sampler as S

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bargs = argparse.Namespace(workload=args.workload, seed=args.seed, impl="b200", roots=args.roots)
    hg, emb_h, roots, _ = bench.make_inputs(bargs, 0)
    dg = G.DeviceGraph(hg, dev)
    smp = S.WalkSampler(dg, hub_threshold=128, depth1=True)
    emb = S.pad_embedding(emb_h, dev)
    bias = torch.zeros(hg.n_node, dtype=torch.float32, device=dev)
    trees = smp.build_trees(roots)
    sample_num = dg.raw_deg[trees.roots.long()]
    plan = smp.plan(trees, sample_num, True)
    dg.hub_tiles(smp.hub_threshold)
    plan.depth1_buffers(smp)
    plan.start_order(smp)

    def one_pass(tag):
        out = smp.run(emb, bias, trees, sample_num, True, seed=args.seed, pass_tag=tag, finalize=False, plan=plan)
        smp.finalize(out)
        smp.emit_d_rows(out)
        return out

    for s in range(args.warmup):
        one_pass(1000 + s)
    torch.cuda.synchronize()
    ctrs = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(args.passes):
            one_pass(2000 + s)
            ctrs.append(plan._flat[:4 * FLAT_CTR_ALL].clone())        # device copy, read after the region
        torch.cuda.synchronize()
    passes = split_levels(kernel_events(prof), args.passes)
    with profile(activities=[ProfilerActivity.CUDA]) as prof_pre:     # precompute: a region of its own
        for s in range(args.passes):
            one_pass(3000 + s)
        torch.cuda.synchronize()
    pre = precompute_kernels(kernel_events(prof_pre), args.passes)
    depth1 = precompute_kernels(kernel_events(prof_pre), args.passes, depth1=True)
    ctr =np.stack([c.view(torch.int32).cpu().numpy().astype(np.int64) for c in ctrs])   # [passes, words]

    levels = {}
    for s in range(1, smp.flat_steps + 1):
        names = sorted({k for per, _ in passes for k in per.get(s, {})})
        levels[str(s)] = {
            "kernels_us": {k: round(float(np.mean([per.get(s, {}).get(k, 0) for per, _ in passes])) / 1e3, 2) for k in names},
            "total_us": round(float(np.mean([sum(per.get(s, {}).values()) for per, _ in passes])) / 1e3, 2),
            "records": int(ctr[:, 1 + 4 * s].mean()), "hub_items": int(ctr[:, 1 + 4 * s + 1].mean()),
            "distinct_keys": int(ctr[:, 1 + 4 * s + 2].mean()),
            "hub_owners": int(ctr[:, FLAT_CTR_WORDS + 3 * s].mean()),
            "hub_work_items": int(ctr[:, FLAT_CTR_WORDS + 3 * s + 1].mean()),
        }
    rec = {
        "tool": "tools/profile_walk_levels.py", "label": args.label, "lib": os.path.basename(os.environ.get("GG_LIB") or _cabi._build.LIB),
        "gpu": gpu_info(), "workload": args.workload, "roots": int(len(roots)), "walks": int(plan.n_walks),
        "flat_steps": smp.flat_steps, "passes": args.passes,
        "levels": levels,
        "start_us": round(float(np.mean([sum(per["start"].values()) for per, _ in passes])) / 1e3, 2),
        "tail_us": round(float(np.mean([sum(per.get("tail", {}).values()) for per, _ in passes])) / 1e3, 2),
        "tail_records": int(ctr[:, 0].mean()),
        "walk_stage_span_us": round(float(np.mean([sp[1] - sp[0] for _, sp in passes])) / 1e3, 2),
        "walk_stage_kernel_sum_us": round(float(np.mean([sum(sum(v.values()) for v in per.values()) for per, _ in passes])) / 1e3, 2),
        "precompute_us": pre, "precompute_total_us": round(sum(pre.values()), 2),
        "depth1_us": depth1, "depth1_total_us": round(sum(depth1.values()), 2),
        "hub_entries": int(dg.hub_tiles(smp.hub_threshold)[3]),
        "note":"device time per pass (mean over the profiled passes); span = first walk-stage kernel start to the tail's "
                "end, kernel_sum = the sum of the stage's kernel durations (the gaps between them are the difference)",
    }
    line = json.dumps(rec)
    print(line)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
