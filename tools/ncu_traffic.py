#!/usr/bin/env python
"""tools/ncu_traffic.py -- turn an ncu capture of one sampling pass into profiles/ncu_traffic.json.

    python tools/ncu_traffic.py k1_metrics.ncu-rep powerlaw_1m@R16384 "<capture description>"

Reads dram__bytes_read.sum + dram__bytes_write.sum and gpu__time_duration.sum per kernel launch (ncu -i ... --page raw
--csv --print-units base), sums them per kernel family, and records the content hash of the kernel sources the
capture was taken from -- bench.py only quotes these numbers while the library it runs was built from the same
sources (graphgan_b200/_build.py: source_hash)."""
import csv
import io
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FAMILIES = ["hub_score_tm_kernel", "root_cdf_kernel", "root_step_kernel", "step1_cdf_kernel", "flat_start_kernel", "flat_enum_kernel",
            "flat_choose_kernel", "walk_kernel", "finalize_kernel",
            "emit_rows_kernel", "bfs_kernel", "adam_kernel", "reward_kernel", "pair_grad_kernel"]


def main():
    rep, key, desc = sys.argv[1], sys.argv[2], (sys.argv[3] if len(sys.argv) > 3 else "")
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv", "--print-units", "base"], stdout=subprocess.PIPE, text=True,
                         check=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    head = rows[0]
    col = {name: k for k, name in enumerate(head)}
    need = ["Kernel Name", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__time_duration.sum"]
    for n in need:
        if n not in col:
            raise SystemExit("metric %s missing from the capture" % n)
    per = {}
    for r in rows[2:]:
        if len(r) < len(head):
            continue
        name = r[col["Kernel Name"]]
        fam = next((f for f in FAMILIES if f in name), None)
        if fam is None:
            continue
        b = float(r[col["dram__bytes_read.sum"]].replace(",", "")) + float(r[col["dram__bytes_write.sum"]].replace(",", ""))
        t = float(r[col["gpu__time_duration.sum"]].replace(",", ""))
        e = per.setdefault(fam, {"launches": 0, "dram_bytes": 0.0, "time_ns": 0.0, "name": name})
        e["launches"] += 1; e["dram_bytes"] += b; e["time_ns"] += t
    from graphgan_b200 import _build
    path = os.path.join(ROOT, "profiles", "ncu_traffic.json")
    try:
        doc = json.load(open(path))
    except (OSError, ValueError):
        doc = {}
    # the hash of the sources the CAPTURED library was built from: pass it (4th argument) when the tree has moved on
    h = sys.argv[4] if len(sys.argv) > 4 else _build.source_hash()
    if doc.get("source_hash") != h:
        doc = {"source_hash": h, "kernels": {}, "detail": {}}
    walk = ["flat_start_kernel", "flat_enum_kernel", "flat_choose_kernel", "walk_kernel"]   # the walk stage (one walk_kernel per pass)
    k1 = ["hub_score_tm_kernel", "root_cdf_kernel", "root_step_kernel", "step1_cdf_kernel"] + walk
    entry = {f: per[f]["dram_bytes"] / per[f]["launches"] for f in per}
    if "walk_kernel" in per:
        passes = per["walk_kernel"]["launches"]             # the capture must cover whole passes
        entry["walk_stage"] = sum(per[f]["dram_bytes"] for f in walk if f in per) / passes
        entry["walk_stage_ncu_us"] = sum(per[f]["time_ns"] for f in walk if f in per) / passes / 1e3
        for f in ("flat_enum_kernel", "flat_choose_kernel", "flat_start_kernel"):
            if f in per:
                entry[f + "_per_pass"] = per[f]["dram_bytes"] / passes
                entry[f + "_ncu_us_per_pass"] = per[f]["time_ns"] / passes / 1e3
        if all(f in per for f in ("hub_score_tm_kernel", "root_cdf_kernel")):
            entry["k1_stage"] = sum(per[f]["dram_bytes"] for f in k1 if f in per) / passes
    doc["kernels"].setdefault(key, {}).update(entry)
    doc["detail"].setdefault(key, {}).update({f: {"launches": per[f]["launches"], "dram_bytes_per_launch": entry[f],
                                                   "ncu_time_us_per_launch": per[f]["time_ns"] / per[f]["launches"] / 1e3,
                                                   "kernel": per[f]["name"]} for f in per})
    doc["capture"] = desc or os.path.basename(rep)
    doc["how"] = "ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none (per launch: read + write)"
    json.dump(doc, open(path, "w"), indent=1)
    print(json.dumps(doc["detail"][key], indent=1))


if __name__ == "__main__":
    main()
