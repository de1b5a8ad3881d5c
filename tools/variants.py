#!/usr/bin/env python
"""tools/variants.py -- build A/B variants of libgraphgan_b200.so (compile-time knobs of csrc/walk_common.cuh) and,
on a GPU box, run the default bench line with each of them:

    python tools/variants.py build             # here (nvcc cross-compiles): writes libgraphgan_b200.<name>.so
    python tools/variants.py run  [--steps N]  # on the GPU box: one JSON summary line per variant
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = {
    "base": [],                                   # defaults of csrc/walk_common.cuh: 3 CTAs/SM, 2048 scores, UNR 4 / 8
    "occ4": ["GG_WALK_MIN_CTAS=4", "GG_SC_CAP=1024", "GG_UNR=2"],    # 4 CTAs/SM at 64 registers
    "occ5": ["GG_WALK_MIN_CTAS=5"],
    "unr2": ["GG_UNR=2"],
    "share0": ["GG_SHARE_LEVELS=0"],              # no shared level: every level runs flat_enum + flat_choose per walk
    "share23": ["GG_SHARE_LEVELS=0xC"],           # levels 2 and 3 shared (default: level 2)
    "hub0": ["GG_SHARE_HUB=0"],                   # shared levels run their hub walks per walk (default: one warp per hub group)
}


def main():
    from graphgan_b200 import _build
    if sys.argv[1] == "build":
        for name, defs in VARIANTS.items():
            print(name, _build.build_variant(name, defs))
        return
    extra = sys.argv[2:]
    for name in VARIANTS:
        path = os.path.join(ROOT, "graphgan_b200", "libgraphgan_b200.%s.so" % name)
        if not os.path.exists(path):
            continue
        env = dict(os.environ, GG_LIB=path)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--no-cpu-baseline", "--verify", "4", "--g-steps", "0",
                            "--steps", "30", "--warmup", "3"] + extra, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        try:
            d = json.loads(r.stdout.strip().splitlines()[-1])
            k = d["roofline"]["k1_stage"]
            print(json.dumps({"variant": name, "defines": VARIANTS[name], "value": d["value"], "e2e": d["e2e"]["value"],
                              "ms_per_step": d["ms_per_step"], "pre_ms": k["hub_scores_root_cdf_ms"], "depth1_ms": k["root_step_step1_cdf_ms"],
                              "walk_ms": k["walk_kernel_ms"], "parity": d["parity"]}))
        except Exception as e:      # noqa: BLE001
            print(json.dumps({"variant": name, "error": str(e), "stderr": r.stderr[-600:]}))
        sys.stdout.flush()


if __name__ == "__main__":
    main()
