#!/usr/bin/env python
"""tools/count_level_repeats.py -- how often walks of one root stand on the same node at the same step (CPU only).

From step 2 on, a walk's candidate list is [tree father] + children(node) in its root's BFS tree, so the list, its
scores and its CDF depend on (root, node) alone.  This counts, on bench.py's C3 inputs (graph, embeddings, roots,
seed 0, pass tag 2000, zero bias), how many choices ("visits") fall on how many distinct (root, node) pairs per step,
and the embedding rows an on-demand step gathers (1 + n for a node below the score-cache threshold) per visit and once
per pair.  For score-cached (hub) nodes, whose steps gather no rows, it weights each visit by its list length instead:
the list entries ([father] + children, what the softmax / CDF passes run over) and the adjacency entries the tree-bit
enumeration scans (the node's degree), per visit and once per pair, and the largest group (visits of one pair).  The walks come from the canonical C oracle (oracle/canonical.py: walk_pass, D mode, paths recorded) on a
uniform random sample of the bench's roots.

    python tools/count_level_repeats.py [--roots 2048]
"""
import argparse
import collections
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--roots", type=int, default=2048, help="roots sampled from the bench's 16 384")
    p.add_argument("--hub-threshold", type=int, default=128)
    p.add_argument("--chunk", type=int, default=32, help="roots per oracle call")
    args = p.parse_args()
    from graphgan_b200 import graph as G, synth
    from oracle import canonical as can

    t0 = time.time()
    n = 1_000_000
    hg = G.HostGraph(synth.power_law(n, 20, seed=0), None, n_node=n)            # bench.py: powerlaw_1m, seed 0
    deg = np.diff(hg.indptr)
    emb = can.pad_rows(synth.embeddings(n, 128, seed=1), 128)
    bias = np.zeros(n, np.float32)
    roots_all = synth.pick_roots(hg.degrees(), 16384, seed=0)
    sel = np.sort(np.random.RandomState(5).choice(len(roots_all), min(args.roots, len(roots_all)), replace=False))
    print("setup %.1f s" % (time.time() - t0), file=sys.stderr, flush=True)

    visits, distinct = collections.Counter(), collections.Counter()       # (step bucket, cached) -> count
    rows_visit, rows_distinct = collections.Counter(), collections.Counter()
    list_visit, list_distinct = collections.Counter(), collections.Counter()   # hub nodes: list entries
    scan_visit, scan_distinct = collections.Counter(), collections.Counter()   # hub nodes: adjacency entries scanned
    largest = collections.Counter()
    lens = collections.Counter()
    walks = 0
    for c0 in range(0, len(sel), args.chunk):
        rts = roots_all[sel[c0:c0 + args.chunk]]
        par = can.bfs_parents(hg.indptr, hg.adj, rts)
        bits = np.zeros((hg.adj.shape[0] + 31) // 32 + 1, np.uint32)
        res = can.walk_pass(emb, bias, hg.indptr, hg.adj, rts, par, deg[rts], True, bits, seed=0, pass_tag=2000, max_path=64)
        for k in range(len(rts)):
            seen = collections.Counter()
            pk = par[k]
            for w in range(res.walk_ptr[k], res.walk_ptr[k + 1]):
                walks += 1
                if res.status[w] != can.DONE:
                    continue
                L = int(res.path_len[w])
                lens[L] += 1
                path = res.paths[w, :L]
                for s in range(2, L - 1):                   # path[s] is the node the walk chooses from at step s
                    x = int(path[s])
                    cached = bool(deg[x] >= args.hub_threshold)
                    key = (min(s, 5), cached)
                    children = int(np.count_nonzero(pk[hg.adj[hg.indptr[x]:hg.indptr[x + 1]]] == x))
                    nrows = 0 if cached else 2 + children
                    nlist, nscan = 1 + children, int(deg[x])
                    visits[key] += 1
                    rows_visit[key] += nrows
                    list_visit[key] += nlist
                    scan_visit[key] += nscan
                    if (s, x) not in seen:
                        distinct[key] += 1
                        rows_distinct[key] += nrows
                        list_distinct[key] += nlist
                        scan_distinct[key] += nscan
                    seen[(s, x)] += 1
                    largest[key] = max(largest[key], seen[(s, x)])
        print("%d roots, %.1f s" % (c0 + len(rts), time.time() - t0), file=sys.stderr, flush=True)

    print("roots %d, walks %d, path lengths %s" % (len(sel), walks, sorted(lens.items())))
    print("| step | node kind | visits | distinct (root, node) | visits / distinct | rows: per walk | rows: once per (root, node) |")
    print("|---|---|---|---|---|---|---|")
    for key in sorted(visits):
        s, cached = key
        print("| %s | %s | %d | %d | %.2f | %s | %s |" % (
            "%d" % s if s < 5 else "5+", "cached (hub)" if cached else "not cached", visits[key], distinct[key],
            visits[key] / max(distinct[key], 1), "-" if cached else rows_visit[key], "-" if cached else rows_distinct[key]))
    print()
    print("| step | hub visits | distinct (root, node) | list entries: per visit -> once per key | "
          "adjacency entries scanned: per visit -> once | largest group |")
    print("|---|---|---|---|---|---|")
    for key in sorted(k for k in visits if k[1]):
        s = key[0]
        print("| %s | %d | %d | %d -> %d (%.2fx) | %d -> %d (%.2fx) | %d |" % (
            "%d" % s if s < 5 else "5+", visits[key], distinct[key], list_visit[key], list_distinct[key],
            list_visit[key] / max(list_distinct[key], 1), scan_visit[key], scan_distinct[key],
            scan_visit[key] / max(scan_distinct[key], 1), largest[key]))
    print("steps >= 2: %d visits on %d distinct (root, node); rows %d -> %d" % (
        sum(visits.values()), sum(distinct.values()), sum(rows_visit.values()), sum(rows_distinct.values())))


if __name__ == "__main__":
    main()
