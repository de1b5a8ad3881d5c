"""Graph containers: the reference's adjacency semantics laid out for the GPU.

The reference keeps ``graph: dict node -> list of neighbours`` in edge-file order, both
directions, duplicates and self-loops included (src/utils.py:12-47).  That order is part of
the sampling semantics (it is the BFS discovery order, graph_gan.py:96-107, and therefore the
candidate order of every softmax).  Here the same information is two CSRs:

  raw  CSR : graph[i] verbatim            -> positives of prepare_data_for_d, sample_num
  walk CSR : first occurrences, no self-loops -> BFS trees and walks (the only entries the
             reference's ``used_nodes`` filter can ever turn into children)
"""
import numpy as np

from . import _cabi

# Entries per work item of the hub score pass.  A target's hub entries run 4.8 long on average at the benchmarked power
# law (p99 34, longest 2 407): the cap keeps one target from becoming the launch's tail, and bounds how long the other
# three 8-lane groups of a warp wait on the longest item among them.
HUB_ITEM_CAP = 32


def read_edge_file(path):
    """src/utils.py:50-54: whitespace separated integer pairs, one edge per line."""
    if path == "" or path is None:
        return np.zeros((0, 2), np.int64)
    with open(path, "r") as f:
        rows = [ln.split() for ln in f if ln.strip()]
    return np.asarray(rows, dtype=np.int64).reshape(-1, 2)


class HostGraph:
    """Reference-order adjacency on the host, as flat numpy arrays."""

    def __init__(self, train_edges, test_edges=None, n_node=None):
        train = np.asarray(train_edges, np.int64).reshape(-1, 2)
        test = np.zeros((0, 2), np.int64) if test_edges is None else np.asarray(test_edges, np.int64).reshape(-1, 2)
        ids = np.unique(np.concatenate([train.ravel(), test.ravel()])) if (train.size + test.size) else np.zeros(0, np.int64)
        # utils.py:47 returns len(nodes); ids are assumed to be 0..n-1 like the reference does
        self.n_node = int(ids.shape[0]) if n_node is None else int(n_node)
        if ids.size and (ids[0] < 0 or ids[-1] >= self.n_node):
            raise ValueError("node ids must lie in [0, n_node)")
        n = self.n_node
        # graph[a].append(b); graph[b].append(a) per edge, in file order (utils.py:36-37)
        src = np.empty(2 * train.shape[0], np.int64)
        dst = np.empty(2 * train.shape[0], np.int64)
        src[0::2], src[1::2] = train[:, 0], train[:, 1]
        dst[0::2], dst[1::2] = train[:, 1], train[:, 0]
        order = np.argsort(src, kind="stable")
        src_s, dst_s = src[order], dst[order]
        self.raw_indptr = np.zeros(n + 1, np.int64)
        np.cumsum(np.bincount(src_s, minlength=n), out=self.raw_indptr[1:])
        self.raw_adj = dst_s.astype(np.int32)
        # walk CSR: drop self-loops, keep the first occurrence of every (src, dst)
        keep = src_s != dst_s
        s2, d2 = src_s[keep], dst_s[keep]
        key = s2 * n + d2
        _, first = np.unique(key, return_index=True)
        first.sort()
        s3, d3 = s2[first], d2[first]
        self.indptr = np.zeros(n + 1, np.int64)
        np.cumsum(np.bincount(s3, minlength=n), out=self.indptr[1:])
        self.adj = d3.astype(np.int32)
        self.max_deg = int(np.diff(self.indptr).max()) if n else 0

    @classmethod
    def from_arrays(cls, n_node, raw_indptr, raw_adj, indptr, adj):
        """Re-create a HostGraph from the four arrays a previous instance held (e.g. a cache on disk)."""
        g = cls.__new__(cls)
        g.n_node = int(n_node)
        g.raw_indptr, g.raw_adj = np.asarray(raw_indptr, np.int64), np.asarray(raw_adj, np.int32)
        g.indptr, g.adj = np.asarray(indptr, np.int64), np.asarray(adj, np.int32)
        assert g.raw_indptr.shape == g.indptr.shape == (g.n_node + 1,)
        g.max_deg = int(np.diff(g.indptr).max()) if g.n_node else 0
        return g

    @classmethod
    def from_files(cls, train_filename, test_filename=""):
        """utils.read_edges(train_filename, test_filename) (src/utils.py:12-47)."""
        return cls(read_edge_file(train_filename), read_edge_file(test_filename))

    def neighbors(self, i):
        """graph[i] exactly as the reference holds it."""
        return self.raw_adj[self.raw_indptr[i]:self.raw_indptr[i + 1]]

    def __getitem__(self, i):
        """``graph[i]`` as reference-style code indexes it (graph_gan.py:190: ``pos = self.graph[i]``)."""
        return self.neighbors(int(i)).tolist()

    def __len__(self):
        return self.n_node

    def degrees(self):
        """len(graph[i]) == sample_num of prepare_data_for_d (graph_gan.py:190-191)."""
        return np.diff(self.raw_indptr)


class DeviceGraph:
    """HostGraph uploaded once; owns the father-removal bitset (graph_gan.py:258-259)."""

    def __init__(self, host, device):
        import torch
        _cabi.lib()  # fail loudly now if the CUDA library is unavailable
        self.host = host
        self.device = torch.device(device)
        self.n_node = host.n_node
        self.max_deg = host.max_deg
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)
        # adj (and edge_score below) carry 4 padding entries: the TMA staging of hub lists copies whole 16-byte units
        self.indptr, self.adj = t(host.indptr), t(np.concatenate([host.adj, np.zeros(4, np.int32)]))[:host.adj.shape[0]]
        same = host.raw_adj.shape == host.adj.shape and np.array_equal(host.raw_adj, host.adj)
        self.raw_indptr = self.indptr if same else t(host.raw_indptr)
        self.raw_adj = self.adj if same else t(host.raw_adj)
        self.raw_deg = t(host.degrees().astype(np.int64))
        self.n_bit_words = (host.adj.shape[0] + 31) // 32 + 1
        self.d1_bits = torch.zeros(self.n_bit_words, dtype=torch.int32, device=self.device)

    def reverse_entries(self):
        """rev[e] = index of the entry (v -> u) for e = (u -> v) (gg_reverse_entries; device int32 [nnz], cached), or None
        when the walk CSR is not symmetric -- the tree builder then stays top-down (csrc/bfs.cu)."""
        import torch
        if not hasattr(self, "_rev"):
            nnz = int(self.host.adj.shape[0])
            rev = torch.empty(max(nnz, 1), dtype=torch.int32, device=self.device)
            missing = torch.zeros(1, dtype=torch.int32, device=self.device)
            st = torch.cuda.current_stream(self.device).cuda_stream
            _cabi.check(_cabi.lib().gg_reverse_entries(self.n_node, nnz, self.indptr.data_ptr(), self.adj.data_ptr(),
                                                       rev.data_ptr(), missing.data_ptr(), st), "gg_reverse_entries")
            self._rev = rev if int(missing.item()) == 0 else None
        return self._rev

    def entry_mult(self):
        """mult[e] = the number of times adj[e] occurs in the raw list graph[u] of the entry's row u: n_ca of the walk-CSR
        entry e = (c -> a), duplicates counted (device int32 [nnz], cached; computed once per graph on the host, like the
        walk CSR itself).  p_true(a | c) = mult[e] / |graph[c]| (DESIGN.md section 5.8)."""
        import torch
        if not hasattr(self, "_mult"):
            h, n = self.host, self.n_node
            key_raw = np.repeat(np.arange(n, dtype=np.int64), np.diff(h.raw_indptr)) * n + h.raw_adj
            key = np.repeat(np.arange(n, dtype=np.int64), np.diff(h.indptr)) * n + h.adj
            u, cnt = np.unique(key_raw, return_counts=True)
            mult = cnt[np.searchsorted(u, key)].astype(np.int32) if key.shape[0] else np.zeros(0, np.int32)
            self._mult = torch.from_numpy(np.concatenate([mult, np.zeros(1, np.int32)])).to(self.device)[:max(key.shape[0], 1)]
        return self._mult

    def hub_tiles(self, threshold, item_cap=HUB_ITEM_CAP):
        """Work list of gg_hub_scores, target-major: the walk-CSR entries e = (u -> v) of the nodes u whose degree is
        >= threshold, stably sorted by target v, as pairs (u, e) (device int32 [n_entries, 2]), and the work items
        (v, first pair, count, 0) (device int32 [n_items, 4]) that cut each target's run of pairs into pieces of at most
        `item_cap`.  Returns (items, pairs, n_items, n_entries).  Built on the device; static per graph; cached."""
        import torch
        key = (int(threshold), int(item_cap))
        if getattr(self, "_hub_key", None) != key:
            dev, i64 = self.device, torch.int64
            deg_h = np.diff(self.host.indptr)
            hubs_h = np.flatnonzero(deg_h >= threshold)
            n_entries = int(deg_h[hubs_h].sum())
            items = torch.zeros((0, 4), dtype=torch.int32, device=dev)
            pairs = torch.zeros((0, 2), dtype=torch.int32, device=dev)
            if n_entries:
                hubs = torch.from_numpy(hubs_h).to(dev)
                cnt = self.indptr[hubs + 1] - self.indptr[hubs]
                src = torch.repeat_interleave(hubs, cnt, output_size=n_entries)                  # hub-major order
                run0 = torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt, output_size=n_entries)
                e = self.indptr[src] + (torch.arange(n_entries, dtype=i64, device=dev) - run0)
                tgt, order = torch.sort(self.adj[e], stable=True)
                pairs = torch.stack([src[order], e[order]], 1).to(torch.int32).contiguous()
                v, run = torch.unique_consecutive(tgt, return_counts=True)
                pieces = (run + item_cap - 1) // item_cap
                n_items = int(pieces.sum().item())
                p0 = torch.cumsum(pieces, 0) - pieces                                            # first piece of each run
                r = torch.repeat_interleave(torch.arange(v.shape[0], dtype=i64, device=dev), pieces, output_size=n_items)
                k = torch.arange(n_items, dtype=i64, device=dev) - p0[r]                         # piece index in its run
                first = (torch.cumsum(run, 0) - run)[r] + k * item_cap
                count = torch.clamp(run[r] - k * item_cap, max=item_cap)
                items = torch.stack([v[r].to(i64), first, count, torch.zeros_like(first)], 1).to(torch.int32).contiguous()
            self._hub_key = key
            self._hub = (items, pairs, int(items.shape[0]), n_entries)
            if not hasattr(self, "edge_score"):
                self.edge_score = torch.empty(self.host.adj.shape[0] + 4, dtype=torch.float32, device=self.device)[:max(self.host.adj.shape[0], 1)]
        return self._hub

    def reset_tree_mutations(self):
        """Forget every father removal (== reloading the reference's tree cache)."""
        self.d1_bits.zero_()
