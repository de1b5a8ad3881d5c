"""Host driver of K1, the graph-softmax walk (csrc/walk.cu), and of the tree builder.

Batched replacement for ``GraphGAN.sample`` (reference src/GraphGAN/graph_gan.py:225-270):
instead of one Python call per root it runs every walk of a batch of roots in one kernel
launch.  Torch tensors are used purely as device-memory containers; all computation happens
in libgraphgan_b200.so through the C ABI (include/graphgan_b200.h).
"""
import ctypes as C
import os

import numpy as np

from . import _cabi
from ._cabi import ptr

RNG_PHILOX, RNG_STREAM = 0, 1
NOTRUN, DONE, VOID, SKIPPED = 0, 1, 2, 3
CNT = dict(steps=0, sum_l=1, accepted=2, ok_roots=3, path_overflow=4, raw_steps=5, raw_sum_l=6, stream_used=7,
           rows_gathered=8, cyc_enum=9, cyc_score=10, cyc_choose=11, cyc_step0=12, cyc_step1=13, cyc_step2p=14, cyc_walk=15)


LD_MAX = 512   # widest row stride the kernels accept (gg::ld_supported in csrc/gg_common.cuh)


def round_up(x, m):
    return (x + m - 1) // m * m


def pad_embedding(emb, device=None):
    """float64/32 [N, d] -> fp32 [N, ld] device tensor, ld = 32 * 2^k >= d (32, 64, 128, 256 or 512), zero padded
    (the tf fp32 variable of generator.py:11-14 in the HBM layout of DESIGN.md section 2)."""
    import torch
    e = emb.float() if isinstance(emb, torch.Tensor) else torch.as_tensor(np.asarray(emb, np.float64).astype(np.float32))
    n, d = e.shape
    if d > LD_MAX:
        raise ValueError("n_emb = %d is not supported: at most %d (the kernels are instantiated for row strides 32, 64, 128, "
                         "256 and 512)" % (d, LD_MAX))
    ld = 32
    while ld < d:      # zero columns add exactly +0 to every canonical dot, so the amount of padding is invisible
        ld *= 2
    out = torch.zeros((n, ld), dtype=torch.float32, device=device if device is not None else e.device)
    out[:, :d] = e.to(out.device)
    return out


class TreeBatch:
    """BFS trees of a batch of roots (``trees[root]`` of graph_gan.py:84-108) as one bit per walk-CSR entry:
    bit e of row k <=> adj[e] is a child of entry e's source node in the tree of roots[k] (csrc/bfs.cu)."""

    def __init__(self, roots, tree_bits, graph=None):
        self.roots = roots            # device int32 [R]
        self.tree_bits = tree_bits    # device int32 [R, tree_words] (bit patterns)
        self.graph = graph

    def slice(self, lo, hi):
        return TreeBatch(self.roots[lo:hi].contiguous(), self.tree_bits[lo:hi].contiguous(), self.graph)

    def select(self, idx):
        return TreeBatch(self.roots[idx].contiguous(), self.tree_bits[idx].contiguous(), self.graph)

    def parent_arrays(self, rows=None):
        """int32 [R', N] parent arrays (root and unreachable nodes: -1) of all / the selected rows -- the form the
        oracle and host-side consumers use; expanded on the device by gg_tree_parent."""
        import torch
        g, lib = self.graph, _cabi.lib()
        bits = self.tree_bits if rows is None else self.tree_bits[rows].contiguous()
        roots = self.roots if rows is None else self.roots[rows].contiguous()
        R = int(bits.shape[0])
        out = torch.empty((R, g.n_node), dtype=torch.int32, device=bits.device)
        st = torch.cuda.current_stream(bits.device).cuda_stream
        for lo in range(0, R, 32768):
            hi = min(R, lo + 32768)
            _cabi.check(lib.gg_tree_parent(g.n_node, ptr(g.indptr), ptr(g.adj), hi - lo, ptr(roots[lo:hi]), ptr(bits[lo:hi]),
                                           int(bits.shape[1]), ptr(out[lo:hi]), st), "gg_tree_parent")
        return out


class WalkOutput:
    """Device-side results of one pass (everything stays on the GPU until asked for)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def counters_host(self):
        c = self.counters.cpu().numpy().astype(np.uint64)
        return {k: int(c[i]) for k, i in CNT.items()}


class WalkPlan:
    """Everything about a pass that does not depend on the embeddings: the walk list of a root batch
    (walk_ptr), the root-CDF offsets, and the output buffers (reused by every run with this plan)."""

    def __init__(self, sampler, trees, sample_num, for_d, max_path):
        import torch
        dev, g = sampler.device, sampler.g
        R = int(trees.roots.shape[0])
        self.trees, self.for_d, self.max_path, self.n_roots = trees, bool(for_d), int(max_path), R
        if isinstance(sample_num, int):
            self.walk_ptr = torch.arange(R + 1, dtype=torch.int64, device=dev) * sample_num
            self.n_walks = R * sample_num
        else:
            self.walk_ptr = torch.zeros(R + 1, dtype=torch.int64, device=dev)
            self.walk_ptr[1:] = torch.cumsum(sample_num.to(torch.int64), 0)      # plumbing: prefix of sample_num
            self.n_walks = int(self.walk_ptr[-1].item())
        nw = self.walk_ptr[1:] - self.walk_ptr[:-1]
        self.walk_slot = torch.repeat_interleave(torch.arange(R, dtype=torch.int32, device=dev), nw,
                                                 output_size=self.n_walks) if self.n_walks else None
        r = trees.roots.long()
        self.rq_ptr = torch.zeros(R + 1, dtype=torch.int64, device=dev)
        self.rq_ptr[1:] = torch.cumsum(g.indptr[r + 1] - g.indptr[r], 0)       # prefix of the roots' walk degrees
        self.nq = int(self.rq_ptr[-1].item())
        nq = max(self.nq, 1)
        self.root_q = torch.empty(nq, dtype=torch.float64, device=dev)
        self.root_sc = torch.empty(nq, dtype=torch.float32, device=dev)
        self._s1 = None
        self._order = None
        W = max(self.n_walks, 1)
        i32 = lambda *s: torch.empty(s, dtype=torch.int32, device=dev)
        self.samples, self.status, self.first_edge, self.wsteps, self.wsuml = i32(W), i32(W), i32(W), i32(W), i32(W)
        self.paths = i32(W, max_path) if max_path > 0 else None
        self.path_len = i32(W) if max_path > 0 else None
        self.root_ok = torch.zeros(max(R, 1), dtype=torch.int32, device=dev)
        self.counters = torch.zeros(16, dtype=torch.int64, device=dev)
        self.row_ptr = torch.empty(R + 1, dtype=torch.int64, device=dev)
        self.n_rows = torch.zeros(1, dtype=torch.int64, device=dev)
        self.rows = [i32(max(2 * self.n_walks, 1)) for _ in range(3)] if for_d else None


    def start_order(self, sampler):
        """Order in which walk_kernel starts the walks: roots whose neighbourhood holds the largest hub first
        (a walk that steps onto a 10 k-neighbour node costs ~100x a median one; started last it would be the
        tail of the launch), walks of one root kept together (they share the tree row in L2).  Static per
        plan; plumbing only (one gather, one segment max, one sort)."""
        if self._order is None and self.n_walks > 0 and self.nq > 0:
            torch, g, dev = sampler.torch, sampler.g, sampler.device
            R = self.n_roots
            deg_r = self.rq_ptr[1:] - self.rq_ptr[:-1]
            slot = torch.repeat_interleave(torch.arange(R, dtype=torch.int64, device=dev), deg_r, output_size=self.nq)
            ent = g.indptr[self.trees.roots.long()[slot]] + (torch.arange(self.nq, dtype=torch.int64, device=dev) - self.rq_ptr[slot])
            c = g.adj[ent].long()
            key = torch.zeros(R, dtype=torch.int64, device=dev).scatter_reduce_(0, slot, g.indptr[c + 1] - g.indptr[c], "amax")
            perm = torch.argsort(key, descending=True, stable=True)
            nw = (self.walk_ptr[1:] - self.walk_ptr[:-1])[perm]
            first = torch.cumsum(nw, 0) - nw                                  # position of each root's first walk in the order
            base = torch.repeat_interleave(self.walk_ptr[:-1][perm] - first, nw, output_size=self.n_walks)
            self._order = (base + torch.arange(self.n_walks, dtype=torch.int64, device=dev)).to(torch.int32)
        return self._order

    def flat_buffer(self, sampler):
        """scratch of the level-synchronous steps (csrc/walk.cu: flat_*_kernel), sized by the library"""
        key = (sampler.flat_steps, sampler.hub_threshold)
        if getattr(self, "_flat_key", None) != key:
            nbytes = C.c_int64(0)
            _cabi.check(sampler.lib.gg_walk_flat_bytes(self.n_walks, sampler.hub_threshold, sampler.flat_steps, C.byref(nbytes)),
                        "gg_walk_flat_bytes")
            self._flat = sampler.torch.empty(max(nbytes.value, 16), dtype=sampler.torch.uint8, device=sampler.device)
            self._flat_key = key
        return self._flat

    def depth1_buffers(self, sampler):
        """Static layout of the depth-1 CDF cache (csrc/walk.cu: step1_cdf_kernel): one slice of degree(child) + 1
        entries per (root, neighbour) pair.  Built on first use (plumbing: gathers + one cumsum)."""
        if self._s1 is None:
            torch, g, dev = sampler.torch, sampler.g, sampler.device
            deg_r = self.rq_ptr[1:] - self.rq_ptr[:-1]
            slot = torch.repeat_interleave(torch.arange(self.n_roots, dtype=torch.int32, device=dev), deg_r, output_size=self.nq)
            r = self.trees.roots.long()[slot.long()]
            ent = g.indptr[r] + (torch.arange(self.nq, dtype=torch.int64, device=dev) - self.rq_ptr[slot.long()])
            c = g.adj[ent].long()
            ptr_ = torch.zeros(self.nq + 1, dtype=torch.int64, device=dev)
            ptr_[1:] = torch.cumsum(g.indptr[c + 1] - g.indptr[c] + 1, 0)
            total = max(int(ptr_[-1].item()), 1)
            i32 = lambda k: torch.empty(max(k, 1), dtype=torch.int32, device=dev)
            order = torch.argsort(g.indptr[c + 1] - g.indptr[c], descending=True, stable=True).to(torch.int32)
            self._s1 = dict(slot=slot, ptr=ptr_, cnt=i32(self.nq), n=i32(self.nq), ids=i32(total), order=order,
                            q=torch.empty(total, dtype=torch.float64, device=dev), first=i32(self.n_walks))
        return self._s1


def _gref_window(window):
    """the window of expected_g_grad / expected_g_moments: config.window_size's range, 1 .. 8"""
    window = int(window)
    if not 1 <= window <= 8:
        raise ValueError("window must be 1 .. 8, got %d" % window)
    return window


class WalkSampler:
    def __init__(self, graph, hub_threshold=128, depth1=True, hub_first=True, tma=True):
        import torch
        self.torch = torch
        self.g = graph
        self.device = graph.device
        self.lib = _cabi.lib()
        self.max_cand = graph.max_deg + 1
        self.hub_threshold = int(hub_threshold)   # 0 disables both per-pass reuses (pure on-demand path)
        # one CDF per (root, depth-1 child) pair that occurs (needs reuse): the walks of a root that pick the same child
        # share its candidate list (5.5x fewer neighbour probes at step 1 on C3); the builder kernel pulls the pairs
        # from a queue, largest lists first (hub_first), because a 13.8k-entry hub list occupies one warp for ~0.5-1 ms
        self.depth1 = bool(depth1)
        self.tma = bool(tma)                      # cp.async.bulk staging of hub lists (csrc/walk.cu); False = plain loads (A/B)
        self.hub_first = bool(hub_first)          # start order of the walks (WalkPlan.start_order); results do not depend on it
        nbytes = C.c_int64(0)
        _cabi.check(self.lib.gg_walk_scratch_bytes(self.max_cand, C.byref(nbytes)), "gg_walk_scratch_bytes")
        self.scratch = torch.empty(max(nbytes.value, 16), dtype=torch.uint8, device=self.device)
        self.work_counter = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._bfs_scratch = None
        # tree builder: direction-optimising BFS (csrc/bfs.cu).  < 0: library default ratio, 0: top-down + small sorted
        # bottom-up levels only; the trees are identical in every mode (tests/test_walk_gpu.py)
        self.bfs_bottom_up_ratio = float(os.environ.get("GG_BFS_BU_RATIO", "-1"))
        self.bfs_flags = 0
        # level-synchronous walk steps (csrc/walk.cu: flat_*_kernel) for steps 1..flat_steps; 0 = persistent kernel only
        self.flat_steps = int(os.environ.get("GG_FLAT_STEPS", "4"))

    def _stream(self):
        return self.torch.cuda.current_stream(self.device).cuda_stream

    # ------------------------------------------------------------------ trees
    def build_trees(self, roots):
        """construct_trees (graph_gan.py:84-108) for ``roots`` on the GPU -> TreeBatch."""
        torch = self.torch
        roots_d = roots if isinstance(roots, torch.Tensor) else torch.as_tensor(np.asarray(roots, np.int32)).to(self.device)
        R, N = int(roots_d.shape[0]), self.g.n_node
        nnz = int(self.g.adj.shape[0])
        words = C.c_int64(0)
        _cabi.check(self.lib.gg_tree_words(nnz, C.byref(words)), "gg_tree_words")
        tree_bits = torch.empty((R, words.value), dtype=torch.int32, device=self.device)
        if self._bfs_scratch is None:
            nbytes = C.c_int64(0)
            _cabi.check(self.lib.gg_bfs_scratch_bytes(N, int(self.g.adj.shape[0]), C.byref(nbytes)), "gg_bfs_scratch_bytes")
            self._bfs_scratch = torch.empty(max(nbytes.value, 16), dtype=torch.uint8, device=self.device)
        rev = self.g.reverse_entries() if self.bfs_bottom_up_ratio != 0.0 else None
        _cabi.check(self.lib.gg_bfs_build_ex(N, nnz, ptr(self.g.indptr), ptr(self.g.adj), ptr(rev) if rev is not None else None,
                                             R, ptr(roots_d), ptr(tree_bits), words.value, ptr(self._bfs_scratch),
                                             self._bfs_scratch.numel(), float(self.bfs_bottom_up_ratio), int(self.bfs_flags),
                                             self._stream()),
                    "gg_bfs_build_ex")
        return TreeBatch(roots_d, tree_bits, self.g)

    # ------------------------------------------------------------------ K1
    def plan(self, trees, sample_num, for_d, max_path=0):
        return WalkPlan(self, trees, sample_num, for_d, max_path)

    def _desc(self, emb, bias, plan, *, seed, pass_tag, update_ratio, rng_mode, stream, reuse, phase_mask=0):
        torch = self.torch
        assert emb.dtype == torch.float32 and emb.is_contiguous() and bias.dtype == torch.float32
        t, d = plan.trees, _cabi.WalkDesc()
        d.n_node, d.ld = self.g.n_node, int(emb.shape[1])
        d.emb, d.bias, d.indptr, d.adj = ptr(emb), ptr(bias), ptr(self.g.indptr), ptr(self.g.adj)
        d.n_roots, d.roots, d.walk_ptr, d.n_walks = plan.n_roots, ptr(t.roots), ptr(plan.walk_ptr), plan.n_walks
        d.tree_bits, d.tree_words = ptr(t.tree_bits), int(t.tree_bits.shape[1])
        d.for_d, d.rng_mode, d.d1_bits = int(plan.for_d), rng_mode, ptr(self.g.d1_bits)
        d.seed, d.pass_tag, d.max_path = seed, pass_tag, plan.max_path
        d.stream, d.n_stream = (ptr(stream), int(stream.numel())) if stream is not None else (None, 0)
        d.update_ratio, d.max_cand, d.phase_mask = float(update_ratio), self.max_cand, int(phase_mask)
        d.no_tma = 0 if self.tma else 1
        d.samples, d.status, d.first_edge, d.wsteps, d.wsuml = (ptr(plan.samples), ptr(plan.status), ptr(plan.first_edge),
                                                                 ptr(plan.wsteps), ptr(plan.wsuml))
        d.paths, d.path_len, d.counters = ptr(plan.paths), ptr(plan.path_len), ptr(plan.counters)
        d.scratch, d.scratch_bytes, d.work_counter = ptr(self.scratch), self.scratch.numel(), ptr(self.work_counter)
        d.rq_ptr, d.walk_slot = ptr(plan.rq_ptr), ptr(plan.walk_slot)
        if self.hub_first and rng_mode == RNG_PHILOX:
            d.walk_order = ptr(plan.start_order(self))
        if reuse:
            self.g.hub_tiles(self.hub_threshold)
            d.edge_score, d.hub_threshold, d.root_q = ptr(self.g.edge_score), self.hub_threshold, ptr(plan.root_q)
            if self.depth1 and rng_mode == RNG_PHILOX and plan.nq > 0 and plan.n_walks > 0:
                b = plan.depth1_buffers(self)
                d.s1_nq, d.s1_slot, d.s1_ptr, d.s1_cnt, d.s1_n = plan.nq, ptr(b["slot"]), ptr(b["ptr"]), ptr(b["cnt"]), ptr(b["n"])
                d.s1_q, d.s1_ids, d.first_idx = ptr(b["q"]), ptr(b["ids"]), ptr(b["first"])
                if self.hub_first:
                    d.s1_order = ptr(b["order"])
                if self.flat_steps > 0:
                    buf = plan.flat_buffer(self)
                    d.flat_buf, d.flat_bytes, d.flat_steps = ptr(buf), buf.numel(), self.flat_steps
        return d

    def precompute(self, emb, bias, plan, desc=None):
        """Per-pass reuse (csrc/hub.cu): hub adjacency scores, then one CDF per root.  Depends on the
        embeddings, so it belongs to every pass; `run` calls it unless told otherwise."""
        d = desc if desc is not None else self._desc(emb, bias, plan, seed=0, pass_tag=0, update_ratio=1.0,
                                                     rng_mode=RNG_PHILOX, stream=None, reuse=True)
        items, pairs, n_items, _ = self.g.hub_tiles(self.hub_threshold)
        st = self._stream()
        _cabi.check(self.lib.gg_hub_scores(n_items, ptr(items), ptr(pairs), ptr(emb), ptr(bias), int(emb.shape[1]),
                                           ptr(self.g.edge_score), st), "gg_hub_scores")
        _cabi.check(self.lib.gg_root_cdf(C.byref(d), ptr(plan.root_sc), ptr(plan.root_q), st), "gg_root_cdf")

    def run(self, emb, bias, trees, sample_num, for_d, *, seed=0, pass_tag=0, update_ratio=1.0, max_path=0,
            rng_mode=RNG_PHILOX, stream=None, finalize=True, plan=None, reuse=None, precompute=True, phase_mask=0, zero_counters=True):
        """All walks of one pass.  ``sample_num``: int (G mode, config.n_sample_gen) or device int64 [R]
        (D mode, len(graph[root])).  ``reuse`` (default: hub_threshold > 0) turns the per-pass score / CDF
        reuse on; results are bit-identical either way."""
        if plan is None:
            plan = self.plan(trees, sample_num, for_d, max_path)
        reuse = (self.hub_threshold > 0) if reuse is None else bool(reuse)
        if zero_counters:
            plan.counters.zero_()
        d = self._desc(emb, bias, plan, seed=seed, pass_tag=pass_tag, update_ratio=update_ratio, rng_mode=rng_mode,
                       stream=stream, reuse=reuse, phase_mask=phase_mask)
        if reuse and precompute:
            self.precompute(emb, bias, plan, d)
        _cabi.check(self.lib.gg_walk_sample(C.byref(d), self._stream()), "gg_walk_sample")
        out = WalkOutput(walk_ptr=plan.walk_ptr, n_walks=plan.n_walks, n_roots=plan.n_roots, for_d=plan.for_d,
                         max_path=plan.max_path, samples=plan.samples, status=plan.status, first_edge=plan.first_edge,
                         wsteps=plan.wsteps, wsuml=plan.wsuml, paths=plan.paths, path_len=plan.path_len,
                         root_ok=plan.root_ok, counters=plan.counters, roots=trees.roots, plan=plan)
        if finalize:
            self.finalize(out)
        return out

    # ------------------------------------------------------------------ exact generator distribution
    def distribution(self, emb, bias, trees, *, reuse=None, max_scratch_bytes=None, counters=None):
        """G(v | root) for every root of ``trees``: the exact probability that one G-mode walk (graph_gan.py:225-270)
        from the root stops at v, under the current father-removal bits (csrc/gdist.cu, DESIGN.md section 5.1).
        Returns device fp64 ``dist [R, N]`` and int32 ``root_ok [R]`` (0: the root's walks void; its row is all zero).
        ``reuse`` (default: hub_threshold > 0) scores hub lists from the per-pass cache -- the same bits either way.  The
        roots run in chunks whose scratch stays within ``max_scratch_bytes`` (default 2 GiB, env GG_GDIST_SCRATCH);
        ``counters`` (optional device int64 [16]) receives the embedding rows fetched in slot rows_gathered."""
        torch = self.torch
        R, N = int(trees.roots.shape[0]), self.g.n_node
        dist = torch.empty((R, N), dtype=torch.float64, device=self.device)
        root_ok = torch.empty(R, dtype=torch.int32, device=self.device)
        for _ in self._distribution_chunks(emb, bias, trees, reuse, max_scratch_bytes, counters, dist, root_ok):
            pass
        return dist, root_ok

    def d_distribution(self, emb, bias, trees, *, reuse=None, max_scratch_bytes=None):
        """The D-mode walk law (csrc/gdist.cu, DESIGN.md section 5.7): for every root of ``trees``, P_D(v | root), the
        exact probability that one D-mode walk (graph_gan.py:225-270, for_d=True) stops at v, and p_void, the probability
        that it lands on a depth-1 leaf and so voids the root's D pass (graph_gan.py:255-257).  A D walk removes the root
        from every depth-1 list whatever the father-removal bits hold, so the law does not depend on them, and the walks
        of one root are independent draws from it.  Returns device fp64 ``P_D [R, N]``, fp64 ``p_void [R]`` and int32
        ``root_ok [R]`` (1 iff the root has children; sum_v P_D = 1 - p_void then).  ``reuse`` and the chunking as for
        ``distribution``."""
        torch = self.torch
        R, N = int(trees.roots.shape[0]), self.g.n_node
        dist = torch.empty((R, N), dtype=torch.float64, device=self.device)
        root_ok = torch.empty(R, dtype=torch.int32, device=self.device)
        p_void = torch.empty(R, dtype=torch.float64, device=self.device)
        for _ in self._distribution_chunks(emb, bias, trees, reuse, max_scratch_bytes, None, dist, root_ok, p_void=p_void):
            pass
        return dist, p_void, root_ok

    def _law_desc(self, emb, bias, trees, reuse, counters):
        """the descriptor of the generator's law for gg_generator_dist / gg_game_value_grad (the per-chunk fields n_roots,
        roots, tree_bits are the caller's); with ``reuse``, the hub scores are refreshed first"""
        g = self.g
        d = _cabi.WalkDesc()
        d.n_node, d.ld = g.n_node, int(emb.shape[1])
        d.emb, d.bias, d.indptr, d.adj = ptr(emb), ptr(bias), ptr(g.indptr), ptr(g.adj)
        d.tree_words, d.d1_bits, d.counters = int(trees.tree_bits.shape[1]), ptr(g.d1_bits), ptr(counters)
        if reuse:
            items, pairs, n_items, _ = g.hub_tiles(self.hub_threshold)
            _cabi.check(self.lib.gg_hub_scores(n_items, ptr(items), ptr(pairs), ptr(emb), ptr(bias), int(emb.shape[1]),
                                               ptr(g.edge_score), self._stream()), "gg_hub_scores")
            d.edge_score, d.hub_threshold = ptr(g.edge_score), self.hub_threshold
        return d

    def _distribution_chunks(self, emb, bias, trees, reuse, max_scratch_bytes, counters, dist=None, root_ok=None,
                             extra_bytes=None, p_void=None, d_mode=False):
        """gg_generator_dist over the roots of ``trees`` in chunks whose scratch fits the budget; yields (lo, hi, dist rows,
        root_ok rows) per chunk.  The rows go to dist[lo:hi] / root_ok[lo:hi] when those are given, else to one chunk-sized
        buffer that the next chunk overwrites.  ``extra_bytes(k)``: the caller's own scratch for a chunk of k roots, counted
        against the same budget (None: nothing).  With ``d_mode`` (implied by ``p_void``), gg_generator_dist_d instead:
        the D-mode law, and each chunk yields (lo, hi, dist rows, root_ok rows, p_void rows), the p_void rows going to
        p_void[lo:hi] when given, else to a chunk-sized buffer."""
        torch, g = self.torch, self.g
        R, N, nnz = int(trees.roots.shape[0]), g.n_node, int(g.adj.shape[0])
        if R == 0:
            return
        assert emb.dtype == torch.float32 and emb.is_contiguous() and bias.dtype == torch.float32
        reuse = (self.hub_threshold > 0) if reuse is None else bool(reuse)
        scratch_bytes = lambda k: self._scratch_size("gg_generator_dist_scratch_bytes", N, nnz, k)
        per_root = scratch_bytes(1) + (extra_bytes(1) if extra_bytes is not None else 0)
        chunk = self._chunk_size(R, N, per_root, max_scratch_bytes)
        scratch = torch.empty(max(scratch_bytes(chunk), 16), dtype=torch.uint8, device=self.device)
        if dist is None:
            dist = torch.empty((chunk, N), dtype=torch.float64, device=self.device)
            root_ok = torch.empty(chunk, dtype=torch.int32, device=self.device)
            rows = lambda lo, hi: (dist[:hi - lo], root_ok[:hi - lo])
        else:
            rows = lambda lo, hi: (dist[lo:hi], root_ok[lo:hi])
        d_mode = d_mode or p_void is not None
        if d_mode and p_void is None:
            p_void = torch.empty(chunk, dtype=torch.float64, device=self.device)
            pv_rows = lambda lo, hi: p_void[:hi - lo]
        else:
            pv_rows = lambda lo, hi: p_void[lo:hi]
        d = self._law_desc(emb, bias, trees, reuse, counters)
        st = self._stream()
        for lo in range(0, R, chunk):
            hi = min(R, lo + chunk)
            dr, okr = rows(lo, hi)
            d.n_roots, d.roots, d.tree_bits = hi - lo, ptr(trees.roots[lo:hi]), ptr(trees.tree_bits[lo:hi])
            if d_mode:
                pvr = pv_rows(lo, hi)
                _cabi.check(self.lib.gg_generator_dist_d(C.byref(d), ptr(dr), ptr(pvr), ptr(okr), ptr(scratch),
                                                         scratch.numel(), st), "gg_generator_dist_d")
                yield lo, hi, dr, okr, pvr
                continue
            _cabi.check(self.lib.gg_generator_dist(C.byref(d), ptr(dr), ptr(okr), ptr(scratch), scratch.numel(), st),
                        "gg_generator_dist")
            yield lo, hi, dr, okr

    # ------------------------------------------------------------------ game value V(G, D)
    def game_value(self, g_emb, g_bias, d_emb, d_bias, trees, *, max_scratch_bytes=None, reuse=None):
        """The GraphGAN game value per root (Wang et al., AAAI-18, Eq. 1), exactly: V_c = pos_c + neg_c with
        pos_c = E_{v ~ p_true(.|c)} log D(v, c), the mean over graph[c] (raw adjacency: duplicates and self-loops count),
        and neg_c = E_{v ~ G(.|c)} log(1 - D(v, c)) under the generator's exact G-mode law (``distribution``, current
        father-removal bits).  D(v, c) = sigmoid(s), s = the discriminator's fp32 score; log D = -bce(s, 1) and
        log(1 - D) = -bce(s, 0) in fp64 (csrc/value.cu, DESIGN.md section 5.2).
        ``g_emb, g_bias``: the generator's padded rows and bias; ``d_emb, d_bias``: the discriminator's.
        Returns device (pos fp64 [R], neg fp64 [R], ok int32 [R]); ok = 0 (pos = neg = 0) for a root without neighbours
        or whose G walks void.  The roots run in the chunks of ``distribution`` (same budget rule): G(. | c) exists for
        one chunk at a time.  The bits do not depend on the chunking or on the order of the roots."""
        torch, g = self.torch, self.g
        assert d_emb.dtype == torch.float32 and d_emb.is_contiguous() and d_bias.dtype == torch.float32
        assert int(d_emb.shape[0]) == g.n_node and int(d_bias.shape[0]) == g.n_node
        R, N = int(trees.roots.shape[0]), g.n_node
        pos = torch.zeros(R, dtype=torch.float64, device=self.device)
        neg = torch.zeros(R, dtype=torch.float64, device=self.device)
        ok = torch.zeros(R, dtype=torch.int32, device=self.device)
        st, scratch = self._stream(), None
        for lo, hi, dist, root_ok in self._distribution_chunks(g_emb, g_bias, trees, reuse, max_scratch_bytes, None):
            nb = self._scratch_size("gg_game_value_scratch_bytes", N, hi - lo)
            if scratch is None or scratch.numel() < nb:
                scratch = torch.empty(max(nb, 16), dtype=torch.uint8, device=self.device)
            _cabi.check(self.lib.gg_game_value(N, int(d_emb.shape[1]), ptr(d_emb), ptr(d_bias), ptr(g.raw_indptr),
                                               ptr(g.raw_adj), hi - lo, ptr(trees.roots[lo:hi]), ptr(dist), ptr(root_ok),
                                               ptr(pos[lo:hi]), ptr(neg[lo:hi]), ptr(ok[lo:hi]), ptr(scratch),
                                               scratch.numel(), st), "gg_game_value")
        return pos, neg, ok

    # ------------------------------------------------------------------ generator gradient of V(G, D)
    def game_value_grad(self, g_emb, g_bias, d_emb, d_bias, trees, *, max_scratch_bytes=None, reuse=None):
        """``game_value`` and the exact gradient of sum_{ok c} V_c with respect to the generator's parameters (csrc/
        value_grad.cu, DESIGN.md section 5.3): the policy gradient sum_v G(v | c) grad log G(v | c) log(1 - D(v, c)) of
        the paper, evaluated exactly over the BFS trees under the step law of ``distribution``.
        Returns device (pos fp64 [R], neg fp64 [R], ok int32 [R]) in the order of ``trees`` -- the bits of ``game_value``
        -- and (grad_emb fp64 [N, ld], grad_bias fp64 [N]) for the padded rows ``g_emb`` (pad columns exactly 0) and
        ``g_bias``.  The roots are taken in ascending id order (stable for duplicates), in chunks under the budget rule of
        ``distribution`` (``max_scratch_bytes``, default 2 GiB or env GG_GDIST_SCRATCH), each coordinate one fp64 chain
        over the roots: the bits do not depend on the chunking, the order of the roots or the call."""
        torch, g = self.torch, self.g
        assert g_emb.dtype == torch.float32 and g_emb.is_contiguous() and g_bias.dtype == torch.float32
        assert d_emb.dtype == torch.float32 and d_emb.is_contiguous() and d_bias.dtype == torch.float32
        assert d_emb.shape == g_emb.shape and int(d_bias.shape[0]) == g.n_node and int(g_emb.shape[0]) == g.n_node
        R, N, nnz = int(trees.roots.shape[0]), g.n_node, int(g.adj.shape[0])
        pos = torch.zeros(R, dtype=torch.float64, device=self.device)
        neg = torch.zeros(R, dtype=torch.float64, device=self.device)
        ok = torch.zeros(R, dtype=torch.int32, device=self.device)
        grad_emb = torch.zeros(tuple(g_emb.shape), dtype=torch.float64, device=self.device)
        grad_bias = torch.zeros(N, dtype=torch.float64, device=self.device)
        if R == 0:
            return pos, neg, ok, grad_emb, grad_bias
        order, st_trees = self._by_root_id(trees)
        reuse = (self.hub_threshold > 0) if reuse is None else bool(reuse)
        scratch_bytes = lambda k: self._scratch_size("gg_game_value_grad_scratch_bytes", N, nnz, k)
        chunk = self._chunk_size(R, N, scratch_bytes(1), max_scratch_bytes)
        scratch = torch.empty(max(scratch_bytes(chunk), 16), dtype=torch.uint8, device=self.device)
        sp, sn, so = (torch.zeros_like(x) for x in (pos, neg, ok))
        d = self._law_desc(g_emb, g_bias, st_trees, reuse, None)
        st = self._stream()
        for lo in range(0, R, chunk):
            hi = min(R, lo + chunk)
            d.n_roots, d.roots, d.tree_bits = hi - lo, ptr(st_trees.roots[lo:hi]), ptr(st_trees.tree_bits[lo:hi])
            _cabi.check(self.lib.gg_game_value_grad(C.byref(d), ptr(d_emb), ptr(d_bias), ptr(g.raw_indptr), ptr(g.raw_adj),
                                                    ptr(sp[lo:hi]), ptr(sn[lo:hi]), ptr(so[lo:hi]), ptr(grad_emb),
                                                    ptr(grad_bias), ptr(scratch), scratch.numel(), st), "gg_game_value_grad")
        pos[order], neg[order], ok[order] = sp, sn, so
        return pos, neg, ok, grad_emb, grad_bias

    # ------------------------------------------------------------------ discriminator gradient of V(G, D)
    @staticmethod
    def scratch_budget(max_scratch_bytes=None):
        """The device bytes the exact-game entry points may hold at once: ``max_scratch_bytes``, else env GG_GDIST_SCRATCH,
        else 2 GiB."""
        return int(max_scratch_bytes if max_scratch_bytes is not None else os.environ.get("GG_GDIST_SCRATCH", 2 << 30))

    def _chunk_size(self, R, N, per_root, max_scratch_bytes):
        """roots per chunk of the exact-game entry points: as many as the scratch budget holds at ``per_root`` bytes
        each, at most R, and fewer than 2^31 / N (the [chunk, N] planes are indexed in int32)"""
        return max(1, min(R, self.scratch_budget(max_scratch_bytes) // max(per_root, 1), ((1 << 31) - 1) // max(N, 1)))

    def _scratch_size(self, fn, *args):
        """the bytes the scratch-size entry point ``fn`` (its name) gives for ``args``"""
        nb = C.c_int64(0)
        _cabi.check(getattr(self.lib, fn)(*args, C.byref(nb)), fn)
        return nb.value

    def _by_root_id(self, trees):
        """(order, sorted trees): the rows of ``trees`` in ascending root id order (stable for duplicates), so that the
        bits of a sum over roots do not depend on their order; the trees are not copied when already sorted"""
        torch = self.torch
        R = int(trees.roots.shape[0])
        order = torch.argsort(trees.roots.long(), stable=True)
        return order, trees if bool(torch.equal(order, torch.arange(R, device=order.device))) else trees.select(order)

    def _given_law_chunks(self, law, order, max_scratch_bytes, extra_bytes):
        """The chunks of ``_distribution_chunks`` for a law computed earlier: ``law = (dist [R, N], root_ok [R])`` from
        ``distribution`` of the trees whose rows ``order`` selects.  Yields (lo, hi, dist rows, root_ok rows) of the roots
        order[lo:hi]; the rows are gathered per chunk (8 N bytes per root, counted with ``extra_bytes`` against the budget)
        unless ``order`` is the identity."""
        torch = self.torch
        dist, root_ok = law
        R, N = int(order.shape[0]), self.g.n_node
        if (dist.dtype != torch.float64 or tuple(dist.shape) != (R, N) or not dist.is_contiguous()
                or root_ok.dtype != torch.int32 or tuple(root_ok.shape) != (R,)):
            raise ValueError("law must be distribution's (dist fp64 [%d, %d], root_ok int32 [%d]) for the same trees"
                             % (R, N, R))
        ident = bool(torch.equal(order, torch.arange(R, device=order.device)))
        per_root = extra_bytes(1) + (0 if ident else 8 * N)
        chunk = self._chunk_size(R, N, per_root, max_scratch_bytes)
        for lo in range(0, R, chunk):
            hi = min(R, lo + chunk)
            if ident:
                yield lo, hi, dist[lo:hi], root_ok[lo:hi]
            else:
                idx = order[lo:hi]
                yield lo, hi, dist.index_select(0, idx), root_ok.index_select(0, idx)

    def game_value_grad_d(self, g_emb, g_bias, d_emb, d_bias, trees, *, max_scratch_bytes=None, reuse=None, law=None):
        """``game_value`` and the exact gradient of sum_{ok c} V_c with respect to the discriminator's parameters (csrc/
        value_dgrad.cu, DESIGN.md section 5.4): the expectation of the reference's D-step gradient (discriminator.py:26-30)
        with the raw neighbours as positives and G-mode negatives, negated, without the L2 term.  D ascends V, so this is
        the direction in which D improves.
        Returns device (pos fp64 [R], neg fp64 [R], ok int32 [R]) in the order of ``trees`` -- the bits of ``game_value``
        -- and (grad_emb fp64 [N, ld], grad_bias fp64 [N]) for the padded rows ``d_emb`` (pad columns exactly 0) and
        ``d_bias``.  The roots are taken in ascending id order (stable for duplicates), in the chunks of ``distribution``
        with this gradient's scratch counted against the same budget (``max_scratch_bytes``, default 2 GiB or env
        GG_GDIST_SCRATCH), each coordinate one fp64 chain over the roots: the bits do not depend on the chunking, the order
        of the roots or the call.
        ``law``: ``distribution(g_emb, g_bias, trees)``'s (dist, root_ok), computed earlier for these same trees under the
        same generator and removal bits; it is used instead of recomputing the law, with identical bits (DESIGN.md section
        5.5: a D phase holds G fixed)."""
        torch, g = self.torch, self.g
        assert d_emb.dtype == torch.float32 and d_emb.is_contiguous() and d_bias.dtype == torch.float32
        assert int(d_emb.shape[0]) == g.n_node and int(d_bias.shape[0]) == g.n_node
        R, N, ld = int(trees.roots.shape[0]), g.n_node, int(d_emb.shape[1])
        pos = torch.zeros(R, dtype=torch.float64, device=self.device)
        neg = torch.zeros(R, dtype=torch.float64, device=self.device)
        ok = torch.zeros(R, dtype=torch.int32, device=self.device)
        grad_emb = torch.zeros(tuple(d_emb.shape), dtype=torch.float64, device=self.device)
        grad_bias = torch.zeros(N, dtype=torch.float64, device=self.device)
        if R == 0:
            return pos, neg, ok, grad_emb, grad_bias
        order, st_trees = self._by_root_id(trees)
        value_bytes = lambda k: self._scratch_size("gg_game_value_scratch_bytes", N, k)
        grad_bytes = lambda k: self._scratch_size("gg_game_value_grad_d_scratch_bytes", N, ld, k)
        sp, sn, so = (torch.zeros_like(x) for x in (pos, neg, ok))
        st, vs, ds = self._stream(), None, None
        extra = lambda k: value_bytes(k) + grad_bytes(k)
        if law is None:
            chunks = self._distribution_chunks(g_emb, g_bias, st_trees, reuse, max_scratch_bytes, None, extra_bytes=extra)
        else:
            chunks = self._given_law_chunks(law, order, max_scratch_bytes, extra)
        for lo, hi, dist, root_ok in chunks:
            if vs is None:                                              # the first chunk is the largest
                vs = torch.empty(max(value_bytes(hi - lo), 16), dtype=torch.uint8, device=self.device)
                ds = torch.empty(max(grad_bytes(hi - lo), 16), dtype=torch.uint8, device=self.device)
            roots = st_trees.roots[lo:hi]
            _cabi.check(self.lib.gg_game_value(N, ld, ptr(d_emb), ptr(d_bias), ptr(g.raw_indptr), ptr(g.raw_adj), hi - lo,
                                               ptr(roots), ptr(dist), ptr(root_ok), ptr(sp[lo:hi]), ptr(sn[lo:hi]),
                                               ptr(so[lo:hi]), ptr(vs), vs.numel(), st), "gg_game_value")
            _cabi.check(self.lib.gg_game_value_grad_d(N, ld, ptr(d_emb), ptr(d_bias), ptr(g.raw_indptr), ptr(g.raw_adj),
                                                      hi - lo, ptr(roots), ptr(dist), ptr(root_ok), ptr(grad_emb),
                                                      ptr(grad_bias), ptr(ds), ds.numel(), st), "gg_game_value_grad_d")
        pos[order], neg[order], ok[order] = sp, sn, so
        return pos, neg, ok, grad_emb, grad_bias

    # ------------------------------------------------------------------ expected reference G step
    def expected_g_grad(self, g_emb, g_bias, d_emb, d_bias, trees, *, window, max_scratch_bytes=None, reuse=None):
        """The exact expectation, per G-mode walk, of the reference's generator step (csrc/value_gref.cu, DESIGN.md section
        5.6): the window pairs of the walk's body (graph_gan.py:272-291, ``window`` = config.window_size, 1 .. 8), each
        weighted by D's reward and differentiated as generator.py:22-31 does, with the sampled pairs held fixed.  The law is
        ``distribution``'s (current father-removal bits); lambda_gen and the 1 / batch mean are not included.
        Returns device (n_pairs fp64 [R]: the expected pairs per walk, root_ok int32 [R]) in the order of ``trees``, and
        (grad_emb fp64 [N, ld], grad_bias fp64 [N]) for the padded rows ``g_emb`` (pad columns exactly 0) and ``g_bias``.
        The roots are taken in ascending id order (stable for duplicates), in chunks under the budget rule of
        ``distribution`` (``max_scratch_bytes``, default 2 GiB or env GG_GDIST_SCRATCH), each coordinate one fp64 chain
        over the roots: the bits do not depend on the chunking, the order of the roots or the call."""
        window = _gref_window(window)
        n_pairs, ok, _, _, grad_emb, grad_bias, _ = self._expected_g(g_emb, g_bias, d_emb, d_bias, trees, window,
                                                                     max_scratch_bytes, reuse, False, False)
        return n_pairs, ok, grad_emb, grad_bias

    def expected_g_moments(self, g_emb, g_bias, d_emb, d_bias, trees, *, window, max_scratch_bytes=None, reuse=None,
                           per_node=False):
        """``expected_g_grad`` and the second moment of one G walk's step (DESIGN.md section 5.9).  A walk that stops at y
        adds the fixed vector s(y), the window-pair gradient of its body; per root c, sq_c = sum_y P(y) |s(y)|^2 and
        mn_c = |m_c|^2, m_c the root's expected step (its share of grad_emb / grad_bias), norms over rows and biases.
        sq_c - mn_c is the trace of the covariance of one walk's step, and a pass of n walks per root has
        E|S|^2 = n^2 |sum_c m_c|^2 + n sum_c (sq_c - mn_c).
        Returns device (n_pairs, root_ok, sq fp64 [R], mn fp64 [R], grad_emb, grad_bias), and with ``per_node`` also
        sq_node fp64 [R, N] (|s(y)|^2 per node, 0 at the root and at nodes not reached), in the order of ``trees``.
        n_pairs, root_ok, grad_emb and grad_bias are the bits of ``expected_g_grad``; the chunking and its budget are
        the same (more scratch per root), and no bit depends on the chunking, the order of the roots or the call."""
        window = _gref_window(window)
        out = self._expected_g(g_emb, g_bias, d_emb, d_bias, trees, window, max_scratch_bytes, reuse, True, per_node)
        return out if per_node else out[:6]

    def _expected_g(self, g_emb, g_bias, d_emb, d_bias, trees, window, max_scratch_bytes, reuse, moments, per_node):
        """the chunk loop of expected_g_grad (moments False) and expected_g_moments: (n_pairs, ok, sq, mn, grad_emb,
        grad_bias, sq_node); sq / mn are None without moments, sq_node None without per_node"""
        torch, g = self.torch, self.g
        assert g_emb.dtype == torch.float32 and g_emb.is_contiguous() and g_bias.dtype == torch.float32
        assert d_emb.dtype == torch.float32 and d_emb.is_contiguous() and d_bias.dtype == torch.float32
        assert d_emb.shape == g_emb.shape and int(d_bias.shape[0]) == g.n_node and int(g_emb.shape[0]) == g.n_node
        R, N, nnz = int(trees.roots.shape[0]), g.n_node, int(g.adj.shape[0])
        n_pairs = torch.zeros(R, dtype=torch.float64, device=self.device)
        ok = torch.zeros(R, dtype=torch.int32, device=self.device)
        sq, mn = (torch.zeros(R, dtype=torch.float64, device=self.device) for _ in range(2)) if moments else (None, None)
        sq_node = torch.zeros((R, N), dtype=torch.float64, device=self.device) if per_node else None
        grad_emb = torch.zeros(tuple(g_emb.shape), dtype=torch.float64, device=self.device)
        grad_bias = torch.zeros(N, dtype=torch.float64, device=self.device)
        if R == 0:
            return n_pairs, ok, sq, mn, grad_emb, grad_bias, sq_node
        order, st_trees = self._by_root_id(trees)
        reuse = (self.hub_threshold > 0) if reuse is None else bool(reuse)
        name = "gg_expected_g_moments" if moments else "gg_expected_g_grad"
        scratch_bytes = lambda k: self._scratch_size(name + "_scratch_bytes", N, nnz, k, window)
        chunk = self._chunk_size(R, N, scratch_bytes(1), max_scratch_bytes)
        scratch = torch.empty(max(scratch_bytes(chunk), 16), dtype=torch.uint8, device=self.device)
        sn, so = torch.zeros_like(n_pairs), torch.zeros_like(ok)
        ssq, smn = (torch.zeros_like(sq), torch.zeros_like(mn)) if moments else (None, None)
        snode = torch.empty_like(sq_node) if per_node else None
        d = self._law_desc(g_emb, g_bias, st_trees, reuse, None)
        st = self._stream()
        for lo in range(0, R, chunk):
            hi = min(R, lo + chunk)
            d.n_roots, d.roots, d.tree_bits = hi - lo, ptr(st_trees.roots[lo:hi]), ptr(st_trees.tree_bits[lo:hi])
            if moments:
                rc = self.lib.gg_expected_g_moments(C.byref(d), ptr(d_emb), ptr(d_bias), window, ptr(sn[lo:hi]),
                                                    ptr(so[lo:hi]), ptr(ssq[lo:hi]), ptr(smn[lo:hi]),
                                                    ptr(snode[lo:hi]) if per_node else None, ptr(grad_emb), ptr(grad_bias),
                                                    ptr(scratch), scratch.numel(), st)
            else:
                rc = self.lib.gg_expected_g_grad(C.byref(d), ptr(d_emb), ptr(d_bias), window, ptr(sn[lo:hi]), ptr(so[lo:hi]),
                                                 ptr(grad_emb), ptr(grad_bias), ptr(scratch), scratch.numel(), st)
            _cabi.check(rc, name)
        n_pairs[order], ok[order] = sn, so
        if moments:
            sq[order], mn[order] = ssq, smn
        if per_node:
            sq_node[order] = snode
        return n_pairs, ok, sq, mn, grad_emb, grad_bias, sq_node

    # ------------------------------------------------------------------ expected reference D step
    def expected_d_grad(self, g_emb, g_bias, d_emb, d_bias, trees, *, max_scratch_bytes=None, reuse=None):
        """The exact expectation of the reference's discriminator step of one pass (csrc/value_dgrad.cu, DESIGN.md section
        5.7): E[-grad sum_rows bce] over the rows prepare_data_for_d (graph_gan.py:182-202) emits for each root c -- deg_c =
        |graph[c]| label-1 pairs from the raw list and deg_c label-0 pairs from D-mode walks, all kept with probability
        P_acc = (1 - p_void)^deg_c, the negatives then independent draws from Q = P_D / (1 - p_void) (``d_distribution``).
        lambda_dis, the 1 / batch mean and update_ratio are not included; the law is conditional on the root being drawn.
        The sign is the descent direction of the reference's D loss, so it compares directly with ``game_value_grad_d``.
        Returns device (accept fp64 [R]: P_acc, 0 where ok_ref = 0; p_void fp64 [R]; ok_ref int32 [R]: 1 iff deg_c > 0,
        the root has children and P_acc > 0) in the order of ``trees``, and (grad_emb fp64 [N, ld], grad_bias fp64 [N])
        for the padded rows ``d_emb`` (pad columns exactly 0) and ``d_bias``.  The roots are taken in ascending id order
        (stable for duplicates), in the chunks of ``d_distribution`` with this step's scratch counted against the same
        budget (``max_scratch_bytes``, default 2 GiB or env GG_GDIST_SCRATCH), each coordinate one fp64 chain over the
        roots: the bits do not depend on the chunking, the order of the roots or the call."""
        torch, g = self.torch, self.g
        assert g_emb.dtype == torch.float32 and g_emb.is_contiguous() and g_bias.dtype == torch.float32
        assert d_emb.dtype == torch.float32 and d_emb.is_contiguous() and d_bias.dtype == torch.float32
        assert int(d_emb.shape[0]) == g.n_node and int(d_bias.shape[0]) == g.n_node
        R, N, ld = int(trees.roots.shape[0]), g.n_node, int(d_emb.shape[1])
        accept = torch.zeros(R, dtype=torch.float64, device=self.device)
        p_void = torch.zeros(R, dtype=torch.float64, device=self.device)
        grad_emb = torch.zeros(tuple(d_emb.shape), dtype=torch.float64, device=self.device)
        grad_bias = torch.zeros(N, dtype=torch.float64, device=self.device)
        if R == 0:
            return accept, p_void, torch.zeros(0, dtype=torch.int32, device=self.device), grad_emb, grad_bias
        order, st_trees = self._by_root_id(trees)
        grad_bytes = lambda k: self._scratch_size("gg_expected_d_grad_scratch_bytes", N, ld, k)
        sa, sv = torch.zeros_like(accept), torch.zeros_like(p_void)
        st, ds = self._stream(), None
        for lo, hi, dist, root_ok, pv in self._distribution_chunks(g_emb, g_bias, st_trees, reuse, max_scratch_bytes, None,
                                                                   extra_bytes=grad_bytes, d_mode=True):
            if ds is None:                                              # the first chunk is the largest
                ds = torch.empty(max(grad_bytes(hi - lo), 16), dtype=torch.uint8, device=self.device)
            sv[lo:hi] = pv
            _cabi.check(self.lib.gg_expected_d_grad(N, ld, ptr(d_emb), ptr(d_bias), ptr(g.raw_indptr), ptr(g.raw_adj),
                                                    hi - lo, ptr(st_trees.roots[lo:hi]), ptr(dist), ptr(pv), ptr(root_ok),
                                                    ptr(sa[lo:hi]), ptr(grad_emb), ptr(grad_bias), ptr(ds), ds.numel(), st),
                        "gg_expected_d_grad")
        accept[order], p_void[order] = sa, sv
        return accept, p_void, (accept > 0).to(torch.int32), grad_emb, grad_bias

    # ------------------------------------------------------------------ the value against the best discriminator
    def _best_response_chunks(self, g_emb, g_bias, trees, max_scratch_bytes, reuse, grad):
        """(order, sorted trees, chunk size, scratch, descriptor) of best_response / best_response_grad"""
        torch, g = self.torch, self.g
        assert g_emb.dtype == torch.float32 and g_emb.is_contiguous() and g_bias.dtype == torch.float32
        assert int(g_emb.shape[0]) == g.n_node and int(g_bias.shape[0]) == g.n_node
        R, N, nnz = int(trees.roots.shape[0]), g.n_node, int(g.adj.shape[0])
        order, st_trees = self._by_root_id(trees)
        reuse = (self.hub_threshold > 0) if reuse is None else bool(reuse)
        fn = "gg_best_response_grad_scratch_bytes" if grad else "gg_best_response_scratch_bytes"
        scratch_bytes = lambda k: self._scratch_size(fn, N, nnz, k)
        chunk = self._chunk_size(R, N, scratch_bytes(1), max_scratch_bytes)
        scratch = torch.empty(max(scratch_bytes(chunk), 16), dtype=torch.uint8, device=self.device)
        return order, st_trees, chunk, scratch, self._law_desc(g_emb, g_bias, st_trees, reuse, None)

    def best_response(self, g_emb, g_bias, trees, *, max_scratch_bytes=None, reuse=None):
        """The game value against the best discriminator per root (csrc/best_response.cu, DESIGN.md section 5.8):
        vstar_c = max_D V_c(G, D) = 2 JSD(p_true(.|c) || G(.|c)) - log 4, with p_true(a | c) = n_ca / |graph[c]| over the
        raw list and G the generator's exact G-mode law (``distribution``, current father-removal bits) at c's neighbours,
        which are the depth-1 nodes of c's tree: only the depth-1 lists are built.  hit_c = sum_a G(a | c), the
        generator's mass on the true neighbours.  Returns device (vstar fp64 [R], hit fp64 [R], ok int32 [R]) in the order
        of ``trees``; ok is ``game_value``'s (vstar = hit = 0 where ok = 0).  The roots are taken in ascending id order, in
        chunks under the budget rule of ``distribution`` (``max_scratch_bytes``, default 2 GiB or env GG_GDIST_SCRATCH):
        the bits do not depend on the chunking, the order of the roots or the call."""
        torch, g = self.torch, self.g
        R = int(trees.roots.shape[0])
        vstar = torch.zeros(R, dtype=torch.float64, device=self.device)
        hit = torch.zeros(R, dtype=torch.float64, device=self.device)
        ok = torch.zeros(R, dtype=torch.int32, device=self.device)
        if R == 0:
            return vstar, hit, ok
        order, st_trees, chunk, scratch, d = self._best_response_chunks(g_emb, g_bias, trees, max_scratch_bytes, reuse, False)
        sv, sh, so = torch.zeros_like(vstar), torch.zeros_like(hit), torch.zeros_like(ok)
        mult, st = g.entry_mult(), self._stream()
        for lo in range(0, R, chunk):
            hi = min(R, lo + chunk)
            d.n_roots, d.roots, d.tree_bits = hi - lo, ptr(st_trees.roots[lo:hi]), ptr(st_trees.tree_bits[lo:hi])
            _cabi.check(self.lib.gg_best_response(C.byref(d), ptr(g.raw_indptr), ptr(mult), ptr(sv[lo:hi]), ptr(sh[lo:hi]),
                                                  ptr(so[lo:hi]), ptr(scratch), scratch.numel(), st), "gg_best_response")
        vstar[order], hit[order], ok[order] = sv, sh, so
        return vstar, hit, ok

    def best_response_grad(self, g_emb, g_bias, trees, *, max_scratch_bytes=None, reuse=None):
        """``best_response`` and the exact gradient of sum_{ok c} vstar_c with respect to the generator's parameters
        (DESIGN.md section 5.8): section 5.3's policy gradient with log(1 - D*) for D* = p / (p + G), held fixed (envelope
        theorem).  Returns device (vstar fp64 [R], hit fp64 [R], ok int32 [R]) in the order of ``trees`` -- the bits of
        ``best_response`` -- and (grad_emb fp64 [N, ld], grad_bias fp64 [N]) for the padded rows ``g_emb`` (pad columns
        exactly 0) and ``g_bias``; lambda_gen is not included.  The roots are taken in ascending id order, in chunks under
        the budget rule of ``distribution``; two fp64 accumulators per walk-CSR entry (16 bytes each) are held for the
        whole call and turned into the gradient once at the end: the bits do not depend on the chunking, the order of the
        roots or the call.  Needs a symmetric walk CSR (``DeviceGraph.reverse_entries``)."""
        torch, g = self.torch, self.g
        R, N, nnz = int(trees.roots.shape[0]), g.n_node, int(g.adj.shape[0])
        vstar = torch.zeros(R, dtype=torch.float64, device=self.device)
        hit = torch.zeros(R, dtype=torch.float64, device=self.device)
        ok = torch.zeros(R, dtype=torch.int32, device=self.device)
        grad_emb = torch.zeros(tuple(g_emb.shape), dtype=torch.float64, device=self.device)
        grad_bias = torch.zeros(N, dtype=torch.float64, device=self.device)
        if R == 0:
            return vstar, hit, ok, grad_emb, grad_bias
        rev = g.reverse_entries()
        if rev is None:
            raise ValueError("best_response_grad needs a symmetric walk CSR (every entry has a reverse entry)")
        order, st_trees, chunk, scratch, d = self._best_response_chunks(g_emb, g_bias, trees, max_scratch_bytes, reuse, True)
        sv, sh, so = torch.zeros_like(vstar), torch.zeros_like(hit), torch.zeros_like(ok)
        acc_coef = torch.zeros(max(nnz, 1), dtype=torch.float64, device=self.device)
        acc_bias = torch.zeros(max(nnz, 1), dtype=torch.float64, device=self.device)
        mult, st = g.entry_mult(), self._stream()
        for lo in range(0, R, chunk):
            hi = min(R, lo + chunk)
            d.n_roots, d.roots, d.tree_bits = hi - lo, ptr(st_trees.roots[lo:hi]), ptr(st_trees.tree_bits[lo:hi])
            _cabi.check(self.lib.gg_best_response_grad(C.byref(d), ptr(g.raw_indptr), ptr(mult), ptr(rev), ptr(sv[lo:hi]),
                                                       ptr(sh[lo:hi]), ptr(so[lo:hi]), ptr(acc_coef), ptr(acc_bias),
                                                       ptr(scratch), scratch.numel(), st), "gg_best_response_grad")
        _cabi.check(self.lib.gg_best_response_spmm(N, int(g_emb.shape[1]), ptr(g.indptr), ptr(g.adj), ptr(g_emb),
                                                   ptr(acc_coef), ptr(acc_bias), ptr(grad_emb), ptr(grad_bias), st),
                    "gg_best_response_spmm")
        vstar[order], hit[order], ok[order] = sv, sh, so
        return vstar, hit, ok, grad_emb, grad_bias

    def finalize(self, out):
        _cabi.check(self.lib.gg_walk_finalize(out.n_roots, ptr(out.walk_ptr), int(out.for_d), ptr(out.samples),
                                              ptr(out.status), ptr(out.first_edge), ptr(out.wsteps), ptr(out.wsuml),
                                              ptr(out.path_len), ptr(self.g.d1_bits), ptr(out.root_ok),
                                              ptr(out.counters), self._stream()), "gg_walk_finalize")

    def emit_d_rows(self, out):
        """prepare_data_for_d's (center, neighbor, label) rows (graph_gan.py:192-201), on device."""
        p = out.plan
        center, neighbor, label = p.rows
        _cabi.check(self.lib.gg_emit_d_rows(out.n_roots, ptr(out.roots), ptr(out.walk_ptr), ptr(self.g.raw_indptr),
                                            ptr(self.g.raw_adj), ptr(out.root_ok), ptr(out.samples), ptr(p.row_ptr),
                                            ptr(center), ptr(neighbor), ptr(label), ptr(p.n_rows), self._stream()),
                    "gg_emit_d_rows")
        return center, neighbor, label, p.n_rows
