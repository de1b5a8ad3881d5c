"""Re-hosted trainer: the reference's ``GraphGAN`` class (src/GraphGAN/graph_gan.py:17-319) with the
same method names, whose bodies batch over roots and call the CUDA hot path.

What is accelerated (SURVEY.md section 8): ``construct_trees`` (GPU BFS), ``sample`` /
``prepare_data_for_d`` / ``prepare_data_for_g`` (K1 + finalize + row/pair emission, all on device),
``discriminator.reward`` and the two update ops (K2 + K3).  What is only re-hosted (thin, not
accelerated): the epoch loop, the text dumps and the link-prediction check.

Differences from the reference that a caller can observe, all documented in DESIGN.md:
  * training rows are device int32/fp32 tensors, not Python lists (len() and slicing still work);
  * walks draw from Philox keyed by (config.seed, pass, root, walk, step) instead of the global
    MT19937 stream, so results do not depend on the number of GPUs or on root order;
  * BFS trees are parent arrays built on the GPU; there is no pickle cache (config.cache_filename
    is ignored) because the dict-of-lists form is O(N^2).
"""
import os

import numpy as np

from . import config
from . import evaluation as lp
from . import io
from .discriminator import Discriminator
from .generator import Generator
from .graph import DeviceGraph, HostGraph
from .sampler import WalkSampler
from .session import Session
from ._cabi import ptr
from . import _cabi
import ctypes as C


def check_exact_mode(cfg, world):
    """Refuse exact-game training (cfg.exact_roots > 0, DESIGN.md section 5.5) in a run of more than one process: its
    steps are single-process."""
    if getattr(cfg, "exact_roots", 0) > 0 and world > 1:
        raise ValueError("config.exact_roots = %d trains on one process only, not %d (set exact_roots = 0 under torchrun)"
                         % (cfg.exact_roots, world))


def _device():
    dev = config.device
    if "LOCAL_RANK" in os.environ and str(dev).startswith("cuda"):
        dev = "cuda:%d" % int(os.environ["LOCAL_RANK"])
    return dev


class GraphGAN(object):
    def __init__(self, host_graph=None, node_embed_init_d=None, node_embed_init_g=None):
        import torch
        self.torch = torch
        self.device = torch.device(_device())
        if self.device.type == "cuda":
            torch.cuda.set_device(self.device)
        print("reading graphs...")
        self.host_graph = host_graph if host_graph is not None else HostGraph.from_files(config.train_filename,
                                                                                         config.test_filename)
        self.n_node = self.host_graph.n_node
        self.graph = self.host_graph            # graph[i] == self.host_graph.neighbors(i)
        self.root_nodes = [i for i in range(self.n_node)]

        print("reading initial embeddings...")
        # graph_gan.py:24-29: the discriminator's file is read first (it consumes the global RNG first)
        self.node_embed_init_d = node_embed_init_d if node_embed_init_d is not None else io.read_embeddings(
            filename=config.pretrain_emb_filename_d, n_node=self.n_node, n_embed=config.n_emb)
        self.node_embed_init_g = node_embed_init_g if node_embed_init_g is not None else io.read_embeddings(
            filename=config.pretrain_emb_filename_g, n_node=self.n_node, n_embed=config.n_emb)

        self.device_graph = DeviceGraph(self.host_graph, self.device)
        self.sampler = WalkSampler(self.device_graph)
        self.lib = _cabi.lib()

        # BFS trees: resident for all roots when they fit (the reference's pickle cache, graph_gan.py:31-46)
        self.trees, self._tree_key = None, None
        import torch.distributed as _d
        if not (_d.is_available() and _d.is_initialized() and _d.get_world_size() > 1) and \
                self._tree_bytes(self.n_node) <= config.tree_cache_bytes:
            print("constructing BFS-trees...")
            self.trees = self.construct_trees(self.root_nodes)

        print("building GAN model...")
        self.discriminator = None
        self.generator = None
        self.build_generator()
        self.build_discriminator()
        self.sess = Session()
        self.shuffle_rng = np.random.RandomState(config.seed)
        self.pass_counter = 0
        self.last_counters = {}
        self.exact_trace = []                   # (phase, step, mean V, n_ok) of every exact step (config.exact_roots > 0)
        # one process per GPU: roots are sharded, rows all-gathered, updates data parallel (parallel.py)
        import torch.distributed as dist
        self.dist = dist if (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1) else None
        self.rank = self.dist.get_rank() if self.dist else 0
        self.world = self.dist.get_world_size() if self.dist else 1
        if self.dist:
            from .parallel import DataParallelStep
            self._dp_d, self._dp_g = DataParallelStep(self.discriminator), DataParallelStep(self.generator)

    # ------------------------------------------------------------------ trees (graph_gan.py:63-108)
    def _tree_bytes(self, n_roots):
        """device bytes of the tree rows of `n_roots` roots: one bit per walk-CSR entry each (csrc/bfs.cu)"""
        return n_roots * 4 * ((int(self.host_graph.adj.shape[0]) + 31) // 32 + 1)

    def construct_trees(self, nodes):
        """BFS trees of ``nodes`` -> sampler.TreeBatch (parent arrays on the GPU)."""
        return self.sampler.build_trees(np.asarray(nodes, np.int32))

    def construct_trees_with_mp(self, nodes):
        """Kept for source compatibility (graph_gan.py:63-82); the GPU builder needs no process pool."""
        self.trees = self.construct_trees(nodes)

    def build_generator(self):
        self.generator = Generator(n_node=self.n_node, node_emd_init=self.node_embed_init_g, device=self.device)
        self.generator.sampler = self.sampler     # Generator.relevance: G(v | root) over this graph's BFS trees

    def build_discriminator(self):
        self.discriminator = Discriminator(n_node=self.n_node, node_emd_init=self.node_embed_init_d, device=self.device)

    # ------------------------------------------------------------------ root batching
    def _root_batches(self, roots):
        roots = np.asarray(roots, np.int32)
        if self.dist:   # this rank's contiguous, degree-balanced block of the root list (same for D and G passes)
            from .parallel import balanced_root_ranges
            lo, hi = balanced_root_ranges(self.host_graph.degrees()[roots] + 1, self.world)[self.rank]
            roots = roots[lo:hi]
            key = (lo, hi, hash(roots.tobytes()))           # the cached trees belong to exactly these roots
            if self.trees is not None and self._tree_key != key:
                self.trees = None
            if self.trees is None and self._tree_bytes(max(hi - lo, 1)) <= config.tree_cache_bytes:
                self.trees, self._tree_key = self.construct_trees(roots), key
            if self.trees is not None:
                yield self.trees
                return
        if self.trees is not None and roots.shape[0] == self.n_node and np.array_equal(roots, np.arange(self.n_node)):
            yield self.trees
            return
        for s in range(0, roots.shape[0], config.root_batch):
            yield self.construct_trees(roots[s:s + config.root_batch])

    # ------------------------------------------------------------------ the game value V(G, D) (DESIGN.md section 5.2)
    def game_value(self, roots):
        """V_c(G, D) = pos_c + neg_c of the current generator and discriminator for every root c of ``roots`` (Wang et al.,
        AAAI-18, Eq. 1), exactly: sampler.WalkSampler.game_value.  Returns device (pos fp64, neg fp64, ok int32)."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        g, d = self.generator, self.discriminator
        return self.sampler.game_value(g.emb, g.bias_t, d.emb, d.bias_t, self._trees_of(roots))

    def game_value_grad(self, roots):
        """game_value(roots) and the exact gradient of sum_{ok c} V_c with respect to the generator's padded rows and biases
        (DESIGN.md section 5.3): sampler.WalkSampler.game_value_grad.  Returns device (pos, neg, ok, grad_emb fp64 [N, ld],
        grad_bias fp64 [N]); pos, neg and ok are the bits of game_value."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        g, d = self.generator, self.discriminator
        return self.sampler.game_value_grad(g.emb, g.bias_t, d.emb, d.bias_t, self._trees_of(roots))

    def game_value_grad_d(self, roots):
        """game_value(roots) and the exact gradient of sum_{ok c} V_c with respect to the discriminator's padded rows and
        biases (DESIGN.md section 5.4): sampler.WalkSampler.game_value_grad_d.  Returns device (pos, neg, ok, grad_emb fp64
        [N, ld], grad_bias fp64 [N]); pos, neg and ok are the bits of game_value."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        g, d = self.generator, self.discriminator
        return self.sampler.game_value_grad_d(g.emb, g.bias_t, d.emb, d.bias_t, self._trees_of(roots))

    def expected_g_grad(self, roots):
        """The exact expectation, per G-mode walk, of the reference's generator step over the window pairs of the walks
        from ``roots`` (DESIGN.md section 5.6), with config.window_size and the current models: sampler.WalkSampler.
        expected_g_grad.  Returns device (n_pairs fp64, root_ok int32, grad_emb fp64 [N, ld], grad_bias fp64 [N])."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        g, d = self.generator, self.discriminator
        return self.sampler.expected_g_grad(g.emb, g.bias_t, d.emb, d.bias_t, self._trees_of(roots),
                                            window=config.window_size)

    def expected_g_moments(self, roots):
        """expected_g_grad(roots) and the second moment of one walk's step per root (DESIGN.md section 5.9), with
        config.window_size and the current models: sampler.WalkSampler.expected_g_moments.  Returns device (n_pairs,
        root_ok, sq fp64, mn fp64, grad_emb fp64 [N, ld], grad_bias fp64 [N])."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        g, d = self.generator, self.discriminator
        return self.sampler.expected_g_moments(g.emb, g.bias_t, d.emb, d.bias_t, self._trees_of(roots),
                                               window=config.window_size)

    def expected_d_grad(self, roots):
        """The exact expectation of the reference's discriminator step of one pass over ``roots`` (DESIGN.md section 5.7),
        with the current models: sampler.WalkSampler.expected_d_grad.  Returns device (accept fp64, p_void fp64, ok_ref
        int32, grad_emb fp64 [N, ld], grad_bias fp64 [N])."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        g, d = self.generator, self.discriminator
        return self.sampler.expected_d_grad(g.emb, g.bias_t, d.emb, d.bias_t, self._trees_of(roots))

    def best_response(self, roots):
        """The game value against the best discriminator, vstar_c = max_D V_c(G, D) = 2 JSD(p_true(.|c) || G(.|c)) - log 4,
        and G's mass on the true neighbours, for every root c of ``roots`` (DESIGN.md section 5.8), with the current
        generator: sampler.WalkSampler.best_response.  Returns device (vstar fp64, hit fp64, ok int32)."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        g = self.generator
        return self.sampler.best_response(g.emb, g.bias_t, self._trees_of(roots))

    def best_response_grad(self, roots):
        """best_response(roots) and the exact gradient of sum_{ok c} vstar_c with respect to the generator's padded rows
        and biases (DESIGN.md section 5.8): sampler.WalkSampler.best_response_grad.  Returns device (vstar, hit, ok,
        grad_emb fp64 [N, ld], grad_bias fp64 [N])."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        g = self.generator
        return self.sampler.best_response_grad(g.emb, g.bias_t, self._trees_of(roots))

    def _trees_of(self, roots):
        """the trees of ``roots``: rows of the resident trees when they hold every one of them, else built"""
        t = self.trees
        if t is not None and roots.shape[0]:
            have = t.roots.cpu().numpy()
            if have.shape[0] and np.all(have[1:] > have[:-1]):      # the resident trees' roots are ascending ids
                idx = np.minimum(np.searchsorted(have, roots), have.shape[0] - 1)
                if np.array_equal(have[idx], roots):
                    return t.select(self.torch.as_tensor(idx.astype(np.int64)).to(self.device))
        return self.construct_trees(roots)

    def value_roots(self):
        """The roots of the value line: config.value_roots of them, seeded by config.seed and fixed for the run so that
        epochs compare.  Under torchrun, rank 0 (which evaluates) holds father-removal bits for its own root shard
        only, so the sample comes from that shard."""
        key = (int(config.value_roots), int(config.seed))
        if getattr(self, "_value_key", None) != key:
            from . import synth
            deg = self.host_graph.degrees()
            lo, hi = 0, self.n_node
            if self.dist:
                from .parallel import balanced_root_ranges
                lo, hi = balanced_root_ranges(deg[np.asarray(self.root_nodes)] + 1, self.world)[self.rank]
            self._value_roots = (synth.pick_roots(deg[lo:hi], key[0], seed=key[1]).astype(np.int64) + lo).astype(np.int32)
            self._value_key = key
        return self._value_roots

    def value_line(self):
        """The line evaluation() appends: "value:<mean V> pos:<mean pos> neg:<mean neg> roots:<ok roots>", the means taken
        over the ok roots of value_roots() (nan when there are none).  With config.value_grad, " gnorm:<norm>" follows:
        the 2-norm of the gradient of the mean V over (E_G[:, :n_emb], b_G), exact (game_value_grad).  With
        config.value_grad_d, " dnorm:<norm>" comes last: the same for the discriminator, over (E_D[:, :n_emb], b_D)
        (game_value_grad_d).  With config.value_gcos, " gcos:<cos>" follows them: the cosine over (E_G[:, :n_emb], b_G)
        between the expectation of the reference's generator step (expected_g_grad) and the gradient of the sum of V
        (game_value_grad; computed for it alone when value_grad is off).  A positive value means the reference's step, which
        descends its own loss, descends V on average.  With config.value_dcos, " dcos:<cos>" comes last: the cosine over
        (E_D[:, :n_emb], b_D) between the expectation of the reference's D step of one pass (expected_d_grad) and the
        gradient of the sum of V (game_value_grad_d; computed for it alone when value_grad_d is off).  A positive value
        means the reference's D step ascends V on average.  With config.value_jsd, " jsd:<mean JSD> hit:<mean hit>" comes
        last: the Jensen-Shannon divergence of the generator from the data and the generator's mass on the true
        neighbours (best_response), means over the roots whose best-response ok is 1.  With config.value_gsnr,
        " gsnr:<snr>" comes last: n |M|^2 / sum_c var_c over the ok roots (expected_g_moments), n = config.n_sample_gen,
        M = sum_c m_c the expected step of the reference's G pass and var_c = sq_c - mn_c the trace of the covariance of
        one walk's step: the signal-to-noise ratio of one sampled G pass (nan without ok roots or when sum var_c <= 0)."""
        vg, vd = getattr(config, "value_grad", False), getattr(config, "value_grad_d", False)
        if vg:
            pos, neg, ok, g_emb, g_bias = self.game_value_grad(self.value_roots())
        if vd:
            out = self.game_value_grad_d(self.value_roots())
            d_emb, d_bias = out[3:]
            if not vg:
                pos, neg, ok = out[:3]
        if not (vg or vd):
            pos, neg, ok = self.game_value(self.value_roots())
        pos, neg, ok = (x.cpu().numpy() for x in (pos, neg, ok))
        sel = ok == 1
        n = int(sel.sum())
        v, p, q = ((pos + neg)[sel].mean(), pos[sel].mean(), neg[sel].mean()) if n else (np.nan,) * 3
        line = "value:%r pos:%r neg:%r roots:%d" % (float(v), float(p), float(q), n)
        if getattr(config, "value_grad", False):
            sq = float((g_emb[:, :self.generator.n_emb] ** 2).sum().item() + (g_bias ** 2).sum().item())
            line += " gnorm:%r" % (float(np.sqrt(sq) / n) if n else np.nan)
        if vd:
            sq = float((d_emb[:, :self.discriminator.n_emb] ** 2).sum().item() + (d_bias ** 2).sum().item())
            line += " dnorm:%r" % (float(np.sqrt(sq) / n) if n else np.nan)
        if getattr(config, "value_gcos", False):
            if not vg:
                g_emb, g_bias = self.game_value_grad(self.value_roots())[3:]
            r_emb, r_bias = self.expected_g_grad(self.value_roots())[2:]
            k = self.generator.n_emb
            dot = float((r_emb[:, :k] * g_emb[:, :k]).sum().item() + (r_bias * g_bias).sum().item())
            nr = float(np.sqrt((r_emb[:, :k] ** 2).sum().item() + (r_bias ** 2).sum().item()))
            ng = float(np.sqrt((g_emb[:, :k] ** 2).sum().item() + (g_bias ** 2).sum().item()))
            line += " gcos:%r" % (dot / (nr * ng) if nr > 0 and ng > 0 else np.nan)
        if getattr(config, "value_dcos", False):
            if not vd:
                d_emb, d_bias = self.game_value_grad_d(self.value_roots())[3:]
            r_emb, r_bias = self.expected_d_grad(self.value_roots())[3:]
            k = self.discriminator.n_emb
            dot = float((r_emb[:, :k] * d_emb[:, :k]).sum().item() + (r_bias * d_bias).sum().item())
            nr = float(np.sqrt((r_emb[:, :k] ** 2).sum().item() + (r_bias ** 2).sum().item()))
            nd = float(np.sqrt((d_emb[:, :k] ** 2).sum().item() + (d_bias ** 2).sum().item()))
            line += " dcos:%r" % (dot / (nr * nd) if nr > 0 and nd > 0 else np.nan)
        if getattr(config, "value_jsd", False):
            vs, ht, okb = (x.cpu().numpy() for x in self.best_response(self.value_roots()))
            sb = okb == 1
            nb = int(sb.sum())
            jsd = float((vs[sb] / 2 + np.log(2.0)).mean()) if nb else np.nan
            line += " jsd:%r hit:%r" % (jsd, float(ht[sb].mean()) if nb else np.nan)
        if getattr(config, "value_gsnr", False):
            _, okg, sq, mn, r_emb, r_bias = self.expected_g_moments(self.value_roots())
            sg = (okg == 1).cpu().numpy()
            var = float((sq - mn).cpu().numpy()[sg].sum())
            k = self.generator.n_emb
            m2 = float((r_emb[:, :k] ** 2).sum().item() + (r_bias ** 2).sum().item())
            line += " gsnr:%r" % (int(config.n_sample_gen) * m2 / var if sg.any() and var > 0 else np.nan)
        return line + "\n"

    # ------------------------------------------------------------------ training on the exact game (DESIGN.md section 5.5)
    def exact_roots(self):
        """The roots of exact training: config.exact_roots non-isolated roots seeded by config.seed (all of them when
        exact_roots reaches their number), fixed for the run."""
        key = (int(config.exact_roots), int(config.seed))
        if getattr(self, "_exact_key", None) != key:
            from . import synth
            self._exact_roots = synth.pick_roots(self.host_graph.degrees(), key[0], seed=key[1])
            self._exact_key = key
        return self._exact_roots

    def _exact_trees(self, roots):
        """the trees of ``roots``, taken from the resident trees or built, once: they do not change during a run"""
        key = roots.tobytes()
        if getattr(self, "_exact_tree_key", None) != key:
            self._exact_tree_cache, self._exact_tree_key = self._trees_of(roots), key
        return self._exact_tree_cache

    def exact_d_step(self, roots, *, law=None, max_scratch_bytes=None):
        """One Adam step of the discriminator on the exact gradient of the mean game value over the ok roots of ``roots``:
        game_value_grad_d, then apply_dense_grad with scale -1/n_ok (D ascends V; the L2 term is the model's own).
        ``law``: the generator's law for these roots (sampler.WalkSampler.distribution of their trees), reused instead of
        recomputed.  A step without ok roots changes nothing.  Returns the pre-step device (pos, neg, ok)."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        g, d = self.generator, self.discriminator
        pos, neg, ok, gE, gb = self.sampler.game_value_grad_d(g.emb, g.bias_t, d.emb, d.bias_t, self._exact_trees(roots),
                                                              max_scratch_bytes=max_scratch_bytes, law=law)
        n_ok = int(ok.sum().item())
        if n_ok:
            d.apply_dense_grad(gE, gb, -1.0 / n_ok)
        return pos, neg, ok

    def exact_g_step(self, roots, *, max_scratch_bytes=None):
        """One Adam step of the generator on the exact gradient of the mean game value over the ok roots of ``roots``:
        game_value_grad, then apply_dense_grad with scale +1/n_ok (G descends V).  A step without ok roots changes nothing.
        Returns the pre-step device (pos, neg, ok)."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        g, d = self.generator, self.discriminator
        pos, neg, ok, gE, gb = self.sampler.game_value_grad(g.emb, g.bias_t, d.emb, d.bias_t, self._exact_trees(roots),
                                                            max_scratch_bytes=max_scratch_bytes)
        n_ok = int(ok.sum().item())
        if n_ok:
            g.apply_dense_grad(gE, gb, 1.0 / n_ok)
        return pos, neg, ok

    def exact_jsd_step(self, roots, *, max_scratch_bytes=None):
        """One Adam step of the generator on the exact gradient of the mean Jensen-Shannon divergence JSD_c = vstar_c / 2
        + log 2 over the ok roots of ``roots`` (DESIGN.md section 5.8): best_response_grad, then apply_dense_grad with
        scale +1/(2 n_ok) (the L2 term is the model's own, as in exact_g_step).  A step without ok roots changes nothing.
        Returns the pre-step device (vstar, hit, ok)."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        g = self.generator
        vstar, hit, ok, gE, gb = self.sampler.best_response_grad(g.emb, g.bias_t, self._exact_trees(roots),
                                                                 max_scratch_bytes=max_scratch_bytes)
        n_ok = int(ok.sum().item())
        if n_ok:
            g.apply_dense_grad(gE, gb, 1.0 / (2 * n_ok))
        return vstar, hit, ok

    def exact_d_phase(self, roots, steps, *, max_scratch_bytes=None):
        """``steps`` exact D steps.  G is fixed meanwhile, so its law over the roots is computed once when it fits the
        scratch budget of the exact-game entry points (8 bytes per root and node; ``max_scratch_bytes``, default env
        GG_GDIST_SCRATCH or 2 GiB), else recomputed by every step -- the same bits either way.  Returns the steps' pre-step
        (pos, neg, ok)."""
        roots = np.asarray(roots.cpu() if isinstance(roots, self.torch.Tensor) else roots, np.int32).reshape(-1)
        law = None
        if steps > 0 and roots.shape[0] * self.n_node * 8 <= self.sampler.scratch_budget(max_scratch_bytes):
            law = self.sampler.distribution(self.generator.emb, self.generator.bias_t, self._exact_trees(roots),
                                            max_scratch_bytes=max_scratch_bytes)
        return [self.exact_d_step(roots, law=law, max_scratch_bytes=max_scratch_bytes) for _ in range(steps)]

    def _exact_phase(self, phase, outs):
        """append the steps of one phase to exact_trace and print the phase's line"""
        vals = []
        for step, (pos, neg, ok) in enumerate(outs):
            pos, neg, ok = (x.cpu().numpy() for x in (pos, neg, ok))
            sel = ok == 1
            n = int(sel.sum())
            v = float((pos + neg)[sel].mean()) if n else float("nan")
            self.exact_trace.append((phase, step, v, n))
            vals.append(v)
        if vals:
            print("exact %s: %d steps, mean V %r -> %r before the first / last step, %d roots"
                  % (phase, len(vals), vals[0], vals[-1], self.exact_trace[-1][3]))

    def _next_tag(self):
        self.pass_counter += 1
        return self.pass_counter

    # ------------------------------------------------------------------ graph_gan.py:182-202
    def prepare_data_for_d(self, roots=None):
        """positive and negative samples for the discriminator -> (center_nodes, neighbor_nodes, labels)
        as device tensors (int32, int32, fp32), rows in the reference's order."""
        torch = self.torch
        tag = self._next_tag()
        cs, ns, ls = [], [], []
        tot = dict(steps=0, sum_l=0, accepted=0)
        for trees in self._root_batches(self.root_nodes if roots is None else roots):
            sample_num = self.device_graph.raw_deg[trees.roots.long()]
            out = self.sampler.run(self.generator.emb, self.generator.bias_t, trees, sample_num, True,
                                   seed=config.seed, pass_tag=tag, update_ratio=float(config.update_ratio))
            c, n, l, n_rows = self.sampler.emit_d_rows(out)
            k = int(n_rows.item())
            cs.append(c[:k]); ns.append(n[:k]); ls.append(l[:k])
            cnt = out.counters_host()
            for key in tot:
                tot[key] += cnt[key]
        self.last_counters = tot
        cat = lambda xs, dt: torch.cat(xs) if xs else torch.zeros(0, dtype=dt, device=self.device)
        c, n, l = cat(cs, torch.int32), cat(ns, torch.int32), cat(ls, torch.int32)
        if self.dist:   # every rank ends up with the full row lists, in root order
            from .parallel import all_gather_varlen
            c, n, l = all_gather_varlen(c), all_gather_varlen(n), all_gather_varlen(l)
        return c, n, l.float()

    # ------------------------------------------------------------------ graph_gan.py:204-223
    def prepare_data_for_g(self, roots=None):
        """sample nodes for the generator -> (node_1, node_2, reward) device tensors."""
        torch = self.torch
        tag = self._next_tag()
        n1s, n2s = [], []
        st = torch.cuda.current_stream(self.device).cuda_stream
        for trees in self._root_batches(self.root_nodes if roots is None else roots):
            out = self.sampler.run(self.generator.emb, self.generator.bias_t, trees, int(config.n_sample_gen), False,
                                   seed=config.seed, pass_tag=tag, update_ratio=float(config.update_ratio),
                                   max_path=config.max_path_len)
            if out.counters_host()["path_overflow"]:
                raise RuntimeError("a walk is longer than config.max_path_len=%d" % config.max_path_len)
            W = out.n_walks
            pair_ptr = torch.empty(W + 1, dtype=torch.int64, device=self.device)
            n_pairs = torch.zeros(1, dtype=torch.int64, device=self.device)
            # count first (capacity 0), then emit
            _cabi.check(self.lib.gg_window_pairs(W, ptr(out.paths), ptr(out.path_len), out.max_path, int(config.window_size),
                                                 ptr(pair_ptr), None, None, ptr(n_pairs), 0, st), "gg_window_pairs")
            m = int(n_pairs.item())
            n1 = torch.empty(max(m, 1), dtype=torch.int32, device=self.device)
            n2 = torch.empty(max(m, 1), dtype=torch.int32, device=self.device)
            _cabi.check(self.lib.gg_window_pairs(W, ptr(out.paths), ptr(out.path_len), out.max_path, int(config.window_size),
                                                 ptr(pair_ptr), ptr(n1), ptr(n2), ptr(n_pairs), m, st), "gg_window_pairs")
            n1s.append(n1[:m]); n2s.append(n2[:m])
        node_1 = torch.cat(n1s) if n1s else torch.zeros(0, dtype=torch.int32, device=self.device)
        node_2 = torch.cat(n2s) if n2s else torch.zeros(0, dtype=torch.int32, device=self.device)
        if self.dist:
            from .parallel import all_gather_varlen
            node_1, node_2 = all_gather_varlen(node_1), all_gather_varlen(node_2)
        reward = self.discriminator.reward_pairs(node_1, node_2)     # graph_gan.py:220-222, one fetch for all pairs
        return node_1, node_2, reward

    # ------------------------------------------------------------------ graph_gan.py:225-270 (single-root form)
    def sample(self, root, tree, sample_num, for_d):
        """Reference-shaped call: one root -> (samples, paths) as Python lists, or (None, None).
        ``tree`` may be a TreeBatch holding this root or anything else (then the tree is rebuilt)."""
        from .sampler import DONE, TreeBatch
        torch = self.torch
        if not (isinstance(tree, TreeBatch) and int(tree.roots.shape[0]) == 1 and int(tree.roots[0]) == root):
            tree = self.construct_trees([root])
        if sample_num == 0:
            return [], []
        out = self.sampler.run(self.generator.emb, self.generator.bias_t, tree, int(sample_num), bool(for_d),
                               seed=config.seed, pass_tag=self._next_tag(), max_path=config.max_path_len)
        if not int(out.root_ok[0]):
            return None, None
        samples = out.samples[:sample_num].cpu().tolist()
        plen, paths = out.path_len.cpu().numpy(), out.paths.cpu().numpy()
        return samples, [paths[w, :plen[w]].tolist() for w in range(sample_num)]

    @staticmethod
    def get_node_pairs_from_path(path):
        """path = [1, 0, 2, 4, 2], window_size = 2 -> [[1,0],[1,2],[0,1],[0,2],[0,4],[2,1],[2,0],[2,4],[4,0],[4,2]]
        (graph_gan.py:272-291; the batched device version is gg_window_pairs)."""
        body, w, pairs = path[:-1], config.window_size, []
        for pos, center in enumerate(body):
            for other in range(max(pos - w, 0), min(pos + w + 1, len(body))):
                if other != pos:
                    pairs.append([center, body[other]])
        return pairs

    # ------------------------------------------------------------------ graph_gan.py:122-180
    def train(self):
        check_exact_mode(config, self.world)
        exact = config.exact_roots > 0
        torch = self.torch
        ckpt = os.path.join(config.model_log, "model.checkpoint.pt")
        if config.load_model and os.path.isfile(ckpt):
            print("loading the checkpoint: %s" % ckpt)
            self.load(ckpt)
        self.write_embeddings_to_file()
        self.evaluation(self)
        print("start training...")
        for epoch in range(config.n_epochs):
            print("epoch %d" % epoch)
            if epoch > 0 and epoch % config.save_steps == 0:
                self.save(ckpt)
            if exact:       # full-expectation steps on V(G, D): no walks, so no removal bits, passes or shuffles change
                roots = self.exact_roots()
                self._exact_phase("D", self.exact_d_phase(roots, config.n_epochs_dis))
                self._exact_phase("G", [self.exact_g_step(roots) for _ in range(config.n_epochs_gen)])
                self.write_embeddings_to_file()
                self.evaluation(self)
                continue
            # D-steps
            center_nodes = neighbor_nodes = labels = None
            for d_epoch in range(config.n_epochs_dis):
                if d_epoch % config.dis_interval == 0:
                    center_nodes, neighbor_nodes, labels = self.prepare_data_for_d()
                train_size = len(center_nodes)
                start_list = list(range(0, train_size, config.batch_size_dis))
                self.shuffle_rng.shuffle(start_list)
                # the per-batch sess.run loop of graph_gan.py:152-157, enqueued from C (identical steps)
                if self.dist:
                    self._dp_d.train_steps(center_nodes, neighbor_nodes, labels, start_list, config.batch_size_dis)
                else:
                    self.discriminator.train_steps(center_nodes, neighbor_nodes, labels, start_list, config.batch_size_dis)
            # G-steps
            node_1 = node_2 = reward = None
            for g_epoch in range(config.n_epochs_gen):
                if g_epoch % config.gen_interval == 0:
                    node_1, node_2, reward = self.prepare_data_for_g()
                train_size = len(node_1)
                start_list = list(range(0, train_size, config.batch_size_gen))
                self.shuffle_rng.shuffle(start_list)
                if self.dist:
                    self._dp_g.train_steps(node_1, node_2, reward, start_list, config.batch_size_gen)
                else:
                    self.generator.train_steps(node_1, node_2, reward, start_list, config.batch_size_gen)   # graph_gan.py:171-176
            self.write_embeddings_to_file()
            self.evaluation(self)
        print("training completes")

    # ------------------------------------------------------------------ graph_gan.py:293-319
    def write_embeddings_to_file(self):
        if self.rank != 0:      # replicas are bit-identical; one writer
            return
        modes = [self.generator, self.discriminator]
        for i in range(2):
            os.makedirs(os.path.dirname(config.emb_filenames[i]) or ".", exist_ok=True)
            if config.binary_embeddings:      # [N, n_emb] fp32 straight from the device (the text form is minutes at N = 1M)
                io.write_embeddings_binary(config.emb_filenames[i] + ".f32", modes[i])
            if config.text_embeddings:
                io.write_embeddings(config.emb_filenames[i], self.sess.run(modes[i].embedding_matrix))

    @staticmethod
    def evaluation(self):
        results = []
        if getattr(self, "rank", 0) != 0:
            return results
        if config.app == "link_prediction":
            modes = [self.generator, self.discriminator]
            for i in range(2):
                if config.device_eval:        # from the device-resident embeddings (csrc/eval.cu): no text round trip
                    lpe = lp.DeviceLinkPredictEval(modes[i], config.test_filename, config.test_neg_filename)
                else:
                    lpe = lp.LinkPredictEval(config.emb_filenames[i], config.test_filename, config.test_neg_filename,
                                             self.n_node, config.n_emb)
                results.append(config.modes[i] + ":" + str(lpe.eval_link_prediction()) + "\n")
        if getattr(config, "value_roots", 0) > 0:
            results.append(self.value_line())
        os.makedirs(os.path.dirname(config.result_filename) or ".", exist_ok=True)
        with open(config.result_filename, mode="a+") as f:
            f.writelines(results)
        return results

    # ------------------------------------------------------------------ checkpoint (tf.train.Saver stand-in)
    def save(self, path):
        """Replicas are bit-identical, so rank 0 alone writes (to a temporary file, then an atomic rename).  The
        father-removal bits (graph_gan.py:258-259) are per root, i.e. per rank shard: they are OR-reduced over the
        ranks first, so the file holds the removals of every root."""
        torch = self.torch
        bits = self.device_graph.d1_bits.clone()
        if self.dist:       # OR over the ranks (NCCL has no bitwise reduction: gather, then OR locally)
            parts = [torch.empty_like(bits) for _ in range(self.world)]
            self.dist.all_gather(parts, bits)
            for p_ in parts:
                bits |= p_
        if self.rank == 0:
            os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
            rs = self.shuffle_rng.get_state()
            state = {"generator": self.generator.state_dict(), "discriminator": self.discriminator.state_dict(),
                     "d1_bits": bits.cpu(), "pass_counter": torch.tensor(self.pass_counter),
                     "shuffle_rng": {"keys": torch.from_numpy(rs[1].astype(np.int64)), "pos": int(rs[2]),
                                     "has_gauss": int(rs[3]), "cached_gaussian": float(rs[4])}}
            tmp = "%s.tmp.%d" % (path, os.getpid())
            torch.save(state, tmp)
            os.replace(tmp, path)
        if self.dist:
            self.dist.barrier()

    def load(self, path):
        """Every rank reads the same file; the OR-ed removal bits only add bits for roots of other shards, which this
        rank's walks never look at."""
        sd = self.torch.load(path, weights_only=True, map_location="cpu")
        self.generator.load_state_dict(sd["generator"])
        self.discriminator.load_state_dict(sd["discriminator"])
        self.device_graph.d1_bits.copy_(sd["d1_bits"].to(self.device))
        self.pass_counter = int(sd["pass_counter"])
        r = sd["shuffle_rng"]
        self.shuffle_rng.set_state(("MT19937", r["keys"].numpy().astype(np.uint32), r["pos"], r["has_gauss"],
                                    r["cached_gaussian"]))
