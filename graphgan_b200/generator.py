"""``Generator`` with the reference's constructor and attribute surface (src/GraphGAN/generator.py:5-31).

Attributes that are TF tensors/ops in the reference are opaque ``Fetch`` handles here, evaluated by
``session.Session.run(fetch, feed_dict)``; the parameters live in HBM (model.PairModel).  The new
trainer calls the batched methods (``step``, ``all_score_matrix``) directly.
"""
from . import config
from .model import Fetch, PairModel, Placeholder


class Generator(PairModel):
    _step_mode = 1  # generator loss (generator.py:26-29)

    def __init__(self, n_node, node_emd_init, device=None):
        super().__init__(n_node, node_emd_init, lr=config.lr_gen, lam=config.lambda_gen, device=device)
        # generator.py:11-15
        self.embedding_matrix = Fetch(self, "embedding_matrix")
        self.bias_vector = Fetch(self, "bias_vector")
        # generator.py:17-19
        self.node_id = Placeholder(self, "node_id")
        self.node_neighbor_id = Placeholder(self, "node_neighbor_id")
        self.reward = Placeholder(self, "reward")
        # generator.py:21-26
        self.all_score = Fetch(self, "all_score")
        self.node_embedding = Fetch(self, "node_embedding")
        self.node_neighbor_embedding = Fetch(self, "node_neighbor_embedding")
        self.bias = Fetch(self, "bias")
        self.score = Fetch(self, "score")
        self.prob = Fetch(self, "prob")
        # generator.py:28-31
        self.loss = Fetch(self, "loss")
        self.g_updates = Fetch(self, "g_updates")

    def g_step(self, node_id, node_neighbor_id, reward):
        """sess.run(generator.g_updates, {node_id, node_neighbor_id, reward}) (graph_gan.py:173-176)."""
        self.step(node_id, node_neighbor_id, reward)

    def relevance(self, roots, nodes=None, sampler=None):
        """G(v | root) of the current generator: the exact probability that one generator walk from the root stops at v
        (csrc/gdist.cu, DESIGN.md section 5.1), under the graph's current father-removal bits.  ``sampler``: the
        sampler.WalkSampler of the graph (default: the one GraphGAN attaches as ``self.sampler``).
        nodes=None: device fp64 rows [len(roots), N]; otherwise ``nodes`` pairs with ``roots`` element by element and the
        result is dist[root_k, nodes_k] (fp64 [len(roots)]).  A root whose walks void has an all-zero row."""
        import numpy as np
        torch = self.torch
        smp = sampler if sampler is not None else getattr(self, "sampler", None)
        if smp is None:
            raise ValueError("relevance needs the graph's WalkSampler (pass sampler=...)")
        r = np.asarray(roots.cpu() if isinstance(roots, torch.Tensor) else roots, np.int64).reshape(-1)
        if nodes is None:
            dist, _ = smp.distribution(self.emb, self.bias_t, smp.build_trees(r.astype(np.int32)))
            return dist
        v = torch.as_tensor(np.asarray(nodes.cpu() if isinstance(nodes, torch.Tensor) else nodes, np.int64).reshape(-1))
        if v.shape[0] != r.shape[0]:
            raise ValueError("roots and nodes must have the same length")
        uniq, inv = np.unique(r, return_inverse=True)
        dist, _ = smp.distribution(self.emb, self.bias_t, smp.build_trees(uniq.astype(np.int32)))
        return dist[torch.as_tensor(inv).to(dist.device), v.to(dist.device)]
