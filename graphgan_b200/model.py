"""Device-resident pair model shared by Generator and Discriminator.

Holds what the reference's TF graph holds per model (generator.py:10-15 / discriminator.py:10-15
plus the AdamOptimizer slots created by ``minimize`` at generator.py:30-31 /
discriminator.py:31-32): embedding_matrix [N, ld] fp32 (zero padded to ld = round_up(n_emb, 32)),
bias_vector [N], Adam m/v for both and the beta powers -- and drives K2 / K3 through the C ABI.
"""
import ctypes as C

import numpy as np

from . import _cabi
from ._cabi import ptr
from .sampler import pad_embedding

MAX_BATCH = 1024  # GG_MAX_BATCH


class Fetch:
    """Opaque handle standing where the reference exposes a tf.Tensor / tf.Operation attribute."""

    def __init__(self, owner, kind):
        self.owner, self.kind = owner, kind

    def __repr__(self):
        return "<Fetch %s.%s>" % (type(self.owner).__name__, self.kind)


class Placeholder(Fetch):
    """tf.placeholder stand-in: only ever used as a feed_dict key."""


class PairModel:
    _step_mode = None  # 0 discriminator loss, 1 generator loss

    def __init__(self, n_node, node_emd_init, lr, lam, device=None):
        import torch
        from . import config
        self.torch = torch
        self.lib = _cabi.lib()
        self.n_node = n_node
        self.node_emd_init = node_emd_init
        dev = torch.device(device if device is not None else config.device)
        self.device = dev
        init = node_emd_init if isinstance(node_emd_init, torch.Tensor) else np.asarray(node_emd_init)
        assert init.shape[0] == n_node
        self.n_emb = int(init.shape[1])
        self.emb = pad_embedding(init, dev)                       # tf.get_variable("embedding", ...) fp32
        self.ld = int(self.emb.shape[1])
        self.bias_t = torch.zeros(n_node, dtype=torch.float32, device=dev)   # tf.Variable(tf.zeros([n_node]))
        z = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)
        self.m_emb, self.v_emb, self.m_bias, self.v_bias = z(n_node, self.ld), z(n_node, self.ld), z(n_node), z(n_node)
        self.row_slot = torch.full((n_node,), -1, dtype=torch.int32, device=dev)
        self.uniq_ids = torch.zeros(2 * MAX_BATCH, dtype=torch.int32, device=dev)
        self.n_unique = torch.zeros(1, dtype=torch.int32, device=dev)
        self.sync_words = torch.zeros(8, dtype=torch.int64, device=dev)     # flag, counter, cycle breakdown of gg_train_loop
        self.grad_rows = z(2 * MAX_BATCH, self.ld)
        self._emb2 = self._bias2 = None          # second parameter buffers of gg_train_fused (allocated on first use)
        self._scratch = None                     # multi-CTA gradient scratch (batches above GG_MAX_BATCH; first use)
        self.grad_bias = z(2 * MAX_BATCH)
        # tf.train.AdamOptimizer defaults
        self.lr, self.lam = np.float32(lr), np.float32(lam)
        self.beta1, self.beta2, self.eps = np.float32(0.9), np.float32(0.999), np.float32(1e-8)
        self.beta1_power, self.beta2_power = self.beta1, self.beta2
        self.step_count = 0

    # ------------------------------------------------------------------ helpers
    def _dev_i32(self, a):
        torch = self.torch
        if isinstance(a, torch.Tensor):
            return a.to(device=self.device, dtype=torch.int32).contiguous()
        return torch.as_tensor(np.ascontiguousarray(np.asarray(a), dtype=np.int32)).to(self.device)

    def _dev_f32(self, a):
        torch = self.torch
        if isinstance(a, torch.Tensor):
            return a.to(device=self.device, dtype=torch.float32).contiguous()
        return torch.as_tensor(np.ascontiguousarray(np.asarray(a), dtype=np.float32)).to(self.device)

    def _stream(self):
        return self.torch.cuda.current_stream(self.device).cuda_stream

    def lr_t(self):
        """lr * sqrt(1 - beta2^t) / (1 - beta1^t), fp32 like TF's graph computes it."""
        one = np.float32(1)
        return np.float32(self.lr * np.sqrt(one - self.beta2_power) / (one - self.beta1_power))

    # ------------------------------------------------------------------ K2 + K3: one optimizer step
    def step(self, node_id, node_neighbor_id, aux):
        """sess.run(d_updates | g_updates, feed_dict) of graph_gan.py:154-157 / 173-176."""
        i, j, a = self._dev_i32(node_id), self._dev_i32(node_neighbor_id), self._dev_f32(aux)
        B = int(i.shape[0])
        if B == 0:
            return
        st = self._stream()
        if B > MAX_BATCH:
            scratch = self._large_batch_buffers(B)
            _cabi.check(self.lib.gg_pair_grad_ex(self._step_mode, B, 0, ptr(i), ptr(j), ptr(a), ptr(self.emb), ptr(self.bias_t),
                                                 self.ld, C.c_float(float(self.lam)), ptr(self.n_unique), ptr(self.uniq_ids),
                                                 ptr(self.grad_rows), ptr(self.grad_bias), ptr(self.row_slot), ptr(scratch),
                                                 scratch.numel(), 0, st), "gg_pair_grad_ex")
            self.apply_adam()
            return
        _cabi.check(self.lib.gg_pair_grad(self._step_mode, B, 0, ptr(i), ptr(j), ptr(a), ptr(self.emb), ptr(self.bias_t),
                                          self.ld, C.c_float(float(self.lam)), ptr(self.n_unique), ptr(self.uniq_ids),
                                          ptr(self.grad_rows), ptr(self.grad_bias), ptr(self.row_slot), st),
                    "gg_pair_grad")
        self.apply_adam()

    def train_steps(self, node_id, node_neighbor_id, aux, start_list, batch_size, persistent=None):
        """All optimizer steps of one inner epoch (graph_gan.py:149-157 / 168-176): ``start_list`` is the shuffled
        list of batch starts; rows come from the device arrays.  Identical to calling ``step`` per batch.  Batches above
        GG_MAX_BATCH pairs run in the C loop (the persistent loops keep a one-CTA gradient)."""
        if batch_size > MAX_BATCH and persistent:
            raise ValueError("the persistent step loops take at most GG_MAX_BATCH=%d pairs per batch, not %d (use persistent=None)"
                             % (MAX_BATCH, batch_size))
        i, j, a = self._dev_i32(node_id), self._dev_i32(node_neighbor_id), self._dev_f32(aux)
        starts = np.ascontiguousarray(np.asarray(start_list, np.int64))
        if starts.size == 0:
            return
        b1p, b2p = C.c_float(float(self.beta1_power)), C.c_float(float(self.beta2_power))
        if batch_size > MAX_BATCH:
            scratch = self._large_batch_buffers(batch_size)
            _cabi.check(self.lib.gg_train_steps_ex(self._step_mode, int(i.shape[0]), starts.ctypes.data_as(C.c_void_p),
                                                   int(starts.size), int(batch_size), ptr(i), ptr(j), ptr(a), self.n_node, self.ld,
                                                   ptr(self.emb), ptr(self.m_emb), ptr(self.v_emb), ptr(self.bias_t), ptr(self.m_bias),
                                                   ptr(self.v_bias), C.c_float(float(self.lam)), ptr(self.n_unique), ptr(self.uniq_ids),
                                                   ptr(self.grad_rows), ptr(self.grad_bias), ptr(self.row_slot), C.c_float(float(self.lr)),
                                                   C.c_float(float(self.beta1)), C.c_float(float(self.beta2)), C.c_float(float(self.eps)),
                                                   C.byref(b1p), C.byref(b2p), ptr(scratch), scratch.numel(), self._stream()),
                        "gg_train_steps_ex")
            self.beta1_power, self.beta2_power = np.float32(b1p.value), np.float32(b2p.value)
            self.step_count += int(starts.size)
            return
        if persistent is None:
            # the persistent loops win while the sweep is small (C1, 4 MB of E/m/v: 11.0 us/step fused, 13.9 two-barrier, 18.4
            # as two launches per step); from ~60 MB on the sweep is faster as its own full-occupancy launch (N = 40k,
            # ld = 128: 42.9 us against 45.5; N = 1M: 0.83 ms against 1.0 ms)
            persistent = 12 * self.n_node * self.ld <= (16 << 20)
        if persistent:
            starts_d = self.torch.as_tensor(starts).to(self.device)
            if persistent == "two-barrier":   # gg_train_loop: CTA 0 computes the gradient, flag, sweep, counter
                _cabi.check(self.lib.gg_train_loop(self._step_mode, int(i.shape[0]), ptr(starts_d), int(starts.size),
                                                   int(batch_size), ptr(i), ptr(j), ptr(a), self.n_node, self.ld, ptr(self.emb),
                                                   ptr(self.m_emb), ptr(self.v_emb), ptr(self.bias_t), ptr(self.m_bias), ptr(self.v_bias),
                                                   C.c_float(float(self.lam)), ptr(self.n_unique), ptr(self.uniq_ids), ptr(self.grad_rows),
                                                   ptr(self.grad_bias), ptr(self.row_slot), C.c_float(float(self.lr)),
                                                   C.c_float(float(self.beta1)), C.c_float(float(self.beta2)), C.c_float(float(self.eps)),
                                                   C.byref(b1p), C.byref(b2p), ptr(self.sync_words), self._stream()), "gg_train_loop")
            else:                              # gg_train_fused: one barrier per step, parameters ping-pong
                if self._emb2 is None:
                    self._emb2, self._bias2 = self.torch.empty_like(self.emb), self.torch.empty_like(self.bias_t)
                _cabi.check(self.lib.gg_train_fused(self._step_mode, int(i.shape[0]), ptr(starts_d), int(starts.size),
                                                    int(batch_size), ptr(i), ptr(j), ptr(a), self.n_node, self.ld, ptr(self.emb),
                                                    ptr(self.m_emb), ptr(self.v_emb), ptr(self.bias_t), ptr(self.m_bias), ptr(self.v_bias),
                                                    ptr(self._emb2), ptr(self._bias2), C.c_float(float(self.lam)),
                                                    C.c_float(float(self.lr)), C.c_float(float(self.beta1)), C.c_float(float(self.beta2)),
                                                    C.c_float(float(self.eps)), C.byref(b1p), C.byref(b2p), ptr(self.sync_words),
                                                    self._stream()), "gg_train_fused")
            self._keep = (starts_d, i, j, a)     # keep the device arrays alive until the stream has consumed them
            self.beta1_power, self.beta2_power = np.float32(b1p.value), np.float32(b2p.value)
            self.step_count += int(starts.size)
            return
        _cabi.check(self.lib.gg_train_steps(self._step_mode, int(i.shape[0]), starts.ctypes.data_as(C.c_void_p), int(starts.size),
                                            int(batch_size), ptr(i), ptr(j), ptr(a), self.n_node, self.ld, ptr(self.emb),
                                            ptr(self.m_emb), ptr(self.v_emb), ptr(self.bias_t), ptr(self.m_bias), ptr(self.v_bias),
                                            C.c_float(float(self.lam)), ptr(self.n_unique), ptr(self.uniq_ids), ptr(self.grad_rows),
                                            ptr(self.grad_bias), ptr(self.row_slot), C.c_float(float(self.lr)),
                                            C.c_float(float(self.beta1)), C.c_float(float(self.beta2)), C.c_float(float(self.eps)),
                                            C.byref(b1p), C.byref(b2p), self._stream()), "gg_train_steps")
        self.beta1_power, self.beta2_power = np.float32(b1p.value), np.float32(b2p.value)
        self.step_count += int(starts.size)

    def _large_batch_buffers(self, B, scratch_bytes=None):
        """Grow uniq_ids / grad_rows / grad_bias to 2B entries and the scratch to `scratch_bytes` (default: the multi-CTA
        gradient's size at B); allocated on first use: models that never see a batch above GG_MAX_BATCH keep today's buffers."""
        torch = self.torch
        if self.uniq_ids.numel() < 2 * B:
            self.uniq_ids = torch.zeros(2 * B, dtype=torch.int32, device=self.device)
            self.grad_rows = torch.zeros((2 * B, self.ld), dtype=torch.float32, device=self.device)
            self.grad_bias = torch.zeros(2 * B, dtype=torch.float32, device=self.device)
        if scratch_bytes is None:
            n = C.c_int64(0)
            _cabi.check(self.lib.gg_pair_grad_scratch_bytes(int(B), self.ld, C.byref(n)), "gg_pair_grad_scratch_bytes")
            scratch_bytes = n.value
        if self._scratch is None or self._scratch.numel() < scratch_bytes:
            self._scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=self.device)   # caching allocator: 512-byte aligned
        return self._scratch

    def apply_adam(self):
        st = self._stream()
        _cabi.check(self.lib.gg_adam_apply(self.n_node, self.ld, ptr(self.emb), ptr(self.m_emb), ptr(self.v_emb),
                                           ptr(self.bias_t), ptr(self.m_bias), ptr(self.v_bias), ptr(self.n_unique),
                                           ptr(self.uniq_ids), ptr(self.grad_rows), ptr(self.grad_bias),
                                           ptr(self.row_slot), C.c_float(float(self.lr_t())), C.c_float(float(self.beta1)),
                                           C.c_float(float(self.beta2)), C.c_float(float(self.eps)), st), "gg_adam_apply")
        self.beta1_power = np.float32(self.beta1_power * self.beta1)
        self.beta2_power = np.float32(self.beta2_power * self.beta2)
        self.step_count += 1

    def apply_dense_grad(self, acc_emb, acc_bias, scale):
        """One Adam step from a dense fp64 gradient (DESIGN.md section 5.5): g = f32(scale * acc + lam * x) per element,
        with ``acc_emb`` fp64 [N, ld] and ``acc_bias`` fp64 [N] as game_value_grad / game_value_grad_d return them.  The
        L2 term is the model's own: lam on every row, and on every bias for the discriminator only (generator.py:28-29 has
        no bias L2).  Shares lr_t, the beta powers and step_count with apply_adam, so sampled and exact steps continue one
        Adam state."""
        torch = self.torch
        for a, shape in ((acc_emb, (self.n_node, self.ld)), (acc_bias, (self.n_node,))):
            if a.dtype != torch.float64 or tuple(a.shape) != shape or not a.is_contiguous() or a.device != self.emb.device:
                raise ValueError("apply_dense_grad takes contiguous fp64 device gradients of shape %s" % (shape,))
        lam_b = self.lam if self._step_mode == 0 else np.float32(0)
        _cabi.check(self.lib.gg_adam_apply_dense(self.n_node, self.ld, ptr(self.emb), ptr(self.m_emb), ptr(self.v_emb),
                                                 ptr(self.bias_t), ptr(self.m_bias), ptr(self.v_bias), ptr(acc_emb),
                                                 ptr(acc_bias), C.c_double(float(scale)), C.c_float(float(self.lam)),
                                                 C.c_float(float(lam_b)), C.c_float(float(self.lr_t())),
                                                 C.c_float(float(self.beta1)), C.c_float(float(self.beta2)),
                                                 C.c_float(float(self.eps)), self._stream()), "gg_adam_apply_dense")
        self.beta1_power = np.float32(self.beta1_power * self.beta1)
        self.beta2_power = np.float32(self.beta2_power * self.beta2)
        self.step_count += 1

    # ------------------------------------------------------------------ fetches
    def reward_pairs(self, node_id, node_neighbor_id):
        """log(1 + exp(clip(score, -10, 10))) for M pairs -> device fp32 [M] (discriminator.py:33-34)."""
        torch = self.torch
        i, j = self._dev_i32(node_id), self._dev_i32(node_neighbor_id)
        out = torch.empty(max(int(i.shape[0]), 1), dtype=torch.float32, device=self.device)
        _cabi.check(self.lib.gg_pair_reward(int(i.shape[0]), ptr(i), ptr(j), ptr(self.emb), ptr(self.bias_t), self.ld,
                                            ptr(out), self._stream()), "gg_pair_reward")
        return out[:int(i.shape[0])]

    def all_score_matrix(self):
        """generator.all_score (generator.py:21), materialised: small graphs only."""
        torch = self.torch
        out = torch.empty((self.n_node, self.n_node), dtype=torch.float32, device=self.device)
        _cabi.check(self.lib.gg_all_score(self.n_node, ptr(self.emb), ptr(self.bias_t), self.ld, ptr(out), self._stream()),
                    "gg_all_score")
        return out

    def embedding_numpy(self):
        """sess.run(model.embedding_matrix) (graph_gan.py:298) -> [N, n_emb] fp32."""
        return self.emb[:, :self.n_emb].cpu().numpy()

    # compatibility-only fetches (never fetched by the reference's training loop); torch indexing
    def _score_t(self, i, j):
        i, j = self._dev_i32(i).long(), self._dev_i32(j).long()
        return (self.emb[i] * self.emb[j]).sum(1) + self.bias_t[j]

    # ------------------------------------------------------------------ checkpoint (SURVEY section 5)
    def state_dict(self):
        return {"emb": self.emb.cpu(), "bias": self.bias_t.cpu(), "m_emb": self.m_emb.cpu(), "v_emb": self.v_emb.cpu(),
                "m_bias": self.m_bias.cpu(), "v_bias": self.v_bias.cpu(), "beta1_power": float(self.beta1_power),
                "beta2_power": float(self.beta2_power), "step_count": self.step_count, "n_emb": self.n_emb}

    def load_state_dict(self, sd):
        for name, key in (("emb", "emb"), ("bias_t", "bias"), ("m_emb", "m_emb"), ("v_emb", "v_emb"),
                          ("m_bias", "m_bias"), ("v_bias", "v_bias")):
            getattr(self, name).copy_(sd[key].to(self.device))
        self.beta1_power, self.beta2_power = np.float32(sd["beta1_power"]), np.float32(sd["beta2_power"])
        self.step_count = int(sd["step_count"])
