"""One process per GPU (torch.distributed / NCCL over NVLink): how the hot path shards.

SURVEY.md section 8e.  Sampling shards by ROOTS and needs no collective: every rank holds the replicated
graph and embeddings, takes a contiguous block of the root list, and -- because the walk RNG is Philox keyed
by (root, walk, step) -- produces exactly the rows a single GPU would produce for those roots.  Rows are
all-gathered so that every rank sees the same training set (the reference's lists, in root order).

Updates are data parallel: every rank scores its slice of the mini-batch (K2), ONE collective per step
exchanges the compact gradients (ids + summed rows; a few KB at 64 pairs, latency bound, NVLS-friendly), every rank
merges them in the same rank-major order (gg_grad_merge; gg_grad_merge_ex, multi-CTA, above GG_MAX_BATCH pairs) and
applies the same K3 Adam sweep, so replicas stay bit-identical without broadcasting parameters.  The step lives in
the C library (csrc/comm.cu: gg_dp_step, gg_dp_train_steps, and their _ex forms for any batch size) with a
library-owned NCCL communicator; torch.distributed only carries the 128-byte unique id.
"""
import ctypes as C

import numpy as np

from . import _cabi
from ._cabi import ptr
from .model import MAX_BATCH
from .sampler import LD_MAX


def block_range(n, rank, world):
    """Contiguous block of [0, n) owned by `rank` (sizes differ by at most one, rank order = item order)."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def balanced_root_ranges(weights, world):
    """Contiguous split of the root list into `world` blocks of roughly equal total weight (work of a root
    ~ its degree times the candidate lists it meets); keeps root order, so the concatenation of the ranks'
    rows equals the single-GPU row order."""
    w = np.asarray(weights, np.float64)
    cum = np.concatenate([[0.0], np.cumsum(w)])
    cuts = [int(np.searchsorted(cum, cum[-1] * r / world, side="left")) for r in range(world + 1)]
    cuts[0], cuts[-1] = 0, len(w)
    return [(min(cuts[r], cuts[r + 1]), cuts[r + 1]) for r in range(world)]


def all_gather_varlen(t, group=None):
    """Concatenate 1-D tensors of different lengths from every rank, in rank order (works on gloo and nccl)."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    n = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n, group=group)
    sizes = [int(s.item()) for s in sizes]
    m = max(sizes + [1])
    pad = torch.zeros(m, dtype=t.dtype, device=t.device)
    pad[:t.shape[0]] = t
    outs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(outs, pad, group=group)
    return torch.cat([o[:k] for o, k in zip(outs, sizes)])


def create_comm(group=None):
    """NCCL communicator OWNED BY THE C LIBRARY (csrc/comm.cu) over the ranks of `group`: rank 0 creates the unique id,
    torch.distributed (any backend) broadcasts its 128 bytes, every rank calls ncclCommInitRank on its current device."""
    import torch
    import torch.distributed as dist
    lib = _cabi.lib()
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    buf = C.create_string_buffer(128)
    if rank == 0:
        _cabi.check(lib.gg_comm_unique_id(buf), "gg_comm_unique_id")
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
    t = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone().to(dev)
    dist.broadcast(t, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    raw = bytes(t.cpu().numpy().tobytes())
    handle = C.c_void_p()
    _cabi.check(lib.gg_comm_init(C.create_string_buffer(raw, 128), rank, world, C.byref(handle)), "gg_comm_init")
    return handle


def connect_peer_memory(comm, capacity_floats, group=None):
    """Peer-memory transport of the data-parallel step (csrc/comm.cu): every rank creates its exchange buffer, the 64-byte
    CUDA IPC handles are all-gathered with torch.distributed, every rank maps its peers' buffers (NVLink P2P)."""
    import torch
    import torch.distributed as dist
    lib = _cabi.lib()
    world = dist.get_world_size(group)
    buf = C.create_string_buffer(64)
    _cabi.check(lib.gg_comm_p2p_export(comm, int(capacity_floats), buf), "gg_comm_p2p_export")
    dev = torch.device("cuda", torch.cuda.current_device())
    mine = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone().to(dev)
    allh = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(allh, mine, group=group)
    raw = b"".join(bytes(h.cpu().numpy().tobytes()) for h in allh)
    _cabi.check(lib.gg_comm_p2p_connect(comm, C.create_string_buffer(raw, 64 * world)), "gg_comm_p2p_connect")


class DataParallelStep:
    """Data-parallel replacement for PairModel.step / train_steps: same arguments (the WHOLE mini-batch, identical on
    every rank).  The step -- gradient of this rank's rows, ONE ncclAllGather of the compact gradients, rank-major merge,
    Adam sweep -- runs inside the C library on the caller's stream (gg_dp_step / gg_dp_train_steps)."""

    _comm = None        # one library-owned communicator per process
    _p2p_capacity = 0   # floats of the peer-memory exchange buffer (0: not connected)
    transport = None    # "nccl" or "p2p" once use() has run

    def __init__(self, model, group=None, transport="nccl"):
        import torch
        import torch.distributed as dist
        self.torch, self.dist, self.model, self.group = torch, dist, model, group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.lib = _cabi.lib()
        if DataParallelStep._comm is None:
            DataParallelStep._comm = create_comm(group)
        self.comm = DataParallelStep._comm
        self._cap = None
        self.transport = None
        self.use(transport)

    def use(self, transport):
        """"nccl": one ncclAllGather per step; "p2p": the gradient kernel itself stores into every peer's exchange buffer
        over NVLink (CUDA IPC mapped) and the merge kernel waits on flags -- no collective call.  Same results bit for bit."""
        assert transport in ("nccl", "p2p")
        if transport == "p2p" and DataParallelStep._p2p_capacity == 0:
            # batches up to 256 pairs at any row stride (ld up to LD_MAX)
            cap_floats = self.world * int(self.lib.gg_grad_buf_floats(2 * (-(-256 // self.world)), LD_MAX))
            connect_peer_memory(self.comm, cap_floats, self.group)
            DataParallelStep._p2p_capacity = cap_floats
        self.transport = transport

    def _check_batch(self, B):
        """Above GG_MAX_BATCH pairs only the NCCL transport has a path (multi-CTA gradient and merge); the peer-memory
        exchange is sized for small batches and fused into a one-CTA kernel.  Refuse before communicating."""
        if B > MAX_BATCH and self.transport != "nccl":
            raise ValueError("data-parallel steps above GG_MAX_BATCH=%d pairs per batch (here %d) need the nccl transport, not %s"
                             % (MAX_BATCH, B, self.transport))

    def _large_batch_scratch(self, B):
        """Model gradient buffers of 2B entries and the scratch of gg_dp_scratch_bytes (shared with PairModel's)."""
        m, n = self.model, C.c_int64(0)
        _cabi.check(self.lib.gg_dp_scratch_bytes(self.world, int(B), m.ld, C.byref(n)), "gg_dp_scratch_bytes")
        return m._large_batch_buffers(int(B), n.value)

    def _select(self):
        _cabi.check(self.lib.gg_comm_use_p2p(self.comm, 1 if self.transport == "p2p" else 0), "gg_comm_use_p2p")

    def _buffers(self, cap):
        torch, m = self.torch, self.model
        if self._cap != cap:
            nf = int(self.lib.gg_grad_buf_floats(cap, m.ld))
            self.local = torch.zeros(nf, dtype=torch.float32, device=m.device)
            self.gathered = torch.empty(self.world * nf, dtype=torch.float32, device=m.device)
            self._cap, self._nf = cap, nf
        return self.local, self.gathered

    def step(self, node_id, node_neighbor_id, aux):
        m = self.model
        i, j, a = m._dev_i32(node_id), m._dev_i32(node_neighbor_id), m._dev_f32(aux)
        B = int(i.shape[0])
        if B == 0:
            return
        self._check_batch(B)
        cap = 2 * (-(-B // self.world))
        local, gathered = self._buffers(cap)
        self._select()
        f = lambda x: C.c_float(float(x))
        if B > MAX_BATCH:
            scratch = self._large_batch_scratch(B)
            _cabi.check(self.lib.gg_dp_step_ex(self.comm, m._step_mode, B, ptr(i), ptr(j), ptr(a), m.n_node, m.ld, ptr(m.emb),
                                               ptr(m.m_emb), ptr(m.v_emb), ptr(m.bias_t), ptr(m.m_bias), ptr(m.v_bias), f(m.lam),
                                               ptr(local), ptr(gathered), cap, ptr(m.n_unique), ptr(m.uniq_ids), ptr(m.grad_rows),
                                               ptr(m.grad_bias), ptr(m.row_slot), f(m.lr_t()), f(m.beta1), f(m.beta2), f(m.eps),
                                               ptr(scratch), scratch.numel(), 0, m._stream()), "gg_dp_step_ex")
            m.beta1_power = np.float32(m.beta1_power * m.beta1)
            m.beta2_power = np.float32(m.beta2_power * m.beta2)
            m.step_count += 1
            return
        _cabi.check(self.lib.gg_dp_step(self.comm, m._step_mode, B, ptr(i), ptr(j), ptr(a), m.n_node, m.ld, ptr(m.emb), ptr(m.m_emb),
                                        ptr(m.v_emb), ptr(m.bias_t), ptr(m.m_bias), ptr(m.v_bias), f(m.lam), ptr(local), ptr(gathered),
                                        cap, ptr(m.n_unique), ptr(m.uniq_ids), ptr(m.grad_rows), ptr(m.grad_bias), ptr(m.row_slot),
                                        f(m.lr_t()), f(m.beta1), f(m.beta2), f(m.eps), m._stream()), "gg_dp_step")
        m.beta1_power = np.float32(m.beta1_power * m.beta1)
        m.beta2_power = np.float32(m.beta2_power * m.beta2)
        m.step_count += 1

    def train_steps(self, node_id, node_neighbor_id, aux, start_list, batch_size):
        """All steps of one inner epoch (graph_gan.py:149-157 / 168-176) enqueued from C, one collective each."""
        self._check_batch(batch_size)
        m = self.model
        i, j, a = m._dev_i32(node_id), m._dev_i32(node_neighbor_id), m._dev_f32(aux)
        starts = np.ascontiguousarray(np.asarray(start_list, np.int64))
        if starts.size == 0:
            return
        cap = 2 * (-(-int(batch_size) // self.world))
        local, gathered = self._buffers(cap)
        self._select()
        f = lambda x: C.c_float(float(x))
        b1p, b2p = f(m.beta1_power), f(m.beta2_power)
        if batch_size > MAX_BATCH:
            scratch = self._large_batch_scratch(batch_size)
            _cabi.check(self.lib.gg_dp_train_steps_ex(self.comm, m._step_mode, int(i.shape[0]), starts.ctypes.data_as(C.c_void_p),
                                                      int(starts.size), int(batch_size), ptr(i), ptr(j), ptr(a), m.n_node, m.ld,
                                                      ptr(m.emb), ptr(m.m_emb), ptr(m.v_emb), ptr(m.bias_t), ptr(m.m_bias),
                                                      ptr(m.v_bias), f(m.lam), ptr(local), ptr(gathered), cap, ptr(m.n_unique),
                                                      ptr(m.uniq_ids), ptr(m.grad_rows), ptr(m.grad_bias), ptr(m.row_slot), f(m.lr),
                                                      f(m.beta1), f(m.beta2), f(m.eps), C.byref(b1p), C.byref(b2p), ptr(scratch),
                                                      scratch.numel(), 0, m._stream()), "gg_dp_train_steps_ex")
        else:
            _cabi.check(self.lib.gg_dp_train_steps(self.comm, m._step_mode, int(i.shape[0]), starts.ctypes.data_as(C.c_void_p),
                                                   int(starts.size), int(batch_size), ptr(i), ptr(j), ptr(a), m.n_node, m.ld,
                                                   ptr(m.emb), ptr(m.m_emb), ptr(m.v_emb), ptr(m.bias_t), ptr(m.m_bias), ptr(m.v_bias),
                                                   f(m.lam), ptr(local), ptr(gathered), cap, ptr(m.n_unique), ptr(m.uniq_ids),
                                                   ptr(m.grad_rows), ptr(m.grad_bias), ptr(m.row_slot), f(m.lr), f(m.beta1), f(m.beta2),
                                                   f(m.eps), C.byref(b1p), C.byref(b2p), m._stream()), "gg_dp_train_steps")
        self._keep = (i, j, a)
        m.beta1_power, m.beta2_power = np.float32(b1p.value), np.float32(b2p.value)
        m.step_count += int(starts.size)

    def stats(self):
        r, w, v, n = C.c_int32(0), C.c_int32(0), C.c_int32(0), C.c_uint64(0)
        _cabi.check(self.lib.gg_comm_info(self.comm, C.byref(r), C.byref(w), C.byref(v), C.byref(n)), "gg_comm_info")
        return {"rank": r.value, "comm_nranks": w.value, "nccl_version": v.value, "collectives_issued": int(n.value),
                "bytes_per_rank_per_step": 4 * int(getattr(self, "_nf", 0)), "transport": self.transport,
                "kind": "ncclAllGather (fp32) inside gg_dp_step" if self.transport == "nccl" else
                        "peer stores into every rank's exchange buffer from the gradient kernel + flag wait in the merge kernel (gg_dp_step, p2p)"}
