"""ctypes binding of libgraphgan_b200.so (include/graphgan_b200.h).

This is the whole FFI: plain pointers, sizes and one POD descriptor.  There is no CPU
fallback -- if the shared object cannot be built or loaded, importing a product module that
needs it raises."""
import ctypes as C
import os

from . import _build

_LIB = None
ABI_VERSION = 11   # == GG_ABI_VERSION of include/graphgan_b200.h


class GGError(RuntimeError):
    pass


class WalkDesc(C.Structure):
    """struct gg_walk_desc (include/graphgan_b200.h)."""
    _fields_ = [
        ("n_node", C.c_int64), ("ld", C.c_int32),
        ("emb", C.c_void_p), ("bias", C.c_void_p), ("indptr", C.c_void_p), ("adj", C.c_void_p),
        ("n_roots", C.c_int64), ("roots", C.c_void_p), ("tree_bits", C.c_void_p), ("tree_words", C.c_int64),
        ("walk_ptr", C.c_void_p),
        ("n_walks", C.c_int64), ("for_d", C.c_int32), ("rng_mode", C.c_int32), ("d1_bits", C.c_void_p),
        ("seed", C.c_uint64), ("pass_tag", C.c_uint32), ("max_path", C.c_int32),
        ("stream", C.c_void_p), ("n_stream", C.c_int64), ("update_ratio", C.c_double),
        ("max_cand", C.c_int32), ("phase_mask", C.c_int32),
        ("samples", C.c_void_p), ("status", C.c_void_p), ("first_edge", C.c_void_p), ("wsteps", C.c_void_p),
        ("wsuml", C.c_void_p), ("paths", C.c_void_p), ("path_len", C.c_void_p), ("counters", C.c_void_p),
        ("scratch", C.c_void_p), ("scratch_bytes", C.c_int64), ("work_counter", C.c_void_p),
        ("edge_score", C.c_void_p), ("root_q", C.c_void_p), ("rq_ptr", C.c_void_p),
        ("hub_threshold", C.c_int32), ("no_tma", C.c_int32), ("walk_slot", C.c_void_p),
        ("s1_nq", C.c_int64), ("s1_slot", C.c_void_p), ("s1_ptr", C.c_void_p), ("s1_cnt", C.c_void_p), ("s1_n", C.c_void_p),
        ("s1_q", C.c_void_p), ("s1_ids", C.c_void_p), ("first_idx", C.c_void_p), ("s1_order", C.c_void_p), ("walk_order", C.c_void_p),
        ("flat_buf", C.c_void_p), ("flat_bytes", C.c_int64), ("flat_steps", C.c_int32), ("flat_reserved", C.c_int32),
    ]


# name -> (restype, argtypes); every symbol include/graphgan_b200.h declares
_P, _I32, _I64, _F = C.c_void_p, C.c_int32, C.c_int64, C.c_float
SIGNATURES = {
    "gg_last_error": (C.c_char_p, []),
    "gg_abi_version": (C.c_int, []),
    "gg_hub_scores": (C.c_int, [_I64, _P, _P, _P, _P, _I32, _P, _P]),
    "gg_root_cdf": (C.c_int, [C.POINTER(WalkDesc), _P, _P, _P]),
    "gg_walk_scratch_bytes": (C.c_int, [_I32, C.POINTER(_I64)]),
    "gg_walk_flat_bytes": (C.c_int, [_I64, _I32, _I32, C.POINTER(_I64)]),
    "gg_walk_sample": (C.c_int, [C.POINTER(WalkDesc), _P]),
    "gg_generator_dist_scratch_bytes": (C.c_int, [_I64, _I64, _I64, C.POINTER(_I64)]),
    "gg_generator_dist": (C.c_int, [C.POINTER(WalkDesc), _P, _P, _P, _I64, _P]),
    "gg_generator_dist_d": (C.c_int, [C.POINTER(WalkDesc), _P, _P, _P, _P, _I64, _P]),
    "gg_game_value_scratch_bytes": (C.c_int, [_I64, _I64, C.POINTER(_I64)]),
    "gg_game_value": (C.c_int, [_I64, _I32, _P, _P, _P, _P, _I64, _P, _P, _P, _P, _P, _P, _P, _I64, _P]),
    "gg_game_value_grad_scratch_bytes": (C.c_int, [_I64, _I64, _I64, C.POINTER(_I64)]),
    "gg_game_value_grad": (C.c_int, [C.POINTER(WalkDesc), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I64, _P]),
    "gg_game_value_grad_d_scratch_bytes": (C.c_int, [_I64, _I32, _I64, C.POINTER(_I64)]),
    "gg_game_value_grad_d": (C.c_int, [_I64, _I32, _P, _P, _P, _P, _I64, _P, _P, _P, _P, _P, _P, _I64, _P]),
    "gg_expected_g_grad_scratch_bytes": (C.c_int, [_I64, _I64, _I64, _I32, C.POINTER(_I64)]),
    "gg_expected_g_grad": (C.c_int, [C.POINTER(WalkDesc), _P, _P, _I32, _P, _P, _P, _P, _P, _I64, _P]),
    "gg_expected_g_moments_scratch_bytes": (C.c_int, [_I64, _I64, _I64, _I32, C.POINTER(_I64)]),
    "gg_expected_g_moments": (C.c_int, [C.POINTER(WalkDesc), _P, _P, _I32, _P, _P, _P, _P, _P, _P, _P, _P, _I64, _P]),
    "gg_expected_d_grad_scratch_bytes": (C.c_int, [_I64, _I32, _I64, C.POINTER(_I64)]),
    "gg_expected_d_grad": (C.c_int, [_I64, _I32, _P, _P, _P, _P, _I64, _P, _P, _P, _P, _P, _P, _P, _P, _I64, _P]),
    "gg_best_response_scratch_bytes": (C.c_int, [_I64, _I64, _I64, C.POINTER(_I64)]),
    "gg_best_response": (C.c_int, [C.POINTER(WalkDesc), _P, _P, _P, _P, _P, _P, _I64, _P]),
    "gg_best_response_grad_scratch_bytes": (C.c_int, [_I64, _I64, _I64, C.POINTER(_I64)]),
    "gg_best_response_grad": (C.c_int, [C.POINTER(WalkDesc), _P, _P, _P, _P, _P, _P, _P, _P, _P, _I64, _P]),
    "gg_best_response_spmm": (C.c_int, [_I64, _I32, _P, _P, _P, _P, _P, _P, _P, _P]),
    "gg_walk_finalize": (C.c_int, [_I64, _P, _I32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "gg_emit_d_rows": (C.c_int, [_I64, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "gg_bfs_scratch_bytes": (C.c_int, [_I64, _I64, C.POINTER(_I64)]),
    "gg_tree_words": (C.c_int, [_I64, C.POINTER(_I64)]),
    "gg_bfs_build": (C.c_int, [_I64, _I64, _P, _P, _I64, _P, _P, _I64, _P, _I64, _P]),
    "gg_reverse_entries": (C.c_int, [_I64, _I64, _P, _P, _P, _P, _P]),
    "gg_bfs_build_ex": (C.c_int, [_I64, _I64, _P, _P, _P, _I64, _P, _P, _I64, _P, _I64, C.c_float, C.c_int32, _P]),
    "gg_tree_parent": (C.c_int, [_I64, _P, _P, _I64, _P, _P, _I64, _P, _P]),
    "gg_pair_reward": (C.c_int, [_I64, _P, _P, _P, _P, _I32, _P, _P]),
    "gg_all_score": (C.c_int, [_I64, _P, _P, _I32, _P, _P]),
    "gg_pair_grad": (C.c_int, [_I32, _I32, _I32, _P, _P, _P, _P, _P, _I32, _F, _P, _P, _P, _P, _P, _P]),
    "gg_pair_grad_scratch_bytes": (C.c_int, [_I32, _I32, C.POINTER(_I64)]),
    "gg_pair_grad_ex": (C.c_int, [_I32, _I32, _I32, _P, _P, _P, _P, _P, _I32, _F, _P, _P, _P, _P, _P, _P, _I64, _I32, _P]),
    "gg_grad_buf_floats": (_I64, [_I32, _I32]),
    "gg_grad_merge": (C.c_int, [_I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _P]),
    "gg_grad_merge_scratch_bytes": (C.c_int, [_I32, _I32, _I32, C.POINTER(_I64)]),
    "gg_grad_merge_ex": (C.c_int, [_I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _P, _I64, _I32, _P]),
    "gg_comm_unique_id": (C.c_int, [_P]),
    "gg_comm_init": (C.c_int, [_P, _I32, _I32, C.POINTER(C.c_void_p)]),
    "gg_comm_destroy": (C.c_int, [_P]),
    "gg_comm_info": (C.c_int, [_P, C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I32), C.POINTER(C.c_uint64)]),
    "gg_comm_p2p_export": (C.c_int, [_P, _I64, _P]),
    "gg_comm_p2p_connect": (C.c_int, [_P, _P]),
    "gg_comm_use_p2p": (C.c_int, [_P, _I32]),
    "gg_dp_step": (C.c_int, [_P, _I32, _I32, _P, _P, _P, _I64, _I32, _P, _P, _P, _P, _P, _P, _F, _P, _P, _I32, _P, _P, _P, _P, _P,
                            _F, _F, _F, _F, _P]),
    "gg_dp_train_steps": (C.c_int, [_P, _I32, _I64, _P, _I64, _I32, _P, _P, _P, _I64, _I32, _P, _P, _P, _P, _P, _P, _F, _P, _P, _I32,
                                   _P, _P, _P, _P, _P, _F, _F, _F, _F, C.POINTER(C.c_float), C.POINTER(C.c_float), _P]),
    "gg_dp_scratch_bytes": (C.c_int, [_I32, _I32, _I32, C.POINTER(_I64)]),
    "gg_dp_step_ex": (C.c_int, [_P, _I32, _I32, _P, _P, _P, _I64, _I32, _P, _P, _P, _P, _P, _P, _F, _P, _P, _I32, _P, _P, _P, _P, _P,
                               _F, _F, _F, _F, _P, _I64, _I32, _P]),
    "gg_dp_train_steps_ex": (C.c_int, [_P, _I32, _I64, _P, _I64, _I32, _P, _P, _P, _I64, _I32, _P, _P, _P, _P, _P, _P, _F, _P, _P, _I32,
                                      _P, _P, _P, _P, _P, _F, _F, _F, _F, C.POINTER(C.c_float), C.POINTER(C.c_float), _P, _I64,
                                      _I32, _P]),
    "gg_set_adam_path": (C.c_int, [C.c_char_p]),
    "gg_adam_apply": (C.c_int, [_I64, _I32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _F, _F, _F, _F, _P]),
    "gg_adam_apply_dense": (C.c_int, [_I64, _I32, _P, _P, _P, _P, _P, _P, _P, _P, C.c_double, _F, _F, _F, _F, _F, _F, _P]),
    "gg_train_steps": (C.c_int, [_I32, _I64, _P, _I64, _I32, _P, _P, _P, _I64, _I32, _P, _P, _P, _P, _P, _P, _F, _P, _P, _P, _P, _P,
                                _F, _F, _F, _F, C.POINTER(C.c_float), C.POINTER(C.c_float), _P]),
    "gg_train_steps_ex": (C.c_int, [_I32, _I64, _P, _I64, _I32, _P, _P, _P, _I64, _I32, _P, _P, _P, _P, _P, _P, _F, _P, _P, _P, _P, _P,
                                   _F, _F, _F, _F, C.POINTER(C.c_float), C.POINTER(C.c_float), _P, _I64, _P]),
    "gg_train_loop": (C.c_int, [_I32, _I64, _P, _I64, _I32, _P, _P, _P, _I64, _I32, _P, _P, _P, _P, _P, _P, _F, _P, _P, _P, _P, _P,
                               _F, _F, _F, _F, C.POINTER(C.c_float), C.POINTER(C.c_float), _P, _P]),
    "gg_train_fused": (C.c_int, [_I32, _I64, _P, _I64, _I32, _P, _P, _P, _I64, _I32, _P, _P, _P, _P, _P, _P, _P, _P, _F,
                                _F, _F, _F, _F, C.POINTER(C.c_float), C.POINTER(C.c_float), _P, _P]),
    "gg_pair_dot_f64": (C.c_int, [_I64, _P, _P, _P, _I32, _P, _P]),
    "gg_link_pred_acc": (C.c_int, [_I64, _P, _P, _P]),
    "gg_unpad_rows": (C.c_int, [_I64, _I32, _I32, _P, _P, _P]),
    "gg_window_pairs": (C.c_int, [_I64, _P, _P, _I32, _I32, _P, _P, _P, _P, _I64, _P]),
}


def lib():
    """Load (building first if the .so is absent).  Raises GGError on any failure."""
    global _LIB
    if _LIB is None:
        path = os.environ.get("GG_LIB") or _build.LIB      # GG_LIB: an A/B variant built by tools/variants.py
        if path == _build.LIB and _build.stale():      # missing, or built from other sources than the tree holds (content hash)
            if os.path.exists(path) and _build.nvcc_path() is None:
                raise GGError("libgraphgan_b200.so was built from different sources and there is no nvcc to rebuild it")
            try:
                _build.build()
            except Exception as e:  # noqa: BLE001
                raise GGError("libgraphgan_b200.so is missing or stale and could not be built: %s" % e) from e
        try:
            handle = C.CDLL(path)
        except OSError as e:
            raise GGError("cannot load %s: %s" % (path, e)) from e
        for name, (res, args) in SIGNATURES.items():
            try:
                fn = getattr(handle, name)
            except AttributeError as e:
                raise GGError("libgraphgan_b200.so does not export %s (stale build?)" % name) from e
            fn.restype, fn.argtypes = res, args
        if handle.gg_abi_version() != ABI_VERSION:
            raise GGError("ABI version mismatch")
        _LIB = handle
    return _LIB


def check(rc, what=""):
    if rc != 0:
        msg = lib().gg_last_error()
        raise GGError("%s failed (rc=%d): %s" % (what, rc, msg.decode() if msg else "?"))


def ptr(t):
    """device pointer of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()
