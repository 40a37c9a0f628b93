"""ctypes binding of libgnnrag_b200.so (include/gnnrag_b200.h).  No CPU fallback: if the library is
missing the import fails loudly."""
import ctypes
import os

from . import _build

c_i32p = ctypes.c_void_p
c_f32p = ctypes.c_void_p
c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_i64 = ctypes.c_int64
c_u32 = ctypes.c_uint32
c_size = ctypes.c_size_t
c_dbl = ctypes.c_double

# name -> (restype, argtypes); mirrors include/gnnrag_b200.h one to one
SIGNATURES = {
    "gr_abi_version": (c_int, []),
    "gr_last_error": (ctypes.c_char_p, []),
    "gr_set_option": (c_int, [ctypes.c_char_p, c_i64]),
    "gr_csr_build_workspace_bytes": (c_size, [c_i64, c_i64]),
    "gr_csr_build": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_i64, c_i64, c_i64,
                             c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p,
                             c_i32p, c_i32p, c_void_p, c_size, c_void_p]),
    "gr_gather_f32": (c_int, [c_f32p, c_i32p, c_f32p, c_i64, c_void_p]),
    "gr_linear": (c_int, [c_f32p, c_i64, c_f32p, c_i64, c_f32p, c_f32p, c_i64, c_i64, c_f32p, c_i64,
                          c_i64, c_i64, c_i64, c_u32, c_void_p]),
    "gr_linear_tc_workspace_bytes": (c_size, [c_i64, c_i64, c_i64]),
    "gr_linear_tc": (c_int, [c_f32p, c_i64, c_f32p, c_i64, c_f32p, c_f32p, c_i64, c_i64, c_i64, c_i64,
                             c_u32, c_void_p, c_size, c_void_p]),
    "gr_aggregate": (c_int, [c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_i64,
                             c_i64, c_i64, c_f32p, c_int, c_int, c_int, c_int, c_i64, c_void_p]),
    "gr_aggregate_backward": (c_int, [c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_i64, c_i64,
                                      c_i64, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_i64, c_void_p]),
    "gr_aggregate_dual": (c_int, [c_i32p, c_i32p, c_i32p, c_f32p, c_i32p, c_i32p, c_i32p, c_f32p,
                                  c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_i64, c_i64, c_i64,
                                  c_void_p, c_void_p, c_i64,
                                  c_int, c_int, c_int, c_int, c_i64, c_void_p]),
    "gr_pad_table256": (c_int, [c_f32p, c_i64, c_i64, c_int, c_f32p, c_void_p]),
    "gr_aggregate_dual_abs_supported": (c_int, [c_int, c_int, c_i64, c_i64]),
    "gr_aggregate_dual_abs": (c_int, [c_i32p, c_i32p, c_i32p, c_f32p, c_i32p, c_i32p, c_i32p, c_f32p,
                                     c_f32p, c_f32p, c_f32p, c_i64, c_f32p, c_void_p, c_void_p, c_i64, c_i64, c_i64,
                                     c_int, c_int, c_int, c_int, c_i64, c_i32p, c_void_p]),
    "gr_fused_profile_read": (c_int, [c_void_p, c_int]),
    "gr_fused_layer_supported": (c_int, [c_i64, c_i64, c_i64, c_int, c_i64]),
    "gr_fused_layer_workspace_bytes": (c_size, [c_i64, c_i64, c_int, c_i64]),
    "gr_fused_layer": (c_int, [c_i32p, c_i32p, c_i32p, c_f32p, c_i32p, c_i32p, c_i32p, c_f32p,
                               c_f32p, c_f32p, c_f32p, c_f32p, c_void_p, c_void_p, c_i64, c_i64, c_f32p,
                               c_i64, c_f32p, c_f32p, c_i64, c_void_p, c_void_p, c_i64, c_f32p, c_f32p,
                               c_int, c_int, c_int, c_int, c_i64, c_i64, c_u32, c_void_p, c_size, c_void_p, c_size,
                               c_void_p]),
    "gr_fused_ell_bytes": (c_size, [c_int, c_int, c_i64]),
    "gr_fused_ell_build": (c_int, [c_i32p, c_i32p, c_i32p, c_f32p, c_i32p, c_i32p, c_i32p, c_f32p, c_int, c_int, c_i64,
                                   c_void_p, c_size, c_void_p]),
    "gr_debug_store_probe": (c_int, [c_void_p, c_void_p, c_i64, c_i64, c_int, c_int, c_int, c_void_p]),
    "gr_type_layer": (c_int, [c_i32p, c_i32p, c_f32p, c_i32p, c_i32p, c_f32p, c_f32p, c_f32p, c_i64,
                              c_void_p, c_void_p, c_i64,
                              c_int, c_int, c_int, c_i64, c_void_p]),
    "gr_linear_tc_planes_workspace_bytes": (c_size, [c_i64, c_i64]),
    "gr_linear_tc_planes": (c_int, [c_void_p, c_void_p, c_i64, c_f32p, c_i64, c_f32p, c_f32p, c_i64,
                                    c_void_p, c_void_p, c_i64, c_f32p, c_f32p, c_i64, c_i64, c_i64,
                                    c_i64, c_i64, c_u32, c_void_p, c_size, c_void_p]),
    "gr_split_bf16": (c_int, [c_f32p, c_i64, c_i64, c_i64, c_void_p, c_void_p, c_i64, c_void_p]),
    "gr_masked_softmax": (c_int, [c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, c_int, c_int, c_void_p]),
    "gr_graft_stage_workspace_bytes": (c_size, [c_i64, c_i64]),
    "gr_graft_stage": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_i64, c_void_p,
                               c_int, c_int, c_i64, c_i64, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p,
                               c_i32p, c_void_p, c_size, c_void_p]),
    "gr_graft_attention": (c_int, [c_f32p, c_f32p, c_int, c_f32p, c_i64, c_i64, c_void_p, c_int, c_i64, c_int,
                                   c_i32p, c_i32p, c_i32p, c_int, c_f32p, c_f32p, c_f32p, c_i32p, c_void_p]),
    "gr_graft_aggregate": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_f32p, c_f32p, c_i64,
                                   c_f32p, c_i64, c_f32p, c_dbl, c_f32p, c_i64, c_void_p, c_void_p, c_i64,
                                   c_i64, c_i64, c_i64, c_f32p, c_f32p, c_int, c_int, c_int, c_void_p]),
    "gr_graft_dropout_mask": (c_int, [c_void_p, c_dbl, c_i64, c_int, c_void_p, c_void_p]),
    "gr_graft_aggregate_train": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_i64, c_f32p, c_i64,
                                         c_void_p, c_dbl, c_f32p, c_i64, c_int, c_int, c_int, c_void_p]),
    "gr_graft_aggregate_backward": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_i64, c_f32p,
                                            c_i64, c_void_p, c_dbl, c_f32p, c_i64, c_f32p, c_f32p, c_i64, c_f32p, c_i64,
                                            c_int, c_int, c_int, c_void_p]),
    "gr_graft_attention_backward": (c_int, [c_f32p, c_f32p, c_int, c_f32p, c_i64, c_i64, c_void_p, c_int, c_i64,
                                            c_int, c_f32p, c_f32p, c_f32p, c_i64, c_void_p]),
    "gr_type_layer_backward": (c_int, [c_i32p, c_i32p, c_f32p, c_i32p, c_i32p, c_f32p, c_f32p, c_i64, c_f32p, c_i64,
                                       c_f32p, c_i64, c_int, c_int, c_int, c_i64, c_void_p]),
    "gr_csr_row_of": (c_int, [c_i32p, c_i64, c_i32p, c_void_p]),
    "gr_aggregate_backward_det_workspace_bytes": (c_size, [c_int, c_int, c_int, c_int, c_i64]),
    "gr_aggregate_backward_det": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p,
                                          c_i64, c_i64, c_i64, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int, c_int,
                                          c_i64, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i64, c_void_p, c_size,
                                          c_void_p]),
    "gr_type_layer_backward_det_workspace_bytes": (c_size, [c_i64, c_int]),
    "gr_type_layer_backward_det": (c_int, [c_i32p, c_f32p, c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_i32p, c_i32p,
                                           c_i32p, c_f32p, c_i64, c_f32p, c_i64, c_f32p, c_i64, c_i64, c_int, c_i64,
                                           c_void_p, c_size, c_void_p]),
    "gr_graft_aggregate_backward_det_workspace_bytes": (c_size, [c_i64, c_int]),
    "gr_graft_aggregate_backward_det": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_i64,
                                                c_f32p, c_i64, c_void_p, c_dbl, c_f32p, c_i64, c_f32p, c_f32p, c_i64,
                                                c_f32p, c_i64, c_int, c_int, c_int, c_i32p, c_i32p, c_i32p, c_i32p,
                                                c_i32p, c_i64, c_i64, c_void_p, c_size, c_void_p]),
    "gr_graft_attention_backward_det_workspace_bytes": (c_size, [c_int, c_i64, c_int, c_int]),
    "gr_graft_attention_backward_det": (c_int, [c_f32p, c_f32p, c_int, c_f32p, c_i64, c_i64, c_void_p, c_int, c_i64,
                                                c_int, c_f32p, c_f32p, c_f32p, c_i64, c_i32p, c_i32p, c_void_p,
                                                c_size, c_void_p]),
    "gr_aggregate_ex": (c_int, [c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_f32p, c_f32p, c_void_p, c_i64, c_i64, c_i64,
                                c_f32p, c_int, c_int, c_int, c_int, c_i64, c_u32, c_void_p]),
    "gr_aggregate_backward_ex": (c_int, [c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_f32p, c_f32p, c_void_p, c_i64,
                                         c_i64, c_i64, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_i64, c_u32,
                                         c_void_p]),
    "gr_aggregate_backward_det_ex": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_f32p, c_f32p, c_void_p,
                                             c_i64, c_i64, c_i64, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int, c_int,
                                             c_i64, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i64, c_void_p, c_size,
                                             c_u32, c_void_p]),
    "gr_type_layer_ex": (c_int, [c_i32p, c_i32p, c_f32p, c_i32p, c_i32p, c_f32p, c_f32p, c_void_p, c_i64,
                                 c_void_p, c_void_p, c_i64, c_int, c_int, c_int, c_i64, c_u32, c_void_p]),
    "gr_type_layer_backward_ex": (c_int, [c_i32p, c_i32p, c_f32p, c_i32p, c_i32p, c_f32p, c_void_p, c_i64, c_void_p,
                                          c_i64, c_f32p, c_i64, c_int, c_int, c_int, c_i64, c_u32, c_void_p]),
    "gr_type_layer_backward_det_ex": (c_int, [c_i32p, c_f32p, c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_i32p, c_i32p,
                                              c_i32p, c_void_p, c_i64, c_void_p, c_i64, c_f32p, c_i64, c_i64, c_int,
                                              c_i64, c_void_p, c_size, c_u32, c_void_p]),
    "gr_graft_aggregate_train_ex": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_i64, c_void_p,
                                            c_i64, c_void_p, c_dbl, c_void_p, c_i64, c_int, c_int, c_int, c_u32,
                                            c_void_p]),
    "gr_graft_aggregate_backward_ex": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_i64,
                                               c_void_p, c_i64, c_void_p, c_dbl, c_void_p, c_i64, c_f32p, c_f32p, c_i64,
                                               c_void_p, c_i64, c_int, c_int, c_int, c_u32, c_void_p]),
    "gr_graft_aggregate_backward_det_ex": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_i64,
                                                   c_void_p, c_i64, c_void_p, c_dbl, c_void_p, c_i64, c_f32p, c_f32p,
                                                   c_i64, c_void_p, c_i64, c_int, c_int, c_int, c_i32p, c_i32p,
                                                   c_i32p, c_i32p, c_i32p, c_i64, c_i64, c_void_p, c_size, c_u32,
                                                   c_void_p]),
    "gr_frontier_rows": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_f32p, c_i64, c_i32p, c_i32p, c_void_p]),
    "gr_frontier_fixup": (c_int, [c_i32p, c_i32p, c_i32p, c_f32p, c_i32p, c_i32p, c_i32p, c_f32p, c_f32p,
                                  c_f32p, c_f32p, c_f32p, c_void_p, c_void_p, c_i64, c_f32p, c_i64, c_f32p,
                                  c_f32p, c_void_p, c_void_p, c_i64, c_f32p, c_f32p, c_i32p, c_i32p,
                                  c_int, c_int, c_int, c_int, c_void_p]),
    "gr_score_softmax": (c_int, [c_f32p, c_i64, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p,
                                 c_int, c_int, c_int, c_void_p]),
    "gr_instructions": (c_int, [c_f32p, c_f32p, c_void_p, c_i64, c_void_p, c_void_p, c_f32p, c_f32p, c_f32p,
                                c_f32p, c_f32p, c_f32p, c_int, c_int, c_int, c_int, c_void_p]),
    "gr_query_reform": (c_int, [c_f32p, c_f32p, c_i64, c_f32p, c_void_p, c_void_p, c_f32p, c_f32p,
                                c_int, c_int, c_int, c_int, c_void_p]),
    "gr_kl_loss_pred": (c_int, [c_f32p, c_f32p, c_f32p, c_f32p, c_void_p, c_int, c_int, c_void_p]),
    "gr_lstm_max_hidden": (c_size, []),
    "gr_lstm_forward": (c_int, [c_f32p, c_f32p, c_f32p, c_f32p, c_int, c_int, c_int, c_void_p]),
    "gr_seed_retrieve": (c_int, [c_f32p, c_f32p, c_i64, c_f32p, c_int, c_int, c_int, c_void_p]),
    "gr_rank_workspace_bytes": (c_size, [c_int, c_int]),
    "gr_rank_candidates": (c_int, [c_f32p, c_void_p, c_f32p, c_i64, c_dbl, c_i32p, c_i32p, c_i32p,
                                   c_int, c_int, c_void_p, c_size, c_void_p]),
    "gr_paths_workspace_bytes": (c_size, [c_int, c_int, c_int, c_int]),
    "gr_shortest_path_nodes": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_int,
                                       c_i32p, c_i32p, c_int, c_void_p, c_i32p, c_int, c_int,
                                       c_void_p, c_size, c_void_p]),
    "gr_rule_adj_workspace_bytes": (c_size, [c_i64]),
    "gr_rule_adj_build": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i64, c_i64,
                                  c_i32p, c_i32p, c_i32p, c_i32p, c_void_p, c_size, c_void_p]),
    "gr_rule_level_workspace_bytes": (c_size, [c_i64]),
    "gr_rule_level_count": (c_int, [c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p, c_int, c_int, c_i32p, c_i32p,
                                    c_i64, c_i32p, c_void_p, c_i32p, c_i32p, c_void_p, c_size, c_void_p]),
    "gr_rule_level_emit": (c_int, [c_i32p, c_i32p, c_i32p, c_void_p, c_i64, c_i64, c_i32p, c_i32p, c_i32p,
                                   c_void_p]),
    "gr_rule_paths_write": (c_int, [c_void_p, c_void_p, c_i32p, c_i32p, c_void_p, c_void_p, c_int, c_i64, c_i32p,
                                    c_void_p]),
}

_lib = None


def lib_path():
    return _build.LIB_PATH


def load(build_if_missing=True):
    """Load (building first if needed and possible).  Raises ImportError when unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if build_if_missing and _build.needs_build():
        try:
            _build.build()
        except Exception as e:  # noqa: BLE001
            if not os.path.exists(path):
                raise ImportError("libgnnrag_b200.so is not built and nvcc failed: %s" % e)
    if not os.path.exists(path):
        raise ImportError("libgnnrag_b200.so not found at %s (run `python -m gnn_rag_b200._build`)" % path)
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            raise ImportError("libgnnrag_b200.so does not export %s (stale build?)" % name)
        fn.restype = res
        fn.argtypes = args
    if lib.gr_abi_version() != 1:
        raise ImportError("libgnnrag_b200.so ABI version mismatch")
    _lib = lib
    return lib


class GrError(RuntimeError):
    pass


def check(rc):
    if rc != 0:
        msg = load().gr_last_error()
        raise GrError("libgnnrag_b200 error %d: %s" % (rc, msg.decode() if msg else "?"))
