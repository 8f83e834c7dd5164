"""ctypes binding of libdirb200.so (the C ABI declared in include/dirb200.h).

The library is built in-tree by ``build_ext.py`` (nvcc, sm_90a).  There is no CPU or PyTorch
fallback: if the shared object is missing, importing this module raises, and every compute
call raises ``DirbError`` on a machine without an sm_90 GPU.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libdirb200.so")


class DirbError(RuntimeError):
    def __init__(self, status, message):
        super().__init__("dirb200 error %d: %s" % (status, message))
        self.status = status


if not os.path.exists(LIB_PATH):
    raise ImportError("%s not found - build it with `python deep-image-retrieval_b200/build_ext.py` "
                      "(or __graft_entry__.build()); there is no fallback path" % LIB_PATH)

_lib = C.CDLL(LIB_PATH)

p = C.c_void_p
i32 = C.c_int
i64 = C.c_int64
f32 = C.c_float
f64 = C.c_double

# name -> (restype, argtypes).  Must list every symbol declared in include/dirb200.h.
SIGNATURES = {
    "dirb200_version": (i32, []),
    "dirb200_last_error": (C.c_char_p, []),
    "dirb200_device_check": (i32, [i32]),
    "dirb200_set_global_option": (i32, [C.c_char_p, f64]),
    "dirb200_get_global_option": (i32, [C.c_char_p, C.POINTER(f64)]),
    "dirb200_net_create": (i32, [C.c_char_p, i32, C.POINTER(p)]),
    "dirb200_net_set_option": (i32, [p, C.c_char_p, f64]),
    "dirb200_net_set_tensor": (i32, [p, C.c_char_p, p, C.POINTER(i64), i32]),
    "dirb200_net_finalize": (i32, [p]),
    "dirb200_net_forward": (i32, [p, p, i32, i32, i32, p, p, p]),
    "dirb200_net_forward_host": (i32, [p, p, i32, i32, i32, p]),
    "dirb200_net_forward_u8": (i32, [p, p, i32, i32, i32, p, p, p]),
    "dirb200_net_forward_host_u8": (i32, [p, p, i32, i32, i32, p]),
    "dirb200_net_forward_ragged_u8": (i32, [p, p, i32, i32, i32, p, p, p, p]),
    "dirb200_net_forward_ragged": (i32, [p, p, i32, i32, i32, p, p, p, p]),
    "dirb200_resize_bilinear_u8": (i32, [p, i32, i32, i32, i32, i32, p, p]),
    "dirb200_resize_coeffs": (i32, [i32, i32, p, p, C.POINTER(i32)]),
    "dirb200_jpeg_probe": (i32, [p, C.c_size_t, C.POINTER(i32)]),
    "dirb200_jpeg_decoder_create": (i32, [i32, C.POINTER(p)]),
    "dirb200_jpeg_decoder_set_option": (i32, [p, C.c_char_p, f64]),
    "dirb200_jpeg_decoder_decode": (i32, [p, i32, p, p, p, p, p, C.POINTER(i32), p]),
    "dirb200_jpeg_debug_coefficients": (i32, [p, i32, p, C.c_size_t, C.POINTER(i32), p]),
    "dirb200_jpeg_decoder_destroy": (i32, [p]),
    "dirb200_net_debug_stage": (i32, [p, C.c_char_p, p, C.c_size_t, C.POINTER(i32), p]),
    "dirb200_net_profile": (i32, [p, C.POINTER(f64)]),
    "dirb200_net_profile_table": (i32, [p, p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "dirb200_net_last_launches": (i32, [p, C.POINTER(i64), C.POINTER(f64)]),
    "dirb200_net_destroy": (i32, [p]),
    "dirb200_nchw_to_nhwc8": (i32, [p, i32, i32, i32, p, p]),
    "dirb200_conv_bn_act": (i32, [p, i32, i32, i32, i32, p, i32, i32, i32, i32, i32, p, p, p, i32, i32, p, p]),
    "dirb200_conv_c23": (i32, [p, i32, i32, i32, i32, p, p, p, p, p, p, p, p, i32, p]),
    "dirb200_conv_c31": (i32, [p, i32, i32, i32, i32, p, p, p, p, p, p, p, p, p, p]),
    "dirb200_stem_workspace_bytes": (C.c_size_t, [i32, i32, i32]),
    "dirb200_stem_pack_weight": (i32, [p, p]),
    "dirb200_stem_conv": (i32, [p, i32, i32, i32, p, p, p, p, p, p]),
    "dirb200_stem_pool": (i32, [p, i32, i32, i32, i32, p, p, p, p, p, p, p]),
    "dirb200_maxpool_3x3s2": (i32, [p, i32, i32, i32, i32, p, p]),
    "dirb200_head_workspace_floats": (C.c_size_t, [i32, i32, i32, i32]),
    "dirb200_head_pool_fc_l2": (i32, [p, i32, i32, i32, i32, f32, f32, i32, p, p, i32, p, p, p, p]),
    "dirb200_pool_scales": (i32, [p, i32, i64, i32, i32, f32, i32, p, p]),
    "dirb200_l2_normalize": (i32, [p, i64, i32, f32, p, p, p]),
    "dirb200_center_bias": (i32, [p, i32, i32, i32, i32, f32, p]),
    "dirb200_whiten": (i32, [p, i64, i32, p, p, p, i32, i32, p, p, p]),
    "dirb200_f32_to_f16": (i32, [p, i64, p, p]),
    "dirb200_index_create": (i32, [i32, i32, C.POINTER(p)]),
    "dirb200_index_set_db": (i32, [p, p, p, i64, i64]),
    "dirb200_index_set_option": (i32, [p, C.c_char_p, f64]),
    "dirb200_index_search": (i32, [p, p, i32, i32, p, p, p]),
    "dirb200_index_search_max_queries": (i32, [p, i32, C.POINTER(C.c_int)]),
    "dirb200_index_search_begin": (i32, [p, p, i32, i32, i32, p, p]),
    "dirb200_index_search_finish": (i32, [p, p, p, p, p, p]),
    "dirb200_index_check": (i32, [p]),
    # filtered exact search: an allow bitmap on the index, and per-query row exclusion into such a bitmap
    "dirb200_index_set_allow": (i32, [p, p, i64, i64]),
    "dirb200_allow_exclude": (i32, [p, i32, i64, p, p, p]),
    "dirb200_index_last_stats": (i32, [p, C.POINTER(i64)]),
    "dirb200_index_last_profile": (i32, [p, C.POINTER(f64)]),
    "dirb200_index_target_scores": (i32, [p, p, i32, p, p, i32, p, p]),
    "dirb200_index_rank_count": (i32, [p, p, i32, p, p, p, p, p, i32, p, p]),
    "dirb200_index_count_ge": (i32, [p, p, i32, p, p, i32, p, p, p]),
    "dirb200_index_destroy": (i32, [p]),
    "dirb200_topk_merge": (i32, [p, p, i32, i32, i32, i64, p, p, p]),
    "dirb200_exchange_create": (i32, [i32, i32, i32, i32, i32, C.POINTER(p)]),
    "dirb200_exchange_ipc_handle": (i32, [p, p]),
    "dirb200_exchange_open": (i32, [p, p]),
    "dirb200_exchange_open_local": (i32, [p, C.POINTER(p)]),
    "dirb200_exchange_close_peers": (i32, [p]),
    "dirb200_exchange_destroy": (i32, [p]),
    "dirb200_index_search_sharded": (i32, [p, p, p, i32, i32, i32, p, p, p]),
    "dirb200_index_search_sharded_phase": (i32, [p, p, i32, p, i32, i32, i32, p, p, p]),
    "dirb200_scores_exact": (i32, [p, i32, p, i64, i32, p, p]),
    "dirb200_aqe_expand": (i32, [p, i32, i32, p, p, p, i32, f64, i32, i64, i64, p, p]),
    # the statistics of sklearn's PCA.fit (_pca.py, _fit_full): the column sums behind mean_, and the centred Gram that
    # replaces the covariance_eigh branch's X^T X - n m m^T
    "dirb200_col_sums_f64": (i32, [p, i64, i32, p, p]),
    "dirb200_gram_f64": (i32, [p, i64, i32, p, p, p]),
    # the AP / TAP losses of loss.py: histogram + fp64 finalisation, and the elementwise backward
    "dirb200_aploss_forward": (i32, [p, p, i64, i64, i32, p, i32, p, p, p, p]),
    "dirb200_aploss_backward": (i32, [p, p, i64, i64, i32, p, p, p, p, p]),
    # diffusion re-ranking (Zhou et al. 2003, Iscen et al. 2017): mutual-kNN graph, seeds, batched CG, rank counts
    "dirb200_diffusion_graph_workspace_bytes": (C.c_size_t, [i64, i32]),
    "dirb200_diffusion_graph": (i32, [p, p, i64, i32, i32, f64, p, p, p, p, p]),
    "dirb200_diffusion_seeds": (i32, [p, p, i32, i32, f64, i64, p, p]),
    "dirb200_diffusion_solve_workspace_bytes": (C.c_size_t, [i64, i32]),
    "dirb200_diffusion_solve": (i32, [p, p, p, i64, p, i32, f64, i32, f64, p, p, p, p, p]),
    "dirb200_diffusion_rank_count_workspace_bytes": (C.c_size_t, [i32, i32]),
    "dirb200_diffusion_rank_count": (i32, [p, i64, i32, p, p, p, p, i32, p, p, p, p]),
    "dirb200_diffusion_topk_workspace_bytes": (C.c_size_t, [i32, i32]),
    "dirb200_diffusion_topk": (i32, [p, i64, i32, i32, p, p, p, p]),
    # truncated diffusion: each query on the subgraph of its own top-m rows, all CG iterations in one launch
    "dirb200_diffusion_graph_weights": (i32, [p, p, i64, i32, i32, f64, p, p, p, p, p, p, p]),
    "dirb200_diffusion_trunc_build_workspace_bytes": (C.c_size_t, [i32, i32]),
    "dirb200_diffusion_trunc_build": (i32, [p, p, p, i64, i32, p, p, i32, i32, i32, f64, p, p, p, p, p, p, p, p, p]),
    "dirb200_diffusion_trunc_solve_workspace_bytes": (C.c_size_t, [i32, i32]),
    "dirb200_diffusion_trunc_solve": (i32, [p, p, p, i32, p, i32, i32, f64, i32, f64, p, p, p, p, p]),
    "dirb200_diffusion_trunc_topk_workspace_bytes": (C.c_size_t, [i32, i32, i32]),
    "dirb200_diffusion_trunc_topk": (i32, [p, p, i32, i32, p, p, i32, i32, p, p, p, p]),
    "dirb200_diffusion_trunc_rank_count": (i32, [p, p, i32, i32, p, p, p, i32, p, p, p, p]),
    # range search, triangular self-join and the connected components of its pair graph
    "dirb200_index_range_search": (i32, [p, p, i32, f64, C.POINTER(i64), p]),
    "dirb200_index_self_join": (i32, [p, i64, i64, f64, C.POINTER(i64), p]),
    "dirb200_index_join_fetch": (i32, [p, p, p, p, p]),
    "dirb200_index_join_stats": (i32, [p, C.POINTER(i64), C.POINTER(f64)]),
    "dirb200_join_components_workspace_bytes": (C.c_size_t, [i64]),
    "dirb200_join_components": (i32, [p, p, i64, i64, p, p, p]),
    "dirb200_join_groups_workspace_bytes": (C.c_size_t, [i64]),
    "dirb200_join_groups": (i32, [p, i64, p, p, p, C.POINTER(i64), p]),
    "dirb200_index_nearest": (i32, [p, p, i32, p, p, p]),
    "dirb200_index_nearest_stats": (i32, [p, C.POINTER(i64)]),
    "dirb200_index_set_lists": (i32, [p, p, p, p, i32, p]),
    "dirb200_index_search_lists": (i32, [p, p, i32, i32, p, i32, p, p, p]),
    "dirb200_index_lists_stats": (i32, [p, C.POINTER(i64), C.POINTER(f64)]),
    # spherical k-means around the exact top-1 assignment: sizes + objective, empty-cluster relocation, centre update,
    # k-means++ draws
    "dirb200_kmeans_stats_workspace_bytes": (C.c_size_t, [i64, i32]),
    "dirb200_kmeans_stats": (i32, [p, p, p, i64, i32, p, p, C.POINTER(i64), p]),
    "dirb200_kmeans_relocate_workspace_bytes": (C.c_size_t, [i64]),
    "dirb200_kmeans_relocate": (i32, [p, p, i64, i32, p, p, C.POINTER(i64), p]),
    "dirb200_kmeans_update_workspace_bytes": (C.c_size_t, [i64, i32, i32]),
    "dirb200_kmeans_update": (i32, [p, i64, i32, p, p, i32, p, p, C.POINTER(i64), p]),
    "dirb200_kmeans_pp_workspace_bytes": (C.c_size_t, [i64, i32]),
    "dirb200_kmeans_pp": (i32, [p, i64, i32, i64, p, i32, p, p, p]),
    # product quantisation of the inverted lists: codeword assignment / encoding, codebook update, ADC tables, and
    # the scan, selection and exact refinement of one query block
    "dirb200_pq_assign": (i32, [p, i64, i32, p, p, p, i32, p, i32, p]),
    "dirb200_pq_update": (i32, [p, i64, i32, p, p, p, i32, p, p, p]),
    "dirb200_pq_tables": (i32, [p, i32, i32, p, i32, p, p]),
    "dirb200_pq_search_ws_bytes": (C.c_size_t, [i32, i64, i32]),
    "dirb200_pq_search": (i32, [p, i32, i32, p, i32, p, p, i32, p, p, p, p, i64, p, i32, i32, p, p, p, p, p]),
    # graph search over a pruned kNN graph: forward edges, reverse edges merged in, best-first traversal
    "dirb200_graph_prune": (i32, [p, i64, i32, i32, p, p]),
    "dirb200_graph_merge": (i32, [p, i64, i32, p, p, p, p]),
    "dirb200_graph_search_smem_bytes": (C.c_size_t, [i32, i32, i32, i32, i32]),
    "dirb200_graph_search": (i32, [p, i32, i32, p, i64, p, i32, p, i32, i32, i32, i32, i32, p, p, p, p, p, p, p]),
}

for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(_lib, _name)     # AttributeError here = the .so is stale / does not export the ABI
    _fn.restype = _res
    _fn.argtypes = _args


def last_error() -> str:
    msg = _lib.dirb200_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def call(name, *args):
    """Call a status-returning entry point; raise DirbError on a non-zero status."""
    status = getattr(_lib, name)(*args)
    if status != 0:
        raise DirbError(status, last_error())


def raw(name):
    return getattr(_lib, name)


def version() -> int:
    return _lib.dirb200_version()


def loaded_path() -> str:
    return LIB_PATH
