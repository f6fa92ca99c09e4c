"""ctypes binding of libpolyb200.so (include/poly_b200.h).

The library is the product: there is no Python/NumPy/PyTorch compute fallback.  If the
shared object is missing, or no sm_90 device is usable, importing works (so that the
CPU-only test tier can check the exported symbols) but every compute call raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libpolyb200.so")

PG_OK, PG_ERR_CUDA, PG_ERR_ARG, PG_ERR_NO_DEVICE, PG_ERR_PANIC, PG_ERR_UNSUPPORTED, PG_ERR_NOMEM = range(7)
PG_ITEM_OK, PG_ITEM_PANIC, PG_ITEM_UNSUPPORTED = 0, 1, 2
PG_SKETCH_PAD_ZERO = 1
PG_SKETCH_TAIL_KEEP = 2
PG_KMER_CANONICAL = 1
PG_PAIRS_UPPER = 1


class PolyError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libpolyb200 error {code}: {msg}")
        self.code = code


class GoPanic(IndexError):
    """Raised where the Go reference would panic (index out of range)."""


_u8p, _u32p, _u64p, _i64p, _i32p, _i16p, _f64p = (C.c_void_p,) * 7  # raw addresses (host or device)

_SIGS = {
    "pg_version": (C.c_int, []),
    "pg_init": (C.c_int, [C.c_int]),
    "pg_thread_device": (C.c_int, [C.c_int]),
    "pg_numa_bind_thread": (C.c_int, [C.c_int, C.POINTER(C.c_int)]),
    "pg_shutdown": (C.c_int, []),
    "pg_last_error": (C.c_char_p, []),
    "pg_last_kernel": (C.c_char_p, []),
    "pg_launch_count": (C.c_uint64, []),
    "pg_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "pg_device_sm_count": (C.c_int, [C.POINTER(C.c_int)]),
    "pg_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_size_t]),
    "pg_host_free": (C.c_int, [C.c_void_p]),
    "pg_dev_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_size_t]),
    "pg_dev_free": (C.c_int, [C.c_void_p]),
    "pg_memcpy_h2d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pg_memcpy_d2h": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "pg_stream_sync": (C.c_int, [C.c_void_p]),
    "pg_mash_sketch_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, _u32p, C.c_uint64, _u32p, _i32p]),
    "pg_mash_sketch_uniform": (C.c_int, [_u8p, C.c_uint64, C.c_uint32, C.c_int32, C.c_int32, C.c_uint32, _u32p, C.c_uint64, _i32p]),
    "pg_mash_sketch_batch_dev": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, _u32p, C.c_uint64, _u32p, _i32p, C.c_void_p]),
    "pg_mash_sketch_uniform_dev": (C.c_int, [_u8p, C.c_uint64, C.c_uint32, C.c_int32, C.c_int32, C.c_uint32, _u32p, C.c_uint64, _i32p, C.c_void_p]),
    "pg_mash_sketch_groups": (C.c_int, [_u8p, _u64p, C.c_uint64, _u64p, C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, _u32p, C.c_uint64, _u32p]),
    "pg_mash_sketch_groups_dev": (C.c_int, [_u8p, _u64p, C.c_uint64, _u64p, C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, _u32p, C.c_uint64, _u32p,
                                            C.c_void_p]),
    "pg_mash_sketch_groups_flags": (C.c_int, [_u8p, _u64p, C.c_uint64, _u64p, C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, C.c_uint32, _u32p,
                                              C.c_uint64, _u32p]),
    "pg_mash_sketch_groups_flags_dev": (C.c_int, [_u8p, _u64p, C.c_uint64, _u64p, C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, C.c_uint32,
                                                  _u32p, C.c_uint64, _u32p, C.c_void_p]),
    "pg_mash_sketcher_create": (C.c_int, [C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, C.c_uint64, C.POINTER(C.c_void_p)]),
    "pg_mash_sketcher_create_flags": (C.c_int, [C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, C.c_uint64, C.c_uint32, C.POINTER(C.c_void_p)]),
    "pg_mash_sketcher_add": (C.c_int, [C.c_void_p, _u8p, _u64p, C.c_uint64, _u64p, C.c_uint64, C.c_uint64]),
    "pg_mash_sketcher_add_dev": (C.c_int, [C.c_void_p, _u8p, _u64p, C.c_uint64, _u64p, C.c_uint64, C.c_uint64, C.c_void_p]),
    "pg_mash_sketcher_rows": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, _u32p, C.c_uint64, _u32p, _u8p, _u64p]),
    "pg_mash_sketcher_rows_dev": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, _u32p, C.c_uint64, _u32p, _u8p, _u64p, C.c_void_p]),
    "pg_mash_sketcher_free": (C.c_int, [C.c_void_p]),
    "pg_mash_dist": (C.c_int, [_u32p, _u32p, C.c_uint64, _u32p, _u32p, C.c_uint64, C.c_uint64, C.c_int32, C.c_int32, _u64p, _u64p, _u32p, _u32p,
                               _f64p, _f64p]),
    "pg_mash_dist_dev": (C.c_int, [_u32p, _u32p, C.c_uint64, _u32p, _u32p, C.c_uint64, C.c_uint64, C.c_int32, C.c_int32, _u64p, _u64p, _u32p,
                                   _u32p, _f64p, _f64p, C.c_void_p]),
    "pg_mash_dist_within": (C.c_int, [_u32p, _u32p, C.c_uint64, _u32p, _u32p, C.c_uint64, C.c_uint64, C.c_int32, C.c_int32, _u64p, _u64p,
                                      C.c_double, C.c_double, C.c_uint32, _u32p, _u32p, _u32p, _u32p, _f64p, _f64p, C.c_uint64,
                                      C.POINTER(C.c_uint64)]),
    "pg_mash_dist_within_dev": (C.c_int, [_u32p, _u32p, C.c_uint64, _u32p, _u32p, C.c_uint64, C.c_uint64, C.c_int32, C.c_int32, _u64p, _u64p,
                                          C.c_double, C.c_double, C.c_uint32, _u32p, _u32p, _u32p, _u32p, _f64p, _f64p, C.c_uint64,
                                          _u64p, C.c_void_p]),
    "pg_ipc_export": (C.c_int, [C.c_void_p, C.c_void_p]),
    "pg_ipc_import": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "pg_ipc_close": (C.c_int, [C.c_void_p]),
    "pg_mash_sketch_uniform_gather_dev": (C.c_int, [_u8p, C.c_uint64, C.c_uint32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p), C.c_int32, C.c_int32, C.c_void_p]),
    "pg_mash_sketch_uniform_scatter_dev": (C.c_int, [_u8p, C.c_uint64, C.c_uint32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p), C.c_int32, C.c_int32, C.c_uint64, C.c_void_p]),
    "pg_mash_sketch_uniform_multi": (C.c_int, [_u8p, C.c_uint64, C.c_uint32, C.c_int32, C.c_int32, C.c_uint32, _u32p, C.c_uint64, _i32p, _i32p, C.c_int32]),
    "pg_mash_sketch_batch_multi": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, _u32p, C.c_uint64, _u32p, _i32p, _i32p, C.c_int32]),
    "pg_mash_sketch_distance_multi": (C.c_int, [_u8p, C.c_uint64, C.c_uint32, C.c_int32, C.c_int32, _i32p, C.c_int32, _u32p, _u32p, _f64p]),
    "pg_mash_similarity_pairs": (C.c_int, [_u32p, _u64p, C.c_uint64, _u32p, _u32p, C.c_uint64, _i64p, _f64p, _f64p, _i32p]),
    "pg_mash_similarity_pairs_dev": (C.c_int, [_u32p, _u64p, C.c_uint64, _u32p, _u32p, C.c_uint64, _i64p, _f64p, _f64p, _i32p, C.c_void_p]),
    "pg_mash_distance_block": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_uint64, C.c_uint64, _u32p, _f64p]),
    "pg_mash_distance_block_dev": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_uint64, C.c_uint64, _u32p, _f64p, C.c_void_p]),
    "pg_mash_distance_sparse": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_uint64, C.c_uint64, C.c_uint32, _u32p, _u32p, _u32p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "pg_mash_distance_sparse_dev": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_uint64, C.c_uint64, C.c_uint32, _u32p, _u32p, _u32p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "pg_mash_cluster": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_uint32, _u32p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "pg_mash_cluster_dev": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_uint32, _u32p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_mash_dereplicate": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_uint32, C.c_uint32, _u32p, C.POINTER(C.c_uint64)]),
    "pg_mash_dereplicate_dev": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_uint32, C.c_uint32, _u32p, C.c_void_p, C.c_void_p]),
    "pg_mash_index_create": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.POINTER(C.c_void_p)]),
    "pg_mash_index_create_dev": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "pg_mash_index_query": (C.c_int, [C.c_void_p, _u32p, C.c_uint64, C.c_int32, C.c_uint32, C.c_uint32, _u32p, _u32p, _f64p, _u32p]),
    "pg_mash_index_query_dev": (C.c_int, [C.c_void_p, _u32p, C.c_uint64, C.c_int32, C.c_uint32, C.c_uint32, _u32p, _u32p, _f64p, _u32p, C.c_void_p]),
    "pg_mash_index_free": (C.c_int, [C.c_void_p]),
    "pg_mash_index_add": (C.c_int, [C.c_void_p, _u32p, C.c_uint64, C.c_int32]),
    "pg_mash_index_add_dev": (C.c_int, [C.c_void_p, _u32p, C.c_uint64, C.c_int32, C.c_void_p]),
    "pg_mash_index_query_within": (C.c_int, [C.c_void_p, _u32p, C.c_uint64, C.c_int32, C.c_uint32, _u64p, _u32p, _u32p, _f64p, C.c_uint64,
                                             C.POINTER(C.c_uint64)]),
    "pg_mash_index_query_within_dev": (C.c_int, [C.c_void_p, _u32p, C.c_uint64, C.c_int32, C.c_uint32, _u64p, _u32p, _u32p, _f64p, C.c_uint64,
                                                 _u64p, C.c_void_p]),
    "pg_mash_dereplicator_create": (C.c_int, [C.c_int32, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]),
    "pg_mash_dereplicator_add": (C.c_int, [C.c_void_p, _u32p, C.c_uint64, C.c_int32, _u32p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "pg_mash_dereplicator_add_dev": (C.c_int, [C.c_void_p, _u32p, C.c_uint64, C.c_int32, _u32p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                               C.c_void_p]),
    "pg_mash_dereplicator_reps": (C.c_int, [C.c_void_p, _u32p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "pg_mash_dereplicator_index": (C.c_void_p, [C.c_void_p]),
    "pg_mash_dereplicator_free": (C.c_int, [C.c_void_p]),
    "pg_mash_clusterer_create": (C.c_int, [C.c_int32, C.c_uint32, C.POINTER(C.c_void_p)]),
    "pg_mash_clusterer_add": (C.c_int, [C.c_void_p, _u32p, C.c_uint64, C.c_int32, _u32p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                        C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "pg_mash_clusterer_add_dev": (C.c_int, [C.c_void_p, _u32p, C.c_uint64, C.c_int32, _u32p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                            C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_void_p]),
    "pg_mash_clusterer_labels": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, _u32p]),
    "pg_mash_clusterer_labels_dev": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, _u32p, C.c_void_p]),
    "pg_mash_clusterer_index": (C.c_void_p, [C.c_void_p]),
    "pg_mash_clusterer_free": (C.c_int, [C.c_void_p]),
    "pg_mash_screen_create": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]),
    "pg_mash_screen_create_dev": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "pg_mash_screen_add": (C.c_int, [C.c_void_p, _u8p, _u64p, C.c_uint64]),
    "pg_mash_screen_add_dev": (C.c_int, [C.c_void_p, _u8p, _u64p, C.c_uint64, C.c_void_p]),
    "pg_mash_screen_reset": (C.c_int, [C.c_void_p]),
    "pg_mash_screen_results": (C.c_int, [C.c_void_p, _u32p, _f64p, _u64p]),
    "pg_mash_screen_results_dev": (C.c_int, [C.c_void_p, _u32p, _f64p, _u64p, C.c_void_p]),
    "pg_mash_screen_winners": (C.c_int, [C.c_void_p, _u32p, _f64p, _u64p]),
    "pg_mash_screen_winners_dev": (C.c_int, [C.c_void_p, _u32p, _f64p, _u64p, C.c_void_p]),
    "pg_mash_screen_create_samples": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, C.POINTER(C.c_void_p)]),
    "pg_mash_screen_create_samples_dev": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "pg_mash_screen_create_flags": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]),
    "pg_mash_screen_create_flags_dev": (C.c_int, [_u32p, C.c_uint64, C.c_int32, C.c_int32, C.c_uint32, C.c_uint32, C.c_void_p,
                                                  C.POINTER(C.c_void_p)]),
    "pg_mash_screen_add_samples": (C.c_int, [C.c_void_p, _u8p, _u64p, _u32p, C.c_uint64]),
    "pg_mash_screen_add_samples_dev": (C.c_int, [C.c_void_p, _u8p, _u64p, _u32p, C.c_uint64, C.c_void_p]),
    "pg_mash_screen_results_samples": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, _u32p, _f64p, _u64p]),
    "pg_mash_screen_results_samples_dev": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, _u32p, _f64p, _u64p, C.c_void_p]),
    "pg_mash_screen_winners_samples": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, _u32p, _f64p, _u64p]),
    "pg_mash_screen_winners_samples_dev": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, _u32p, _f64p, _u64p, C.c_void_p]),
    "pg_mash_screen_free": (C.c_int, [C.c_void_p]),
    "pg_sw_score_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, _u8p, C.c_uint64, C.c_int32, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p]),
    "pg_sw_score_batch_dev": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_uint64, _u8p, C.c_uint64, C.c_int32, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p, C.c_void_p]),
    "pg_sw_align_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, _u8p, C.c_uint64, C.c_int32, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p, _u8p, _u8p, C.c_uint64, _u32p, _i32p]),
    "pg_nw_align_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, _u8p, C.c_uint64, C.c_int32, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p, _u8p, _u8p, C.c_uint64, _u32p, _i32p]),
    "pg_nw_score_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, _u8p, C.c_uint64, C.c_int32, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p]),
    "pg_nw_score_batch_dev": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_uint64, _u8p, C.c_uint64, C.c_int32, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p, C.c_void_p]),
    "pg_sw_score_pairs": (C.c_int, [_u8p, _u64p, C.c_uint64, _u8p, _u64p, C.c_uint64, _u32p, _u32p, C.c_uint64, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p]),
    "pg_nw_score_pairs": (C.c_int, [_u8p, _u64p, C.c_uint64, _u8p, _u64p, C.c_uint64, _u32p, _u32p, C.c_uint64, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p]),
    "pg_sw_score_pairs_dev": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_uint64, _u8p, _u64p, C.c_uint64, C.c_uint64, _u32p, _u32p, C.c_uint64, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p, C.c_void_p]),
    "pg_nw_score_pairs_dev": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_uint64, _u8p, _u64p, C.c_uint64, C.c_uint64, _u32p, _u32p, C.c_uint64, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p, C.c_void_p]),
    "pg_sw_align_pairs": (C.c_int, [_u8p, _u64p, C.c_uint64, _u8p, _u64p, C.c_uint64, _u32p, _u32p, C.c_uint64, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p, _u8p, _u8p, C.c_uint64, _u32p, _i32p]),
    "pg_nw_align_pairs": (C.c_int, [_u8p, _u64p, C.c_uint64, _u8p, _u64p, C.c_uint64, _u32p, _u32p, C.c_uint64, _i16p, _i16p, _i64p, C.c_int32, C.c_int32, C.c_int64, _i64p, _i32p, _i64p, _u8p, _u8p, C.c_uint64, _u32p, _i32p]),
    "pg_tm_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_double, C.c_double, C.c_double, _f64p, _f64p, _f64p, _i32p]),
    "pg_tm_batch_dev": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_double, C.c_double, C.c_double, _f64p, _f64p, _f64p, _i32p, C.c_void_p]),
    "pg_design_primers_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_double, _u32p, _u32p, _i32p]),
    "pg_pcr_minimal_primer_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_double, _u32p, _i32p]),
    "pg_find_sites_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, _u8p, _u64p, C.c_uint32, C.c_uint32, _u32p, _u64p, _u32p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "pg_fastq_ingest": (C.c_int, [_u8p, C.c_uint64, _u8p, C.c_uint64, _u64p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.POINTER(C.c_uint64)]),
    "pg_fastq_ingest_dev": (C.c_int, [_u8p, C.c_uint64, _u8p, C.c_uint64, _u64p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.c_void_p]),
    "pg_fastq_ingest_records": (C.c_int, [_u8p, C.c_uint64, _u8p, C.c_uint64, _u64p, _u64p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.POINTER(C.c_uint64)]),
    "pg_fastq_ingest_records_dev": (C.c_int, [_u8p, C.c_uint64, _u8p, C.c_uint64, _u64p, _u64p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.c_void_p]),
    "pg_fasta_ingest": (C.c_int, [_u8p, C.c_uint64, C.c_uint32, C.c_uint32, _u8p, C.c_uint64, _u64p, _u8p, C.c_uint64, _u64p, C.c_uint64,
                                  C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.POINTER(C.c_uint64)]),
    "pg_fasta_ingest_dev": (C.c_int, [_u8p, C.c_uint64, C.c_uint32, C.c_uint32, _u8p, C.c_uint64, _u64p, _u8p, C.c_uint64, _u64p, C.c_uint64,
                                      C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.c_void_p]),
    "pg_seqhash_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_int32, C.c_uint32, _u8p, _i32p, _u64p]),
    "pg_seqhash_batch_dev": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_int32, C.c_uint32, _u8p, _i32p, _u64p, C.c_uint64, C.c_void_p]),
    "pg_least_rotation_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, _u64p]),
    "pg_clone_digest_batch": (C.c_int, [_u8p, _u64p, _u8p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_int32, _u32p, _i32p, _u8p, C.c_uint64, _u64p, _u8p,
                                        C.c_uint64, _u64p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "pg_clone_golden_gate_batch": (C.c_int, [_u8p, _u64p, _u8p, C.c_uint64, _u64p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint64, _u8p, _u64p, _u8p,
                                             _u8p, _u64p, _i32p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "pg_clone_circular_ligate_batch": (C.c_int, [_u8p, _u64p, _u8p, _u64p, C.c_uint64, _u64p, C.c_uint64, C.c_uint64, C.c_uint64, _u8p, _u64p, _u8p,
                                                 _u8p, _u64p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "pg_fold_zuker_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_double, _f64p, _u8p, _u64p, _i32p]),
    "pg_fragment_batch": (C.c_int, [_u8p, _u64p, C.c_uint64, C.c_int64, C.c_int64, _u8p, _u64p, C.c_uint64, _u8p, _u64p, C.c_uint64, _i32p, _f64p,
                                    _i64p, _i64p, _u64p, _u64p, C.c_uint64, _u64p]),
    "pg_fragment_set_efficiency_batch": (C.c_int, [_u8p, _u64p, _u64p, C.c_uint64, _f64p]),
    "pg_fragment_next_overhangs_batch": (C.c_int, [_u8p, _u64p, _u64p, C.c_uint64, _u8p, _u32p, _f64p]),
    "pg_synth_reads_dev": (C.c_int, [_u8p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint64, C.c_int32, C.c_uint32, C.c_void_p]),
}
EXPORTS = tuple(_SIGS)

_lib = None


def lib():
    """The loaded shared object; raises (loudly) if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C poly_b200/csrc`). poly_b200 has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            f = getattr(L, name)
            f.restype = res
            f.argtypes = args
        _lib = L
    return _lib


def last_error() -> str:
    return (lib().pg_last_error() or b"").decode("utf-8", "replace")


def check(rc: int, allow=()) -> int:
    if rc != PG_OK and rc not in allow:
        raise PolyError(rc, last_error())
    return rc


def ptr(a) -> int:
    """Address of a NumPy array (host) or torch tensor (host or device); None -> NULL."""
    if a is None:
        return None
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    return a.ctypes.data
