"""ctypes binding of the C ABI declared in include/buffalo_b200.h.

The shared library is built in-tree (buffalo_b200/libbuffalo_b200.so) by
``buffalo_b200/csrc/build.sh`` (nvcc, sm_90a only).  There is no CPU fallback: if the
library is missing, loading raises; if no Hopper (sm_90) GPU is present, ``init`` fails with the
library's error string.
"""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbuffalo_b200.so")
_SRC_DIR = os.path.join(_HERE, "csrc")

_lib = None

_vp, _i32, _i64, _f, _d, _sz = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_double, C.c_size_t
_cs = C.c_char_p
_pd = C.POINTER(C.c_double)
_pi64 = C.POINTER(C.c_int64)

# name -> (restype, argtypes); one line per declaration in include/buffalo_b200.h
PROTOTYPES = {
    "bfl_last_error": (_cs, []),
    "bfl_abi_version": (C.c_int, []),
    "bfl_compiled_sm": (C.c_int, []),
    "bfl_require_device": (C.c_int, []),
    "bfl_kernel_launch_count": (_i64, []),
    "bfl_ipc_open": (_vp, [_vp]),
    "bfl_ipc_close": (C.c_int, [_vp]),
    "bfl_dev_alloc": (_vp, [_sz]),
    "bfl_dev_free": (C.c_int, [_vp]),
    "bfl_ipc_export": (C.c_int, [_vp, _vp]),
    # ALS
    "bfl_als_create": (_vp, []),
    "bfl_als_destroy": (None, [_vp]),
    "bfl_als_init": (C.c_int, [_vp, _cs]),
    "bfl_als_init_json": (C.c_int, [_vp, _cs]),
    "bfl_als_get_vdim": (C.c_int, [_vp]),
    "bfl_als_initialize_model": (C.c_int, [_vp, _vp, _i32, _vp, _i32]),
    "bfl_als_set_placeholder": (C.c_int, [_vp, _vp, _vp, _sz]),
    "bfl_als_precompute": (C.c_int, [_vp, C.c_int]),
    "bfl_als_partial_update": (C.c_int, [_vp, _i32, _i32, _vp, _vp, _vp, C.c_int, _pd, _pd]),
    "bfl_als_bind_factors_device": (C.c_int, [_vp, _vp, _i64, _vp, _i64]),
    "bfl_als_bind_csr_device": (C.c_int, [_vp, C.c_int, _vp, _vp, _vp, _i64, _i64]),
    "bfl_als_precompute_device": (C.c_int, [_vp, C.c_int, _vp]),
    "bfl_als_precompute_rows_device": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp]),
    "bfl_als_update_device": (C.c_int, [_vp, C.c_int, _i64, _i64, _vp, _vp]),
    "bfl_als_set_peer_replicas": (C.c_int, [_vp, C.c_int, C.c_int, C.POINTER(_vp)]),
    "bfl_als_explain_device": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp]),
    "bfl_als_posterior_sample_device": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, C.c_int, _vp, C.c_uint32, _f, _vp,
                                                  _vp, _vp]),
    "bfl_als_gram_device": (_vp, [_vp]),
    "bfl_als_gram_device_mut": (_vp, [_vp]),
    # SGD (BPRMF / WARP)
    "bfl_sgd_create": (_vp, [C.c_int]),
    "bfl_sgd_destroy": (None, [_vp]),
    "bfl_sgd_init": (C.c_int, [_vp, _cs]),
    "bfl_sgd_init_json": (C.c_int, [_vp, _cs]),
    "bfl_sgd_get_vdim": (C.c_int, [_vp]),
    "bfl_sgd_initialize_model": (C.c_int, [_vp, _vp, _i32, _vp, _i32, _vp, _i64]),
    "bfl_sgd_bind_factors_device": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _i64]),
    "bfl_sgd_set_cumulative_table": (C.c_int, [_vp, _vp, _i32]),
    "bfl_sgd_set_placeholder": (C.c_int, [_vp, _vp, _sz]),
    "bfl_sgd_bind_csr_device": (C.c_int, [_vp, _vp, _vp, _i64, _i64]),
    "bfl_sgd_launch_workers": (C.c_int, [_vp]),
    "bfl_sgd_wait_until_done": (C.c_int, [_vp]),
    "bfl_sgd_join": (C.c_int, [_vp, _pd]),
    "bfl_sgd_add_jobs": (C.c_int, [_vp, _i32, _i32, _vp, _vp]),
    "bfl_sgd_add_jobs_device": (C.c_int, [_vp, _i64, _i64, _vp]),
    "bfl_sgd_update_parameters": (C.c_int, [_vp]),
    "bfl_sgd_update_parameters_device": (C.c_int, [_vp, _vp]),
    "bfl_sgd_synchronize": (C.c_int, [_vp, C.c_int]),
    "bfl_sgd_compute_loss": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _pd]),
    "bfl_sgd_apply_triples_device": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _f, _vp]),
    "bfl_sgd_sample_device": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp]),
    "bfl_sgd_grad_device": (_vp, [_vp, C.c_int]),
    "bfl_sgd_count_device": (_vp, [_vp, C.c_int]),
    "bfl_sgd_set_trace_device": (C.c_int, [_vp, _vp, _vp]),
    "bfl_sgd_epoch": (C.c_int, [_vp]),
    "bfl_sgd_current_lr": (_d, [_vp]),
    "bfl_sgd_read_stats": (C.c_int, [_vp, _pd, _pi64]),
    "bfl_sgd_reduce_items_device": (C.c_int, [_vp, _vp]),
    "bfl_sgd_segment_len": (C.c_int, []),
    "bfl_sgd_fold_in_items_device": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _i64,
                                               _vp, _vp, C.c_int, _vp, _vp, _vp]),
    # PLSI
    "bfl_plsi_create": (_vp, []),
    "bfl_plsi_destroy": (None, [_vp]),
    "bfl_plsi_init": (C.c_int, [_vp, _cs]),
    "bfl_plsi_init_json": (C.c_int, [_vp, _cs]),
    "bfl_plsi_get_vdim": (C.c_int, [_vp]),
    "bfl_plsi_initialize_model": (C.c_int, [_vp, _vp, _i32, _vp, _i32]),
    "bfl_plsi_set_model": (C.c_int, [_vp, _vp, _i32, _vp, _i32]),
    "bfl_plsi_reset": (C.c_int, [_vp]),
    "bfl_plsi_partial_update": (C.c_int, [_vp, _i32, _i32, _vp, _vp, _vp, _pd]),
    "bfl_plsi_normalize": (C.c_int, [_vp, _f, _f]),
    "bfl_plsi_swap": (C.c_int, [_vp]),
    "bfl_plsi_release": (C.c_int, [_vp]),
    "bfl_plsi_bind_factors_device": (C.c_int, [_vp, _vp, _i64, _vp, _i64]),
    "bfl_plsi_bind_csr_device": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64]),
    "bfl_plsi_update_device": (C.c_int, [_vp, _i64, _i64, _vp, _vp]),
    "bfl_plsi_normalize_device": (C.c_int, [_vp, _f, _f, _vp]),
    "bfl_plsi_swap_device": (C.c_int, [_vp, _vp]),
    "bfl_plsi_partial_update_items": (C.c_int, [_vp, _i32, _i32, _vp, _vp, _vp]),
    "bfl_plsi_item_segment_len": (C.c_int, []),
    "bfl_plsi_bind_colwise_csr_device": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64]),
    "bfl_plsi_update_items_device": (C.c_int, [_vp, _i64, _i64, _vp]),
    "bfl_plsi_fold_in_device": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _vp, _i64, _i64, _vp, C.c_int, _f, _vp]),
    # evaluation top-k
    "bfl_topk_device": (C.c_int, [_vp, _i64, C.c_int, _vp, _i64, C.c_int, _vp, C.c_int, C.c_int, _vp, _vp, _vp]),
    "bfl_topk_host": (C.c_int, [_vp, _i64, C.c_int, _vp, _i64, C.c_int, _vp, C.c_int, C.c_int, _vp, _vp]),
    # batch serving top-k
    "bfl_serve_create": (_vp, []),
    "bfl_serve_destroy": (None, [_vp]),
    "bfl_serve_set_items": (C.c_int, [_vp, _vp, _i64, C.c_int, C.c_int, _vp]),
    "bfl_serve_bind_items_device": (C.c_int, [_vp, _vp, _i64, C.c_int, C.c_int, _vp]),
    "bfl_serve_set_queries": (C.c_int, [_vp, _vp, _i64, C.c_int]),
    "bfl_serve_bind_queries_device": (C.c_int, [_vp, _vp, _i64, C.c_int]),
    "bfl_serve_set_pool": (C.c_int, [_vp, _vp, _i64]),
    "bfl_serve_topk": (C.c_int, [_vp, _vp, _i64, C.c_int, _vp, _vp]),
    "bfl_serve_topk_device": (C.c_int, [_vp, _vp, _i64, C.c_int, _vp, _vp, _vp]),
    "bfl_seen_topk": (C.c_int, [_vp, _vp, _i64, C.c_int, _vp, _vp, _vp, _vp]),
    "bfl_seen_topk_device": (C.c_int, [_vp, _vp, _i64, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bfl_cand_topk": (C.c_int, [_vp, _vp, _i64, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bfl_cand_topk_device": (C.c_int, [_vp, _vp, _i64, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bfl_cand_set_budget": (C.c_int, [_vp, _i64]),
    "bfl_mmr_rerank_device": (C.c_int, [_vp, _vp, _vp, _i64, C.c_int, C.c_int, C.c_float, _vp, _vp, _vp]),
    "bfl_category_walk_device": (C.c_int, [_vp, _vp, _i64, C.c_int, _vp, _vp, _vp, C.c_int, C.c_int, C.c_int, _vp, _vp,
                                           _vp, _vp]),
    # IVF index
    "bfl_ivf_create": (_vp, []),
    "bfl_ivf_destroy": (None, [_vp]),
    "bfl_ivf_attach": (C.c_int, [_vp]),
    "bfl_ivf_build_device": (C.c_int, [_vp, _vp, _i64, C.c_int, C.c_int, _vp, C.c_int, C.c_int, C.c_uint64]),
    "bfl_ivf_search_device": (C.c_int, [_vp, _vp, _i64, C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp]),
    "bfl_ivf_set_batch_rows": (C.c_int, [_vp, _i64]),
    "bfl_ivf_info": (C.c_int, [_vp, _pi64, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "bfl_ivf_read": (C.c_int, [_vp, _vp, _vp, _vp]),
    # validation metrics
    "bfl_eval_unsorted_rows_device": (C.c_int, [_vp, _vp, _i64, _vp, _vp]),
    "bfl_eval_topk_masked_device": (C.c_int, [_vp, _i64, C.c_int, _vp, _i64, C.c_int, _vp, C.c_int, C.c_int, _vp, _vp,
                                              _vp, _vp, _vp]),
    "bfl_eval_ranking_terms_device": (C.c_int, [_vp, _i64, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp]),
    "bfl_eval_score_terms_device": (C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _i64, _vp, _vp]),
    "bfl_eval_sum_device": (C.c_int, [_vp, _i64, C.c_int, _vp, _vp]),
    # offline evaluation
    "bfl_eval_cutoff_terms_device": (C.c_int, [_vp, _i64, C.c_int, _vp, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp, _i64,
                                               _vp]),
    "bfl_eval_ild_device": (C.c_int, [_vp, _i64, C.c_int, C.c_int, _vp, C.c_int, C.c_int, _vp, C.c_int, _vp, _i64, _vp]),
    "bfl_eval_coverage_mark_device": (C.c_int, [_vp, _i64, C.c_int, _vp, C.c_int, _vp, _vp]),
    "bfl_eval_coverage_count_device": (C.c_int, [_vp, _i64, C.c_int, _vp, _vp]),
    # ingest helpers
    "bfl_csr_from_triples_device": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, C.c_int, _vp, _vp, _vp, _vp]),
    "bfl_csr_from_triples_host": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, C.c_int, _vp, _vp, _vp]),
    "bfl_popularity_table_device": (C.c_int, [_vp, _i64, _i32, C.c_int, _vp, _vp]),
    "bfl_popularity_table_host": (C.c_int, [_vp, _i64, _i32, C.c_int, _vp]),
    # MatrixMarket ingest
    "bfl_mm_ingest_create": (_vp, [_i32, _i32, _i64, _i64, _i64, _i64]),
    "bfl_mm_ingest_destroy": (None, [_vp]),
    "bfl_mm_ingest_staging": (C.c_int, [_vp, C.c_int, C.POINTER(_vp)]),
    "bfl_mm_ingest_feed": (C.c_int, [_vp, C.c_int, _i64, C.c_int]),
    "bfl_mm_ingest_finish": (C.c_int, [_vp, _pi64, C.POINTER(_i32), _pi64, _pi64, _pi64]),
    "bfl_mm_ingest_slow_tokens": (C.c_int, [_vp, _i64, _vp, _vp, _vp]),
    "bfl_mm_ingest_patch_values": (C.c_int, [_vp, _vp, _vp, _i64]),
    "bfl_mm_ingest_split": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _vp]),
    "bfl_mm_ingest_build": (C.c_int, [_vp, C.c_int, _vp, _vp, _vp]),
    "bfl_mm_ingest_stats": (C.c_int, [_vp, _pd, _pi64]),
    "bfl_stream_ingest_create": (_vp, [_i64, C.c_uint64, _vp, _i32, _i32]),
    "bfl_stream_ingest_destroy": (None, [_vp]),
    "bfl_stream_ingest_staging": (C.c_int, [_vp, C.c_int, C.POINTER(_vp)]),
    "bfl_stream_ingest_load_iid": (C.c_int, [_vp, _vp, _vp, _i64]),
    "bfl_stream_ingest_feed": (C.c_int, [_vp, C.c_int, _i64, C.c_int]),
    "bfl_stream_ingest_finish": (C.c_int, [_vp, _pi64, _pi64, C.POINTER(_i32), C.POINTER(_i32), _pi64]),
    "bfl_stream_ingest_names": (C.c_int, [_vp, _vp, _vp]),
    "bfl_stream_ingest_split": (C.c_int, [_vp, _i32, C.c_int, _i64, _vp, _i64, C.c_int, _pi64, _pi64]),
    "bfl_stream_ingest_vali": (C.c_int, [_vp, _vp, _vp, _vp]),
    "bfl_stream_ingest_build": (C.c_int, [_vp, C.c_int, _vp, _vp, _vp]),
    "bfl_stream_ingest_stats": (C.c_int, [_vp, _pd, _pi64]),
}


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a into buffalo_b200/libbuffalo_b200.so."""
    srcs = [os.path.join(_SRC_DIR, f) for f in os.listdir(_SRC_DIR) if f.endswith((".cu", ".cuh", ".sh"))]
    srcs.append(os.path.join(_HERE, "..", "include", "buffalo_b200.h"))
    newest = max(os.path.getmtime(s) for s in srcs if os.path.exists(s))
    if force or not os.path.isfile(LIB_PATH) or os.path.getmtime(LIB_PATH) < newest:
        out = subprocess.run(["bash", os.path.join(_SRC_DIR, "build.sh")], stdout=subprocess.PIPE,
                             stderr=subprocess.STDOUT, text=True)
        if verbose or out.returncode != 0:
            print(out.stdout)
        if out.returncode != 0:
            raise RuntimeError("nvcc build of libbuffalo_b200.so failed:\n" + out.stdout)
    return LIB_PATH


def lib():
    """Load the shared library (raises if it has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise RuntimeError(
                "buffalo_b200/libbuffalo_b200.so is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). There is no CPU fallback.")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(handle, name)  # AttributeError if the header and the library disagree
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


class BackendError(RuntimeError):
    """Raised when a C-ABI call returns a non-zero status (the reference throws
    std::runtime_error through Cython's `except +`, buffalo/algo/cuda/_als.pyx:14-22)."""


def check(status, what=""):
    if status != 0:
        msg = lib().bfl_last_error()
        raise BackendError("%s failed (status %d): %s" % (what, status, msg.decode("utf-8", "replace") if msg else ""))
    return status
