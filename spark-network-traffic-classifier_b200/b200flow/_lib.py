"""ctypes binding of libb200flow.so (include/b200flow.h).

The CUDA library is the product path: there is no CPU fallback.  Importing this module
without a built libb200flow.so, or calling into it without a CUDA device, raises.
"""
import ctypes as C
import os

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200flow.so")

F32, F64, I32 = 0, 1, 2
SRC_F32, SRC_F64, SRC_I32, SRC_INDEX, SRC_ONEHOT = 0, 1, 2, 3, 4

SLOT_DTYPE = np.dtype([("kind", "<i4"), ("src_off", "<i4"), ("lut_off", "<i4"), ("lut_len", "<i4"),
                       ("hot", "<i4"), ("reserved", "<i4"), ("mean", "<f8"), ("scale", "<f8")])
SPLIT_DTYPE = np.dtype([("feat", "<i4"), ("kind", "<i4"), ("bin_thr", "<i4"), ("flags", "<i4"),
                        ("gain", "<f8"), ("impurity", "<f8"), ("mask", "<u8", (4,))])
NODE_DTYPE = np.dtype([("feat", "<i4"), ("kind_bin", "<i4"), ("left", "<i4"), ("nid", "<u4")])
assert SLOT_DTYPE.itemsize == 40 and SPLIT_DTYPE.itemsize == 64 and NODE_DTYPE.itemsize == 16


class B200FlowError(RuntimeError):
    pass


class UnsupportedParamError(B200FlowError, ValueError):
    """a parameter value MLlib accepts but the CUDA path does not implement (entropy impurity, maxBins > 256, ...): a
    ValueError, so the pyspark shim reports it as IllegalArgumentException; CUDA/runtime failures stay B200FlowError."""


_P, _I32, _I64, _U64, _F64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_double

# name -> argtypes, exactly the prototypes of include/b200flow.h
_SIGNATURES = {
    "b200flow_category_counts": [_P, _I64, _I32, _I32, _I32, _P, _P],
    "b200flow_category_counts_multi": [_P, _I64, _I32, _I32, _P, _P, _P, _P],
    "b200flow_encode": [_P, _I64, _I32, _P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _P, _I32, _P, _P, _P],
    "b200flow_sample_records": [_P, _I64, _I32, _P, _I32, _P, _I32, _U64, _U64, _I64, _P, _I64, _P, _P],
    "b200flow_encode_bins": [_P, _I64, _I32, _P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _I32, _P, _I32, _P, _P, _P],
    "b200flow_column_moments": [_P, _I32, _I64, _I32, _I64, _P, _P, _P, _P],
    "b200flow_sample_rows": [_P, _I32, _I64, _I32, _I64, _U64, _U64, _I64, _P, _I64, _P, _P],
    "b200flow_find_splits": [_P, _I64, _I32, _I32, _P, _I32, _P, _P, _P, _P],
    "b200flow_bin_rows": [_P, _I32, _I64, _I32, _I64, _P, _P, _P, _I32, _P, _P, _I32, _P, _P],
    "b200flow_dedup_rows": [_P, _I64, _I32, _I32, _P, _P, _I64, _P, _P, _P, _P, _P, _P, _P, _P],
    "b200flow_bag_weights": [_U64, _I32, _I64, _I64, _P, _P, _P, _P, _I64, _P, _P],
    "b200flow_group_rows": [_P, _I64, _I64, _P, _P, _P, _P, _P, _P],
    "b200flow_bag_count": [_P, _I32, _I64, _P, _P],
    "b200flow_bag_fill": [_P, _I32, _I64, _P, _P, _P],
    "b200flow_exclusive_scan_i32_to_i64": [_P, _I64, _P, _P, _P],
    "b200flow_feature_subsets": [_U64, _I32, _P, _P, _I32, _I32, _P, _P],
    "b200flow_hist_level": [_P, _I32, _I32, _P, _I32, _P, _P, _P, _I64, _I32, _P, _I32, _I32, _I32, _P, _P],
    "b200flow_score_level": [_P, _I32, _P, _I32, _I32, _I32, _P, _P, _I32, _I32, _I32, _F64, _P, _P, _P, _P, _P],
    "b200flow_grow_level": [_I32, _P, _P, _P, _P, _P, _P, _P, _I32, _P, _P, _P, _P, _I64, _P, _P, _P, _P, _P, _P, _P],
    "b200flow_route_hist_level": [_P, _I32, _I32, _P, _P, _P, _I32, _P, _P, _P, _P, _I64, _I32, _P, _P, _P, _P, _P, _I32, _I32,
                                  _I32, _P, _I32, _P],
    "b200flow_pack_records": [_P, _I32, _I64, _I32, _P, _I32, _P, _P],
    "b200flow_partition_level": [_P, _I32, _P, _P, _I32, _P, _P, _P, _I64, _I32, _P, _P, _P],
    "b200flow_plan_route": [_I32, _P, _P, _P, _I32, _P, _P, _P, _P, _P],
    "b200flow_next_segments": [_I32, _P, _P, _P, _P, _P, _P, _P, _P],
    "b200flow_finalize_forest": [_I64, _P, _I32, _P, _P],
    "b200flow_build_top_nodes": [_P, _P, _I64, _I32, _I32, _P, _P],
    "b200flow_forest_layout_size": [_P, _P, _I64, _I32, _I32, _P, _P, _P],
    "b200flow_build_forest_layout": [_P, _P, _P, _P, _P, _I64, _I32, _I32, _I32, _P, _P, _P, _P],
    "b200flow_predict_forest": [_P, _I32, _I32, _I64, _P, _P, _I32, _I32, _P, _P, _P, _P],
    "b200flow_gather_rows": [_P, _I32, _P, _I64, _P, _P],
    "b200flow_confusion": [_P, _P, _I64, _I32, _P, _P],
    "b200flow_predict_grid_confusion": [_P, _I32, _I32, _I64, _P, _P, _P, _P, _P, _I32, _I32, _I32, _P, _I32, _P, _I32, _P, _I32,
                                        _I32, _I32, _P, _P],
    "b200flow_predict_grid_scores": [_P, _I32, _I32, _I64, _P, _P, _P, _P, _I32, _I32, _I32, _P, _I32, _P, _I32, _P, _I32, _I32,
                                     _P],
    "b200flow_binary_counts": [_P, _I64, _P, _P, _I64, _I32, _I64, _P, _I64, _P, _P, _P, _I64, _P, _P, _P],
    "b200flow_binary_curve": [_P, _P, _P, _I64, _P, _I32, _I32, _P, _P, _P, _P, _P, _P, _P],
    "b200flow_kmeans_assign": [_P, _I64, _I32, _I64, _P, _I32, _P, _P, _P],
    "b200flow_group_sums": [_P, _I64, _P, _I64, _I32, _I32, _I64, _P, _P, _P],
    "b200flow_group_sums_chain": [_P, _I64, _I32, _I32, _P, _P],
    "b200flow_kmeans_row_keys": [_U64, _I64, _I64, _P, _P],
    "b200flow_kmeans_select": [_U64, _I64, _I64, _I32, _P, _I32, _F64, _P, _P],
    "b200flow_silhouette_rows": [_P, _I64, _I32, _I64, _P, _P, _P, _P, _P, _I32, _P, _P],
    "b200flow_bkm_assign": [_P, _I64, _I32, _I64, _P, _I32, _P, _P, _I32, _P, _P, _P, _P, _P],
    "b200flow_bkm_predict": [_P, _I64, _I32, _I64, _P, _P, _P, _P, _I32, _I32, _P, _P, _P],
    "b200flow_mlp_loss_grad": [_P, _I32, _I64, _I64, _P, _P, _I32, _P, _I64, _P, _P],
    "b200flow_mlp_forward": [_P, _I32, _I64, _I64, _P, _I32, _P, _P, _P],
    "b200flow_svc_loss_grad": [_P, _I32, _I64, _I64, _I32, _P, _P, _I64, _P, _P, _I64, _P, _P],
    "b200flow_svc_margins": [_P, _I32, _I64, _I64, _I32, _I64, _P, _P, _P],
    "b200flow_linreg_loss_grad": [_P, _I32, _I64, _I64, _I32, _P, _P, _P, _F64, _F64, _P, _P, _F64, _I32, _I64, _P, _P],
    "b200flow_aft_loss_grad": [_P, _I32, _I64, _I64, _I32, _P, _P, _P, _P, _P, _P, _I64, _P, _P],
    "b200flow_glm_rows": [_P, _I32, _I64, _I64, _I32, _P, _P, _P, _P, _F64, _F64, _I32, _I32, _F64, _F64, _I32, _I64, _P, _P,
                          _P],
    "b200flow_isotonic_fit": [_P, _I32, _I64, _P, _I64, _P, _I64, _I64, _I32, _I64, _P, _I64, _P, _P, _P, _P, _P],
    "b200flow_isotonic_predict": [_P, _I32, _I64, _I64, _P, _P, _I64, _P, _P],
    "b200flow_column_stats": [_P, _I64, _I64, _I32, _P, _I32, _F64, _P, _P],
    "b200flow_column_sums": [_P, _I64, _I64, _I32, _P, _I32, _F64, _P, _P, _P],
    "b200flow_quantile_hist": [_P, _I64, _I64, _I32, _P, _I32, _F64, _I64, _P, _I32, _I64, _P, _P],
    "b200flow_quantile_step": [_I64, _I32, _P, _P, _I32, _P],
    "b200flow_bucketize": [_P, _I64, _I64, _I32, _P, _P, _P, _P, _P, _P, _P],
    "b200flow_impute_fill": [_P, _I64, _I64, _I32, _P, _I32, _F64, _P, _P, _P],
    "b200flow_min_max": [_P, _I64, _I64, _I32, _P, _P, _P, _F64, _F64, _P, _P],
    "b200flow_mode_keys": [_P, _I64, _I64, _P, _I32, _F64, _P, _P, _P],
    "b200flow_mode": [_P, _I64, _P, _I64, _P, _P],
    "b200flow_fm_loss_grad": [_P, _I32, _I64, _I64, _I32, _I32, _P, _P, _I64, _P, _F64, _U64, _I64, _P, _P],
    "b200flow_fm_regression_loss_grad": [_P, _I32, _I64, _I64, _I32, _I32, _P, _P, _F64, _U64, _I64, _P, _P],
    "b200flow_fm_raw": [_P, _I32, _I64, _I64, _I32, _I32, _I64, _P, _P, _P],
    "b200flow_gmm_estep": [_P, _I64, _I32, _I64, _I32, _P, _P, _P, _I64, _P, _P, _P, _P],
    "b200flow_gmm_moments": [_P, _I64, _I32, _I64, _I32, _P, _I64, _P, _P],
    "b200flow_centered_gram": [_P, _I64, _I32, _I64, _P, _I64, _P, _P],
    "b200flow_weighted_centered_gram": [_P, _I64, _I32, _I64, _P, _P, _I64, _P, _P],
    "b200flow_pca_project": [_P, _I64, _I32, _I64, _P, _I32, _P, _P],
    "b200flow_distinct_values": [_P, _I64, _I32, _I64, _P, _P, _P, _P],
    "b200flow_dictionary_ids": [_P, _I64, _I64, _P, _I32, _P, _P],
    "b200flow_contingency_counts": [_P, _I64, _I32, _I64, _P, _I32, _P, _P, _I64, _P, _P],
    "b200flow_group_centered_moments": [_P, _I64, _I32, _I64, _P, _I32, _P, _P, _F64, _I64, _P, _P],
    "b200flow_gbt_hist_level": [_P, _I32, _P, _P, _I32, _P, _P, _P, _I64, _I32, _P, _I32, _I32, _P, _P],
    "b200flow_gbt_hist_level_classes": [_P, _I32, _P, _P, _I64, _P, _I32, _P, _P, _P, _I64, _I32, _P, _I32, _I32, _P, _P],
    "b200flow_gbt_score_level": [_P, _I32, _P, _I32, _I32, _P, _P, _I32, _I32, _I32, _I32, _I32, _F64, _P, _P, _P, _P, _P],
    "b200flow_gbt_leaf_values": [_I64, _P, _P, _P, _I32, _P, _P],
    "b200flow_gbt_update": [_P, _I32, _I32, _I64, _P, _P, _P, _I32, _I32, _I32, _P, _P, _P],
    "b200flow_gbt_update_classes": [_P, _I32, _I32, _I64, _I32, _P, _P, _P, _I32, _I32, _I32, _I32, _P, _P, _P],
    "b200flow_gbt_output": [_P, _I64, _P, _P, _P, _P],
    "b200flow_reg_labels": [_P, _I64, _P, _I32, _I32, _P, _P],
    "b200flow_reg_tree_weights": [_P, _I32, _I64, _P, _P],
    "b200flow_reg_grid": [_P, _I32, _I32, _P, _I64, _I32, _I32, _I32, _P, _P],
    "b200flow_reg_leaf_table": [_I64, _P, _I32, _I32, _P, _I32, _P],
    "b200flow_reg_divide": [_P, _I64, _F64, _P, _P],
    "b200flow_gbr_leaf_values": [_I64, _P, _P, _I32, _F64, _I32, _P, _P],
    "b200flow_gbr_update": [_P, _I32, _I32, _P, _I64, _P, _P, _P, _I32, _I32, _P, _P, _P, _P],
    "b200flow_reg_eval_max": [_P, _P, _I64, _I32, _F64, _P, _P],
    "b200flow_reg_eval_sums": [_P, _P, _I64, _I32, _F64, _I32, _I32, _I32, _I32, _P, _P],
    "b200flow_random_split": [_U64, _I64, _I64, _P, _I32, _P, _P],
    "b200flow_compact_rows": [_P, _I64, _I32, _P, _I32, _P, _P, _P, _P],
    "b200flow_csv_count_lines": [_P, _I64, _P, _P, _P],
    "b200flow_csv_line_starts": [_P, _I64, _P, _P, _P],
    "b200flow_csv_infer": [_P, _I64, _P, _I64, _I32, _I32, _P, _P, _P, _P],
    "b200flow_csv_dictionary": [_P, _I64, _P, _I64, _I32, _I32, _P, _P, _P, _I32, _P, _P],
    "b200flow_csv_parse": [_P, _I64, _P, _I64, _I32, _I32, _P, _P, _P, _P, _I32, _P, _I32, _P, _P],
}
EXPORTS = sorted(list(_SIGNATURES) + ["b200flow_last_error", "b200flow_version", "b200flow_route_hist_config",
                                       "b200flow_packed_layout", "b200flow_binary_counts_scratch",
                                       "b200flow_group_sums_chunks", "b200flow_mlp_config",
                                       "b200flow_svc_config", "b200flow_fm_config",
                                       "b200flow_isotonic_scratch", "b200flow_mode_scratch"])

_lib = None
launches = 0   # kernels of OURS launched so far (counted per C-ABI call); bench.py reads the delta over the timed region
_KERNELS_PER_CALL = {"b200flow_grow_level": 3, "b200flow_compact_rows": 3, "b200flow_route_hist_level": 2, "b200flow_dedup_rows": 5, "b200flow_group_rows": 3}


def load():
    """dlopen libb200flow.so and declare every prototype; raises if the library is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200FlowError("libb200flow.so is not built (%s missing): run `python -c 'import __graft_entry__ as g; "
                                "g.build()'` or `make -C spark-network-traffic-classifier_b200/csrc`. There is no CPU "
                                "fallback for the product path." % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        for name, args in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.argtypes = args
            fn.restype = C.c_int
        lib.b200flow_last_error.restype = C.c_char_p
        lib.b200flow_version.restype = C.c_int
        lib.b200flow_route_hist_config.argtypes = [_I32] * 5 + [C.POINTER(_I32), C.POINTER(_I32)]
        lib.b200flow_route_hist_config.restype = C.c_int
        lib.b200flow_packed_layout.argtypes = [_I32, _P, _I32, _P, C.POINTER(_I32)]
        lib.b200flow_packed_layout.restype = C.c_int
        lib.b200flow_binary_counts_scratch.argtypes = [_I32, _I64, C.POINTER(_I64)]
        lib.b200flow_binary_counts_scratch.restype = C.c_int
        lib.b200flow_group_sums_chunks.argtypes = [_I64, _I64, C.POINTER(_I64)]
        lib.b200flow_group_sums_chunks.restype = C.c_int
        lib.b200flow_mlp_config.argtypes = [_P, _I32, C.POINTER(_I64), C.POINTER(_I64)]
        lib.b200flow_mlp_config.restype = C.c_int
        lib.b200flow_svc_config.argtypes = [_I32, _I64, C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I64)]
        lib.b200flow_svc_config.restype = C.c_int
        lib.b200flow_fm_config.argtypes = [_I32, _I32, _I64, C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I64)]
        lib.b200flow_fm_config.restype = C.c_int
        lib.b200flow_isotonic_scratch.argtypes = [_I64, C.POINTER(_I64)]
        lib.b200flow_isotonic_scratch.restype = C.c_int
        lib.b200flow_mode_scratch.argtypes = [_I64, C.POINTER(_I64)]
        lib.b200flow_mode_scratch.restype = C.c_int
        _lib = lib
    return _lib


def route_hist_config(F, m, n_bins, n_classes, rec_bytes=0):
    """launch shape of the fused route + histogram kernel: (chunk_rows, m_pass) or None when it cannot run (host-only call).
    rec_bytes: size of the packed records it gathers (packed_layout), 0 for byte records."""
    ch, mp = _I32(0), _I32(0)
    ok = load().b200flow_route_hist_config(int(F), int(m), int(n_bins), int(n_classes), int(rec_bytes), C.byref(ch), C.byref(mp))
    return (int(ch.value), int(mp.value)) if ok else None


def packed_layout(feat_bins, n_classes):
    """bit-packed TreePoint layout of the level kernel (host-only call): (desc int32[F + 1], rec_bytes); rec_bytes == 0 means
    the byte records stay (packing would not save a 16-byte granule)."""
    fb = np.ascontiguousarray(feat_bins, dtype=np.int32)
    desc = np.zeros(fb.shape[0] + 1, np.int32)
    rb = _I32(0)
    lib = load()
    if lib.b200flow_packed_layout(int(fb.shape[0]), fb.ctypes.data, int(n_classes), desc.ctypes.data, C.byref(rb)) != 0:
        raise B200FlowError("b200flow_packed_layout failed: %s" % lib.b200flow_last_error().decode())
    return desc, int(rb.value)


def binary_counts_scratch(S, n):
    """bytes of device scratch b200flow_binary_counts needs for S segments of n scores (host-only call)."""
    out = _I64(0)
    lib = load()
    if lib.b200flow_binary_counts_scratch(int(S), int(n), C.byref(out)) != 0:
        raise B200FlowError("b200flow_binary_counts_scratch failed: %s" % lib.b200flow_last_error().decode())
    return int(out.value)


def isotonic_scratch(n):
    """bytes of device scratch b200flow_isotonic_fit needs for n rows (host-only call)."""
    out = _I64(0)
    lib = load()
    if lib.b200flow_isotonic_scratch(int(n), C.byref(out)) != 0:
        raise B200FlowError("b200flow_isotonic_scratch failed: %s" % lib.b200flow_last_error().decode())
    return int(out.value)


def mode_scratch(M):
    """bytes of device scratch b200flow_mode needs for M keys (host-only call)."""
    out = _I64(0)
    lib = load()
    if lib.b200flow_mode_scratch(int(M), C.byref(out)) != 0:
        raise B200FlowError("b200flow_mode_scratch failed: %s" % lib.b200flow_last_error().decode())
    return int(out.value)


def group_sums_chunks(row_offset, n_rows):
    """number of 4096-row global chunks that rows [row_offset, row_offset + n_rows) touch (host-only call)."""
    out = _I64(0)
    lib = load()
    if lib.b200flow_group_sums_chunks(int(row_offset), int(n_rows), C.byref(out)) != 0:
        raise B200FlowError("b200flow_group_sums_chunks failed: %s" % lib.b200flow_last_error().decode())
    return int(out.value)


def mlp_config(layers):
    """(P, shared-memory bytes) of the MLP kernels for a layer list (host-only call); raises UnsupportedParamError beyond
    the kernels' limits."""
    la = np.ascontiguousarray(layers, dtype=np.int32)
    P, sm = _I64(0), _I64(0)
    lib = load()
    if lib.b200flow_mlp_config(la.ctypes.data, int(la.shape[0]), C.byref(P), C.byref(sm)) != 0:
        raise UnsupportedParamError("layers %s: %s" % (list(map(int, la)), lib.b200flow_last_error().decode()))
    return int(P.value), int(sm.value)


def svc_config(D, K):
    """(columns per class block, class blocks, shared-memory bytes) of the LinearSVC kernels (host-only call); raises
    UnsupportedParamError beyond the kernels' limits."""
    kb, nb, sm = _I32(0), _I32(0), _I64(0)
    lib = load()
    if lib.b200flow_svc_config(int(D), int(K), C.byref(kb), C.byref(nb), C.byref(sm)) != 0:
        raise UnsupportedParamError("LinearSVC with %d features: %s" % (int(D), lib.b200flow_last_error().decode()))
    return int(kb.value), int(nb.value), int(sm.value)


def fm_config(D, factor_size, K):
    """(classes per class block, class blocks, shared-memory bytes) of the FMClassifier kernels (host-only call); raises
    UnsupportedParamError beyond the kernels' limits."""
    kb, nb, sm = _I32(0), _I32(0), _I64(0)
    lib = load()
    if lib.b200flow_fm_config(int(D), int(factor_size), int(K), C.byref(kb), C.byref(nb), C.byref(sm)) != 0:
        raise UnsupportedParamError("FMClassifier with %d features and factorSize %d: %s"
                                    % (int(D), int(factor_size), lib.b200flow_last_error().decode()))
    return int(kb.value), int(nb.value), int(sm.value)


def ptr(t):
    """device pointer of a torch tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise B200FlowError("b200flow kernels need CUDA tensors (got %s); there is no CPU fallback" % t.device)
    if not t.is_contiguous():
        raise B200FlowError("b200flow kernels need contiguous tensors")
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def call(name, *args):
    """invoke one entry point on torch's current stream and raise on a non-zero return code."""
    global launches
    lib = load()
    rc = getattr(lib, name)(*args, stream())
    launches += _KERNELS_PER_CALL.get(name, 1)
    if rc != 0:
        raise B200FlowError("%s failed (%d): %s" % (name, rc, lib.b200flow_last_error().decode()))


def h2d(a, device):
    """small host array -> device tensor through a pinned staging block, asynchronously.  A pageable cudaMemcpy blocks the
    host until the stream reaches it, which stops the level loop from running ahead of the GPU; pinned + non_blocking does
    not (torch's caching host allocator keeps the block alive until the copy has run)."""
    t = torch.from_numpy(np.ascontiguousarray(a))
    if torch.device(device).type != "cuda":
        return t.clone()
    return t.pin_memory().to(device, non_blocking=True)


def require_cuda():
    if not torch.cuda.is_available():
        raise B200FlowError("no CUDA device: the b200flow product path has no CPU fallback")
    load()


def dtype_code(t):
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.float64:
        return F64
    raise B200FlowError("dense matrices must be float32 or float64, got %s" % t.dtype)
