"""Shared helpers for the parity tests: build the same encode plan for the CUDA path and the oracle."""
import numpy as np
import torch

import oracle
from b200flow import dist as bdist
from b200flow import encode as enc
from b200flow import synth


def kdd_luts_oracle(rec_np, schema, dicts):
    luts, ordered = {}, {}
    for col in synth.KDD_CATEGORICAL + ["label"]:
        counts = oracle.category_counts(rec_np, schema.row_bytes, schema.offsets[col], len(dicts[col]))
        ordered[col], luts[col] = oracle.string_index_order(counts, dicts[col])
    return luts, ordered


def kdd_luts_gpu(rec, schema, dicts, group=None):
    """with a process group, every rank counts its own rows and the counts are summed over the group, so every rank
    orders the categories as one process holding all the rows would"""
    luts, ordered = {}, {}
    for col in synth.KDD_CATEGORICAL + ["label"]:
        counts = enc.category_counts(rec, schema, col, len(dicts[col]))
        if group is not None:
            bdist.all_reduce_sum_(counts, group)
        ordered[col], luts[col] = enc.string_index_order(counts.cpu().numpy(), dicts[col])
    return luts, ordered


def kdd_plan(schema, luts, ordered, onehot=False, label=True):
    """script-faithful plan (kdd99.py:39-46): the 38 numeric columns in file order, then the 3 indexed columns;
    onehot=True replaces the indexed columns by dropLast one-hot blocks (north_star full encode)."""
    plan = enc.EncodePlan(schema)
    for c in synth.KDD_COLUMNS:
        if c not in synth.KDD_CATEGORICAL and c != "label":
            plan.add_numeric(c)
    for c in synth.KDD_CATEGORICAL:
        if onehot:
            plan.add_onehot(c, luts[c], len(ordered[c]))
        else:
            plan.add_index(c, luts[c])
    if label:
        plan.set_label("label", luts["label"])
    return plan


def oracle_encode(plan, rec_np):
    loff, llo, lln = plan.label if plan.label else (-1, 0, 0)
    return oracle.encode(rec_np, plan.schema.row_bytes, plan.slot_array(), plan.lut_array(), loff, llo, lln, plan.check_nan)


def forests_equal(ex_gpu, ex_orc):
    """exact comparison of two canonical forest exports; returns list of mismatching keys."""
    bad = []
    if len(ex_gpu["nid"]) != len(ex_orc["nid"]):
        return ["num_nodes %d vs %d" % (len(ex_gpu["nid"]), len(ex_orc["nid"]))]
    for k in ("tree", "nid", "feat", "kind", "bin_thr", "is_leaf", "mask", "counts"):
        if not np.array_equal(np.asarray(ex_gpu[k]).astype(np.int64) if k != "mask" else ex_gpu[k],
                              np.asarray(ex_orc[k]).astype(np.int64) if k != "mask" else ex_orc[k]):
            bad.append(k)
    internal = ex_orc["is_leaf"] == 0
    if not np.array_equal(ex_gpu["gain"][internal], ex_orc["gain"][internal]):
        bad.append("gain")
    return bad
