"""Bit-packed TreePoint records of the fused level kernel: the host layout (b200flow_packed_layout) and the pack kernel."""
import numpy as np
import pytest
import torch

import oracle
from b200flow import _lib, forest as fr, synth
from util import forests_equal, kdd_luts_gpu, kdd_luts_oracle, kdd_plan, oracle_encode


def _fields(desc):
    word, shift, mask = desc & 0xff, (desc >> 8) & 0xff, desc >> 16
    return word, shift, mask


def _check_layout(feat_bins, C):
    desc, rec_bytes = _lib.packed_layout(feat_bins, C)
    word, shift, mask = _fields(desc)
    width = np.array([int(mk).bit_length() for mk in mask])
    assert (mask == (1 << width) - 1).all()
    assert (shift + width <= 32).all()                                        # no field crosses a word
    for w in np.unique(word):                                                  # fields of one word do not overlap
        bits = 0
        for f in np.nonzero(word == w)[0]:
            assert bits & (int(mask[f]) << int(shift[f])) == 0
            bits |= int(mask[f]) << int(shift[f])
    values = np.append(np.asarray(feat_bins), C)
    assert (mask >= values - 1).all()                                          # every width covers n_bins - 1 and C - 1 ...
    assert (width == np.maximum(1, [int(v - 1).bit_length() for v in values])).all()   # ... and no more
    if rec_bytes:
        assert rec_bytes % 16 == 0 and (word.max() + 1) * 4 <= rec_bytes
    return desc, rec_bytes


def _kdd_feat_bins(n_classes):
    # the bins of the benchmark's KDD fit (max_bins 70), from the CPU oracle's findSplits on the synthetic generator
    rec, dicts = synth.make_kdd(200000, n_classes, seed=3)
    schema = synth.kdd_schema()
    rn = rec.numpy()
    luts, ordered = kdd_luts_oracle(rn, schema, dicts)
    x, _, _ = oracle_encode(kdd_plan(schema, luts, ordered), rn)
    arity = np.array([0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL], np.int32)
    mpb, _, _ = oracle.build_metadata(len(x), 41, n_classes, arity, 70, 100)
    _, n_thr, _ = oracle.find_splits(x, 2019, int(min(1.0, max(mpb * mpb, 10000) / len(x)) * 4294967296.0), arity, mpb)
    return np.where(arity > 0, arity, n_thr + 1).astype(np.int32), len(ordered["label"])


@pytest.mark.parametrize("n_classes", [5, 23])
def test_kdd_records_pack_into_32_bytes(n_classes):
    fb, C = _kdd_feat_bins(n_classes)
    _, rec_bytes = _check_layout(fb, C)
    assert rec_bytes == 32
    assert _lib.route_hist_config(41, 7, int(fb.max()), C, rec_bytes) is not None


@pytest.mark.parametrize("C", [6, 14, 15])
def test_78_features_of_7_bits_keep_byte_records(C):
    # CICIDS width with every feature at 65-78 bins (7 bits): 80 packed bytes are 5 granules, as many as the 79-byte record.
    # (The benchmark's CICIDS fits have many few-bin columns and pack to 64 bytes.)
    for bins in (78, 65):
        assert _check_layout(np.full(78, bins, np.int32), C)[1] == 0


def test_power_of_two_bin_counts_get_exact_widths():
    for k in range(0, 9):
        fb = np.full(3, 1 << k, np.int32)
        desc, _ = _check_layout(fb, 2)
        assert (_fields(desc)[2][:3] == max(1, (1 << k) - 1)).all()
    desc, _ = _check_layout(np.array([2, 3, 4, 5, 129, 256, 1], np.int32), 256)
    assert _fields(desc)[2].tolist() == [1, 3, 3, 7, 255, 255, 1, 255]


def test_more_than_255_features_keep_byte_records():
    # the level kernel does not take records of more than 255 features (unfused kernels): the layout must not fail them
    assert _lib.packed_layout(np.full(300, 2, np.int32), 2)[1] == 0
    assert _lib.route_hist_config(300, 18, 32, 2) is None


def test_packing_needs_a_saved_granule():
    assert _check_layout(np.full(14, 2, np.int32), 2)[1] == 0                  # 15 bytes: one granule either way
    assert _check_layout(np.full(16, 2, np.int32), 2)[1] == 16                 # 17 bytes (two granules) -> 17 bits
    assert _check_layout(np.full(200, 256, np.int32), 2)[1] == 0               # nothing to save at 8 bits per bin


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 1000, 70001])
def test_unpacked_fields_equal_the_byte_records(n):
    fb, C = np.array([70, 2, 3, 16, 17, 256, 1, 5, 70, 12] * 4 + [9], np.int32), 23
    desc, rec_bytes = _check_layout(fb, C)
    assert rec_bytes == 32
    g = np.random.default_rng(n)
    tp = np.zeros((n, fr.tp_stride(41)), np.uint8)
    tp[:, :41] = g.integers(0, fb, size=(n, 41))
    tp[:, 41] = g.integers(0, C, size=n)
    packed = fr.pack_records(torch.from_numpy(tp).cuda(), 41, torch.from_numpy(desc).cuda(), rec_bytes).cpu().numpy()
    words = packed.view(np.uint32)
    word, shift, mask = _fields(desc)
    got = (words[:, word] >> shift.astype(np.uint32)) & mask.astype(np.uint32)
    assert np.array_equal(got, tp[:, :42].astype(np.uint32))
    used = np.zeros(rec_bytes // 4, np.uint64)
    for f in range(42):
        used[word[f]] |= np.uint64(int(mask[f]) << int(shift[f]))
    assert not (words.astype(np.uint64) & ~used).any()                         # no stray bits outside the fields


def _dense(n, F, C, seed):
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    x = torch.rand((n, F), dtype=torch.float64, device="cuda", generator=g)
    y = ((x[:, 0] > 0.5).to(torch.int64) + (x[:, 1] + x[:, 2] > 1.0).to(torch.int64)) % C
    flip = torch.rand(n, device="cuda", generator=g) < 0.05
    y = torch.where(flip, torch.randint(0, C, (n,), device="cuda", generator=g), y)
    return x, y.to(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("case,rec_bytes", [("dense20", 16), ("kdd", 32), ("dense60", 48)])
def test_packed_fits_build_the_byte_record_forest(case, rec_bytes, monkeypatch):
    # each packed record size (1, 2 and 3 granules) through the fused kernel against the unfused kernels on byte records
    if case == "kdd":
        rec, dicts = synth.make_kdd(60000, 5, seed=19, device="cuda")
        schema = synth.kdd_schema()
        luts, ordered = kdd_luts_gpu(rec, schema, dicts)
        x, y, _ = kdd_plan(schema, luts, ordered).run(rec, torch.float64)
        arity, C, max_bins = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL], len(ordered["label"]), 70
    else:
        F = 20 if case == "dense20" else 60
        C, max_bins = 3, 4 if case == "dense20" else 32                       # 2 or 5 bits per feature
        x, y = _dense(40000, F, C, F)
        arity = [0] * F
    p = fr.ForestParams(num_trees=5, max_bins=max_bins, max_depth=8, seed=7)
    monkeypatch.setattr(fr, "FUSED", False)
    want = fr.fit_forest(x, y, C, arity, p)
    assert want.train_stats["record_format"] == "bytes"
    monkeypatch.setattr(fr, "FUSED", True)
    got = fr.fit_forest(x, y, C, arity, p)
    assert (got.train_stats["record_format"], got.train_stats["record_bytes"]) == ("packed", rec_bytes)
    eg, ew = got.export(), want.export()
    assert forests_equal(eg, ew) == [] and np.array_equal(eg["gain"], ew["gain"])


@pytest.mark.gpu
def test_fit_with_more_than_255_features_runs_on_byte_records():
    F, C = 300, 3
    x, y = _dense(3000, F, C, 5)
    p = fr.ForestParams(num_trees=3, max_bins=16, max_depth=4, seed=11)
    model = fr.fit_forest(x, y, C, [0] * F, p)
    assert model.train_stats["record_format"] == "bytes" and model.train_stats["route_chunk"] == 0
    fo, _ = oracle.fit_forest(x.cpu().numpy(), y.cpu().numpy(), C, [0] * F, num_trees=3, max_bins=16, max_depth=4, seed=11)
    assert forests_equal(model.export(), fo.export()) == []
