"""Edge cases of the fused encode path (csrc/encode.cu) that the KDD / CICIDS record sets never reach.

encode_kernel: both thread -> slot mappings (n_out <= 256 and above), the shared rank pre-pass and the inline lookups
(1 to 12 categorical sources), slot de-duplication on and off (n_out <= 1024 and above), the LUT pool in shared and in
global memory, scaled slots of every kind, f64 fields at offsets = 4 (mod 8), label-only plans, tile sizes R and the TMA
ring around a ragged last tile, the two-stage ring and the width limit.  encode_bins_kernel and sample_records_kernel:
the fp64 threshold table in global memory, the float table fed by non-f32 sources, maxBins 2 and 256, categorical
arities 254-256 with out-of-range cells, F + 1 not a multiple of the warp count.  StandardScaler.fit (column_moments)
against exact sums, and the routing of categorical values a model never saw.

Every f64 output is compared bit for bit with the CPU oracle; an f32 output must be the oracle's fp64 value rounded once
(the kernel computes in fp64 and rounds once to the output type), so it is compared bit for bit too."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle
from b200flow import _lib, encode as enc, forest as fr
from b200flow._lib import SRC_F32, SRC_F64, SRC_INDEX, SRC_ONEHOT, ptr
from util import oracle_encode

DEV = "cuda"
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
PKG = os.path.join(ROOT, "spark-network-traffic-classifier_b200")

U = 2.0 ** -53                                   # unit roundoff of fp64


def _gamma(k):
    """Higham's gamma_k = k u / (1 - k u): the relative error bound of k chained fp64 roundings."""
    return k * U / (1.0 - k * U)


# ------------------------------------------------------------------------------- encode launch arithmetic
def _enc_launch(n_rows, row_bytes, n_out, out_bytes, lut_total, stages=3, budget_kb=52):
    """(R, dynamic shared memory bytes, grid) of encode_kernel.  Restates b200flow_encode in csrc/encode.cu, the lines
    from `const int fixed_bytes = ...` to `int grid = ...`, with kEncStages = kEncOutBufs = 3, kEncMaxCat = 8,
    sizeof(b200flow_slot) = 40 and kNumSMs = 132."""
    lut_smem = lut_total * 4 if 0 < lut_total <= 4096 else 0
    fixed = 3 * 8 + n_out * 40 + lut_smem + 1024 + 3 * 9 * 4 + 4 * (n_out + 1)
    per_row = row_bytes * stages + n_out * out_bytes * 3 + 8 + 8 * 4
    budget = budget_kb * 1024 - fixed
    R = budget // per_row if budget > 0 else 0
    R = min(max(R, 4), 512) & ~3
    R = min(R, (n_rows + 3) & ~3)
    in_stride = (R * row_bytes + 127) & ~127
    out_stride = (R * n_out * out_bytes + 127) & ~127
    smem = (stages * in_stride + 3 * out_stride + 3 * 8 + (2 * R + 2) * 4 + n_out * 40 + lut_smem + 16 + 3 * 9 * 4 +
            R * 8 * 4 + 4 * (n_out + 1))
    ctas = min(max((220 * 1024) // (smem + 1024), 1), 8)
    return R, smem, min((n_rows + R - 1) // R, 132 * ctas)


# static shared memory of encode_kernel (ptxas: 128 bytes): sh_ncat, padded to the 128-byte alignment of the dynamic window
ENC_STATIC_SMEM = 128
# f64 records in, f64 vector out: the widest plan whose tile of R = 4 rows, with the static 128 bytes, fits 227 KB
ENC_F64_WIDTH_LIMIT = 980


def test_encode_launch_restatement_pins_the_width_limit_and_the_minimum_tile():
    R, smem, _ = _enc_launch(10 ** 6, 8 * ENC_F64_WIDTH_LIMIT, ENC_F64_WIDTH_LIMIT, 8, 0)
    assert R == 4 and smem + ENC_STATIC_SMEM <= 227 * 1024
    assert _enc_launch(10 ** 6, 8 * (ENC_F64_WIDTH_LIMIT + 1), ENC_F64_WIDTH_LIMIT + 1, 8, 0)[1] + ENC_STATIC_SMEM > 227 * 1024
    schema, _, plan = _wide_case()
    assert schema.row_bytes >= 2000 and _enc_launch(10 ** 6, schema.row_bytes, plan.n_out, 8, len(plan.lut_array()))[0] == 4


# ------------------------------------------------------------------------------- records and plans
F32_EDGES = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1e-45, 1e-40, 1.0 + 2.0 ** -23, 16777216.0, 3.4028235e38, -2.5],
                     np.float32)
# 1 + 2^-24 and 16777217 sit exactly halfway between two floats (round to even), 1 + 2^-24 + 2^-52 just above;
# 2^53 + 1 is not a double (it reads as 2^53), 2^53 + 2 is
F64_EDGES = np.array([np.nan, np.inf, -np.inf, -0.0, 5e-324, 1e-310, 2.0 ** 53 + 2.0, float(2 ** 53 + 1), 1.0 + 2.0 ** -24,
                      1.0 + 2.0 ** -24 + 2.0 ** -52, 16777217.0, 1e300, -1e-300, 0.1], np.float64)
I32_EDGES = np.array([-2 ** 31, 2 ** 31 - 1, 0, -1, 2 ** 24 + 1, -(2 ** 24 + 1)], np.int64)


def _records(schema, n, seed, code_sizes, edge_frac=0.05):
    """n random records of `schema` (numpy structured array): numbers over many magnitudes with edge values mixed in,
    dictionary codes in [-3, K + 3) (negative, unseen and >= the LUT length) plus a few huge ones."""
    rng = np.random.default_rng(seed)
    a = np.zeros(n, schema.numpy_dtype())
    for name, typ in zip(schema.names, schema.types):
        edge = rng.random(n) < edge_frac
        if typ == "code":
            v = rng.integers(-3, code_sizes[name] + 3, n)
            v[edge] = rng.choice(np.array([2 ** 31 - 1, -2 ** 31, 1 << 20]), int(edge.sum()))
        elif typ == "i32":
            v = np.where(rng.random(n) < 0.5, rng.integers(-1000, 1000, n), rng.integers(-2 ** 31, 2 ** 31, n))
            v[edge] = rng.choice(I32_EDGES, int(edge.sum()))
        else:
            v = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 6, n)).astype(np.float32 if typ == "f32" else np.float64)
            v[edge] = rng.choice(F32_EDGES if typ == "f32" else F64_EDGES, int(edge.sum()))
        a[name] = v
    return a


def _dev(a, schema):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(len(a), schema.row_bytes).copy()).to(DEV)


def _lut(K, rng, unseen=0.1):
    """StringIndexer LUT of a K-code dictionary: about `unseen` of the codes never occurred (rank -1)."""
    seen = rng.random(K) >= unseen
    lut = np.full(K, -1, np.int32)
    lut[seen] = rng.permutation(int(seen.sum()))
    return lut


class _Plan:
    """EncodePlan builder that registers ONE LUT per categorical field, so that several slots share a source (encode_kernel
    de-duplicates sources on field offset + LUT offset + LUT length).  scaled: every slot gets a (mean, scale), among them
    identity, zero and negative scales."""

    def __init__(self, schema, seed, code_sizes, scaled=False):
        self.schema, self.sizes, self.scaled = schema, code_sizes, scaled
        self.p = enc.EncodePlan(schema)
        self.rng = np.random.default_rng(seed)
        self.src = {}

    def _ms(self):
        if not self.scaled:
            return 0.0, 1.0
        r = self.rng
        return float(r.choice([0.0, r.normal() * 3.0, 1e9])), float(r.choice([1.0, 0.0, -2.5, 1.0 / r.uniform(0.1, 10.0)]))

    def source(self, field):
        if field not in self.src:
            lut = _lut(self.sizes[field], self.rng)
            off, ln = self.p._add_lut(lut)
            self.src[field] = (off, ln, int((lut >= 0).sum()))
        return self.src[field]

    def num(self, field):
        self.p.add_numeric(field, *self._ms())
        return self

    def index(self, field):
        off, ln, _ = self.source(field)
        self.p.slots.append((SRC_INDEX, self.schema.offsets[field], off, ln, 0) + self._ms())
        return self

    def onehot(self, field, width=None):
        off, ln, nr = self.source(field)
        for k in range(nr if width is None else width):
            self.p.slots.append((SRC_ONEHOT, self.schema.offsets[field], off, ln, k) + self._ms())
        return self

    def label(self, field):
        self.p.set_label(field, _lut(self.sizes[field], self.rng))
        return self


def _mixed_schema(n_codes):
    """two (f32, f64, i32) triples — the f64 fields sit at offsets 4 and 20, = 4 (mod 8) — then n_codes code fields and a
    code label."""
    fields = []
    for j in range(2):
        fields += [("x%d" % j, "f32"), ("d%d" % j, "f64"), ("i%d" % j, "i32")]
    fields += [("c%d" % i, "code") for i in range(n_codes)] + [("lab", "code")]
    schema = enc.RecordSchema(fields)
    assert schema.offsets["d0"] % 8 == 4 and schema.offsets["d1"] % 8 == 4
    return schema


_SWEEP_SIZES = {"c0": 40, "c1": 12, "c2": 300, "c3": 7, "lab": 9}


def _sweep_plan(n_out, seed, scaled=False, label=True):
    """n_out slots cycling through numeric, INDEX and ONEHOT slots of four sources; c0 feeds an INDEX slot and a ONEHOT
    block.  The last one-hot block is cut to land on n_out exactly."""
    schema = _mixed_schema(4)
    b = _Plan(schema, seed, _SWEEP_SIZES, scaled)
    cycle = [("num", "x0"), ("index", "c0"), ("num", "d0"), ("onehot", "c1"), ("num", "i0"), ("index", "c2"),
             ("onehot", "c0"), ("num", "d1"), ("onehot", "c3"), ("num", "x1"), ("num", "i1")]
    k = 0
    while b.p.n_out < n_out:
        kind, f = cycle[k % len(cycle)]
        k += 1
        if kind == "onehot":
            b.onehot(f, width=min(n_out - b.p.n_out, b.source(f)[2]))
        else:
            getattr(b, kind)(f)
    if label:
        b.label("lab")
    assert b.p.n_out == n_out
    return schema, b.p


def _wide_case():
    """about 2 KB per record: 500 f32 fields, two f64 fields at offsets = 4 (mod 8), a code and a label — R is 4."""
    fields = [("w%d" % i, "f32") for i in range(500)] + [("q", "i32"), ("a", "f64"), ("b", "f64"), ("c0", "code"),
                                                           ("lab", "code")]
    schema = enc.RecordSchema(fields)
    assert schema.offsets["a"] % 8 == 4 and schema.offsets["b"] % 8 == 4
    sizes = {"c0": 30, "lab": 5}
    b = _Plan(schema, 3, sizes)
    for i in range(0, 500, 25):
        b.num("w%d" % i)
    b.num("a").index("c0").num("b").onehot("c0", 10).num("q").label("lab")
    return schema, sizes, b.p


def _same_bits(got, want, what=""):
    """bit-for-bit equality; NaNs are compared by position only (the identity f32 path moves their bits unchanged)."""
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, want.shape, got.dtype, want.dtype)
    ng, nw = np.isnan(got), np.isnan(want)
    assert np.array_equal(ng, nw), "%s: NaN positions differ" % what
    ui = np.uint32 if got.dtype == np.float32 else np.uint64
    g, w = np.where(ng, got.dtype.type(0), got), np.where(nw, want.dtype.type(0), want)
    diff = np.argwhere(g.view(ui) != w.view(ui))
    assert diff.size == 0, "%s: %d values differ, first at %s: got %r, want %r" % (
        what, len(diff), tuple(diff[0]), got[tuple(diff[0])], want[tuple(diff[0])])


def _check_encode(plan, a, out_dtype, check_nan, rec=None):
    plan.check_nan = check_nan
    rec = _dev(a, plan.schema) if rec is None else rec
    got, lab, valid = plan.run(rec, out_dtype)
    want, want_lab, want_valid = oracle_encode(plan, np.ascontiguousarray(a).view(np.uint8))
    what = "n=%d n_out=%d %s check_nan=%d" % (len(a), plan.n_out, out_dtype, check_nan)
    _same_bits(got.cpu().numpy(), want if out_dtype == torch.float64 else want.astype(np.float32), what)
    assert np.array_equal(valid.cpu().numpy(), want_valid), what
    if plan.label is not None:
        assert np.array_equal(lab.cpu().numpy(), want_lab), what
    else:
        assert lab is None


# ------------------------------------------------------------------------------- encode_kernel
@pytest.mark.gpu
@pytest.mark.parametrize("n_out", [1, 255, 256, 257, 1000, 1100])
def test_encode_slot_mappings_match_oracle(n_out):
    # <= 256: one fixed slot per thread (rp = 256 / n_out rows per slot); above: threads stride over the slots;
    # above 1024: no slot de-duplication (every categorical slot looks its code up inline)
    schema, plan = _sweep_plan(n_out, seed=n_out)
    a = _records(schema, 1501, seed=100 + n_out, code_sizes=_SWEEP_SIZES)
    for dt in (torch.float32, torch.float64):
        _check_encode(plan, a, dt, check_nan=1)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["blocks", "plain_index"])
@pytest.mark.parametrize("n_src", [1, 8, 9, 12])
def test_encode_categorical_sources_shared_and_inline(n_src, layout):
    # blocks: one-hot blocks (>= 3 slots per source) use the shared rank pre-pass for the first kEncMaxCat = 8 sources and
    # inline lookups beyond; every third source also feeds an INDEX slot.  plain_index: one INDEX slot per source, so
    # n_cat_slots < 3 * nc and every lookup falls back to inline.
    schema = _mixed_schema(12)
    sizes = dict({"c%d" % i: 4 + 3 * i for i in range(12)}, lab=6)
    b = _Plan(schema, n_src, sizes)
    for i in range(n_src):
        b.num(["x0", "d0", "i0", "x1", "d1", "i1"][i % 6])
        if layout == "blocks":
            b.onehot("c%d" % i)
            if i % 3 == 0:
                b.index("c%d" % i)
        else:
            b.index("c%d" % i)
    b.label("lab")
    a = _records(schema, 2003, seed=7 * n_src, code_sizes=sizes)
    for dt in (torch.float32, torch.float64):
        for cn in (0, 1):
            _check_encode(b.p, a, dt, cn)


@pytest.mark.gpu
def test_encode_lut_pool_in_global_memory():
    # a 5000-code dictionary: the pool exceeds 4096 entries and stays in global memory (lut_in_smem = 0)
    schema = _mixed_schema(3)
    sizes = {"c0": 5000, "c1": 9, "c2": 300, "lab": 7}
    b = _Plan(schema, 11, sizes)
    b.index("c0").num("d0").onehot("c1").index("c2").onehot("c0", 20).num("x1").label("lab")
    assert len(b.p.lut_array()) > 4096
    a = _records(schema, 3001, seed=12, code_sizes=sizes)
    assert (a["c0"] < 0).any() and (a["c0"] >= 5000).any()
    for dt in (torch.float32, torch.float64):
        _check_encode(b.p, a, dt, check_nan=1)


@pytest.mark.gpu
@pytest.mark.parametrize("n_out", [40, 300])
@pytest.mark.parametrize("check_nan", [0, 1])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.float64])
def test_encode_scaled_slots_and_unaligned_f64(n_out, check_nan, out_dtype):
    # every slot kind with a (mean, scale): the INDEX / ONEHOT hot and cold constants, scaled I32, F32 and F64 fields
    # (the F64 ones at offsets = 4 (mod 8) holding NaN, +-inf, -0.0, subnormals and 2^53 + 2)
    schema, plan = _sweep_plan(n_out, seed=5 + n_out, scaled=True)
    kinds = {s[0] for s in plan.slots}
    assert kinds == {0, 1, 2, 3, 4} and any(s[5] != 0.0 or s[6] != 1.0 for s in plan.slots)
    a = _records(schema, 2500, seed=n_out, code_sizes=_SWEEP_SIZES, edge_frac=0.2)
    _check_encode(plan, a, out_dtype, check_nan)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["label_only", "no_label"])
def test_encode_label_only_and_unlabelled_plans(case):
    schema = _mixed_schema(1)
    sizes = {"c0": 5, "lab": 9}
    b = _Plan(schema, 17, sizes)
    b.num("x0").num("d0").num("i0").num("d1")
    if case == "label_only":
        b.label("lab")                                       # the label is the only categorical source (ncat = 0)
    a = _records(schema, 777, seed=18, code_sizes=sizes)
    assert case == "no_label" or ((a["lab"] < 0) | (a["lab"] >= 9)).any()     # unseen label codes
    for dt in (torch.float32, torch.float64):
        _check_encode(b.p, a, dt, check_nan=1)


def _row_count_case(kind):
    if kind == "mixed":
        schema, plan = _sweep_plan(40, seed=21)
        return schema, _SWEEP_SIZES, plan, torch.float32
    schema, sizes, plan = _wide_case()
    return schema, sizes, plan, torch.float64


def _straddling_rows(schema, plan, dt, which, stages=3):
    R, _, grid = _enc_launch(10 ** 8, schema.row_bytes, plan.n_out, 4 if dt == torch.float32 else 8,
                             len(plan.lut_array()), stages)
    return R, {"R-1": R - 1, "R": R, "R+1": R + 1,
               "ring-1": (grid * stages - 1) * R + 3, "ring+1": (grid * stages + 1) * R + 3}[which]


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["R-1", "R", "R+1", "ring-1", "ring+1"])
@pytest.mark.parametrize("kind", ["mixed", "wide"])
def test_encode_row_counts_straddling_the_tile_and_the_ring(kind, which):
    # one ragged tile around R, and the load ring wrapping (grid * stages tiles) with a ragged last tile of 3 rows
    schema, sizes, plan, dt = _row_count_case(kind)
    R, n = _straddling_rows(schema, plan, dt, which)
    assert (kind == "wide") == (R == 4)
    a = _records(schema, n, seed=n, code_sizes=sizes)
    _check_encode(plan, a, dt, check_nan=1)


def _knob_cases():
    """(name, plan, records, out dtype) run by a child process under B200FLOW_ENC_STAGES=2, B200FLOW_ENC_SMEM_KB=12.
    With a 12 KB budget the 300-slot plan has no room left (R falls back to 4), the others get small tiles."""
    out = []
    schema, plan = _sweep_plan(40, seed=31)
    R, _, grid = _enc_launch(10 ** 8, schema.row_bytes, plan.n_out, 4, len(plan.lut_array()), stages=2, budget_kb=12)
    for n in (R - 1, (grid * 2 - 1) * R + 3, (grid * 2 + 1) * R + 3):
        out.append(("mixed_%d" % n, plan, _records(schema, n, seed=n, code_sizes=_SWEEP_SIZES), torch.float32))
    schema, plan = _sweep_plan(300, seed=32, scaled=True)
    assert _enc_launch(10 ** 8, schema.row_bytes, 300, 8, len(plan.lut_array()), stages=2, budget_kb=12)[0] == 4
    out.append(("scaled_300", plan, _records(schema, 4099, seed=33, code_sizes=_SWEEP_SIZES), torch.float64))
    schema, sizes, plan = _wide_case()
    out.append(("wide", plan, _records(schema, 1203, seed=34, code_sizes=sizes), torch.float64))
    for _, p, _, _ in out:
        p.check_nan = 1
    return out


_KNOB_CHILD = r"""
import sys
sys.path[:0] = [%r, %r, %r]
import numpy as np, torch
import test_encode_edges as t
res = {}
for name, plan, a, dt in t._knob_cases():
    x, lab, valid = plan.run(t._dev(a, plan.schema), dt)
    res[name + "/x"] = x.cpu().numpy(); res[name + "/lab"] = lab.cpu().numpy(); res[name + "/valid"] = valid.cpu().numpy()
torch.cuda.synchronize()
np.savez(sys.argv[1], **res)
"""


@pytest.mark.gpu
def test_encode_two_stage_ring_and_small_budget(tmp_path):
    # both knobs are read once per process (static locals in b200flow_encode), so they run in a child of their own
    env = dict(os.environ, B200FLOW_ENC_STAGES="2", B200FLOW_ENC_SMEM_KB="12")
    dst = str(tmp_path / "knobs.npz")
    subprocess.run([sys.executable, "-c", _KNOB_CHILD % (ROOT, PKG, TESTS), dst], env=env, timeout=600, check=True)
    got = np.load(dst)
    for name, plan, a, dt in _knob_cases():
        want, want_lab, want_valid = oracle_encode(plan, a.view(np.uint8))
        _same_bits(got[name + "/x"], want if dt == torch.float64 else want.astype(np.float32), name)
        assert np.array_equal(got[name + "/lab"], want_lab) and np.array_equal(got[name + "/valid"], want_valid), name


@pytest.mark.gpu
def test_encode_width_limit():
    # f64 records in, f64 vector out: ENC_F64_WIDTH_LIMIT slots run; one more is refused before any launch
    for D in (ENC_F64_WIDTH_LIMIT, ENC_F64_WIDTH_LIMIT + 1):
        schema = enc.RecordSchema([("v%d" % i, "f64") for i in range(D)])
        plan = enc.EncodePlan(schema)
        for i in range(D):
            plan.add_numeric("v%d" % i)
        a = _records(schema, 37, seed=D, code_sizes={})
        if D == ENC_F64_WIDTH_LIMIT:
            _check_encode(plan, a, torch.float64, check_nan=1)
            continue
        out = torch.full((37, D), 7.0, dtype=torch.float64, device=DEV)
        with pytest.raises(_lib.B200FlowError, match=r"record too wide.*row_bytes=%d n_out=%d" % (8 * D, D)):
            plan.run(_dev(a, schema), torch.float64, out=out)
        torch.cuda.synchronize()                             # no CUDA error is left pending either
        assert bool((out == 7.0).all())                      # nothing was launched


# ------------------------------------------------------------------------------- encode -> bins, findSplits sample
def _field(a, schema, off, kind):
    raw = np.ascontiguousarray(a).view(np.uint8).reshape(len(a), schema.row_bytes)
    w = 8 if kind == SRC_F64 else 4
    return raw[:, off:off + w].copy().view(np.float64 if kind == SRC_F64 else np.float32 if kind == SRC_F32 else np.int32)[:, 0]


def _expected_bad(plan, a, x, arity):
    """(bad[0], bad[1]) of encode_bins: categorical cells that are non-integral or outside [0, arity); NaN cells of f32 / f64
    slots (with check_nan) + INDEX / ONEHOT cells whose code has no rank + labels without a rank."""
    cat = arity > 0
    xv = x[:, cat]
    bad0 = int((~((xv == np.floor(xv)) & (xv >= 0) & (xv < arity[cat]))).sum())
    lut = plan.lut_array()

    def no_rank(off, lo, ln):
        codes = _field(a, plan.schema, off, None)
        inside = (codes >= 0) & (codes < ln)
        return int((~inside | (lut[lo + np.clip(codes, 0, ln - 1)] < 0)).sum())
    bad1 = 0
    for kind, off, lo, ln, _, _, _ in plan.slots:
        if kind in (SRC_F32, SRC_F64):
            bad1 += int(np.isnan(_field(a, plan.schema, off, kind)).sum()) if plan.check_nan else 0
        elif kind >= SRC_INDEX:
            bad1 += no_rank(off, lo, ln)
    if plan.label is not None:
        bad1 += no_rank(*plan.label)
    return bad0, bad1


def _bins_case(name):
    """-> (schema, records, plan, arity, maxBins, round_f32)"""
    if name.startswith("cicids_f64"):                       # CICIDS-shaped: 78 f64 fields + the label, one constant column
        schema = enc.RecordSchema([("f%d" % i, "f64") for i in range(78)] + [("Label", "code")])
        sizes = {"Label": 15}
        a = _records(schema, 20000, seed=41, code_sizes=sizes, edge_frac=0.01)
        a["f5"] = 3.25
        b = _Plan(schema, 42, sizes)
        for i in range(78):
            b.num("f%d" % i)
        b.label("Label")
        b.p.check_nan = 1
        return schema, a, b.p, np.zeros(78, np.int32), int(name.split("_")[-1]), 0
    if name.startswith("int_index") or name == "maxbins_2":  # I32 and INDEX numbers as continuous features
        schema = _mixed_schema(2)
        sizes = {"c0": 300, "c1": 20, "lab": 6}
        a = _records(schema, 6000, seed=43, code_sizes=sizes)
        b = _Plan(schema, 44, sizes)
        b.num("i0").index("c0").index("c1").num("d0")
        b.p.add_numeric("x1", 0.5, -3.0).add_numeric("i1", 3.5, 1.0 / 7.0)      # scaled f32 and i32 slots
        b.label("lab")
        arity = np.array([0, 0, b.src["c1"][2], 0, 0, 0], np.int32)
        return schema, a, b.p, arity, 2 if name == "maxbins_2" else 32, int(name == "int_index_rf32")
    if name == "f32_index":                                  # unscaled f32 / INDEX / ONEHOT: the float table, no round_f32
        schema = _mixed_schema(2)
        sizes = {"c0": 300, "c1": 5, "lab": 6}
        a = _records(schema, 5000, seed=45, code_sizes=sizes)
        b = _Plan(schema, 46, sizes)
        b.num("x0").index("c0").onehot("c1").num("x1").label("lab")
        arity = np.array([0, 0] + [2] * b.src["c1"][2] + [0], np.int32)
        return schema, a, b.p, arity, 64, 0
    F = int(name[1:])
    if F == 1:                                               # one f32 feature, no label
        schema = enc.RecordSchema([("x0", "f32")])
        a = _records(schema, 4099, seed=47, code_sizes={})
        plan = enc.EncodePlan(schema).add_numeric("x0")
        plan.check_nan = 1
        return schema, a, plan, np.zeros(1, np.int32), 32, 0
    # F = 15 or 47: numbers, categorical i32 fields of arity 254, 255, 256 (values in [-2, arity + 3)), an f64 field of
    # arity 10 holding half-integers, and (F = 47) a 5000-code dictionary: the LUT pool in global memory
    fields = [("x%d" % i, "f32") for i in range(F - 8)] + [("d0", "f64"), ("k254", "i32"), ("k255", "i32"),
                                                           ("k256", "i32"), ("h10", "f64"), ("i0", "i32"),
                                                           ("c0", "code"), ("c1", "code"), ("lab", "code")]
    schema = enc.RecordSchema(fields)
    sizes = {"c0": 5000 if F == 47 else 50, "c1": 12, "lab": 7}
    a = _records(schema, 7001, seed=F, code_sizes=sizes, edge_frac=0.02)
    rng = np.random.default_rng(F + 1)
    for k in (254, 255, 256):
        a["k%d" % k] = rng.integers(-2, k + 3, len(a))
    a["h10"] = rng.integers(-1, 12, len(a)) + 0.5 * (rng.random(len(a)) < 0.1)
    b = _Plan(schema, F + 2, sizes)
    for i in range(F - 8):
        b.num("x%d" % i)
    b.num("d0").num("k254").num("k255").num("k256").num("h10").num("i0").index("c0").index("c1").label("lab")
    b.p.check_nan = 1
    arity = np.array([0] * (F - 8) + [0, 254, 255, 256, 10, 0, 0, b.src["c1"][2]], np.int32)
    return schema, a, b.p, arity, 256, 0


BINS_CASES = ["cicids_f64_128", "cicids_f64_256", "int_index", "int_index_rf32", "f32_index", "maxbins_2", "F1", "F15", "F47"]


def _encoded(plan, a, round_f32):
    x, y, _ = oracle_encode(plan, a.view(np.uint8))
    return (x.astype(np.float32).astype(np.float64) if round_f32 else x), y


@pytest.mark.gpu
@pytest.mark.parametrize("name", BINS_CASES)
def test_encode_bins_edges_match_oracle(name):
    schema, a, plan, arity, mb, rf32 = _bins_case(name)
    F = plan.n_out
    assert len(arity) == F
    x, y = _encoded(plan, a, rf32)
    thr, n_thr, _ = oracle.find_splits(np.where(np.isnan(x), 0.0, x), 7, 1 << 32, arity, mb)
    if name.startswith("cicids"):
        assert (n_thr > mb // 2).sum() >= 70 and n_thr[5] == 0          # long tables, and the constant column
        assert (F * (mb - 1) + 256) * 8 > 56 * 1024                       # the fp64 table stays in global memory
    tp_o, _ = oracle.bin_rows(x, thr, n_thr, arity, mb, y if plan.label is not None else None)
    src = fr._RecordSource(_dev(a, schema), plan, round_f32=bool(rf32))
    bad = torch.zeros(2, dtype=torch.int32, device=DEV)
    tp, lab = src.bin(_lib.h2d(thr, DEV), _lib.h2d(n_thr, DEV), _lib.h2d(arity, DEV), mb, bad, want_label_out=True)
    tp = tp.cpu().numpy()
    assert tp.shape[0] == len(a) and tp.shape[1] >= F + 1 and tp.shape[1] % 16 == 0
    diff = np.argwhere(tp[:, :F + 1] != tp_o[:, :F + 1])
    assert diff.size == 0, "%d bins differ, first (row, feature) %s" % (len(diff), tuple(diff[0]))
    assert not tp[:, F + 1:].any()
    assert tuple(bad.cpu().tolist()) == _expected_bad(plan, a, x, arity)
    if plan.label is not None:
        assert np.array_equal(lab.cpu().numpy(), y)


@pytest.mark.gpu
@pytest.mark.parametrize("name,rf32,row_offset", [("int_index", 0, 0), ("int_index_rf32", 1, 2 ** 32 - 1500),
                                                  ("F47", 0, 123457)])
def test_sample_records_is_the_oracle_sample(name, rf32, row_offset):
    # the findSplits sample: rows whose first Philox word (keyed by the GLOBAL row) is below keep_threshold, encoded
    # through the plan; slot order comes from an atomic, so each column is compared as a multiset
    schema, a, plan, _, _, _ = _bins_case(name)
    n, F = len(a), plan.n_out
    seed, keep = 0x5EED, int(0.37 * 2 ** 32)
    rows = [i for i in range(n) if int(oracle.philox(seed, oracle.PURPOSE_SAMPLE, (row_offset + i) & 0xFFFFFFFF,
                                                     (row_offset + i) >> 32)[0]) < keep]
    x, _ = _encoded(plan, a, rf32)
    src = fr._RecordSource(_dev(a, schema), plan, round_f32=bool(rf32))
    cap = n
    sample = torch.full((F * cap,), -7.0, dtype=torch.float64, device=DEV)
    n_s = torch.zeros(1, dtype=torch.int32, device=DEV)
    src.sample(seed, keep, row_offset, sample, cap, n_s)
    assert int(n_s.item()) == len(rows)
    s = sample.view(F, cap).cpu().numpy()
    for f in range(F):
        assert np.array_equal(np.sort(s[f, :len(rows)]), np.sort(x[rows, f]), equal_nan=True), f
    assert (s[:, len(rows):] == -7.0).all()


# ------------------------------------------------------------------------------- StandardScaler.fit: column moments
def _moments_data(n, D, seed):
    """columns of 1e9 + N(0, 1) (the case a one-pass variance gets wrong), constant 0.1 and 1/3, and N(0, 1) at assorted
    scales."""
    rng = np.random.default_rng(seed)
    x = np.empty((n, D))
    for d in range(D):
        k = d % 4
        x[:, d] = (1e9 + rng.standard_normal(n) if k == 0 else np.full(n, 0.1) if k == 1 else np.full(n, 1.0 / 3.0)
                   if k == 2 else rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4))
    return x


MOMENT_SHAPES = [(1, 257), (2, 256), (3, 255), (4097, 600), (4097, 1), (10 ** 6, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,D", MOMENT_SHAPES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_column_moments_within_summation_bounds(n, D, dtype):
    x = torch.from_numpy(_moments_data(n, D, seed=n + D)).to(dtype)
    xh = x.to(torch.float64).numpy()                       # the values the kernel reads, exactly
    mean, std = enc.column_moments(x.to(DEV))
    mean, std = mean.cpu().numpy(), std.cpu().numpy()
    for d in range(D):
        col = xh[:, d]
        mu = math.fsum(col) / n                             # correctly rounded sum: off by at most 2u|mu|
        mean_abs = math.fsum(np.abs(col)) / n
        # mean: the sum of n values in any order is within gamma_(n-1) * sum|x| of the exact sum; the division adds
        # u|mu|; the reference adds 2u|mu|  ->  gamma_(n+2) * mean|x|
        tol_mean = _gamma(n + 2) * mean_abs
        assert abs(mean[d] - mu) <= tol_mean, (d, mean[d], mu, tol_mean)
        if (col == col[0]).all():
            assert std[d] == 0.0, (d, std[d])               # a constant column has std exactly 0
            continue
        dev = col - mu
        q = math.fsum(dev * dev) + n * tol_mean ** 2       # >= sum (x - mean_gpu)^2, the squares the second pass sums
        var = (math.fsum(dev * dev) - math.fsum(dev) ** 2 / n) / (n - 1)
        # second pass: each shifted square carries 3 roundings and the sum gamma_(n-1); the correction s^2/n is bounded
        # by the same q (Cauchy-Schwarz) and its error by 2 gamma_n q; the reference's own error is 3u q  ->  4 gamma_(n+4) q
        tol_var = 4 * _gamma(n + 4) * q / (n - 1) + U * var
        # |sqrt(a) - sqrt(b)| <= |a - b| / sqrt(b), plus the rounding of the sqrt and of the division
        tol_std = tol_var / math.sqrt(var) + 2 * U * math.sqrt(var)
        assert abs(std[d] - math.sqrt(var)) <= tol_std, (d, std[d], math.sqrt(var), tol_std)


@pytest.mark.gpu
@pytest.mark.parametrize("n,D", [(3, 255), (4097, 257), (4097, 600)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("shifted", [False, True])
def test_column_moments_c_abi_with_row_pitch(n, D, dtype, shifted):
    # ld > D: the columns past D are NaN and must never be read
    ld = D + 5
    xh = _moments_data(n, D, seed=D).astype(np.float32 if dtype == torch.float32 else np.float64)
    buf = torch.full((n, ld), float("nan"), dtype=dtype)
    buf[:, :D] = torch.from_numpy(xh)
    buf = buf.to(DEV)
    shift = xh.astype(np.float64)[0] + 0.5 if shifted else None
    s = torch.zeros(D, dtype=torch.float64, device=DEV)
    q = torch.zeros(D, dtype=torch.float64, device=DEV)
    _lib.call("b200flow_column_moments", ptr(buf), _lib.dtype_code(buf), n, D, ld,
              ptr(_lib.h2d(shift, DEV) if shifted else None), ptr(s), ptr(q))
    s, q = s.cpu().numpy(), q.cpu().numpy()
    for d in range(D):
        v = xh[:, d].astype(np.float64) - (shift[d] if shifted else 0.0)     # the shifted values, rounded as the kernel does
        # n values summed in any order: within gamma_(n-1) sum|v| (resp. sum v^2, the squares being rounded alike);
        # the correctly rounded reference adds u|sum|
        assert abs(s[d] - math.fsum(v)) <= _gamma(n) * math.fsum(np.abs(v)), d
        assert abs(q[d] - math.fsum(v * v)) <= _gamma(n) * math.fsum(v * v), d


@pytest.mark.gpu
@pytest.mark.parametrize("with_mean,with_std", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("branch,D", [("plan", 40), ("dense", 40), ("dense", 300)])
def test_standard_scaler_transform_is_numpy_bit_for_bit(branch, D, with_mean, with_std):
    # "plan": the scaler fuses into the VectorAssembler's encode plan over the raw records; "dense": a vector without
    # record provenance goes through a dense f64 plan (D = 300: threads stride over the slots)
    from pyspark.ml.feature import StandardScaler, VectorAssembler
    from pyspark.sql import ColumnData, DataFrame
    n = 3001
    xh = _moments_data(n, D, seed=D)
    if branch == "plan":
        schema = enc.RecordSchema([("v%d" % i, "f32" if i % 5 == 3 else "f64") for i in range(D)])
        a = np.zeros(n, schema.numpy_dtype())
        for i in range(D):
            a["v%d" % i] = xh[:, i]
        df = VectorAssembler(inputCols=schema.names, outputCol="v").transform(DataFrame.fromRecords(_dev(a, schema), schema, {}))
    else:
        df = DataFrame(n, None, None, {}, {"v": ColumnData("vector", torch.from_numpy(xh).to(DEV), "f64")})
    model = StandardScaler(inputCol="v", outputCol="s", withMean=with_mean, withStd=with_std).fit(df)
    out = model.transform(df)
    assert (out._cols["s"].prov is not None and out._cols["s"].prov[0] == "plan") == (branch == "plan")
    x = out._cols["v"].data.to(torch.float64).cpu().numpy()
    assert (model.std[1::4] == 0.0).all() and (model.std[2::4] == 0.0).all()
    mean = model.mean if with_mean else np.zeros(D)
    scale = np.where(model.std != 0, 1.0 / np.where(model.std != 0, model.std, 1.0), 0.0) if with_std else np.ones(D)
    got = out._cols["s"].data.cpu().numpy()
    _same_bits(got, (x - mean) * scale, "StandardScaler(%s, %s)" % (with_mean, with_std))
    if with_std:
        assert (got[:, 1::4] == 0.0).all() and (got[:, 2::4] == 0.0).all()  # constant columns scale to exactly 0


# ------------------------------------------------------------------------------- categorical values a model never saw
def _mllib_leaves(ex, thresholds, arity, x):
    """the leaf each row of x reaches, walking the exported tree 0 with MLlib's Node.predictImpl on the RAW values:
    ContinuousSplit goes left iff value <= threshold; CategoricalSplit (Split.scala) keeps the smaller side,
    isLeft = |leftCategories| <= numCategories / 2, and shouldGoLeft is `value in leftCategories` when isLeft, else
    `value not in rightCategories`."""
    at = {int(nid): i for i, (t, nid) in enumerate(zip(ex["tree"], ex["nid"])) if t == 0}
    leaves = []
    for row in x:
        nid = 1
        while not ex["is_leaf"][at[nid]]:
            i = at[nid]
            f = int(ex["feat"][i])
            v = float(row[f])
            if arity[f] == 0:
                left = v <= thresholds[f, ex["bin_thr"][i]]
            else:
                cats = {c for c in range(arity[f]) if (int(ex["mask"][i][c >> 6]) >> (c & 63)) & 1}
                left = (v in cats) if len(cats) <= arity[f] // 2 else (v not in set(range(arity[f])) - cats)
            nid = 2 * nid + (0 if left else 1)
        leaves.append(at[nid])
    return leaves


def _routing_data(A):
    """8 rows per category of feature 0 (arity A), feature 1 alternating 0 / 1.  The label is 1 below category A - 56;
    from A - 56 up it equals feature 1.  The root then splits feature 0 with left set {A - 56, ..., A - 1}, which holds
    the top category and is small enough (56 <= A / 2) that MLlib sends any unseen value right."""
    cat = np.repeat(np.arange(A), 8).astype(np.float64)
    f1 = np.tile([0.0, 1.0], 4 * A)
    y = np.where(cat < A - 56, 1, f1 > 0.5).astype(np.int32)
    return np.stack([cat, f1], 1), y


def _routing_fit(A):
    x, y = _routing_data(A)
    p = fr.ForestParams(num_trees=1, max_bins=256, max_depth=2, bootstrap=False, seed=1)
    return fr.fit_forest(torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV), 2, [A, 0], p)


@pytest.mark.gpu
def test_unseen_categories_route_right_at_every_split():
    # arity 255: the out-of-range bin 255 is no category, so a value the fit never saw must take MLlib's route at every
    # split, through the dense (bin_rows) and the record (encode_bins) paths.  (With arity 256, which build_metadata now
    # refuses, bin 255 is category 255: these values followed it into the left set and predicted 0 instead of 1.)
    A = 255
    model = _routing_fit(A)
    ex = model.export()
    root = np.flatnonzero((ex["tree"] == 0) & (ex["nid"] == 1))[0]
    left = [c for c in range(256) if (int(ex["mask"][root][c >> 6]) >> (c & 63)) & 1]
    assert ex["feat"][root] == 0 and A - 1 in left and len(left) <= A // 2
    tests = np.array([[v, f1] for v in (300.0, 1.5, -1.0, float(A), 256.0, 1e6, A - 1.0, A - 56.0, 0.0, 7.0)
                      for f1 in (0.0, 1.0)])
    leaves = _mllib_leaves(ex, model.thresholds.cpu().numpy(), [A, 0], tests)
    want = np.array([float(np.argmax(ex["counts"][i])) for i in leaves])
    assert want[:12].tolist() == [1.0] * 12                 # unseen values: the pure right leaf
    _, _, pred = model.predict(torch.from_numpy(tests).to(DEV))
    assert np.array_equal(pred.cpu().numpy(), want)
    schema = enc.RecordSchema([("cat", "f64"), ("f1", "f32")])
    plan = enc.EncodePlan(schema).add_numeric("cat").add_numeric("f1")
    a = np.zeros(len(tests), schema.numpy_dtype())
    a["cat"], a["f1"] = tests[:, 0], tests[:, 1]
    _, _, pred_r, _ = model.predict_records(_dev(a, schema), plan)
    assert np.array_equal(pred_r.cpu().numpy(), want)


@pytest.mark.gpu
def test_256_category_feature_is_refused_on_every_fit_path():
    # with 256 categories every uint8 bin is a category and an unseen value would follow category 255
    x, y = _routing_data(256)
    p = fr.ForestParams(num_trees=1, max_bins=256, max_depth=2, bootstrap=False, seed=1)
    with pytest.raises(_lib.UnsupportedParamError, match="256"):
        fr.fit_forest(torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV), 2, [256, 0], p)
    schema = enc.RecordSchema([("cat", "f64"), ("f1", "f32"), ("y", "code")])
    a = np.zeros(len(x), schema.numpy_dtype())
    a["cat"], a["f1"], a["y"] = x[:, 0], x[:, 1], y
    plan = enc.EncodePlan(schema).add_numeric("cat").add_numeric("f1").set_label("y", np.arange(2, dtype=np.int32))
    with pytest.raises(_lib.UnsupportedParamError, match="256"):
        fr.fit_forest_records(_dev(a, schema), plan, 2, [256, 0], p)
    # the pyspark shim: StringIndexer makes the 256-value nominal attribute, DecisionTreeClassifier reports the refusal
    from pyspark.ml.classification import DecisionTreeClassifier
    from pyspark.ml.feature import IllegalArgumentException, StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    cs = enc.RecordSchema([("cat", "code"), ("y", "code")])
    c = np.zeros(len(x), cs.numpy_dtype())
    c["cat"], c["y"] = x[:, 0].astype(np.int32), y
    df = DataFrame.fromRecords(_dev(c, cs), cs, {"cat": ["v%03d" % i for i in range(256)], "y": ["n", "p"]})
    df = StringIndexer(inputCol="cat", outputCol="cat_idx").fit(df).transform(df)
    df = StringIndexer(inputCol="y", outputCol="label").fit(df).transform(df)
    df = VectorAssembler(inputCols=["cat_idx"], outputCol="features").transform(df)
    with pytest.raises(IllegalArgumentException, match="256"):
        DecisionTreeClassifier(maxBins=256, maxDepth=2).fit(df)


def test_build_metadata_refuses_a_256_category_feature():
    with pytest.raises(_lib.UnsupportedParamError, match="256 categories"):
        fr.build_metadata(10000, 3, 2, [0, 256, 3], 256, 1)
    assert isinstance(_lib.UnsupportedParamError("x"), ValueError)             # the shim reports it as IllegalArgumentException
    mpb, kind, m = fr.build_metadata(10000, 3, 2, [0, 255, 3], 256, 1)          # 255 categories leave bin 255 for unseen values
    assert mpb == 256 and kind.tolist() == [0, 1, 1] and m == 3
    with pytest.raises(ValueError, match="maxBins"):                             # MLlib's own check comes first
        fr.build_metadata(10000, 3, 2, [0, 256, 3], 128, 1)
