"""The device CSV reader's field grammar and decimal -> double conversion (csrc/csv_number.h), compiled for the HOST and checked
against Python's own correctly rounded float() / int() — the same semantics as Java's Double.parseDouble / Integer.parseInt that
Spark's CSV reader applies (kdd99.py:25, cicids17.py:19-20).  No GPU needed: the header is `__host__ __device__`."""
import ctypes as C

import numpy as np
import pytest

from csv_corpus import (DOUBLE, INT, LONG, NOT_A_NUMBER, NULL, OK, STRING, UNSUPPORTED, build_host_lib, grammar_literals, long_literals,
                        midpoint_literals, run, writer_literals)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("csvnum"))


def bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def test_classification_follows_spark_inference(lib):
    cases = {"": NULL, "0": INT, "-0": INT, "+17": INT, "007": INT, "2147483647": INT, "-2147483648": INT, "2147483648": LONG,
             "-2147483649": LONG, "9223372036854775807": LONG, "-9223372036854775808": LONG, "9223372036854775808": DOUBLE,
             "12345678901234567890123": DOUBLE, "1.0": DOUBLE, "1.": DOUBLE, ".5": DOUBLE, "-.5e-3": DOUBLE, "1e5": DOUBLE, "1E+5": DOUBLE,
             " 12": DOUBLE, "12 ": DOUBLE, "\t3.5 ": DOUBLE,             # toInt rejects blanks, toDouble trims them
             "NaN": DOUBLE, "Infinity": DOUBLE, "-Infinity": DOUBLE, "+Infinity": DOUBLE, "Inf": DOUBLE, "-Inf": DOUBLE,
             "nan": STRING, "inf": STRING, "infinity": STRING, ".": STRING, "-": STRING, "+": STRING, "e5": STRING, "1e": STRING, "1e+": STRING,
             "1.2.3": STRING, "1,2": STRING, "0x10": STRING, "1f": STRING, "tcp": STRING, "  ": STRING, "1 2": STRING, "--1": STRING, "BENIGN": STRING}
    cls, *_ = run(lib, list(cases))
    assert {k: int(c) for k, c in zip(cases, cls)} == cases


def test_doubles_are_correctly_rounded_fast_path_and_128_bit_path(lib):
    fields = writer_literals(np.random.default_rng(7))
    cls, st, val, _, _ = run(lib, fields)
    want = np.array([float(f) for f in fields])
    assert (cls[st == OK] != STRING).all()
    ok = st == OK
    assert ok.mean() > 0.995 and np.array_equal(bits(val[ok]), bits(want[ok]))     # bit-exact wherever the reader answers
    assert set(np.unique(st[~ok])) <= {UNSUPPORTED}


def test_more_than_19_digits_exact_or_reported(lib):
    fields = long_literals(np.random.default_rng(9))
    fields += ["0.1000000000000000055511151231257827021181583404541015625",        # 0.1's exact binary expansion
               "9007199254740993.0000000000000000000001", "9007199254740993.00000000000000000000", "1" + "0" * 25, "0." + "0" * 30 + "1"]
    cls, st, val, _, _ = run(lib, fields)
    want = np.array([float(f) for f in fields])
    ok = st == OK
    assert np.array_equal(bits(val[ok]), bits(want[ok])) and ok.mean() > 0.99
    assert set(np.unique(st[~ok])) <= {UNSUPPORTED}
    d = dict(zip(fields[-5:], st[-5:]))
    assert d["9007199254740993.0000000000000000000001"] == UNSUPPORTED             # just above a tie: w and w + 1 disagree
    assert d["9007199254740993.00000000000000000000"] == OK and d["1" + "0" * 25] == OK and d["0." + "0" * 30 + "1"] == UNSUPPORTED


def test_special_values_blanks_and_nulls(lib):
    fields = ["", "NaN", "Infinity", "-Infinity", "+Infinity", "Inf", "-Inf", " 1.5 ", "1e400", "1e-400", "abc", "1e28", "1e27"]
    cls, st, val, sti, iv = run(lib, fields)
    assert np.isnan(val[0]) and st[0] == OK and np.isnan(val[1]) and val[2] == np.inf and val[3] == -np.inf and val[4] == np.inf
    assert val[5] == np.inf and val[6] == -np.inf and val[7] == 1.5
    assert st[8] == UNSUPPORTED and st[9] == UNSUPPORTED and st[10] == NOT_A_NUMBER and st[11] == UNSUPPORTED and st[12] == OK and val[12] == 1e27


def test_int32_fields(lib):
    rng = np.random.default_rng(3)
    ints = [int(v) for v in rng.integers(-2 ** 31, 2 ** 31, 50000)] + [0, -0, 2 ** 31 - 1, -2 ** 31]
    fields = [str(v) for v in ints] + ["+5", "0005", "2147483648", "1.0", " 5", "", "-"]
    cls, st, val, sti, iv = run(lib, fields)
    n = len(ints)
    assert (sti[:n] == OK).all() and np.array_equal(iv[:n], np.array(ints, np.int64).astype(np.int32)) and (cls[:n] == INT).all()
    assert list(sti[n:]) == [OK, OK, NOT_A_NUMBER, NOT_A_NUMBER, NOT_A_NUMBER, NOT_A_NUMBER, NOT_A_NUMBER] and iv[n] == 5 and iv[n + 1] == 5


def test_hash_is_fnv1a_and_never_zero(lib):
    lib.csvnum_hash.restype = C.c_uint64
    def fnv(b):
        h = 1469598103934665603
        for c in b:
            h = ((h ^ c) * 1099511628211) & (2 ** 64 - 1)
        return h or 1
    for s in [b"", b"tcp", b"smurf.", b"BENIGN", b"DoS Hulk", bytes(range(256))]:
        assert lib.csvnum_hash(s, len(s)) == fnv(s)


def test_python_restatement_agrees_with_the_product_grammar(lib, tmp_path):
    """oracle/csv_ref.py (the checker of the GPU tests) and csv_number.h must classify and convert every field alike; pandas is
    the independent pin for the column types and values of a plain file."""
    from oracle import csv_ref
    rng = np.random.default_rng(11)
    fields = grammar_literals(rng)
    fields += ["", "NaN", "Infinity", "-Infinity", "+Infinity", "Inf", "-Inf", "+Inf", " 12", "12 ", "1e5", "0x10", "1_000", "١٢", "1d", "1f", "٣.٥"]
    cls, st, val, sti, iv = run(lib, fields)
    raw = [f.encode() for f in fields]
    want_cls = np.array([csv_ref.classify(f) for f in raw])
    assert np.array_equal(cls, want_cls), [(f, int(a), int(b)) for f, a, b in zip(fields, cls, want_cls) if a != b][:10]
    num = (want_cls == DOUBLE) | (want_cls == INT) | (want_cls == LONG) | (want_cls == NULL)
    want_val = np.array([csv_ref.to_double(f) if ok else 0.0 for f, ok in zip(raw, num)])
    ok = num & (st == OK)
    assert np.array_equal(bits(val[ok]), bits(want_val[ok])) and set(np.unique(st[num & ~ok])) <= {UNSUPPORTED}
    assert (st[~num] == NOT_A_NUMBER).all()
    pd = pytest.importorskip("pandas")
    p = str(tmp_path / "plain.csv")
    rows = ["%d,%s,%s,%s" % (rng.integers(-1000, 1000), repr(float(rng.standard_normal())), ["tcp", "udp", "icmp"][int(rng.integers(0, 3))],
                             rng.integers(0, 2 ** 40)) for _ in range(3000)]
    open(p, "w").write("\n".join(rows) + "\n")
    names, types, cols, dicts = csv_ref.read_csv([p], infer_schema=True)
    pdf = pd.read_csv(p, header=None, float_precision="round_trip")   # the default C parser is not correctly rounded
    assert types == ["i32", "f64", "code", "f64"]
    assert np.array_equal(cols["_c0"], pdf[0].to_numpy()) and np.array_equal(cols["_c1"], pdf[1].to_numpy())
    assert [dicts["_c2"][c] for c in cols["_c2"]] == list(pdf[2]) and np.array_equal(cols["_c3"], pdf[3].to_numpy(np.float64))


def test_literals_next_to_rounding_boundaries(lib):
    """The hardest inputs for a decimal -> double converter are literals a hair above or below the midpoint of two adjacent
    doubles.  Built exactly with decimal arithmetic: midpoint, then cut or bumped at the 17th..19th significant digit."""
    fields = midpoint_literals(np.random.default_rng(21))
    cls, st, val, _, _ = run(lib, fields)
    want = np.array([float(f) for f in fields])
    ok = st == OK
    assert np.array_equal(bits(val[ok]), bits(want[ok])) and set(np.unique(st[~ok])) <= {UNSUPPORTED}
    short = np.array([sum(ch.isdigit() for ch in f.split("e")[0].lstrip("0.")) <= 19 for f in fields])
    assert ok[short].all()                                                              # <= 19 digits in range: always answered
