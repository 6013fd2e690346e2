"""The decimal-literal corpora of the CSV reader's number tests and the host build of csrc/csv_number.h that classifies and
converts them.  tests/test_csv_number_host.py runs them through the host build against float() / int();
tests/test_csv_kernels.py runs the same literals through the device kernels and holds them to the host build."""
import ctypes as C
import decimal
import math
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NULL, INT, LONG, DOUBLE, STRING = range(5)
OK, NOT_A_NUMBER, UNSUPPORTED = range(3)


def build_host_lib(out_dir):
    """g++ build of tests/native/csv_number_host.cpp (the same csv_number.h the kernels compile) -> ctypes library"""
    out = os.path.join(str(out_dir), "libcsvnum.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-I", os.path.join(ROOT, "spark-network-traffic-classifier_b200", "csrc"),
                           os.path.join(ROOT, "tests", "native", "csv_number_host.cpp"), "-o", out])
    return C.CDLL(out)


def run(lib, fields):
    """fields (str or bytes) -> (class, double status, double value, int32 status, int32 value), one entry per field"""
    raw = [f if isinstance(f, bytes) else f.encode() for f in fields]
    offs = np.zeros(len(raw) + 1, np.int64)
    np.cumsum([len(r) for r in raw], out=offs[1:])
    blob = np.frombuffer(b"".join(raw) + b"\0", np.uint8)
    n = len(raw)
    cls, st, sti, iv = (np.zeros(n, np.int32) for _ in range(4))
    val = np.zeros(n, np.float64)
    lib.csvnum_batch(C.c_void_p(blob.ctypes.data), C.c_void_p(offs.ctypes.data), C.c_int64(n), C.c_void_p(cls.ctypes.data), C.c_void_p(st.ctypes.data),
                     C.c_void_p(val.ctypes.data), C.c_void_p(sti.ctypes.data), C.c_void_p(iv.ctypes.data))
    return cls, st, val, sti, iv


def writer_literals(rng, n=150000, n_hard=60000):
    """what a CSV writer produces -- repr (shortest round trip), %.6f, %.17g, %.10e over many magnitudes -- then 16-19 digit
    mantissas (beyond 2^53) with small exponents, the neighbours of 2^53 and a few fixed literals"""
    fields = []
    mags = 10.0 ** rng.uniform(-9, 15, n)
    vals = rng.standard_normal(n) * mags
    a, b, c = n // 3, n * 3 // 5, n * 4 // 5
    for v in vals[:a]:
        fields.append(repr(float(v)))
    for v in vals[a:b]:
        fields.append("%.6f" % v)
    for v in vals[b:c]:
        fields.append("%.17g" % v)
    for v in vals[c:n]:
        fields.append("%.10e" % v)
    for _ in range(n_hard):
        nd = int(rng.integers(16, 20))
        w = int(rng.integers(10 ** (nd - 1), 10 ** nd, dtype=np.uint64))
        q = int(rng.integers(-27 + 0, 9))
        s = str(w)
        k = int(rng.integers(0, nd))
        fields.append((s[:k] or "0") + "." + s[k:] + ("e%d" % (q + (nd - k))) if rng.random() < 0.5 else s + "e%d" % q)
    for e in range(-300, 300, 7):                                        # exact binary halfway points written in decimal
        fields.append(str(2 ** 53 + 1)); fields.append(str(2 ** 54 + 2)); fields.append(str(2 ** 53 + 3))
    fields += ["0.1", "0.30000000000000004", "9007199254740993", "9007199254740992.5", "4.35", "0.000001", "123456789012345678",
               "1.7976931348623157e27", "5e-27", "0.00", "1.00", "0.05", "-0.0", "0e999", "000.000"]
    return fields


def long_literals(rng, n=40000):
    """20 to 39 significant digits: exact when the truncated w and w + 1 round alike, refused otherwise"""
    fields = []
    for _ in range(n):
        nd = int(rng.integers(20, 40))
        s = "".join(str(d) for d in rng.integers(0, 10, nd))
        k = int(rng.integers(1, 12))
        fields.append(s[:k] + "." + s[k:])
    return fields


def midpoint_literals(rng, n=30000):
    """literals a hair below and above the midpoint of two adjacent doubles, built exactly with decimal arithmetic: the
    midpoint cut or bumped at the 17th..19th significant digit, and sometimes the exact tie itself (more than 19 digits)"""
    decimal.getcontext().prec = 60
    fields = []
    for _ in range(n):
        d = float(rng.uniform(1, 10)) * 10.0 ** int(rng.integers(-8, 12))
        mid = (decimal.Decimal(d) + decimal.Decimal(math.nextafter(d, math.inf))) / 2     # exact
        digits = int(rng.integers(17, 20))
        q = decimal.Decimal(1).scaleb(mid.adjusted() - digits + 1)
        lo = mid.quantize(q, rounding=decimal.ROUND_FLOOR)
        for v in (lo, lo + q):
            s = format(v, "f") if rng.random() < 0.5 else format(v, "e")
            fields.append(s)
        if digits == 19 and rng.random() < 0.2:
            fields.append(format(mid, "f"))
    return fields


def grammar_literals(rng, n=200000):
    """short random strings over the number grammar's alphabet (digits, signs, '.', exponents, blanks, the letters of NaN /
    Infinity): numbers, near-numbers and strings"""
    alphabet = list("0123456789") * 3 + list("+-.eE ") + list("aNIfnity\t")
    return ["".join(rng.choice(alphabet, size=int(rng.integers(0, 9)))) for _ in range(n)]
