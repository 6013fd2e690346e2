"""The device CSV reader's kernels (csrc/csv.cu, csrc/csv_number.h) at the edges where a tokenizer or a converter goes wrong:

  csv_count_lines / csv_line_starts   newlines at every residue mod 16 and around every 4 KB block edge, CRLF split across two
                                      threads and across two blocks, blank LF / CRLF runs, `\\r\\r\\n`, texts of any length, the
                                      quote flag in the first byte, the last byte of a block and the final partial chunk;
  csv_rows_kernel                     rows of 4063..4096 bytes (LF) and 4063..4095 bytes + CRLF, the first row over the cap,
                                      empty leading / trailing / all fields, one column, 1024 and 1025 columns, ragged rows
                                      whose first offender is far from the first CTA;
  csv_number.h on the device          every literal of the host test's corpora and the fast-path / 128-bit / q = +-27 edges,
                                      classified one literal per column and converted one literal per row, with the
                                      whitespace flags off, on and one at a time;
  dictionaries                        first appearance decided against thousands of later rows, the second file of a glob, two
                                      table growths, 4 KB strings, bytes >= 0x80, strings that differ only in blanks, a full
                                      16-slot table and one whose probes wrap around;
  read_csv(shard=...)                 every world size from 1 to 4 against the full read.

References: a Python list of line starts, oracle/csv_ref.py for records and dictionaries, Python's float() / int() for values,
and the host build of csv_number.h (tests/csv_corpus.py) for which literals the converter answers and which it refuses."""
import numpy as np
import pytest
import torch

from b200flow import _lib, csvio
from csv_corpus import (NOT_A_NUMBER, NULL, OK, STRING, UNSUPPORTED, build_host_lib, grammar_literals, long_literals, midpoint_literals, run,
                        writer_literals)
from oracle import csv_ref

pytestmark = pytest.mark.gpu

DEV = "cuda"
BAD_RAGGED, BAD_RAGGED_FIRST, BAD_LONG, BAD_NUMBER, BAD_UNSUPPORTED, BAD_NUMBER_FIRST, BAD_DICT_FULL, BAD_DICT_MISS = range(8)
U64_MAX = 2 ** 64 - 1
WS = bytes(range(0x21))                       # what the strip flags and Java's trim() remove


# ------------------------------------------------------------------------------------------------ helpers
def _dev(data, pad=b""):
    """bytes -> device buffer (torch allocations are 16-byte aligned, as the line index needs); pad: bytes past the text"""
    return torch.from_numpy(np.frombuffer(bytes(data) + pad, np.uint8).copy()).to(DEV)


def _new_bad(n=1):
    bad = torch.zeros((n, 8), dtype=torch.int64, device=DEV)
    bad[:, BAD_RAGGED_FIRST] = -1
    bad[:, BAD_NUMBER_FIRST] = -1
    return bad


def _u64(t):
    return t.cpu().numpy().view(np.uint64)


def _cols(types, size):
    """column descriptors of numeric columns stored back to back, `size` bytes each"""
    c = np.zeros(len(types), csvio.COL_DTYPE)
    c["type"] = types
    c["rec_off"] = np.arange(len(types)) * size
    c["str_index"] = -1
    return torch.from_numpy(c.view(np.uint8)).to(DEV)


def _table(rows):
    """rows (lists of field bytes) -> (text, row start offsets)"""
    lines = [b",".join(r) for r in rows]
    starts = np.zeros(len(lines), np.int64)
    np.cumsum([len(ln) + 1 for ln in lines[:-1]], out=starts[1:])
    return b"\n".join(lines) + b"\n", starts


def _strip(f, flags):
    if flags & 1:
        f = f.lstrip(WS)
    if flags & 2:
        f = f.rstrip(WS)
    return f


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _fnv(b):
    h = 1469598103934665603
    for c in b:
        h = ((h ^ c) * 1099511628211) & (2 ** 64 - 1)
    return h or 1


def _same_as_ref(paths, **kw):
    """read_csv against csv_ref.read_csv: schema, every record field (doubles bit for bit) and the dictionaries"""
    rec, schema, dicts = csvio.read_csv(paths, **kw)
    names, types, cols, want_dicts = csv_ref.read_csv(paths, **kw)
    assert schema.names == names and schema.types == types, (schema.names, schema.types, names, types)
    n = len(next(iter(cols.values()))) if cols else 0
    assert rec.shape[0] == n
    host = rec.cpu().numpy().view(schema.numpy_dtype()).reshape(-1) if n else None
    for name, typ in zip(names, types):
        if not n:
            continue
        if typ == "f64":
            assert np.array_equal(_bits(host[name]), _bits(cols[name])), name
        else:
            assert np.array_equal(host[name], cols[name]), name
    assert dicts == want_dicts
    return rec, schema, dicts


def _write(tmp_path, name, data):
    p = str(tmp_path / name)
    with open(p, "wb") as f:
        f.write(data if isinstance(data, bytes) else data.encode())
    return p


# ------------------------------------------------------------------------------------------------ line index
def _ref_starts(data):
    """offset of every non-empty line: csv_ref's rule (split at '\\n', drop one trailing '\\r', skip empty lines)"""
    out, o = [], 0
    for seg in data.split(b"\n"):
        if seg[:-1] if seg.endswith(b"\r") else seg:
            out.append(o)
        o += len(seg) + 1
    return out


def _check_index(data):
    """the two line-index kernels, called directly on `data` followed by quotes the kernels must not read"""
    n = len(data)
    text = _dev(data, b'"' * 48)
    n_blocks = (n + 4095) // 4096
    counts = torch.full((n_blocks,), -1, dtype=torch.int32, device=DEV)
    flags = torch.zeros(1, dtype=torch.int64, device=DEV)
    _lib.call("b200flow_csv_count_lines", _lib.ptr(text), n, _lib.ptr(counts), _lib.ptr(flags))
    want = _ref_starts(data)
    c = counts.cpu().numpy().astype(np.int64)
    assert c.tolist() == np.bincount(np.asarray(want, np.int64) // 4096, minlength=n_blocks).tolist()
    assert int(flags.item()) == (1 if b'"' in data else 0)
    bases = torch.from_numpy(np.concatenate([[0], np.cumsum(c)[:-1]]).astype(np.int64)).to(DEV)
    starts = torch.full((len(want) + 1,), -1, dtype=torch.int64, device=DEV)       # one sentinel past the end
    _lib.call("b200flow_csv_line_starts", _lib.ptr(text), n, _lib.ptr(bases), _lib.ptr(starts))
    got = starts.cpu().numpy()
    assert got[:-1].tolist() == want and got[-1] == -1


def test_line_index_newlines_at_every_residue_and_block_edge():
    L = 3 * 4096 + 37
    for r in range(16):                                                   # a line start at every residue mod 16
        b = bytearray(b"a" * L)
        b[r::16] = b"\n" * len(range(r, L, 16))
        _check_index(bytes(b))
    for d1 in range(-3, 3):                                               # one or two newlines on either side of each 4 KB edge
        for d2 in range(d1, 3):
            b = bytearray(b"x,1" * (L // 3 + 1))[:L]
            for k in (1, 2, 3):
                b[k * 4096 + d1] = b[k * 4096 + d2] = ord("\n")
            _check_index(bytes(b))


def test_line_index_crlf_split_between_threads_and_blocks():
    L = 3 * 4096 + 21
    pats = [b"\r\n", b"\n\r\n", b"\r\n\r\n", b"\n\r\r\n", b"\n\r\ra", b"\n\n", b"\n\ra\n", b"\r\r\n\r\n"]
    for at in (15, 31, 4095, 8191, 4096 * 3 - 1):                          # the last byte of a thread's 16 / of a block
        for pat in pats:
            for shift in range(-len(pat), 2):
                b = bytearray(b"ab,c" * (L // 4 + 1))[:L]
                b[at + shift:at + shift + len(pat)] = pat
                _check_index(bytes(b))
    # a CRLF whose '\r' is the last byte of every thread's 16 bytes, and "\r\r\n" lines starting at every residue
    b = bytearray(b"q" * L)
    for p in range(15, L - 1, 16):
        b[p:p + 2] = b"\r\n"
    _check_index(bytes(b))
    parts = []
    for k in range(900):
        parts.append(b"x" * (k % 37) + b"\n\r\r\n")
    _check_index(b"".join(parts))


def test_line_index_blank_runs_short_texts_and_fuzz():
    rng = np.random.default_rng(1)
    pieces = [b"", b"\r", b"\r\r", b"a", b"a\r", b"ab,c", b"\ra", b"1,2,3"]
    for seed_len in (3 * 4096 + 5, 2 * 4096 + 16, 4096, 4095, 12345):
        lines = [pieces[int(i)] for i in rng.integers(0, len(pieces), seed_len // 2)]
        _check_index(b"\n".join(lines)[:seed_len])
    for _ in range(6):                                                    # every local pattern of '\n', '\r' at every alignment
        n = int(rng.integers(3 * 4096, 4 * 4096))
        _check_index(bytes(rng.choice(np.frombuffer(b"\n\r\ra,", np.uint8), n).tobytes()))
    for t in [b"a", b"\n", b"\r", b"\r\n", b"abc", b"abc\r", b"a,b,c\n", b"\n\n\r\n\n", b"x" * 4095, b"x" * 4096, b"x" * 4097,
              b"x" * 4095 + b"\n", b"x" * 4096 + b"\n", b"\n" + b"x" * 4096, b"y" * 17, b"y" * 33 + b"\r"]:
        _check_index(t)                                                   # single lines, lengths not a multiple of 16


def test_line_index_quote_flag():
    base = b"a,b\n" * 3000 + b"c,dd\n"                                     # 12005 bytes: a final partial chunk of 5
    n = len(base)
    assert n % 16 != 0
    _check_index(base)
    for p in (0, 4095, 8191, n - n % 16, n - 1, n - 2):
        b = bytearray(base)
        b[p] = ord('"')
        _check_index(bytes(b))


def test_read_csv_files_without_newline_globs_and_blank_lines_before_headers(tmp_path):
    p1 = _write(tmp_path, "a.csv", "\n\r\n\nname,val,n\nx,1.5,1\ny,2,2\nz,,3")                     # no trailing newline
    p2 = _write(tmp_path, "b.csv", "\r\n\r\nname,val,n\r\nw,-0,4\r\n\r\nx,1e5,5\r\n\r\n")
    p3 = _write(tmp_path, "c.csv", "")
    p4 = _write(tmp_path, "d.csv", "\n\n")
    p5 = _write(tmp_path, "e.csv", "name,val,n\nv,7,6\r")                                            # ends in a lone '\r'
    _same_as_ref([p1, p2, p3, p4, p5], header=True, infer_schema=True)
    _same_as_ref([p5, p4, p2, p1], header=True, infer_schema=False)
    q = _write(tmp_path, "one.csv", "1,abc,2.5")
    _same_as_ref([q], infer_schema=True)
    _same_as_ref([q, q, q], infer_schema=True)


# ------------------------------------------------------------------------------------------------ row tokenizer
@pytest.mark.parametrize("eol", [b"\n", b"\r\n"], ids=["lf", "crlf"])
def test_rows_up_to_the_4096_byte_cap(tmp_path, eol):
    top = 4097 - len(eol)                       # at most 4096 bytes before the '\n', a CRLF's '\r' included
    shapes = [lambda L: b"7," + b"x" * (L - 4) + b",9",                                   # long middle field
              lambda L: b"s%d" % (L % 10) + b"y" * (L - 6) + b",7,9",                      # long first field
              lambda L: b"7,x," + b"0" * (L - 7) + (b"1.5" if L % 2 else b"123")]         # long last numeric field
    for k, shape in enumerate(shapes):
        rows = [shape(L) for L in range(4063, top + 1)]
        assert [len(r) for r in rows] == list(range(4063, top + 1))
        rows = [b"1,a,2"] + rows[:10] + [b"3,b,4"] + rows[10:]
        for tail in (eol, b""):                                           # the longest row last, with and without a newline
            p = _write(tmp_path, "cap%d.csv" % k, eol.join(rows) + tail)
            _same_as_ref([p], infer_schema=True)
            _same_as_ref([p], infer_schema=False)
        over = _write(tmp_path, "over%d.csv" % k, eol.join([b"1,a,2", shape(top + 1), b"3,b,4", shape(top)]) + eol)
        for infer in (True, False):
            with pytest.raises(csvio.CsvFormatError, match=r": 1 row\(s\) are longer than 4096 bytes"):
                csvio.read_csv([over], infer_schema=infer)


def test_empty_fields_and_one_column(tmp_path):
    p = _write(tmp_path, "empty.csv", "1,2,,\n,1,2,3\n,,,\n4,,5,\n7,8,9,10\n,,,x\n")
    _same_as_ref([p], infer_schema=True)
    _same_as_ref([p], infer_schema=False)
    _same_as_ref([p], infer_schema=True, strip_lead=True, strip_trail=True)
    q = _write(tmp_path, "one.csv", "5\n\n6\r\n-7\n+8\n")
    _same_as_ref([q], infer_schema=True)
    r = _write(tmp_path, "one_str.csv", "a\nb\r\n\na\n 1\n")
    _same_as_ref([r], infer_schema=True)
    _same_as_ref([r], infer_schema=False)


def test_1024_columns_and_1025_refused(tmp_path):
    rng = np.random.default_rng(2)
    pick = [["0", "7", "-3", "12"], [".5", "1.", "2e3", "-0"], ["a", "b", "zz", ""], ["9", "", "1", "2"]]
    rows = [",".join(pick[c % 4][int(rng.integers(0, 4))] for c in range(1024)) for _ in range(3000)]
    assert max(len(r) for r in rows) <= 4096
    p = _write(tmp_path, "wide.csv", "\n".join(rows) + "\n")
    _, schema, _ = _same_as_ref([p], infer_schema=True)
    assert len(schema.names) == 1024 and set(schema.types) == {"i32", "f64", "code"}
    h = _write(tmp_path, "wide_header.csv", ",".join("c%d" % i for i in range(1024)) + "\n" + "\n".join(rows[:500]) + "\n")
    _same_as_ref([h], header=True, infer_schema=True)
    w = _write(tmp_path, "wider.csv", "\n".join(r + ",1" for r in rows[:50]) + "\n")
    with pytest.raises(csvio.CsvFormatError, match="more than 1024 columns"):
        csvio.read_csv([w], infer_schema=True)
    data = open(w, "rb").read()
    text, st = _dev(data), torch.tensor(_ref_starts(data), dtype=torch.int64, device=DEV)
    cls, bad = torch.zeros(2 * 1025, dtype=torch.int32, device=DEV), _new_bad()
    with pytest.raises(_lib.B200FlowError, match="bad arguments"):
        _lib.call("b200flow_csv_infer", _lib.ptr(text), len(data), _lib.ptr(st), 50, 1025, 0, _lib.ptr(cls), _lib.ptr(cls[1025:]), _lib.ptr(bad))


@pytest.mark.parametrize("first_kind", ["too_few", "too_many"])
def test_ragged_rows_first_offender(tmp_path, first_kind):
    n = 20000
    rows = ["%d,%d,%d" % (i, i % 7, i % 5) for i in range(n)]
    bad_rows = {9001: "1,2" if first_kind == "too_few" else "1,2,3,4", 12000: "1,2,3,4,5", 15000: "1", n - 1: "1,2,3,"}
    for i, r in bad_rows.items():
        rows[i] = r
    body = "\n".join(rows[:100]) + "\n\n\r\n\n" + "\n".join(rows[100:]) + "\n"       # blank lines are not data rows
    for header in (False, True):
        p = _write(tmp_path, "ragged.csv", ("a,b,c\n\n" if header else "") + body)
        for infer in (True, False):
            with pytest.raises(csvio.CsvFormatError, match=r": 4 row\(s\) do not have 3 fields \(first: data row 9001\)"):
                csvio.read_csv([p], header=header, infer_schema=infer)


# ------------------------------------------------------------------------------------------------ decimal converter
def _edge_literals():
    out = []
    mants = ["1", "5", "9", "9007199254740991", "9007199254740992", "9007199254740993", "9007199254740994", "12345678901234567",
             "1234567890123456789", "9999999999999999999", "9223372036854775807"]
    for k in (21, 22, 23, 26, 27, 28, 29):                               # Clinger's |q| <= 22 and the 128-bit |q| <= 27
        for m in mants:
            for sg in ("", "-"):
                out += ["%s%se%d" % (sg, m, k), "%s%se-%d" % (sg, m, k), "%s%sE+%d" % (sg, m, k)]
    for d in range(-3, 4):                                               # 2^53 +- 1
        v = 2 ** 53 + d
        out += [str(v), "%d.0" % v, "%d.5" % v, "-%d" % v, "%de1" % v, "%de-1" % v, "0.%de16" % v, "%d.00000000000000000001" % v]
    for w in ("1", "7", "123456789", "1234567890123456789", "9999999999999999999"):
        for q in range(-30, 31):
            out.append("%se%d" % (w, q))
        for q in (26, 27, 28, 29):                                       # q from dropped digits: w and zeros past the 19th
            out.append(w + "0" * (q + 19 - len(w)))
            out.append(w + "1" + "0" * (q + 18 - len(w)))
        for q in (-26, -27, -28, -29):                                   # q from the fraction's length
            out.append("0." + "0" * (-q - len(w)) + w)
            out.append("-." + "0" * (-q - len(w)) + w)
        out.append(w + ".123456789e27")
        out.append(w + "." + "0" * 30 + "1e-1")
    for w in ("1234567890123456789", "9007199254740993000", "1000000000000000001", "9999999999999999999"):   # 19 digits, leading zeros
        out += ["000" + w, "-000" + w, "0000." + w, "0.000" + w, "000" + w + ".000", "00" + w + "e8", "0" * 30 + w,
                "0." + "0" * 8 + w, "0." + "0" * 9 + w, "+0" + w + "e-27", "0" + w + "0"]
    out += ["-0.0", "-0", "+0", "0", "0.0e0", "-0e-999", "0e999", "-.0", "NaN", "Infinity", "+Infinity", "-Infinity", "Inf", "+Inf",
            "-Inf", "inf", "INF", "nan", "+NaN", "-NaN", "1e400", "-1e-400", "1.7976931348623157e308", "4.9e-324"]
    return out


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp("csvnum"))


@pytest.fixture(scope="module")
def corpus():
    """every literal of the host test's generated corpora and the edge literals, as field bytes, ~20% with blanks around"""
    fields = (writer_literals(np.random.default_rng(7)) + long_literals(np.random.default_rng(9)) + midpoint_literals(np.random.default_rng(21))
              + grammar_literals(np.random.default_rng(11)) + _edge_literals())
    rng = np.random.default_rng(5)
    pads = [b"", b"", b"", b"", b"", b"", b"", b" ", b"\t", b" \t "]
    raw = []
    for f in fields:
        b = f.encode()
        assert not any(c in b for c in b',\n\r"')
        raw.append(pads[int(rng.integers(0, len(pads)))] + b + pads[int(rng.integers(0, len(pads)))])
    return raw


def _pack(raw):
    """literals -> rows of at most 1024 fields and 4096 bytes (never a lone empty field: that would be a blank line)"""
    rows, a, size = [], 0, -1
    for i, f in enumerate(raw):
        if i > a and (i - a == 1024 or size + 1 + len(f) > 4096):
            rows.append((a, i)); a, size = i, -1
        size += 1 + len(f)
    rows.append((a, len(raw)))
    assert all(b - a >= 2 or raw[a] for a, b in rows)
    return rows


@pytest.mark.parametrize("flags", [0, 1, 2, 3])
def test_device_class_per_literal_equals_the_host_converter(host, corpus, flags):
    lits = sorted(corpus, key=len)                                        # the shortest fill rows of 1024 columns
    rows = _pack(lits)
    text, starts = _table([lits[a:b] for a, b in rows])
    t, st = _dev(text), torch.from_numpy(starts).to(DEV)
    out = torch.zeros((2, len(lits)), dtype=torch.int32, device=DEV)
    bad = _new_bad()
    for i, (a, b) in enumerate(rows):                                     # one row per call: each column's class is one literal's
        _lib.call("b200flow_csv_infer", _lib.ptr(t), len(text), _lib.ptr(st[i:i + 1]), 1, b - a, flags, _lib.ptr(out[0, a:b]),
                  _lib.ptr(out[1, a:b]), _lib.ptr(bad))
    got = out.cpu().numpy()
    assert not _u64(bad)[0, [BAD_RAGGED, BAD_LONG]].any()
    want = run(host, [_strip(f, flags) for f in lits])[0]
    wrong = np.nonzero(got[0] != want)[0]
    assert not len(wrong), [(lits[i], int(got[0, i]), int(want[i])) for i in wrong[:10]]
    assert np.array_equal(got[1], (want == NULL).astype(np.int32))
    assert max(b - a for a, b in rows) == 1024


@pytest.mark.parametrize("flags", [0, 3])
def test_device_doubles_bit_for_bit_one_literal_per_row(host, corpus, flags):
    s = [_strip(f, flags) for f in corpus]
    st = run(host, s)[1]
    keep = [i for i in range(len(corpus)) if st[i] == OK and corpus[i]]   # an empty literal alone would be a blank line
    text, starts = _table([[corpus[i]] for i in keep])
    n = len(keep)
    t, st, cols = _dev(text), torch.from_numpy(starts).to(DEV), _cols([csvio.CSV_DOUBLE], 8)
    rec = torch.zeros((n, 8), dtype=torch.uint8, device=DEV)
    bad = _new_bad()
    _lib.call("b200flow_csv_parse", _lib.ptr(t), len(text), _lib.ptr(st), n, 1, flags, _lib.ptr(cols), None, None, None, 4, _lib.ptr(rec), 8,
              _lib.ptr(bad))
    assert _u64(bad)[0].tolist() == [0, U64_MAX, 0, 0, 0, U64_MAX, 0, 0]
    got = _bits(rec.cpu().numpy().view(np.float64).reshape(-1))
    want = _bits([csv_ref.to_double(s[i]) for i in keep])                # float(), with Java's NaN / Infinity spellings
    wrong = np.nonzero(got != want)[0]
    assert not len(wrong), [(corpus[keep[i]], hex(int(got[i])), hex(int(want[i]))) for i in wrong[:10]]
    assert n > 350000


def _batches(host, literals, flags, col_type, width, rows_per_batch):
    """literals in `width`-column tables of one type, one parse call per batch of rows -> per batch: the device's bad[] and
    values, and the host build's status and value of every literal"""
    size = 8 if col_type == csvio.CSV_DOUBLE else 4
    n = len(literals) - len(literals) % width
    rows = [literals[i:i + width] for i in range(0, n, width)]
    text, starts = _table(rows)
    t, st = _dev(text), torch.from_numpy(starts).to(DEV)
    cols = _cols([col_type] * width, size)
    nb = (len(rows) + rows_per_batch - 1) // rows_per_batch
    rec = torch.zeros((len(rows), width * size), dtype=torch.uint8, device=DEV)
    bad = _new_bad(nb)
    for k in range(nb):
        r0, r1 = k * rows_per_batch, min(len(rows), (k + 1) * rows_per_batch)
        _lib.call("b200flow_csv_parse", _lib.ptr(t), len(text), _lib.ptr(st[r0:r1]), r1 - r0, width, flags, _lib.ptr(cols), None, None, None, 4,
                  _lib.ptr(rec[r0:r1]), width * size, _lib.ptr(bad[k]))
    _, st_d, val, st_i, iv = run(host, [_strip(f, flags) for f in literals[:n]])
    return _u64(bad), rec.cpu().numpy(), (st_d, val) if col_type == csvio.CSV_DOUBLE else (st_i, iv), n


def _check_batches(bad, status, width, rows_per_batch):
    per = width * rows_per_batch
    for k in range(bad.shape[0]):
        s = status[k * per:(k + 1) * per]
        off = np.nonzero(s != OK)[0]
        first = U64_MAX if not len(off) else ((int(off[0]) // width) << 16) | (int(off[0]) % width)
        assert (int(bad[k, BAD_NUMBER]), int(bad[k, BAD_UNSUPPORTED]), int(bad[k, BAD_NUMBER_FIRST])) == \
            (int((s == NOT_A_NUMBER).sum()), int((s == UNSUPPORTED).sum()), first), k
        assert not bad[k, [BAD_RAGGED, BAD_LONG, BAD_DICT_MISS]].any()


@pytest.mark.parametrize("flags", [0, 1, 2, 3])
def test_device_refusals_and_first_offender_equal_the_host_converter(host, corpus, flags):
    """the numeric literals (answered or refused) in 8-column DOUBLE tables, with a few non-numbers mixed in: per batch the
    device's UNSUPPORTED / not-a-number counts and first offender (row, column) are the host's, and every answer is float()'s"""
    s = [_strip(f, flags) for f in corpus]
    cls, st = run(host, s)[:2]
    lits = [f for i, f in enumerate(corpus) if st[i] != NOT_A_NUMBER or (cls[i] == STRING and i % 500 == 0)]
    W, R = 8, 256
    bad, rec, (status, _), n = _batches(host, lits, flags, csvio.CSV_DOUBLE, W, R)
    assert (status == UNSUPPORTED).sum() > 1000
    _check_batches(bad, status, W, R)
    got = _bits(rec.view(np.float64).reshape(-1))
    ok = np.nonzero(status == OK)[0]
    want = _bits([csv_ref.to_double(_strip(lits[i], flags)) for i in ok])
    assert np.array_equal(got[ok], want)


@pytest.mark.parametrize("flags", [0, 1, 2, 3])
def test_device_int32_fields(host, flags):
    rng = np.random.default_rng(17)
    vals = [int(v) for v in rng.integers(-2 ** 31, 2 ** 31, 30000)]
    lits = []
    for v in vals:
        r = rng.random()
        lits.append("+%d" % v if r < 0.1 and v >= 0 else ("%s%010d" % ("-" if v < 0 else "", abs(v)) if r < 0.2 else str(v)))
    edge = ["2147483647", "-2147483648", "+2147483647", "-02147483648", "0002147483647", "-0", "+0", "0", "0" * 25 + "7", "-" + "0" * 30,
            "2147483646", "-2147483647", "2147483648", "-2147483649", "+2147483648", "4294967296", "9223372036854775807",
            "00000000000000000002147483648", "99999999999999999999", "+-1", "--1", "1.0", "1e3", "", "-", "+", "0x1", "1 2", "NaN"]
    for i, e in enumerate(edge):
        lits.insert(int(rng.integers(0, len(lits))), e)
    pads = [b"", b"", b"", b"", b" ", b"\t", b"  "]
    raw = [pads[int(rng.integers(0, len(pads)))] + f.encode() + pads[int(rng.integers(0, len(pads)))] for f in lits]
    W, R = 4, 64
    bad, rec, (status, ival), n = _batches(host, raw, flags, csvio.CSV_INT32, W, R)
    _check_batches(bad, status, W, R)
    got = rec.view(np.int32).reshape(-1)
    ok = np.nonzero(status == OK)[0]
    assert np.array_equal(got[ok], np.array([int(_strip(raw[i], flags)) for i in ok], np.int64).astype(np.int32))
    assert np.array_equal(got[ok], ival[ok])
    assert (status != OK).sum() >= (17 if flags == 3 else 1000)         # without both flags, padded literals are not ints


# ------------------------------------------------------------------------------------------------ dictionaries
def test_dictionary_first_appearance_against_later_rows(tmp_path):
    rng = np.random.default_rng(3)
    vals = ["k%03d" % i for i in rng.permutation(96)]
    col = vals + [vals[int(i)] for i in rng.integers(0, 96, 60000)]
    hot = ["hot"] + ["" if rng.random() < 0.01 else ("hot" if rng.random() < 0.99 else "c%d" % rng.integers(0, 50)) for _ in col[1:]]
    p = _write(tmp_path, "hot.csv", "\n".join("%d,%s,%s" % (i, a, b) for i, (a, b) in enumerate(zip(col, hot))) + "\n")
    _, _, dicts = _same_as_ref([p], infer_schema=True)
    assert dicts["_c1"] == vals and dicts["_c2"][0] == "hot"


def test_dictionary_values_first_seen_in_the_second_file(tmp_path):
    a = _write(tmp_path, "a.csv", "proto,svc\n" + "tcp,http\nudp,\ntcp,dns\n" * 500)
    b = _write(tmp_path, "b.csv", "proto,svc\nicmp,ntp\ntcp,http\nsctp,ssh\n" + "udp,ssh\n" * 3000 + "gre,x\n")
    _same_as_ref([a, b], header=True, infer_schema=True)
    _same_as_ref([b, a], header=True, infer_schema=True)


@pytest.mark.parametrize("n_distinct", [3000, 20000])
def test_dictionary_grows(tmp_path, n_distinct):
    """the table starts at 4096 slots per column and grows by 8x whenever a column fills more than half of it"""
    rng = np.random.default_rng(n_distinct)
    vals = ["v%d" % i for i in rng.permutation(n_distinct)]
    col = vals + [vals[int(i)] for i in rng.integers(0, n_distinct, 20000)]
    col = [col[0]] + [col[int(i)] for i in rng.permutation(np.arange(1, len(col)))]
    p = _write(tmp_path, "many.csv", "\n".join("%s,%d" % (v, i) for i, v in enumerate(col)) + "\n")
    _, _, dicts = _same_as_ref([p], infer_schema=True)
    assert len(dicts["_c0"]) == n_distinct


def test_dictionary_long_strings_and_high_bytes(tmp_path):
    rng = np.random.default_rng(4)
    letters = np.frombuffer(b"abcdefghij", np.uint8)
    base = bytes(rng.choice(letters, 4090).tobytes())
    longs = [base[:L] for L in (3990, 4000, 4050, 4089, 4090)] + [b"Z" + base[1:4090], base[:4089] + b"Z"]
    highs = [bytes(rng.integers(0x80, 0x100, int(rng.integers(1, 9)), dtype=np.uint8).tobytes()) for _ in range(200)]
    highs += ["é".encode(), "日本".encode(), "Web Attack – Brute Force".encode(), b"\xff\xfe", b"\x80", b"\x81"]
    rows = []
    for i in range(6000):
        v = longs[int(rng.integers(0, len(longs)))] if i % 3 == 0 else highs[int(rng.integers(0, len(highs)))]
        rows.append(v + b",%d" % (i % 11))
    p = _write(tmp_path, "strings.csv", b"\n".join(rows) + b"\n")
    _same_as_ref([p], infer_schema=True)


@pytest.mark.parametrize("lead,trail", [(False, False), (True, False), (False, True), (True, True)])
def test_dictionary_strings_that_differ_in_blanks(tmp_path, lead, trail):
    vals = ["a", " a", "a ", "\ta\t", " a \t", "b", " b", "b\t", "  ", "", " 5", "5 ", "5"]
    rng = np.random.default_rng(6)
    rows = ["%s,%s,%d" % (vals[int(rng.integers(0, len(vals)))], [" 5", "5 ", "5", "\t7"][i % 4], i) for i in range(4000)]
    p = _write(tmp_path, "blanks.csv", "\n".join(rows) + "\n")
    _same_as_ref([p], infer_schema=True, strip_lead=lead, strip_trail=trail)


def _dict_call(rows, cap_log2, guard=16):
    """b200flow_csv_dictionary on one string column (column 1 of `rows`), with guard words either side of the table"""
    text, starts = _table(rows)
    cap = 1 << cap_log2
    keys = torch.zeros(cap + 2 * guard, dtype=torch.int64, device=DEV)
    pos_len = torch.full((cap + 2 * guard,), 0x5A5A5A5A, dtype=torch.int64, device=DEV)
    pos_len[guard:guard + cap] = np.iinfo(np.int64).max
    bad = _new_bad()
    t, st = _dev(text), torch.from_numpy(starts).to(DEV)
    cols = torch.from_numpy(np.array([(csvio.CSV_INT32, 0, -1, 0), (csvio.CSV_STRING, 4, 0, 0)], csvio.COL_DTYPE).view(np.uint8)).to(DEV)
    _lib.call("b200flow_csv_dictionary", _lib.ptr(t), len(text), _lib.ptr(st), len(rows), 2, 0, _lib.ptr(cols), _lib.ptr(keys[guard:guard + cap]),
              _lib.ptr(pos_len[guard:guard + cap]), cap_log2, _lib.ptr(bad))
    k, pl = keys.cpu().numpy(), pos_len.cpu().numpy()
    assert not k[:guard].any() and not k[guard + cap:].any()
    assert (pl[:guard] == 0x5A5A5A5A).all() and (pl[guard + cap:] == 0x5A5A5A5A).all()
    first = {}
    for r, row in enumerate(rows):
        first.setdefault(row[1], (int(starts[r]) + len(row[0]) + 1) << 16 | len(row[1]))
    return t, st, cols, k[guard:guard + cap].view(np.uint64), pl[guard:guard + cap], _u64(bad)[0], first


def test_dictionary_full_table_counts_and_stays_inside():
    vals = [b"d%02d" % i for i in range(20)]
    _, _, _, keys, pl, bad, first = _dict_call([[b"%d" % i, v] for i, v in enumerate(vals)], 4)
    assert int(bad[BAD_DICT_FULL]) == 4 and (keys != 0).all()
    by_hash = {_fnv(v): v for v in vals}
    assert len(set(keys.tolist())) == 16 and set(keys.tolist()) <= set(by_hash)
    for k, p in zip(keys.tolist(), pl.tolist()):
        assert p == first[by_hash[k]]


def test_dictionary_probes_wrap_around_a_nearly_full_table():
    home = lambda v: (lambda h: (h ^ (h >> 32)) & 15)(_fnv(v))
    cands = [b"w%d" % i for i in range(2000)]
    vals = [v for v in cands if home(v) == 15][:8] + [v for v in cands if home(v) == 14][:7]      # 15 values homed at the end
    rng = np.random.default_rng(8)
    order = [vals[int(i)] for i in rng.permutation(15)]
    col = order + [vals[int(i)] for i in rng.integers(0, 15, 6000)]
    rows = [[b"%d" % i, v] for i, v in enumerate(col)]
    t, st, cols, keys, pl, bad, first = _dict_call(rows, 4)
    assert int(bad[BAD_DICT_FULL]) == 0 and int((keys == 0).sum()) == 1
    assert set(keys[keys != 0].tolist()) == {_fnv(v) for v in vals}
    by_hash = {_fnv(v): v for v in vals}
    for s in np.nonzero(keys)[0]:
        v = by_hash[int(keys[s])]
        assert pl[s] == first[v]
        h = home(v)
        assert all(keys[(h + j) % 16] for j in range((int(s) - h) % 16))                        # no hole between home and slot
    # lookups walk the same wrapped probe sequence: codes in order of first appearance
    code = {v: c for c, v in enumerate(order)}
    slot_code = torch.tensor([code[by_hash[int(k)]] if k else -1 for k in keys], dtype=torch.int32, device=DEV)
    keys_d, pl_d = torch.from_numpy(keys.view(np.int64).copy()).to(DEV), torch.from_numpy(pl.copy()).to(DEV)
    rec = torch.zeros((len(rows), 8), dtype=torch.uint8, device=DEV)
    bad2 = _new_bad()
    _lib.call("b200flow_csv_parse", _lib.ptr(t), int(t.numel()), _lib.ptr(st), len(rows), 2, 0, _lib.ptr(cols), _lib.ptr(keys_d), _lib.ptr(pl_d),
              _lib.ptr(slot_code), 4, _lib.ptr(rec), 8, _lib.ptr(bad2))
    assert _u64(bad2)[0].tolist() == [0, U64_MAX, 0, 0, 0, U64_MAX, 0, 0]
    got = rec.cpu().numpy().view(np.int32).reshape(-1, 2)
    assert got[:, 1].tolist() == [code[v] for v in col] and got[:, 0].tolist() == list(range(len(col)))


# ------------------------------------------------------------------------------------------------ sharded reads
def test_sharded_reads_concatenate_to_the_full_read(tmp_path):
    rng = np.random.default_rng(10)
    rows = ["%d,%s,%s,%s" % (i, repr(float(rng.standard_normal())), ["tcp", "udp"][i % 2], "late%d" % (i % 3) if i > 9000 else "x")
            for i in range(10007)]
    a = _write(tmp_path, "a.csv", "n,v,p,s\n" + "\n".join(rows[:6000]) + "\n")
    b = _write(tmp_path, "b.csv", "\n\nn,v,p,s\r\n" + "\r\n".join(rows[6000:]))
    tiny = _write(tmp_path, "tiny.csv", "n,v,p,s\n1,2.5,tcp,q\n2,3.5,udp,r\n3,,tcp,q\n")
    for paths in ([a, b], [tiny]):
        full, schema, dicts = _same_as_ref(paths, header=True, infer_schema=True)
        for w in (1, 2, 3, 4):
            parts = []
            for r in range(w):
                rec, sch, d = csvio.read_csv(paths, header=True, infer_schema=True, shard=(r, w))
                assert sch.names == schema.names and sch.types == schema.types and d == dicts
                parts.append(rec)
            assert torch.equal(torch.cat(parts), full)
