"""CSV files -> AoS flow records on the device (SURVEY.md 8f-3).

`spark.read.csv(path_or_glob, inferSchema=True, header=...)` (kdd99.py:25, cicids17.py:19-20) made GPU-native: the host only
reads the files' BYTES into pinned memory and copies them to the GPU; the line index, Spark's per-column type inference, the
string dictionaries and the text -> int32 / float64 / dictionary-code conversion are CUDA kernels (csrc/csv.cu), with Java's
correctly rounded parseDouble semantics (csrc/csv_number.h).  The host touches text again only for the header line and to
fetch each DISTINCT string once (a few dozen per column).

No CPU fallback: quoted fields, ragged rows, rows over 4096 bytes or numeric literals the exact converter cannot round raise
CsvFormatError.  (The pyspark shim keeps a pandas reader as an explicit opt-in `option("b200flow.csvEngine", "host")`, and the
tests use pandas / Python's float() as the checker.)
"""
import numpy as np
import torch

from ._lib import B200FlowError, call, ptr, require_cuda
from .encode import RecordSchema

CSV_NULL, CSV_INT32, CSV_INT64, CSV_DOUBLE, CSV_STRING = 0, 1, 2, 3, 4
COL_DTYPE = np.dtype([("type", "<i4"), ("rec_off", "<i4"), ("str_index", "<i4"), ("reserved", "<i4")])
_TEXT_BLOCK = 4096                       # bytes of text per line-index block (csv.cu kIdxThreads * 16)
_I64_MAX = np.iinfo(np.int64).max
_U64_MAX = np.iinfo(np.uint64).max


class CsvFormatError(B200FlowError, ValueError):
    """input the device CSV reader does not accept (it never guesses): quoted fields, ragged rows, inexact literals"""


_STAGE_BYTES = 32 << 20
_stage = []                              # two pinned staging blocks, allocated once (page-locking costs more than the copy)


def _load_text(paths, device):
    """files -> one device byte buffer (every file ends with a newline) + the files' base offsets + each file's first 64 KB.
    Double-buffered: the next block is read from the file while the previous one is on its way to the GPU."""
    import os
    sizes = [os.path.getsize(p) for p in paths]
    total = sum(s + 1 for s in sizes)
    text = torch.empty(total + (-total) % 16 + 16, dtype=torch.uint8, device=device)
    if not _stage:
        _stage.extend(torch.empty(_STAGE_BYTES, dtype=torch.uint8, pin_memory=True) for _ in range(2))
    copy_stream = torch.cuda.Stream(device)
    copy_stream.wait_stream(torch.cuda.current_stream(device))
    free = [None, None]                                                  # event: the block's last copy has left the host
    bases, heads, o, k = [], [], 0, 0
    for p, s in zip(paths, sizes):
        bases.append(o)
        last = 0x0A
        with open(p, "rb") as f:
            done = 0
            while done < s:
                blk = _stage[k & 1]
                if free[k & 1] is not None:
                    free[k & 1].synchronize()
                got = f.readinto(memoryview(blk.numpy())[:min(_STAGE_BYTES, s - done)])
                if not got:
                    raise IOError("short read of %s" % p)
                if done == 0:
                    heads.append(bytes(blk.numpy()[:min(got, 1 << 16)]))
                last = int(blk[got - 1])
                with torch.cuda.stream(copy_stream):
                    text[o:o + got].copy_(blk[:got], non_blocking=True)
                    ev = torch.cuda.Event(); ev.record(copy_stream); free[k & 1] = ev
                o += got; done += got; k += 1
        if s == 0:
            heads.append(b"")
        if last != 0x0A:
            with torch.cuda.stream(copy_stream):
                text[o:o + 1].fill_(0x0A)
            o += 1
    with torch.cuda.stream(copy_stream):
        text[o:].fill_(0x0A)
    torch.cuda.current_stream(device).wait_stream(copy_stream)
    return text, o, bases, heads


def _first_line(head):
    """(offset, bytes) of the first non-empty line of a file, from its first 64 KB (host; header / column count only)"""
    o = 0
    while o < len(head):
        nl = head.find(b"\n", o)
        if nl < 0:
            nl = len(head)
        line = head[o:nl]
        if line.endswith(b"\r"):
            line = line[:-1]
        if line:
            return o, line
        o = nl + 1
    return len(head), b""


def _dedup_names(names):
    low = [n.lower() for n in names]
    return [n + str(i) if low.count(n.lower()) > 1 else n for i, n in enumerate(names)]    # Spark appends the position to duplicates


def index_lines(text, n_bytes):
    """device line index -> (row_starts int64[n_rows] device tensor, saw_quote)."""
    dev = text.device
    n_blocks = (n_bytes + _TEXT_BLOCK - 1) // _TEXT_BLOCK
    counts = torch.zeros(n_blocks + 1, dtype=torch.int32, device=dev)
    flags = torch.zeros(1, dtype=torch.int64, device=dev)
    call("b200flow_csv_count_lines", ptr(text), n_bytes, ptr(counts), ptr(flags))
    bases = torch.cumsum(counts, 0, dtype=torch.int64)                     # inclusive; exclusive = shifted
    head = torch.cat([bases[-1:], flags]).cpu()
    n_rows, saw_quote = int(head[0]), bool(head[1] & 1)
    ex = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), bases[:-1]])
    row_starts = torch.empty(max(n_rows, 1), dtype=torch.int64, device=dev)
    call("b200flow_csv_line_starts", ptr(text), n_bytes, ptr(ex), ptr(row_starts))
    return row_starts[:n_rows], saw_quote


def _new_bad(dev):
    bad = torch.zeros(8, dtype=torch.int64, device=dev)
    bad[1] = -1; bad[5] = -1                                                # ~0 as uint64: the "first offender" minima
    return bad


def _raise_bad(bad, names, what):
    b = bad.cpu().numpy().view(np.uint64)
    if b[0]:
        raise CsvFormatError("%s: %d row(s) do not have %d fields (first: data row %d)" % (what, int(b[0]), len(names), int(b[1])))
    if b[2]:
        raise CsvFormatError("%s: %d row(s) are longer than 4096 bytes" % (what, int(b[2])))
    if b[3] or b[4]:
        r, c = int(b[5] >> np.uint64(16)), int(b[5] & np.uint64(0xFFFF))
        raise CsvFormatError("%s: %d field(s) do not parse as their column's type and %d numeric literal(s) are outside the exact "
                             "converter's range (first: data row %d, column %r)" % (what, int(b[3]), int(b[4]), r, names[c] if c < len(names) else c))
    if b[7]:
        raise CsvFormatError("%s: %d string field(s) collide in the 64-bit dictionary hash" % (what, int(b[7])))


def read_csv(paths, header=False, infer_schema=False, strip_lead=False, strip_trail=False, device=None, stats=None, shard=None):
    """-> (records uint8[n_rows, row_bytes] on the device, RecordSchema, {string column: [values in order of first appearance]})
    stats (optional dict): receives the wall time of each phase in seconds (adds a device synchronize per phase).
    shard = (rank, world): one process per GPU — the line index, the column types and the dictionaries come from ALL rows
    (every rank gets the same schema and codes), but only this rank's contiguous block of rows is converted and returned."""
    import time
    require_cuda()
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    paths = list(paths)
    t_last = [time.perf_counter()]

    def lap(name):
        if stats is not None:
            torch.cuda.synchronize(dev)
            now = time.perf_counter()
            stats[name] = stats.get(name, 0.0) + now - t_last[0]
            t_last[0] = now

    text, n_bytes, bases, heads = _load_text(paths, dev)
    lap("read_files_h2d_s")
    flags = (1 if strip_lead else 0) | (2 if strip_trail else 0)
    row_starts, saw_quote = index_lines(text, n_bytes)
    lap("line_index_s")
    if saw_quote:
        raise CsvFormatError("quoted fields are not supported by the device CSV reader (use option('b200flow.csvEngine', 'host'))")
    first = [(b + o, ln) for b, (o, ln) in zip(bases, (_first_line(h) for h in heads))]
    lead = next((ln for _, ln in first if ln), b"")
    if header:
        names = [c.decode("utf-8", "replace") for c in lead.split(b",")]
        names = [c.strip() if (strip_lead or strip_trail) else c for c in names]
        names = _dedup_names(names)
        hdr = torch.tensor([o for o, ln in first if ln], dtype=torch.int64, device=dev)
        if hdr.numel():
            row_starts = row_starts[~torch.isin(row_starts, hdr)].contiguous()            # every file's own header line
    else:
        names = ["_c%d" % i for i in range(len(lead.split(b",")) if lead else 0)]
    n_cols, n_rows = len(names), int(row_starts.shape[0])
    if n_cols == 0:
        return torch.empty((0, 4), dtype=torch.uint8, device=dev), RecordSchema([]), {}
    if n_cols > 1024:
        raise CsvFormatError("more than 1024 columns")

    # ---- column types: Spark's inference order null < int < long < double < string
    if infer_schema and n_rows:
        cls = torch.zeros(2 * n_cols, dtype=torch.int32, device=dev)
        bad = _new_bad(dev)
        call("b200flow_csv_infer", ptr(text), n_bytes, ptr(row_starts), n_rows, n_cols, flags, ptr(cls), ptr(cls[n_cols:]), ptr(bad))
        _raise_bad(bad, names, "inferSchema")
        cls = cls.cpu().numpy()
        col_class, col_null = cls[:n_cols], cls[n_cols:]
    else:
        col_class, col_null = np.full(n_cols, CSV_STRING, np.int32), np.zeros(n_cols, np.int32)
    lap("infer_schema_s")
    fields, cols = [], np.zeros(n_cols, COL_DTYPE)
    str_cols = []
    for c, name in enumerate(names):
        k = int(col_class[c])
        if k == CSV_INT32 and not col_null[c]:
            typ, ctype = "i32", CSV_INT32
        elif k in (CSV_INT32, CSV_INT64, CSV_DOUBLE):
            typ, ctype = "f64", CSV_DOUBLE                                   # nullable ints and longs are read as doubles (null -> NaN)
        else:
            typ, ctype = "code", CSV_STRING                                  # strings, and columns that are empty everywhere
            str_cols.append(c)
        fields.append((name, typ))
        cols[c]["type"] = ctype
        cols[c]["str_index"] = len(str_cols) - 1 if ctype == CSV_STRING else -1
    schema = RecordSchema(fields)
    for c, name in enumerate(names):
        cols[c]["rec_off"] = schema.offsets[name]
    cols_d = torch.from_numpy(cols.view(np.uint8)).to(dev)

    # ---- string dictionaries: hash tables on the device, one host read of the distinct values
    dicts, keys, pos_len, slot_code, cap_log2 = {}, None, None, None, 4
    if str_cols and n_rows:
        cap_log2 = 12
        while True:
            keys = torch.zeros((len(str_cols), 1 << cap_log2), dtype=torch.int64, device=dev)
            pos_len = torch.full((len(str_cols), 1 << cap_log2), _I64_MAX, dtype=torch.int64, device=dev)
            bad = _new_bad(dev)
            call("b200flow_csv_dictionary", ptr(text), n_bytes, ptr(row_starts), n_rows, n_cols, flags, ptr(cols_d), ptr(keys), ptr(pos_len),
                 cap_log2, ptr(bad))
            occ = (keys != 0)
            full = int(bad[6].item()) or int(occ.sum(1).max().item()) > (1 << cap_log2) // 2
            if not full:
                break
            cap_log2 += 3
            if cap_log2 > 26:
                raise CsvFormatError("a string column has more than 2^25 distinct values")
        _raise_bad(bad, names, "dictionary")
        occ_h, pl_h = occ.cpu().numpy(), pos_len.cpu().numpy()
        code_h = np.full(occ_h.shape, -1, np.int32)
        # the distinct values' bytes: one gather on the device, one copy back
        v_all = pl_h[occ_h]
        lens = (v_all & 0xFFFF).astype(np.int64)
        ends_ = np.cumsum(lens)
        idx = np.repeat((v_all >> 16) - (ends_ - lens), lens) + np.arange(int(ends_[-1]) if len(ends_) else 0)
        blob = text[torch.from_numpy(idx).to(dev)].cpu().numpy().tobytes() if len(idx) else b""
        at = dict(zip(v_all.tolist(), (ends_ - lens).tolist()))
        for si, c in enumerate(str_cols):
            slots = np.nonzero(occ_h[si])[0]
            slots = slots[np.argsort(pl_h[si, slots], kind="stable")]        # order of first appearance in the file(s)
            values, code_of = [], {}
            for sl in slots:
                v = int(pl_h[si, sl]); ln = v & 0xFFFF
                s = blob[at[v]:at[v] + ln].decode("utf-8", "replace")
                if s not in code_of:
                    code_of[s] = len(values); values.append(s)
                code_h[si, sl] = code_of[s]
            dicts[names[c]] = values
        slot_code = torch.from_numpy(code_h).to(dev)
    for c in str_cols:
        dicts.setdefault(names[c], [])

    lap("dictionaries_s")
    if shard is not None:
        from .dist import shard_bounds
        lo, hi = shard_bounds(n_rows, int(shard[0]), int(shard[1]))
        row_starts = row_starts[lo:hi].contiguous()
        n_rows = hi - lo
    # ---- fields -> records
    rec = torch.zeros((max(n_rows, 1), schema.row_bytes), dtype=torch.uint8, device=dev)
    if n_rows:
        bad = _new_bad(dev)
        call("b200flow_csv_parse", ptr(text), n_bytes, ptr(row_starts), n_rows, n_cols, flags, ptr(cols_d), ptr(keys), ptr(pos_len), ptr(slot_code),
             cap_log2, ptr(rec), schema.row_bytes, ptr(bad))
        _raise_bad(bad, names, "parse")
    lap("parse_s")
    return rec[:n_rows], schema, dicts
