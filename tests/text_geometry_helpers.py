"""Builders and readers for tests/test_text_geometry_gpu.py: the kernels' geometry constants re-read from the sources, CSV and JSON
files with records planted at exact byte offsets, frames whose rows have chosen text lengths, and the launch records of a write."""
from __future__ import annotations

import os
import re

import numpy as np

import csv_oracle as co

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "rust-dataframe_b200", "csrc")

THREAD, WARP, CTA = 16, 512, 4096      # bytes of a tokenizer / newline-pass thread, warp and CTA
STATE_NAMES = {co.SR: "StartRecord", co.SF: "StartField", co.IF: "InField", co.IQ: "InQuoted", co.QQ: "QuoteInQuoted"}
CLASSES = {"delim": b",", "quote": b'"', "cr": b"\r", "lf": b"\n", "other": None}
U8, U32, U64 = 4, 6, 7   # BDF dtype ids in the launch records


# ---- constants from the sources ------------------------------------------------------------------------------------

def source(name: str) -> str:
    with open(os.path.join(CSRC, name)) as fh:
        return fh.read()


def constant(text: str, name: str, env: dict) -> int:
    """The value of `constexpr ... name = <expr>;` in text, its casts and integer suffixes dropped, names from env."""
    m = re.search(r"\b" + name + r"\s*=\s*([^;]+);", text)
    assert m, name
    expr = re.sub(r"\((?:size_t|int64_t|unsigned|int|long long)\)", "", m.group(1))
    expr = re.sub(r"\b(\d+)(?:u|ull|ll|LL)\b", r"\1", expr)
    return int(eval(expr, {"__builtins__": {}}, dict(env)))


# ---- CSV files with planted bytes -----------------------------------------------------------------------------------

def classify(b: int) -> str:
    return {ord(","): "delim", ord('"'): "quote", 13: "cr", 10: "lf"}.get(b, "other")


def pair_record(state: int, cls: str, i: int, c: int):
    """(before, after, id, check) of one `id,p,check` record such that the DFA is in `state` after `before` and the first byte of
    `after` is of class `cls`.  A record whose id or check is empty gives None there."""
    I, C = b"%d" % i, b"%d" % c
    t = {
        (co.SR, "delim"): (b"", b",p," + C + b"\n", None, c),
        (co.SR, "quote"): (b"", b'"' + I + b'",p,' + C + b"\n", i, c),
        (co.SR, "cr"): (b"", b"\r\n" + I + b",p," + C + b"\n", i, c),
        (co.SR, "lf"): (b"", b"\n" + I + b",p," + C + b"\n", i, c),
        (co.SR, "other"): (b"", I + b",p," + C + b"\n", i, c),
        (co.SF, "delim"): (I + b",", b"," + C + b"\n", i, c),
        (co.SF, "quote"): (I + b",", b'"p",' + C + b"\n", i, c),
        (co.SF, "cr"): (I + b",p,", b"\r\n", i, None),
        (co.SF, "lf"): (I + b",p,", b"\n", i, None),
        (co.SF, "other"): (I + b",", b"p," + C + b"\n", i, c),
        (co.IF, "delim"): (I, b",p," + C + b"\n", i, c),
        (co.IF, "quote"): (I + b",a", b'"b,' + C + b"\n", i, c),
        (co.IF, "cr"): (I + b",p," + C, b"\r\n", i, c),
        (co.IF, "lf"): (I + b",p," + C, b"\n", i, c),
        (co.IF, "other"): (I + b",a", b"b," + C + b"\n", i, c),
        (co.IQ, "delim"): (I + b',"a', b',b",' + C + b"\n", i, c),
        (co.IQ, "quote"): (I + b',"ab', b'",' + C + b"\n", i, c),
        (co.IQ, "cr"): (I + b',"a', b'\rb",' + C + b"\n", i, c),
        (co.IQ, "lf"): (I + b',"a', b'\nb",' + C + b"\n", i, c),
        (co.IQ, "other"): (I + b',"a', b'b",' + C + b"\n", i, c),
        (co.QQ, "delim"): (I + b',"ab"', b"," + C + b"\n", i, c),
        (co.QQ, "quote"): (I + b',"a"', b'"b",' + C + b"\n", i, c),
        (co.QQ, "cr"): (I + b',p,"' + C + b'"', b"\r\n", i, c),
        (co.QQ, "lf"): (I + b',p,"' + C + b'"', b"\n", i, c),
        (co.QQ, "other"): (I + b',"a"', b"b," + C + b"\n", i, c),
        # beyond the 25 pairs: a CRLF split by the edge, and a "" escape whose first quote starts the unit
        ("crlf", "lf"): (I + b",p," + C + b"\r", b"\n", i, c),
        ("escape", "quote"): (I + b',"a', b'""b",' + C + b"\n", i, c),
    }
    return t[(state, cls)]


PAIRS = [(s, k) for s in (co.SR, co.SF, co.IF, co.IQ, co.QQ) for k in CLASSES] + [("crlf", "lf"), ("escape", "quote")]
PAIR_STATE = {"crlf": co.SR, "escape": co.IQ}


def edge_kind(off: int) -> str:
    return "cta" if off % CTA == 0 else "warp" if off % WARP == 0 else "thread" if off % THREAD == 0 else "none"


class CsvPlan:
    """An `id,p,check` file built record by record: filler records of any length, and records planted so that one byte lands on an
    exact offset.  ids and checks are unique Int64 values, so a shifted field shows in either column."""

    def __init__(self, header: bool = True):
        self.buf = bytearray(b"id,p,check\n" if header else b"")
        self.header = header
        self.ids, self.checks, self.starts = [], [], []
        self.plants = []   # (edge offset, state, class, start of the previous record, end of the planted record, id, check)
        self.n = 0

    def _next(self):
        self.n += 1
        return self.n, 3 * self.n + 1

    def _add(self, rec: bytes, i, c):
        self.starts.append(len(self.buf))
        self.buf += rec
        self.ids.append(i)
        self.checks.append(c)

    def fill_to(self, target: int, long_ok: bool = True):
        """Filler records `id,xxx,check` up to exactly `target` bytes."""
        while target - len(self.buf) > 300:
            i, c = self._next()
            self._add(b"%d,%s,%d\n" % (i, b"x" * (100 if long_ok else 40), c), i, c)
        i, c = self._next()
        base = len(b"%d,,%d\n" % (i, c))
        k = target - len(self.buf) - base
        assert k >= 0, (target, len(self.buf))
        self._add(b"%d,%s,%d\n" % (i, b"x" * k, c), i, c)

    def plant_at(self, edge: int, state, cls: str):
        i, c = self._next()
        before, after, pi, pc = pair_record(state, cls, i, c)
        self.fill_to(edge - len(before))
        prev = self.starts[-1]
        self._add(before + after, pi, pc)
        self.plants.append((edge, state, cls, prev, len(self.buf), pi, pc))

    def next_edge(self, kind: str, rng, gap: int = 40) -> int:
        unit = {"thread": THREAD, "warp": WARP, "cta": CTA}[kind]
        e = (len(self.buf) + gap + 30 + int(rng.integers(0, 3 * unit if kind == "thread" else 1)) + unit - 1) // unit * unit
        while edge_kind(e) != kind:
            e += unit
        return e

    @property
    def rows(self):
        return len(self.ids)

    def fields(self):
        return 3 * (self.rows + (1 if self.header else 0))

    def check_plants(self):
        """Each planted byte is where it was meant to be, the DFA state before it is the one named (csv_oracle.states from the
        previous record's start, where the state is StartRecord), and csv_oracle.records reads the planted record as built."""
        data = bytes(self.buf)
        for edge, state, cls, prev, end, pi, pc in self.plants:
            st = co.states(data[prev:edge + 1])
            assert st[edge - prev] == PAIR_STATE.get(state, state), (edge, state, cls)
            if state == "crlf":
                assert data[edge - 1] == 13 and data[edge] == 10
            assert classify(data[edge]) == cls, (edge, state, cls)
            recs = co.records(data[prev:end])
            want = [b"" if pi is None else b"%d" % pi, b"" if pc is None else b"%d" % pc]
            assert [recs[-1][0], recs[-1][2]] == want and len(recs[-1]) == 3, (edge, state, cls, recs[-1])


# ---- frames whose rows have chosen text lengths ----------------------------------------------------------------------

def int_columns(extras, ncols: int, salt: int = 0):
    """ncols Int64 columns, row r's values together 18 * ncols + extras[r] characters long (extras[r] <= 2 * ncols): each value
    is 10^17 + x (18 digits), 10^18 + x (19) or -(10^18 + x) (20), x unique per value."""
    extras = np.asarray(extras, np.int64)
    n = extras.size
    x = (np.arange(n, dtype=np.int64)[:, None] * ncols + np.arange(ncols) + salt * 7919).astype(np.int64)
    left = extras.copy()
    cols = []
    for j in range(ncols):
        e = np.minimum(left, 2)
        left -= e
        v = np.where(e == 0, 10 ** 17 + x[:, j], 10 ** 18 + x[:, j])
        cols.append(np.where(e == 2, -v, v).astype(np.int64))
    assert (left == 0).all()
    return cols


def cta_extras(base: int, rows_per_cta: int = 256):
    """Per-row extra characters for: three CTAs whose text is 24575, 24576 and 24577 bytes, then 17 CTAs one byte longer than
    `base` * rows (so, from a 16-byte aligned start, every CTA after them starts one byte further into the 16-byte word)."""
    out = []
    for t in (24575, 24576, 24577):
        e = t - base * rows_per_cta
        q, r = divmod(e, rows_per_cta)
        out += [q + 1] * r + [q] * (rows_per_cta - r)
    for _ in range(17):
        out += [1] + [0] * (rows_per_cta - 1)
    return out


def cta_texts(text: bytes, rows_per_cta: int = 256):
    """The byte length of each CTA's rows in a text of newline-ended rows."""
    lens = np.array([len(x) + 1 for x in text.split(b"\n")[:-1]], np.int64)
    return [int(lens[s:s + rows_per_cta].sum()) for s in range(0, lens.size, rows_per_cta)]


# ---- launch records -------------------------------------------------------------------------------------------------

def recorded(ctx, kernel: str, fn):
    """fn() with launch records on: the records of `kernel`."""
    ctx.synchronize()
    ctx.profile_read()
    ctx.profile_enable(True)
    try:
        fn()
        ctx.synchronize()
        return [r for r in ctx.profile_read() if r["kernel"] == kernel]
    finally:
        ctx.profile_enable(False)


def csv_write_blocks(recs):
    """(rows, text bytes) of each block of a CSV write: its emit record (BDF_U8) counts 8 bytes a row plus the text."""
    return [(r["rows"], r["bytes"] - 8 * r["rows"]) for r in recs if r["dtype"] == U8]


def json_write_blocks(recs):
    """(rows, text bytes) of each block of a JSON write: the row emit records (BDF_U8 with the text's bytes; element emits count 0)."""
    return [(r["rows"], r["bytes"]) for r in recs if r["dtype"] == U8 and r["bytes"] > 0]


def json_write_windows(recs):
    """Rows of each window of a JSON write: the row measure (BDF_U64) two records before each cut (-1 after the row scan, BDF_U32)."""
    return [recs[i - 2]["rows"] for i in range(2, len(recs)) if recs[i]["dtype"] == -1 and recs[i - 1]["dtype"] == U32 and recs[i - 2]["dtype"] == U64]


# ---- device columns to host ------------------------------------------------------------------------------------------

def host(col):
    """(values as bit patterns, valid mask, [chunk lengths], [has a bitmap]) of a device column."""
    vals, valid, lens, hv = [], [], [], []
    for a in col.download():
        m = a.valid_mask()
        if hasattr(a, "value_bits"):
            v = np.asarray(a.value_bits(), dtype=bool)
        else:
            v = np.asarray(a.value_slice())
            if v.dtype.kind == "f":
                v = v.view(f"u{v.dtype.itemsize}")
        vals.append(v); valid.append(np.asarray(m, dtype=bool)); lens.append(a.length); hv.append(a.validity is not None)
    return np.concatenate(vals), np.concatenate(valid), lens, hv


def list_host(lc):
    """(rows: None or [element bits or None], [chunk lengths], [has a bitmap]) of a device list column."""
    rows, lens, hv = [], [], []
    for ch in lc.download():
        lens.append(ch.length)
        hv.append(ch.validity is not None)
        vals = np.asarray(ch.values.value_slice())
        if vals.dtype.kind == "f":
            vals = vals.view(f"u{vals.dtype.itemsize}")
        vm = ch.values.valid_mask()
        lm = [True] * ch.length if ch.validity is None else [bool((ch.validity[k >> 3] >> (k & 7)) & 1) for k in range(ch.length)]
        assert ch.offsets[0] == 0
        for k in range(ch.length):
            s, e = int(ch.offsets[k]), int(ch.offsets[k + 1])
            rows.append(None if not lm[k] else [int(vals[j]) if vm[j] else None for j in range(s, e)])
    return rows, lens, hv
