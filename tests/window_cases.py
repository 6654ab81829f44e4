"""Window functions for the tests: a per-row restatement of DESIGN.md §6 (viii), an input table with ties, NULLs, one-row
partitions and a partition holding most rows, and the stage plans that run a window node.

The restatement works on Python values as pyarrow returns them (int, Decimal, float, str, bool, date) and computes exactly:
integers and decimals with Python integers, float sums with math.fsum.  Rows come out in input order with one value per
window expression, as the operator appends its columns."""
from __future__ import annotations

import datetime
import decimal
import functools
import math
import struct
from typing import Any, Dict, List, Optional, Sequence

import numpy as np
import pyarrow as pa

from ballista_b200 import plan as P

c = P.col

SCHEMA = [P.field("rid", "i64"), P.field("g", "i32", True), P.field("h", "utf8", True), P.field("o", "i64", True),
          P.field("ks", "utf8", True), P.field("i32", "i32", True), P.field("i64", "i64", True), P.field("u64", "u64", True),
          P.field("dec", P.dec(12, 2), True), P.field("f64", "f64", True), P.field("dt", "date32", True), P.field("b", "bool", True)]
TYPES = {f["name"]: f["type"] for f in SCHEMA}


def make_table(n: int, seed: int, n_groups: int = 7, null_frac: float = 0.1) -> pa.Table:
    """n rows.  g: n_groups partition ids, skewed so that one holds most rows, plus one-row partitions; o: an order key with
    many ties; every value column about `null_frac` NULL."""
    rng = np.random.default_rng(seed)

    def nulls():
        return rng.random(n) < null_frac

    def arr(values, typ, nf=null_frac):
        m = rng.random(n) < nf
        return pa.array([None if m[i] else values[i] for i in range(n)], type=typ)

    g = [int(x) for x in np.minimum(rng.geometric(0.6, n) - 1, n_groups - 1)]
    for i in range(min(n, 3)):
        g[i] = 1000 + i  # one-row partitions
    words = ["", "a", "AIR", "MAIL", "TRUCK", "longer than seven", "é"]
    h = [words[int(x)] for x in rng.integers(0, 3, n)]
    o = [int(x) for x in rng.integers(0, max(2, n // 8), n)]
    ks = ["".join(chr(97 + int(k)) for k in rng.integers(0, 3, int(rng.integers(0, 3)))) for _ in range(n)]
    i32 = [int(x) for x in rng.integers(-2 ** 31, 2 ** 31, n)]
    i64 = [int(x) for x in rng.integers(-10 ** 15, 10 ** 15, n)]
    u64 = [int(x) for x in rng.integers(0, 2 ** 63, n, dtype=np.uint64) * 2 + rng.integers(0, 2, n, dtype=np.uint64)]
    dec = [decimal.Decimal(int(x)).scaleb(-2) for x in rng.integers(-10 ** 9, 10 ** 9, n)]
    f64 = [float(x) for x in rng.normal(0, 1e6, n)]
    dt = [int(x) for x in rng.integers(8000, 12000, n)]
    b = [bool(x) for x in rng.integers(0, 2, n)]
    cols = [pa.array(list(range(n)), pa.int64()), arr(g, pa.int32(), 0.05), arr(h, pa.string(), 0.05), arr(o, pa.int64(), 0.05),
            arr(ks, pa.string()), arr(i32, pa.int32()), arr(i64, pa.int64()), arr(u64, pa.uint64()), arr(dec, pa.decimal128(12, 2)),
            arr(f64, pa.float64()), arr(dt, pa.int32()).cast(pa.date32()), arr(b, pa.bool_())]
    return pa.Table.from_arrays(cols, names=[f["name"] for f in SCHEMA])


def register(e, name: str, table: pa.Table, parts: int = 1) -> None:
    e.drop_table(name)
    step = max((table.num_rows + parts - 1) // parts, 1)
    for p in range(parts):
        sl = table.slice(min(table.num_rows, p * step), step).combine_chunks()
        batch = sl.to_batches()[0] if sl.num_rows else pa.RecordBatch.from_arrays(
            [pa.array([], type=f.type) for f in table.schema], schema=table.schema)
        e.register_batch(name, p, batch)


def stages(plan) -> List[P.Stage]:
    return [P.Stage(1, P.shuffle_writer(plan, 1))]


# ---- the restatement -------------------------------------------------------------------------------------------------
def _f64_key(v: float) -> int:
    b = struct.unpack("<q", struct.pack("<d", v))[0]
    return b ^ ((b >> 63) & 0x7FFFFFFFFFFFFFFF)


def _value_key(v):
    if isinstance(v, float):
        return _f64_key(v)
    if isinstance(v, str):
        return v.encode()
    if isinstance(v, bool):
        return int(v)
    return v


def _cmp_key(a, b, asc: bool, nulls_first: bool) -> int:
    if a is None or b is None:
        if a is None and b is None:
            return 0
        return (-1 if a is None else 1) * (1 if nulls_first else -1)
    ka, kb = _value_key(a), _value_key(b)
    c_ = (ka > kb) - (ka < kb)
    return c_ if asc else -c_


def _same(a, b) -> bool:
    return (a is None and b is None) or (a is not None and b is not None and _value_key(a) == _value_key(b))


def _frame(frame: Optional[dict], i: int, ps: int, pe: int, qs: int, qe: int):
    frame = frame or P.range_(P.UNBOUNDED_PRECEDING, P.CURRENT_ROW)
    rows = frame["units"] == "rows"
    s, e = frame["start"], frame["end"]
    fs = {"unbounded_preceding": ps, "preceding": i - s.get("n", 0), "current_row": i if rows else qs,
          "following": i + s.get("n", 0)}[s["kind"]]
    fe = {"unbounded_following": pe, "preceding": i - e.get("n", 0) + 1, "current_row": i + 1 if rows else qe,
          "following": i + e.get("n", 0) + 1}[e["kind"]]
    fs, fe = min(max(fs, ps), pe), min(max(fe, ps), pe)
    return fs, max(fe, fs)


def _wrap64(v: int, signed: bool) -> int:
    v &= (1 << 64) - 1
    return v - (1 << 64) if signed and v >= 1 << 63 else v


def _dec_scale(t) -> int:
    return t["dec"][1]


def _agg(fn: str, vals: List[Any], typ, count_star: bool):
    if fn == "count":
        return len(vals) if count_star else sum(v is not None for v in vals)
    xs = [v for v in vals if v is not None]
    if not xs:
        return None
    if fn in ("min", "max"):
        best = xs[0]
        for v in xs[1:]:
            if (_value_key(v) < _value_key(best)) if fn == "min" else (_value_key(v) > _value_key(best)):
                best = v
        return best
    if isinstance(typ, dict):  # Decimal128: exact unscaled arithmetic
        s = _dec_scale(typ)
        tot = sum(int(v.scaleb(s)) for v in xs)
        if fn == "sum":
            return decimal.Decimal(tot).scaleb(-s)
        rs = min(38, s + 4)
        q = abs(tot) * 10 ** (rs - s) // len(xs)
        return decimal.Decimal(q if tot >= 0 else -q).scaleb(-rs)
    if typ == "f64" or fn == "avg":
        tot = math.fsum(float(v) for v in xs)
        return tot if fn == "sum" else tot / len(xs)
    return _wrap64(sum(xs), typ != "u64")


def evaluate(table: pa.Table, exprs: Sequence[dict], partition: Sequence[str], order: Sequence[tuple]) -> Dict[str, list]:
    """The window values of every row, in input order.  partition: column names; order: (name, asc, nulls_first)."""
    cols = {n: table.column(n).to_pylist() for n in table.column_names}
    n = table.num_rows

    def cmp(a, b):
        for p_ in partition:
            r = _cmp_key(cols[p_][a], cols[p_][b], True, False)
            if r:
                return r
        for name, asc, nf in order:
            r = _cmp_key(cols[name][a], cols[name][b], asc, nf)
            if r:
                return r
        return (a > b) - (a < b)  # stable: ties keep their input order

    idx = sorted(range(n), key=functools.cmp_to_key(cmp))
    out = {w["name"]: [None] * n for w in exprs}
    i = 0
    while i < n:
        j = i
        while j < n and all(_same(cols[p_][idx[j]], cols[p_][idx[i]]) for p_ in partition):
            j += 1
        part = idx[i:j]
        rows = len(part)
        # peer groups
        starts = [0]
        for k in range(1, rows):
            if not all(_same(cols[name][part[k]], cols[name][part[k - 1]]) for name, _, _ in order):
                starts.append(k)
        bounds = starts + [rows]
        peer_of = [0] * rows
        for gi in range(len(starts)):
            for k in range(bounds[gi], bounds[gi + 1]):
                peer_of[k] = gi
        for k in range(rows):
            gi = peer_of[k]
            qs, qe = bounds[gi], bounds[gi + 1]
            r = part[k]
            for w in exprs:
                fn, args = w["fn"], w.get("args", [])
                if fn == "row_number":
                    v = k + 1
                elif fn == "rank":
                    v = qs + 1
                elif fn == "dense_rank":
                    v = gi + 1
                elif fn == "percent_rank":
                    v = qs / (rows - 1) if rows > 1 else 0.0
                elif fn == "cume_dist":
                    v = qe / rows
                elif fn == "ntile":
                    nb = args[0]["lit"]["v"]
                    q, rem = divmod(rows, nb)
                    big = rem * (q + 1)
                    v = (k // (q + 1) if k < big else rem + (k - big) // q) + 1
                elif fn in ("lag", "lead"):
                    off = args[1]["lit"]["v"] if len(args) > 1 else 1
                    d = args[2]["lit"]["v"] if len(args) > 2 else None
                    j2 = k - off if fn == "lag" else k + off
                    v = cols[args[0]["col"]][part[j2]] if 0 <= j2 < rows else _lit_value(d, TYPES.get(args[0]["col"]))
                else:
                    fs, fe = _frame(w.get("frame"), k, 0, rows, qs, qe)
                    frame_rows = part[fs:fe]
                    if fn == "first_value":
                        v = cols[args[0]["col"]][frame_rows[0]] if frame_rows else None
                    elif fn == "last_value":
                        v = cols[args[0]["col"]][frame_rows[-1]] if frame_rows else None
                    elif fn == "nth_value":
                        m = args[1]["lit"]["v"]
                        v = cols[args[0]["col"]][frame_rows[m - 1]] if len(frame_rows) >= m else None
                    else:
                        name = args[0]["col"] if args and "col" in args[0] else None
                        vals = [cols[name][x] for x in frame_rows] if name else [1] * len(frame_rows)
                        v = _agg(fn, vals, TYPES.get(name, "i64"), name is None)
                out[w["name"]][r] = v
        i = j
    return out


def _lit_value(v, typ):
    if v is None:
        return None
    if typ == "date32":
        return datetime.date(1970, 1, 1) + datetime.timedelta(days=v)
    if isinstance(typ, dict):
        return decimal.Decimal(int(v)).scaleb(-typ["dec"][1])
    return v


def frame_abs_sum(table: pa.Table, w: dict, partition, order) -> Dict[int, tuple]:
    """For a float SUM / AVG: per input row, (m, Σ|x|) over the frame's non-NULL values -- the error bound's inputs."""
    name = w["args"][0]["col"]
    absw = dict(w, fn="sum", name="__abs")
    t2 = table.set_column(table.column_names.index(name), name,
                          pa.array([None if v is None else abs(float(v)) for v in table.column(name).to_pylist()], pa.float64()))
    cnt = dict(w, fn="count", name="__cnt")
    types = dict(TYPES)
    TYPES[name] = "f64"
    try:
        ev = evaluate(t2, [absw, cnt], partition, order)
    finally:
        TYPES.clear()
        TYPES.update(types)
    return {i: (ev["__cnt"][i], ev["__abs"][i] or 0.0) for i in range(table.num_rows)}
