"""Shared by the AggregateExec tests: input columns of every type the engine aggregates, at the edges of each type; the
stage plans that run COUNT(*), COUNT, SUM, AVG, MIN and MAX in every aggregate mode; and a plain-Python reference of
what they return, written from the rules below and sharing nothing with plan.hpp or the CPU oracle.

Values are carried "raw": integers, dates and timestamps as Python ints, decimals as their unscaled ints, floats as
their bit patterns, booleans as bools, strings as str.

Rules (DataFusion's, [EXT] where DESIGN §6 says so):
- Result types: COUNT is Int64; SUM(signed int) Int64, SUM(unsigned) UInt64, SUM(float) Float64, SUM(Decimal(p, s))
  Decimal(min(38, p + 10), s); AVG(decimal) Decimal(min(38, p + 4), min(38, s + 4)), AVG(anything else) Float64; MIN
  and MAX keep the argument's type.
- Integer and decimal SUMs wrap (add_wrapping): to 64 bits, to 128 bits for decimals.
- Decimal AVG is sum * 10^k // count truncated toward zero (k = result scale - input scale); it fails when sum * 10^k
  leaves the i128 range or when the quotient has more digits than the result precision.
- Float SUM and AVG are exact here (fractions); the device may differ by the order-independent bound
  (n - 1) * u * sum|x| (over the count for AVG, plus the division's half ulp).  A NaN, or +inf with -inf, gives NaN.
- Float MIN and MAX follow the IEEE total order of the bit patterns: NaN above +inf, -0.0 below 0.0, NaNs ordered by
  sign and payload.
- Group keys are equal when their bit patterns are (floats), their UTF-8 bytes are (strings), their unscaled values
  are (decimals); NULL is a group of its own.
- A group whose argument is all NULL gives NULL for SUM, AVG, MIN and MAX and 0 for COUNT.  An empty input gives one
  row without keys and no rows with keys."""
from __future__ import annotations

import decimal
import json
import random
import struct
from fractions import Fraction

import numpy as np
import pyarrow as pa

from ballista_b200 import driver, engine
from ballista_b200 import plan as P

c = P.col
_EXACT = decimal.Context(prec=80)   # the default 28 digits would round 29- to 38-digit decimals

_NAN_BITS64 = [0x7FF8000000000000, 0x7FF8000000000123, 0xFFF8000000000000, 0xFFF80000000000A5, 0x7FF0000000000001]
_NAN_BITS32 = [0x7FC00000, 0x7FC00123, 0xFFC00000, 0xFFC000A5, 0x7F800001]


def _f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def _f32_bits(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


# F32_EDGES holds a signalling NaN, 0x7F800001: widened by the hardware it would become the Float64 of 0x7FC00001
# specials shared by both float widths, as values (the NaNs are added as bit patterns above)
_FLOAT_SPECIALS = [0.0, -0.0, float("inf"), float("-inf"), 5e-324, -5e-324, 2.0 ** 53 + 2, 2.0 ** 53, -(2.0 ** 53),
                   1.5, -2.25, 1e300, -1e300, 1e-310]
F64_EDGES = sorted({_f64_bits(x) for x in _FLOAT_SPECIALS} | {_f64_bits(2.0 ** 53 - 1), _f64_bits(2.0 ** 53 + 1)}) + _NAN_BITS64
F32_EDGES = sorted({_f32_bits(x) for x in [0.0, -0.0, float("inf"), float("-inf"), 1.5, -2.25, 2.0 ** 24, 3e38, -3e38]}
                   | {0x00000001, 0x80000001, 0x4B800001}) + _NAN_BITS32

# name -> (kind, arrow type, IR type, precision/scale or bits, edge values)
TYPES = {
    "i8": ("int", pa.int8(), "i8", 8, [-128, 127, -1, 0]),
    "i16": ("int", pa.int16(), "i16", 16, [-32768, 32767, -1]),
    "i32": ("int", pa.int32(), "i32", 32, [-2 ** 31, 2 ** 31 - 1, -1]),
    "i64": ("int", pa.int64(), "i64", 64, [-2 ** 63, 2 ** 63 - 1, -1, 1]),
    "u8": ("uint", pa.uint8(), "u8", 8, [0, 255]),
    "u16": ("uint", pa.uint16(), "u16", 16, [0, 65535]),
    "u32": ("uint", pa.uint32(), "u32", 32, [0, 2 ** 32 - 1, 2 ** 31]),
    "u64": ("uint", pa.uint64(), "u64", 64, [0, 2 ** 64 - 1, 2 ** 63, 2 ** 63 - 1]),
    "f32": ("float", pa.float32(), "f32", 32, F32_EDGES),
    "f64": ("float", pa.float64(), "f64", 64, F64_EDGES),
    "d5_2": ("dec", pa.decimal128(5, 2), P.dec(5, 2), (5, 2), [-99999, 99999, 0, -1]),
    "d15_2": ("dec", pa.decimal128(15, 2), P.dec(15, 2), (15, 2), [-10 ** 15 + 1, 10 ** 15 - 1]),
    "d18_0": ("dec", pa.decimal128(18, 0), P.dec(18, 0), (18, 0), [-10 ** 18 + 1, 10 ** 18 - 1, 2 ** 59]),
    # |x| >= 2^63: the sums carry into and borrow from the high 64 bits with mixed signs
    "d20_3": ("dec", pa.decimal128(20, 3), P.dec(20, 3), (20, 3), [10 ** 20 - 1, -10 ** 20 + 1, 2 ** 64 - 1, -(2 ** 64) + 1, 2 ** 63]),
    "d38_0": ("dec", pa.decimal128(38, 0), P.dec(38, 0), (38, 0), [2 ** 80, -(2 ** 80), 2 ** 64, -(2 ** 64) - 1]),
    "d38_10": ("dec", pa.decimal128(38, 10), P.dec(38, 10), (38, 10), [2 ** 90, -(2 ** 90) + 7, 1, -1]),
    "date32": ("date", pa.date32(), "date32", 32, [-2 ** 31, 2 ** 31 - 1, 0, -1]),
    "ts": ("ts", pa.timestamp("ns"), "ts", 64, [-2 ** 63, 2 ** 63 - 1, 0]),
    "bool": ("bool", pa.bool_(), "bool", 1, [True, False]),
    "utf8": ("utf8", pa.string(), "utf8", 0, ["", "a", "a\0", "abcdefgh", "é", "日本語", "\U0001F600", "zz", "abc"]),
}
# the rows every column puts its edge values at: both sides of the 1024-row tile boundaries, and the last row
EDGE_ROWS = (0, 1, 1022, 1023, 1024, 1025, 2047, 2048)

FORMS = ("nn", "nv", "n")   # non-nullable; nullable without NULLs; nullable with NULLs


def _random_value(kind, bits, rng: random.Random):
    if kind == "int" or kind in ("date", "ts"):
        return rng.randrange(-(1 << (bits - 1)), 1 << (bits - 1))
    if kind == "uint":
        return rng.randrange(0, 1 << bits)
    if kind == "bool":
        return rng.random() < 0.5
    raise AssertionError(kind)


def random_values(t: str, n: int, seed: int):
    """n raw values of type t: edge values at EDGE_ROWS and the last row, random values elsewhere."""
    kind, _at, _it, bits, edges = TYPES[t]
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        if kind == "float":
            if rng.random() < 0.3:
                out.append(rng.choice(edges))
            else:
                x = rng.uniform(-1e6, 1e6) * (10.0 ** rng.randrange(-3, 4))
                out.append(_f64_bits(x) if bits == 64 else _f32_bits(x))
        elif kind == "dec":
            p, _s = bits
            m = min(10 ** p - 1, 2 ** 90)
            out.append(rng.choice(edges) if rng.random() < 0.2 else rng.randrange(-m, m + 1))
        elif kind == "utf8":
            out.append(rng.choice(edges) if rng.random() < 0.5 else "".join(rng.choice("abcxyz\0é") for _ in range(rng.randrange(0, 12))))
        else:
            out.append(rng.choice(edges) if rng.random() < 0.2 else _random_value(kind, bits, rng))
    for k, i in enumerate([r for r in EDGE_ROWS if r < n] + ([n - 1] if n else [])):
        out[i] = edges[k % len(edges)]
    return out


def to_arrow(t: str, vals, nulls=None) -> pa.Array:
    """raw values (None = NULL) -> an Arrow array of type t; nulls: an optional validity override (True = NULL)."""
    kind, at, _it, bits, _e = TYPES[t]
    if nulls is not None:
        vals = [None if m else v for v, m in zip(vals, nulls)]
    mask = np.array([v is None for v in vals], dtype=bool)
    if kind == "float":
        u, f = (np.uint64, np.float64) if bits == 64 else (np.uint32, np.float32)
        return pa.array(np.array([0 if v is None else v for v in vals], dtype=u).view(f), type=at, mask=mask)
    if kind == "dec":
        s = bits[1]
        return pa.array([None if v is None else decimal.Decimal(v).scaleb(-s, _EXACT) for v in vals], type=at)
    if kind in ("date", "ts"):
        return pa.array(vals, pa.int32() if kind == "date" else pa.int64()).view(at)
    return pa.array(vals, type=at)


def raw_values(arr) -> list:
    """An Arrow column -> its raw values (None = NULL)."""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    t = arr.type
    valid = arr.is_valid().to_pylist()
    if pa.types.is_floating(t):
        u = np.uint32 if t == pa.float32() else np.uint64
        bits = np.frombuffer(arr.buffers()[1], dtype=u, count=arr.offset + len(arr))[arr.offset:] if len(arr) else []
        return [int(b) if v else None for b, v in zip(bits, valid)]
    if pa.types.is_decimal(t):
        return [None if x is None else int(x.scaleb(t.scale, _EXACT)) for x in arr.to_pylist()]
    if pa.types.is_date32(t):
        return arr.view(pa.int32()).to_pylist()
    if pa.types.is_timestamp(t):
        return arr.view(pa.int64()).to_pylist()
    return arr.to_pylist()


def make_table(arg_types, n: int, seed: int, key_cols=None) -> pa.Table:
    """One column per (type, form) of arg_types in the three forms, named v_<type>_<form>, plus key columns:
    key_cols: name -> (type, raw values) or name -> Arrow array."""
    cols, fields = [], []
    rng = random.Random(seed)
    for i, t in enumerate(arg_types):
        vals = random_values(t, n, seed * 131 + i)
        for form in FORMS:
            nulls = [rng.random() < 0.25 for _ in range(n)] if form == "n" else None
            if form == "n" and n:
                nulls[rng.randrange(n)] = False
            cols.append(to_arrow(t, vals, nulls))
            fields.append(pa.field(f"v_{t}_{form}", TYPES[t][1], nullable=form != "nn"))
    for name, kv in (key_cols or {}).items():
        arr = kv if isinstance(kv, (pa.Array, pa.ChunkedArray)) else to_arrow(kv[0], kv[1])
        cols.append(arr)
        fields.append(pa.field(name, arr.type, nullable=arr.null_count > 0))
    return pa.Table.from_arrays(cols, schema=pa.schema(fields))


def ir_schema(table: pa.Table):
    """The IR fields of a table built by make_table (nullable as its Arrow field says)."""
    ir_of = {str(v[1]): v[2] for v in TYPES.values()}
    return [P.field(f.name, ir_of[str(f.type)], f.nullable) for f in table.schema]


# ---- result types ---------------------------------------------------------------------------------------------------
def result_type(fn: str, t: str | None) -> pa.DataType:
    if fn in ("count", "count_star"):
        return pa.int64()
    kind, at, _it, bits, _e = TYPES[t]
    if fn in ("min", "max"):
        return at
    if fn == "sum":
        if kind == "dec":
            return pa.decimal128(min(38, bits[0] + 10), bits[1])
        return {"int": pa.int64(), "uint": pa.uint64(), "float": pa.float64()}[kind]
    if fn == "avg":
        if kind == "dec":
            return pa.decimal128(min(38, bits[0] + 4), min(38, bits[1] + 4))
        return pa.float64()
    raise AssertionError(fn)


# ---- reference ------------------------------------------------------------------------------------------------------
class AggOverflow(Exception):
    """The reference's decimal AVG failed: the engine must fail the task with an execution error."""


class Approx:
    """A float SUM / AVG: the exact value (a Fraction, or 'nan' / 'inf' / '-inf') and the error the device may add."""

    def __init__(self, exact, bound):
        self.exact, self.bound = exact, bound

    def matches(self, bits: int) -> bool:
        x = struct.unpack("<d", struct.pack("<Q", bits))[0]
        if isinstance(self.exact, str):
            return (x != x) if self.exact == "nan" else x == float(self.exact)
        if x != x or x in (float("inf"), float("-inf")):
            return False
        return abs(Fraction(x) - self.exact) <= self.bound

    def __repr__(self):
        return f"Approx({self.exact if isinstance(self.exact, str) else float(self.exact)!r} +- {float(self.bound):.3g})"


U64 = Fraction(1, 1 << 53)   # unit roundoff of Float64


def _float_of(kind, bits, v) -> float:
    """The Float64 a raw value becomes before it is summed or averaged (a cast, exact for f32, rounded for integers)."""
    if kind == "float":
        return struct.unpack("<d", struct.pack("<Q", v))[0] if bits == 64 else struct.unpack("<f", struct.pack("<I", v))[0]
    return float(v)


def _float_sum(xs):
    """(exact sum or special, sum of |x|) of Float64 values."""
    if any(x != x for x in xs) or (float("inf") in xs and float("-inf") in xs):
        return "nan", 0
    if float("inf") in xs:
        return "inf", 0
    if float("-inf") in xs:
        return "-inf", 0
    fr = [Fraction(x) for x in xs]
    return sum(fr, Fraction(0)), sum((abs(f) for f in fr), Fraction(0))


def _order_key(kind, bits, v):
    if kind == "float":
        w = bits
        sign = 1 << (w - 1)
        return (v ^ ((1 << w) - 1)) if v & sign else (v | sign)   # IEEE total order as an unsigned key
    if kind == "utf8":
        return v.encode("utf-8")
    return v


def _wrap(v, bits, signed):
    v &= (1 << bits) - 1
    return v - (1 << bits) if signed and v >> (bits - 1) else v


def aggregate_values(fn: str, t: str | None, vals):
    """One aggregate over one group's raw argument values (None = NULL); count_star takes the row count as vals."""
    if fn == "count_star":
        return len(vals)
    xs = [v for v in vals if v is not None]
    if fn == "count":
        return len(xs)
    if not xs:
        return None
    kind, _at, _it, bits, _e = TYPES[t]
    if fn in ("min", "max"):
        pick = min if fn == "min" else max
        return pick(xs, key=lambda v: _order_key(kind, bits, v))
    if fn == "sum" and kind in ("int", "uint"):
        return _wrap(sum(xs), 64, kind == "int")
    if kind == "dec":
        s = _wrap(sum(xs), 128, True)
        if fn == "sum":
            return s
        p, sc = bits
        k = min(38, sc + 4) - sc
        prod = s * 10 ** k
        if not -(1 << 127) <= prod < (1 << 127):
            raise AggOverflow("sum * 10^k beyond i128")
        q = abs(prod) // len(xs) * (1 if prod >= 0 else -1)
        if abs(q) >= 10 ** min(38, p + 4):
            raise AggOverflow("average beyond the result precision")
        return q
    fl = [_float_of(kind, bits, v) for v in xs]
    exact, mag = _float_sum(fl)
    bound = (len(fl) - 1) * U64 * mag
    if fn == "sum":
        return Approx(exact, bound)
    if isinstance(exact, str):
        return Approx(exact, 0)
    mean = exact / len(fl)
    return Approx(mean, bound / len(fl) + U64 * abs(mean) + Fraction(1, 1 << 1074))


def key_of(kind_vals):
    """A hashable group key from raw key values: floats by bits, decimals by unscaled value, strings by UTF-8 bytes."""
    return tuple(("s", v.encode("utf-8")) if isinstance(v, str) else v for v in kind_vals)


def reference(table: pa.Table, keys, aggs) -> dict:
    """{group key: [result per aggregate]} of an aggregate with group keys `keys` (column names) and aggregates `aggs`
    [(fn, column name or None, output name)].  No keys: one group, (), even for an empty input."""
    n = table.num_rows
    kv = [raw_values(table.column(k)) for k in keys]
    groups: dict = {}
    if not keys:
        groups[()] = list(range(n))
    for i in range(n):
        if keys:
            groups.setdefault(key_of([col[i] for col in kv]), []).append(i)
    args = {a: raw_values(table.column(a)) for _fn, a, _nm in aggs if a is not None}
    type_of = {f.name: _type_name(f.type) for f in table.schema}
    out = {}
    for g, rows in groups.items():
        out[g] = [aggregate_values(fn, type_of.get(a), rows if fn == "count_star" else [args[a][i] for i in rows]) for fn, a, _nm in aggs]
    return out


def _type_name(t: pa.DataType) -> str:
    for name, v in TYPES.items():
        if v[1] == t:
            return name
    raise KeyError(t)


def results_of(table: pa.Table, n_keys: int) -> dict:
    """The engine's output as {group key: [raw result per aggregate]}; a repeated group key is an error."""
    cols = [raw_values(table.column(i)) for i in range(table.num_columns)]
    out = {}
    for r in range(table.num_rows):
        k = key_of([cols[i][r] for i in range(n_keys)])
        assert k not in out, f"group {k!r} emitted twice"
        out[k] = [cols[i][r] for i in range(n_keys, table.num_columns)]
    return out


def mismatches(got: dict, want: dict, names) -> list:
    """Differences between results_of() and reference(); empty when the engine is right."""
    bad = []
    if set(got) != set(want):
        bad.append(("groups", sorted(map(repr, set(got) ^ set(want)))[:8]))
        return bad
    for k, w in want.items():
        for name, gv, wv in zip(names, got[k], w):
            ok = (gv is not None and wv.matches(gv)) if isinstance(wv, Approx) else gv == wv
            if not ok:
                bad.append((k, name, gv, wv))
    return bad[:12]


def check_types(table: pa.Table, aggs, key_types) -> None:
    """The output schema: the keys' types, then result_type of each aggregate.  aggs: [(fn, argument type or None)]."""
    want = list(key_types) + [result_type(fn, None if at is None else _type_name(at)) for fn, at in aggs]
    assert [f.type for f in table.schema] == want, (table.schema, want)


# ---- plans ----------------------------------------------------------------------------------------------------------
MODES = ("final_partitioned", "final", "single", "single_partitioned")
FN_IR = {"count_star": "count", "count": "count", "sum": "sum", "avg": "avg", "min": "min", "max": "max"}


def stages(mode: str, schema, keys, aggs, n_out: int = 16, table: str = "agg_t"):
    """Stage plans of one AggregateExec over the scan of `table` in `mode`:
    - final_partitioned: Partial -> hash shuffle on the keys into n_out partitions -> FinalPartitioned;
    - final: Partial -> one partition -> Final;
    - single: Single over the scan (register the table as one partition);
    - single_partitioned: the rows hash-shuffled on the keys into n_out partitions -> SinglePartitioned.
    keys: column names; aggs: [(fn, column name or None, output name)]."""
    idx = {f["name"]: i for i, f in enumerate(schema)}
    gb = [(c(idx[k]), k) for k in keys]
    pagg = [P.agg(FN_IR[fn], None if a is None else c(idx[a]), nm) for fn, a, nm in aggs]
    scan = P.scan(table, schema)
    nk = len(keys)
    if mode == "single":
        return [P.Stage(1, P.shuffle_writer(P.aggregate("Single", gb, pagg, scan), 1))]
    if mode == "single_partitioned":
        assert nk
        return [P.Stage(1, P.shuffle_writer(scan, 1, [c(idx[k]) for k in keys], n_out)),
                P.Stage(2, P.shuffle_writer(P.aggregate("SinglePartitioned", gb, pagg, P.shuffle_reader(1, schema)), 2))]
    partial = P.aggregate("Partial", gb, pagg, scan)
    typed = json.loads(engine.plan_typed_json(json.dumps(partial)))
    part = typed["schema"]
    faggs = [P.agg(a["fn"], None, a["name"], ta["input_type"] if a["fn"] == "avg" else None) for a, ta in zip(pagg, typed["aggr"])]
    fgb = [(c(i), k) for i, k in enumerate(keys)]
    if mode == "final_partitioned" and nk:
        return [P.Stage(1, P.shuffle_writer(partial, 1, [c(i) for i in range(nk)], n_out)),
                P.Stage(2, P.shuffle_writer(P.aggregate("FinalPartitioned", fgb, faggs, P.shuffle_reader(1, part)), 2))]
    return [P.Stage(1, P.shuffle_writer(partial, 1)),
            P.Stage(2, P.shuffle_writer(P.aggregate("Final", fgb, faggs, P.coalesce_partitions(P.shuffle_reader(1, part))), 2), n_tasks=1)]


def register(e, table: pa.Table, parts: int, name: str = "agg_t") -> None:
    try:
        e.drop_table(name)
    except Exception:
        pass
    n = table.num_rows
    for p in range(parts):
        sl = table.slice(n * p // parts, n * (p + 1) // parts - n * p // parts).combine_chunks()
        e.register_batch(name, p, sl.to_batches()[0] if sl.num_rows else
                         pa.RecordBatch.from_arrays([pa.array([], type=f.type) for f in table.schema], schema=table.schema))


def run(e, table: pa.Table, mode: str, keys, aggs, job: str, parts: int = 3, n_out: int = 16) -> pa.Table:
    """Register the columns of `table` the aggregate reads (one partition for Single, else `parts`) and run it in `mode`."""
    table = table.select(list(dict.fromkeys(list(keys) + [a for _fn, a, _nm in aggs if a is not None])))
    register(e, table, 1 if mode == "single" else parts)
    return driver.run_stages(e, stages(mode, ir_schema(table), keys, aggs, n_out), job)


def check(e, table: pa.Table, mode: str, keys, aggs, job: str, parts: int = 3, want=None, n_out: int = 16) -> pa.Table:
    """Run and compare with the reference: output types, then every group's results."""
    got = run(e, table, mode, keys, aggs, job, parts, n_out)
    key_types = [table.schema.field(k).type for k in keys]
    check_types(got, [(fn, None if a is None else table.schema.field(a).type) for fn, a, _nm in aggs], key_types)
    if want is None:
        want = reference(table, keys, aggs)
    bad = mismatches(results_of(got, len(keys)), want, [nm for _fn, _a, nm in aggs])
    assert not bad, f"{mode}: {bad}"
    return got


# ---- the argument matrix --------------------------------------------------------------------------------------------
def fn_groups(t: str):
    """The aggregates of each plan over one argument column of type t (at most 6 accumulators per plan, so that a plan
    with few groups can take the register sink)."""
    if TYPES[t][0] in ("date", "ts", "bool", "utf8"):
        return [("count_star", "count", "min", "max")]
    return [("count_star", "count", "sum", "avg"), ("min", "max")]


def arg_aggs(t: str, form: str, fns):
    col = f"v_{t}_{form}"
    return [(fn, None if fn == "count_star" else col, f"{fn}_{t}_{form}") for fn in fns]


def arg_table(n: int = 4097, seed: int = 7, groups: int = 4) -> pa.Table:
    """Every argument type in its three forms, plus a non-nullable Int64 key `g` with `groups` values."""
    rng = random.Random(seed)
    g = [rng.randrange(groups) - 2 for _ in range(n)]
    return make_table(list(TYPES), n, seed, {"g": ("i64", g)})


def snan_table():
    """Float32 groups where a signalling NaN decides MIN or MAX, and signalling and quiet NaN keys with one payload."""
    inf, one, m_one = 0x7F800000, 0x3F800000, 0xBF800000
    rows = [(0, 0x7F800001), (0, 0x7FC00000), (0, one),          # MAX: the quiet NaN above the signalling one
            (1, 0x7F800001), (1, one), (1, inf | 0x80000000),     # MAX: the signalling NaN
            (2, 0xFF800001), (2, m_one),                          # MIN: the negative signalling NaN
            (3, 0xFF800001), (3, 0xFFC00000)]                     # MIN: the negative quiet NaN below it
    rows = rows * 3
    keys = [0x7F800001, 0x7FC00001] * (len(rows) // 2)
    return make_table([], len(rows), 1, {"g": ("i64", [r[0] for r in rows]), "x": ("f32", [r[1] for r in rows]),
                                          "kf": ("f32", keys)})


SNAN_AGGS = [("min", "x", "mn"), ("max", "x", "mx"), ("count_star", None, "c")]


# ---- the key matrix -------------------------------------------------------------------------------------------------
def key_domains():
    """Key type -> raw values that sit at the type's edges."""
    big = 10 ** 37
    return {
        "i64": [-2 ** 63, 2 ** 63 - 1, 0, -1],
        "u64": [2 ** 63, 2 ** 64 - 1, 0, 2 ** 63 - 1],
        "i32": [-2 ** 31, 2 ** 31 - 1, -1, 0],
        "date32": [-2 ** 31, 2 ** 31 - 1, 0, 1],
        "u32": [2 ** 32 - 1, 0, 2 ** 31, 2 ** 31 - 1],
        "i8": [-1, -128, 127, 0],
        "u8": [255, 0, 128, 1],
        "d38_0": [big, -big, 2 ** 64, 2 ** 64 + 1, -(2 ** 64)],
        "bool": [True, False],
        "f32": F32_EDGES,
        "f64": F64_EDGES,
        "utf8": ["", "a", "a\0", "abc", "abcd", "abcdefg", "abcdefgh", "a much longer string", "é", "日本"],
    }


KEY_SHAPES = {t: [t] for t in key_domains()}
KEY_SHAPES.update({"i32+u32": ["i32", "u32"], "i8+u8": ["i8", "u8"], "date32+i32": ["date32", "i32"], "utf8+i64": ["utf8", "i64"],
                   "f64+f32": ["f64", "f32"], "bool+d38_0": ["bool", "d38_0"]})
KEY_AGGS = [("count_star", None, "cnt"), ("sum", "v_i64_nn", "s"), ("min", "v_f64_n", "mn"), ("max", "v_utf8_n", "mx")]


def key_table(shape: str, n: int, seed: int, nullable: bool) -> tuple:
    """(table, key column names): the key columns of `shape` over their edge domains (with about one NULL in seven when
    nullable), plus the value columns KEY_AGGS reads."""
    rng = random.Random(seed)
    dom = key_domains()
    keys = {}
    for t in KEY_SHAPES[shape]:
        vals = [rng.choice(dom[t]) for _ in range(n)]
        nulls = [nullable and rng.random() < 1 / 7 for _ in range(n)]
        keys[f"k_{t}"] = to_arrow(t, vals, nulls if nullable else None)
    table = make_table(["i64", "f64", "utf8"], n, seed, keys)
    return table, list(keys)
