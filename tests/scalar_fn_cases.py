"""The scalar functions of DESIGN.md §3 restated per row in plain Python (the rules of the §6 table), an edge-case table
that puts NULLs in every argument position, and the projection that calls every function and alias over it.

The restatement is pinned against independent computations (datetime, pyarrow.compute, math, sqlite3, str) by
tests/test_scalar_functions.py; the device is checked bit-exactly against it by tests/test_gpu_scalar_functions.py."""
import datetime
import decimal
import math
import struct

import numpy as np
import pyarrow as pa

from ballista_b200 import plan as P

c = P.col
D = decimal.Decimal
EPOCH_ORDINAL = datetime.date(1970, 1, 1).toordinal()
PARTS = ["year", "quarter", "month", "week", "day", "doy", "dow"]
INT_MIN = {"i8": -2**7, "i16": -2**15, "i32": -2**31, "i64": -2**63}


class Overflow(Exception):
    pass


# ---- per-row rules ---------------------------------------------------------------------------------------------------------
def date_part(part, days):
    if days is None:
        return None
    d = datetime.date.fromordinal(EPOCH_ORDINAL + days)
    return {"year": d.year, "quarter": (d.month - 1) // 3 + 1, "month": d.month, "week": d.isocalendar()[1], "day": d.day,
            "doy": d.timetuple().tm_yday, "dow": d.isoweekday() % 7}[part]


def abs_(x, typ=None):
    if x is None:
        return None
    if typ in INT_MIN and x == INT_MIN[typ]:
        raise Overflow(typ)
    if isinstance(x, float):
        return math.fabs(x)
    return -x if x < 0 else x


def _f32(v):
    return float(np.float32(v))


def _round_half_away(y):
    if math.isnan(y) or math.isinf(y):
        return y
    t = math.trunc(y)
    if abs(y - t) >= 0.5:   # y - t is exact: t is y with its fraction removed
        t += 1 if y > 0 else -1
    return math.copysign(float(t), y)


def round_(x, n=0, f32=False):
    if x is None or n is None:
        return None
    p = 10.0 ** abs(n)
    if f32:
        f = np.float32(p) if n >= 0 else np.float32(1.0) / np.float32(p)
        y = np.float32(x) * f
        return float(np.float32(_round_half_away(float(y))) / f)
    f = p if n >= 0 else 1.0 / p
    return _round_half_away(x * f) / f


def floor_(x):
    if x is None or not math.isfinite(x):
        return x
    return math.copysign(float(math.floor(x)), x) if math.floor(x) == 0 else float(math.floor(x))


def ceil_(x):
    if x is None or not math.isfinite(x):
        return x
    return math.copysign(float(math.ceil(x)), x) if math.ceil(x) == 0 else float(math.ceil(x))


def _same(a, b):
    if isinstance(a, float):  # total order: NaN = NaN, -0.0 != 0.0
        return struct.pack("<d", a) == struct.pack("<d", b)
    return a == b


def nullif(a, b):
    return None if (a is not None and b is not None and _same(a, b)) else a


def coalesce(*xs):
    return next((x for x in xs if x is not None), None)


def char_length(s):
    return None if s is None else len(s)


def octet_length(s):
    return None if s is None else len(s.encode())


def starts_with(s, p):
    return None if s is None or p is None else s.startswith(p)


def ends_with(s, p):
    return None if s is None or p is None else s.endswith(p)


def trim(side, s, chars=" "):
    if s is None or chars is None:
        return None
    return {"btrim": s.strip, "ltrim": s.lstrip, "rtrim": s.rstrip}[side](chars)


# ---- the edge-case table ----------------------------------------------------------------------------------------------------
EDGE_DAYS = [0, -1, 1, 59, 60, 365, 366, -719162, -719163 + 365, 2932896, 11016, 11017, 10956, 10957, 10958, 10959, 10960,
             10961, 10962, 13878, 13879, 13880, 13881, 13882, 13883, 13884, 14244, 14245, 14246, 14609, 14610, 14611, 14612,
             16435, 16436, 16437, -25567, -25568, -36524, -36525, -141427, 47481, 47482]
STRS = ["", " ", "   ", " a ", "  héllo wörld  ", "日本語", " 日本 ", "xxabcxx", "€uro€", "ab€", "€", "a", "MAIL", "TRUCK  ",
        "  REG AIR", "COLLECT COD", "ümlaut", "naïve café", "x€x€", "🙂 smile 🙂", "\t tab", "abc", "ab", "b"]
PREFIXES = ["", "a", "ab", "日", "€", " ", "xyz", "abc", "🙂", "TRUCK"]
FLOATS = [0.0, -0.0, 0.5, -0.5, 1.5, 2.5, -2.5, 0.49999999999999994, 1.005, 2.675, -1.2345, 123.456, 1e300, -1e300,
          float("nan"), float("inf"), float("-inf"), 1e-300, 5e-324, 9007199254740993.0, 0.125, -7.75, 314.159, 1e22, 4.5e15]
ROUND_DIGITS = [-3, 0, 2, 22]


def edge_table(n=3500, seed=7):
    """n rows (>= 3 full 1024-row tiles plus a partial one); every column has NULLs spread across the tiles"""
    rng = np.random.default_rng(seed)

    def pick(vals, null_every):
        out = []
        for r in range(n):
            if (r * 7919 + null_every) % null_every == 0:
                out.append(None)
            else:
                out.append(vals[int(rng.integers(len(vals)))])
        return out

    days = pick(EDGE_DAYS + [int(v) for v in rng.integers(-719162, 2932896, 200)], 11)
    cols = {
        "d": pa.array(days, pa.int32()).cast(pa.date32()),
        "i8": pa.array(pick([0, 1, -1, 127, -127, 5, -100], 13), pa.int8()),
        "i16": pa.array(pick([0, 1, -1, 32767, -32767, -300], 9), pa.int16()),
        "i32": pa.array(pick([0, 7, -7, 2**31 - 1, -(2**31 - 1), 123456], 10), pa.int32()),
        "i64": pa.array(pick([0, 3, -3, 2**63 - 1, -(2**63 - 1), -5000000000], 12), pa.int64()),
        "u8": pa.array(pick([0, 1, 255, 128], 8), pa.uint8()),
        "u64": pa.array(pick([0, 1, 2**64 - 1, 2**63], 14), pa.uint64()),
        "f32": pa.array([None if v is None else _f32(v) for v in pick(FLOATS, 15)], pa.float32()),
        "f64": pa.array(pick(FLOATS, 16), pa.float64()),
        "f64b": pa.array(pick(FLOATS[:8] + [float("nan")], 6), pa.float64()),
        "dec": pa.array(pick([D("0.00"), D("-1.25"), D("9999999999999.99"), D("-9999999999999.99"), D("3.10")], 17), pa.decimal128(15, 2)),
        "s": pa.array(pick(STRS, 18), pa.string()),
        "p": pa.array(pick(PREFIXES, 19), pa.string()),
        "b": pa.array(pick([True, False], 20), pa.bool_()),
        "b2": pa.array(pick([True, False], 21), pa.bool_()),
        "k": pa.array(pick([0, 1, 2, -3], 22), pa.int32()),
    }
    return pa.table(cols)


SCHEMA = [P.field("d", "date32", True), P.field("i8", "i8", True), P.field("i16", "i16", True), P.field("i32", "i32", True),
          P.field("i64", "i64", True), P.field("u8", "u8", True), P.field("u64", "u64", True), P.field("f32", "f32", True),
          P.field("f64", "f64", True), P.field("f64b", "f64", True), P.field("dec", P.dec(15, 2), True), P.field("s", "utf8", True),
          P.field("p", "utf8", True), P.field("b", "bool", True), P.field("b2", "bool", True), P.field("k", "i32", True)]

TRIM_SET = "x€ "


def projections():
    """(output name, IR expression, per-row reference over a dict row, result Arrow type); abs over the signed minimum is not
    here (its overflow is an error, tested on its own)"""
    out = []
    for part in PARTS:
        out.append((f"dp_{part}", P.fn(f"date_part_{part}", c("d")), lambda r, part=part: date_part(part, r["d"]), pa.int32()))
    for col, typ in (("i8", pa.int8()), ("i16", pa.int16()), ("i32", pa.int32()), ("i64", pa.int64()), ("u8", pa.uint8()),
                     ("u64", pa.uint64()), ("f32", pa.float32()), ("f64", pa.float64()), ("dec", pa.decimal128(15, 2))):
        out.append((f"abs_{col}", P.fn("abs", c(col)), lambda r, col=col: abs_(r[col]), typ))
    for n in ROUND_DIGITS:
        out.append((f"round_f64_{n}".replace("-", "m"), P.fn("round", c("f64"), P.lit_i64(n)), lambda r, n=n: round_(r["f64"], n), pa.float64()))
        out.append((f"round_f32_{n}".replace("-", "m"), P.fn("round", c("f32"), P.lit_i64(n)), lambda r, n=n: round_(r["f32"], n, True), pa.float32()))
    out += [
        ("round_f64", P.fn("round", c("f64")), lambda r: round_(r["f64"]), pa.float64()),
        ("round_null_digits", P.fn("round", c("f64"), P.lit_null("i64")), lambda r: None, pa.float64()),
        ("floor_f64", P.fn("floor", c("f64")), lambda r: floor_(r["f64"]), pa.float64()),
        ("ceil_f64", P.fn("ceil", c("f64")), lambda r: ceil_(r["f64"]), pa.float64()),
        ("floor_f32", P.fn("floor", c("f32")), lambda r: floor_(r["f32"]), pa.float32()),
        ("ceil_f32", P.fn("ceil", c("f32")), lambda r: ceil_(r["f32"]), pa.float32()),
        ("nullif_i32", P.fn("nullif", c("i32"), c("k")), lambda r: nullif(r["i32"], r["k"]), pa.int32()),
        ("nullif_i32_lit", P.fn("nullif", c("k"), P.lit_i32(0)), lambda r: nullif(r["k"], 0), pa.int32()),
        ("nullif_f64", P.fn("nullif", c("f64"), c("f64b")), lambda r: nullif(r["f64"], r["f64b"]), pa.float64()),
        ("nullif_dec", P.fn("nullif", c("dec"), P.lit_dec(310, 15, 2)), lambda r: nullif(r["dec"], D("3.10")), pa.decimal128(15, 2)),
        ("nullif_s", P.fn("nullif", c("s"), c("p")), lambda r: nullif(r["s"], r["p"]), pa.string()),
        ("nullif_b", P.fn("nullif", c("b"), c("b2")), lambda r: nullif(r["b"], r["b2"]), pa.bool_()),
        ("nullif_date", P.fn("nullif", c("d"), P.lit_date("1970-01-01")), lambda r: nullif(r["d"], 0), pa.date32()),
        ("coalesce_i32", P.fn("coalesce", c("i32"), c("k"), P.lit_i32(-1)), lambda r: coalesce(r["i32"], r["k"], -1), pa.int32()),
        ("coalesce_s", P.fn("coalesce", c("s"), c("p")), lambda r: coalesce(r["s"], r["p"]), pa.string()),
        ("coalesce_f64", P.fn("coalesce", c("f64"), c("f64b")), lambda r: coalesce(r["f64"], r["f64b"]), pa.float64()),
        ("coalesce_one", P.fn("coalesce", c("dec")), lambda r: r["dec"], pa.decimal128(15, 2)),
        ("char_length", P.fn("character_length", c("s")), lambda r: char_length(r["s"]), pa.int32()),
        ("octet_length", P.fn("octet_length", c("s")), lambda r: octet_length(r["s"]), pa.int32()),
        ("starts_with", P.fn("starts_with", c("s"), c("p")), lambda r: starts_with(r["s"], r["p"]), pa.bool_()),
        ("ends_with", P.fn("ends_with", c("s"), c("p")), lambda r: ends_with(r["s"], r["p"]), pa.bool_()),
        ("starts_with_lit", P.fn("starts_with", c("s"), P.lit_utf8("ab")), lambda r: starts_with(r["s"], "ab"), pa.bool_()),
        ("ends_with_lit", P.fn("ends_with", c("s"), P.lit_utf8("€")), lambda r: ends_with(r["s"], "€"), pa.bool_()),
    ]
    for side in ("btrim", "ltrim", "rtrim"):
        out.append((side, P.fn(side, c("s")), lambda r, side=side: trim(side, r["s"]), pa.string()))
        out.append((side + "_set", P.fn(side, c("s"), P.lit_utf8(TRIM_SET)), lambda r, side=side: trim(side, r["s"], TRIM_SET), pa.string()))
    out.append(("btrim_null_set", P.fn("btrim", c("s"), P.lit_null("utf8")), lambda r: None, pa.string()))
    out.append(("btrim_empty_set", P.fn("btrim", c("s"), P.lit_utf8("")), lambda r: r["s"], pa.string()))
    return out


def expected(table, projs):
    rows = table.to_pylist()
    for r in rows:  # dates as day numbers, as the engine sees them
        if r["d"] is not None:
            r["d"] = (r["d"] - datetime.date(1970, 1, 1)).days
    res = {}
    for name, _, fn, _ in projs:
        res[name] = [fn(r) for r in rows]
    return res


def same_values(got, want):
    """bit-exact comparison of two value lists (floats by their bits, so -0.0 != 0.0 and NaN == NaN)"""
    if len(got) != len(want):
        return False
    for g, w in zip(got, want):
        if (g is None) != (w is None):
            return False
        if isinstance(w, float) or isinstance(g, float):
            if struct.pack("<d", float(g)) != struct.pack("<d", float(w)):
                return False
        elif isinstance(w, datetime.date) or isinstance(g, datetime.date):
            gd = g if isinstance(g, int) else (g - datetime.date(1970, 1, 1)).days
            wd = w if isinstance(w, int) else (w - datetime.date(1970, 1, 1)).days
            if gd != wd:
                return False
        elif g != w:
            return False
    return True
