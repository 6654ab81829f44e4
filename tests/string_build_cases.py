"""The string builders of DESIGN.md §6 (xi) restated per row in plain Python: concat, `||`, concat_ws, repeat, reverse and
CAST(x AS Utf8) of integers, Decimal128, Date32 and Bool.  An edge-case table puts NULLs, empty strings, multi-byte UTF-8
and a row over 64 KB in every argument position.

The restatement is pinned against independent computations (sqlite3, pyarrow.compute.cast, Python str) by
tests/test_string_build.py; the device is checked byte for byte against it by tests/test_gpu_string_build.py."""
import datetime
import decimal

import pyarrow as pa

from ballista_b200 import plan as P

c = P.col
EPOCH_ORDINAL = datetime.date(1970, 1, 1).toordinal()
ROW_LIMIT = 2**31 - 1


class TooLong(Exception):
    pass


# ---- per-row rules ---------------------------------------------------------------------------------------------------------
def concat(*xs):
    """never NULL: NULL arguments are skipped"""
    out = "".join(x for x in xs if x is not None)
    if len(out.encode()) > ROW_LIMIT:
        raise TooLong("concat")
    return out


def str_concat(a, b):
    return None if a is None or b is None else a + b


def concat_ws(sep, *xs):
    """NULL iff the separator is; NULL arguments are skipped with no separator for them"""
    return None if sep is None else sep.join(x for x in xs if x is not None)


def repeat(s, n):
    if s is None or n is None:
        return None
    if n <= 0:
        return ""
    if len(s.encode()) * n > ROW_LIMIT:
        raise TooLong("repeat")
    return s * n


def reverse(s):
    return None if s is None else s[::-1]   # code points, not bytes


def cast_int(v):
    return None if v is None else str(v)


def cast_decimal(unscaled, scale):
    """arrow's Decimal128 display: exactly `scale` fractional digits, a leading 0 below one, no point at scale 0"""
    if unscaled is None:
        return None
    digits = str(abs(unscaled))
    sign = "-" if unscaled < 0 else ""
    if scale == 0:
        return sign + digits
    digits = digits.rjust(scale + 1, "0")
    return sign + digits[:-scale] + "." + digits[-scale:]


def civil_from_days(days):
    """proleptic Gregorian (year, month, day) of a day number, any year (H. Hinnant's algorithm)"""
    z = days + 719468
    era = z // 146097  # floor division
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = mp + 3 if mp < 10 else mp - 9
    return yoe + era * 400 + (m <= 2), m, d


def cast_date(days):
    """chrono's %Y-%m-%d: four digits within years 0..9999, else an explicit sign and at least four digits"""
    if days is None:
        return None
    y, m, d = civil_from_days(days)
    ys = f"{y:04d}" if 0 <= y <= 9999 else f"{y:+05d}"
    return f"{ys}-{m:02d}-{d:02d}"


def cast_bool(v):
    return None if v is None else ("true" if v else "false")


# ---- the edge-case table -----------------------------------------------------------------------------------------------------
STRINGS = [None, "", "a", "ab", "héllo", "日本語", "𝄞x", "a-b", " ", "zzzzzzzzzzzz", "€", "mixed 😀 ✓", None, "x" * 70000]
SCHEMA = [P.field("k", "i32", False), P.field("a", "utf8", True), P.field("b", "utf8", True), P.field("sep", "utf8", True),
          P.field("n", "i64", True), P.field("i8", "i8", True), P.field("i16", "i16", True), P.field("i32", "i32", True),
          P.field("i64", "i64", True), P.field("u8", "u8", True), P.field("u16", "u16", True), P.field("u32", "u32", True),
          P.field("u64", "u64", True), P.field("dec", P.dec(15, 2), True), P.field("dec0", P.dec(38, 0), True),
          P.field("dec9", P.dec(10, 9), True), P.field("d", "date32", True), P.field("flag", "bool", True)]
INT_EDGES = {
    "i8": [-128, 127, 0, -1], "i16": [-32768, 32767, 0, 9], "i32": [-2**31, 2**31 - 1, 0, -7], "i64": [-2**63, 2**63 - 1, 0, 10**18],
    "u8": [0, 255, 7], "u16": [0, 65535], "u32": [0, 2**32 - 1], "u64": [0, 2**64 - 1, 2**63, 2**63 - 1],
}
DEC_EDGES = {"dec": (2, [-5, 5, 0, 12345, -12345, 10**15 - 1, -(10**15 - 1), 100, -100]),
             "dec0": (0, [0, -1, 10**38 - 1, -(10**38 - 1), 42]),
             "dec9": (9, [1, -1, 10**10 - 1, -(10**10 - 1), 0, 500000000])}
DAY_EDGES = [0, -1, 1, -719162, 2932896, 2932897, -719163, -800000, 11016, 19000, 60 * 365 * 1000, -365 * 3000, 3652424,
             95000000, -95000000]


def edge_table(n=None):
    """one row per combination slice: every column cycles through its edges (NULL every 11th row), n rows"""
    n = n or 4 * len(STRINGS) * 3
    ints = {k: [None if i % 11 == 3 else v[i % len(v)] for i in range(n)] for k, v in INT_EDGES.items()}
    cols = {
        "k": pa.array(range(n), pa.int32()),
        "a": pa.array([STRINGS[i % len(STRINGS)] for i in range(n)], pa.string()),
        "b": pa.array([STRINGS[(i * 5 + 3) % len(STRINGS)] for i in range(n)], pa.string()),
        "sep": pa.array([[", ", None, "", "—"][i % 4] for i in range(n)], pa.string()),
        "n": pa.array([[3, 0, -2, None, 1, 2][i % 6] for i in range(n)], pa.int64()),
    }
    for k, v in ints.items():
        cols[k] = pa.array(v, P_TYPES[k])
    for k, (s, v) in DEC_EDGES.items():
        p = {"dec": 15, "dec0": 38, "dec9": 10}[k]
        cols[k] = pa.array([None if i % 11 == 3 else _dec(v[i % len(v)], s) for i in range(n)], pa.decimal128(p, s))
    cols["d"] = pa.array([None if i % 11 == 3 else DAY_EDGES[i % len(DAY_EDGES)] for i in range(n)], pa.int32()).cast(pa.date32())
    cols["flag"] = pa.array([None if i % 3 == 2 else bool(i % 2) for i in range(n)], pa.bool_())
    return pa.table(cols)


P_TYPES = {"i8": pa.int8(), "i16": pa.int16(), "i32": pa.int32(), "i64": pa.int64(), "u8": pa.uint8(), "u16": pa.uint16(),
           "u32": pa.uint32(), "u64": pa.uint64()}


CTX = decimal.Context(prec=50)


def _dec(unscaled, scale):
    return decimal.Decimal(unscaled).scaleb(-scale, CTX)


def _unscaled(d, scale):
    return None if d is None else int(d.scaleb(scale, CTX))


def _days(d):
    return None if d is None else d.toordinal() - EPOCH_ORDINAL


def projections():
    """(name, expression, per-row rule over a dict of the row's Python values)"""
    s = P.lit_utf8
    out = [
        ("concat_ab", P.fn("concat", c("a"), c("b")), lambda r: concat(r["a"], r["b"])),
        ("concat_lits", P.fn("concat", s("<"), c("a"), P.lit_utf8(None), s(">")), lambda r: concat("<", r["a"], None, ">")),
        ("concat_one", P.fn("concat", c("b")), lambda r: concat(r["b"])),
        ("concat_nested", P.fn("concat", P.fn("reverse", c("a")), c("b"), P.cast(c("i32"), "utf8")),
         lambda r: concat(reverse(r["a"]), r["b"], cast_int(r["i32"]))),
        ("concat_ten", P.fn("concat", *[c("a") if i % 2 else s(str(i)) for i in range(10)]),
         lambda r: concat(*[r["a"] if i % 2 else str(i) for i in range(10)])),
        ("pipe", P.str_concat(c("a"), c("b")), lambda r: str_concat(r["a"], r["b"])),
        ("pipe3", P.str_concat(P.cast(c("i64"), "utf8"), s("-"), c("b")), lambda r: str_concat(str_concat(cast_int(r["i64"]), "-"), r["b"])),
        ("concat_ws", P.fn("concat_ws", c("sep"), c("a"), c("b"), s("z")), lambda r: concat_ws(r["sep"], r["a"], r["b"], "z")),
        ("concat_ws_lit", P.fn("concat_ws", s("|"), c("a"), P.lit_utf8(None), c("b")), lambda r: concat_ws("|", r["a"], None, r["b"])),
        ("concat_ws_many", P.fn("concat_ws", c("sep"), *[[c("a"), c("b"), s("q"), P.lit_utf8(None)][i % 4] for i in range(13)]),
         lambda r: concat_ws(r["sep"], *[[r["a"], r["b"], "q", None][i % 4] for i in range(13)])),
        ("repeat_lit", P.fn("repeat", c("a"), P.lit_i64(3)), lambda r: repeat(r["a"], 3)),
        ("repeat_col", P.fn("repeat", c("b"), c("n")), lambda r: repeat(r["b"], r["n"])),
        ("reverse", P.fn("reverse", c("a")), lambda r: reverse(r["a"])),
    ]
    for k in INT_EDGES:
        out.append((f"cast_{k}", P.cast(c(k), "utf8"), (lambda k: lambda r: cast_int(r[k]))(k)))
    for k, (sc, _) in DEC_EDGES.items():
        out.append((f"cast_{k}", P.cast(c(k), "utf8"), (lambda k, sc: lambda r: cast_decimal(_unscaled(r[k], sc), sc))(k, sc)))
    out.append(("cast_date", P.cast(c("d"), "utf8"), lambda r: cast_date(r["d"])))
    out.append(("cast_bool", P.cast(c("flag"), "utf8"), lambda r: cast_bool(r["flag"])))
    out.append(("cast_null", P.cast(P.lit_null("i64"), "utf8"), lambda r: None))
    return out


def expected(table, rule):
    """the rule over every row; Date32 values as day numbers (Python's date stops at year 9999)"""
    if "d" in table.column_names:
        table = table.set_column(table.column_names.index("d"), "d", table.column("d").cast(pa.int32()))
    rows = table.to_pylist()
    return [rule(r) for r in rows]
