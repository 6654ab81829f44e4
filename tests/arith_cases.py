"""The scalar core of the tile VM -- `+ - * / %`, negation, the six comparisons, the numeric casts and CASE -- restated per
row in plain Python with exact integers, `fractions` and numpy's IEEE scalars, never through csrc/common/plan.hpp or
csrc/host/lower.hpp.  The rules (DESIGN.md §6 (xii)):

  integers   + - *: exact, then wrapped to the type's width.  /: truncates toward zero; a zero divisor is an error; a
             quotient outside the type (its minimum / -1) is an overflow error; UInt64 divides unsigned.
             %: the dividend's sign; MIN % -1 is 0 [EXT] (arrow's mod_checked may raise instead: not settled here).
  decimals   result types from arrow's decimal_op (written out below); operands rescaled to the result scale (+ -) or
             the larger scale (%), Div = a * 10^(s - s1 + s2) / b truncating; every i128 overflow is an error.
  floats     IEEE binary64; Float32 rounded once per operation.  -x flips the sign bit, a NaN's too.
  compares   exact for integers and decimals; floats in IEEE total order (-0.0 < 0.0, NaN above +inf, -NaN below -inf).
  casts      safe: out of range -> NULL; int -> decimal beyond the precision is an error; decimal down-scaling and
             float -> decimal round half away from zero (float -> decimal on the double x * 10.0**s); int -> Float32 is
             rounded once from the integer (Rust's `as f32`).
  CASE       each WHEN on the rows no earlier WHEN took, each THEN / the ELSE only on the rows it takes.

It also builds the edge table (`edge_table`): every integer type at its edges, Float32 / Float64 at the IEEE specials,
Decimal128 at eight (precision, scale) pairs, each in three forms (non-nullable, nullable without NULLs, nullable with
NULLs), with edge rows at 0, 1023, 1024 and the last row of 3 full 1024-row tiles plus a partial one."""
import math
import struct
from decimal import Context, Decimal
from fractions import Fraction

import numpy as np
import pyarrow as pa

from ballista_b200 import plan as P

INTS = {"i8": (8, True), "i16": (16, True), "i32": (32, True), "i64": (64, True),
        "u8": (8, False), "u16": (16, False), "u32": (32, False), "u64": (64, False)}
FLOATS = ("f32", "f64")
DECS = ((5, 2), (9, 0), (15, 2), (18, 4), (20, 0), (28, 6), (38, 0), (38, 10))
I128_MIN, I128_MAX = -(1 << 127), (1 << 127) - 1
N_ROWS = 3 * 1024 + 517
EDGE_ROWS = (0, 1023, 1024, N_ROWS - 1)
CTX = Context(prec=80)  # Decimal arithmetic wide enough for every Decimal128 value, exactly
FORMS = ("nn", "nv", "nl")  # non-nullable; nullable without NULLs (no validity buffer); nullable with NULLs


class Raise(Exception):
    """the engine must fail the plan with an execution error"""


def dec_name(p, s):
    return f"d{p}_{s}"


TYPES = list(INTS) + list(FLOATS) + [dec_name(p, s) for p, s in DECS]


def parse_dec(t):
    p, s = t[1:].split("_")
    return int(p), int(s)


def is_dec(t):
    return t.startswith("d")


def plan_type(t):
    return P.dec(*parse_dec(t)) if is_dec(t) else t


def arrow_type(t):
    if is_dec(t):
        return pa.decimal128(*parse_dec(t))
    return {"i8": pa.int8(), "i16": pa.int16(), "i32": pa.int32(), "i64": pa.int64(), "u8": pa.uint8(), "u16": pa.uint16(),
            "u32": pa.uint32(), "u64": pa.uint64(), "f32": pa.float32(), "f64": pa.float64(), "bool": pa.bool_()}[t]


def int_range(t):
    w, signed = INTS[t]
    return (-(1 << (w - 1)), (1 << (w - 1)) - 1) if signed else (0, (1 << w) - 1)


def wrap(v, t):
    w, signed = INTS[t]
    v &= (1 << w) - 1
    return v - (1 << w) if signed and v >> (w - 1) else v


# ---- floats: values are Python floats; Float32 values are exactly representable in binary32 ----------------------------
def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def f64_from_bits(b):
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def f32_from_bits(b):
    return float(np.array([b], np.uint32).view(np.float32)[0])


def to_f32(x):
    """x rounded once to binary32 (numpy's double -> float conversion rounds to nearest, ties to even)"""
    with np.errstate(all="ignore"):
        return float(np.float32(x))


def int_to_f32(v):
    """the binary32 nearest to the integer v, ties to even, computed on the integer (not through a double)"""
    if v == 0:
        return 0.0
    m, sign = abs(v), -1 if v < 0 else 1
    e = m.bit_length() - 24
    if e > 0:
        q, r = divmod(m, 1 << e)
        half = 1 << (e - 1)
        if r > half or (r == half and q & 1):
            q += 1
        m = q << e
    return sign * float(m)  # m has <= 25 significant bits: exact as a double


def total_key(x):
    """IEEE 754 totalOrder as an integer (f32 values widen exactly, NaN payloads kept)"""
    b = f64_bits(x)
    return b ^ 0xFFFFFFFFFFFFFFFF if b >> 63 else b | (1 << 63)


def float_op(op, a, b, t):
    f = np.float32 if t == "f32" else np.float64
    x, y = f(a), f(b)
    with np.errstate(all="ignore"):
        r = {"+": x + y, "-": x - y, "*": x * y, "/": x / y, "%": np.fmod(x, y)}[op]
    return float(r)


# ---- decimals: (unscaled integer, precision, scale) --------------------------------------------------------------------
def dec_result(op, t1, t2):
    """arrow-arith decimal_op, written from its documentation"""
    (p1, s1), (p2, s2) = t1, t2
    if op in "+-":
        s = max(s1, s2)
        return min(38, max(p1 - s1, p2 - s2) + s + 1), s
    if op == "*":
        return min(38, p1 + p2 + 1), s1 + s2
    if op == "/":
        s = min(38, s1 + 4)
        return min(38, p1 + s - s1 + s2), s
    s = max(s1, s2)
    return min(38, min(p1 - s1, p2 - s2) + s), s


def int_as_dec(t):
    """the Decimal128 an integer type becomes next to a decimal (DataFusion's coerce_numeric_type_to_decimal)"""
    return {"i8": (3, 0), "i16": (5, 0), "i32": (10, 0), "i64": (20, 0), "u8": (3, 0), "u16": (5, 0), "u32": (10, 0), "u64": (20, 0)}[t]


def chk(v):
    if not I128_MIN <= v <= I128_MAX:
        raise Raise("overflow")
    return v


def tdiv(a, b):
    """a / b truncated toward zero, exactly"""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def dec_op(op, a, t1, b, t2):
    p, s = dec_result(op, t1, t2)
    s1, s2 = t1[1], t2[1]
    if op in "+-":
        x, y = chk(a * 10 ** (s - s1)), chk(b * 10 ** (s - s2))
        return chk(x + y if op == "+" else x - y)
    if op == "*":
        return chk(a * b)
    if b == 0:
        raise Raise("div0")
    if op == "/":
        return chk(tdiv(chk(a * 10 ** (s - s1 + s2)), b))
    x, y = chk(a * 10 ** (s - s1)), chk(b * 10 ** (s - s2))
    return x - y * tdiv(x, y)


def round_half_away(fr):
    """the integer nearest to the rational fr, halves away from zero (not Python's round, which rounds halves to even)"""
    q = math.floor(abs(fr))
    if abs(fr) - q >= Fraction(1, 2):
        q += 1
    return q if fr >= 0 else -q


# ---- per-row operators ---------------------------------------------------------------------------------------------------
def arith(op, a, b, t):
    """a op b, both of type t (the result's type), or None; raises Raise for the rows that fail the plan"""
    if a is None or b is None:
        return None
    if t in FLOATS:
        return float_op(op, a, b, t)
    if is_dec(t):
        return dec_op(op, a, parse_dec(t), b, parse_dec(t))
    if op in "+-*":
        return wrap(a + b if op == "+" else a - b if op == "-" else a * b, t)
    if b == 0:
        raise Raise("div0")
    q = tdiv(a, b)
    if op == "/":
        lo, hi = int_range(t)
        if not lo <= q <= hi:
            raise Raise("overflow")
        return q
    return a - b * q


def arith_type(op, t):
    return dec_name(*dec_result(op, parse_dec(t), parse_dec(t))) if is_dec(t) else t


def neg(a, t):
    if a is None:
        return None
    if t in FLOATS:
        return f64_from_bits(f64_bits(a) ^ (1 << 63))
    if is_dec(t):
        return -a
    return wrap(-a, t)


def compare(op, a, b, t):
    if a is None or b is None:
        return None
    if t in FLOATS:
        a, b = total_key(a), total_key(b)
    return {"=": a == b, "<>": a != b, "<": a < b, "<=": a <= b, ">": a > b, ">=": a >= b}[op]


def cast(v, frm, to):
    """CAST(v AS to) for a value of type frm; None for NULL (a NULL input or a safe-cast overflow)"""
    if v is None or frm == to:
        return v
    if frm in INTS and to in INTS:
        lo, hi = int_range(to)
        return v if lo <= v <= hi else None
    if frm in INTS and to == "f64":
        return float(v)  # Python's int -> float rounds once, to nearest even
    if frm in INTS and to == "f32":
        return int_to_f32(v)
    if frm in FLOATS and to in FLOATS:
        return to_f32(v) if to == "f32" else v
    if frm in FLOATS and to in INTS:
        if math.isnan(v) or math.isinf(v):
            return None
        lo, hi = int_range(to)
        q = math.trunc(v)
        return q if lo <= q <= hi else None
    if frm in INTS and is_dec(to):
        p, s = parse_dec(to)
        u = chk(v * 10 ** s)
        if abs(u) >= 10 ** p:
            raise Raise("precision")
        return u
    if is_dec(frm) and to in INTS:
        q = tdiv(v, 10 ** parse_dec(frm)[1])
        lo, hi = int_range(to)
        return q if lo <= q <= hi else None
    if is_dec(frm) and is_dec(to):
        (p1, s1), (p, s) = parse_dec(frm), parse_dec(to)
        u = chk(v * 10 ** (s - s1)) if s >= s1 else round_half_away(Fraction(v, 10 ** (s1 - s)))
        return u if abs(u) < 10 ** p else None
    if frm in FLOATS and is_dec(to):
        if math.isnan(v) or math.isinf(v):
            return None
        p, s = parse_dec(to)
        x = v * float(10 ** s)  # one IEEE multiplication (10.0**s is exact for s <= 22)
        if math.isinf(x):
            return None
        u = round_half_away(Fraction(x))
        return u if abs(u) < 10 ** p else None
    if is_dec(frm) and to in FLOATS:
        x = float(v) / float(10 ** parse_dec(frm)[1])
        return to_f32(x) if to == "f32" else x
    raise ValueError((frm, to))


def case_rows(conds, thens, else_=None):
    """CASE over per-row closures: conds / thens are lists of functions of the row; a THEN raises only when selected"""
    def f(row):
        for c, t in zip(conds, thens):
            if c(row) is True:
                return t(row)
        return else_(row) if else_ else None
    return f


# ---- edge values -------------------------------------------------------------------------------------------------------
NAN_BITS = (0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000123, 0xFFF4000000000456)
NAN32_BITS = (0x7FC00000, 0xFFC00000, 0x7FC00123, 0xFFA00456)


def edges(t):
    if t in INTS:
        lo, hi = int_range(t)
        v = [lo, lo + 1, -1, 0, 1, hi - 1, hi, 2, -3, 7] if lo < 0 else [0, 1, hi - 1, hi, 1 << (INTS[t][0] - 1), 2, 3, 7]
        return [x for x in v if lo <= x <= hi]
    if t == "f64":
        return [0.0, -0.0, math.inf, -math.inf, 5e-324, -2.2250738585072009e-308, 2.0 ** 53 - 1, 2.0 ** 53 + 2, 2.0 ** 63, -2.0 ** 63,
                2.0 ** 64, 1.5, -2.5, 0.125, -1.0, 1e10, 123456.789, 0.005] + [f64_from_bits(b) for b in NAN_BITS]
    if t == "f32":
        return [0.0, -0.0, math.inf, -math.inf, f32_from_bits(1), -f32_from_bits(0x7FFFFF), 2.0 ** 24 - 1, 2.0 ** 24 + 2, 2.0 ** 63,
                -2.0 ** 63, 2.0 ** 64, 1.5, -2.5, 0.125, -1.0, to_f32(1e10), to_f32(123456.789), to_f32(0.005)] + \
            [f32_from_bits(b) for b in NAN32_BITS]
    p, s = parse_dec(t)
    m = 10 ** p - 1
    half = 5 * 10 ** (s - 1) if s else 5
    return [m, -m, 1, -1, 0, half, -half, 7 * 10 ** s, -3 * 10 ** s, 123 * 10 ** s + (half if s else 0), 10 ** (p // 2) + 1]


def column_values(t, which, n=N_ROWS):
    """values of operand column `which` (0: a, 1: b) of type t: the edges, a cycling through them and b shifting by one
    more every cycle of a, so that every pair of edges meets in some row -- the edge rows 0, 1023, 1024 and the last among
    them"""
    e = edges(t)
    return [e[i % len(e)] if which == 0 else e[(i + i // len(e)) % len(e)] for i in range(n)]


def null_mask(which, n=N_ROWS):
    """rows that are NULL in the "nl" form: never an edge row, so each edge row holds a value"""
    k = 7 if which == 0 else 11
    return [i % k == 3 and i not in EDGE_ROWS for i in range(n)]


def arrow_array(t, vals):
    if t == "f32":
        bits = [0 if v is None else int(np.array([v], np.float32).view(np.uint32)[0]) for v in vals]
        arr = np.array(bits, np.uint32).view(np.float32)
        return pa.array(arr, pa.float32(), mask=np.array([v is None for v in vals]))
    if t == "f64":
        return pa.array(np.array([0.0 if v is None else v for v in vals], np.float64), pa.float64(),
                        mask=np.array([v is None for v in vals]))
    if is_dec(t):
        p, s = parse_dec(t)
        return pa.array([None if v is None else Decimal(v).scaleb(-s, CTX) for v in vals], pa.decimal128(p, s))
    return pa.array(vals, arrow_type(t))


def operands(t):
    """{name: python values} of the six operand columns of type t: a / b in each of the three forms"""
    out = {}
    for which, ab in ((0, "a"), (1, "b")):
        vals = column_values(t, which)
        nm = null_mask(which)
        out[f"{ab}_nn"] = vals
        out[f"{ab}_nv"] = vals
        out[f"{ab}_nl"] = [None if m else v for v, m in zip(vals, nm)]
    return out


def edge_table(t, values=None):
    """the table of type t's operand columns (a_nn, a_nv, a_nl, b_nn, b_nv, b_nl) and `row`; its plan schema"""
    values = values or operands(t)
    cols, schema = {}, []
    for name, vals in values.items():
        cols[name] = arrow_array(t, vals)
        schema.append(P.field(name, plan_type(t), not name.endswith("_nn")))
    cols["row"] = pa.array(range(len(next(iter(values.values())))), pa.int32())
    schema.append(P.field("row", "i32", False))
    return pa.table(cols), schema


def literal(t, v):
    """a literal of type t (floats through strings: JSON has no NaN / inf)"""
    if v is None:
        return P.lit_null(plan_type(t))
    if is_dec(t):
        return P.lit_dec(v, *parse_dec(t))
    if t in FLOATS:
        return {"lit": {"t": t, "v": repr(v) if math.isfinite(v) else ("nan" if math.isnan(v) else ("inf" if v > 0 else "-inf"))}}
    return {"lit": {"t": t, "v": str(v) if t == "u64" else v}}


def lit_operand(t):
    """the literal operand of the column-literal shapes: a value no edge pair turns into a failure with"""
    if t in FLOATS:
        return -2.5
    if is_dec(t):
        return 3 * 10 ** parse_dec(t)[1] + 1
    return 3


# ---- results -----------------------------------------------------------------------------------------------------------
def to_python(arr, t):
    """an engine's output column as reference values: decimals as unscaled integers, floats as Python floats"""
    vals = arr.to_pylist()
    if is_dec(t):
        s = parse_dec(t)[1]
        return [None if v is None else int(v.scaleb(s, CTX)) for v in vals]
    if t == "f32":
        a = arr.combine_chunks() if hasattr(arr, "combine_chunks") else arr
        bits = np.frombuffer(a.buffers()[1], np.uint32)[a.offset:a.offset + len(a)]
        return [None if v is None else f32_from_bits(int(b)) for v, b in zip(vals, bits)]
    return vals


def same(got, want, nan_sign=False, ulp=0):
    """bit-exact equality; NaN equals any NaN unless nan_sign (then the sign bit must agree); ulp: allowed distance in
    units of the last place for finite floats"""
    if got is None or want is None:
        return got is None and want is None
    if isinstance(want, float):
        if not isinstance(got, float):
            return False
        if math.isnan(want):
            return math.isnan(got) and (not nan_sign or math.copysign(1, got) == math.copysign(1, want))
        if ulp and math.isfinite(want) and got != 0 and want != 0:
            return abs(f64_bits(got) - f64_bits(want)) <= ulp
        return f64_bits(got) == f64_bits(want)
    return type(got) is type(want) and got == want


def mismatches(got, want, **kw):
    return [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if not same(g, w, **kw)]


# ---- operator matrix ---------------------------------------------------------------------------------------------------
OPS = ("+", "-", "*", "/", "%")
CMPS = ("=", "<>", "<", "<=", ">", ">=")


def result_type(op, ta, tb):
    if ta in FLOATS or tb in FLOATS:
        return "f32" if ta == tb == "f32" else "f64"
    if is_dec(ta) or is_dec(tb):
        da = parse_dec(ta) if is_dec(ta) else int_as_dec(ta)
        db = parse_dec(tb) if is_dec(tb) else int_as_dec(tb)
        return dec_name(*dec_result(op, da, db))
    return ta if ta == tb else "i64"


def arith2(op, a, ta, b, tb):
    """a op b for operands of types ta, tb (one type, or an integer next to a decimal)"""
    if a is None or b is None:
        return None
    rt = result_type(op, ta, tb)
    if is_dec(rt):
        da = parse_dec(ta) if is_dec(ta) else int_as_dec(ta)
        db = parse_dec(tb) if is_dec(tb) else int_as_dec(tb)
        return dec_op(op, a, da, b, db)
    return arith(op, a, b, rt)


def shapes(op, t, form):
    """(name, plan expression, per-row reference over the operand dict, result type) of the four operand shapes"""
    a, b = P.col(f"a_{form}"), P.col(f"b_{form}")
    L = lit_operand(t)
    lit = literal(t, L)
    inner_t = result_type(op, t, t)
    return [
        (f"cc_{form}", P.binop(op, a, b), lambda r: arith2(op, r[f"a_{form}"], t, r[f"b_{form}"], t), inner_t),
        (f"cl_{form}", P.binop(op, a, lit), lambda r: arith2(op, r[f"a_{form}"], t, L, t), inner_t),
        (f"lc_{form}", P.binop(op, lit, b), lambda r: arith2(op, L, t, r[f"b_{form}"], t), inner_t),
        # a register operand: (a op L) op b
        (f"nest_{form}", P.binop(op, P.binop(op, a, lit), b),
         lambda r: arith2(op, arith2(op, r[f"a_{form}"], t, L, t), inner_t, r[f"b_{form}"], t), result_type(op, inner_t, t)),
    ]


def zero_one(t):
    if is_dec(t):
        return 0, 10 ** parse_dec(t)[1]
    return (0.0, 1.0) if t in FLOATS else (0, 1)


def safe_operands(op, t):
    """the operand columns of type t with every row that fails one of op's shapes set to a = 0, b = 1 (which fails none):
    those rows' failures are the error tests' business"""
    vals = operands(t)
    z, o = zero_one(t)
    rows = [dict(zip(vals, r)) for r in zip(*vals.values())]
    for i, r in enumerate(rows):
        for form in FORMS:
            for _, _, ref, _ in shapes(op, t, form):
                try:
                    ref(r)
                except Raise:
                    for k in FORMS:
                        if vals[f"a_{k}"][i] is not None:
                            vals[f"a_{k}"][i] = z
                        if vals[f"b_{k}"][i] is not None:
                            vals[f"b_{k}"][i] = o
                    break
    return vals


def rows_of(vals):
    return [dict(zip(vals, r)) for r in zip(*vals.values())]


def project(exprs, table, schema):
    import queries as Q
    return [Q.Stage(1, P.shuffle_writer(P.project([(e, n) for n, e in exprs], P.scan(table, schema)), 1))]


def check_projection(engine, job, table, schema, rows, cases, **same_kw):
    """run the projection of `cases` ((name, expr, ref, result type)) and compare every column with the reference; returns
    the list of mismatches (name, result type, count, first rows).  A NaN's sign counts only where negation made it
    (columns named neg_*): the NaN f64 arithmetic produces is the platform's default NaN, whose sign differs by CPU."""
    from ballista_b200 import driver
    if len(cases) > 16:  # a pipeline materializes at most 32 output columns
        return [b for i in range(0, len(cases), 16) for b in check_projection(engine, f"{job}-{i}", table, schema, rows, cases[i:i + 16], **same_kw)]
    out = driver.run_stages(engine, project([(n, e) for n, e, _, _ in cases], table, schema), job)
    bad = []
    for name, _, ref, rt in cases:
        want = [ref(r) for r in rows]
        col = out.column(name)
        if col.type != arrow_type(rt):
            bad.append((name, rt, "type", str(col.type)))
            continue
        got = to_python(col, rt)
        mm = mismatches(got, want, nan_sign=name.startswith("neg") and rt == "f64", **same_kw)
        if mm:
            bad.append((name, rt, len(mm), mm[:3]))
    return bad


def cast_cases(frm, targets, rows):
    """(name, expr, ref, rt) for CAST(a_<form> AS to), skipping targets where some row raises (int -> decimal beyond the
    precision; those are the error tests' business); a ulp tolerance flag for decimal -> float above scale 22"""
    out = []
    for to in targets:
        ok = True
        for r in rows:
            try:
                cast(r["a_nn"], frm, to)
            except Raise:
                ok = False
                break
        if not ok:
            continue
        for form in FORMS:
            out.append((f"{to}_{form}", P.cast(P.col(f"a_{form}"), plan_type(to)), lambda r, to=to, form=form: cast(r[f"a_{form}"], frm, to), to))
    return out


# ---- the defects this suite was written for: one small table each ---------------------------------------------------------
U64_MAX = (1 << 64) - 1


def defect_cases():
    """(name, {column: (type, values)}, expression, expected values or Raise)"""
    big = (1 << 62) + (1 << 38) + 1
    return [
        ("u64_div", {"u": ("u64", [U64_MAX, 1 << 63, 7]), "v": ("u64", [2, 3, U64_MAX])}, P.binop("/", P.col("u"), P.col("v")),
         [(1 << 63) - 1, 3074457345618258602, 0]),
        ("u64_mod", {"u": ("u64", [U64_MAX, 1 << 63, 7]), "v": ("u64", [2, 3, U64_MAX])}, P.binop("%", P.col("u"), P.col("v")),
         [1, 2, 7]),
        ("u64_to_dec", {"u": ("u64", [U64_MAX, 1 << 63, 5])}, P.cast(P.col("u"), P.dec(20, 0)), [U64_MAX, 1 << 63, 5]),
        ("u64_plus_dec", {"u": ("u64", [U64_MAX, 1 << 63, 5]), "d": ("d5_2", [1, -1, 0])}, P.binop("+", P.col("u"), P.col("d")),
         [U64_MAX * 100 + 1, (1 << 63) * 100 - 1, 500]),
        ("u64_lt_dec", {"u": ("u64", [U64_MAX, 1 << 63, 5]), "d": ("d5_2", [99999, -99999, 500])}, P.binop("<", P.col("d"), P.col("u")),
         [True, True, False]),
        ("i32_to_u64", {"i": ("i32", [-5, 0, 2 ** 31 - 1])}, P.cast(P.col("i"), "u64"), [None, 0, 2 ** 31 - 1]),
        ("i64_to_u64", {"i": ("i64", [-1, -(1 << 63), 1 << 62])}, P.cast(P.col("i"), "u64"), [None, None, 1 << 62]),
        ("u64_to_i64", {"u": ("u64", [U64_MAX, 1 << 63, (1 << 63) - 1])}, P.cast(P.col("u"), "i64"), [None, None, (1 << 63) - 1]),
        ("u64_to_i16", {"u": ("u64", [U64_MAX, (1 << 64) - 32768, 5])}, P.cast(P.col("u"), "i16"), [None, None, 5]),
        ("f64_to_u64", {"f": ("f64", [-1.0, 2.0 ** 63, 2.0 ** 64, -0.5])}, P.cast(P.col("f"), "u64"), [None, 1 << 63, None, 0]),
        ("dec_to_u64", {"d": ("d38_0", [-1, 1 << 63, U64_MAX, U64_MAX + 1])}, P.cast(P.col("d"), "u64"), [None, 1 << 63, U64_MAX, None]),
        ("f64_to_dec_precision", {"f": ("f64", [1e10, 999.994, 999.995, -999.995])}, P.cast(P.col("f"), P.dec(5, 2)),
         [None, 99999, None, None]),
        ("i64_to_f32", {"l": ("i64", [big, -big, 3])}, P.cast(P.col("l"), "f32"),
         [float((1 << 62) + (1 << 39)), -float((1 << 62) + (1 << 39)), 3.0]),
        ("u64_to_f32", {"u": ("u64", [U64_MAX, (1 << 63) + (1 << 39) + 1])}, P.cast(P.col("u"), "f32"),
         [float(1 << 64), float((1 << 63) + (1 << 40))]),
        ("i32_div_minus1", {"i": ("i32", [5, -2 ** 31, 7]), "j": ("i32", [-1, -1, 2])}, P.binop("/", P.col("i"), P.col("j")), Raise),
        ("i8_div_minus1", {"i": ("i8", [-128]), "j": ("i8", [-1])}, P.binop("/", P.col("i"), P.col("j")), Raise),
        ("i32_mod_minus1", {"i": ("i32", [5, -2 ** 31]), "j": ("i32", [-1, -1])}, P.binop("%", P.col("i"), P.col("j")), [0, 0]),
        ("case_guards_div", {"l": ("i64", [10, 7, -9]), "b": ("i64", [2, 0, 4])},
         P.case([(P.binop("<>", P.col("b"), P.lit_i64(0)), P.binop("/", P.col("l"), P.col("b")))]), [5, None, -2]),
        ("case_else_guards_div", {"l": ("i64", [10, 7, -9]), "b": ("i64", [2, 0, 4])},
         P.case([(P.binop("=", P.col("b"), P.lit_i64(0)), P.lit_i64(-1))], P.binop("/", P.col("l"), P.col("b"))), [5, -1, -2]),
        ("case_when_guards_div", {"l": ("i64", [10, 7, -9]), "b": ("i64", [2, 0, 4])},
         P.case([(P.binop("=", P.col("b"), P.lit_i64(0)), P.lit_i64(0)),
                 (P.binop(">", P.binop("/", P.col("l"), P.col("b")), P.lit_i64(1)), P.lit_i64(1))], P.lit_i64(2)), [1, 0, 2]),
        ("case_guards_cast", {"l": ("i64", [10, 10 ** 12, -9])},
         P.case([(P.binop("<", P.col("l"), P.lit_i64(1000)), P.cast(P.col("l"), P.dec(5, 2)))]), [1000, None, -900]),
        ("case_guards_dec_overflow", {"d": ("d38_0", [10 ** 38 - 1, 5, -7])},
         P.case([(P.binop("<", P.col("d"), P.lit_dec(10 ** 20, 38, 0)), P.binop("*", P.col("d"), P.col("d")))]), [None, 25, 49]),
        ("neg_nan_sign", {"f": ("f64", [f64_from_bits(0x7FF8000000000000), f64_from_bits(0xFFF8000000000001), -0.0])},
         P.binop("<", P.neg(P.col("f")), P.lit_f64(0.0)), [True, False, False]),
    ]


def defect_table(cols):
    """cols: {name: (type, values)} -> (table, schema), every column nullable"""
    t = pa.table({n: arrow_array(ty, v) for n, (ty, v) in cols.items()})
    return t, [P.field(n, plan_type(ty), True) for n, (ty, _) in cols.items()]


def run_defect(engine, name, cols, expr, want):
    """None when the engine gives `want`, else a description of what it gave"""
    from ballista_b200 import driver, engine as E
    t, sch = defect_table(cols)
    import golden_data as G
    G.register(engine, "dfx", t, 1)
    st = project([("r", expr)], "dfx", sch)
    if want is Raise:
        try:
            driver.run_stages(engine, st, f"dfx-{name}")
        except Exception as ex:  # the device's B200Error, the oracle's OracleError: both carry the C ABI code
            return None if getattr(ex, "code", None) == -3 else f"error: {ex!r}"
        return "no error"
    out = driver.run_stages(engine, st, f"dfx-{name}")
    col = out.column("r")
    if pa.types.is_decimal(col.type):
        got = [None if v is None else int(v.scaleb(col.type.scale, CTX)) for v in col.to_pylist()]
    else:
        got = col.to_pylist()
    ok = len(got) == len(want) and all(same(g, w, nan_sign=True) if isinstance(w, float) else g == w and type(g) is type(w)
                                        for g, w in zip(got, want))
    return None if ok else f"{col.type}: {got} != {want}"
