"""Shared by the nested-loop join tests: input tables, filters over both sides, a stage plan around the join, and an
independent pure-Python evaluation (cross product + filter in three-valued logic) of what the join must return."""
from __future__ import annotations

import decimal
import math
import struct

import pyarrow as pa

from ballista_b200 import driver
from ballista_b200 import plan as P

JOIN_TYPES = ["Inner", "Left", "Right", "Full", "LeftSemi", "LeftAnti", "RightSemi", "RightAnti"]
D152, D124, D174 = P.dec(15, 2), P.dec(12, 4), P.dec(17, 4)
SCHEMA = pa.schema([("k", pa.int64()), ("i", pa.int32()), ("dt", pa.date32()), ("m", pa.decimal128(15, 2)),
                    ("m4", pa.decimal128(12, 4)), ("f", pa.float64()), ("s", pa.string()), ("u", pa.uint64())])
IR_SCHEMA = [P.field("k", "i64", True), P.field("i", "i32", True), P.field("dt", "date32", True), P.field("m", D152, True),
             P.field("m4", D124, True), P.field("f", "f64", True), P.field("s", "utf8", True), P.field("u", "u64", True)]
NC = len(IR_SCHEMA)
COL = {f["name"]: i for i, f in enumerate(IR_SCHEMA)}

_F = [float("nan"), -0.0, 0.0, 1.5, -2.25, float("inf"), float("-inf"), None, 3.0]
_S = ["", "a", "ab", "abc", "b", "é", "été", "zz", None, "aÿ", "B"]
_U = [0, 1, 2 ** 63, 2 ** 64 - 1, 2 ** 63 - 1, None, 7]


def make_table(n: int, seed: int, null_every: int = 5) -> pa.Table:
    """n rows with small value domains (so that comparisons tie often), NULLs in every column but k."""
    import random
    r = random.Random(seed)

    def maybe(v, row):
        return None if (row + seed) % null_every == 0 else v
    rows = {c: [] for c in SCHEMA.names}
    for row in range(n):
        rows["k"].append(row)
        rows["i"].append(maybe(r.randrange(-4, 5), row))
        rows["dt"].append(maybe(r.randrange(9000, 9006), row + 1))
        rows["m"].append(maybe(decimal.Decimal(r.randrange(-300, 300)).scaleb(-2), row + 2))
        rows["m4"].append(maybe(decimal.Decimal(r.randrange(-30000, 30000, 50)).scaleb(-4), row + 3))
        rows["f"].append(r.choice(_F))
        rows["s"].append(r.choice(_S))
        rows["u"].append(r.choice(_U))
    arrays = [pa.array(rows[c], type=SCHEMA.field(c).type) for c in SCHEMA.names]
    return pa.Table.from_arrays(arrays, schema=SCHEMA)


def L(name):
    return P.col(COL[name])


def R(name):
    return P.col(NC + COL[name])


def cmp(op, a, b):
    return P.binop(op, a, b)


# name -> filter over left ++ right (None: no filter).  Every separable shape, one-side terms, Kleene combinations.
FILTERS = {
    "none": None,
    "build_only": cmp(">", L("i"), P.lit_i32(0)),
    "probe_only": P.is_not_null(R("s")),
    "int_lt": cmp("<", L("i"), R("i")),
    "int_eq_flipped": cmp("=", R("i"), L("i")),
    "date_ge": cmp(">=", L("dt"), R("dt")),
    "dec_eq": cmp("=", L("m"), R("m")),
    "dec_cast_gt": cmp(">", P.cast(L("m"), D174), R("m4")),
    "f64_lt": cmp("<", L("f"), R("f")),
    "f64_eq": cmp("=", L("f"), R("f")),
    "utf8_lt": cmp("<", L("s"), R("s")),
    "utf8_ge_flipped": cmp(">=", R("s"), L("s")),
    "u64_gt": cmp(">", L("u"), R("u")),
    "band": P.and_(cmp(">=", R("i"), L("i")), cmp("<=", R("i"), P.binop("+", L("i"), P.lit_i32(2)))),
    "not_lt": P.not_(cmp("<", L("i"), R("i"))),
    "or_nulls": P.or_(cmp("=", L("i"), R("i")), P.not_(cmp(">", L("dt"), R("dt")))),
    "mixed": P.and_(P.or_(cmp("<>", L("s"), R("s")), P.is_null(R("i"))), P.not_(cmp("=", L("m"), R("m"))), cmp(">", L("i"), P.lit_i32(-3))),
}


# ---- independent evaluation ----------------------------------------------------------------------------------------
def _total_key(x: float) -> int:
    b = struct.unpack("<q", struct.pack("<d", x))[0]
    return b ^ ((b >> 63) & 0x7FFFFFFFFFFFFFFF)


def _value(e, row, types):
    """(value, type) of an expression over one concatenated row; value None = NULL."""
    if "col" in e:
        return row[e["col"]], types[e["col"]]
    if "lit" in e:
        t = e["lit"]["t"]
        v = e["lit"].get("v")
        if isinstance(t, dict) and v is not None:
            v = decimal.Decimal(int(v)).scaleb(-t["dec"][1])
        return v, t
    if "cast" in e:
        v, _t = _value(e["cast"], row, types)
        return v, e["to"]
    if "bin" in e and e["bin"] == "+":
        a, t = _value(e["l"], row, types)
        b, _ = _value(e["r"], row, types)
        return (None if a is None or b is None else a + b), t
    return _truth(e, row, types), "bool"


def _order(v, t):
    if t == "f64":
        return _total_key(v)
    if t == "utf8":
        return v.encode("utf-8")
    return v


def _truth(e, row, types):
    """Three-valued: True / False / None."""
    if "bin" in e and e["bin"] in ("and", "or"):
        a, b = _truth(e["l"], row, types), _truth(e["r"], row, types)
        if e["bin"] == "and":
            if a is False or b is False:
                return False
            return None if a is None or b is None else True
        if a is True or b is True:
            return True
        return None if a is None or b is None else False
    if "not" in e:
        a = _truth(e["not"], row, types)
        return None if a is None else not a
    if "is_null" in e:
        return _value(e["is_null"], row, types)[0] is None
    if "is_not_null" in e:
        return _value(e["is_not_null"], row, types)[0] is not None
    if "bin" in e:
        (a, ta), (b, tb) = _value(e["l"], row, types), _value(e["r"], row, types)
        if a is None or b is None:
            return None
        x, y = _order(a, ta), _order(b, tb)
        return {"=": x == y, "!=": x != y, "<>": x != y, "<": x < y, "<=": x <= y, ">": x > y, ">=": x >= y}[e["bin"]]
    if "col" in e or "lit" in e:
        return _value(e, row, types)[0]
    raise ValueError(f"expression not covered by the reference evaluator: {e}")


def reference_join(left: pa.Table, right: pa.Table, join_type: str, filt, projection=None):
    """Rows (as tuples, in the join's output order: pairs by probe row then build row, unmatched build rows, unmatched
    probe rows) of NestedLoopJoinExec over `left` (build) and `right` (probe)."""
    lrows, rrows = left.to_pylist(), right.to_pylist()
    lt = [list(r.values()) for r in lrows]
    rt = [list(r.values()) for r in rrows]
    types = [f["type"] for f in IR_SCHEMA] * 2
    pairs = []
    for j, pr in enumerate(rt):
        for i, br in enumerate(lt):
            if filt is None or _truth(filt, br + pr, types) is True:
                pairs.append((i, j))
    lm = {i for i, _ in pairs}
    rm = {j for _, j in pairs}
    nulls = [None] * NC
    if join_type == "LeftSemi":
        return [tuple(lt[i]) for i in range(len(lt)) if i in lm]
    if join_type == "LeftAnti":
        return [tuple(lt[i]) for i in range(len(lt)) if i not in lm]
    if join_type == "RightSemi":
        return [tuple(rt[j]) for j in range(len(rt)) if j in rm]
    if join_type == "RightAnti":
        return [tuple(rt[j]) for j in range(len(rt)) if j not in rm]
    out = [lt[i] + rt[j] for i, j in pairs]
    if join_type in ("Left", "Full"):
        out += [lt[i] + nulls for i in range(len(lt)) if i not in lm]
    if join_type in ("Right", "Full"):
        out += [nulls + rt[j] for j in range(len(rt)) if j not in rm]
    if projection is not None:
        out = [[r[c] for c in projection] for r in out]
    return [tuple(r) for r in out]


# ---- running the join on an engine ---------------------------------------------------------------------------------
def join_stage(join_type: str, filt, projection=None, schema=None):
    sch = schema or IR_SCHEMA
    j = P.nested_loop_join(P.scan("nlj_l", sch), P.scan("nlj_r", sch), join_type, filter=filt, projection=projection)
    return [P.Stage(1, P.shuffle_writer(j, 1))]


def register(engine, left: pa.Table, right: pa.Table, probe_parts: int = 1):
    for t in ("nlj_l", "nlj_r"):
        try:
            engine.drop_table(t)
        except Exception:
            pass
    engine.register_batch("nlj_l", 0, left.combine_chunks().to_batches()[0] if left.num_rows else pa.RecordBatch.from_pylist([], schema=left.schema))
    n = right.num_rows
    for p in range(probe_parts):
        part = right.slice(n * p // probe_parts, n * (p + 1) // probe_parts - n * p // probe_parts).combine_chunks()
        engine.register_batch("nlj_r", p, part.to_batches()[0] if part.num_rows else pa.RecordBatch.from_pylist([], schema=right.schema))


def run_join(engine, job: str, join_type: str, filt, projection=None):
    return driver.run_stages(engine, join_stage(join_type, filt, projection), job)


def rows_of(table):
    if table is None:
        return []
    return list(zip(*[c.to_pylist() for c in table.columns]))   # by position: both sides have the same column names


def canon_rows(rows):
    """Multiset order for comparisons that ignore the output order (NaN made comparable)."""
    def key(v):
        if v is None:
            return (0, "")
        if isinstance(v, float):
            return (1, _total_key(v))
        return (2, repr(v))
    return sorted(rows, key=lambda r: tuple(key(v) for v in r))


def same_rows(a, b):
    """Row lists equal value by value (NaN equal to NaN, -0.0 distinct from 0.0)."""
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            if isinstance(u, float) and isinstance(v, float):
                if _total_key(u) != _total_key(v):
                    return False
            elif u != v:
                return False
    return True


def is_nan(v):
    return isinstance(v, float) and math.isnan(v)
