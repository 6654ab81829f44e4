"""Shared by the hash join tests: build and probe tables with a key column of every type the engine joins on, stage plans
around HashJoinExec (CollectLeft over scans, Partitioned behind a two-stage hash shuffle), a plain-Python reference of
what the join must return, and a pair of distinct two-column Int64 keys whose row hashes collide.

Key equality in the reference is the engine's `=`: floats are equal when their bit patterns are (NaN = NaN only with the
same payload, -0.0 <> 0.0), strings when their UTF-8 bytes are, decimals when their unscaled integers are.  A NULL in
any key keeps the row from matching unless the join has null_equals_null, where NULL matches NULL column by column."""
from __future__ import annotations

import decimal
import random
import struct
from collections import Counter

import numpy as np
import pyarrow as pa

from ballista_b200 import driver
from ballista_b200 import plan as P
import nlj_cases as N

JOIN_TYPES = N.JOIN_TYPES
DEC = P.dec(38, 3)

# name -> (arrow type, IR type, value domain).  Small domains, so that keys repeat on both sides.
_D = decimal.Decimal
KEY_TYPES = {
    "i8": (pa.int8(), "i8", [-128, -1, 0, 1, 127]),
    "i16": (pa.int16(), "i16", [-32768, -1, 0, 2, 32767]),
    "i32": (pa.int32(), "i32", [-2 ** 31, -1, 0, 3, 2 ** 31 - 1]),
    "i64": (pa.int64(), "i64", [-2 ** 63, -1, 0, 4, 2 ** 63 - 1]),
    "u8": (pa.uint8(), "u8", [0, 1, 200, 255]),
    "u16": (pa.uint16(), "u16", [0, 1, 40000, 65535]),
    "u32": (pa.uint32(), "u32", [0, 1, 2 ** 31, 2 ** 32 - 1]),
    "u64": (pa.uint64(), "u64", [0, 1, 2 ** 63, 2 ** 64 - 1]),
    "date32": (pa.date32(), "date32", [-1, 0, 9000, 19000]),
    "ts": (pa.timestamp("ns"), "ts", [-1, 0, 1_600_000_000_000_000_000, 9_000_000_000_000_000_000]),
    "dec": (pa.decimal128(38, 3), DEC, [_D("-1.000"), _D("0.000"), _D("0.001"), _D(2 ** 70).scaleb(-3), _D(-2 ** 70).scaleb(-3)]),
    "utf8": (pa.string(), "utf8", ["", "a", "ab", "é", "日本語", "abcdefghijklmn", "abcdefghijklmo", "a string of twenty-b", "a string of twenty-c"]),
    "bool": (pa.bool_(), "bool", [True, False]),
    # floats as bit patterns: -0.0, 0.0, +inf, -inf, two quiet NaN payloads, a negative NaN, 1.5
    "f32": (pa.float32(), "f32", [0x80000000, 0x00000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7FC00001, 0xFFC00000, 0x3FC00000]),
    "f64": (pa.float64(), "f64", [0x8000000000000000, 0, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000, 0x7FF8000000000001,
                                  0xFFF8000000000000, 0x3FF8000000000000]),
}
KEYS = list(KEY_TYPES)
NAMES = ["id"] + [f"k_{t}" for t in KEYS]
SCHEMA = pa.schema([("id", pa.int64())] + [(f"k_{t}", KEY_TYPES[t][0]) for t in KEYS])
IR_SCHEMA = [P.field("id", "i64", True)] + [P.field(f"k_{t}", KEY_TYPES[t][1], True) for t in KEYS]
NC = len(IR_SCHEMA)
COL = {n: i for i, n in enumerate(NAMES)}

# key shapes: name -> key columns (the same columns on both sides)
SHAPES = {t: [f"k_{t}"] for t in KEYS}
SHAPES["i32_utf8"] = ["k_i32", "k_utf8"]
SHAPES["i16_dec_date32"] = ["k_i16", "k_dec", "k_date32"]


def L(name):
    return P.col(COL[name])


def R(name):
    return P.col(NC + COL[name])


# residual filters over left ++ right, in what nlj_cases._truth evaluates (three-valued, NULLs on both sides)
FILTERS = {
    "none": None,
    "id_or_null": P.or_(P.binop(">", L("id"), R("id")), P.is_null(L("k_u8"))),
}


def _float_array(bits, typ, mask):
    u, f = (np.uint32, np.float32) if typ == pa.float32() else (np.uint64, np.float64)
    return pa.array(np.array(bits, dtype=u).view(f), type=typ, mask=np.array(mask, dtype=bool))


def make_table(n: int, seed: int, null_every: int = 6, domains=None) -> pa.Table:
    """n rows: id = row number (never NULL), then one key column per type drawn from its small domain, NULL in about
    one row in `null_every` of every key column.  `domains` overrides the domain of some types."""
    r = random.Random(seed)
    cols = [pa.array(list(range(n)), pa.int64())]
    for c, t in enumerate(KEYS):
        typ, _ir, dom = KEY_TYPES[t]
        dom = (domains or {}).get(t, dom)
        vals = [r.choice(dom) for _ in range(n)]
        nulls = [r.randrange(null_every) == 0 for _ in range(n)]
        if t in ("f32", "f64"):
            cols.append(_float_array(vals, typ, nulls))
        elif t in ("date32", "ts"):
            cols.append(pa.array([None if m else v for v, m in zip(vals, nulls)], pa.int64()).cast(pa.int32() if t == "date32" else pa.int64()).view(typ))
        else:
            cols.append(pa.array([None if m else v for v, m in zip(vals, nulls)], typ))
    return pa.Table.from_arrays(cols, schema=SCHEMA)


# ---- reference ------------------------------------------------------------------------------------------------------
def key_values(table: pa.Table, name: str):
    """Canonical equality key of every row of a column (None = NULL): floats by bit pattern, strings by UTF-8 bytes,
    decimals by the unscaled integer, temporal types by their integer."""
    arr = table.column(name).combine_chunks()
    valid = arr.is_valid().to_pylist()
    t = arr.type
    if pa.types.is_floating(t):
        u = np.uint32 if t == pa.float32() else np.uint64
        bits = np.frombuffer(arr.buffers()[1], dtype=u)[arr.offset:arr.offset + len(arr)] if len(arr) else []
        return [("f", int(b)) if v else None for b, v in zip(bits, valid)]
    if pa.types.is_decimal(t):
        return [("d", int(x.scaleb(t.scale))) if x is not None else None for x in arr.to_pylist()]
    if pa.types.is_string(t):
        return [("s", x.encode("utf-8")) if x is not None else None for x in arr.to_pylist()]
    if pa.types.is_date32(t) or pa.types.is_timestamp(t):
        return arr.view(pa.int32() if pa.types.is_date32(t) else pa.int64()).to_pylist()
    return arr.to_pylist()


def reference_hash_join(left: pa.Table, right: pa.Table, on, join_type: str, filt=None, projection=None, null_equals_null=False,
                        ir_schema=None):
    """Rows (as tuples, as multisets: the hash join's pair order depends on its atomics) of HashJoinExec with `left` as the
    build side.  `on`: [(left key, right key)], each a column name or the list of key_values of a computed key."""
    ir_schema = ir_schema or IR_SCHEMA

    def keys(table, ks):
        return list(zip(*[k if isinstance(k, list) else key_values(table, k) for k in ks])) if table.num_rows else []
    lk, rk = keys(left, [a for a, _ in on]), keys(right, [b for _, b in on])
    table = {}
    for i, k in enumerate(lk):
        if None in k and not null_equals_null:
            continue
        table.setdefault(k, []).append(i)
    lt = [list(r.values()) for r in left.to_pylist()]
    rt = [list(r.values()) for r in right.to_pylist()]
    types = [f["type"] for f in ir_schema] * 2
    pairs = []
    for j, k in enumerate(rk):
        if None in k and not null_equals_null:
            continue
        for i in table.get(k, ()):
            if filt is None or N._truth(filt, lt[i] + rt[j], types) is True:
                pairs.append((i, j))
    lm = {i for i, _ in pairs}
    rm = {j for _, j in pairs}
    nc = len(ir_schema)
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
        out += [lt[i] + [None] * nc for i in range(len(lt)) if i not in lm]
    if join_type in ("Right", "Full"):
        out += [[None] * nc + rt[j] for j in range(len(rt)) if j not in rm]
    if projection is not None:
        out = [[r[c] for c in projection] for r in out]
    return [tuple(r) for r in out]


def _canon(v):
    return ("f", struct.pack("<d", v)) if type(v) is float else v   # -0.0 <> 0.0, NaN by payload


def same_multiset(got, want):
    """Equal as multisets of rows, floats compared by bit pattern."""
    return len(got) == len(want) and Counter(tuple(map(_canon, r)) for r in got) == Counter(tuple(map(_canon, r)) for r in want)


# ---- plans and running them -----------------------------------------------------------------------------------------
def on_cols(keys, ir_schema=None):
    idx = {f["name"]: i for i, f in enumerate(ir_schema or IR_SCHEMA)}
    return [[P.col(idx[k]), P.col(idx[k])] for k in keys]


def collect_left_stages(keys, join_type, filt=None, projection=None, null_equals_null=False, ir_schema=None, left=None, right=None):
    """One stage: HashJoinExec(CollectLeft) over the scans hj_l (build, read whole by every task) and hj_r (probe)."""
    sch = ir_schema or IR_SCHEMA
    j = P.hash_join(left or P.scan("hj_l", sch), right or P.scan("hj_r", sch), on_cols(keys, sch), join_type, "CollectLeft", filter=filt,
                    projection=projection, null_equals_null=null_equals_null)
    return [P.Stage(1, P.shuffle_writer(j, 1))]


def partitioned_stages(keys, join_type, filt=None, projection=None, null_equals_null=False, n_parts=4, ir_schema=None):
    """Stages 1 and 2 hash-repartition hj_l and hj_r on the keys into n_parts partitions; stage 3 joins partition p of
    one with partition p of the other (HashJoinExec, Partitioned)."""
    sch = ir_schema or IR_SCHEMA
    on = on_cols(keys, sch)
    s1 = P.Stage(1, P.shuffle_writer(P.scan("hj_l", sch), 1, [a for a, _ in on], n_parts))
    s2 = P.Stage(2, P.shuffle_writer(P.scan("hj_r", sch), 2, [b for _, b in on], n_parts))
    j = P.hash_join(P.shuffle_reader(1, sch), P.shuffle_reader(2, sch), on, join_type, "Partitioned", filter=filt, projection=projection,
                    null_equals_null=null_equals_null)
    return [s1, s2, P.Stage(3, P.shuffle_writer(j, 3))]


def _register(engine, name, table, parts):
    try:
        engine.drop_table(name)
    except Exception:
        pass
    n = table.num_rows
    for p in range(parts):
        part = table.slice(n * p // parts, n * (p + 1) // parts - n * p // parts).combine_chunks()
        engine.register_batch(name, p, part.to_batches()[0] if part.num_rows else pa.RecordBatch.from_pylist([], schema=table.schema))


def register(engine, left: pa.Table, right: pa.Table, build_parts: int = 1, probe_parts: int = 1):
    _register(engine, "hj_l", left, build_parts)
    _register(engine, "hj_r", right, probe_parts)


def run(engine, stages, job):
    return N.rows_of(driver.run_stages(engine, stages, job))


# ---- a forced 64-bit row-hash collision ----------------------------------------------------------------------------
M64 = (1 << 64) - 1
_SEED = 0x9E3779B97F4A7C15


def _unxorshift(y, s):
    x = y
    for _ in range(64 // s + 1):
        x = y ^ (x >> s)
    return x & M64


def unmix64(h):
    """Inverse of hash.hpp's mix64 (a bijection: xor-shifts and multiplications by odd constants)."""
    x = _unxorshift(h & M64, 31)
    x = (x * pow(0x94d049bb133111eb, -1, 1 << 64)) & M64
    x = _unxorshift(x, 27)
    x = (x * pow(0xbf58476d1ce4e5b9, -1, 1 << 64)) & M64
    return _unxorshift(x, 30)


def _i64(u):
    return u - (1 << 64) if u >= 1 << 63 else u


def colliding_keys(a1=0, b1=0, b2=1):
    """Two distinct (a, b) Int64 keys with equal row hashes combine_hashes(hash_i64(b), hash_i64(a)): (a1, b1) and
    (a2, b2), a2 found by inverting combine_hashes (an odd multiplier, invertible mod 2^64) and hash_i64."""
    def h(v):
        return _mix64((v + _SEED) & M64)
    target = ((17 * 37 + h(b1)) * 37 + h(a1)) & M64
    ha2 = (target - (17 * 37 + h(b2)) * 37) & M64
    a2 = _i64((unmix64(ha2) - _SEED) & M64)
    return (a1, b1), (a2, b2)


def _mix64(x):
    x &= M64
    x ^= x >> 30
    x = (x * 0xbf58476d1ce4e5b9) & M64
    x ^= x >> 27
    x = (x * 0x94d049bb133111eb) & M64
    x ^= x >> 31
    return x
