"""AggregateExec without a GPU.  First the plain-Python reference of aggregate_cases is pinned against independent
implementations where their semantics coincide with DataFusion's:
- pyarrow's Table.group_by(...).aggregate(...) and sqlite3, for integer, decimal and string keys, on inputs whose sums
  do not overflow;
- Python's `decimal` at 80 digits, for decimal AVG;
- the struct bit patterns, for the total order of float MIN / MAX.
Left out of those comparisons, with the reason:
- float keys: pyarrow and sqlite put -0.0 with 0.0 and every NaN in one group; the engine keys floats by bit pattern;
- float MIN / MAX with NaN or -0.0: pyarrow skips NaN and sqlite has no NaN; the engine uses the IEEE total order;
- wrapping sums: pyarrow's checked sums and sqlite's integers raise or promote on overflow; the engine wraps;
- float SUM / AVG: the other implementations round in their own order; the reference is exact.
Then the CPU oracle is checked against the reference over the whole matrix of aggregate_cases."""
import decimal
import sqlite3
import struct

import pyarrow as pa
import pytest

from ballista_b200 import plan as P
import aggregate_cases as A


# ---- the reference against independent implementations ------------------------------------------------------------
def _int_table(n=600, seed=3):
    import random
    r = random.Random(seed)
    return pa.table({"k": pa.array([r.choice([None, -7, 0, 3, 2 ** 40]) for _ in range(n)], pa.int64()),
                     "s": pa.array([r.choice([None, "", "a", "a\0", "abcdefgh", "é"]) for _ in range(n)], pa.string()),
                     "d": pa.array([None if r.random() < 0.2 else decimal.Decimal(r.randrange(-10 ** 12, 10 ** 12)).scaleb(-3)
                                    for _ in range(n)], pa.decimal128(20, 3)),
                     "v": pa.array([None if r.random() < 0.2 else r.randrange(-10 ** 12, 10 ** 12) for _ in range(n)], pa.int64())})


def _ref(table, keys, specs):
    aggs = [(fn, a, f"{fn}_{a}") for fn, a in specs]
    return A.reference(table, keys, aggs)


@pytest.mark.parametrize("key", ["k", "s", "d"])
def test_reference_matches_pyarrow_group_by(key):
    t = _int_table()
    specs = [("count_star", None), ("count", "v"), ("sum", "v"), ("min", "v"), ("max", "v"), ("sum", "d"), ("min", "s"), ("max", "s")]
    want = _ref(t, [key], specs)
    pa_aggs = [([], "count_all"), ("v", "count"), ("v", "sum"), ("v", "min"), ("v", "max"), ("d", "sum"), ("s", "min"), ("s", "max")]
    got = t.group_by(key, use_threads=False).aggregate(pa_aggs)
    kv = A.raw_values(got.column(key))
    cols = [A.raw_values(got.column(n)) for n in got.column_names if n != key]
    assert len(kv) == len(want)
    for r, k in enumerate(kv):
        row = [col[r] for col in cols]
        w = want[A.key_of([k])]
        assert row == w, (k, row, w)


def test_reference_matches_sqlite():
    t = _int_table(seed=5)
    db = sqlite3.connect(":memory:")
    db.execute("CREATE TABLE t (k INTEGER, s TEXT, v INTEGER)")
    db.executemany("INSERT INTO t VALUES (?, ?, ?)", zip(*(t.column(n).to_pylist() for n in ("k", "s", "v"))))
    for key in ("k", "s"):
        rows = db.execute(f"SELECT {key}, COUNT(*), COUNT(v), SUM(v), MIN(v), MAX(v), MIN(s), MAX(s) FROM t GROUP BY {key}").fetchall()
        want = _ref(t, [key], [("count_star", None), ("count", "v"), ("sum", "v"), ("min", "v"), ("max", "v"), ("min", "s"), ("max", "s")])
        assert len(rows) == len(want)
        for k, *vals in rows:
            assert vals == want[A.key_of([k])], (key, k)


def test_reference_decimal_avg_matches_80_digit_decimal():
    ctx = decimal.Context(prec=80, rounding=decimal.ROUND_DOWN)
    import random
    r = random.Random(9)
    for t in ("d5_2", "d15_2", "d18_0", "d20_3", "d38_0", "d38_10"):
        p, s = A.TYPES[t][3]
        rp, rs = min(38, p + 4), min(38, s + 4)
        for _ in range(40):
            xs = [r.randrange(-10 ** p + 1, 10 ** p) for _ in range(r.randrange(1, 9))]
            try:
                got = A.aggregate_values("avg", t, xs)
            except A.AggOverflow:
                got = None
            exact = ctx.divide(sum(decimal.Decimal(x) for x in xs).scaleb(-s), decimal.Decimal(len(xs)))
            q = int(exact.scaleb(rs).to_integral_value(rounding=decimal.ROUND_DOWN))
            ok = abs(q) < 10 ** rp and abs(sum(xs) * 10 ** (rs - s)) < 2 ** 127
            assert got == (q if ok else None), (t, xs)


def test_reference_decimal_avg_errors():
    # one Decimal(38, 0) row of 9e33: 9e37 as Decimal(38, 4) fits both i128 and 38 digits
    assert A.aggregate_values("avg", "d38_0", [9 * 10 ** 33]) == 9 * 10 ** 37
    # 1.5e34 * 10^4 fits i128 (< 1.7e38) but not 38 digits
    with pytest.raises(A.AggOverflow, match="precision"):
        A.aggregate_values("avg", "d38_0", [15 * 10 ** 33])
    # 2e34 * 10^4 leaves i128
    with pytest.raises(A.AggOverflow, match="i128"):
        A.aggregate_values("avg", "d38_0", [2 * 10 ** 34])
    # truncation toward zero
    assert A.aggregate_values("avg", "d5_2", [-1, -1, 0]) == -6666


def test_reference_float_total_order_and_wrapping():
    def b(x):
        return struct.unpack("<Q", struct.pack("<d", x))[0]
    order = [0xFFF80000000000A5, 0xFFF8000000000000, b(float("-inf")), b(-1.0), b(-5e-324), b(-0.0), b(0.0), b(5e-324), b(1.0),
             b(float("inf")), 0x7FF0000000000001, 0x7FF8000000000000, 0x7FF8000000000123]
    for i in range(len(order)):
        for j in range(i, len(order)):
            assert A.aggregate_values("min", "f64", [order[j], order[i]]) == order[i]
            assert A.aggregate_values("max", "f64", [order[i], order[j]]) == order[j]
    assert A.aggregate_values("sum", "i64", [2 ** 63 - 1, 1]) == -2 ** 63
    assert A.aggregate_values("sum", "u64", [2 ** 64 - 1, 2]) == 1
    assert A.aggregate_values("sum", "d38_0", [2 ** 126, 2 ** 126]) == -2 ** 127
    assert A.aggregate_values("sum", "f64", [b(float("inf")), b(float("-inf"))]).exact == "nan"
    assert A.aggregate_values("min", "utf8", ["a\0", "a", "é", "z"]) == "a"


def test_result_types_match_the_typed_plan():
    """The engine's typing of each aggregate is the result type written down in aggregate_cases."""
    import json
    from ballista_b200 import engine
    arrow_of = {v[2]: v[1] for v in A.TYPES.values() if isinstance(v[2], str)}

    def to_arrow(t):
        return pa.decimal128(*t["dec"]) if isinstance(t, dict) else arrow_of[t]
    t = A.arg_table(4)
    sch = A.ir_schema(t)
    idx = {f["name"]: i for i, f in enumerate(sch)}
    for typ in A.TYPES:
        for fns in A.fn_groups(typ):
            aggs = A.arg_aggs(typ, "n", fns)
            node = P.aggregate("Single", [(P.col(idx["g"]), "g")],
                               [P.agg(A.FN_IR[fn], None if a is None else P.col(idx[a]), nm) for fn, a, nm in aggs], P.scan("agg_t", sch))
            typed = json.loads(engine.plan_typed_json(json.dumps(node)))["schema"][1:]
            assert [to_arrow(f["type"]) for f in typed] == [A.result_type(fn, None if a is None else typ) for fn, a, _ in aggs], typ


# ---- the oracle against the reference ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def arg_table():
    return A.arg_table(1100)


@pytest.mark.parametrize("mode", A.MODES)
@pytest.mark.parametrize("typ", list(A.TYPES))
def test_oracle_arguments(oracle, arg_table, typ, mode):
    for form in A.FORMS:
        for fns in A.fn_groups(typ):
            A.check(oracle, arg_table, mode, ["g"], A.arg_aggs(typ, form, fns), f"oa-{typ}-{form}-{mode}")


@pytest.mark.parametrize("typ", ["i64", "u64", "f32", "d38_0", "utf8"])
def test_oracle_scalar_and_empty(oracle, arg_table, typ):
    for n in (0, 1, 1100):
        t = arg_table.slice(0, n)
        for fns in A.fn_groups(typ):
            A.check(oracle, t, "final", [], A.arg_aggs(typ, "n", fns), f"os-{typ}-{n}")
            A.check(oracle, t, "single", [], A.arg_aggs(typ, "nn", fns), f"os1-{typ}-{n}")
        if n == 0:
            got = A.run(oracle, t, "final_partitioned", ["g"], A.arg_aggs(typ, "n", ["count_star", "max"]), f"oe-{typ}")
            assert got.num_rows == 0


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("mode", A.MODES)
@pytest.mark.parametrize("shape", sorted(A.KEY_SHAPES))
def test_oracle_keys(oracle, shape, mode, nullable):
    table, keys = A.key_table(shape, 700, seed=len(shape), nullable=nullable)
    A.check(oracle, table, mode, keys, A.KEY_AGGS, f"ok-{shape}-{mode}")


@pytest.mark.parametrize("t", ["f32", "f64"])
def test_oracle_groups_float_keys_by_bits(oracle, t):
    """-0.0 and 0.0 are two groups and keep their signs; every NaN payload is a group of its own."""
    dom = A.F32_EDGES if t == "f32" else A.F64_EDGES
    vals = dom * 3
    table = A.make_table(["i64"], len(vals), 1, {f"k_{t}": (t, vals)})
    got = A.check(oracle, table, "single", [f"k_{t}"], [("count_star", None, "cnt")], f"of-{t}")
    assert sorted(A.raw_values(got.column(0))) == sorted(dom)


def test_oracle_float32_signalling_nan(oracle):
    table = A.snan_table()
    want = A.reference(table, ["g"], A.SNAN_AGGS)
    assert [want[(g,)][:2] for g in range(4)] == [[0x3F800000, 0x7FC00000], [0xFF800000, 0x7F800001], [0xFF800001, 0xBF800000],
                                                 [0xFFC00000, 0xFF800001]]
    for mode in A.MODES:
        A.check(oracle, table, mode, ["g"], A.SNAN_AGGS, f"osn-{mode}", want=want)
        got = A.check(oracle, table, mode, ["kf"], [("count_star", None, "c")], f"osk-{mode}")
        assert sorted(A.raw_values(got.column(0))) == [0x7F800001, 0x7FC00001]


def test_oracle_decimal_avg_overflow(oracle):
    for v, fails in ((9 * 10 ** 33, False), (15 * 10 ** 33, True), (2 * 10 ** 34, True)):
        table = A.make_table([], 1, 1, {"k": ("i64", [1]), "x": ("d38_0", [v])})
        aggs = [("avg", "x", "a")]
        if fails:
            with pytest.raises(Exception, match="overflow"):
                A.run(oracle, table, "single", ["k"], aggs, "oav")
        else:
            A.check(oracle, table, "single", ["k"], aggs, "oav")
