"""Grouping sets and the bitwise operators without a GPU: the protobuf fixtures decode to the typed plans they were written
from, refusals carry their code and name, the typing rules of DESIGN.md §6, and the UNION ALL form the GPU tests compare
against (grouping_set_cases.expected, on the CPU oracle) against sqlite3."""
import base64
import json
import os
import sqlite3

import pyarrow as pa
import pytest

import golden_data as G
import grouping_set_cases as GC
from ballista_b200 import engine
from ballista_b200 import plan as P

c = P.col
FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "grouping_set_proto_plans.json")


def _cases():
    with open(FIXTURES) as f:
        return json.load(f)["cases"]


def _typed(ir: str) -> dict:
    return json.loads(engine.plan_typed_json(ir))


@pytest.mark.parametrize("case", [cs for cs in _cases() if "refuse" not in cs], ids=lambda cs: cs["name"])
def test_fixture_decodes_to_its_plan(case):
    for st in case["stages"]:
        decoded = engine.plan_proto_to_json(base64.b64decode(st["proto_b64"]), "job")
        assert _typed(decoded) == _typed(st["ir"]), st["name"]


@pytest.mark.parametrize("case", [cs for cs in _cases() if "refuse" in cs], ids=lambda cs: cs["name"])
def test_fixture_refusals_carry_code_and_name(case):
    with pytest.raises(engine.B200Error) as ei:
        _typed(engine.plan_proto_to_json(base64.b64decode(case["stages"][0]["proto_b64"]), "job"))
    assert ei.value.code == case["refuse"]["code"], str(ei.value)
    assert case["refuse"]["match"] in str(ei.value)


def test_typing_rules():
    scan = P.scan("t", GC.SCHEMA)
    for n in (1, 3, 7):
        names = ["ks", "ki", "kd", "kt", "kf", "kb", "n"][:n]
        t = _typed(json.dumps(P.aggregate("Partial", [(c(k), k) for k in names], [P.agg("sum", c("v"), "s")], scan,
                                          grouping_sets=P.rollup_sets(n))))
        sch = t["schema"]
        assert all(f["nullable"] for f in sch[:n])
        assert sch[n] == {"name": "__grouping_id", "type": "u8", "nullable": False}
        assert t["grouping_sets"] == P.rollup_sets(n)
    # a plain GROUP BY keeps its key nullability and gets no id
    t = _typed(json.dumps(P.aggregate("Single", [(c("ki"), "ki")], [P.agg("count", None, "n")], P.scan("t", [P.field("ki", "i32")]))))
    assert [f["name"] for f in t["schema"]] == ["ki", "n"] and not t["schema"][0]["nullable"] and "grouping_sets" not in t


@pytest.mark.parametrize("bad, code, match", [
    (dict(grouping_sets=[[False], [False]]), -2, "duplicate grouping set 1"),
    (dict(grouping_sets=[[True, False]]), -1, "has 2 entries for 1 keys"),
    (dict(grouping_sets=[]), -1, "empty grouping_sets"),
    (dict(mode="Final"), -1, "Final-mode aggregate carries no grouping sets"),
])
def test_refusals(bad, code, match):
    node = P.aggregate(bad.get("mode", "Single"), [(c("ki"), "ki")], [P.agg("count", None, "n")], P.scan("t", GC.SCHEMA),
                       grouping_sets=bad.get("grouping_sets", [[True]]))
    with pytest.raises(engine.B200Error) as ei:
        _typed(json.dumps(node))
    assert ei.value.code == code and match in str(ei.value), str(ei.value)


def test_more_than_32_sets_is_refused():
    names = ["ks", "ki", "kd", "kt", "kf", "kb"]
    node = P.aggregate("Single", [(c(k), k) for k in names], [P.agg("count", None, "n")], P.scan("t", GC.SCHEMA), grouping_sets=P.cube_sets(6))
    with pytest.raises(engine.B200Error) as ei:
        _typed(json.dumps(node))
    assert ei.value.code == -2 and "64 grouping sets" in str(ei.value)


@pytest.mark.parametrize("ty", ["i8", "i16", "i32", "i64", "u8", "u16", "u32", "u64"])
def test_bitwise_typing(ty):
    scan = P.scan("t", [P.field("a", ty, True), P.field("b", ty), P.field("x", "f64")])
    t = _typed(json.dumps(P.project([(P.binop(op, c("a"), c("b")), op) for op in ["&", "|", "^", "<<", ">>"]], scan)))
    assert [(f["type"], f["nullable"]) for f in t["schema"]] == [(ty, True)] * 5
    for other in (P.binop("&", c("a"), c("x")), P.binop("<<", c("a"), P.lit_f64(1.0))):
        with pytest.raises(engine.B200Error) as ei:
            _typed(json.dumps(P.project([(other, "bad")], scan)))
        assert ei.value.code == -2


def test_oracle_refuses_grouping_sets_and_bitwise(oracle):
    from ballista_b200 import driver
    t = GC.make_table(10, seed=1)
    GC.register(oracle, "gs", t, 1)
    scan = P.scan("gs", GC.SCHEMA)
    for plan in (P.aggregate("Single", [(c("ki"), "ki")], [P.agg("count", None, "n")], scan, grouping_sets=P.rollup_sets(1)),
                 P.project([(P.binop("&", c("ki"), c("ki")), "x")], scan)):
        with pytest.raises(Exception) as ei:
            driver.run_stages(oracle, [P.Stage(1, P.shuffle_writer(plan, 1))], "refuse")
        assert "not computed by this consumer" in str(ei.value)


def _sqlite_union_all(con, table, keys, agg_sql, sets):
    parts = []
    for mask in sets:
        sel = [("NULL" if m else k) for k, m in zip(keys, mask)]
        present = [k for k, m in zip(keys, mask) if not m]
        gb = (" GROUP BY " + ", ".join(present)) if present else ""
        having = "" if present else " HAVING COUNT(*) > 0"  # the () set of an empty input has no row
        parts.append(f"SELECT {', '.join(sel)}, {P.grouping_id(mask)}, {agg_sql} FROM {table}{gb}{having}")
    return con.execute(" UNION ALL ".join(parts)).fetchall()


def _sqlite_table(con, name, table: pa.Table):
    cols = table.column_names
    con.execute(f"CREATE TABLE {name} ({', '.join(cols)})")
    rows = list(zip(*[table.column(c_).to_pylist() for c_ in cols]))
    if rows:
        con.executemany(f"INSERT INTO {name} VALUES ({', '.join('?' * len(cols))})", rows)


def _rows(tbl: pa.Table):
    return sorted((tuple(r.values()) for r in tbl.to_pylist()), key=repr)


@pytest.mark.parametrize("sets_name", ["rollup3", "cube3", "explicit"])
@pytest.mark.parametrize("empty", [False, True])
def test_union_all_form_against_sqlite_aggregate_test_100(oracle, sets_name, empty):
    t = G.load("aggregate_test_100")
    if empty:
        t = t.slice(0, 0)
    keys = ["c1", "c2", "c13"]
    sets = {"rollup3": P.rollup_sets(3), "cube3": P.cube_sets(3), "explicit": [[False, True, True], [True, False, True], [True, True, True]]}[sets_name]
    G.register(oracle, "aggregate_test_100", t, 1)
    aggs = [P.agg("sum", c("c4"), "s"), P.agg("count", None, "n"), P.agg("min", c("c13"), "mn"), P.agg("max", c("c3"), "mx")]
    got = GC.expected(oracle, P.scan("aggregate_test_100", G.ir_schema("aggregate_test_100")), [(c(k), k) for k in keys], aggs, sets, "sq")
    con = sqlite3.connect(":memory:")
    _sqlite_table(con, "t", t.select(["c1", "c2", "c3", "c4", "c13"]))
    want = _sqlite_union_all(con, "t", keys, "SUM(c4), COUNT(*), MIN(c13), MAX(c3)", sets)
    assert _rows(got) == sorted(want, key=repr)


def test_union_all_form_against_sqlite_tpch(oracle):
    from ballista_b200 import tpch  # noqa: F401
    cols = ["l_orderkey", "l_linenumber", "l_returnflag", "l_linestatus", "l_shipmode", "l_shipdate"]
    n = engine.GpuExecutionEngine.tpch_table_rows("lineitem", 5)
    oracle.drop_table("lineitem")
    oracle.tpch_generate("lineitem", 5, 0, 0, n, cols)
    t = pa.Table.from_batches([oracle.export_table("lineitem", 0)])
    sch = [P.field(f.name, {"int64": "i64", "int32": "i32", "string": "utf8", "date32[day]": "date32"}[str(f.type)], f.nullable)
           for f in t.schema]
    keys = ["l_returnflag", "l_linestatus", "l_shipmode"]
    aggs = [P.agg("count", None, "n"), P.agg("sum", c("l_linenumber"), "s"), P.agg("max", c("l_orderkey"), "mx")]
    sets = P.cube_sets(3)
    got = GC.expected(oracle, P.scan("lineitem", sch), [(c(k), k) for k in keys], aggs, sets, "sq-tpch")
    con = sqlite3.connect(":memory:")
    _sqlite_table(con, "li", t.select(keys + ["l_linenumber", "l_orderkey"]))
    want = _sqlite_union_all(con, "li", keys, "COUNT(*), SUM(l_linenumber), MAX(l_orderkey)", sets)
    assert _rows(got) == sorted(want, key=repr)


def _norm(v):
    """one representation for sqlite3 and arrow values: decimals and dates as text, bools as integers"""
    import datetime
    import decimal
    if isinstance(v, bool):
        return int(v)
    if isinstance(v, decimal.Decimal):
        return str(v)
    if isinstance(v, datetime.date):
        return v.isoformat()
    return v


def _norm_rows(rows):
    return sorted((tuple(_norm(v) for v in r) for r in rows), key=repr)


@pytest.mark.parametrize("keys, sets", [
    (["ks", "ki"], P.rollup_sets(2)),
    (["kd", "kt", "kf"], P.cube_sets(3)),
    (["kb", "ks", "kd"], [[False, False, False], [False, True, True], [True, False, True], [True, True, True]]),
    (["kt", "ki"], [[False, False]]),
], ids=["rollup_utf8_i32", "cube_dec_date_f64", "sets_bool_utf8_dec", "one_all_false_set"])
@pytest.mark.parametrize("rows", [0, 2000])
def test_union_all_form_against_sqlite_every_key_type_with_nulls(oracle, keys, sets, rows):
    """keys of every type the engine carries (Utf8, Int32, Decimal128, Date32, Float64, Bool), about 10 % NULL each: a real
    NULL key and a rolled-up one must stay apart (they differ in __grouping_id)"""
    t = GC.make_table(rows, seed=11)
    GC.register(oracle, "gs", t, 1)
    aggs = [P.agg("count", None, "n"), P.agg("count", c("n"), "cn"), P.agg("sum", c("n"), "sn"), P.agg("min", c("s"), "mn"),
            P.agg("max", c("s"), "mx")]
    got = GC.expected(oracle, P.scan("gs", GC.SCHEMA), [(c(k), k) for k in keys], aggs, sets, "sq-types")
    con = sqlite3.connect(":memory:")
    sq = pa.Table.from_arrays([pa.array([_norm(v) for v in t.column(k).to_pylist()]) if t.num_rows else pa.array([], pa.null())
                               for k in keys + ["n", "s"]], names=keys + ["n", "s"])
    _sqlite_table(con, "t", sq)
    want = _sqlite_union_all(con, "t", keys, "COUNT(*), COUNT(n), SUM(n), MIN(s), MAX(s)", sets)
    assert _norm_rows(tuple(r.values()) for r in got.to_pylist()) == _norm_rows(want)
    if rows:
        nulls_in_finest = [r for r in got.to_pylist() if r["__grouping_id"] == P.grouping_id(sets[0]) and r[keys[0]] is None]
        assert nulls_in_finest or sets[0][0], "the data has real NULL keys next to rolled-up ones"


def test_union_all_form_against_sqlite_tpch_orders(oracle):
    cols = ["o_orderkey", "o_custkey", "o_orderstatus", "o_totalprice", "o_orderdate", "o_orderpriority"]
    n = engine.GpuExecutionEngine.tpch_table_rows("orders", 5)
    oracle.drop_table("orders")
    oracle.tpch_generate("orders", 5, 0, 0, n, cols)
    t = pa.Table.from_batches([oracle.export_table("orders", 0)])
    ir = {"int64": "i64", "int32": "i32", "string": "utf8", "date32[day]": "date32"}
    sch = [P.field(f.name, ir.get(str(f.type)) or P.dec(f.type.precision, f.type.scale), f.nullable) for f in t.schema]
    keys = ["o_orderstatus", "o_orderpriority", "o_orderdate"]
    aggs = [P.agg("count", None, "n"), P.agg("sum", c("o_custkey"), "s"), P.agg("min", c("o_orderkey"), "mn")]
    sets = P.rollup_sets(3)
    got = GC.expected(oracle, P.scan("orders", sch), [(c(k), k) for k in keys], aggs, sets, "sq-orders")
    con = sqlite3.connect(":memory:")
    _sqlite_table(con, "o", pa.Table.from_arrays([pa.array([_norm(v) for v in t.column(k).to_pylist()])
                                                  for k in keys + ["o_custkey", "o_orderkey"]], names=keys + ["o_custkey", "o_orderkey"]))
    want = _sqlite_union_all(con, "o", keys, "COUNT(*), SUM(o_custkey), MIN(o_orderkey)", sets)
    assert _norm_rows(tuple(r.values()) for r in got.to_pylist()) == _norm_rows(want)
