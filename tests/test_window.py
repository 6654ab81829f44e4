"""Window functions without a GPU: the typing rules of DESIGN.md §6 (viii), every refusal with its code and the name of the
culprit, the CPU oracle's refusal, and the per-row restatement the GPU tests compare against (window_cases.py) pinned
against sqlite3's window functions."""
import json
import math
import sqlite3

import pyarrow as pa
import pytest

import golden_data as G
import window_cases as W
from ballista_b200 import driver, engine
from ballista_b200 import plan as P

c = P.col
PK, OB = [c("g")], [P.sort_key(c("o"))]


def _typed(node) -> dict:
    return json.loads(engine.plan_typed_json(json.dumps(node)))


def _node(exprs, mode="sorted"):
    return P.window([dict(w, partition_by=w.get("partition_by") or PK, order_by=w.get("order_by") or OB) for w in exprs],
                    P.scan("t", W.SCHEMA), PK, mode)


def test_result_types():
    exprs = [P.win("row_number", "rn"), P.win("rank", "rk"), P.win("dense_rank", "dr"), P.win("percent_rank", "pr"),
             P.win("cume_dist", "cd"), P.win("ntile", "nt", [P.lit_i64(4)]), P.win("lag", "lg", [c("dec")]),
             P.win("lead", "ld", [c("ks"), P.lit_i64(2), P.lit_utf8("x")]), P.win("first_value", "fv", [c("dt")]),
             P.win("last_value", "lv", [c("b")]), P.win("nth_value", "nv", [c("u64"), P.lit_i64(3)]),
             P.win("count", "cs", []), P.win("count", "c1", [P.lit_i64(1)]), P.win("count", "cx", [c("ks")]),
             P.win("sum", "si", [c("i32")]), P.win("sum", "su", [c("u64")]), P.win("sum", "sd", [c("dec")]),
             P.win("sum", "sf", [c("f64")]), P.win("avg", "ai", [c("i32")]), P.win("mean", "ad", [c("dec")]),
             P.win("min", "mi", [c("dt")]), P.win("max", "mb", [c("b")]), P.win("max", "md", [c("dec")])]
    t = _typed(_node(exprs))
    got = [(f["name"], f["type"], f["nullable"]) for f in t["schema"][len(W.SCHEMA):]]
    assert got == [("rn", "u64", False), ("rk", "u64", False), ("dr", "u64", False), ("pr", "f64", False), ("cd", "f64", False),
                   ("nt", "u64", True), ("lg", {"dec": [12, 2]}, True), ("ld", "utf8", True), ("fv", "date32", True),
                   ("lv", "bool", True), ("nv", "u64", True), ("cs", "i64", False), ("c1", "i64", False), ("cx", "i64", False),
                   ("si", "i64", True), ("su", "u64", True), ("sd", {"dec": [22, 2]}, True), ("sf", "f64", True),
                   ("ai", "f64", True), ("ad", {"dec": [16, 6]}, True), ("mi", "date32", True), ("mb", "bool", True),
                   ("md", {"dec": [12, 2]}, True)]
    assert [f["name"] for f in t["schema"][:len(W.SCHEMA)]] == [f["name"] for f in W.SCHEMA]
    assert t["window_expr"][12]["args"] == []  # COUNT(1) is COUNT(*)
    assert t["window_expr"][0]["frame"] == {"units": "range", "start": {"kind": "unbounded_preceding"}, "end": {"kind": "current_row"}}
    assert t["mode"] == "sorted" and _typed(_node(exprs[:1], mode=None))["mode"] is None


@pytest.mark.parametrize("bad, code, match", [
    (P.win("sum", "x", [c("i64")], frame=P.range_(P.preceding(7), P.CURRENT_ROW)), -2, "RANGE window frame with an offset bound (start of sum (x))"),
    (P.win("sum", "x", [c("i64")], frame={"units": "groups", "start": P.UNBOUNDED_PRECEDING, "end": P.CURRENT_ROW}), -2, "GROUPS window frame of sum (x)"),
    (dict(P.win("first_value", "x", [c("i64")]), ignore_nulls=True), -2, "IGNORE NULLS in window function first_value (x)"),
    (dict(P.win("count", "x", [c("i64")]), distinct=True), -2, "DISTINCT window function count (x)"),
    (P.win("stddev", "x", [c("f64")]), -2, "window function stddev (x) is not supported"),
    (P.win("string_agg", "x", [c("ks")]), -2, "window function string_agg (x) is not supported"),
    (P.win("array_agg", "x", [c("ks")]), -2, "window function array_agg (x) is not supported"),
    (P.win("min", "x", [c("ks")]), -2, "min (x) does not support an argument of type utf8"),
    (P.win("sum", "x", [c("dt")]), -2, "sum (x) does not support an argument of type date32"),
    (P.win("ntile", "x", [c("i64")]), -2, "the bucket count of ntile (x) must be an integer literal"),
    (P.win("nth_value", "x", [c("i64"), c("i64")]), -2, "the position of nth_value (x) must be an integer literal"),
    (P.win("lag", "x", [c("i64"), c("i32")]), -2, "the offset of lag (x) must be an integer literal"),
    (P.win("lag", "x", [c("i64"), P.lit_i64(1), P.lit_utf8("a")]), -2, "the default of lag (x) has type utf8"),
    (P.win("rank", "x", partition_by=[c("h")]), -2, "rank (x): its PARTITION BY differs from the node's partition keys"),
    (P.win("sum", "x", [c("i64")], frame=P.rows(P.UNBOUNDED_FOLLOWING, P.CURRENT_ROW)), -1, "sum (x) starts at UNBOUNDED FOLLOWING"),
    (P.win("sum", "x", [c("i64")], frame=P.rows(P.CURRENT_ROW, P.UNBOUNDED_PRECEDING)), -1, "sum (x) ends at UNBOUNDED PRECEDING"),
    (P.win("ntile", "x", [P.lit_i64(0)]), -1, "ntile of ntile (x) needs n >= 1"),
    (P.win("nth_value", "x", [c("i64"), P.lit_i64(0)]), -1, "nth_value of nth_value (x) needs n >= 1"),
], ids=lambda v: v if isinstance(v, str) else None)
def test_refusals(bad, code, match):
    with pytest.raises(engine.B200Error) as ei:
        _typed(_node([P.win("row_number", "rn"), bad]))
    assert ei.value.code == code and match in str(ei.value), str(ei.value)


def test_order_by_must_agree_and_modes():
    other = P.win("rank", "r2", order_by=[P.sort_key(c("o"), False)])
    with pytest.raises(engine.B200Error) as ei:
        _typed(_node([P.win("rank", "r1"), other]))
    assert ei.value.code == -2 and "rank (r2): its ORDER BY differs" in str(ei.value)
    for mode in ("linear", "partially_sorted"):
        with pytest.raises(engine.B200Error) as ei:
            _typed(_node([P.win("rank", "r")], mode=mode))
        assert ei.value.code == -2 and f"window input order mode {mode}" in str(ei.value)


def test_oracle_refuses_window_plans(oracle):
    t = W.make_table(10, seed=1)
    W.register(oracle, "t", t)
    with pytest.raises(Exception) as ei:
        driver.run_stages(oracle, W.stages(_node([P.win("row_number", "rn")])), "refuse")
    assert "window functions are not computed by this consumer" in str(ei.value)


# ---- the restatement against sqlite3 ---------------------------------------------------------------------------------
def _sql_frame(f):
    if f is None:
        return ""
    def b(x):
        return {"unbounded_preceding": "UNBOUNDED PRECEDING", "current_row": "CURRENT ROW", "unbounded_following": "UNBOUNDED FOLLOWING",
                "preceding": f"{x.get('n')} PRECEDING", "following": f"{x.get('n')} FOLLOWING"}[x["kind"]]
    return f" {f['units'].upper()} BETWEEN {b(f['start'])} AND {b(f['end'])}"


def _sql(w, over):
    args = []
    for a in w.get("args", []):
        if "col" in a:
            args.append(a["col"])
        else:
            v = a["lit"]["v"]
            args.append("NULL" if v is None else repr(v) if isinstance(v, str) else str(v))
    fn = w["fn"]
    arg_s = "*" if fn == "count" and not args else ", ".join(args)
    return f"{fn}({arg_s}) OVER ({over}{_sql_frame(w.get('frame'))}) AS {w['name']}"


def _sqlite_rows(table: pa.Table, exprs, partition, order):
    con = sqlite3.connect(":memory:")
    names = ["rid", "g", "h", "o", "ks", "i32", "i64", "f64"]
    con.execute(f"CREATE TABLE t ({', '.join(names)})")
    con.executemany(f"INSERT INTO t VALUES ({', '.join('?' * len(names))})", list(zip(*[table.column(n).to_pylist() for n in names])))
    over = (f"PARTITION BY {', '.join(partition)} " if partition else "") + "ORDER BY " + ", ".join(
        f"{n} {'ASC' if a else 'DESC'} NULLS {'FIRST' if nf else 'LAST'}" for n, a, nf in order)
    q = f"SELECT rid, {', '.join(_sql(w, over) for w in exprs)} FROM t ORDER BY rid"
    return con.execute(q).fetchall()


FRAMES = [None, P.range_(P.UNBOUNDED_PRECEDING, P.UNBOUNDED_FOLLOWING), P.range_(P.CURRENT_ROW, P.UNBOUNDED_FOLLOWING),
          P.range_(P.CURRENT_ROW, P.CURRENT_ROW), P.rows(P.preceding(2), P.CURRENT_ROW), P.rows(P.preceding(3), P.preceding(1)),
          P.rows(P.following(1), P.following(3)), P.rows(P.following(2), P.following(1)), P.rows(P.CURRENT_ROW, P.UNBOUNDED_FOLLOWING)]


def _pin(table, partition, order, frames=FRAMES):
    peer_safe = [P.win("rank", "rk"), P.win("dense_rank", "dr"), P.win("percent_rank", "pr"), P.win("cume_dist", "cd")]
    # with a unique ORDER BY every function is determined; sqlite need not keep the input order among peers
    exact_order = order + [("rid", True, False)]
    full = [P.win("row_number", "rn"), P.win("ntile", "nt", [P.lit_i64(4)]), P.win("lag", "lg", [c("i32"), P.lit_i64(2), P.lit_i64(-1)]),
            P.win("lead", "ld", [c("ks"), P.lit_i64(1)])]
    for k, f in enumerate(frames):
        full += [P.win("count", f"cs{k}", [], frame=f), P.win("count", f"cx{k}", [c("ks")], frame=f), P.win("sum", f"si{k}", [c("i64")], frame=f),
                 P.win("min", f"mn{k}", [c("f64")], frame=f), P.win("max", f"mx{k}", [c("ks")], frame=f),
                 P.win("first_value", f"fv{k}", [c("h")], frame=f), P.win("last_value", f"lv{k}", [c("i32")], frame=f),
                 P.win("nth_value", f"nv{k}", [c("i64"), P.lit_i64(2)], frame=f), P.win("avg", f"av{k}", [c("i32")], frame=f)]
    for exprs, ordr in ((peer_safe, order), (full, exact_order)):
        want = W.evaluate(table, exprs, partition, ordr)
        rows = _sqlite_rows(table, exprs, partition, ordr)
        for j, w in enumerate(exprs):
            got = [r[j + 1] for r in rows]
            for i, (a, b) in enumerate(zip(got, want[w["name"]])):
                if isinstance(b, float) and a is not None:
                    assert math.isclose(a, b, rel_tol=1e-12, abs_tol=1e-9), (w["name"], i, a, b)
                else:
                    assert a == b, (w["name"], i, a, b)


@pytest.mark.parametrize("partition, order", [(["g"], [("o", True, False)]), (["h"], [("f64", False, True)]), ([], [("ks", True, True)])],
                         ids=["int_keys", "utf8_partition_f64_desc", "one_partition"])
def test_restatement_against_sqlite_generated(partition, order):
    _pin(W.make_table(400, seed=21), partition, order)


def test_restatement_against_sqlite_aggregate_test_100():
    t = G.load("aggregate_test_100")
    m = {"rid": pa.array(range(t.num_rows), pa.int64()), "g": t.column("c2").cast(pa.int32()), "h": t.column("c1"), "o": t.column("c3").cast(pa.int64()),
         "ks": t.column("c13"), "i32": t.column("c4").cast(pa.int32()), "i64": t.column("c9").cast(pa.int64()), "f64": t.column("c12")}
    _pin(pa.table(m), ["g"], [("o", True, False)])


def test_restatement_against_sqlite_tpch():
    cols = ["l_orderkey", "l_linenumber", "l_returnflag", "l_shipmode", "l_quantity", "l_shipdate"]
    n = engine.GpuExecutionEngine.tpch_table_rows("lineitem", 1)
    from oracle_ffi import OracleEngine
    o = OracleEngine()
    try:
        o.tpch_generate("lineitem", 1, 0, 0, n, cols)
        li = pa.Table.from_batches([o.export_table("lineitem", 0)])
    finally:
        o.close()
    m = {"rid": pa.array(range(li.num_rows), pa.int64()), "g": li.column("l_linenumber").cast(pa.int32()), "h": li.column("l_returnflag"),
         "o": li.column("l_orderkey").cast(pa.int64()), "ks": li.column("l_shipmode"), "i32": li.column("l_linenumber").cast(pa.int32()),
         "i64": li.column("l_orderkey").cast(pa.int64()), "f64": li.column("l_quantity").cast(pa.float64())}
    _pin(pa.table(m), ["h"], [("o", False, False)], FRAMES[3:8])  # bounded frames: the restatement reads frames row by row
