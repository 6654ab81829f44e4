"""first_value / last_value on the host: the restatement (first_last_cases.py) against sqlite3's FIRST_VALUE / LAST_VALUE
windows and pyarrow's hash_first / hash_last; the result types and partial state schemas of the typed plan in every mode;
every refusal, with its code and the culprit named; the CPU oracle's refusal; the protobuf plans decoding to the typed
plan of the IR they were encoded from, and ordering_req on SUM still refused."""
import base64
import json
import random
import sqlite3

import pyarrow as pa
import pyarrow.compute  # noqa: F401  (registers hash_first / hash_last)
import pytest

import golden_data as G
from ballista_b200 import engine
from ballista_b200 import plan as P
from first_last_cases import final_merge, first_last, grouped, partial_state, stages

c = P.col
UNSUPPORTED = -2  # B200_ERR_UNSUPPORTED (include/b200exec.h)
SCHEMA = [P.field("k", "i32", True), P.field("x", "i64", True), P.field("o", "f64", True), P.field("s", "utf8", True),
          P.field("d", P.dec(38, 2), True), P.field("b", "bool", True), P.field("dt", "date32", True), P.field("ts", "ts", True),
          P.field("f", "f32", True), P.field("u", "u64", True)]


def typed(st, i=0):
    return json.loads(engine.plan_typed_json(st[i].json("j")))["input"]


def refusal(st, i=0):
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(st[i].json("j"))
    return ei.value


def rand_rows(rng, n):
    return [(rng.randint(0, 3), None if rng.random() < 0.2 else rng.randint(-5, 5), None if rng.random() < 0.2 else float(rng.randint(-3, 3)),
             None if rng.random() < 0.2 else rng.choice(["", "a", "ab", "b", "abc"])) for _ in range(n)]


# ---- the restatement against independent engines ----------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_restatement_matches_sqlite_windows(seed):
    """sqlite3 FIRST_VALUE / LAST_VALUE over the whole partition, ordered by the keys and then the input position (the
    engine's tie rule), on data without NaN or -0.0"""
    rng = random.Random(seed)
    rows = rand_rows(rng, rng.randint(1, 300))
    db = sqlite3.connect(":memory:")
    db.execute("create table t (pos integer, k integer, x integer, o real, s text)")
    db.executemany("insert into t values (?, ?, ?, ?, ?)", [(i,) + r for i, r in enumerate(rows)])
    for fn in ("first_value", "last_value"):
        for asc in (True, False):
            for nf in (True, False):
                ob = f"o {'asc' if asc else 'desc'} nulls {'first' if nf else 'last'}, s {'desc' if asc else 'asc'} nulls last, pos"
                q = (f"select k, {fn}(x) over (partition by k order by {ob} rows between unbounded preceding and unbounded following) "
                     "from t order by pos")
                want = dict(db.execute(q).fetchall())
                got = grouped(rows, [0], [(fn, 1, [(2, asc, nf), (3, not asc, False)], False, "v")])
                assert {k[0]: v["v"] for k, v in got.items()} == want, (fn, asc, nf)


@pytest.mark.parametrize("seed", range(4))
def test_restatement_matches_pyarrow_hash_first_last(seed):
    """no ORDER BY: the first / last candidate in input order (pyarrow skips NULLs by default: IGNORE NULLS)"""
    rng = random.Random(seed)
    rows = rand_rows(rng, rng.randint(1, 300))
    t = pa.table({"k": [r[0] for r in rows], "x": [r[1] for r in rows]})
    for fn, pfn in (("first_value", "first"), ("last_value", "last")):
        for skip in (True, False):
            res = t.group_by("k", use_threads=False).aggregate([("x", pfn, pa.compute.ScalarAggregateOptions(skip_nulls=skip))]).to_pydict()
            want = dict(zip(res["k"], res[f"x_{pfn}"]))
            got = grouped(rows, [0], [(fn, 1, [], skip, "v")])
            assert {k[0]: v["v"] for k, v in got.items()} == want


def test_restated_rules():
    nan, inf = float("nan"), float("inf")
    rows = [(0, 1, -0.0), (0, 2, 0.0), (0, 3, nan), (0, 4, -inf), (0, 5, inf)]
    assert first_last("first_value", rows, lambda r: r[1], [lambda r: r[2]], [(True, False)]) == 4
    assert first_last("last_value", rows, lambda r: r[1], [lambda r: r[2]], [(True, False)]) == 3   # NaN greatest
    assert first_last("first_value", rows[:2], lambda r: r[1], [lambda r: r[2]], [(False, False)]) == 2  # -0.0 before +0.0
    tied = [(0, 1, 5), (0, 2, 5), (0, 3, 5)]
    assert first_last("first_value", tied, lambda r: r[1], [lambda r: r[2]], [(True, False)]) == 1
    assert first_last("last_value", tied, lambda r: r[1], [lambda r: r[2]], [(False, True)]) == 3
    assert first_last("first_value", [(0, None, 1), (0, 7, 2)], lambda r: r[1], [lambda r: r[2]], [(True, False)], ignore_nulls=True) == 7
    assert first_last("first_value", [(0, None, 1)], lambda r: r[1], [], [], ignore_nulls=True) is None
    assert first_last("first_value", [(0, 1, "ab"), (0, 2, "a")], lambda r: r[1], [lambda r: r[2]], [(True, False)]) == 2  # prefix first
    # the Final merge over states in reading order equals the rule over all rows in that order
    rng = random.Random(5)
    parts = [rand_rows(rng, 40) for _ in range(3)]
    for fn in ("first_value", "last_value"):
        states = [partial_state(fn, p, lambda r: r[1], [lambda r: r[2]], [(True, True)]) for p in parts]
        assert final_merge(fn, states, [(True, True)]) == first_last(fn, [r for p in parts for r in p], lambda r: r[1], [lambda r: r[2]], [(True, True)])


# ---- typing ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("x", ["x", "o", "s", "d", "b", "dt", "ts", "f", "u"])
def test_result_and_state_types(x):
    types = {f["name"]: f["type"] for f in SCHEMA}
    aggs = [("first_value", c(x), types[x], [(c("o"), True, False), (c("s"), False, True)], False, "a"),
            ("last_value", c(x), types[x], [], True, "b")]
    single = typed(stages(P.scan("t", SCHEMA), aggs, [(c("k"), "k")], [], "Single"))
    assert [(f["name"], f["type"], f["nullable"]) for f in single["schema"]] == [("k", "i32", True), ("a", types[x], True), ("b", types[x], True)]
    a0 = single["aggr"][0]
    assert a0["fn"] == "first_value" and a0["ignore_nulls"] is False and [(k["asc"], k["nulls_first"]) for k in a0["order_by"]] == [(True, False), (False, True)]
    assert single["aggr"][1]["ignore_nulls"] is True and single["aggr"][1]["order_by"] == []
    st = stages(P.scan("t", SCHEMA), aggs, [(c("k"), "k")], [P.field("k", "i32", True)], "Partial")
    part = typed(st)
    assert [(f["name"], f["type"]) for f in part["schema"]] == [("k", "i32"), ("a[first_value]", types[x]), ("o@2", "f64"), ("s@3", "utf8"),
                                                                 ("is_set", "bool"), ("b[last_value]", types[x]), ("is_set", "bool")]
    fin = typed(st, 1)
    assert [(f["name"], f["type"], f["nullable"]) for f in fin["schema"]] == [("k", "i32", True), ("a", types[x], True), ("b", types[x], True)]
    assert [(k["asc"], k["nulls_first"]) for k in fin["aggr"][0]["order_by"]] == [(True, False), (False, True)]
    for mode in ("SinglePartitioned",):
        assert typed(stages(P.scan("t", SCHEMA), aggs, [(c("k"), "k")], [], mode))["mode"] == mode
    scalar = stages(P.scan("t", SCHEMA), aggs, [], [], "Partial")
    assert typed(scalar, 1)["mode"] == "Final"


# ---- refusals -------------------------------------------------------------------------------------------------------------
def test_refusals():
    src = P.scan("t", SCHEMA)
    five = [(c("o"), True, False)] * 5
    e = refusal(stages(src, [("first_value", c("x"), "i64", five, False, "five")], [(c("k"), "k")]))
    assert e.code == UNSUPPORTED and "five" in str(e) and "ordering keys" in str(e)
    plan = P.aggregate("Single", [(c("k"), "k"), (c("s"), "s")], [P.agg("last_value", c("x"), "gs", order_by=[P.sort_key(c("o"))])], src,
                       grouping_sets=[[False, False], [False, True]])
    e = refusal([P.Stage(1, P.shuffle_writer(plan, 1))])
    assert e.code == UNSUPPORTED and "gs" in str(e) and "grouping sets" in str(e)
    # a Final whose state columns do not have the layout: the culprit column is named
    st = stages(src, [("first_value", c("x"), "i64", [(c("o"), True, False)], False, "a")], [(c("k"), "k")], [P.field("k", "i32", True)], "Partial")
    bad = json.loads(st[1].json("j"))
    reader = bad["input"]["input"]
    for name, idx in (("a[first]", 1), ("a[is_set]x", 3)):
        sch = [dict(f) for f in reader["schema"]]
        sch[idx]["name"] = name
        reader["schema"] = sch
        with pytest.raises(engine.B200Error) as ei:
            engine.plan_typed_json(json.dumps(bad))
        assert ei.value.code == UNSUPPORTED and name in str(ei.value)
        reader["schema"] = json.loads(st[1].json("j"))["input"]["input"]["schema"]
    sch = [dict(f) for f in reader["schema"]]
    sch[3]["type"] = "i32"  # is_set of the wrong type
    reader["schema"] = sch
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(json.dumps(bad))
    assert ei.value.code == UNSUPPORTED and "is_set" in str(ei.value)
    # one ordering column fewer than the node's order_by: is_set is not where it should be
    st2 = stages(src, [("first_value", c("x"), "i64", [(c("o"), True, False), (c("s"), True, False)], False, "a")], [(c("k"), "k")],
                 [P.field("k", "i32", True)], "Partial")
    bad = json.loads(st2[1].json("j"))
    bad["input"]["input"]["schema"] = json.loads(st[1].json("j"))["input"]["input"]["schema"]
    with pytest.raises(engine.B200Error):
        engine.plan_typed_json(json.dumps(bad))


def test_cpu_oracle_refuses(oracle):
    from ballista_b200 import driver
    from oracle_ffi import OracleError
    b = pa.record_batch([pa.array([1, 1, 2], pa.int32()), pa.array([3, 5, 7], pa.int64()), pa.array([1.0, 2.0, 0.5])], names=["k", "x", "o"])
    oracle.register_batch("t", 0, b)
    sch = [P.field("k", "i32", False), P.field("x", "i64", True), P.field("o", "f64", True)]
    for fn in ("first_value", "last_value"):
        for ob in ([], [(c("o"), True, False)]):
            with pytest.raises(OracleError, match=f"'{fn}' is not computed"):
                driver.run_stages(oracle, stages(P.scan("t", sch), [(fn, c("x"), "i64", ob, False, "r")], [(c("k"), "k")]), f"orf-{fn}-{len(ob)}")


# ---- the protobuf path ------------------------------------------------------------------------------------------------
with open(G.__file__.replace("golden_data.py", "golden/first_last_proto_plans.json")) as _fh:
    PROTO_CASES = json.load(_fh)["cases"]


def _agg_nodes(node):
    if isinstance(node, dict):
        if node.get("op") == "AggregateExec":
            yield node
        for v in node.values():
            yield from _agg_nodes(v)


@pytest.mark.parametrize("case", [x for x in PROTO_CASES if "ir" in x], ids=[x["name"] for x in PROTO_CASES if "ir" in x])
def test_protobuf_plans_decode_to_the_same_typed_plan(case):
    decoded = json.loads(engine.plan_typed_json(engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]), "job")))
    want = json.loads(engine.plan_typed_json(case["ir"]))
    got_aggs, want_aggs = list(_agg_nodes(decoded)), list(_agg_nodes(want))
    assert len(got_aggs) == len(want_aggs) == 1
    g, w = got_aggs[0], want_aggs[0]
    assert g["mode"] == w["mode"]
    assert g["aggr"] == w["aggr"] or [(a["fn"], a["result_type"], a["order_by"], a["ignore_nulls"]) for a in g["aggr"]] == \
        [(a["fn"], a["result_type"], a["order_by"], a["ignore_nulls"]) for a in w["aggr"]]
    assert [(f["name"], f["type"], f["nullable"]) for f in g["schema"]] == [(f["name"], f["type"], f["nullable"]) for f in w["schema"]]


@pytest.mark.parametrize("case", [x for x in PROTO_CASES if "refusal" in x], ids=[x["name"] for x in PROTO_CASES if "refusal" in x])
def test_protobuf_refusals(case):
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]), "job"))
    assert ei.value.code == UNSUPPORTED and case["refusal"] in str(ei.value)
