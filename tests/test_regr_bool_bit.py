"""regr_* / bool_and / bool_or / bit_and / bit_or / bit_xor on the host: the restated regression formulas against scipy,
the result types and partial state schemas of the typed plan, every refusal (with its code and the function's name), the
CPU oracle's refusal, and the protobuf plans decoding to the IR they were encoded from."""
import base64
import json
import math
import random

import pytest

import golden_data as G
from ballista_b200 import engine
from ballista_b200 import plan as P
from regr_bool_bit_cases import BIT, BOOL, REGR, REGR_STATE, fold, regr_exact, result_type, stages, state_fields

c = P.col
UNSUPPORTED = -2  # B200_ERR_UNSUPPORTED (include/b200exec.h)
SCHEMA = [P.field("k", "i32", True), P.field("x", "i32", True), P.field("y", "f64", True), P.field("d", P.dec(15, 2), True),
          P.field("s", "utf8", True), P.field("b", "bool", True), P.field("i8", "i8", True), P.field("u64", "u64", True),
          P.field("dt", "date32", True)]


def typed(st, i=0):
    return json.loads(engine.plan_typed_json(st[i].json("j")))["input"]


def refusal(st, i=0):
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(st[i].json("j"))
    return ei.value


def one(fn):
    """one aggregate of each kind over SCHEMA: regr_*(y, x), bool over b, bit over i8"""
    if fn in REGR:
        return (fn, c("y"), c("x"), "r", None)
    if fn in BOOL:
        return (fn, c("b"), None, "r", "bool")
    return (fn, c("i8"), None, "r", "i8")


# ---- the restatement against an independent implementation -----------------------------------------------------------
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_restated_regression_matches_scipy(seed):
    from scipy import stats
    rng = random.Random(seed)
    n = rng.randint(3, 400)
    xs = [rng.gauss(10, 4) for _ in range(n)]
    ys = [2.5 * x - 7 + rng.gauss(0, 3) for x in xs]
    lr = stats.linregress(xs, ys)
    assert math.isclose(regr_exact("regr_slope", ys, xs), lr.slope, rel_tol=1e-9)
    assert math.isclose(regr_exact("regr_intercept", ys, xs), lr.intercept, rel_tol=1e-9)
    assert math.isclose(regr_exact("regr_r2", ys, xs), lr.rvalue ** 2, rel_tol=1e-9)


def test_restated_rules():
    assert regr_exact("regr_count", [None, 1.0], [2.0, None]) == 0 and regr_exact("regr_avgx", [None], [1.0]) is None
    assert regr_exact("regr_slope", [1.0], [2.0]) is None and regr_exact("regr_sxx", [1.0], [2.0]) == 0.0
    assert regr_exact("regr_slope", [1.0, 2.0, 3.0], [0.1, 0.1, 0.1]) is None  # sxx = 0
    assert regr_exact("regr_r2", [5.0, 5.0], [1.0, 2.0]) is None                # syy = 0: [EXT] unpinned
    assert regr_exact("regr_slope", [5.0, 5.0], [1.0, 2.0]) == 0.0
    assert regr_exact("regr_avgy", [1.0, 2.0, None], [1.0, None, 3.0]) == 1.0   # only complete pairs count
    assert fold("bool_and", [True, None, False]) is False and fold("bool_or", [None, None]) is None
    assert fold("bit_and", [-128, -1], "i8") == -128 and fold("bit_xor", [1, 3, None], "i32") == 2
    assert fold("bit_or", [1 << 63, 1], "u64") == (1 << 63) + 1 and fold("bit_and", [], "u8") is None


# ---- typing -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", REGR + BOOL + BIT)
def test_result_types_and_state_schema(fn):
    a = one(fn)
    src = P.scan("t", SCHEMA)
    single = typed(stages(src, [a]))
    assert single["aggr"][0]["fn"] == fn
    want = result_type(fn, a[4])
    f = single["schema"][-1]
    assert (f["name"], f["type"], f["nullable"]) == ("r", want, fn != "regr_count")
    assert len(single["aggr"][0]["args"]) == (2 if fn in REGR else 1)
    st = stages(src, [a], keys=[(c("k"), "k")], key_fields=[P.field("k", "i32", True)], mode="Partial")
    states = typed(st, 0)["schema"][1:]
    assert [(s["name"], s["type"]) for s in states] == [(s["name"], s["type"]) for s in state_fields(fn, "r", a[4])]
    final = typed(st, 1)
    assert final["aggr"][0]["fn"] == fn and final["schema"][-1]["type"] == want


@pytest.mark.parametrize("t", ["i8", "i16", "i32", "i64", "u8", "u16", "u32", "u64"])
def test_bit_result_has_the_argument_type(t):
    sch = [P.field("v", t, True)]
    for fn in BIT:
        assert typed(stages(P.scan("t", sch), [(fn, c("v"), None, "r", t)]))["schema"][-1]["type"] == t


@pytest.mark.parametrize("t", ["i8", "u64", "f32", P.dec(15, 2)])
def test_regr_arguments_are_coerced_to_f64(t):
    sch = [P.field("a", t, True), P.field("b", "i64", False)]
    for fn in REGR:
        assert typed(stages(P.scan("t", sch), [(fn, c("a"), c("b"), "r", None)]))["schema"][-1]["type"] == result_type(fn, None)


# ---- refusals -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn,col", [(f, a) for f in REGR for a in ("s", "b", "dt")] + [(f, a) for f in BOOL for a in ("x", "s", "y")] +
                         [(f, a) for f in BIT for a in ("b", "y", "d", "s", "dt")])
def test_argument_types_are_refused(fn, col):
    args = (c("y"), c(col)) if fn in REGR else (c(col), None)
    e = refusal(stages(P.scan("t", SCHEMA), [(fn, args[0], args[1], "r", None)]))
    t = next(f["type"] for f in SCHEMA if f["name"] == col)
    assert e.code == UNSUPPORTED and fn in str(e) and (t if isinstance(t, str) else "dec(") in str(e), str(e)


def test_wrong_argument_counts_are_refused():
    for fn, a, b in (("regr_slope", c("y"), None), ("bool_and", c("b"), c("b")), ("bit_or", c("i8"), c("i8"))):
        with pytest.raises(engine.B200Error, match=fn):
            engine.plan_typed_json(stages(P.scan("t", SCHEMA), [(fn, a, b, "r", None)])[0].json("j"))


@pytest.mark.parametrize("fn", REGR + BOOL + BIT)
def test_distinct_is_refused(fn):
    st = stages(P.scan("t", SCHEMA), [one(fn)])
    st[0].plan["input"]["aggr"][0]["distinct"] = True
    with pytest.raises(engine.B200Error, match="DISTINCT"):
        engine.plan_typed_json(st[0].json("j"))


@pytest.mark.parametrize("fn", REGR + BOOL + BIT)
def test_window_forms_are_refused(fn):
    a = one(fn)
    args = [a[1]] + ([a[2]] if a[2] is not None else [])
    node = P.window([P.win(fn, "w", args, partition_by=[c("k")], order_by=[P.sort_key(c("x"))])], P.scan("t", SCHEMA))
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(P.Stage(1, P.shuffle_writer(node, 1)).json("j"))
    assert ei.value.code == UNSUPPORTED and fn in str(ei.value)


def test_regr_alongside_grouping_sets_is_refused_and_bool_bit_are_accepted():
    keys = [(c("k"), "k"), (c("s"), "s")]
    e = refusal(stages(P.scan("t", SCHEMA), [one("regr_sxy")], keys, grouping_sets=P.rollup_sets(2)))
    assert e.code == UNSUPPORTED and "regr_sxy" in str(e)
    for fn in BOOL + BIT:
        out = typed(stages(P.scan("t", SCHEMA), [one(fn)], keys, grouping_sets=P.cube_sets(2)))
        assert out["schema"][-1]["type"] == one(fn)[4]


@pytest.mark.parametrize("fn,bad", [("regr_slope", ["count", "mean_y", "mean_x", "m2_x", "m2_y", "algo_const"]),
                                    ("regr_r2", ["count", "mean1", "m2_1", "mean2", "m2_2", "algo_const"]),
                                    ("regr_count", ["count", "mean_x", "mean_y", "m2_x", "m2_y", "co"])])
def test_final_with_other_regr_state_layout_is_refused(fn, bad):
    part = [P.field(f"r[{s}]", "u64" if s == "count" else "f64", True) for s in bad]
    plan = P.shuffle_writer(P.aggregate("Final", [], [P.agg(fn, None, "r")], P.shuffle_reader(1, part)), 2)
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(P.Stage(2, plan).json("j"))
    first_bad = next(i for i, s in enumerate(bad) if s != REGR_STATE[i])
    assert ei.value.code == UNSUPPORTED and f"r[{bad[first_bad]}]" in str(ei.value), str(ei.value)


@pytest.mark.parametrize("fn,t", [("bool_and", "i32"), ("bit_xor", "f64"), ("bit_or", "bool")])
def test_final_with_a_wrong_bool_bit_state_type_is_refused(fn, t):
    plan = P.shuffle_writer(P.aggregate("Final", [], [P.agg(fn, None, "r")], P.shuffle_reader(1, [P.field(f"r[{fn}]", t, True)])), 2)
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(P.Stage(2, plan).json("j"))
    assert ei.value.code == UNSUPPORTED and fn in str(ei.value)


def test_cpu_oracle_refuses(oracle):
    """The CPU oracle does not compute these functions: a plan holding one is refused, never evaluated."""
    import pyarrow as pa
    from ballista_b200 import driver
    from oracle_ffi import OracleError
    b = pa.record_batch([pa.array([1, 1, 2], pa.int32()), pa.array([1.0, 2.0, 5.0]), pa.array([True, False, None]),
                         pa.array([3, 5, 7], pa.int64())], names=["k", "y", "b", "v"])
    oracle.register_batch("t", 0, b)
    sch = [P.field("k", "i32", False), P.field("y", "f64", True), P.field("b", "bool", True), P.field("v", "i64", True)]
    for fn in REGR + BOOL + BIT:
        a = (fn, c("y"), c("v"), "r", None) if fn in REGR else (fn, c("b"), None, "r", "bool") if fn in BOOL else (fn, c("v"), None, "r", "i64")
        with pytest.raises(OracleError, match="not computed"):
            driver.run_stages(oracle, stages(P.scan("t", sch), [a], [(c("k"), "k")]), f"orf-{fn}")


# ---- the protobuf path ------------------------------------------------------------------------------------------------
with open(G.__file__.replace("golden_data.py", "golden/regr_bool_bit_proto_plans.json")) as _fh:
    PROTO_CASES = json.load(_fh)["cases"]


def _agg_nodes(node):
    if isinstance(node, dict):
        if node.get("op") == "AggregateExec":
            yield node
        for v in node.values():
            yield from _agg_nodes(v)


@pytest.mark.parametrize("case", PROTO_CASES, ids=[c_["name"] for c_ in PROTO_CASES])
def test_protobuf_plans_decode_to_the_same_typed_plan(case):
    decoded = json.loads(engine.plan_typed_json(engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]), "job")))
    want = json.loads(engine.plan_typed_json(case["ir"]))
    got_aggs, want_aggs = list(_agg_nodes(decoded)), list(_agg_nodes(want))
    assert len(got_aggs) == len(want_aggs) == 1
    g, w = got_aggs[0], want_aggs[0]
    assert g["mode"] == w["mode"]
    assert [(a["fn"], a["result_type"], len(a["args"])) for a in g["aggr"]] == [(a["fn"], a["result_type"], len(a["args"])) for a in w["aggr"]]
    assert [(f["name"], f["type"], f["nullable"]) for f in g["schema"]] == [(f["name"], f["type"], f["nullable"]) for f in w["schema"]]
    assert g["aggr"][0]["fn"] == case["fn"].lower()
