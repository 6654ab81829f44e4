"""VAR / STDDEV / COVAR / CORR on the host: every name and alias the function registry resolves, argument typing, the
Float64 results, the partial state schemas and the refusals (an argument type without a Float64 coercion, DISTINCT, and
a Final whose state columns are laid out differently).  Also pins the exact reference these tests compare against."""
import json
import math

import pytest

import golden_data as G
from ballista_b200 import engine
from ballista_b200 import plan as P
from stat_cases import BIVARIATE, STATE, exact, part_fields, stat_stages, welford

c = P.col
UNSUPPORTED = -2  # B200_ERR_UNSUPPORTED (include/b200exec.h)
SCHEMA = [P.field("x", "i32", True), P.field("y", "f64", True), P.field("d", P.dec(15, 2), True), P.field("s", "utf8", True)]
CANON = {"var": "var_samp", "var_samp": "var_samp", "var_sample": "var_samp", "var_pop": "var_pop", "var_population": "var_pop",
         "stddev": "stddev_samp", "stddev_samp": "stddev_samp", "stddev_pop": "stddev_pop", "covar": "covar_samp",
         "covar_samp": "covar_samp", "covar_pop": "covar_pop", "corr": "corr"}


def typed(stages, i=0):
    return json.loads(engine.plan_typed_json(stages[i].json("j")))["input"]


def refusal(stages, i=0):
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(stages[i].json("j"))
    return ei.value


def args_of(fn):
    return (c("x"), c("y")) if fn in BIVARIATE else (c("x"), None)


@pytest.mark.parametrize("fn", sorted(CANON))
def test_names_types_and_state_schema(fn):
    x, y = args_of(fn)
    src = P.scan("t", SCHEMA)
    single = typed(stat_stages(src, [(fn, x, y, "r")]))
    a = single["aggr"][0]
    assert a["fn"] == CANON[fn]
    assert a["result_type"] == "f64"
    assert single["schema"][-1]["name"] == "r" and single["schema"][-1]["type"] == "f64" and single["schema"][-1]["nullable"]
    assert len(a["args"]) == (2 if fn in BIVARIATE else 1)
    stages = stat_stages(src, [(fn, x, y, "r")], keys=[(c("x"), "k")], key_fields=[P.field("k", "i32", True)], mode="Partial")
    partial = typed(stages, 0)
    states = partial["schema"][1:]
    assert [f["name"] for f in states] == [f"r[{s}]" for s in STATE[fn]]
    assert [f["type"] for f in states] == ["u64"] + ["f64"] * (len(STATE[fn]) - 1)
    final = typed(stages, 1)
    assert final["schema"][-1]["type"] == "f64" and final["aggr"][0]["fn"] == CANON[fn]


@pytest.mark.parametrize("typ", ["i8", "i16", "i32", "i64", "u8", "u16", "u32", "u64", "f32", "f64", P.dec(15, 2), P.dec(38, 10)])
def test_numeric_arguments_are_coerced_to_f64(typ):
    sch = [P.field("a", typ, True), P.field("b", typ, False)]
    for fn in ("var_pop", "stddev", "covar_pop", "corr"):
        x, y = (c("a"), c("b")) if fn in BIVARIATE else (c("a"), None)
        out = typed(stat_stages(P.scan("t", sch), [(fn, x, y, "r")]))
        assert out["schema"][-1]["type"] == "f64"


@pytest.mark.parametrize("typ", ["utf8", "bool", "date32"])
def test_other_argument_types_are_refused(typ):
    sch = [P.field("a", typ, True), P.field("x", "f64", True)]
    for fn, x, y in (("var", c("a"), None), ("covar", c("x"), c("a")), ("corr", c("a"), c("x"))):
        e = refusal(stat_stages(P.scan("t", sch), [(fn, x, y, "r")]))
        assert e.code == UNSUPPORTED and typ in str(e), str(e)


def test_distinct_is_refused():
    st = stat_stages(P.scan("t", SCHEMA), [("stddev", c("x"), None, "r")])
    plan = st[0].plan
    plan["input"]["aggr"][0]["distinct"] = True
    with pytest.raises(engine.B200Error, match="DISTINCT"):
        engine.plan_typed_json(st[0].json("j"))


def test_wrong_argument_count_is_refused():
    with pytest.raises(engine.B200Error):
        engine.plan_typed_json(stat_stages(P.scan("t", SCHEMA), [("corr", c("x"), None, "r")])[0].json("j"))
    with pytest.raises(engine.B200Error):
        engine.plan_typed_json(stat_stages(P.scan("t", SCHEMA), [("var", c("x"), c("y"), "r")])[0].json("j"))


@pytest.mark.parametrize("fn,bad", [("var", ["count", "m2", "mean"]), ("stddev_pop", ["count", "mean", "sum"]),
                                    ("covar", ["count", "mean1", "algo_const", "mean2"]),
                                    ("corr", ["count", "mean1", "mean2", "m2_1", "m2_2", "algo_const"])])
def test_final_with_other_state_layout_is_refused(fn, bad):
    """A Final reads the states by position: a layout it does not know is refused, naming the column, never misread."""
    part = [P.field(f"r[{s}]", "u64" if s == "count" else "f64", True) for s in bad]
    plan = P.shuffle_writer(P.aggregate("Final", [], [P.agg(fn, None, "r")], P.shuffle_reader(1, part)), 2)
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(P.Stage(2, plan).json("j"))
    assert ei.value.code == UNSUPPORTED
    first_bad = next(i for i, s in enumerate(bad) if s != STATE[fn][i])
    assert f"r[{bad[first_bad]}]" in str(ei.value), str(ei.value)


def test_final_state_count_must_be_integer():
    part = [P.field("r[count]", "f64", True), P.field("r[mean]", "f64", True), P.field("r[m2]", "f64", True)]
    plan = P.shuffle_writer(P.aggregate("Final", [], [P.agg("var", None, "r")], P.shuffle_reader(1, part)), 2)
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(P.Stage(2, plan).json("j"))
    assert ei.value.code == UNSUPPORTED


def test_mixed_with_existing_aggregates_schema():
    src = P.scan("t", SCHEMA)
    extra = [("sum", c("x"), "sx", [P.field("sx[sum]", "i64", True)], None),
             ("avg", c("d"), "ad", [P.field("ad[count]", "u64", True), P.field("ad[sum]", P.dec(25, 2), True)], P.dec(15, 2))]
    st = stat_stages(src, [("corr", c("x"), c("d"), "r"), ("var_pop", c("y"), None, "v")], keys=[(c("s"), "k")],
                     key_fields=[P.field("k", "utf8", True)], mode="Partial", extra=extra)
    names = [f["name"] for f in typed(st, 0)["schema"]]
    assert names == ["k"] + [f["name"] for f in part_fields([("corr", 0, 0, "r"), ("var_pop", 0, 0, "v")])] + ["sx[sum]", "ad[count]", "ad[sum]"]
    fin = typed(st, 1)["schema"]
    assert [f["name"] for f in fin] == ["k", "r", "v", "sx", "ad"]
    assert [f["type"] for f in fin][1:3] == ["f64", "f64"]


# ---- the exact reference the device is checked against ----------------------------------------------------------------
def test_exact_reference_rules():
    assert exact("var", []) is None and exact("var_pop", []) is None
    assert exact("var", [3.0]) is None and exact("var_pop", [3.0]) == 0.0 and exact("stddev_pop", [3.0]) == 0.0
    assert exact("var", [1.0, 2.0]) == 0.5 and exact("var_pop", [1.0, 2.0]) == 0.25
    assert exact("covar", [1.0, None, 3.0], [2.0, 5.0, None]) is None  # one complete pair
    assert exact("covar_pop", [1.0, None, 3.0], [2.0, 5.0, None]) == 0.0
    assert exact("corr", [1.0, 2.0, 3.0], [2.0, 4.0, 6.0]) == 1.0
    assert exact("corr", [1.0, 2.0, 3.0], [5.0, 5.0, 5.0]) is None
    assert math.isnan(exact("var", [1.0, math.nan, 2.0])) and math.isnan(exact("var_pop", [1.0, math.inf]))
    # 1e9 + small integers: power sums cancel completely, the exact value does not
    xs = [1e9 + v for v in (0, 1, 2, 3, 4, 5, 6, 7)]
    assert exact("var", xs) == 6.0


def test_reference_goldens_match_the_exact_values():
    """The reference's seven goldens over alltypes_plain (context_basic.rs) are Welford's roundings of these values."""
    t = G.load("alltypes_plain")
    gold = json.load(open(G.__file__.replace("golden_data.py", "golden/reference_stat_aggregates.json")))["cases"]
    assert len(gold) == 7
    for case in gold:
        cols = [[float(v) for v in t.column(a).to_pylist()] for a in case["args"]]
        want = exact(case["fn"], cols[0], cols[1] if len(cols) > 1 else None)
        assert math.isclose(want, case["value"], rel_tol=1e-12, abs_tol=0), case


# ---- DataFusion's computation restated (Welford per row, Chan's merge), pinned against exact arithmetic ------------------
@pytest.mark.parametrize("parts", [1, 2, 5])
def test_welford_restatement_matches_exact(parts):
    import random
    rng = random.Random(5)
    sets = [[], [3.0], [1.0, 2.0], [1.0, 2.0, 4.0], [None, 1.0, None, 7.5, -2.0],
            [float(rng.randint(-50, 50)) for _ in range(300)], [1e6 + rng.random() for _ in range(500)]]
    for xs in sets:
        ys = [None if (x is not None and rng.random() < 0.1) else rng.gauss(0, 1) for x in xs]
        for fn in sorted(STATE):
            y = ys if fn in BIVARIATE else None
            want, got = exact(fn, xs, y), welford(fn, xs, y, parts)
            assert (want is None) == (got is None), (fn, xs, got, want)
            if want is not None:
                # Welford's per-row rounding is ~1e-8 relative on values near 1e6 (and unbounded relative for a
                # correlation near 0): this pins the restatement, not its accuracy
                assert math.isclose(got, want, rel_tol=1e-7, abs_tol=1e-9), (fn, parts, got, want)


def test_welford_restatement_reproduces_the_goldens():
    """The reference's golden values are what DataFusion's Welford computation rounds to: this restatement gives them."""
    t = G.load("alltypes_plain")
    gold = json.load(open(G.__file__.replace("golden_data.py", "golden/reference_stat_aggregates.json")))["cases"]
    for case in gold:
        cols = [[float(v) for v in t.column(a).to_pylist()] for a in case["args"]]
        got = welford(case["fn"], cols[0], cols[1] if len(cols) > 1 else None)
        assert math.isclose(got, case["value"], rel_tol=1e-15, abs_tol=0), (case, got)


def test_cpu_oracle_refuses_instead_of_misreading(oracle):
    """The CPU oracle does not compute these functions: a plan holding one is refused, never evaluated."""
    import pyarrow as pa
    from ballista_b200 import driver
    from oracle_ffi import OracleError
    b = pa.record_batch([pa.array([1, 1, 2], pa.int32()), pa.array([1.0, 2.0, 5.0]), pa.array([10.0, 20.0, 30.0])], names=["k", "x", "y"])
    oracle.register_batch("t", 0, b)
    sch = [P.field("k", "i32", False), P.field("x", "f64", True), P.field("y", "f64", True)]
    for fn, y in (("stddev", None), ("var_pop", None), ("covar", c("y")), ("corr", c("y"))):
        st = stat_stages(P.scan("t", sch), [(fn, c("x"), y, "r")], [(c("k"), "k")], extra=[("sum", c("y"), "sy", [], None)])
        with pytest.raises(OracleError, match="not computed"):
            driver.run_stages(oracle, st, f"orf-{fn}")


# ---- the protobuf path: every name and alias as a Ballista task carries it ------------------------------------------------
with open(G.__file__.replace("golden_data.py", "golden/stat_proto_plans.json")) as _fh:
    PROTO_CASES = json.load(_fh)["cases"]


def _agg_nodes(node):
    if isinstance(node, dict):
        if node.get("op") == "AggregateExec":
            yield node
        for v in node.values():
            yield from _agg_nodes(v)


@pytest.mark.parametrize("case", PROTO_CASES, ids=[c_["name"] for c_ in PROTO_CASES])
def test_protobuf_plans_decode_to_the_same_typed_plan(case):
    import base64
    decoded = json.loads(engine.plan_typed_json(engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]), "job")))
    want = json.loads(engine.plan_typed_json(case["ir"]))
    got_aggs, want_aggs = list(_agg_nodes(decoded)), list(_agg_nodes(want))
    assert len(got_aggs) == len(want_aggs) == 1
    g, w = got_aggs[0], want_aggs[0]
    assert g["mode"] == w["mode"]
    assert [(a["fn"], a["result_type"], len(a["args"])) for a in g["aggr"]] == [(a["fn"], a["result_type"], len(a["args"])) for a in w["aggr"]]
    assert [(f["name"], f["type"]) for f in g["schema"]] == [(f["name"], f["type"]) for f in w["schema"]]
    assert g["aggr"][0]["fn"] == CANON[case["fn"].lower()]
