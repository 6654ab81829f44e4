"""The string builders (DESIGN.md §6 (xi)) on the host: the per-row restatement of tests/string_build_cases.py pinned against
independent computations (sqlite3 for concat / concat_ws / ||, pyarrow.compute.cast for the casts, Python str for reverse
and repeat); result types and nullability; every refusal by name, including the unchanged upper / lower / replace ones; the
CPU oracle still computing integer -> Utf8 and refusing the new functions; the protobuf fixtures decoding to the typed plan
of their IR."""
import base64
import datetime
import json
import os
import sqlite3

import pyarrow as pa
import pyarrow.compute as pc
import pytest

import golden_data as G
import queries as Q
import string_build_cases as S
from ballista_b200 import driver, engine
from ballista_b200 import plan as P

c = P.col
UNSUPPORTED = -2  # B200_ERR_UNSUPPORTED (include/b200exec.h)
HERE = os.path.dirname(os.path.abspath(__file__))
SAMPLE = [None, "", "a", "héllo", "日本語", "𝄞x", " ", "x" * 300]


# ---- the restatement against independent computations ---------------------------------------------------------------------
def test_concat_rules_against_sqlite():
    db = sqlite3.connect(":memory:")
    for a in SAMPLE:
        for b in SAMPLE:
            got = db.execute("SELECT concat(?, ?), ? || ?, concat(?, '-', ?)", (a, b, a, b, a, b)).fetchone()
            assert got == (S.concat(a, b), S.str_concat(a, b), S.concat(a, "-", b)), (a, b)
            if "" in (a, b):
                continue  # sqlite's concat_ws also drops empty values; PostgreSQL and DataFusion keep them (pinned below)
            for sep in (None, "", ", ", "—"):
                want = db.execute("SELECT concat_ws(?, ?, ?, 'z')", (sep, a, b)).fetchone()[0]
                assert S.concat_ws(sep, a, b, "z") == want, (sep, a, b)
    assert db.execute("SELECT concat(NULL, NULL)").fetchone()[0] == S.concat(None, None) == ""
    assert S.concat_ws(", ", None, "", "z") == ", z" and S.concat_ws(None, "a") is None


def test_reverse_and_repeat_against_str():
    for s in SAMPLE:
        assert S.reverse(s) == (None if s is None else "".join(reversed(list(s))))
        for n in (-3, 0, 1, 2, 5, None):
            want = None if s is None or n is None else s * max(n, 0)
            assert S.repeat(s, n) == want
    assert S.reverse("a𝄞é") == "é𝄞a"  # code points, not bytes
    with pytest.raises(S.TooLong):
        S.repeat("ab", 2**30)


def test_integer_casts_against_pyarrow():
    for k, vals in S.INT_EDGES.items():
        arr = pa.array(vals + [None], S.P_TYPES[k])
        assert pc.cast(arr, pa.string()).to_pylist() == [S.cast_int(v) for v in arr.to_pylist()], k


def test_decimal_casts_against_pyarrow():
    for k, (scale, vals) in S.DEC_EDGES.items():
        p = {"dec": 15, "dec0": 38, "dec9": 10}[k]
        arr = pa.array([S._dec(v, scale) for v in vals] + [None], pa.decimal128(p, scale))
        for v, ref in zip(vals + [None], pc.cast(arr, pa.string()).to_pylist()):
            if ref is not None and "E" in ref:
                continue  # Arrow C++ writes values below 1e-6 in scientific notation; arrow-rs does not (pinned below)
            assert S.cast_decimal(v, scale) == ref, (k, v)
    assert S.cast_decimal(1, 9) == "0.000000001" and S.cast_decimal(-10**9 + 1, 9) == "-0.999999999"
    assert S.cast_decimal(-5, 2) == "-0.05" and S.cast_decimal(12345, 2) == "123.45" and S.cast_decimal(7, 0) == "7"


def test_date_casts_against_pyarrow_and_chrono_rule():
    first, last = datetime.date(1, 1, 1).toordinal() - S.EPOCH_ORDINAL, datetime.date(9999, 12, 31).toordinal() - S.EPOCH_ORDINAL
    days = list(range(first, first + 800)) + list(range(-2000, 2000)) + list(range(last - 800, last + 1)) + list(range(first, last, 997))
    arr = pa.array(days, pa.int32()).cast(pa.date32())
    assert pc.cast(arr, pa.string()).to_pylist() == [S.cast_date(d) for d in days]
    assert S.cast_date(last + 1) == "+10000-01-01"
    assert S.cast_date(first - 1) == "0000-12-31"
    assert S.cast_date(first - 367) == "-0001-12-31"


def test_bool_casts_against_pyarrow():
    arr = pa.array([True, False, None])
    assert pc.cast(arr, pa.string()).to_pylist() == [S.cast_bool(v) for v in arr.to_pylist()]


# ---- typing -------------------------------------------------------------------------------------------------------------------
def _typed_projection(e):
    st = Q.Stage(1, P.shuffle_writer(P.project([(e, "r")], P.scan("x", S.SCHEMA)), 1))
    return json.loads(engine.plan_typed_json(st.json("j")))["input"]["schema"][0]


RESULT_TYPES = [
    (P.fn("concat", c("a"), c("b")), False), (P.fn("concat", P.lit_utf8(None)), False),
    (P.str_concat(c("a"), P.lit_utf8("x")), True), (P.str_concat(P.lit_utf8("x"), P.lit_utf8("y")), False),
    (P.fn("concat_ws", P.lit_utf8(","), c("a")), False), (P.fn("concat_ws", c("sep"), P.lit_utf8("x")), True),
    (P.fn("repeat", P.lit_utf8("ab"), P.lit_i64(2)), False), (P.fn("repeat", P.lit_utf8("ab"), c("n")), True),
    (P.fn("reverse", c("a")), True), (P.fn("reverse", P.lit_utf8("ab")), False),
    (P.cast(c("k"), "utf8"), False), (P.cast(c("dec"), "utf8"), True), (P.cast(c("d"), "utf8"), True),
]


@pytest.mark.parametrize("i", range(len(RESULT_TYPES)))
def test_result_types(i):
    e, nullable = RESULT_TYPES[i]
    f = _typed_projection(e)
    assert (f["type"], f["nullable"]) == ("utf8", nullable), e


@pytest.mark.parametrize("e,culprit", [
    (P.fn("concat", c("a"), c("k")), "i32"), (P.str_concat(c("a"), c("n")), "i64"), (P.fn("concat_ws", c("k"), c("a")), "i32"),
    (P.fn("repeat", c("a"), c("k")), "i32"), (P.fn("repeat", c("k"), P.lit_i64(2)), "i32"), (P.fn("reverse", c("d")), "date32"),
] + [(P.fn(f, c("a"), P.lit_i64(3)), f) for f in ("lpad", "rpad", "left", "right", "split_part")]
  + [(P.fn(f, c("a")), f) for f in ("to_hex", "to_char", "translate", "initcap")])
def test_typing_refusals_name_the_culprit(e, culprit):
    with pytest.raises(engine.B200Error) as ei:
        _typed_projection(e)
    assert ei.value.code == UNSUPPORTED and culprit in str(ei.value), str(ei.value)


@pytest.mark.parametrize("f", ["upper", "lower", "replace"])
def test_upper_lower_replace_stay_refused(f):
    """unchanged: the plan IR does not know them (a malformed plan) and the protobuf decoder refuses them by name"""
    with pytest.raises(engine.B200Error) as ei:
        _typed_projection(P.fn(f, c("a")))
    assert ei.value.code == -1 and f"unknown scalar function '{f}'" in str(ei.value)
    with open(os.path.join(HERE, "golden", "scalar_fn_proto_plans.json")) as fh:
        case = next(x for x in json.load(fh)["cases"] if x["refused"] == f)
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]), "job")
    assert ei.value.code == UNSUPPORTED and f in str(ei.value).lower()


# ---- the CPU oracle -------------------------------------------------------------------------------------------------------------
def test_cpu_oracle_casts_integers_and_refuses_the_builders(oracle):
    from oracle_ffi import OracleError
    t = S.edge_table(64).select(["k", "a", "b", "sep", "n", "i8", "i16", "i32", "i64"])
    sch = S.SCHEMA[:9]
    G.register(oracle, "x", t, 1)
    for k in ("i8", "i16", "i32", "i64"):
        st = [Q.Stage(1, P.shuffle_writer(P.project([(P.cast(c(k), "utf8"), "r")], P.scan("x", sch)), 1))]
        got = driver.run_stages(oracle, st, f"o-{k}").column("r").to_pylist()
        assert got == [S.cast_int(v) for v in t.column(k).to_pylist()], k
    for name, e, _ in S.projections():
        if name.startswith("cast_"):
            continue
        st = [Q.Stage(1, P.shuffle_writer(P.project([(e, "r")], P.scan("x", sch)), 1))]
        with pytest.raises(OracleError) as ei:
            driver.run_stages(oracle, st, f"o-{name}")
        assert "not computed by this consumer" in str(ei.value), name


# ---- protobuf --------------------------------------------------------------------------------------------------------------------
with open(os.path.join(HERE, "golden", "string_build_proto_plans.json")) as _fh:
    PROTO_CASES = json.load(_fh)["cases"]
GOOD = [x for x in PROTO_CASES if "refused" not in x]
REFUSED = [x for x in PROTO_CASES if "refused" in x]


def test_fixtures_cover_every_form():
    names = {x["name"].split("/")[0] for x in GOOD}
    assert {"concat", "string_concat", "concat_ws", "repeat", "repeat_column_count", "reverse", "cast_int", "cast_uint64",
            "cast_decimal", "cast_date", "cast_bool", "try_cast_int"} <= names
    assert {x["refused"] for x in REFUSED} == {"lpad", "rpad", "to_hex", "to_char", "left", "right", "split_part", "translate", "initcap"}
    pipe = json.loads(engine.plan_proto_to_json(base64.b64decode(next(x for x in GOOD if x["name"] == "string_concat/projection")["proto_b64"])))
    assert '"bin": "||"' in json.dumps(pipe)


@pytest.mark.parametrize("case", GOOD, ids=[x["name"] for x in GOOD])
def test_protobuf_plans_decode_to_the_same_typed_plan(case):
    decoded = engine.plan_typed_json(engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]), "job"))
    assert json.loads(decoded) == json.loads(engine.plan_typed_json(case["ir"]))


@pytest.mark.parametrize("case", REFUSED, ids=[x["name"] for x in REFUSED])
def test_protobuf_refusals_name_the_function(case):
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]), "job")
    assert ei.value.code == UNSUPPORTED and case["refused"] in str(ei.value), str(ei.value)
