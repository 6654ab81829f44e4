"""Scalar functions (DESIGN.md §3) on the host: the per-row restatement the device is checked against, pinned against
independent computations (datetime, pyarrow.compute, math, decimal, sqlite3, str); result types written down from the
§6 table; every protobuf fixture decoding to the plan it was generated from; and the refusals, each naming the culprit."""
import base64
import datetime
import decimal
import json
import math
import sqlite3

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import golden_data as G
import queries as Q
import scalar_fn_cases as S
from ballista_b200 import driver, engine
from ballista_b200 import plan as P

c = P.col
UNSUPPORTED = -2  # B200_ERR_UNSUPPORTED (include/b200exec.h)


# ---- the restatement against independent computations ---------------------------------------------------------------------
def test_date_parts_against_pyarrow_and_datetime():
    rng = np.random.default_rng(3)
    days = S.EDGE_DAYS + [int(v) for v in rng.integers(-719162, 2932896, 20000)]
    # ISO-week edges (Dec 29 - Jan 4) and leap days of many years, including before 1970
    for y in list(range(1, 40)) + list(range(1890, 2110)) + [2400, 9998, 9999]:
        for m, d in ((12, 29), (12, 30), (12, 31), (1, 1), (1, 2), (1, 3), (1, 4), (2, 28), (3, 1)):
            if y == 9999 and m == 1 and d > 4:
                continue
            days.append((datetime.date(y, m, d) - datetime.date(1970, 1, 1)).days)
        if y % 4 == 0 and (y % 100 != 0 or y % 400 == 0):
            days.append((datetime.date(y, 2, 29) - datetime.date(1970, 1, 1)).days)
    days = [d for d in days if -719162 <= d <= 2932896]
    arr = pa.array(days, pa.int32()).cast(pa.date32())
    ref = {"year": pc.year(arr), "quarter": pc.quarter(arr), "month": pc.month(arr), "week": pc.iso_week(arr),
           "day": pc.day(arr), "doy": pc.day_of_year(arr), "dow": pc.day_of_week(arr, count_from_zero=True, week_start=7)}
    assert min(days) < 0
    for part in S.PARTS:
        want = ref[part].to_pylist()
        got = [S.date_part(part, d) for d in days]
        assert got == want, part
    assert S.date_part("dow", 0) == 4 and S.date_part("week", (datetime.date(2021, 1, 3) - datetime.date(1970, 1, 1)).days) == 53
    assert S.date_part("year", None) is None


def test_abs_floor_ceil_against_math_and_decimal():
    for x in S.FLOATS:
        if math.isfinite(x):
            dx = decimal.Decimal(x)
            assert S.floor_(x) == float(dx.to_integral_value(decimal.ROUND_FLOOR))
            assert S.ceil_(x) == float(dx.to_integral_value(decimal.ROUND_CEILING))
            assert S.abs_(x) == float(abs(dx))
        else:
            assert (math.isnan(S.floor_(x)) and math.isnan(x)) or S.floor_(x) == x
    assert math.copysign(1, S.floor_(-0.0)) < 0 and math.copysign(1, S.ceil_(-0.5)) < 0 and math.copysign(1, S.abs_(-0.0)) > 0
    assert math.isnan(S.abs_(float("nan")))
    for typ, mn in S.INT_MIN.items():
        assert S.abs_(mn + 1, typ) == -(mn + 1)
        with pytest.raises(S.Overflow):
            S.abs_(mn, typ)
    assert S.abs_(decimal.Decimal("-1.25")) == decimal.Decimal("1.25")


@pytest.mark.parametrize("f32", [False, True])
def test_round_rules(f32):
    """half away from zero on x * 10^n, divided back; -0.0, NaN and infinities pass through"""
    assert 10.0 ** 22 == 1e22 and float(int(10 ** 22)) == 1e22   # 10^22 is exact in binary64: the factor is exact
    r = lambda x, n=0: S.round_(x, n, f32)  # noqa: E731
    for x, want in ((0.5, 1.0), (-0.5, -1.0), (1.5, 2.0), (2.5, 3.0), (-2.5, -3.0), (0.4, 0.0), (2.4, 2.0)):
        assert r(x) == want, x
    assert math.copysign(1, r(-0.0)) < 0 and math.copysign(1, r(-0.4)) < 0
    assert math.isnan(r(float("nan"))) and r(float("inf")) == math.inf and r(float("-inf")) == -math.inf
    assert r(499.0, -3) == 0.0
    if not f32:
        assert r(1234.5, -3) == 1000.0 and r(-1500.0, -3) == -2000.0 and r(0.125, 2) == 0.13
        assert r(0.49999999999999994) == 0.0
        assert r(1.005, 2) == 1.0          # 1.005 * 100 = 100.49999999999999 in binary64
        assert r(2.5, 22) == 2.5 and r(1e300, 22) == math.inf   # x * 10^22 overflows: the formula's result
        # the formula against exact decimal arithmetic where x * f is exact
        for x in (1.25, -3.75, 1234.5, 0.5, 7.0):
            for n in (0, 1, 2):
                q = (decimal.Decimal(x) * 10 ** n).to_integral_value(decimal.ROUND_HALF_UP)
                assert r(x, n) == float(q / 10 ** n), (x, n)
    else:  # f = 1 / 10^3 rounded to f32 is not 10^-3: f32 arithmetic gives what it gives, step by step
        assert r(1234.5, -3) == float(np.float32(1.0) / (np.float32(1.0) / np.float32(1000.0)))
        assert r(S._f32(2.675), 2) == float(np.float32(np.float32(268.0) / np.float32(100.0)))


def test_nullif_and_coalesce_against_sqlite():
    db = sqlite3.connect(":memory:")
    vals = [None, 0, 1, -1, 7, "a", "", "日本"]
    for a in vals:
        for b in vals:
            if a is not None and b is not None and type(a) is not type(b):
                continue
            want = db.execute("SELECT nullif(?, ?)", (a, b)).fetchone()[0]
            assert S.nullif(a, b) == want, (a, b)
            for d in (None, 5):
                want = db.execute("SELECT coalesce(?, ?, ?)", (a, b, d)).fetchone()[0]
                assert S.coalesce(a, b, d) == want, (a, b, d)
    # the engine's float equality is the total order of DESIGN §6 (iii), not SQL's IEEE equality
    assert S.nullif(float("nan"), float("nan")) is None and S.nullif(-0.0, 0.0) == -0.0 and S.nullif(0.0, 0.0) is None


def test_string_functions_against_bytes():
    for s in S.STRS:
        b = s.encode()
        assert S.char_length(s) == sum(1 for x in b if x & 0xC0 != 0x80)
        assert S.octet_length(s) == len(b)
        for p in S.PREFIXES:
            assert S.starts_with(s, p) == (b[:len(p.encode())] == p.encode())
            assert S.ends_with(s, p) == (len(p.encode()) <= len(b) and b[len(b) - len(p.encode()):] == p.encode())
    assert S.trim("btrim", "  a b  ") == "a b" and S.trim("ltrim", "  a ") == "a " and S.trim("rtrim", " a  ") == " a"
    assert S.trim("btrim", "\t a \n") == "\t a \n"       # only U+0020 by default
    assert S.trim("btrim", "x€ab€x ", "x€ ") == "ab" and S.trim("ltrim", "€€a€", "€") == "a€" and S.trim("rtrim", "a€€", "€") == "a"
    assert S.trim("btrim", "   ") == "" and S.trim("btrim", "") == "" and S.trim("btrim", "ab", None) is None
    assert S.starts_with("abc", "") is True and S.starts_with(None, "a") is None and S.ends_with("a", None) is None


# ---- result types (written down from the table in DESIGN §6) --------------------------------------------------------------
RESULT_TYPES = [
    (P.fn("date_part_week", c("d")), "i32", True), (P.fn("date_part_dow", c("dn")), "i32", False),
    (P.fn("abs", c("i8")), "i8", True), (P.fn("abs", c("u64")), "u64", True), (P.fn("abs", c("f32")), "f32", True),
    (P.fn("abs", c("dec")), {"dec": [15, 2]}, True), (P.fn("round", c("f64")), "f64", True),
    (P.fn("round", c("f32"), P.lit_i64(-2)), "f32", True), (P.fn("floor", c("f32")), "f32", True), (P.fn("ceil", c("f64")), "f64", True),
    (P.fn("nullif", c("dn"), c("dn")), "date32", True), (P.fn("nullif", c("s"), P.lit_utf8("")), "utf8", True),
    (P.fn("coalesce", c("s"), c("sn")), "utf8", False), (P.fn("coalesce", c("s"), c("p")), "utf8", True),
    (P.fn("coalesce", c("i32"), P.lit_i32(0)), "i32", False), (P.fn("character_length", c("s")), "i32", True),
    (P.fn("octet_length", c("sn")), "i32", False), (P.fn("starts_with", c("sn"), c("s")), "bool", True),
    (P.fn("ends_with", c("sn"), P.lit_utf8("a")), "bool", False), (P.fn("btrim", c("s")), "utf8", True),
    (P.fn("ltrim", c("sn"), P.lit_utf8("x")), "utf8", False), (P.fn("nullif", c("ts"), c("ts")), "ts", True), (P.fn("coalesce", c("ts"), P.lit_null("ts")), "ts", True), (P.fn("rtrim", c("sn"), c("p")), "utf8", True),
]
TYPE_SCHEMA = S.SCHEMA + [P.field("dn", "date32", False), P.field("sn", "utf8", False), P.field("ts", "ts", True)]


def _typed_projection(e):
    st = Q.Stage(1, P.shuffle_writer(P.project([(e, "r")], P.scan("x", TYPE_SCHEMA)), 1))
    return json.loads(engine.plan_typed_json(st.json("j")))["input"]["schema"][0]


@pytest.mark.parametrize("i", range(len(RESULT_TYPES)))
def test_result_types(i):
    e, typ, nullable = RESULT_TYPES[i]
    f = _typed_projection(e)
    assert (f["type"], f["nullable"]) == (typ, nullable), e


# ---- refusals ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("e,culprit", [
    (P.fn("round", c("dec")), "dec(15,2)"), (P.fn("floor", c("i32")), "i32"), (P.fn("ceil", c("dec")), "dec(15,2)"),
    (P.fn("round", c("f64"), P.lit_i64(23)), "23"), (P.fn("round", c("f64"), P.lit_i64(-40)), "-40"),
    (P.fn("date_part_year", P.cast(c("i64"), "ts")), "ts"), (P.fn("date_part_month", c("i32")), "i32"),
    (P.fn("abs", c("s")), "utf8"), (P.fn("character_length", c("i32")), "i32"), (P.fn("btrim", c("s"), c("i32")), "i32"),
    (P.fn("nullif", c("i32"), c("i64")), "i64"), (P.fn("coalesce", c("s"), c("i32")), "i32"),
])
def test_typing_refusals_name_the_type(e, culprit):
    with pytest.raises(engine.B200Error) as ei:
        _typed_projection(e)
    assert ei.value.code == UNSUPPORTED and culprit in str(ei.value), str(ei.value)


with open(G.__file__.replace("golden_data.py", "golden/scalar_fn_proto_plans.json")) as _fh:
    PROTO_CASES = json.load(_fh)["cases"]


def _fns(node, out):
    if isinstance(node, dict):
        if "fn" in node and "args" in node and "type" in node:
            out.append((node["fn"], json.dumps(node["type"])))
        for v in node.values():
            _fns(v, out)
    elif isinstance(node, list):
        for v in node:
            _fns(v, out)
    return out


def test_fixtures_cover_every_function_and_alias():
    spelled = {(x["spelled"].lower(), (x["part"] or "").lower()) for x in PROTO_CASES if not x["refused"]}
    names = {n for n, _ in spelled}
    assert {"date_part", "datepart", "abs", "round", "floor", "ceil", "nullif", "coalesce", "character_length", "char_length",
            "length", "octet_length", "starts_with", "ends_with", "btrim", "trim", "ltrim", "rtrim"} <= names
    assert {p for n, p in spelled if n in ("date_part", "datepart")} == set(S.PARTS)
    shapes = {x["name"].split("/")[1] for x in PROTO_CASES if not x["refused"]}
    assert shapes == {"projection", "filter", "group_key_and_argument"}


@pytest.mark.parametrize("case", [x for x in PROTO_CASES if not x["refused"]], ids=lambda x: x["name"])
def test_protobuf_plans_decode_to_the_same_typed_plan(case):
    decoded = engine.plan_typed_json(engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]), "job"))
    want = engine.plan_typed_json(case["ir"])
    got_fns, want_fns = _fns(json.loads(decoded), []), _fns(json.loads(want), [])
    assert got_fns == want_fns
    assert any(f == case["fn"] for f, _ in got_fns) or case["name"].endswith("/stage2")  # a Final reads the key as a column
    assert json.loads(decoded)["input"]["schema"] == json.loads(want)["input"]["schema"]


@pytest.mark.parametrize("case", [x for x in PROTO_CASES if x["refused"]], ids=lambda x: x["name"])
def test_protobuf_refusals_name_the_function_or_part(case):
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]), "job")
    assert ei.value.code == UNSUPPORTED and case["refused"] in str(ei.value).lower(), str(ei.value)


# ---- the CPU oracle ---------------------------------------------------------------------------------------------------------
def test_cpu_oracle_refuses_the_new_functions_and_keeps_year(oracle):
    """The oracle keeps computing date_part('year') and refuses (code -2) a plan holding any other new function, never
    evaluating it: the device results are checked against scalar_fn_cases instead."""
    from oracle_ffi import OracleError
    t = S.edge_table(64)
    G.register(oracle, "x", t, 1)
    year = [Q.Stage(1, P.shuffle_writer(P.project([(P.fn("date_part_year", c("d")), "y")], P.scan("x", S.SCHEMA)), 1))]
    got = driver.run_stages(oracle, year, "o-year").column("y").to_pylist()
    assert got == S.expected(t, [("y", None, lambda r: S.date_part("year", r["d"]), None)])["y"]
    for name, e, _, _ in S.projections():
        if name.startswith("dp_year"):
            continue
        st = [Q.Stage(1, P.shuffle_writer(P.project([(e, name)], P.scan("x", S.SCHEMA)), 1))]
        with pytest.raises(OracleError) as ei:
            driver.run_stages(oracle, st, f"o-{name}")
        assert ei.value.code == UNSUPPORTED, name
