"""Window plans from protobuf bytes without a GPU: every fixture of tests/golden/window_proto_plans.json decodes to the typed
plan it was written from, and every refused fixture carries its code and the name of its case.  Also the two typing rules
that only show in the typed plan: nth_value / lag / lead positions beyond any partition are clamped, and a LAG / LEAD default
is cast to the argument's type."""
import base64
import json
import os

import pytest

import window_cases as W
from ballista_b200 import engine
from ballista_b200 import plan as P

c = P.col
FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "window_proto_plans.json")


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


def _window(exprs):
    return P.window([dict(w, partition_by=[c("g")], order_by=[P.sort_key(c("o"))]) for w in exprs], P.scan("t", W.SCHEMA), [c("g")])


def test_positions_beyond_any_partition_are_clamped():
    big = 2 ** 63 - 1
    t = _typed(json.dumps(_window([P.win("nth_value", "nv", [c("i64"), P.lit_i64(big)]), P.win("lag", "lg", [c("i64"), P.lit_i64(big)]),
                                   P.win("lead", "ld", [c("i64"), P.lit_i64(-big)]), P.win("nth_value", "n2", [c("i64"), P.lit_i64(7)])])))
    assert [w["n"] for w in t["window_expr"]] == [2 ** 40, -(2 ** 40), -(2 ** 40), 7]


def test_lag_default_is_cast_to_the_argument_type():
    t = _typed(json.dumps(_window([P.win("lag", "a", [c("i32"), P.lit_i64(1), P.lit_i64(-7)]),
                                   P.win("lag", "b", [c("dec"), P.lit_i64(1), P.lit_i64(3)]),
                                   P.win("lag", "c", [c("f64"), P.lit_i64(1), P.lit_i64(2)]),
                                   P.win("lag", "d", [c("dec"), P.lit_i64(1), P.lit_dec(15, 4, 1)])])))
    assert [(w["default"]["lit"]["t"], w["default"]["lit"]["v"]) for w in t["window_expr"]] == [
        ("i32", -7), ({"dec": [12, 2]}, "300"), ("f64", 2.0), ({"dec": [12, 2]}, "150")]
    for bad, what in ((P.win("lag", "x", [c("i32"), P.lit_i64(1), P.lit_i64(2 ** 40)]), "i64"),
                      (P.win("lag", "x", [c("dec"), P.lit_i64(1), P.lit_dec(15, 6, 3)]), "dec(6,3)"),
                      (P.win("lag", "x", [c("i64"), P.lit_i64(1), P.lit_f64(1.5)]), "f64")):
        with pytest.raises(engine.B200Error) as ei:
            _typed(json.dumps(_window([bad])))
        assert ei.value.code == -2 and f"the default of lag (x) has type {what} and does not cast exactly" in str(ei.value), str(ei.value)
