"""ILIKE, the regex operators and regexp_like from protobuf plan bytes, host only: the fixtures of
tests/golden/regex_proto_plans.json (tests/golden/make_regex_proto_plans.py; ballista/core/proto/*.proto) decode into IR
whose typed plan equals the typed plan of the IR they were generated from -- NOT, ILIKE and flags included -- and the refused
cases decode to the same refusal as their IR."""
import base64
import json
import os

import pytest

from ballista_b200 import engine

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "regex_proto_plans.json")) as fh:
    CASES = json.load(fh)["cases"]
GOOD = [c for c in CASES if "code" not in c]
REFUSED = [c for c in CASES if "code" in c]


@pytest.mark.parametrize("case", GOOD, ids=[c["name"] for c in GOOD])
def test_decoded_plan_equals_source_plan(case):
    got_ir = engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]))
    assert json.loads(engine.plan_typed_json(got_ir)) == json.loads(engine.plan_typed_json(case["ir"]))


def test_fixtures_cover_every_form():
    names = {c["name"].split("/")[0] for c in GOOD}
    assert {"ilike", "not_ilike", "match", "imatch", "not_match", "not_imatch", "regexp_like", "regexp_like_flags_i",
            "regexp_like_flags_is", "match_null_pattern"} <= names
    ilike = json.loads(engine.plan_proto_to_json(base64.b64decode(next(c for c in GOOD if c["name"] == "not_ilike/filter")["proto_b64"])))
    pred = ilike["input"]["predicate"]
    assert pred["case_insensitive"] is True and pred["negated"] is True
    plain = engine.plan_proto_to_json(base64.b64decode(next(c for c in GOOD if c["name"] == "like_plain/filter")["proto_b64"]))
    assert "case_insensitive" not in plain  # plain LIKE decodes as before


def _outcome(f):
    try:
        f()
    except engine.B200Error as e:
        return e.code, str(e)
    return 0, ""


@pytest.mark.parametrize("case", REFUSED, ids=[c["name"] for c in REFUSED])
def test_refused_cases_decode_to_the_same_refusal(case):
    raw = base64.b64decode(case["proto_b64"])
    code, msg = _outcome(lambda: engine.plan_typed_json(engine.plan_proto_to_json(raw)))
    assert code == case["code"] and case["needle"] in msg, msg
    if "ilike_column" not in case["name"]:  # the IR has no spelling of an ILIKE over a column pattern
        want = _outcome(lambda: engine.plan_typed_json(case["ir"]))
        assert (code, msg.split(": ", 1)[1]) == (want[0], want[1].split(": ", 1)[1])
