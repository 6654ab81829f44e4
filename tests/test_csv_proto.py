"""CsvScanExecNode (PhysicalPlanNode variant 2) from protobuf plan bytes, host only: the fixtures of
tests/golden/csv_proto_plans.json (tests/golden/make_csv_proto_plans.py; ballista/core/proto/*.proto) decode into
DataSourceExec nodes whose typed plan equals the typed plan of the IR they were generated from, carrying the reader options
and byte ranges for b200_engine_register_csv; the options the device scan does not implement are refused by name."""
import base64
import json
import os
import random

import pytest

from ballista_b200 import engine

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "csv_proto_plans.json")) as fh:
    CASES = json.load(fh)["cases"]
GOOD = [c for c in CASES if "code" not in c]
REFUSED = [c for c in CASES if "code" in c]


def _scans(node, out):
    if isinstance(node, dict):
        if node.get("op") == "DataSourceExec":
            out.append(node)
        for v in node.values():
            _scans(v, out)
    elif isinstance(node, list):
        for v in node:
            _scans(v, out)
    return out


@pytest.mark.parametrize("case", GOOD, ids=[c["name"] for c in GOOD])
def test_decoded_plan_equals_source_plan(case):
    got_ir = engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]))
    assert json.loads(engine.plan_typed_json(got_ir)) == json.loads(engine.plan_typed_json(case["ir"]))
    got, want = _scans(json.loads(got_ir), []), _scans(json.loads(case["ir"]), [])
    assert len(got) == len(want)
    for g, w in zip(got, want):
        for k in ("schema", "projection", "file_groups", "format", "csv", "file_ranges"):
            assert g.get(k) == w.get(k), k


def test_tbl_scans_are_what_tpch_rs_plans():
    names = {c["name"] for c in GOOD}
    assert {"q1/stage1", "q6/stage1", "q3/stage1", "q3/stage2", "header_quote_escape_ranges"} <= names
    node = _scans(json.loads(engine.plan_proto_to_json(base64.b64decode(next(c for c in GOOD if c["name"] == "q1/stage1")["proto_b64"]))), [])[0]
    assert node["table"] == "lineitem" and node["schema"][-1]["name"] == "__placeholder" and len(node["schema"]) == 17
    assert node["csv"] == {"has_header": False, "delimiter": "|", "quote": '"', "escape": None, "newlines_in_values": False}
    assert "file_ranges" not in node


@pytest.mark.parametrize("case", REFUSED, ids=[c["name"] for c in REFUSED])
def test_refusals_name_the_option(case):
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]))
    assert ei.value.code == case["code"] and case["needle"] in str(ei.value)


def test_damaged_csv_scans_decode_to_valid_json_or_an_error():
    rnd = random.Random(20261016)
    outcomes = {"ok": 0, "error": 0}
    for c in GOOD[:3] + [c for c in GOOD if c["name"] == "header_quote_escape_ranges"]:
        raw = base64.b64decode(c["proto_b64"])
        for _ in range(300):
            b = bytearray(raw)
            for _k in range(rnd.randrange(1, 4)):
                b[rnd.randrange(len(b))] ^= 1 << rnd.randrange(8)
            try:
                json.loads(engine.plan_proto_to_json(bytes(b)))
                outcomes["ok"] += 1
            except engine.B200Error:
                outcomes["error"] += 1
    assert outcomes["ok"] > 0 and outcomes["error"] > 0
