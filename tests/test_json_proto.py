"""JsonScanExecNode (PhysicalPlanNode variant 31) from protobuf plan bytes, host only: the fixtures of
tests/golden/json_proto_plans.json (tests/golden/make_json_proto_plans.py; ballista/core/proto/*.proto) decode into
DataSourceExec nodes whose typed plan equals the typed plan of the IR they were generated from, carrying "format": "json" and
the byte ranges for b200_engine_register_json; a schema type the engine does not read is refused."""
import base64
import json
import os
import random

import pytest

from ballista_b200 import engine

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "json_proto_plans.json")) as fh:
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


def _decode(name):
    return json.loads(engine.plan_proto_to_json(base64.b64decode(next(c for c in CASES if c["name"] == name)["proto_b64"])))


@pytest.mark.parametrize("case", GOOD, ids=[c["name"] for c in GOOD])
def test_decoded_plan_equals_source_plan(case):
    got_ir = engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]))
    assert json.loads(engine.plan_typed_json(got_ir)) == json.loads(engine.plan_typed_json(case["ir"]))
    got, want = _scans(json.loads(got_ir), []), _scans(json.loads(case["ir"]), [])
    assert len(got) == len(want)
    for g, w in zip(got, want):
        for k in ("schema", "projection", "file_groups", "format", "file_ranges", "csv"):
            assert g.get(k) == w.get(k), k


def test_json_leaves_carry_format_and_ranges():
    names = {c["name"] for c in GOOD}
    assert {"q1/stage1", "q6/stage1", "q3/stage1", "q3/stage2", "ranges_multi_file", "projection_exprs"} <= names
    node = _scans(_decode("q1/stage1"), [])[0]
    assert node["table"] == "lineitem" and node["format"] == "json" and len(node["schema"]) == 16
    assert node["file_groups"] == [["/data/tpch/lineitem.json"]] and "file_ranges" not in node and "csv" not in node
    node = _scans(_decode("ranges_multi_file"), [])[0]
    assert node["file_ranges"] == [[[0, 4096], [0, 1000]], [[1000, 9000], None]]
    assert node["projection"] == [5, 0, 2]
    # the projection travelled as projection_exprs (FileScanExecConf field 13), not as `projection`
    assert _scans(_decode("projection_exprs"), [])[0]["projection"] == [1, 4]


@pytest.mark.parametrize("case", REFUSED, ids=[c["name"] for c in REFUSED])
def test_refusals(case):
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]))
    assert ei.value.code == case["code"] and case["needle"] in str(ei.value)


def test_damaged_json_scans_decode_to_valid_json_or_an_error():
    rnd = random.Random(20261018)
    outcomes = {"ok": 0, "error": 0}
    for c in GOOD[:3] + [c for c in GOOD if c["name"] in ("ranges_multi_file", "projection_exprs")]:
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
