"""The JSON scan's reference reader (json_reference.py), host only: pinned to hand-written lines for every accepted shape and
every refusal, and cross-checked against pyarrow.json.read_json on generated files both accept."""
import datetime as dt
import json
import random
from decimal import Decimal

import pyarrow as pa
import pyarrow.json as pajson
import pytest

import csv_reference as CR
import json_reference as R


def F(name, t, nullable=False):
    return {"name": name, "type": t, "nullable": nullable}


ACCEPTED = [
    (b'{"a":1}\n{"a":-2}\n', [F("a", "i8")], {"a": [1, -2]}),
    (b'{"a":18446744073709551615}', [F("a", "u64")], {"a": [2 ** 64 - 1]}),
    (b'{"a":1.25,"b":-0}\n', [F("a", {"dec": [5, 2]}), F("b", {"dec": [5, 2]})], {"a": [Decimal("1.25")], "b": [Decimal(0)]}),
    (b'{"a":-0}\n{"a":1e-400}\n{"a":0.1}\n', [F("a", "f64")], {"a": [CR.b64(-0.0), 0, CR.b64(0.1)]}),
    (b'{"a":16777217}\n', [F("a", "f32")], {"a": [CR.b32(16777216.0)]}),
    (b'{"a":"2020-01-31"}\n', [F("a", "date32")], {"a": [dt.date(2020, 1, 31)]}),
    (b'{"a":true}\n{"a":false}\n{"a":null}\n', [F("a", "bool", True)], {"a": [True, False, None]}),
    (b'{"a":""}\n{"a":null}\n{}\n', [F("a", "utf8", True)], {"a": ["", None, None]}),
    (b'{"a":"\\u00e9\\ud83d\\ude00\\n\\/","z":[{"q":[]}]}\r\n', [F("a", "utf8")], {"a": ["é😀\n/"]}),
    (b'{"\\u0061":7}\n', [F("a", "i32")], {"a": [7]}),
    (b'\n \t\r\n{ "a" : 1 } \r\n\n', [F("a", "i32")], {"a": [1]}),
    (b'{"a":1,"a":2}\n', [F("b", "i32", True)], {"b": [None]}),   # duplicate keys that are not materialised
    (b'', [F("a", "i32")], {"a": []}),
    (b'{"x":' + b'[' * 64 + b']' * 64 + b'}', [F("a", "i32", True)], {"a": [None]}),
]


@pytest.mark.parametrize("data,schema,want", ACCEPTED)
def test_accepted_lines(data, schema, want):
    assert R.read(data, schema) == want


REFUSED = [
    (b'{"a":1,\n"b":2}\n', R.INVALID, 1, None),
    (b'{"a":1}{"a":2}\n', R.INVALID, 1, None),
    (b'[{"a":1}]\n', R.INVALID, 1, None),
    (b'{"a":1} 2\n', R.INVALID, 1, None),
    (b'{"a":NaN}\n', R.INVALID, 1, None),
    (b'{"a":Infinity}\n', R.INVALID, 1, None),
    (b'{"a":"\\ud800"}\n', R.INVALID, 1, None),
    (b'{"a":"\x01"}\n', R.INVALID, 1, None),
    (b'{"a":"\xed\xa0\x80"}\n', R.INVALID, 1, None),
    (b'{"a":01}\n', R.INVALID, 1, None),
    (b'{"x":' + b'[' * 65 + b']' * 65 + b'}', R.UNSUPPORTED, 1, None),
    (b'{"a":1}\n\n{"a":1,"a":1}\n', R.INVALID, 2, "a"),
    (b'{"a":"1"}\n', R.INVALID, 1, "a"),
    (b'{"a":1.5}\n', R.INVALID, 1, "a"),
    (b'{"a":1e0}\n', R.INVALID, 1, "a"),
    (b'{"a":128}\n', R.INVALID, 1, "a"),
    (b'{"a":null}\n', R.INVALID, 1, "a"),
    (b'{}\n', R.INVALID, 1, "a"),
    (b'{"a":[1]}\n', R.INVALID, 1, "a"),
]


@pytest.mark.parametrize("data,code,record,column", REFUSED)
def test_refused_lines(data, code, record, column):
    with pytest.raises(R.Refused) as ei:
        R.read(data, [F("a", "i8")])
    assert (ei.value.code, ei.value.record, ei.value.column) == (code, record, column)


def test_byte_offsets_skip_blank_lines():
    with pytest.raises(R.Refused) as ei:
        R.read(b'{"a":1}\n  \n{"a":"x"}\n', [F("a", "i32")])
    assert (ei.value.record, ei.value.offset) == (2, 11)


def _generated(seed, n=400):
    rng = random.Random(seed)
    lines = []
    for i in range(n):
        o = {}
        if rng.random() < 0.9:
            o["i"] = R.Num(str(rng.randint(-2 ** 63, 2 ** 63 - 1)))
        if rng.random() < 0.9:
            x = rng.uniform(-1e6, 1e6) * 10 ** rng.randint(-30, 30)
            o["f"] = R.Num(repr(x))
        if rng.random() < 0.9:
            o["s"] = "".join(rng.choice("ab é日😀\"\\\n\t/{}[],:") for _ in range(rng.randint(0, 12)))
        if rng.random() < 0.9:
            o["b"] = rng.random() < 0.5
        if rng.random() < 0.3:
            o["junk"] = {"x": [1, {"y": "z"}]}
        if rng.random() < 0.1:
            o["s"] = None
        lines.append(R.dumps_record(o))
    return ("\n".join(lines) + "\n").encode()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_reference_agrees_with_pyarrow(tmp_path, seed):
    data = _generated(seed)
    schema = [F("i", "i64", True), F("f", "f64", True), F("s", "utf8", True), F("b", "bool", True)]
    want = R.read(data, schema)
    path = tmp_path / "g.json"
    path.write_bytes(data)
    pa_schema = pa.schema([("i", pa.int64()), ("f", pa.float64()), ("s", pa.string()), ("b", pa.bool_())])
    got = pajson.read_json(str(path), parse_options=pajson.ParseOptions(explicit_schema=pa_schema, unexpected_field_behavior="ignore"))
    assert {n: CR.canon_values(got.column(n)) for n in got.column_names} == want


def test_dumps_record_round_trips():
    o = {"a": R.Num("1.50"), "s": "é\"x", "n": None}
    line = R.dumps_record(o)
    assert line == '{"a":1.50,"s":"é\\"x","n":null}'
    assert json.loads(line) == {"a": 1.5, "s": 'é"x', "n": None}
