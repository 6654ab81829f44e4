"""Newline-delimited JSON scan on the device (b200_engine_register_json): every result is compared column by column with the
reference reader of json_reference.py (Python's json, exact arithmetic for numbers), float bits included, and every refusal
with the code, file, column, record and byte offset the reference gives."""
import base64
import json
import os
import random
import struct
from decimal import Decimal
from fractions import Fraction

import pyarrow as pa
import pytest

import csv_reference as CR
import json_reference as R
import ballista_b200 as bb
from ballista_b200 import driver, tpch
from util import assert_tables_equal

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F = bb.plan.field


def write(tmp_path, data: bytes, name="t.json"):
    p = os.path.join(str(tmp_path), name)
    with open(p, "wb") as f:
        f.write(data)
    return p


def scan(gpu, files, schema, table="jsont", partition=0, columns=None):
    gpu.drop_table(table)
    gpu.register_json(table, partition, files, schema, columns=columns)
    return pa.Table.from_batches([gpu.export_table(table, partition)])


def values(t: pa.Table):
    return {n: CR.canon_values(t.column(n)) for n in t.column_names}


def check(gpu, tmp_path, data: bytes, schema, columns=None):
    want = R.read(data, schema, columns)
    got = scan(gpu, write(tmp_path, data), schema, columns=columns)
    assert got.column_names == list(want)
    assert got.num_rows == len(next(iter(want.values()))) if want else True
    assert values(got) == want
    return got


def refused(gpu, tmp_path, data: bytes, schema, name="bad.json", columns=None):
    with pytest.raises(R.Refused) as w:
        R.read(data, schema, columns)
    want = w.value
    path = write(tmp_path, data, name)
    gpu.drop_table("bad")
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_json("bad", 0, path, schema, columns=columns)
    msg = str(ei.value)
    assert ei.value.code == want.code, (msg, want)
    assert name in msg and f"record {want.record} (byte offset {want.offset})" in msg, (msg, want)
    if want.column is not None:
        assert f"column '{want.column}'" in msg, (msg, want)
    with pytest.raises(bb.B200Error):
        gpu.export_table("bad", 0)
    ok = scan(gpu, write(tmp_path, b'{"a":1}\n{"a":2}\n', "ok.json"), [F("a", "i32")])
    assert ok.column("a").to_pylist() == [1, 2]
    return msg


ALL_TYPES = [F("i8", "i8", True), F("u8", "u8", True), F("i16", "i16", True), F("u16", "u16", True), F("i32", "i32", True),
             F("u32", "u32", True), F("i64", "i64", True), F("u64", "u64", True), F("d", {"dec": [38, 4]}, True),
             F("d2", {"dec": [5, 2]}, True), F("f", "f64", True), F("g", "f32", True), F("t", "date32", True), F("b", "bool", True),
             F("s", "utf8", True)]

EDGE = [
    ("types", b'{"i8":-128,"u8":255,"i16":-32768,"u16":65535,"i32":-2147483648,"u32":4294967295,"i64":-9223372036854775808,'
              b'"u64":18446744073709551615,"d":12345678901234567890123456789012.3456,"d2":-999.99,"f":-0,"g":1.5e-3,'
              b'"t":"2000-02-29","b":true,"s":"x"}\n'
              b'{"i8":127,"u8":0,"i16":32767,"u16":0,"i32":2147483647,"u32":0,"i64":9223372036854775807,"u64":0,"d":-0.5,"d2":0,'
              b'"f":1E308,"g":-0.0,"t":"1969-12-31","b":false,"s":""}\n'
              b'{"d":0.0001,"d2":1.5,"f":5e-324,"g":3.4028235e38,"t":"0001-01-01","s":"\\u0000"}\n', ALL_TYPES),
    ("nulls_missing_unknown", b'{"a":null,"b":null}\n{}\n{"zz":[1,{"x":[[]]}],"a":1,"q":{"a":2,"b":"s"}}\n'
                              b'{"b":"{}[]\\",:\\\\","z":"{}[]\\",:\\\\"}\n', [F("a", "i64", True), F("b", "utf8", True)]),
    ("escapes", b'{"s":"\\"\\\\\\/\\b\\f\\n\\r\\t","k":1}\n{"s":"\\u00e9\\u65e5\\ud83d\\ude00\\u0041","k":2}\n'
                b'{"\\u0073":"escaped key","\\u006b":3}\n{"s":"\xc3\xa9\xe6\x97\xa5\xf0\x9f\x98\x80 raw","k":4}\n'
                b'{"s":"","k":5}\n{"s":null,"k":6}\n', [F("s", "utf8", True), F("k", "i32")]),
    ("crlf_blank_ws", b'\n  \r\n{"a":1}\r\n\t\n{"a":2}  \r\n\r\n\n{ "a" : 3 }', [F("a", "i32")]),
    ("empty", b'', [F("a", "i32")]),
    ("blank_only", b'\n \n\r\n\t\n', [F("a", "i32")]),
    ("deep_unknown", b'{"x":' + b'[' * 64 + b']' * 64 + b',"a":1,"y":' + b'{"k":' * 63 + b'{}' + b'}' * 63 + b'}\n', [F("a", "i32")]),
    ("nested_in_strings", b'{"a":"[[[[{{{{","b":"}}]]"}\n', [F("a", "utf8"), F("b", "utf8")]),
    ("bools_dates", b'{"b":true,"t":"9999-12-31"}\n{"b":false,"t":"1970-01-01"}\n', [F("b", "bool"), F("t", "date32")]),
]


@pytest.mark.parametrize("name,data,schema", EDGE, ids=[e[0] for e in EDGE])
def test_edge_shapes(gpu, tmp_path, name, data, schema):
    check(gpu, tmp_path, data, schema)


def test_string_of_one_megabyte_and_more_than_2_20_rows(gpu, tmp_path):
    big = "".join(chr(0x41 + (i % 26)) for i in range(1 << 20))
    data = ('{"s":"' + big + '\\u00e9","k":1}\n{"s":"' + big[:1000] + '\\\\x","k":2}\n').encode()
    check(gpu, tmp_path, data, [F("s", "utf8"), F("k", "i32")])
    n = (1 << 20) + 123
    data = "".join('{"k":%d,"v":"%s"}\n' % (i, "x" * (i % 5)) for i in range(n)).encode()
    got = scan(gpu, write(tmp_path, data, "many.json"), [F("k", "i64"), F("v", "utf8")])
    assert got.num_rows == n
    assert got.column("k").to_pylist() == list(range(n))
    assert got.column("v").to_pylist()[-7:] == ["x" * (i % 5) for i in range(n - 7, n)]


def _float_strings(seed=5):
    rng = random.Random(seed)
    out = []
    for _ in range(20000):
        x = struct.unpack("<d", struct.pack("<Q", rng.getrandbits(64)))[0]
        if x != x or x in (float("inf"), float("-inf")):
            continue
        r = repr(x)
        out.append(r if "e" in r or "." in r else r + ".0")
    for _ in range(10000):
        nd = rng.randint(1, 40)
        digits = str(rng.randint(1, 9)) + "".join(rng.choice("0123456789") for _ in range(nd - 1))
        pos = rng.randint(1, nd)
        s = rng.choice(["", "-"]) + digits[:pos] + ("." + digits[pos:] if pos < nd else "")
        if rng.random() < 0.7:
            s += "e%d" % rng.randint(-340, 330)
        out.append(s)
    for _ in range(200):
        m = rng.getrandbits(52) | (1 << 52)
        out.append(CR.fraction_to_decimal(Fraction(2 * m + 1) * Fraction(2) ** (rng.randint(-1074, 900) - 1)))
        m32 = rng.getrandbits(23) | (1 << 23)
        out.append(CR.fraction_to_decimal(Fraction(2 * m32 + 1) * Fraction(2) ** (rng.randint(-149, 100) - 1)))
    half = CR.fraction_to_decimal(Fraction(2 ** 53 + 1, 2 ** 53) * Fraction(1, 2 ** 1000))
    out += [half, half + "0" * 200, half + "0" * 120 + "1", "1." + "0" * 900 + "1", "0." + "9" * 1000, "1" * 1200 + "e-1200",
            "-0", "-0.0", "0e10", "1e400", "-1e400", "1e-400"]
    return [s if not s.startswith(".") else "0" + s for s in out]


def test_floats_correctly_rounded(gpu, tmp_path):
    strs = _float_strings()
    data = "".join('{"d":%s,"f":%s}\n' % (s, s) for s in strs).encode()
    check(gpu, tmp_path, data, [F("d", "f64"), F("f", "f32")])


def test_random_ranges_hold_every_record_once(gpu, tmp_path):
    rng = random.Random(3)
    for eol in (b"\n", b"\r\n"):
        lines = [('{"k":%d,"s":"%s"}' % (i, "ab" * (i % 7))).encode() for i in range(3000)]
        data = b""
        for i, ln in enumerate(lines):
            data += ln + eol + (b"  " + eol if i % 97 == 0 else b"")
        path = write(tmp_path, data, "ranges.json")
        size = len(data)
        for k in (1, 2, 7, 23):
            cuts = sorted(set([0, size] + [rng.randrange(1, size) for _ in range(k - 1)]))
            got = []
            for p in range(len(cuts) - 1):
                t = scan(gpu, [(path, cuts[p], cuts[p + 1])], [F("k", "i64"), F("s", "utf8")], table="rng", partition=p)
                got += t.column("k").to_pylist()
            assert got == list(range(3000)), (eol, cuts)


def test_several_files_in_order_and_errors_name_the_right_file(gpu, tmp_path):
    a = write(tmp_path, b'{"k":1}\n{"k":2}\n', "a.json")
    b = write(tmp_path, b'\n{"k":3}', "b.json")
    c = write(tmp_path, b'{"k":4}\n{"k":5}\n{"k":6}\n', "c.json")
    sch = [F("k", "i64")]
    got = scan(gpu, [a, b, (c, 0, 9), (c, 9, 100)], sch)
    assert got.column("k").to_pylist() == [1, 2, 3, 4, 5, 6]
    bad = write(tmp_path, b'{"k":7}\n\n{"k":"8"}\n', "bad.json")
    with pytest.raises(bb.B200Error) as ei:
        scan(gpu, [a, b, bad], sch)
    assert "bad.json" in str(ei.value) and "column 'k', record 2 (byte offset 9)" in str(ei.value), str(ei.value)


def test_duplicate_and_empty_column_lists(gpu, tmp_path):
    path = write(tmp_path, b'{"a":1,"b":"x"}\n{"a":2,"b":"y"}\n')
    sch = [F("a", "i32"), F("b", "utf8")]
    gpu.drop_table("dup")
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_json("dup", 0, path, sch, columns=["a", "a"])
    assert ei.value.code == -1 and "twice" in str(ei.value)
    # an empty list materialises nothing, but the records are still counted and checked
    gpu.register_json("dup", 0, path, sch, columns=[])
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_json("dup", 0, write(tmp_path, b'{"a":1}\n{"a":1,}\n', "short.json"), sch, columns=[])
    assert ei.value.code == -1 and "record 2" in str(ei.value)
    assert scan(gpu, path, sch, columns=["b", "a"]).column_names == ["b", "a"]


S1 = [F("a", "i32", True)]
MALFORMED = [
    ("split_object", b'{"a":1,\n"b":2}\n', S1),
    ("two_objects", b'{"a":1}{"a":2}\n', S1),
    ("top_array", b'{"a":1}\n[1,2]\n', S1),
    ("top_scalar", b'{"a":1}\n"x"\n', S1),
    ("trailing", b'{"a":1} x\n', S1),
    ("unterminated_string", b'{"a":1,"b":"abc}\n', S1),
    ("control_in_string", b'{"a":1,"b":"a\tb"}\n', S1),
    ("bad_utf8", b'{"a":1,"b":"\xff"}\n', S1),
    ("overlong_utf8", b'{"a":1,"b":"\xc0\xaf"}\n', S1),
    ("bad_escape", b'{"a":1,"b":"\\x"}\n', S1),
    ("short_u", b'{"a":1,"b":"\\u12"}\n', S1),
    ("lone_high", b'{"a":1,"b":"\\ud800x"}\n', S1),
    ("lone_low", b'{"a":1,"b":"\\udc00"}\n', S1),
    ("nan", b'{"a":1,"b":NaN}\n', S1),
    ("infinity", b'{"a":1,"b":-Infinity}\n', S1),
    ("leading_zero", b'{"a":1,"b":01}\n', S1),
    ("bare_dot", b'{"a":1,"b":1.}\n', S1),
    ("plus", b'{"a":1,"b":+1}\n', S1),
    ("bad_literal", b'{"a":1,"b":tru}\n', S1),
    ("mismatched", b'{"a":1,"b":[}\n', S1),
    ("missing_colon", b'{"a" 1}\n', S1),
    ("trailing_comma", b'{"a":1,}\n', S1),
    ("single_quotes", b"{'a':1}\n", S1),
    ("duplicate_key", b'{"a":1}\n{"a":1,"a":2}\n', S1),
    ("duplicate_escaped_key", b'{"a":1,"\\u0061":2}\n', S1),
    ("too_deep", b'{"x":' + b'[' * 65 + b']' * 65 + b'}\n', S1),
    ("string_in_int", b'{"a":"1"}\n', S1),
    ("fraction_in_int", b'{"a":1.0}\n', S1),
    ("exponent_in_int", b'{"a":1e2}\n', S1),
    ("int_range", b'{"a":2147483648}\n', S1),
    ("unsigned_minus", b'{"a":-1}\n', [F("a", "u32", True)]),
    ("object_in_int", b'{"a":{"b":1}}\n', S1),
    ("array_in_utf8", b'{"a":[1]}\n', [F("a", "utf8", True)]),
    ("number_in_utf8", b'{"a":1}\n', [F("a", "utf8", True)]),
    ("bool_in_int", b'{"a":true}\n', S1),
    ("string_in_bool", b'{"a":"true"}\n', [F("a", "bool", True)]),
    ("number_in_date", b'{"a":20200101}\n', [F("a", "date32", True)]),
    ("bad_date", b'{"a":"2021-02-29"}\n', [F("a", "date32", True)]),
    ("dec_exponent", b'{"a":1e2}\n', [F("a", {"dec": [10, 2]}, True)]),
    ("dec_scale", b'{"a":1.255}\n', [F("a", {"dec": [10, 2]}, True)]),
    ("dec_precision", b'{"a":1000.00}\n', [F("a", {"dec": [5, 2]}, True)]),
    ("null_non_nullable", b'{"a":1}\n{"a":null}\n', [F("a", "i32")]),
    ("missing_non_nullable", b'{"a":1}\n\n{"b":1}\n', [F("a", "i32")]),
]


@pytest.mark.parametrize("name,data,schema", MALFORMED, ids=[m[0] for m in MALFORMED])
def test_malformed_is_refused_and_engine_keeps_working(gpu, tmp_path, name, data, schema):
    refused(gpu, tmp_path, data, schema, name + ".json")


def test_refusals(gpu, tmp_path):
    path = write(tmp_path, b'{"a":1}\n')
    sch = [F("a", "i32")]
    for extra, code, needle in (({"newline_delimited": False}, -2, "newline_delimited"), ({"compression": "GZIP"}, -2, "compression")):
        with pytest.raises(bb.B200Error) as ei:
            gpu.register_json_json("ref", 0, json.dumps({"files": [path], "schema": sch, **extra}))
        assert ei.value.code == code and needle in str(ei.value), (extra, str(ei.value))
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_json("ref", 0, path, [F("a", "ts"), F("b", "i32")])
    assert ei.value.code == -2 and "'a'" in str(ei.value)
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_json("ref", 0, os.path.join(str(tmp_path), "missing.json"), sch)
    assert ei.value.code == -5
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_json_json("ref", 0, "{not json")
    assert ei.value.code == -1
    assert scan(gpu, path, sch).column("a").to_pylist() == [1]


def test_launch_accounting(gpu, tmp_path):
    """A scan's launches are counted where they are enqueued and do not grow with the rows: records (3), fields (1) and one
    converter per column at least; the column images after the scan depend on the values, so the values repeat."""
    sch = [F("k", "i64"), F("s", "utf8"), F("d", {"dec": [12, 2]})]
    counts = []
    for n in (10, 5000):
        path = write(tmp_path, ('{"k":7,"s":"vv","d":1.25}\n' * n).encode(), f"n{n}.json")
        gpu.drop_table("acc")
        before = gpu.kernel_launches()
        gpu.register_json("acc", 0, path, sch)
        counts.append(gpu.kernel_launches() - before)
    assert counts[0] >= 4 + len(sch) and counts[0] == counts[1], counts


def _lineitem_json(oracle, oracle_lib, tmp_path, msf=20):
    n = oracle_lib.lib().oracle_tpch_table_rows(b"lineitem", msf)
    cols = [f["name"] for f in tpch.SCHEMAS["lineitem"]]
    oracle.drop_table("lineitem")
    oracle.tpch_generate("lineitem", msf, 0, 0, n, cols)
    host = pa.Table.from_batches([oracle.export_table("lineitem", 0)])
    path = os.path.join(str(tmp_path), "lineitem.json")
    rows = host.to_pylist()
    with open(path, "w") as fh:
        for r in rows:
            fh.write("{" + ",".join(json.dumps(k) + ":" + (str(v) if isinstance(v, (int, Decimal)) else json.dumps(str(v)))
                                    for k, v in r.items()) + "}\n")
    return host, path


def test_q1_q6_from_json_lineitem(gpu, oracle, oracle_lib, tmp_path):
    host, path = _lineitem_json(oracle, oracle_lib, tmp_path)
    cols = list(dict.fromkeys(tpch.Q1_COLUMNS + tpch.Q6_COLUMNS))
    schema = tpch.SCHEMAS["lineitem"]
    n = host.num_rows
    oracle.drop_table("lineitem")
    oracle.tpch_generate("lineitem", 20, 0, 0, n, cols)
    tpch.TABLE_LAYOUT["lineitem"] = cols
    try:
        gpu.drop_table("lineitem")
        gpu.register_json("lineitem", 0, path, schema, columns=cols)
        for name, st in (("q1", tpch.q1(4)), ("q6", tpch.q6(4))):
            got = driver.run_stages(gpu, st, f"json-{name}")
            want = driver.run_stages(oracle, st, f"json-{name}")
            assert_tables_equal(got, want, sort=False)
    finally:
        tpch.TABLE_LAYOUT.clear()
    # the whole table read back equals what was written
    got = scan(gpu, path, schema, table="li_all")
    for c in ("l_orderkey", "l_extendedprice", "l_shipdate", "l_comment"):
        assert got.column(c).to_pylist() == host.column(c).to_pylist(), c


def test_q1_q6_prepared_from_json_plan_bytes(gpu, oracle, oracle_lib, tmp_path):
    """The stage plans as a scheduler ships them (JsonScanExecNode leaves over lineitem.json), the table registered from the
    decoded node's file group the way an executor-side shim does it."""
    with open(os.path.join(GOLD, "json_proto_plans.json")) as fh:
        proto = {c["name"]: base64.b64decode(c["proto_b64"]) for c in json.load(fh)["cases"]}
    host, path = _lineitem_json(oracle, oracle_lib, tmp_path)
    n = host.num_rows

    class FromProto:
        def __init__(self, e, q):
            self._e, self._q = e, q

        def __getattr__(self, k):
            return getattr(self._e, k)

        def create_query_stage_exec(self, job_id, stage_id, plan_json):
            return self._e.create_query_stage_exec_proto(job_id, stage_id, proto[f"{self._q}/stage{stage_id}"])

    for q in ("q1", "q6"):
        node = json.loads(bb.engine.plan_proto_to_json(proto[f"{q}/stage1"]))
        while node.get("op") != "DataSourceExec":
            node = node["input"]
        assert node["format"] == "json" and node["file_groups"] == [["/data/tpch/lineitem.json"]]
        gpu.drop_table("lineitem")
        driver.register_json_scan(gpu, node, 0, {"/data/tpch/lineitem.json": path})
        layout = [f["name"] for f in node["schema"][:max(node["projection"]) + 1]]
        oracle.drop_table("lineitem")
        oracle.tpch_generate("lineitem", 20, 0, 0, n, layout)
        tpch.TABLE_LAYOUT["lineitem"] = layout
        try:
            stages = getattr(tpch, q)(4)
            got = driver.run_stages(FromProto(gpu, q), stages, f"jsonpb-{q}")
            want = driver.run_stages(oracle, stages, f"jsonpb-{q}")
            assert_tables_equal(got, want, sort=False)
        finally:
            tpch.TABLE_LAYOUT.clear()
