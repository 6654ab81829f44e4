"""CSV / TPC-H .tbl scan on the device (b200_engine_register_csv): every result is compared column by column with the
reference reader of csv_reference.py (pyarrow.csv configured to the scan's rules, exact Python arithmetic for floats), float
bits included."""
import os
import random
import struct

import pyarrow as pa
import pytest

import csv_reference as R
import golden_data as G
import queries as Q
import ballista_b200 as bb
from ballista_b200 import driver, tpch
from util import assert_tables_equal

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CSV_DIR = os.path.join(GOLD, "csv")
REF = G.reference_expectations()
F = bb.plan.field


def scan(gpu, path, schema, table="csvt", partition=0, **kw):
    gpu.drop_table(table)
    gpu.register_csv(table, partition, path, schema, **kw)
    return pa.Table.from_batches([gpu.export_table(table, partition)])


def write(tmp_path, data: bytes, name="t.csv"):
    p = os.path.join(str(tmp_path), name)
    with open(p, "wb") as f:
        f.write(data)
    return p


def values(t: pa.Table):
    return {n: R.canon_values(t.column(n)) for n in t.column_names}


def test_aggregate_test_100_equals_golden(gpu):
    schema = G.ir_schema("aggregate_test_100")
    got = scan(gpu, os.path.join(CSV_DIR, "aggregate_test_100.csv"), schema, has_header=True)
    want = G.load("aggregate_test_100")
    assert got.column_names == want.column_names
    assert values(got) == values(want)
    # config[0] and the remote-sql variant run from the scanned table
    gpu.drop_table("aggregate_test_100")
    size = os.path.getsize(os.path.join(CSV_DIR, "aggregate_test_100.csv"))
    for p, (s, e) in enumerate(((0, size // 2), (size // 2, size))):
        gpu.register_csv("aggregate_test_100", p, [(os.path.join(CSV_DIR, "aggregate_test_100.csv"), s, e)], schema, has_header=True)
    out = driver.run_stages(gpu, Q.q_config0("aggregate_test_100", schema), "csv-c0")
    assert {str(k): v for k, v in zip(out.column(0).to_pylist(), out.column(1).to_pylist())} == REF["config0_min_b_group_a"]
    out = driver.run_stages(gpu, Q.q_remote_sql("aggregate_test_100", schema), "csv-rs").sort_by("c1")
    assert out.column("c1").to_pylist() == REF["remote_sql_groups"]


def test_python_test_csv_without_final_newline(gpu):
    got = scan(gpu, os.path.join(CSV_DIR, "test.csv"), [F("a", "i64"), F("b", "i64")], has_header=True)
    a, b = got.column("a").to_pylist(), got.column("b").to_pylist()
    assert [x for x in a if x > 2] == REF["python_filter_a_gt_2"]["a"]
    assert [y for x, y in zip(a, b) if x > 2] == REF["python_filter_a_gt_2"]["b"]


@pytest.mark.parametrize("name", ["customer", "part", "orders", "nation", "supplier", "partsupp", "region", "lineitem_partition0",
                                  "lineitem_partition1"])
def test_scheduler_tbl_fixtures(gpu, name):
    table = name.split("_")[0]
    path = os.path.join(CSV_DIR, name + ".tbl")
    schema = tpch.tbl_schema(table)
    real = [f["name"] for f in schema[:-1]]
    got = scan(gpu, path, schema, columns=real, delimiter="|")
    want = R.read(path, schema, delimiter="|").select(real)
    assert values(got) == values(want)
    # the empty last field is NULL, and `__placeholder` is declared non-nullable: materialising it is refused
    with pytest.raises(bb.B200Error) as ei:
        scan(gpu, path, schema, delimiter="|")
    assert ei.value.code == -1 and "'__placeholder', record 1" in str(ei.value)
    cols = [schema[-2]["name"], schema[0]["name"]]
    got = scan(gpu, path, schema, columns=cols, delimiter="|")
    assert got.column_names == cols
    assert values(got) == values(want.select(cols))


def _lineitem_tbl(oracle, oracle_lib, tmp_path, msf=20):
    n = oracle_lib.lib().oracle_tpch_table_rows(b"lineitem", msf)
    cols = [f["name"] for f in tpch.SCHEMAS["lineitem"]]
    oracle.drop_table("lineitem")
    oracle.tpch_generate("lineitem", msf, 0, 0, n, cols)
    host = pa.Table.from_batches([oracle.export_table("lineitem", 0)])
    path = os.path.join(str(tmp_path), "lineitem.tbl")
    R.write_tbl(host, path)
    return host, path


def test_q1_q6_from_tbl_and_ranges(gpu, oracle, oracle_lib, tmp_path):
    host, path = _lineitem_tbl(oracle, oracle_lib, tmp_path)
    cols = list(dict.fromkeys(tpch.Q1_COLUMNS + tpch.Q6_COLUMNS))
    schema = tpch.tbl_schema("lineitem")
    n = host.num_rows
    oracle.drop_table("lineitem")
    oracle.tpch_generate("lineitem", 20, 0, 0, n, cols)
    tpch.TABLE_LAYOUT["lineitem"] = cols
    try:
        launches = gpu.kernel_launches()
        gpu.drop_table("lineitem")
        gpu.register_csv("lineitem", 0, path, schema, columns=cols, delimiter="|")
        assert gpu.kernel_launches() > launches
        for name, st in (("q1", tpch.q1(4)), ("q6", tpch.q6(4))):
            got = driver.run_stages(gpu, st, f"csv-{name}")
            want = driver.run_stages(oracle, st, f"csv-{name}")
            assert_tables_equal(got, want, sort=False)
    finally:
        tpch.TABLE_LAYOUT.clear()
    # every split of the file into consecutive ranges yields every row exactly once, in order
    data = open(path, "rb").read()
    size = len(data)
    rng = random.Random(7)
    nl = [i for i in range(size) if data[i] == 10]
    for k in (1, 2, 5, 9):
        cuts = sorted(set([0, size] + [rng.randrange(1, size) for _ in range(k - 1)] + [nl[rng.randrange(len(nl))] + 1, nl[5]]))
        gpu.drop_table("li_r")
        for p in range(len(cuts) - 1):
            gpu.register_csv("li_r", p, [(path, cuts[p], cuts[p + 1])], schema, columns=["l_orderkey", "l_linenumber", "l_comment"],
                             delimiter="|")
        parts = [pa.Table.from_batches([gpu.export_table("li_r", p)]) for p in range(len(cuts) - 1)]
        got = pa.concat_tables([t.cast(parts[0].schema) for t in parts])
        assert got.column("l_orderkey").to_pylist() == host.column("l_orderkey").to_pylist()
        assert got.column("l_linenumber").to_pylist() == host.column("l_linenumber").to_pylist()
        assert got.column("l_comment").to_pylist() == host.column("l_comment").to_pylist()


def test_ranges_across_crlf(gpu, tmp_path):
    rows = [f"{i},{'x' * (i % 7)}" for i in range(200)]
    data = "\r\n".join(rows).encode() + b"\r\n"
    path = write(tmp_path, data)
    schema = [F("a", "i64"), F("b", "utf8", True)]
    size = len(data)
    for cut in range(0, size + 1, 3):
        got = []
        for p, (s, e) in enumerate(((0, cut), (cut, size))):
            got += scan(gpu, [(path, s, e)], schema, table="crlf", partition=p).column("a").to_pylist()
        assert got == list(range(200)), cut


EDGE = [
    # (name, bytes, schema, options)
    ("quoted", b'a,"x,y"\nb,"line1\nline2"\nc,"he said ""hi"""\n"d",\n', [F("k", "utf8"), F("v", "utf8", True)], {}),
    ("escaped", b'1,"a\\"b"\n2,"c\\\\d"\n3,"e""f"\n', [F("k", "i32"), F("v", "utf8")], {"escape": "\\"}),
    ("newlines", b'1,"a\r\nb"\r\n2,"c\rd"\n', [F("k", "i32"), F("v", "utf8")], {"newlines_in_values": True}),
    ("crlf_cr_blank", b'1,x\r\n\r\n2,y\r3,z\n\n\n4,w', [F("k", "i32"), F("v", "utf8")], {}),
    ("header_only", b'k,v\n', [F("k", "i32"), F("v", "utf8")], {"has_header": True}),
    ("empty", b'', [F("k", "i32"), F("v", "utf8")], {}),
    ("one_column", b'5\n6\n\n7', [F("k", "i64")], {}),
    ("nulls", b',,,,,,,\n1,2.5,3.5,1.25,2020-01-01,true,s,"x"\n"","","","","","","",""\n',
     [F("i", "i32", True), F("f", "f64", True), F("g", "f32", True), F("d", {"dec": [10, 2]}, True), F("t", "date32", True),
      F("b", "bool", True), F("s", "utf8", True), F("q", "utf8", True)], {}),
    ("utf8", "é,日本語\n😀,\"a,ü\"\n".encode(), [F("a", "utf8"), F("b", "utf8")], {}),
    ("ints", b'-128,255,-32768,65535,-2147483648,4294967295,-9223372036854775808,18446744073709551615\n'
             b'127,0,32767,0,2147483647,0,9223372036854775807,0\n+1,+2,+3,+4,+5,+6,+7,+8\n',
     [F("a", "i8"), F("b", "u8"), F("c", "i16"), F("d", "u16"), F("e", "i32"), F("f", "u32"), F("g", "i64"), F("h", "u64")], {}),
    ("decimals", b'99999999999999999999999999999999999999,-1.5,.25\n-99999999999999999999999999999999999999,+2,-.5\n0,0.0,0\n',
     [F("a", {"dec": [38, 0]}), F("b", {"dec": [5, 2]}), F("c", {"dec": [3, 2]})], {}),
    ("dates", b'0001-01-01\n1970-01-01\n2000-02-29\n9999-12-31\n1969-12-31\n', [F("d", "date32")], {}),
    ("bools", b'true\nFALSE\nTrue\nfAlSe\n', [F("b", "bool")], {}),
    ("tab_delim_quote", b"1\t'a\tb'\n2\t'c''d'\n", [F("k", "i32"), F("v", "utf8")], {"delimiter": "\t", "quote": "'"}),
]


@pytest.mark.parametrize("name,data,schema,opts", EDGE, ids=[e[0] for e in EDGE])
def test_edge_shapes(gpu, tmp_path, name, data, schema, opts):
    path = write(tmp_path, data)
    got = scan(gpu, path, schema, **opts)
    want = R.expected_edge(name)
    assert got.num_rows == len(want[schema[0]["name"]])
    assert values(got) == want


def _float_strings(seed=11):
    rng = random.Random(seed)
    out = []
    for _ in range(50000):
        x = struct.unpack("<d", struct.pack("<Q", rng.getrandbits(64)))[0]
        if x != x or x in (float("inf"), float("-inf")):
            continue
        out.append(repr(x))
        out.append("%.17g" % x)
    for _ in range(20000):
        nd = rng.randint(1, 40)
        digits = "".join(rng.choice("0123456789") for _ in range(nd))
        pos = rng.randint(0, nd)
        s = (rng.choice(["", "-", "+"]) + digits[:pos] + ("." + digits[pos:] if pos < nd else "") +
             ("e%d" % rng.randint(-340, 330) if rng.random() < 0.7 else ""))
        out.append(s)
    # subnormals, overflow, underflow, exact halfway points (of doubles and of floats) that need the exact comparison
    out += ["4.9406564584124654e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "2.2250738585072011e-308",
            "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308", "1e309", "-1e400", "1e-400",
            "9007199254740993", "9007199254740995", "9007199254740993.000000000000000000000001", "16777217", "16777219",
            "1.40129846e-45", "7.00649232e-46", "7.006492321624086e-46", "3.4028235677973366e38", "3.4028235e38", "3.4028236e38",
            "0.1", "0.3", "123456789012345678901234567890", "inf", "-Infinity", "NaN", "-0", "-0.0", "+0e10", "0.000", ".5", "5.",
            "1E5", "1e+5", "1e-5"]
    # exact halfway points between adjacent doubles and adjacent floats, printed in full
    from fractions import Fraction
    for _ in range(300):
        m = rng.getrandbits(52) | (1 << 52)
        e = rng.randint(-1074, 900)
        h = Fraction(2 * m + 1) * Fraction(2) ** (e - 1)
        out.append(R.fraction_to_decimal(h))
        m32 = rng.getrandbits(23) | (1 << 23)
        e32 = rng.randint(-149, 100)
        out.append(R.fraction_to_decimal(Fraction(2 * m32 + 1) * Fraction(2) ** (e32 - 1)))
    return out


def test_floats_correctly_rounded(gpu, tmp_path):
    strs = _float_strings()
    path = write(tmp_path, ("\n".join(f"{s},{s}" for s in strs) + "\n").encode())
    got = scan(gpu, path, [F("d", "f64"), F("f", "f32")])
    d_bits = struct.unpack(f"<{len(strs)}Q", got.column("d").combine_chunks().buffers()[1][:8 * len(strs)])
    f_bits = struct.unpack(f"<{len(strs)}I", got.column("f").combine_chunks().buffers()[1][:4 * len(strs)])
    bad = []
    for s, db, fb in zip(strs, d_bits, f_bits):
        wd, wf = R.f64_bits(s), R.f32_bits(s)
        if (db != wd and not (R.is_nan64(db) and R.is_nan64(wd))) or (fb != wf and not (R.is_nan32(fb) and R.is_nan32(wf))):
            bad.append((s, hex(db), hex(wd), hex(fb), hex(wf)))
    assert not bad, bad[:10]


MALFORMED = [
    ("fields_short", b'1,2\n3\n', [F("a", "i32"), F("b", "i32")], "record 2"),
    ("fields_long", b'1,2\n3,4,5\n', [F("a", "i32"), F("b", "i32")], "record 2"),
    ("not_int", b'1\n 2\n', [F("a", "i32")], "column 'a', record 2"),
    ("int_range", b'1\n128\n', [F("a", "i8")], "column 'a', record 2"),
    ("unsigned_minus", b'-1\n', [F("a", "u32")], "column 'a', record 1"),
    ("dec_scale", b'1.25\n1.255\n', [F("a", {"dec": [10, 2]})], "record 2"),
    ("dec_exp", b'1e2\n', [F("a", {"dec": [10, 2]})], "exponent"),
    ("dec_precision", b'1000.00\n', [F("a", {"dec": [5, 2]})], "precision"),
    ("bad_float", b'1.5\n1.5x\n', [F("a", "f64")], "record 2"),
    ("bad_date", b'2021-02-29\n', [F("a", "date32")], "date"),
    ("loose_date", b'2021-2-01\n', [F("a", "date32")], "date"),
    ("bad_bool", b'yes\n', [F("a", "bool")], "boolean"),
    ("bad_utf8", b'ok\n\xff\xfe\n', [F("a", "utf8")], "UTF-8"),
    ("null_non_nullable", b'1\n""\n', [F("a", "i32")], "column 'a', record 2"),
]


@pytest.mark.parametrize("name,data,schema,needle", MALFORMED, ids=[m[0] for m in MALFORMED])
def test_malformed_is_refused_and_engine_keeps_working(gpu, tmp_path, name, data, schema, needle):
    path = write(tmp_path, data, name + ".csv")
    gpu.drop_table("bad")
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_csv("bad", 0, path, schema)
    assert ei.value.code == -1, str(ei.value)
    assert needle in str(ei.value) and name + ".csv" in str(ei.value), str(ei.value)
    with pytest.raises(bb.B200Error):
        gpu.export_table("bad", 0)
    ok = scan(gpu, write(tmp_path, b'1,x\n2,y\n', "ok.csv"), [F("a", "i32"), F("b", "utf8")])
    assert ok.column("a").to_pylist() == [1, 2]


def test_refusals(gpu, tmp_path):
    path = write(tmp_path, b'1,2\n')
    sch = [F("a", "i32"), F("b", "i32")]
    cases = [
        ({"comment": "#"}, -2, "comment"),
        ({"truncate_rows": True}, -2, "truncate_rows"),
        ({"delimiter": ",,"}, -1, "delimiter"),
        ({"quote": ""}, -1, "quote"),
        ({"escape": "ab"}, -1, "escape"),
    ]
    import json
    for extra, code, needle in cases:
        spec = {"files": [{"path": path}], "schema": sch, **extra}
        with pytest.raises(bb.B200Error) as ei:
            gpu.register_csv_json("ref", 0, json.dumps(spec))
        assert ei.value.code == code and needle in str(ei.value), (extra, str(ei.value))
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_csv("ref", 0, [(path, 0, 2)], sch, newlines_in_values=True)
    assert ei.value.code == -2 and "newlines_in_values" in str(ei.value)
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_csv("ref", 0, path, [F("a", "ts"), F("b", "i32")])
    assert ei.value.code == -2 and "'a'" in str(ei.value) and "ts" in str(ei.value)
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_csv("ref", 0, os.path.join(str(tmp_path), "missing.csv"), sch)
    assert ei.value.code == -5
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_csv_json("ref", 0, "{not json")
    assert ei.value.code == -1
    assert scan(gpu, path, sch).column("b").to_pylist() == [2]


def test_duplicate_and_empty_column_lists(gpu, tmp_path):
    path = write(tmp_path, b'1,x\n2,y\n')
    sch = [F("a", "i32"), F("b", "utf8")]
    gpu.drop_table("dup")
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_csv("dup", 0, path, sch, columns=["a", "a"])
    assert ei.value.code == -1 and "twice" in str(ei.value)
    # an empty list materialises nothing (a count(*) scan of a .tbl file): no NULL check on `__placeholder`, records
    # still counted and their field counts still checked
    gpu.register_csv("dup", 0, os.path.join(CSV_DIR, "nation.tbl"), tpch.tbl_schema("nation"), columns=[], delimiter="|")
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_csv("dup", 0, write(tmp_path, b'1,x\n2\n', "short.csv"), sch, columns=[])
    assert ei.value.code == -1 and "record 2" in str(ei.value)
    assert scan(gpu, path, sch, columns=["b", "a"]).column_names == ["b", "a"]


def test_several_files_in_order_and_errors_name_the_right_file(gpu, tmp_path):
    a = write(tmp_path, b'k,v\n1,a\n2,b\n', "a.csv")
    b = write(tmp_path, b'k,v\n3,c', "b.csv")
    c = write(tmp_path, b'k,v\n4,d\n5,"e"\n6,f\n', "c.csv")
    sch = [F("k", "i64"), F("v", "utf8")]
    got = scan(gpu, [a, b, (c, 0, 10), (c, 10, 100)], sch, has_header=True)
    assert got.column("k").to_pylist() == [1, 2, 3, 4, 5, 6]
    assert got.column("v").to_pylist() == ["a", "b", "c", "d", "e", "f"]
    bad = write(tmp_path, b'k,v\n7,g\nx,h\n', "bad.csv")
    with pytest.raises(bb.B200Error) as ei:
        scan(gpu, [a, b, bad], sch, has_header=True)
    assert "bad.csv" in str(ei.value) and "column 'k', record 2 (byte offset 8)" in str(ei.value), str(ei.value)


def test_floats_beyond_the_kept_digits(gpu, tmp_path):
    # more than 800 significant digits: the digits past the kept ones only matter as "non-zero" (ties break upwards)
    from fractions import Fraction
    half = R.fraction_to_decimal(Fraction(2 ** 53 + 1, 2 ** 53) * Fraction(1, 2 ** 1000))   # a double halfway point, 730+ digits
    strs = [half, half + "0" * 200, half + "0" * 120 + "1", "1." + "0" * 900 + "1", "0." + "9" * 1000, "1" * 1200 + "e-1200"]
    path = write(tmp_path, ("\n".join(f"{s},{s}" for s in strs) + "\n").encode())
    got = scan(gpu, path, [F("d", "f64"), F("f", "f32")])
    assert R.canon_values(got.column("d")) == [R.f64_bits(s) for s in strs]
    assert R.canon_values(got.column("f")) == [R.f32_bits(s) for s in strs]


def test_q1_q6_prepared_from_csv_plan_bytes(gpu, oracle, oracle_lib, tmp_path):
    """The stage plans as a scheduler ships them (CsvScanExecNode leaves over lineitem.tbl), the table registered from the
    decoded node's own options and file group the way an executor-side shim does it."""
    import base64
    import json
    with open(os.path.join(GOLD, "csv_proto_plans.json")) as fh:
        proto = {c["name"]: base64.b64decode(c["proto_b64"]) for c in json.load(fh)["cases"]}
    host, path = _lineitem_tbl(oracle, oracle_lib, tmp_path)
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
        assert node["format"] == "csv" and node["file_groups"] == [["/data/tpch/lineitem.tbl"]]
        gpu.drop_table("lineitem")
        driver.register_csv_scan(gpu, node, 0, {"/data/tpch/lineitem.tbl": path})
        layout = [f["name"] for f in node["schema"][:max(node["projection"]) + 1]]
        oracle.drop_table("lineitem")
        oracle.tpch_generate("lineitem", 20, 0, 0, n, layout)
        tpch.TABLE_LAYOUT["lineitem"] = layout
        try:
            stages = getattr(tpch, q)(4)
            got = driver.run_stages(FromProto(gpu, q), stages, f"csvpb-{q}")
            want = driver.run_stages(oracle, stages, f"csvpb-{q}")
            assert_tables_equal(got, want, sort=False)
        finally:
            tpch.TABLE_LAYOUT.clear()
