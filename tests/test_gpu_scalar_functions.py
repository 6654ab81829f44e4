"""GPU: the scalar functions of DESIGN.md §3 on the device, bit-exact against the per-row restatement in scalar_fn_cases.py
(itself pinned against datetime / pyarrow / math / sqlite3 / str by test_scalar_functions.py): in projections over several
1024-row tiles, as FilterExec predicates (on the tile VM, not the fast filter), as group keys and aggregate arguments over
SF1 lineitem through Partial -> hash shuffle -> FinalPartitioned, from the protobuf fixtures, and the errors."""
import base64
import datetime
import json
import os
from decimal import Decimal

import pyarrow as pa
import pyarrow.compute as pc
import pytest

import golden_data as G
import queries as Q
import scalar_fn_cases as S
from ballista_b200 import driver, engine
from ballista_b200 import plan as P

pytestmark = pytest.mark.gpu
c = P.col
HERE = os.path.dirname(os.path.abspath(__file__))
EXECUTION, UNSUPPORTED = -3, -2


def _project(exprs, table="x", schema=S.SCHEMA):
    return [Q.Stage(1, P.shuffle_writer(P.project([(e, n) for n, e in exprs], P.scan(table, schema)), 1))]


@pytest.fixture(scope="module")
def edge():
    return S.edge_table()


@pytest.mark.parametrize("parts", [1, 3])
def test_projection_of_every_function(gpu, edge, parts):
    """>= 3 full 1024-row tiles plus a partial one, NULLs in every argument position across the tiles"""
    G.register(gpu, "x", edge, parts)
    projs = S.projections()
    want = S.expected(edge, projs)
    vm0 = gpu.counter("vm")
    bad = []
    for i in range(0, len(projs), 6):
        chunk = projs[i:i + 6]
        out = driver.run_stages(gpu, _project([(n, e) for n, e, _, _ in chunk]), f"sf-proj-{parts}-{i}")
        assert out.num_rows == edge.num_rows
        for name, _, _, typ in chunk:
            got = out.column(name).to_pylist()
            if out.schema.field(name).type != typ or not S.same_values(got, want[name]):
                rows = [(r, g, w) for r, (g, w) in enumerate(zip(got, want[name])) if not S.same_values([g], [w])]
                bad.append((name, str(out.schema.field(name).type), len(rows), rows[:4]))
    assert not bad, bad
    assert gpu.counter("vm") > vm0


def test_date_part_year_unchanged(gpu, oracle, edge):
    """date_part('year') now runs as OP_DATE_PART(year): the oracle still computes it, and the two agree"""
    for e in (gpu, oracle):
        G.register(e, "x", edge, 2)
    st = _project([("y", P.fn("date_part_year", c("d"))), ("y2", P.binop("+", P.fn("date_part_year", c("d")), P.lit_i32(1)))])
    got, want = driver.run_stages(gpu, st, "sf-year"), driver.run_stages(oracle, st, "sf-year")
    assert got.column("y").to_pylist() == want.column("y").to_pylist() == S.expected(edge, [("y", None, lambda r: S.date_part("year", r["d"]), None)])["y"]
    assert got.column("y2").to_pylist() == want.column("y2").to_pylist()


FILTERS = [
    ("starts_with", P.fn("starts_with", c("s"), c("p")), lambda r: S.starts_with(r["s"], r["p"])),
    ("ends_with_lit", P.fn("ends_with", c("s"), P.lit_utf8("€")), lambda r: S.ends_with(r["s"], "€")),
    ("month_gt_6", P.binop(">", P.fn("date_part_month", c("d")), P.lit_i32(6)), lambda r: None if r["d"] is None else S.date_part("month", r["d"]) > 6),
    ("week_eq_53", P.binop("=", P.fn("date_part_week", c("d")), P.lit_i32(53)), lambda r: None if r["d"] is None else S.date_part("week", r["d"]) == 53),
    ("char_length_gt_3", P.binop(">", P.fn("character_length", c("s")), P.lit_i32(3)), lambda r: None if r["s"] is None else len(r["s"]) > 3),
    ("btrim_eq", P.binop("=", P.fn("btrim", c("s")), P.lit_utf8("a")), lambda r: None if r["s"] is None else S.trim("btrim", r["s"]) == "a"),
    ("nullif_not_null", P.is_not_null(P.fn("nullif", c("k"), P.lit_i32(0))), lambda r: S.nullif(r["k"], 0) is not None),
    ("abs_round", P.binop(">=", P.fn("round", P.fn("abs", c("f64")), P.lit_i64(0)), P.lit_f64(2.0)),   # NaN sorts above all
     lambda r: None if r["f64"] is None else (S.round_(abs(r["f64"])) >= 2.0 or r["f64"] != r["f64"])),
    ("coalesce_ceil", P.binop("<", P.fn("coalesce", P.fn("ceil", c("f64")), P.lit_f64(-1.0)), P.lit_f64(1.0)),
     lambda r: S.coalesce(S.ceil_(r["f64"]), -1.0) < 1.0),
]


@pytest.mark.parametrize("name,pred,ref", FILTERS, ids=[f[0] for f in FILTERS])
def test_filter_predicates_keep_row_order(gpu, edge, name, pred, ref):
    rows = edge.to_pylist()
    for r in rows:
        if r["d"] is not None:
            r["d"] = (r["d"] - datetime.date(1970, 1, 1)).days
    want = [i for i, r in enumerate(rows) if ref(r) is True]
    t = edge.append_column("row", pa.array(range(edge.num_rows), pa.int32()))
    G.register(gpu, "x", t, 1)
    sch = S.SCHEMA + [P.field("row", "i32", False)]
    st = [Q.Stage(1, P.shuffle_writer(P.filter_(pred, P.scan("x", sch), projection=[len(sch) - 1]), 1))]
    ff0, vm0 = gpu.counter("fastfilter"), gpu.counter("vm")
    out = driver.run_stages(gpu, st, f"sf-filter-{name}")
    got = [] if out is None else out.column("row").to_pylist()
    assert len(want) > 0 and got == want
    assert gpu.counter("fastfilter") == ff0 and gpu.counter("vm") > vm0, "the tile VM, not the fast filter kernel, runs these"


def test_group_key_and_aggregate_argument_sf1(gpu):
    """GROUP BY date_part('month', l_shipdate), character_length(btrim(l_shipmode)) with sum(abs(l_quantity - 25)),
    sum(round(CAST(l_extendedprice AS DOUBLE))) and count(*), SF1 lineitem in 4 partitions, Partial -> FinalPartitioned"""
    cols = ["l_quantity", "l_extendedprice", "l_shipdate", "l_shipmode"]
    msf, parts = 1000, 4
    import oracle_ffi
    n = oracle_ffi.lib().oracle_tpch_table_rows(b"lineitem", msf)
    gpu.drop_table("lineitem")
    step = (n + parts - 1) // parts
    for p in range(parts):
        gpu.tpch_generate("lineitem", msf, p, p * step, min(n, (p + 1) * step), cols)
    data = pa.Table.from_batches([gpu.export_table("lineitem", p) for p in range(parts)])
    sch = [P.field("l_quantity", P.dec(15, 2), False), P.field("l_extendedprice", P.dec(15, 2), False), P.field("l_shipdate", "date32", False),
           P.field("l_shipmode", "utf8", False)]
    scan = P.scan("lineitem", sch)
    month = P.fn("date_part_month", c("l_shipdate"))
    mlen = P.fn("character_length", P.fn("btrim", c("l_shipmode")))
    absq = P.fn("abs", P.binop("-", c("l_quantity"), P.lit_dec(2500, 15, 2)))
    rnd = P.fn("round", P.cast(c("l_extendedprice"), "f64"), P.lit_i64(0))
    part = P.aggregate("Partial", [(month, "m"), (mlen, "len")], [P.agg("sum", absq, "sa"), P.agg("sum", rnd, "sr"), P.agg("count", None, "n")], scan)
    st1 = Q.Stage(1, P.shuffle_writer(part, 1, [c(0), c(1)], 4))
    fields = json.loads(engine.plan_typed_json(st1.json("j")))["input"]["schema"]
    fin = P.aggregate("FinalPartitioned", [(c(0), "m"), (c(1), "len")],
                      [P.agg("sum", c(2), "sa", input_type=P.dec(16, 2)), P.agg("sum", c(3), "sr", input_type="f64"), P.agg("count", c(4), "n")],
                      P.shuffle_reader(1, fields))
    st = [st1, Q.Stage(2, P.shuffle_writer(fin, 2))]
    fused0, gb0 = gpu.counter("fused"), gpu.counter("groupby")
    got = driver.run_stages(gpu, st, "sf-group")
    assert gpu.counter("fused") == fused0 and gpu.counter("groupby") == gb0, "the matchers refuse programs holding the new ops"
    # independent: pyarrow's month / utf8_length / utf8_trim and Python's Decimal and float arithmetic
    m = pc.month(data.column("l_shipdate")).to_pylist()
    ln = pc.utf8_length(pc.utf8_trim(data.column("l_shipmode"), " ")).to_pylist()
    q = data.column("l_quantity").to_pylist()
    ep = data.column("l_extendedprice").to_pylist()
    want = {}
    for i in range(data.num_rows):
        k = (m[i], ln[i])
        a = want.setdefault(k, [Decimal(0), [], 0])
        a[0] += abs(q[i] - Decimal("25.00"))
        a[1].append(S.round_(float(ep[i])))
        a[2] += 1
    g = {(r["m"], r["len"]): r for r in got.to_pylist()}
    assert set(g) == set(want) and len(want) > 12
    for k, (sa, sr, cnt) in want.items():
        assert g[k]["sa"] == sa and g[k]["n"] == cnt
        # each rounded value is an integer and every partial sum stays below 2^53: exact in binary64, in any order
        assert g[k]["sr"] == float(sum(Decimal(v) for v in sr))


with open(os.path.join(HERE, "golden", "scalar_fn_proto_plans.json")) as _fh:
    PROTO_CASES = json.load(_fh)["cases"]


class _FromProto:
    def __init__(self, eng, cases):
        self._e, self._c = eng, cases

    def __getattr__(self, name):
        return getattr(self._e, name)

    def create_query_stage_exec(self, job_id, stage_id, plan_json):
        return self._e.create_query_stage_exec_proto(job_id, stage_id, base64.b64decode(self._c[stage_id]["proto_b64"]))


def _fixture_table():
    t = S.edge_table(2500, seed=11)
    return pa.table({"k": t.column("k"), "x": t.column("i64").cast(pa.int64()), "f": t.column("f64"), "d": t.column("d"),
                     "s": t.column("s"), "t": t.column("p")})


def test_every_fixture_runs_from_its_bytes(gpu):
    """each plan decoded from its protobuf bytes gives, on the device, what its source IR gives (the functions' results
    themselves are checked against the restatement by the tests above)"""
    G.register(gpu, "t", _fixture_table(), 2)
    groups = {}
    for case in PROTO_CASES:
        if not case["refused"]:
            groups.setdefault(case["name"].rsplit("/", 1)[0], {})[int(case["name"].rsplit("stage", 1)[1])] = case
    assert len(groups) >= 3 * 25
    for j, (name, cases) in enumerate(sorted(groups.items())):
        stages = [Q.Stage(i, json.loads(cases[i]["ir"])) for i in sorted(cases)]
        got = driver.run_stages(_FromProto(gpu, cases), stages, f"sf-proto-{j}")
        want = driver.run_stages(gpu, stages, f"sf-ir-{j}")
        if want is None:
            assert got is None or got.num_rows == 0, name
            continue
        ordered = "/projection" in name or "/filter" in name
        a = got.to_pylist() if ordered else sorted(got.to_pylist(), key=repr)
        b = want.to_pylist() if ordered else sorted(want.to_pylist(), key=repr)
        assert S.same_values([repr(r) for r in a], [repr(r) for r in b]), name


def test_nullif_and_coalesce_over_timestamps(gpu):
    ns = [None, 0, 1_600_000_000_123_456_789, -5, 7, None, 7] * 500
    other = [1, None, 1_600_000_000_123_456_789, -5, 8, None, 0] * 500
    t = pa.table({"a": pa.array(ns, pa.timestamp("ns")), "b": pa.array(other, pa.timestamp("ns"))})
    G.register(gpu, "tsx", t, 2)
    sch = [P.field("a", "ts", True), P.field("b", "ts", True)]
    st = _project([("n", P.fn("nullif", c("a"), c("b"))), ("c", P.fn("coalesce", c("a"), c("b")))], "tsx", sch)
    out = driver.run_stages(gpu, st, "sf-ts")
    assert out.column("n").cast(pa.int64()).to_pylist() == [S.nullif(x, y) for x, y in zip(ns, other)]
    assert out.column("c").cast(pa.int64()).to_pylist() == [S.coalesce(x, y) for x, y in zip(ns, other)]


def test_abs_overflow_is_an_execution_error(gpu):
    for typ, pat in (("i64", pa.int64()), ("i32", pa.int32()), ("i8", pa.int8())):
        t = pa.table({"v": pa.array([1, None, S.INT_MIN[typ], 5] * 700, pat)})
        G.register(gpu, "ov", t, 1)
        st = _project([("a", P.fn("abs", c("v")))], "ov", [P.field("v", typ, True)])
        with pytest.raises(engine.B200Error) as ei:
            driver.run_stages(gpu, st, f"sf-ovf-{typ}")
        assert ei.value.code == EXECUTION, str(ei.value)
        # the engine runs the next plan correctly
        t2 = pa.table({"v": pa.array([1, None, S.INT_MIN[typ] + 1, -5], pat)})
        G.register(gpu, "ov", t2, 1)
        out = driver.run_stages(gpu, st, f"sf-ovf-next-{typ}")
        assert out.column("a").to_pylist() == [1, None, -(S.INT_MIN[typ] + 1), 5]


@pytest.mark.parametrize("e,culprit", [(P.fn("round", c("f64"), c("i64")), "digit count"), (P.fn("btrim", c("s"), c("p")), "character set")])
def test_non_literal_operands_are_refused(gpu, edge, e, culprit):
    G.register(gpu, "x", edge, 1)
    with pytest.raises(engine.B200Error) as ei:
        driver.run_stages(gpu, _project([("r", e)]), "sf-nonlit")
    assert ei.value.code == UNSUPPORTED and culprit in str(ei.value), str(ei.value)
