"""first_value / last_value on the device against the plain-Python restatement (first_last_cases.py), bit-exact: every
value type and every ordering key type (nullable keys, DESC, NULLS FIRST / LAST, multi-key orderings, Utf8 keys longer
than 14 bytes that share prefixes, Decimal128 beyond 64 bits, floats with NaN and -0.0), all-tied groups, IGNORE NULLS
with all-NULL groups; the five modes, Partial -> shuffle -> Final over several input partitions; the register sink
(<= 4 groups) and the global sink, told apart by the kernel timer families; other aggregates in the same node; the
DISTINCT ON shape sharing one chain; plans decoded from protobuf bytes; a TPC-H-shaped query over generated lineitem."""
import base64
import datetime
import decimal
import json
import math
import struct

import numpy as np
import pyarrow as pa
import pytest

import golden_data as G
from ballista_b200 import driver, engine
from ballista_b200 import plan as P
from first_last_cases import final_merge, grouped, partial_only, partial_state, stages

pytestmark = pytest.mark.gpu
c = P.col

COLS = [("k4", "i32", pa.int32(), False), ("kg", "i64", pa.int64(), False), ("seq", "i64", pa.int64(), False),
        ("i8", "i8", pa.int8(), True), ("i16", "i16", pa.int16(), True), ("i32", "i32", pa.int32(), True), ("i64", "i64", pa.int64(), True),
        ("u8", "u8", pa.uint8(), True), ("u16", "u16", pa.uint16(), True), ("u32", "u32", pa.uint32(), True), ("u64", "u64", pa.uint64(), True),
        ("f32", "f32", pa.float32(), True), ("f64", "f64", pa.float64(), True), ("b", "bool", pa.bool_(), True),
        ("dec", P.dec(38, 0), pa.decimal128(38, 0), True), ("dt", "date32", pa.date32(), True), ("ts", "ts", pa.timestamp("ns"), True),
        ("s", "utf8", pa.string(), True), ("xn", "i32", pa.int32(), True)]
NAMES = [n for n, _, _, _ in COLS]
IDX = {n: i for i, n in enumerate(NAMES)}
SCHEMA = [P.field(n, t, nl) for n, t, _, nl in COLS]
TYPES = {n: t for n, t, _, _ in COLS}
VALUE_COLS = ["i8", "i16", "i32", "i64", "u8", "u16", "u32", "u64", "f32", "f64", "b", "dec", "dt", "ts", "s"]
PREFIX = "a shared prefix longer than fourteen bytes/"


def make_rows(n, seed, kg_size=5):
    """k4: 4 groups, kg: groups of kg_size rows; small value domains so that ties are common; xn: NULL in every row of
    group k4 = 3 (an all-NULL group for IGNORE NULLS) and in some others"""
    rng = np.random.default_rng(seed)
    floats = [0.0, -0.0, 1.5, -1.5, float("nan"), float("inf"), -float("inf"), struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000001))[0]]
    strs = ["", "a", "ab", PREFIX, PREFIX + "x", PREFIX + "xy", PREFIX + "x" * 20, PREFIX + "x" * 20 + "z", "b" * 30]
    rows = []
    for i in range(n):
        nul = lambda p=0.12: rng.random() < p  # noqa: E731
        k4 = i % 4
        r = [k4, i // kg_size, i,
             None if nul() else int(rng.integers(-3, 4)), None if nul() else int(rng.integers(-32768, 32768)),
             None if nul() else int(rng.integers(-5, 5)), None if nul() else int(rng.integers(-(1 << 62), 1 << 62)) * (1 if i % 3 else -1),
             None if nul() else int(rng.integers(0, 4)), None if nul() else int(rng.integers(0, 65536)),
             None if nul() else int(rng.integers(0, 6)), None if nul() else (int(rng.integers(0, 3)) << 62) | int(rng.integers(0, 3)),
             None if nul() else float(np.float32(floats[int(rng.integers(0, len(floats)))])) if rng.random() < 0.7 else float(np.float32(rng.normal())),
             None if nul() else floats[int(rng.integers(0, len(floats)))],
             None if nul() else bool(rng.integers(0, 2)),
             None if nul() else decimal.Decimal(int(rng.integers(-2, 3)) * (1 << 70) + int(rng.integers(-3, 3))),
             None if nul() else datetime.date(2020, 1, 1) + datetime.timedelta(days=int(rng.integers(-3, 3))),
             None if nul() else int(rng.integers(-3, 3)) * 1_000_000_000_000,
             None if nul() else strs[int(rng.integers(0, len(strs)))],
             None if (k4 == 3 or nul(0.3)) else int(rng.integers(0, 1000))]
        rows.append(r)
    return rows


def to_batch(rows):
    cols = list(zip(*rows)) if rows else [[] for _ in NAMES]
    return pa.record_batch([pa.array(list(v), t) for v, (_, _, t, _) in zip(cols, COLS)], names=NAMES)


def ref_rows(rows):
    """the rows as pyarrow gives them back, so that the restatement and the result hold the same Python types"""
    if not rows:
        return []
    d = to_batch(rows).to_pydict()
    return [tuple(d[n][i] for n in NAMES) for i in range(len(rows))]


def register(gpu, name, rows, parts):
    gpu.drop_table(name)
    step = max((len(rows) + parts - 1) // parts, 1)
    for p in range(parts):
        gpu.register_batch(name, p, to_batch(rows[p * step:(p + 1) * step]))


def same(v, w):
    if isinstance(w, float) and isinstance(v, float):
        return struct.pack("<d", v) == struct.pack("<d", w)
    return v == w and type(v) is type(w)


def check(got, key_names, want):
    assert got.num_rows == len(want), (got.num_rows, len(want))
    for r in got.to_pylist():
        g = tuple(r[k] for k in key_names)
        assert g in want, g
        for nm, w in want[g].items():
            assert same(r[nm], w), (g, nm, r[nm], w)


def agg_spec(fn, x, ob, ign=False, name=None):
    """(plan tuple, restatement tuple) of one aggregate; ob: [(column, asc, nulls_first)]"""
    name = name or f"{fn}_{x}_" + "_".join(f"{k}{int(a)}{int(n)}" for k, a, n in ob) + ("_ign" if ign else "")
    return ((fn, c(x), TYPES[x], [(c(k), a, n) for k, a, n in ob], ign, name),
            (fn, IDX[x], [(IDX[k], a, n) for k, a, n in ob], ign, name))


def run(gpu, rows, aggs, key, mode, job, parts=3):
    register(gpu, job, rows, parts if mode == "Partial" else 1)
    keys = [(c(key), key)] if key else []
    kf = [P.field(key, TYPES[key], False)] if key else []
    plan_aggs = [a for a, _ in aggs]
    want = grouped(ref_rows(rows), [IDX[key]] if key else [], [b for _, b in aggs])
    got = driver.run_stages(gpu, stages(P.scan(job, SCHEMA), plan_aggs, keys, kf, mode), job)
    check(got, [key] if key else [], want)
    return got


@pytest.fixture()
def timed(gpu):
    gpu.set_config("b200.metrics.kernel_timing", "on")
    yield gpu
    gpu.set_config("b200.metrics.kernel_timing", "off")


def value_sets():
    """each value type under a few orderings of each key type: single keys ASC / DESC with either NULL placement, and
    multi-key orderings; at most four aggregates per node"""
    out = []
    for i, x in enumerate(VALUE_COLS):
        k1 = VALUE_COLS[(i + 3) % len(VALUE_COLS)]
        k2 = VALUE_COLS[(i + 7) % len(VALUE_COLS)]
        out.append([agg_spec("first_value", x, [(k1, True, False)]), agg_spec("last_value", x, [(k1, False, True)]),
                    agg_spec("first_value", x, [(k2, False, False), (k1, True, True)]), agg_spec("last_value", x, [])])
    return out


@pytest.mark.parametrize("mode", ["Single", "SinglePartitioned", "Partial"])
@pytest.mark.parametrize("key,sink", [("k4", "pipeline_agg_reg"), ("kg", "pipeline_agg_global"), (None, "pipeline_agg_reg")])
def test_types_orderings_modes_and_sinks(timed, mode, key, sink):
    gpu = timed
    rows = make_rows(3001, 7)
    for j, aggs in enumerate(value_sets()):
        gpu.kernel_stats(reset=True)
        run(gpu, rows, aggs, key, mode, f"fl-{mode}-{key}-{j}")
        ks = gpu.kernel_stats()
        assert "pipeline_fused_agg" not in ks and "groupby_hash_agg" not in ks, ks
        assert "pipeline_agg_first_last" in ks, ks
        if mode != "Partial":
            assert sink in ks, ks
            if sink == "pipeline_agg_reg":
                assert "pipeline_agg_global" not in ks, ks


@pytest.mark.parametrize("n", [0, 1, 2, 1025, (1 << 18) + 3])
def test_row_counts(gpu, n):
    rows = make_rows(n, n + 1, kg_size=7)
    aggs = [agg_spec("first_value", "s", [("f64", True, False), ("seq", False, True)]), agg_spec("last_value", "dec", [("s", True, True)]),
            agg_spec("last_value", "xn", [("i8", False, False)], ign=True), agg_spec("first_value", "f32", [])]
    for key in ("k4", "kg", None):
        for mode in ("Single", "Partial"):
            run(gpu, rows, aggs, key, mode, f"flr-{n}-{key}-{mode}")


def test_ties_ignore_nulls_and_empty_groups(gpu):
    """every row of a group tied on the ordering (the earliest wins first_value, the latest last_value); IGNORE NULLS over
    a group whose values are all NULL, and without IGNORE NULLS a NULL value can win"""
    rows = make_rows(2000, 3)
    for r in rows:
        r[IDX["i8"]] = 1 if r[0] != 2 else None
    aggs = [agg_spec("first_value", "seq", [("i8", True, False)]), agg_spec("last_value", "seq", [("i8", False, True)]),
            agg_spec("first_value", "xn", [("i8", True, False)], ign=True), agg_spec("last_value", "xn", [("u8", True, True)])]
    for mode in ("Single", "Partial"):
        got = run(gpu, rows, aggs, "k4", mode, f"flt-{mode}")
        for r in got.to_pylist():
            assert r[aggs[2][0][5]] is None if r["k4"] == 3 else r[aggs[2][0][5]] is not None
    # Partial over 3 partitions: the restatement of the Final merge over the states in partition order is the same thing
    states = []
    for p in range(3):
        part = ref_rows(rows[p * 667:(p + 1) * 667])
        states.append(partial_state("last_value", [r for r in part if r[0] == 1], lambda r: r[IDX["seq"]], [lambda r: r[IDX["i8"]]], [(False, True)]))
    assert final_merge("last_value", states, [(False, True)]) == max(r[IDX["seq"]] for r in rows if r[0] == 1)


def test_partial_states(gpu):
    rows = make_rows(3001, 11)
    rr = ref_rows(rows)
    aggs = [agg_spec("first_value", "s", [("f64", True, False), ("dec", False, True)], name="a"),
            agg_spec("last_value", "f32", [("s", True, True)], ign=True, name="b")]
    register(gpu, "flp", rows, 1)
    got = driver.run_stages(gpu, partial_only(P.scan("flp", SCHEMA), [a for a, _ in aggs], [(c("k4"), "k4")]), "flp")
    assert got.schema.names == ["k4", "a[first_value]", "f64@12", "dec@14", "is_set", "b[last_value]", "s@17", "is_set"]
    cols = got.to_pydict()
    for i, k in enumerate(cols["k4"]):
        grp = [r for r in rr if r[0] == k]
        wa = partial_state("first_value", grp, lambda r: r[IDX["s"]], [lambda r: r[IDX["f64"]], lambda r: r[IDX["dec"]]], [(True, False), (False, True)])
        wb = partial_state("last_value", [r for r in grp if r[IDX["f32"]] is not None], lambda r: r[IDX["f32"]], [lambda r: r[IDX["s"]]], [(True, True)])
        row = [got.column(j)[i].as_py() for j in range(got.num_columns)]
        assert all(same(v, w) for v, w in zip(row[1:5], wa)), (row, wa)
        assert all(same(v, w) for v, w in zip(row[5:8], wb)), (row, wb)


def test_other_aggregates_stay_exact(gpu):
    """SUM / COUNT / VAR next to first / last in one AggregateExec"""
    rows = make_rows(4001, 5)
    rr = ref_rows(rows)
    fl = [agg_spec("last_value", "s", [("ts", True, False)])]
    register(gpu, "flo", rows, 1)
    for mode in ("Single", "SinglePartitioned"):
        aggs = [a for a, _ in fl]
        pagg = [P.agg("sum", c("i32"), "s32"), P.agg("count", c("i8"), "c8"), P.agg("var_pop", c("i16"), "v16")]
        st = stages(P.scan("flo", SCHEMA), aggs, [(c("k4"), "k4")], [P.field("k4", "i32", False)], mode)
        node = st[0].plan["input"]
        node["aggr"] = pagg + node["aggr"]
        got = driver.run_stages(gpu, st, f"flo-{mode}").to_pylist()
        want = grouped(rr, [0], [b for _, b in fl])
        assert len(got) == 4
        for r in got:
            grp = [q for q in rr if q[0] == r["k4"]]
            assert r["s32"] == sum(q[IDX["i32"]] for q in grp if q[IDX["i32"]] is not None)
            assert r["c8"] == sum(1 for q in grp if q[IDX["i8"]] is not None)
            v = [q[IDX["i16"]] for q in grp if q[IDX["i16"]] is not None]
            m = sum(v) / len(v)
            assert math.isclose(r["v16"], sum((a - m) ** 2 for a in v) / len(v), rel_tol=1e-12)
            assert same(r[fl[0][0][5]], want[(r["k4"],)][fl[0][0][5]])


def test_distinct_on_shares_one_chain(gpu):
    """SELECT DISTINCT ON (kg) i32, s, f64 ... ORDER BY kg, seq DESC: one first_value per column, one ordering, one chain of
    passes over the rows (two non-NULL Int64 keys: one word each, the position word and the capture)"""
    rows = make_rows(5000, 13)
    ob = [("kg", True, False), ("seq", False, True)]
    aggs = [agg_spec("first_value", x, ob) for x in ("i32", "s", "f64")]
    for mode in ("Single", "Partial"):  # Partial: the Final merges three states per group under one chain too
        before = gpu.counter("first_last_passes")
        run(gpu, rows, aggs, "kg", mode, f"fld-{mode}")
        # kg, seq, position, capture: one chain.  Partial -> FinalPartitioned: that in each of the 3 Partial tasks; each of
        # the 3 Final tasks reads every aggregate's own state columns, so it runs one chain per aggregate, of the state's kg
        # and seq (nullable: a NULL-rank word each), position and capture
        assert gpu.counter("first_last_passes") - before == (4 if mode == "Single" else 3 * 4 + 3 * 3 * 6), mode


def test_long_string_keys(gpu):
    """Utf8 ordering keys of hundreds of bytes that differ only near their ends: the pass count follows the longest key"""
    rows = make_rows(600, 17)
    rng = np.random.default_rng(2)
    for r in rows:
        r[IDX["s"]] = None if rng.random() < 0.1 else "p" * int(rng.integers(100, 300)) + chr(97 + int(rng.integers(0, 3)))
    aggs = [agg_spec("first_value", "seq", [("s", True, False)]), agg_spec("last_value", "seq", [("s", False, False)])]
    for mode in ("Single", "Partial"):
        run(gpu, rows, aggs, "k4", mode, f"fls-{mode}")


def test_lineitem_latest_shipmode(gpu):
    """SELECT l_orderkey, last_value(l_shipmode ORDER BY l_shipdate, l_linenumber) ... GROUP BY l_orderkey over generated
    lineitem (SF 0.01, three partitions, Partial -> FinalPartitioned), against the restatement over the same rows"""
    cols = ["l_orderkey", "l_linenumber", "l_shipdate", "l_shipmode"]
    gpu.drop_table("lineitem")
    n = 60000
    for p in range(3):
        gpu.tpch_generate("lineitem", 10, p, p * n // 3, (p + 1) * n // 3, cols)
    t = pa.Table.from_batches([gpu.export_table("lineitem", p) for p in range(3)])
    sch = [P.field(f.name, {pa.int64(): "i64", pa.int32(): "i32", pa.date32(): "date32"}.get(f.type, "utf8"), f.nullable) for f in t.schema]
    ob = [(c("l_shipdate"), True, False), (c("l_linenumber"), True, False)]
    aggs = [("last_value", c("l_shipmode"), "utf8", ob, False, "m")]
    kt = next(f["type"] for f in sch if f["name"] == "l_orderkey")
    got = driver.run_stages(gpu, stages(P.scan("lineitem", sch), aggs, [(c("l_orderkey"), "l_orderkey")], [P.field("l_orderkey", kt, False)], "Partial"), "fll")
    d = t.to_pydict()
    best = {}
    for k, ln, sd, m in zip(d["l_orderkey"], d["l_linenumber"], d["l_shipdate"], d["l_shipmode"]):
        if k not in best or (sd, ln) >= best[k][0]:
            best[k] = ((sd, ln), m)
    res = {r["l_orderkey"]: r["m"] for r in got.to_pylist()}
    assert res == {k: v[1] for k, v in best.items()}
    gpu.drop_table("lineitem")


def test_protobuf_plans_run_like_their_ir(gpu):
    """every fixture stage pair decoded from protobuf bytes computes what its IR computes, and both match the restatement"""
    with open(G.__file__.replace("golden_data.py", "golden/first_last_proto_plans.json")) as fh:
        cases = [x for x in json.load(fh)["cases"] if "ir" in x]
    rng = np.random.default_rng(4)
    n = 3000
    b = pa.record_batch([pa.array([int(v) for v in rng.integers(0, 6, n)], pa.int32()),
                         pa.array([None if rng.random() < 0.2 else int(v) for v in rng.integers(-9, 9, n)], pa.int64()),
                         pa.array([None if rng.random() < 0.1 else float(v) for v in rng.integers(0, 5, n)], pa.float64()),
                         pa.array([None if rng.random() < 0.1 else PREFIX + str(v) for v in rng.integers(0, 4, n)], pa.string())],
                        names=["k", "x", "o", "s"])
    gpu.drop_table("t")
    for p in range(3):
        gpu.register_batch("t", p, b.slice(p * n // 3, n // 3))
    by_plan = {}
    for cs in cases:
        by_plan.setdefault(cs["name"].rsplit("/", 1)[0], []).append(cs)
    ran = 0
    for name, sts in by_plan.items():
        if len(sts) == 1:
            continue  # a Single aggregate over three partitions aggregates each on its own: covered by the IR tests
        scalar = "scalar" in name
        decoded = [P.Stage(i + 1, json.loads(engine.plan_proto_to_json(base64.b64decode(s["proto_b64"]), "job")), 1 if scalar and i else None)
                   for i, s in enumerate(sts)]
        ir = [P.Stage(i + 1, json.loads(s["ir"]), 1 if scalar and i else None) for i, s in enumerate(sts)]
        job = name.replace("/", "-")
        got = sorted(driver.run_stages(gpu, decoded, job + "-pb").to_pylist(), key=lambda r: r.get("k", 0))
        want = sorted(driver.run_stages(gpu, ir, job + "-ir").to_pylist(), key=lambda r: r.get("k", 0))
        assert len(got) == len(want) > 0, name
        for g, w in zip(got, want):
            assert all(same(g[k], w[k]) for k in w), (name, g, w)
        ran += 1
    assert ran >= 4
