"""ROLLUP / CUBE / GROUPING SETS on the device against the UNION ALL form on the CPU oracle (grouping_set_cases.py): keys of
every type with real NULLs, every accumulator kind of the global sink, Single and Partial -> hash shuffle ->
FinalPartitioned over 1, 2 and 4 input partitions, a table that outgrows its first capacity class, TPC-H q1 with
ROLLUP(l_returnflag, l_linestatus) through three stages, GROUPING() in its bitwise form, the bitwise operators at every
integer width, the committed protobuf fixtures, and the engine after every refused plan."""
import base64
import json
import os

import numpy as np
import pyarrow as pa
import pytest

import grouping_set_cases as GC
from ballista_b200 import driver, engine, tpch
from ballista_b200 import plan as P
from util import assert_tables_equal

pytestmark = pytest.mark.gpu
c = P.col
RTOL = 1e-12
FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "grouping_set_proto_plans.json")

KEY_SETS = [
    # (keys, sets)
    (["ks"], P.rollup_sets(1)),
    (["ks", "ki"], P.rollup_sets(2)),
    (["kd", "kt", "kf"], P.rollup_sets(3)),
    (["ki", "kd", "ks"], P.cube_sets(3)),
    (["kb", "kf"], [[False, False]]),                       # GROUPING SETS ((kb, kf)): one all-false set, still with the id
    (["kt", "ks"], [[False, True], [True, False], [True, True]]),  # GROUPING SETS ((kt), (ks), ())
]


def _keys(names):
    return [(c(n), n) for n in names]


@pytest.fixture()
def timed(gpu):
    gpu.set_config("b200.metrics.kernel_timing", "on")
    gpu.kernel_stats(reset=True)
    yield gpu
    gpu.set_config("b200.metrics.kernel_timing", "off")


@pytest.mark.parametrize("case", range(len(KEY_SETS)))
def test_single_mode_matches_union_all(timed, oracle, case):
    gpu = timed
    names, sets = KEY_SETS[case]
    t = GC.make_table(3000, seed=case)
    GC.register(gpu, "gs", t, 1)
    GC.register(oracle, "gs", t, 1)
    scan = P.scan("gs", GC.SCHEMA)
    fused0, gb0 = gpu.counter("fused"), gpu.counter("groupby")
    got = driver.run_stages(gpu, GC.single_stages(scan, _keys(names), GC.AGGS, sets), f"gs-single-{case}")
    want = GC.expected(oracle, scan, _keys(names), GC.AGGS, sets, f"gs-single-{case}")
    assert_tables_equal(got, want, f64_rtol=RTOL)
    ks = gpu.kernel_stats()
    assert ks.get("pipeline_agg_gsets", {}).get("launches", 0) >= 1, ks.keys()
    assert gpu.counter("fused") == fused0 and gpu.counter("groupby") == gb0


@pytest.mark.parametrize("parts", [1, 2, 4])
@pytest.mark.parametrize("case", range(len(KEY_SETS)))
def test_partial_final_matches_union_all(gpu, oracle, case, parts):
    names, sets = KEY_SETS[case]
    t = GC.make_table(2000, seed=100 + case)
    GC.register(gpu, "gs", t, parts)
    GC.register(oracle, "gs", t, 1)
    scan = P.scan("gs", GC.SCHEMA)
    # the FinalPartitioned merge of all twelve aggregates would take more than the 16 table accumulators one holds
    aggs = GC.AGGS[:2] + GC.AGGS[4:5] + GC.AGGS[6:8] + GC.AGGS[9:10]
    got = driver.run_stages(gpu, GC.two_stages(scan, _keys(names), aggs, sets), f"gs-pf-{case}-{parts}")
    want = GC.expected(oracle, scan, _keys(names), aggs, sets, f"gs-pf-{case}-{parts}")
    assert_tables_equal(got, want, f64_rtol=RTOL)


@pytest.mark.parametrize("case", range(len(KEY_SETS)))
def test_partial_states_match_union_all(gpu, oracle, case):
    """the Partial node's own output: keys, __grouping_id and the state columns (one input partition: one row per group)"""
    names, sets = KEY_SETS[case]
    t = GC.make_table(2500, seed=200 + case)
    GC.register(gpu, "gs", t, 1)
    GC.register(oracle, "gs", t, 1)
    scan = P.scan("gs", GC.SCHEMA)
    aggs = GC.AGGS[:2] + GC.AGGS[3:6] + GC.AGGS[6:8] + GC.AGGS[9:10]
    st = [P.Stage(1, P.shuffle_writer(P.aggregate("Partial", _keys(names), aggs, scan, grouping_sets=sets), 1))]
    got = driver.run_stages(gpu, st, f"gs-partial-{case}")
    want = GC.expected(oracle, scan, _keys(names), aggs, sets, f"gs-partial-{case}", mode="Partial")
    assert_tables_equal(got, want, f64_rtol=RTOL)


def test_null_key_next_to_its_rolled_up_twin(gpu):
    t = pa.table({"k": pa.array([1, None, None, 2], pa.int32()), "x": pa.array([10, 20, 30, 40], pa.int64())})
    GC.register(gpu, "nk", t, 1)
    scan = P.scan("nk", [P.field("k", "i32", True), P.field("x", "i64")])
    got = driver.run_stages(gpu, GC.single_stages(scan, [(c("k"), "k")], [P.agg("sum", c("x"), "s"), P.agg("count", None, "n")],
                                                  P.rollup_sets(1)), "nk")
    rows = sorted(zip(*[got.column(i).to_pylist() for i in range(4)]), key=lambda r: (r[1], r[0] is None, r[0] or 0))
    assert rows == [(1, 0, 10, 1), (2, 0, 40, 1), (None, 0, 50, 2), (None, 1, 100, 4)]
    assert got.schema.field("__grouping_id").type == pa.uint8()


def test_empty_input_gives_no_rows(gpu):
    t = GC.make_table(0, seed=1)
    GC.register(gpu, "gse", t, 2)
    scan = P.scan("gse", GC.SCHEMA)
    for sets in (P.rollup_sets(2), [[True, True]]):
        got = driver.run_stages(gpu, GC.two_stages(scan, _keys(["ks", "ki"]), GC.AGGS[:4], sets), "gse")
        assert got.num_rows == 0


def test_table_outgrows_its_first_class(timed):
    gpu = timed
    # CUBE of two unique keys: 3 n + 1 groups, more than the first table (sized for one group per input row) holds
    n = 1_000_000
    k = np.arange(n, dtype=np.int64) * 7919 % (1 << 40)
    x = np.arange(n, dtype=np.int64) % 1000 - 500
    GC.register(gpu, "big", pa.table({"k": k, "k2": -k, "x": x}), 1)
    scan = P.scan("big", [P.field("k", "i64"), P.field("k2", "i64"), P.field("x", "i64")])
    got = driver.run_stages(gpu, GC.single_stages(scan, [(c("k"), "k"), (c("k2"), "k2")],
                                                  [P.agg("sum", c("x"), "s"), P.agg("count", None, "n"), P.agg("min", c("x"), "m")],
                                                  P.cube_sets(2)), "big")
    assert got.num_rows == 3 * n + 1
    gid = got.column("__grouping_id").to_numpy()
    for g, key in ((0, "k"), (1, "k"), (2, "k2")):
        part = got.filter(pa.array(gid == g))
        order = np.argsort(part.column(key).to_numpy())
        src = np.argsort(k if key == "k" else -k)
        assert np.array_equal(part.column(key).to_numpy()[order], (k if key == "k" else -k)[src])
        assert np.array_equal(part.column("s").to_numpy()[order], x[src])
        assert np.array_equal(part.column("m").to_numpy()[order], x[src])
    total = got.filter(pa.array(gid == 3))
    assert total.column("k").to_pylist() == [None] and total.column("k2").to_pylist() == [None]
    assert total.column("s").to_pylist() == [int(x.sum())] and total.column("n").to_pylist() == [n]
    assert total.column("m").to_pylist() == [int(x.min())]
    assert gpu.kernel_stats()["pipeline_agg_gsets"]["launches"] >= 2  # the first table overflowed and the run grew it


def _q1_rollup_stages(n_out=4):
    """q1's scan, filter and projection under ROLLUP(l_returnflag, l_linestatus), Partial -> FinalPartitioned -> merge"""
    q1 = tpch.q1(n_out)
    partial = q1[0].plan["input"]
    partial = dict(partial, grouping_sets=P.rollup_sets(2))
    keys = [P.sort_key(c(0)), P.sort_key(c(1)), P.sort_key(c(2))]
    t = GC.typed(partial)
    st1 = P.Stage(1, P.shuffle_writer(partial, 1, [c(0), c(1), c(2)], n_out))
    faggs = [P.agg(a["fn"], None, a["name"], a["input_type"] if a["fn"] == "avg" else None) for a in t["aggr"]]
    final = P.aggregate("FinalPartitioned", [(c(i), t["schema"][i]["name"]) for i in range(3)], faggs, P.shuffle_reader(1, t["schema"]))
    ft = GC.typed(final)
    st2 = P.Stage(2, P.shuffle_writer(P.sort(keys, final, preserve_partitioning=True), 2))
    st3 = P.Stage(3, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(2, ft["schema"])), 3), n_tasks=1)
    return [st1, st2, st3], partial


def test_tpch_q1_rollup_three_stages(gpu, oracle):
    msf = 20
    n = engine.GpuExecutionEngine.tpch_table_rows("lineitem", msf)
    gpu.drop_table("lineitem")
    gpu.tpch_generate("lineitem", msf, 0, 0, n // 2, tpch.Q1_COLUMNS)
    gpu.tpch_generate("lineitem", msf, 1, n // 2, n, tpch.Q1_COLUMNS)
    oracle.drop_table("lineitem")
    oracle.tpch_generate("lineitem", msf, 0, 0, n, tpch.Q1_COLUMNS)
    stages, partial = _q1_rollup_stages()
    fused0 = gpu.counter("fused")
    got = driver.run_stages(gpu, stages, "q1r")
    assert gpu.counter("fused") == fused0
    assert got.num_rows == 4 + 3 + 1  # (flag, status), (flag), ()
    keys = [(k["expr"], k["name"]) for k in partial["group_by"]]
    want = GC.expected(oracle, partial["input"], keys, partial["aggr"], P.rollup_sets(2), "q1r")
    assert_tables_equal(got, want)


def test_grouping_function_projection(gpu):
    """GROUPING(ks) and GROUPING(ks, ki) as DataFusion's analyzer leaves them: CAST of & / >> over __grouping_id"""
    t = GC.make_table(1500, seed=7)
    GC.register(gpu, "gs", t, 2)
    scan = P.scan("gs", GC.SCHEMA)
    aggs = [P.agg("sum", c("q"), "sum_q"), P.agg("count", None, "cnt")]
    st = GC.two_stages(scan, _keys(["ks", "ki"]), aggs, P.cube_sets(2))
    final = st[1].plan["input"]
    u8 = lambda v: {"lit": {"t": "u8", "v": v}}  # noqa: E731
    g_a = P.cast(P.binop("&", P.binop(">>", c(2), u8(1)), u8(1)), "i32")
    g_ab = P.cast(P.binop("&", c(2), u8(3)), "i32")
    proj = P.project([(c(0), "ks"), (c(1), "ki"), (c(2), "__grouping_id"), (g_a, "grouping(ks)"), (g_ab, "grouping(ks, ki)"),
                      (c(3), "sum_q")], final)
    got = driver.run_stages(gpu, [st[0], P.Stage(2, P.shuffle_writer(proj, 2))], "gs-grouping")
    ids = got.column("__grouping_id").to_pylist()
    assert sorted(set(ids)) == [0, 1, 2, 3]
    assert got.column("grouping(ks)").to_pylist() == [(i >> 1) & 1 for i in ids]
    assert got.column("grouping(ks, ki)").to_pylist() == [i & 3 for i in ids]
    assert got.schema.field("grouping(ks)").type == pa.int32()


WIDTHS = [("i8", pa.int8(), 8, True), ("i16", pa.int16(), 16, True), ("i32", pa.int32(), 32, True), ("i64", pa.int64(), 64, True),
          ("u8", pa.uint8(), 8, False), ("u16", pa.uint16(), 16, False), ("u32", pa.uint32(), 32, False), ("u64", pa.uint64(), 64, False)]


def rust_bitwise(op, a, b, bits, signed):
    """Rust's & | ^ wrapping_shl wrapping_shr on the two's complement images, read back in the type"""
    m = (1 << bits) - 1
    ua, ub = a & m, b & m
    if op == "&":
        r = ua & ub
    elif op == "|":
        r = ua | ub
    elif op == "^":
        r = ua ^ ub
    elif op == "<<":
        r = (ua << (ub & (bits - 1))) & m
    else:
        sh = ub & (bits - 1)
        r = ((a >> sh) if signed else (ua >> sh)) & m
    return r - (1 << bits) if signed and r >> (bits - 1) else r


@pytest.mark.parametrize("w", WIDTHS, ids=[w[0] for w in WIDTHS])
def test_bitwise_operators_every_width(gpu, w):
    ir, at, bits, signed = w
    rng = np.random.default_rng(bits + signed)
    lo, hi = (-(1 << (bits - 1)), (1 << (bits - 1)) - 1) if signed else (0, (1 << bits) - 1)
    n = 600
    a = [int(x) for x in rng.integers(lo, hi, n, endpoint=True, dtype=np.int64 if signed or bits < 64 else np.uint64)]
    b = [int(x) for x in rng.integers(lo, hi, n, endpoint=True, dtype=np.int64 if signed or bits < 64 else np.uint64)]
    a[:6] = [lo, hi, 0, 1, lo, hi]
    b[:6] = [bits, bits + 1, -1 if signed else hi, bits - 1, 0, 3]
    an = [None if i % 17 == 5 else v for i, v in enumerate(a)]
    GC.register(gpu, "bw", pa.table({"a": pa.array(an, at), "b": pa.array(b, at)}), 2)
    scan = P.scan("bw", [P.field("a", ir, True), P.field("b", ir)])
    ops = ["&", "|", "^", "<<", ">>"]
    proj = P.project([(P.binop(op, c("a"), c("b")), op) for op in ops], scan)
    got = driver.run_stages(gpu, [P.Stage(1, P.shuffle_writer(proj, 1))], f"bw-{ir}")
    # the table's partitions come back in order
    for op in ops:
        col = got.column(op)
        assert col.type == at
        want = [None if x is None else rust_bitwise(op, x, y, bits, signed) for x, y in zip(an, b)]
        assert col.to_pylist() == want, op


def test_proto_fixtures_run_on_the_device(gpu, oracle):
    """every accepted fixture, its stages decoded from protobuf bytes, over aggregate_test_100 in 1, 2 and 4 partitions"""
    import golden_data as G
    with open(FIXTURES) as f:
        cases = [cs for cs in json.load(f)["cases"] if "refuse" not in cs]
    t = G.load("aggregate_test_100")
    G.register(oracle, "aggregate_test_100", t, 1)
    for parts in (1, 2, 4):
        G.register(gpu, "aggregate_test_100", t, parts)
        for cs in cases:
            if len(cs["stages"]) == 1 and parts > 1:
                continue  # a Single aggregate groups each input partition on its own
            run = cs["run"]
            stages = [P.Stage(i + 1, json.loads(engine.plan_proto_to_json(base64.b64decode(st["proto_b64"]), "job")))
                      for i, st in enumerate(cs["stages"])]
            job = f"fx-{cs['name']}-{parts}".replace("/", "-")
            got = driver.run_stages(gpu, stages, job)
            nk = len(run["keys"])
            if run["grouping_projection"]:
                ids = got.column("__grouping_id").to_pylist()
                for name, kidx in run["grouping_projection"]:
                    want_g = [sum(((i >> (nk - 1 - k)) & 1) << (len(kidx) - 1 - j) for j, k in enumerate(kidx)) for i in ids]
                    assert got.column(name).to_pylist() == want_g, name
                got = got.drop_columns([n for n, _ in run["grouping_projection"]])
            want = GC.expected(oracle, json.loads(run["input_ir"]), [(k["expr"], k["name"]) for k in run["keys"]], run["aggs"],
                               run["sets"], job)
            assert_tables_equal(got, want, f64_rtol=RTOL)


def test_engine_runs_after_every_refused_plan(gpu):
    t = GC.make_table(200, seed=9)
    GC.register(gpu, "gs", t, 1)
    scan = P.scan("gs", GC.SCHEMA)
    bad = [
        P.aggregate("Single", _keys(["ks", "ki"]), GC.AGGS, scan, grouping_sets=[[False, True], [False, True]]),
        P.aggregate("Single", _keys(["ks", "ki", "kd", "kt", "kf", "kb", "n", "s"]), GC.AGGS, scan, grouping_sets=P.rollup_sets(8)),
        P.aggregate("Single", _keys(["ks"]), [P.agg("var", c("v"), "var_v")], scan, grouping_sets=P.rollup_sets(1)),
        P.aggregate("Single", _keys(["ks", "ki"]), GC.AGGS, scan, grouping_sets=[[True]]),
        P.aggregate("Final", _keys(["ks"]), [P.agg("count", None, "cnt")], scan, grouping_sets=[[True]]),
        P.project([(P.binop("&", c("ki"), c("n")), "mixed")], scan),
    ]
    for i, b in enumerate(bad):
        with pytest.raises(engine.B200Error):
            gpu.create_query_stage_exec("bad", 1 + i, json.dumps(P.shuffle_writer(b, 1 + i)))
    got = driver.run_stages(gpu, GC.single_stages(scan, _keys(["ks"]), [P.agg("count", None, "cnt")], P.rollup_sets(1)), "after-bad")
    assert sum(got.column("cnt").to_pylist()) == 2 * t.num_rows
