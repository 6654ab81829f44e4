"""Window functions on the device against the per-row restatement (window_cases.py): every function over every frame kind
and argument type, inputs of 0 to 300,000 rows with 100 k partitions or one, a Float64 frame sum a prefix difference would
ruin, the reference scheduler's window stage over TPC-H lineitem, top-N per group over an aggregate, the sort the operator
skips below a matching SortExec, refusals, and the operator's metrics."""
import base64
import ctypes as C
import json
import math
import os
import threading

import pyarrow as pa
import pytest

import window_cases as W
from ballista_b200 import driver, engine
from ballista_b200 import plan as P

pytestmark = pytest.mark.gpu
c = P.col
EPS = 2.0 ** -52

FRAMES = {
    "default": None,
    "range_unbounded": P.range_(P.UNBOUNDED_PRECEDING, P.UNBOUNDED_FOLLOWING),
    "range_current_to_end": P.range_(P.CURRENT_ROW, P.UNBOUNDED_FOLLOWING),
    "range_peers": P.range_(P.CURRENT_ROW, P.CURRENT_ROW),
    "rows_running": P.rows(P.UNBOUNDED_PRECEDING, P.CURRENT_ROW),
    "rows_2p_cur": P.rows(P.preceding(2), P.CURRENT_ROW),
    "rows_1p_1f": P.rows(P.preceding(1), P.following(1)),
    "rows_3p_1p": P.rows(P.preceding(3), P.preceding(1)),
    "rows_1f_3f": P.rows(P.following(1), P.following(3)),
    "rows_cur_end": P.rows(P.CURRENT_ROW, P.UNBOUNDED_FOLLOWING),
    "rows_5p_end": P.rows(P.preceding(5), P.UNBOUNDED_FOLLOWING),
    "rows_start_2f": P.rows(P.UNBOUNDED_PRECEDING, P.following(2)),
    "rows_all": P.rows(P.UNBOUNDED_PRECEDING, P.UNBOUNDED_FOLLOWING),
    "rows_empty": P.rows(P.following(2), P.following(1)),
    "rows_wide": P.rows(P.preceding(40), P.following(59)),
}
PART = ["g"]
ORDER = [("o", True, False)]


def _keys(partition, order):
    return [c(p) for p in partition], [P.sort_key(c(n), asc, nf) for n, asc, nf in order]


def _run(gpu, table, exprs, partition=PART, order=ORDER, sorted_input=False, job="w"):
    W.register(gpu, "wt", table)
    pk, ob = _keys(partition, order)
    exprs = [dict(w, partition_by=pk, order_by=ob) for w in exprs]
    src = P.scan("wt", W.SCHEMA)
    if sorted_input:
        src = P.sort([P.sort_key(k) for k in pk] + ob, src)
    return driver.run_stages(gpu, W.stages(P.window(exprs, src, pk)), job)


def _check(got: pa.Table, table: pa.Table, exprs, partition=PART, order=ORDER):
    if got is None:
        assert table.num_rows == 0
        return
    assert got.num_rows == table.num_rows
    assert got.column("rid").to_pylist() == list(range(table.num_rows)), "rows must come out in input order"
    want = W.evaluate(table, exprs, partition, order)
    for w in exprs:
        g, e = got.column(w["name"]).to_pylist(), want[w["name"]]
        arg = w.get("args", [{}])[0].get("col") if w.get("args") else None
        float_sum = w["fn"] in ("sum", "avg") and (W.TYPES.get(arg) == "f64" or (w["fn"] == "avg" and not isinstance(W.TYPES.get(arg), dict)))
        if not float_sum:
            bad = [(i, g[i], e[i]) for i in range(len(e)) if not (g[i] == e[i] and (g[i] is None) == (e[i] is None))]
            assert not bad, (w["name"], bad[:5])
            continue
        bounds = W.frame_abs_sum(table, w, partition, order)
        for i in range(len(e)):
            if e[i] is None or g[i] is None:
                assert g[i] is None and e[i] is None, (w["name"], i, g[i], e[i])
                continue
            m, sabs = bounds[i]
            tol = (m + 1) * EPS * sabs / (m if w["fn"] == "avg" else 1)
            assert abs(g[i] - e[i]) <= tol, (w["name"], i, g[i], e[i], tol)


def _aggs_for(frame, tag):
    f = FRAMES[frame]
    out = [P.win("count", f"cnt_star_{tag}", [], frame=f), P.win("count", f"cnt_ks_{tag}", [c("ks")], frame=f),
           P.win("first_value", f"first_ks_{tag}", [c("ks")], frame=f), P.win("last_value", f"last_dt_{tag}", [c("dt")], frame=f),
           P.win("nth_value", f"nth_dec_{tag}", [c("dec"), P.lit_i64(2)], frame=f)]
    for col_ in ("i32", "i64", "u64", "dec", "f64"):
        out += [P.win("sum", f"sum_{col_}_{tag}", [c(col_)], frame=f), P.win("min", f"min_{col_}_{tag}", [c(col_)], frame=f),
                P.win("max", f"max_{col_}_{tag}", [c(col_)], frame=f)]
    out += [P.win("avg", f"avg_dec_{tag}", [c("dec")], frame=f), P.win("avg", f"avg_f64_{tag}", [c("f64")], frame=f),
            P.win("avg", f"avg_i32_{tag}", [c("i32")], frame=f), P.win("min", f"min_dt_{tag}", [c("dt")], frame=f),
            P.win("max", f"max_b_{tag}", [c("b")], frame=f)]
    return out


RANKING = [P.win("row_number", "rn"), P.win("rank", "rk"), P.win("dense_rank", "drk"), P.win("percent_rank", "prk"),
           P.win("cume_dist", "cd"), P.win("ntile", "nt3", [P.lit_i64(3)]), P.win("ntile", "nt50", [P.lit_i64(50)]),
           P.win("lag", "lag_i64", [c("i64")]), P.win("lead", "lead2_ks", [c("ks"), P.lit_i64(2)]),
           P.win("lag", "lag_dec_d", [c("dec"), P.lit_i64(1), P.lit_dec(-5, 12, 2)]),
           P.win("lead", "lead_neg_dt", [c("dt"), P.lit_i64(-3)]), P.win("lag", "lag_h_d", [c("h"), P.lit_i64(1), P.lit_utf8("none")]),
           P.win("lag", "lag_b", [c("b"), P.lit_i64(4)])]


@pytest.mark.parametrize("frame", list(FRAMES))
def test_framed_functions_every_type(gpu, frame):
    t = W.make_table(1000, seed=7)
    exprs = _aggs_for(frame, frame)
    _check(_run(gpu, t, exprs, job=f"w-{frame}"), t, exprs)


@pytest.mark.parametrize("partition, order", [
    (["g"], [("o", True, False)]),
    (["h"], [("f64", False, True)]),               # Utf8 partition key, DESC NULLS FIRST over floats
    (["g", "h"], [("ks", True, True), ("dt", False, False)]),
    ([], [("o", False, False)]),                   # one partition
    (["g"], []),                                   # no ORDER BY: the partition is one peer group
], ids=["g_o", "utf8_f64desc", "two_keys", "no_partition", "no_order"])
def test_ranking_and_offsets(gpu, partition, order):
    t = W.make_table(1000, seed=3)
    _check(_run(gpu, t, RANKING, partition, order, job="w-rank"), t, RANKING, partition, order)


@pytest.mark.parametrize("n", [0, 1, 1000, 300_000])
def test_sizes(gpu, n):
    t = W.make_table(n, seed=n)
    exprs = RANKING[:6] + _aggs_for("rows_2p_cur", "a")[5:8]
    if n <= 1000:  # the restatement reads every frame row by row: unbounded frames are quadratic in Python
        exprs += [P.win("sum", "run_f64", [c("f64")]), P.win("max", "wmax", [c("i64")], frame=FRAMES["rows_wide"])]
    _check(_run(gpu, t, exprs, job=f"w-size-{n}"), t, exprs)


def test_many_partitions_and_one(gpu):
    n = 300_000
    t = W.make_table(n, seed=5)
    t = t.set_column(1, "g", pa.array([i % 100_000 for i in range(n)], pa.int32()))
    exprs = [P.win("row_number", "rn"), P.win("sum", "s", [c("i64")], frame=FRAMES["rows_1p_1f"]), P.win("lag", "lg", [c("dec")])]
    _check(_run(gpu, t, exprs, job="w-100k"), t, exprs)
    _check(_run(gpu, t, exprs, partition=[], job="w-one"), t, exprs, partition=[])


def test_float_frame_sum_after_a_large_value(gpu):
    """1e15 then small values, 3-row frames: a difference of running sums would leave nothing of the small values."""
    n = 5000
    t = W.make_table(n, seed=1, null_frac=0.0)
    vals = [1e15] + [0.1 * (i % 7) + 1e-3 for i in range(n - 1)]
    t = t.set_column(t.column_names.index("f64"), "f64", pa.array(vals, pa.float64()))
    t = t.set_column(1, "g", pa.array([0] * n, pa.int32())).set_column(3, "o", pa.array(list(range(n)), pa.int64()))
    exprs = [P.win("sum", "s3", [c("f64")], frame=P.rows(P.preceding(2), P.CURRENT_ROW)),
             P.win("avg", "a3", [c("f64")], frame=P.rows(P.preceding(1), P.following(1)))]
    got = _run(gpu, t, exprs, job="w-prec")
    _check(got, t, exprs)
    s3 = got.column("s3").to_pylist()
    assert abs(s3[100] - math.fsum(vals[98:101])) <= 4 * EPS * math.fsum(abs(v) for v in vals[98:101])


def test_matching_sort_below_is_not_repeated(gpu):
    t = W.make_table(3000, seed=9)
    exprs = RANKING[:3] + [P.win("sum", "s", [c("i64")])]
    s0 = gpu.counter("window_sorts")
    got_sorted = _run(gpu, t, exprs, sorted_input=True, job="w-sorted")
    assert gpu.counter("window_sorts") == s0, "a SortExec by (partition keys, order keys) feeds the window: no second sort"
    got_plain = _run(gpu, t, exprs, job="w-plain")
    assert gpu.counter("window_sorts") == s0 + 1
    _check(got_plain, t, exprs)
    # the sorted plan's rows come out in the sort's order; the window values per row are the same
    by_rid = {r["rid"]: r for r in got_sorted.to_pylist()}
    for r in got_plain.to_pylist():
        assert {w["name"]: r[w["name"]] for w in exprs} == {w["name"]: by_rid[r["rid"]][w["name"]] for w in exprs}


def test_top_n_per_group_over_an_aggregate(gpu, oracle):
    t = W.make_table(5000, seed=11)
    for e in (gpu, oracle):
        W.register(e, "wt", t)
    agg = P.aggregate("Single", [(c("g"), "g"), (c("o"), "o")], [P.agg("sum", c("i64"), "s")], P.scan("wt", W.SCHEMA))
    base = driver.run_stages(oracle, W.stages(agg), "w-topn-base")
    ob = [P.sort_key(c("s"), False, False), P.sort_key(c("o"))]
    win = P.window([P.win("row_number", "rn", [], [c("g")], ob)], agg, [c("g")])
    plan = P.filter_(P.binop("<=", c("rn"), P.lit_i64(3)), win)
    got = driver.run_stages(gpu, W.stages(plan), "w-topn")
    rows = base.to_pylist()
    want = []
    for g in {r["g"] for r in rows}:
        grp = sorted([r for r in rows if r["g"] == g], key=lambda r: ((r["s"] is None), -(r["s"] or 0), (r["o"] is None, r["o"])))
        want += [(g, r["o"], r["s"], k + 1) for k, r in enumerate(grp[:3])]
    key = lambda x: tuple((v is None, v) for v in x)
    assert sorted(((r["g"], r["o"], r["s"], r["rn"]) for r in got.to_pylist()), key=key) == sorted(want, key=key)


def test_reference_planner_stage_on_lineitem(gpu):
    """rank() OVER (PARTITION BY l_shipmode ORDER BY l_shipdate DESC) <= 100 after a hash shuffle on l_shipmode.  The window
    stage is the reference scheduler's (planner.rs:1128-1178): SortExec(l_shipmode ASC NULLS LAST, l_shipdate DESC) ->
    BoundedWindowAggExec (mode Sorted) -> FilterExec.  Simplified around it: the scan projects the four columns the query
    reads instead of a ProjectionExec, the last stage only gathers the partitions (no final SortPreservingMergeExec on
    (l_shipdate, rk)), and the rows are compared as a set."""
    cols = ["l_orderkey", "l_linenumber", "l_shipmode", "l_shipdate"]
    n = engine.GpuExecutionEngine.tpch_table_rows("lineitem", 20)
    gpu.drop_table("lineitem")
    gpu.tpch_generate("lineitem", 20, 0, 0, n // 2, cols)
    gpu.tpch_generate("lineitem", 20, 1, n // 2, n, cols)
    sch = [P.field("l_orderkey", "i64"), P.field("l_linenumber", "i32"), P.field("l_shipmode", "utf8"), P.field("l_shipdate", "date32")]
    full = driver.run_stages(gpu, [P.Stage(1, P.shuffle_writer(P.scan("lineitem", sch), 1))], "w-li-all")
    pk, ob = [c("l_shipmode")], [P.sort_key(c("l_shipdate"), False, True)]
    want_rank = W.evaluate(full, [P.win("rank", "rk")], ["l_shipmode"], [("l_shipdate", False, True)])["rk"]
    want = sorted((r["l_orderkey"], r["l_linenumber"], k) for r, k in zip(full.to_pylist(), want_rank) if k <= 100)
    for parts in (2, 4):
        s1 = P.Stage(1, P.shuffle_writer(P.scan("lineitem", sch), 1, [c("l_shipmode")], parts))
        srt = P.sort([P.sort_key(c("l_shipmode"), True, False), P.sort_key(c("l_shipdate"), False, True)], P.shuffle_reader(1, sch))
        w = P.window([P.win("rank", "rk", [], pk, ob, P.range_(P.UNBOUNDED_PRECEDING, P.CURRENT_ROW))], srt, pk)
        s2 = P.Stage(2, P.shuffle_writer(P.filter_(P.binop("<=", c("rk"), P.lit_i64(100)), w), 2))
        s3 = P.Stage(3, P.shuffle_writer(P.coalesce_partitions(P.shuffle_reader(2, sch + [P.field("rk", "u64")])), 3), n_tasks=1)
        s0 = gpu.counter("window_sorts")
        got = driver.run_stages(gpu, [s1, s2, s3], f"w-li-{parts}")
        assert gpu.counter("window_sorts") == s0
        assert sorted((r["l_orderkey"], r["l_linenumber"], r["rk"]) for r in got.to_pylist()) == want


@pytest.mark.parametrize("bad", [
    P.win("sum", "x", [c("i64")], frame=P.range_(P.preceding(3), P.CURRENT_ROW)),
    P.win("sum", "x", [c("i64")], frame={"units": "groups", "start": P.UNBOUNDED_PRECEDING, "end": P.CURRENT_ROW}),
    dict(P.win("lag", "x", [c("i64")]), ignore_nulls=True),
    dict(P.win("count", "x", [c("i64")]), distinct=True),
    P.win("var_samp", "x", [c("f64")]),
    P.win("max", "x", [c("ks")]),
    P.win("ntile", "x", [c("i64")]),
])
def test_refusals_leave_the_engine_working(gpu, bad):
    t = W.make_table(100, seed=2)
    with pytest.raises(engine.B200Error) as ei:
        _run(gpu, t, [bad], job="w-bad")
    assert ei.value.code == -2, str(ei.value)
    exprs = [P.win("row_number", "rn")]
    _check(_run(gpu, t, exprs, job="w-after"), t, exprs)


def test_metrics_and_kernel_families(gpu):
    t = W.make_table(20_000, seed=4)
    gpu.set_config("b200.metrics.kernel_timing", "on")
    gpu.kernel_stats(reset=True)
    try:
        exprs = [P.win("rank", "rk"), P.win("sum", "s", [c("f64")], frame=FRAMES["rows_1p_1f"]), P.win("lead", "ld", [c("i32")])]
        W.register(gpu, "wt", t)
        pk, ob = _keys(PART, ORDER)
        plan = P.window([dict(w, partition_by=pk, order_by=ob) for w in exprs], P.scan("wt", W.SCHEMA), pk)
        metrics = []
        driver.run_stages(gpu, W.stages(plan), "w-met", metrics_out=metrics)
        ks = gpu.kernel_stats()
    finally:
        gpu.set_config("b200.metrics.kernel_timing", "off")
    for fam in ("window_sort", "window_bounds", "window_scan", "window_frames"):
        assert ks.get(fam, {}).get("launches", 0) >= 1 and ks[fam]["bytes"] > 0, (fam, sorted(ks))
    ops = [m for _, stage in metrics for m in stage if m["name"] == "WindowAggExec"]
    assert ops and all(m["input_rows"] == t.num_rows and m["output_rows"] == t.num_rows and m["kernel_launches"] > 0 for m in ops), metrics


FIXTURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "window_proto_plans.json")


def _fixtures():
    with open(FIXTURES) as f:
        return [cs for cs in json.load(f)["cases"] if "refuse" not in cs]


@pytest.mark.parametrize("case", _fixtures(), ids=lambda cs: cs["name"])
def test_proto_fixtures_run_on_the_device(gpu, case):
    """Every accepted fixture, decoded from its protobuf bytes, gives the rows of its source plan; the window stages over
    the generated table are also held to the restatement."""
    if case["table"] == "wt":
        t = W.make_table(1000, seed=17)
        W.register(gpu, "wt", t)
    else:
        n = engine.GpuExecutionEngine.tpch_table_rows("lineitem", 20)
        gpu.drop_table("lineitem")
        gpu.tpch_generate("lineitem", 20, 0, 0, n // 2, ["l_orderkey", "l_linenumber", "l_shipmode", "l_shipdate"])
        gpu.tpch_generate("lineitem", 20, 1, n // 2, n, ["l_orderkey", "l_linenumber", "l_shipmode", "l_shipdate"])
    job = case["name"].replace("/", "-")
    decoded = [P.Stage(i + 1, json.loads(engine.plan_proto_to_json(base64.b64decode(st["proto_b64"]), "job")))
               for i, st in enumerate(case["stages"])]
    source = [P.Stage(i + 1, json.loads(st["ir"])) for i, st in enumerate(case["stages"])]
    got = driver.run_stages(gpu, decoded, job + "-proto")
    want = driver.run_stages(gpu, source, job + "-ir")
    key = lambda r: tuple((v is None, str(v)) for v in r)  # noqa: E731
    assert sorted(map(key, (tuple(r.values()) for r in got.to_pylist()))) == sorted(map(key, (tuple(r.values()) for r in want.to_pylist())))
    if case["table"] == "wt":
        node = json.loads(case["stages"][0]["ir"])["input"]
        exprs = [dict(w, fn="avg" if w["fn"] == "mean" else w["fn"]) for w in node["window_expr"]]
        _check(got, t, exprs, [k["col"] for k in node["partition_keys"]],
               [(k["expr"]["col"], k["asc"], k["nulls_first"]) for k in exprs[0]["order_by"]])


def test_cancelled_window_task_stores_nothing(gpu):
    """A window task cancelled while it runs (or, failing that, before it starts) fails with B200_ERR_CANCELLED and leaves no
    partition stored; the engine keeps working."""
    cols = ["l_orderkey", "l_suppkey", "l_extendedprice", "l_shipdate"]
    n = engine.GpuExecutionEngine.tpch_table_rows("lineitem", 1000)
    gpu.drop_table("lineitem")
    gpu.tpch_generate("lineitem", 1000, 0, 0, n, cols)
    sch = [P.field("l_orderkey", "i64"), P.field("l_suppkey", "i64"), P.field("l_extendedprice", P.dec(15, 2)), P.field("l_shipdate", "date32")]
    pk, ob = [c("l_suppkey")], [P.sort_key(c("l_shipdate"))]
    w = P.window([P.win("rank", "rk", [], pk, ob), P.win("sum", "s", [c("l_extendedprice")], pk, ob, P.rows(P.preceding(9), P.following(10))),
                  P.win("lag", "lg", [c("l_orderkey")], pk, ob)], P.scan("lineitem", sch), pk)
    st = P.Stage(1, P.shuffle_writer(w, 1))
    cancelled_while_running = False
    for k, delay in enumerate((0.02, 0.005, 0.001, None)):
        job = f"win-cancel{k}"
        flag = C.c_int32(1 if delay is None else 0)
        q = gpu.create_query_stage_exec(job, 1, st.json(job))
        timer = threading.Timer(delay, lambda: setattr(flag, "value", 1)) if delay is not None else None
        if timer:
            timer.start()
        cancelled = False
        try:
            q.execute_query_stage(0, cancel_flag=flag)
        except engine.B200Error as ex:
            assert ex.code == -6, str(ex)
            cancelled = True
        if timer:
            timer.join()
        q.release()
        if cancelled:
            assert gpu.partition_rows(job, 1, 0) < 0
            cancelled_while_running = delay is not None
            break
        gpu.remove_job_data(job)
    assert cancelled
    t = W.make_table(200, seed=8)
    exprs = [P.win("row_number", "rn")]
    _check(_run(gpu, t, exprs, job="w-after-cancel"), t, exprs)
    print("cancelled while running:", cancelled_while_running)
