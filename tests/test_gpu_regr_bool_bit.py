"""regr_* / bool_and / bool_or / bit_and / bit_or / bit_xor on the device against the plain-Python restatement
(regr_bool_bit_cases.py): bool / bit results and regr_count bit-exact, the other regr_* values within the bounds the
VAR / CORR tests justify and their NULL pattern exact; Single and Partial -> shuffle -> Final / FinalPartitioned; the
register sink (<= 4 groups) and the global sink (many groups), told apart by the kernel timer families; 0 to 2^20 + 3
rows; constant regression arguments; grouping sets against the UNION ALL form; plans decoded from protobuf bytes."""
import base64
import json
import math

import numpy as np
import pyarrow as pa
import pytest

import golden_data as G
from ballista_b200 import driver, engine
from ballista_b200 import plan as P
from regr_bool_bit_cases import BIT, BOOL, REGR, fold, grouped, partial_only, regr_exact, regr_state, stages, union_all
from stat_cases import rel_close

pytestmark = pytest.mark.gpu
c = P.col
RTOL = 1e-10
PA = {"i8": pa.int8(), "i16": pa.int16(), "i32": pa.int32(), "i64": pa.int64(), "u8": pa.uint8(), "u16": pa.uint16(),
      "u32": pa.uint32(), "u64": pa.uint64()}
NAMES = ["k3", "kg", "kb"] + list(PA) + ["b", "y", "x"]


@pytest.fixture()
def timed(gpu):
    gpu.set_config("b200.metrics.kernel_timing", "on")
    yield gpu
    gpu.set_config("b200.metrics.kernel_timing", "off")


def make_rows(n, seed):
    """k3: 3 groups, kg: groups of 3 rows (the last one may be shorter), kb: 4 groups whose b is all true, all false,
    mixed and all NULL; every integer width with its extremes (Int8 -128, UInt64 with the top bit set); y, x with NULLs on
    either side"""
    rng = np.random.default_rng(seed)
    i = np.arange(n)
    cols = [(i % 3).tolist(), (i // 3).tolist(), (i % 4).tolist()]
    for t, ty in PA.items():
        dt = ty.to_pandas_dtype()
        info = np.iinfo(dt)
        v = rng.integers(info.min, info.max, size=n, dtype=dt, endpoint=True)
        v[i % 7 == 0] = info.min if t.startswith("i") else info.max
        cols.append([None if m else int(a) for a, m in zip(v, rng.random(n) < 0.1)])
    mixed = rng.random(n) < 0.5
    bnull = rng.random(n) < 0.1
    cols.append([None if (k == 3 or (k < 3 and m)) else (True if k == 0 else False if k == 1 else bool(mx))
                 for k, m, mx in zip(cols[2], bnull, mixed)])
    xv = rng.integers(-50, 50, size=n).astype(np.float64)
    xn = rng.random(n) < 0.1
    yv = np.where(xn, rng.normal(size=n), 2.5 * xv + 7 + rng.normal(size=n))
    yn = rng.random(n) < 0.1
    cols.append([None if m else float(a) for a, m in zip(yv, yn)])
    cols.append([None if m else float(a) for a, m in zip(xv, xn)])
    return list(zip(*cols))


def to_batch(rows):
    cols = list(zip(*rows)) if rows else [[] for _ in NAMES]
    types = [pa.int32(), pa.int64(), pa.int32()] + list(PA.values()) + [pa.bool_(), pa.float64(), pa.float64()]
    return pa.record_batch([pa.array(list(v), t) for v, t in zip(cols, types)], names=NAMES)


SCHEMA = [P.field("k3", "i32", False), P.field("kg", "i64", False), P.field("kb", "i32", False)] + \
         [P.field(t, t, True) for t in PA] + [P.field("b", "bool", True), P.field("y", "f64", True), P.field("x", "f64", True)]
IDX = {n: i for i, n in enumerate(NAMES)}


def register(gpu, name, rows, parts):
    gpu.drop_table(name)
    step = max((len(rows) + parts - 1) // parts, 1)
    for p in range(parts):
        gpu.register_batch(name, p, to_batch(rows[p * step:(p + 1) * step]))


def agg_sets(big):
    """one AggregateExec per argument: a column's three bit functions, its COUNT and COUNT(*) are 5 accumulators, within
    the register sink's 6.  The nine regr_* over one pair share one AggregateExec in every stage.  Over 2^20 rows only
    regr_count (the other regr_* take exact rational arithmetic per row in the reference)."""
    out = [[(fn, c(t), None, f"{fn}_{t}", t) for fn in BIT] for t in (("i8", "i64", "u64") if big else PA)]
    out.append([(fn, c("b"), None, fn, "bool") for fn in BOOL])
    out.append([(fn, c("y"), c("x"), fn, None) for fn in (["regr_count"] if big else REGR)])
    return out


def check(got, key_names, want):
    assert got.num_rows == len(want), (got.num_rows, len(want))
    for r in got.to_pylist():
        g = tuple(r[k] for k in key_names)
        assert g in want, g
        for nm, w in want[g].items():
            v = r[nm]
            if isinstance(w, float) or w is None and isinstance(v, float):
                assert rel_close(v, w, RTOL), (g, nm, v, w)
            else:
                assert v == w and type(v) is type(w), (g, nm, v, w)


@pytest.mark.parametrize("n", [0, 1, 2, 1023, 1024, 1025, 4097, (1 << 20) + 3])
def test_row_counts_sinks_and_modes(timed, n):
    gpu = timed
    big = n > 5000
    rows = make_rows(n, n)
    for key, sink in (("k3", "pipeline_agg_reg"), ("kg", "pipeline_agg_global"), (None, "pipeline_agg_reg")):
        keys = [(c(key), key)] if key else []
        kf = [P.field(key, "i32" if key == "k3" else "i64", False)] if key else []
        for mode in ("Single", "SinglePartitioned", "Partial"):
            register(gpu, "rbb", rows, 3 if mode == "Partial" else 1)
            for aggs in agg_sets(big):
                want = grouped(rows, [IDX[key]] if key else [], [(fn, IDX[a["col"]], IDX[b["col"]] if b else None, nm, t) for fn, a, b, nm, t in aggs])
                gpu.kernel_stats(reset=True)
                got = driver.run_stages(gpu, stages(P.scan("rbb", SCHEMA), aggs, keys, kf, mode), f"rbb-{n}-{key}-{aggs[0][3]}-{mode}")
                ks = gpu.kernel_stats()
                check(got, [key] if key else [], want)
                assert "pipeline_fused_agg" not in ks and "groupby_hash_agg" not in ks, ks
                if n > 4 and mode != "Partial":  # a plan of fewer rows has at most 4 groups on either key
                    assert sink in ks, ks
                    if sink == "pipeline_agg_reg":
                        assert "pipeline_agg_global" not in ks, ks
                    if aggs[0][0] in REGR:  # regr_count alone needs only the pass-1 count
                        assert (sink + "_pass2" in ks) == (len(aggs) > 1), ks


def test_partial_states(gpu):
    rows = make_rows(4097, 5)
    register(gpu, "rbs", rows, 1)
    for aggs in agg_sets(False):
        got = driver.run_stages(gpu, partial_only(P.scan("rbs", SCHEMA), aggs, [(c("k3"), "k3")]), f"rbs-{aggs[0][3]}").to_pylist()
        groups = {}
        for r in rows:
            groups.setdefault(r[0], []).append(r)
        assert len(got) == 3
        for r in got:
            rs = groups[r["k3"]]
            for fn, a, b, nm, t in aggs:
                if fn in REGR:
                    n, mx, my, m2x, m2y, co = regr_state([q[IDX["y"]] for q in rs], [q[IDX["x"]] for q in rs])
                    assert r[f"{nm}[count]"] == n
                    for s, w in (("mean_x", mx), ("mean_y", my), ("m2_x", m2x), ("m2_y", m2y)):
                        assert rel_close(r[f"{nm}[{s}]"], w, 1e-12), (nm, s, r[f"{nm}[{s}]"], w)
                    assert abs(r[f"{nm}[algo_const]"] - co) <= 1e-12 * math.sqrt(m2x * m2y), (nm, r, co)
                else:
                    w = fold(fn, [q[IDX[a["col"]]] for q in rs], t)
                    assert r[f"{nm}[{fn}]"] == w, (nm, r, w)


def test_constant_regression_arguments(gpu):
    """x constant within a group (0.1, 1e12 + 0.1), y constant, both: sxx / syy exactly 0 and slope, intercept, r2 NULL;
    through Partial -> Final the group's rows are split 1 / 2 / 4 over three partitions, one of them with a state of
    count 0 (its only row has x NULL)"""
    def row(k, y, x):
        return (k, 0, 0) + (None,) * len(PA) + (None, y, x)
    parts = [[], [], []]
    for p, cnt in enumerate((1, 2, 4)):
        for j in range(cnt):
            parts[p].append(row(0, float(j + 3 * p), 0.1))
            parts[p].append(row(1, float(j * j - p), 1e12 + 0.1))
            parts[p].append(row(2, 0.1, float(j + p)))
            parts[p].append(row(3, 1e12 + 0.1, 0.1))
            parts[p].append(row(4, 5.0, float(j)))  # a single-row group in the first partition, a regular one overall
    parts[2].append(row(0, 1.0, None))
    allrows = [r for p in parts for r in p]
    aggs = [(fn, c("y"), c("x"), fn, None) for fn in REGR]
    want = grouped(allrows, [0], [(fn, IDX["y"], IDX["x"], fn, None) for fn in REGR])
    for g in (0, 1, 3):
        assert want[(g,)]["regr_sxx"] == 0.0 and want[(g,)]["regr_slope"] is None and want[(g,)]["regr_r2"] is None
    for mode in ("Single", "Partial"):
        gpu.drop_table("rbc")
        if mode == "Single":
            gpu.register_batch("rbc", 0, to_batch(allrows))
        else:
            for p in range(3):
                gpu.register_batch("rbc", p, to_batch(parts[p]))
        got = driver.run_stages(gpu, stages(P.scan("rbc", SCHEMA), aggs, [(c("k3"), "k3")], [P.field("k3", "i32", False)], mode),
                                f"rbc-{mode}")
        check(got, ["k3"], want)
        for r in got.to_pylist():
            if r["k3"] in (0, 1, 3):
                assert r["regr_sxx"] == 0.0, r


@pytest.mark.parametrize("keyed", [True, False])
def test_constant_regression_arguments_register_sink(timed, keyed):
    """The same rule on the register sink (at most 4 groups, or none), with negative constants, whose total-order keys are
    negative: a wrong identity of the range's largest key, a lost high word or swapped bounds in the flush would show.
    Thousands of rows per group, so many threads and CTAs fold and combine the ranges.  Single runs on the register sink
    alone; Partial's first stage runs there too (a Final always runs on the global sink)."""
    gpu = timed
    rng = np.random.default_rng(23)

    def row(k, y, x):
        return (k, 0, 0) + (None,) * len(PA) + (None, y, x)
    consts = [(-0.1, None), (-(1e12 + 0.1), None), (None, -0.1), (-(1e12 + 0.1), 0.1)]  # (x, y); None: varying
    rows = []
    for i in range(6000):
        k = i % 4 if keyed else 1
        cx, cy = consts[k]
        v = float(rng.integers(-40, 40))
        rows.append(row(k, cy if cy is not None else v + float(rng.normal()), cx if cx is not None else v))
    rows.append(row(rows[0][0], 3.0, None))  # x NULL: not counted, and not in the range
    aggs = [(fn, c("y"), c("x"), fn, None) for fn in REGR]
    want = grouped(rows, [0] if keyed else [], [(fn, IDX["y"], IDX["x"], fn, None) for fn in REGR])
    for g, w in want.items():
        assert w["regr_r2"] is None  # sxx = 0 or syy = 0 in every group
        assert (w["regr_slope"] is None) == (consts[g[0] if keyed else 1][0] is not None)  # y constant: slope 0
    keys, kf = ([(c("k3"), "k3")], [P.field("k3", "i32", False)]) if keyed else ([], [])
    for mode in ("Single", "Partial"):
        register(gpu, "rbr", rows, 1 if mode == "Single" else 3)
        gpu.kernel_stats(reset=True)
        got = driver.run_stages(gpu, stages(P.scan("rbr", SCHEMA), aggs, keys, kf, mode), f"rbr-{keyed}-{mode}")
        ks = gpu.kernel_stats()
        check(got, ["k3"] if keyed else [], want)
        for r in got.to_pylist():
            g = r["k3"] if keyed else 1
            assert (r["regr_sxx"] == 0.0) == (consts[g][0] is not None) or g == 2, r
            if consts[g][1] is not None:
                assert r["regr_syy"] == 0.0 and r["regr_sxy"] == 0.0, r
        assert "pipeline_agg_reg" in ks and "pipeline_agg_reg_pass2" in ks, ks
        if mode == "Single":
            assert "pipeline_agg_global" not in ks, ks


def test_all_nine_and_corr_share_one_aggregate(timed):
    gpu = timed
    rows = make_rows(3000, 9)
    register(gpu, "rbn", rows, 1)
    aggs = [(fn, c("y"), c("x"), fn, None) for fn in REGR]
    plan = [P.Stage(1, P.shuffle_writer(P.aggregate("Single", [(c("k3"), "k3")], [P.agg(fn, a, nm, arg2=b) for fn, a, b, nm, _ in aggs] +
                                                     [P.agg("corr", c("x"), "cr", arg2=c("y"))], P.scan("rbn", SCHEMA)), 1))]
    gpu.kernel_stats(reset=True)
    got = driver.run_stages(gpu, plan, "rbn")
    ks = gpu.kernel_stats()
    assert "pipeline_agg_reg" in ks and "pipeline_agg_global" not in ks, ks
    want = grouped(rows, [0], [(fn, IDX["y"], IDX["x"], fn, None) for fn in REGR])
    check(got.drop_columns(["cr"]), ["k3"], want)
    for r in got.to_pylist():
        rs = [q for q in rows if q[0] == r["k3"]]
        r2 = regr_exact("regr_r2", [q[IDX["y"]] for q in rs], [q[IDX["x"]] for q in rs])
        assert rel_close(r["cr"] ** 2, r2, 1e-9), r
    # Partial -> hash shuffle -> FinalPartitioned, one AggregateExec per stage: the Partial extracts the shared state once
    # for the nine, and the Final (whose aggregates carry their arguments, as a Ballista plan does) merges it once
    register(gpu, "rbn", rows, 3)
    st = stages(P.scan("rbn", SCHEMA), aggs, [(c("k3"), "k3")], [P.field("k3", "i32", False)], "Partial")
    assert len(st) == 2
    check(driver.run_stages(gpu, st, "rbn-partial"), ["k3"], want)
    # without the arguments a Final cannot tell that the states are one pair's: each is merged on its own, and nine take
    # more accumulators and co-moments than one AggregateExec holds -- refused, never run partly
    with pytest.raises(engine.B200Error, match="too many"):
        driver.run_stages(gpu, stages(P.scan("rbn", SCHEMA), aggs, [(c("k3"), "k3")], [P.field("k3", "i32", False)], "Partial",
                                      final_args=False), "rbn-noargs")


@pytest.mark.parametrize("sets", ["rollup", "cube"])
def test_grouping_sets_against_union_all(gpu, sets):
    rows = make_rows(5000, 13)
    gs = P.rollup_sets(2) if sets == "rollup" else P.cube_sets(2)
    aggs = [(fn, c("b"), None, fn, "bool") for fn in BOOL] + [(fn, c("i64"), None, fn, "i64") for fn in BIT] + [("bit_xor", c("u8"), None, "xu8", "u8")]
    want = union_all(rows, [IDX["k3"], IDX["kb"]], gs, [(fn, IDX[a["col"]], None, nm, t) for fn, a, _, nm, t in aggs])
    for mode in ("Single", "Partial"):
        register(gpu, "rbg", rows, 1 if mode == "Single" else 3)
        keys = [(c("k3"), "k3"), (c("kb"), "kb")]
        if mode == "Single":
            st = stages(P.scan("rbg", SCHEMA), aggs, keys, grouping_sets=gs)
        else:
            kf = [P.field("k3", "i32", True), P.field("kb", "i32", True), P.field("__grouping_id", "u8", False)]
            st = stages(P.scan("rbg", SCHEMA), aggs, keys, kf, "Partial", grouping_sets=gs)
            st[1].plan["input"]["group_by"].append({"expr": c(2), "name": "__grouping_id"})
        got = driver.run_stages(gpu, st, f"rbg-{sets}-{mode}")
        check(got, ["k3", "kb", "__grouping_id"], want)


def test_protobuf_plans_run_like_their_ir(gpu):
    from decimal import Decimal
    with open(G.__file__.replace("golden_data.py", "golden/regr_bool_bit_proto_plans.json")) as fh:
        cases = json.load(fh)["cases"]
    rng = np.random.default_rng(17)
    n = 3000
    cols = [pa.array([int(v) for v in rng.integers(0, 4, n)], pa.int32()),
            pa.array([None if rng.random() < 0.1 else int(v) for v in rng.integers(-10**6, 10**6, n)], pa.int64()),
            pa.array([None if rng.random() < 0.1 else Decimal(int(v)).scaleb(-2) for v in rng.integers(-10**8, 10**8, n)], pa.decimal128(15, 2)),
            pa.array(rng.normal(size=n), pa.float64()),
            pa.array([None if rng.random() < 0.1 else bool(v) for v in rng.random(n) < 0.9], pa.bool_()),
            pa.array([None if rng.random() < 0.1 else int(v) for v in rng.integers(0, 1 << 16, n)], pa.uint16())]
    b = pa.record_batch(cols, names=["k", "x", "y", "z", "b", "u"])
    gpu.drop_table("t")
    for p in range(2):
        gpu.register_batch("t", p, b.slice(p * n // 2, n // 2))
    by_plan = {}
    for cs in cases:
        by_plan.setdefault(cs["name"].rsplit("/", 1)[0], []).append(cs)
    for name, sts in by_plan.items():
        if len(sts) == 1:
            continue  # a Single aggregate over two partitions groups each on its own: covered by the IR tests
        scalar = "scalar" in name
        decoded = [P.Stage(i + 1, json.loads(engine.plan_proto_to_json(base64.b64decode(s["proto_b64"]), "job")), 1 if scalar and i else None)
                   for i, s in enumerate(sts)]
        ir = [P.Stage(i + 1, json.loads(s["ir"]), 1 if scalar and i else None) for i, s in enumerate(sts)]
        job = name.replace("/", "-")
        got = driver.run_stages(gpu, decoded, job + "-pb").to_pylist()
        want = driver.run_stages(gpu, ir, job + "-ir").to_pylist()
        key = (lambda r: r.get("k", 0))
        got.sort(key=key)
        want.sort(key=key)
        assert len(got) == len(want) and len(got) > 0, name
        for g, w in zip(got, want):
            for col in w:
                if isinstance(w[col], float):
                    assert rel_close(g[col], w[col], 1e-12), (name, col, g[col], w[col])
                else:
                    assert g[col] == w[col], (name, col, g[col], w[col])
