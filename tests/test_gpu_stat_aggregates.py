"""VAR / STDDEV / COVAR / CORR on the device against exact rational arithmetic: the NULL rules at n = 0 / 1 / 2, NaN,
CORR at zero variance, every argument type, ill-conditioned inputs (where power sums lose every digit), TPC-H lineitem on
the register sink (4 groups), the global sink (l_suppkey) and without keys, mixed with SUM / AVG / MIN, Single and
Partial -> hash shuffle -> Final; and the reference's seven goldens over alltypes_plain."""
import json
import math

import numpy as np
import pyarrow as pa
import pytest

import golden_data as G
from ballista_b200 import driver
from ballista_b200 import plan as P
from stat_cases import check_result, grouped_exact, rel_close, stat_stages, welford

pytestmark = pytest.mark.gpu
c = P.col
ALL = ["var", "var_samp", "var_sample", "var_pop", "var_population", "stddev", "stddev_samp", "stddev_pop"]
BI = ["covar", "covar_samp", "covar_pop", "corr"]


@pytest.fixture()
def timed(gpu):
    gpu.set_config("b200.metrics.kernel_timing", "on")
    yield gpu
    gpu.set_config("b200.metrics.kernel_timing", "off")


def _register(gpu, table, batch, parts):
    gpu.drop_table(table)
    step = max((batch.num_rows + parts - 1) // parts, 1)
    for p in range(parts):
        gpu.register_batch(table, p, batch.slice(p * step, step))


def _aggs(x="x", y="y"):
    return [(fn, c(x), None, fn) for fn in ALL] + [(fn, c(x), c(y), fn) for fn in BI]


def _agg_sets():
    """every name, over four AggregateExecs: merging the states of all twelve in one Final takes more than the 16 table
    accumulators and 6 co-moments one holds (such a plan is refused with B200_ERR_UNSUPPORTED)"""
    a = _aggs()
    return [a[:4], a[4:8], a[8:11], a[11:]]


def _names(aggs):
    return [n for *_, n in aggs]


def _exact_aggs(aggs, x="x", y="y"):
    return [(fn, x, y if a2 is not None else None, n) for fn, _, a2, n in aggs]


def _run_modes(gpu, table, batch, schema, keys, key_fields, agg_sets, rtol, job, parts=2, xname="x", yname="y"):
    for i, aggs in enumerate(agg_sets):
        want = grouped_exact(pa.Table.from_batches([batch]), [n for _, n in keys], _exact_aggs(aggs, xname, yname))
        for mode in ("Single", "Partial"):
            _register(gpu, table, batch, 1 if mode == "Single" else parts)
            got = driver.run_stages(gpu, stat_stages(P.scan(table, schema), aggs, keys, key_fields, mode), f"{job}-{i}-{mode}")
            check_result(got, [n for _, n in keys], want, _names(aggs), rtol)


def unit_batch():
    """groups: 0 empty of values, 1 one value, 2 two values, 3 NaN, 4 constant y (corr at zero variance), 5 general with
    NULLs on either side, 6 all NULL"""
    rows = [(1, 3.0, 4.0), (2, 1.0, 2.0), (2, 2.5, -1.0), (3, 1.0, 1.0), (3, math.nan, 2.0), (3, 2.0, 3.0),
            (4, 1.0, 5.0), (4, 2.0, 5.0), (4, 4.0, 5.0), (0, None, 1.0), (0, None, None), (6, None, None)]
    rng = np.random.default_rng(3)
    for _ in range(200):
        rows.append((5, None if rng.random() < 0.1 else float(rng.integers(-50, 50)), None if rng.random() < 0.1 else float(rng.normal())))
    k, x, y = zip(*rows)
    return pa.record_batch([pa.array(k, pa.int32()), pa.array(x, pa.float64()), pa.array(y, pa.float64())], names=["k", "x", "y"])


UNIT_SCHEMA = [P.field("k", "i32", False), P.field("x", "f64", True), P.field("y", "f64", True)]


def test_unit_sets_keyed_and_scalar(gpu):
    b = unit_batch()
    aggs = _aggs()
    _run_modes(gpu, "su", b, UNIT_SCHEMA, [(c("k"), "k")], [P.field("k", "i32", False)], _agg_sets(), 1e-12, "su-k")
    _run_modes(gpu, "su", b, UNIT_SCHEMA, [], [], _agg_sets(), 1e-12, "su-s")
    got = driver.run_stages(gpu, stat_stages(P.scan("su", UNIT_SCHEMA), aggs, [(c("k"), "k")]), "su-rules").to_pylist()
    by = {r["k"]: r for r in got}
    assert by[1]["var"] is None and by[1]["var_pop"] == 0.0 and by[1]["corr"] is None
    assert by[2]["covar"] is not None and by[0]["var_pop"] is None and by[6]["stddev_pop"] is None
    assert math.isnan(by[3]["var"]) and by[4]["corr"] is None  # [EXT] corr at zero variance is NULL


@pytest.mark.parametrize("typ", [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64(),
                                 pa.float32(), pa.float64(), pa.decimal128(15, 2), pa.decimal128(38, 10)])
def test_argument_types(gpu, typ):
    from decimal import Decimal
    rng = np.random.default_rng(7)
    n = 5000
    k = rng.integers(0, 3, n)
    if pa.types.is_decimal(typ):
        vals = [None if rng.random() < 0.05 else Decimal(int(rng.integers(-10**6, 10**6))).scaleb(-typ.scale) for _ in range(n)]
    elif pa.types.is_floating(typ):
        vals = [None if rng.random() < 0.05 else float(np.float32(rng.normal(10, 3))) for _ in range(n)]
    else:
        lo = 0 if pa.types.is_unsigned_integer(typ) else -100
        vals = [None if rng.random() < 0.05 else int(rng.integers(lo, 100)) for _ in range(n)]
    b = pa.record_batch([pa.array(k, pa.int32()), pa.array(vals, typ), pa.array(list(reversed(vals)), typ)], names=["k", "x", "y"])
    tn = str(typ).replace("(", "_").replace(")", "").replace(",", "_").replace(" ", "")
    irt = {"int8": "i8", "int16": "i16", "int32": "i32", "int64": "i64", "uint8": "u8", "uint16": "u16", "uint32": "u32",
           "uint64": "u64", "float": "f32", "double": "f64"}
    t = P.dec(typ.precision, typ.scale) if pa.types.is_decimal(typ) else irt[str(typ)]
    sch = [P.field("k", "i32", False), P.field("x", t, True), P.field("y", t, True)]
    _run_modes(gpu, "sty_" + tn, b, sch, [(c("k"), "k")], [P.field("k", "i32", False)], _agg_sets(), 1e-12, "sty-" + tn)


@pytest.mark.parametrize("keys", [0, 3, 5000])
def test_ill_conditioned(timed, keys):
    """1e9 + small integers and 1e12 + U(0,1): naive power sums return 0 or noise here; two passes keep 1e-12 over raw rows.
    Partial -> Final is bounded by the states themselves: even a correctly rounded Float64 mean near 1e9 or 1e12 is off
    by up to half an ulp (6e-8 / 6e-5), and the merge's n_i * (mean_i - mean)^2 terms carry that into m2 as up to
    2 * sum n_i |mean_i - mean| * 6e-5.  With 11-33 k rows per state (keys 0 and 3: |mean_i - mean| ~ 0.002) that is a few
    1e-6 of m2: held to 1e-5.  With ~7 rows per state (5000 keys, 3 partitions) it is up to ~1e-4: held to 1e-3.  Power
    sums miss both by many orders of magnitude (on these values they return a negative variance or one 1e12 times too
    large)."""
    gpu = timed
    rng = np.random.default_rng(11)
    n = 100000
    x = 1e9 + rng.integers(0, 8, n).astype(np.float64)
    y = 1e12 + rng.random(n)
    k = rng.integers(0, max(keys, 1), n).astype(np.int32)
    b = pa.record_batch([pa.array(k), pa.array(x), pa.array(y)], names=["k", "x", "y"])
    sch = [P.field("k", "i32", False), P.field("x", "f64", False), P.field("y", "f64", False)]
    kk = [(c("k"), "k")] if keys else []
    kf = [P.field("k", "i32", False)] if keys else []
    sets = [[("var", c("x"), None, "vx"), ("stddev_pop", c("y"), None, "sy"), ("var_pop", c("y"), None, "vy")],
            [("covar", c("x"), c("y"), "cv"), ("corr", c("x"), c("y"), "cr")]]
    for i, aggs in enumerate(sets):
        want = grouped_exact(pa.Table.from_batches([b]), ["k"] if keys else [],
                             [(fn, x["col"], y["col"] if y else None, n) for fn, x, y, n in aggs])
        for mode in ("Single", "Partial"):
            _register(gpu, "sic", b, 1 if mode == "Single" else 3)
            gpu.kernel_stats(reset=True)
            got = driver.run_stages(gpu, stat_stages(P.scan("sic", sch), aggs, kk, kf, mode), f"sic-{keys}-{i}-{mode}")
            ks = gpu.kernel_stats()
            if mode == "Single" or i == 0:
                check_result(got, ["k"] if keys else [], want, _names(aggs), 1e-12 if mode == "Single" else 1e-5 if keys <= 3 else 1e-3)
            else:
                # a covariance near 0 has no relative bound: the states' rounding is measured against sqrt(var x * var y),
                # and corr (within [-1, 1]) absolutely
                spread = grouped_exact(pa.Table.from_batches([b]), ["k"] if keys else [], [("var", "x", None, "vx"), ("var", "y", None, "vy")])
                assert got.num_rows == len(want)
                for r in got.to_pylist():
                    g = (r["k"],) if keys else ()
                    tol = 1e-5 if keys <= 3 else 1e-3
                    assert abs(r["cv"] - want[g]["cv"]) <= tol * math.sqrt(spread[g]["vx"] * spread[g]["vy"]), (g, r, want[g])
                    assert abs(r["cr"] - want[g]["cr"]) <= tol, (g, r, want[g])
            sink = "pipeline_agg_global" if keys > 4 else "pipeline_agg_reg"
            assert sink in ks and sink + "_pass2" in ks, ks


def _lineitem(gpu, oracle, msf=10, parts=2):
    """TPC-H lineitem at msf / 1000 of scale factor 1, generated by the CPU oracle and registered on the device as batches"""
    import oracle_ffi
    cols = ["l_suppkey", "l_quantity", "l_extendedprice", "l_discount", "l_returnflag", "l_linestatus"]
    n = oracle_ffi.lib().oracle_tpch_table_rows(b"lineitem", msf)
    bounds = [n * p // parts for p in range(parts + 1)]
    oracle.drop_table("lineitem")
    gpu.drop_table("li")
    batches = []
    for p in range(parts):
        oracle.tpch_generate("lineitem", msf, p, bounds[p], bounds[p + 1], cols)
        batches.append(oracle.export_table("lineitem", p))
        gpu.register_batch("li", p, batches[-1])
    return pa.Table.from_batches(batches), batches


def test_lineitem_sinks_modes_and_mixed(timed, oracle):
    gpu = timed
    table, batches = _lineitem(gpu, oracle)
    sch = [P.field(f.name, P.dec(f.type.precision, f.type.scale) if pa.types.is_decimal(f.type) else
                   {"int64": "i64", "int32": "i32", "string": "utf8"}[str(f.type)], f.nullable) for f in batches[0].schema]
    aggs = [("stddev", c("l_extendedprice"), None, "sd"), ("var_pop", c("l_quantity"), None, "vp"),
            ("corr", c("l_quantity"), c("l_extendedprice"), "cr"), ("covar_pop", c("l_discount"), c("l_extendedprice"), "cp")]
    exact_aggs = [("stddev", "l_extendedprice", None, "sd"), ("var_pop", "l_quantity", None, "vp"),
                  ("corr", "l_quantity", "l_extendedprice", "cr"), ("covar_pop", "l_discount", "l_extendedprice", "cp")]
    q, e, d = (batches[0].schema.field(n).type for n in ("l_quantity", "l_extendedprice", "l_discount"))
    extra = [("sum", c("l_quantity"), "sq", [P.field("sq[sum]", P.dec(min(38, q.precision + 10), q.scale), True)], None),
             ("avg", c("l_extendedprice"), "ae", [P.field("ae[count]", "u64", True), P.field("ae[sum]", P.dec(min(38, e.precision + 10), e.scale), True)],
              P.dec(e.precision, e.scale)),
             ("min", c("l_discount"), "md", [P.field("md[min]", P.dec(d.precision, d.scale), True)], None)]
    shapes = [([(c("l_returnflag"), "rf"), (c("l_linestatus"), "ls")], [P.field("rf", "utf8", False), P.field("ls", "utf8", False)],
               ["l_returnflag", "l_linestatus"], "pipeline_agg_reg"),
              ([(c("l_suppkey"), "sk")], [P.field("sk", "i64", False)], ["l_suppkey"], "pipeline_agg_global"),
              ([], [], [], "pipeline_agg_reg")]
    for keys, kf, knames, sink in shapes:
        want = grouped_exact(table, knames, exact_aggs)
        df_way = grouped_exact(table, knames, exact_aggs, welford)  # what DataFusion's Welford accumulators compute
        names = [k for _, k in keys]
        for mode in ("Single", "Partial"):
            if mode == "Single":
                gpu.drop_table("li1")
                gpu.register_batch("li1", 0, pa.Table.from_batches(batches).combine_chunks().to_batches()[0])
            src = P.scan("li1" if mode == "Single" else "li", sch)
            gpu.kernel_stats(reset=True)
            alone = driver.run_stages(gpu, stat_stages(src, aggs[:3], keys, kf, mode), f"sla-{len(keys)}-{mode}")
            ks = gpu.kernel_stats()
            check_result(alone, names, want, ["sd", "vp", "cr"], 1e-10)
            check_result(alone, names, df_way, ["sd", "vp", "cr"], 1e-10)
            assert sink in ks and sink + "_pass2" in ks, ks
            assert "pipeline_fused_agg" not in ks and "groupby_hash_agg" not in ks, ks
            # mixed with SUM / AVG / MIN in one AggregateExec: more than the register sink's six accumulators, so this
            # one may run on the global table, whatever its group count
            mixed = [aggs[0], aggs[2]]
            got = driver.run_stages(gpu, stat_stages(src, mixed, keys, kf, mode, extra=extra), f"sli-{len(keys)}-{mode}")
            renamed = {tuple(r[n] for n in names): r for r in got.to_pylist()}
            assert got.num_rows == len(want), (got.num_rows, len(want))
            for g, w in want.items():
                r = renamed[g]
                for nm in ("sd", "cr"):
                    assert rel_close(r[nm], w[nm], 1e-10), (g, nm, r[nm], w[nm])
            # the existing aggregates in the same AggregateExec against pyarrow
            tk = table.group_by(knames).aggregate([("l_quantity", "sum"), ("l_extendedprice", "mean"), ("l_discount", "min")]) if knames else None
            if tk is not None:
                ref = {tuple(r[k] for k in knames): r for r in tk.to_pylist()}
                for g, r in renamed.items():
                    assert r["sq"] == ref[g]["l_quantity_sum"] and r["md"] == ref[g]["l_discount_min"], g
                    assert abs(float(r["ae"]) - float(ref[g]["l_extendedprice_mean"])) < 1e-2, g


def test_empty_input_and_all_null(gpu):
    sch = UNIT_SCHEMA
    empty = pa.record_batch([pa.array([], pa.int32()), pa.array([], pa.float64()), pa.array([], pa.float64())], names=["k", "x", "y"])
    for mode in ("Single", "Partial"):
        _register(gpu, "se", empty, 1 if mode == "Single" else 2)
        for i, aggs in enumerate(_agg_sets()):
            got = driver.run_stages(gpu, stat_stages(P.scan("se", sch), aggs, [], [], mode), f"se-{i}-{mode}")
            assert got.num_rows == 1 and all(v is None for v in got.to_pylist()[0].values())
            got = driver.run_stages(gpu, stat_stages(P.scan("se", sch), aggs, [(c("k"), "k")], [P.field("k", "i32", False)], mode), f"se-k-{i}-{mode}")
            assert got.num_rows == 0
    nulls = pa.record_batch([pa.array([1, 1, 2], pa.int32()), pa.array([None, None, 1.0], pa.float64()), pa.array([None, 2.0, None], pa.float64())],
                            names=["k", "x", "y"])
    _run_modes(gpu, "sn", nulls, sch, [(c("k"), "k")], [P.field("k", "i32", False)], _agg_sets(), 1e-12, "sn")


def test_reference_goldens(gpu):
    """context_basic.rs:329-438, run as the reference does: Partial over two partitions, then Final"""
    t = G.load("alltypes_plain")
    gold = json.load(open(G.__file__.replace("golden_data.py", "golden/reference_stat_aggregates.json")))["cases"]
    sch = G.ir_schema("alltypes_plain")
    G.register(gpu, "test", t, 2)
    for i, g in enumerate(gold):  # one query each, as the reference runs them
        agg = (g["fn"], c(g["args"][0]), c(g["args"][1]) if len(g["args"]) > 1 else None, "r")
        got = driver.run_stages(gpu, stat_stages(P.scan("test", sch), [agg], mode="Partial"), f"sgold-{i}").to_pylist()[0]["r"]
        assert math.isclose(got, g["value"], rel_tol=1e-12, abs_tol=0), (g, got)
