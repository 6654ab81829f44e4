"""MIN / MAX over Utf8 and UInt64 on the device, in every aggregate mode, on both VM aggregate sinks (register sink for a
few groups, global hash table for many), against the CPU oracle and pyarrow: Utf8 columns from Arrow batches (offsets),
from Parquet (BYTE_ARRAY views) and from string expressions; the compare-and-swap worst cases at one group; results that
outlive their input; UInt64 states across 2^63, including states read from a shuffle file pyarrow wrote."""
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from ballista_b200 import driver
from ballista_b200 import plan as P
from ballista_b200.plan import Stage
from test_oracle_minmax import AGGS, SCHEMA, minmax_batch, minmax_stages, pyarrow_minmax
from util import assert_tables_equal

pytestmark = pytest.mark.gpu
c = P.col


def _register(engines, table, batch, parts=2):
    step = (batch.num_rows + parts - 1) // parts
    for e in engines:
        e.drop_table(table)
        for p in range(parts):
            e.register_batch(table, p, batch.slice(p * step, step))


def _run(gpu, oracle, stages, job, want=None):
    gpu.kernel_stats(reset=True)
    got = driver.run_stages(gpu, stages, job)
    ks = gpu.kernel_stats()
    ref = driver.run_stages(oracle, stages, job)
    assert_tables_equal(got, ref)
    if want is not None:
        assert_tables_equal(got, want)
    return ks, got


@pytest.fixture()
def timed(gpu):
    gpu.set_config("b200.metrics.kernel_timing", "on")
    yield gpu
    gpu.set_config("b200.metrics.kernel_timing", "off")


# n_keys = 3: keys 0, 1, 2 and NULL -- the register sink's four groups.  MIN + MAX + COUNT(*) + the non-NULL count of a
# nullable column are four accumulators: one column at a time fits the register sink's six.
@pytest.mark.parametrize("n_keys,sink,agg_sets", [(3, "pipeline_agg_reg", [AGGS[:2], AGGS[2:]]), (150000, "pipeline_agg_global", [AGGS])])
def test_minmax_all_modes_both_sinks(timed, oracle, n_keys, sink, agg_sets):
    gpu = timed
    n = 400000 if n_keys > 4 else 60000
    b = minmax_batch(n, 21, n_keys=n_keys)
    _register((gpu, oracle), "mm", b)
    _register((gpu, oracle), "mm1", b, parts=1)
    for aggs in agg_sets:
        # (the scalar form of the seven-accumulator set is one group on the global table: its UInt64 MIN / MAX then
        # serialise on the 128-bit integer lock of that one cell, which is slow and not what this test is about)
        for keyed in ((True, False) if len(aggs) == 2 else (True,)):
            want = pyarrow_minmax(b, keyed, aggs)
            for mode, table in (("Single", "mm1"), ("Partial", "mm")):
                job = f"g-{n_keys}-{aggs[0][1]}-{keyed}-{mode}"
                ks, _ = _run(gpu, oracle, minmax_stages(keyed, mode, P.scan(table, SCHEMA), aggs), job, want)
                assert "groupby_hash_agg" not in ks and "pipeline_fused_agg" not in ks, ks
                assert sink in ks, ks


def test_minmax_parquet_strings(timed, oracle, tmp_path):
    """BYTE_ARRAY columns decoded on the device arrive as string views, not Arrow offsets"""
    gpu = timed
    b = minmax_batch(30000, 22).select(["k", "s"])
    path = str(tmp_path / "mm.parquet")
    pq.write_table(pa.Table.from_batches([b]), path, row_group_size=7000)
    gpu.drop_table("mmpq")
    gpu.register_parquet("mmpq", 0, path)
    oracle.drop_table("mmpq")
    oracle.register_batch("mmpq", 0, b)
    for keyed in (True, False):
        for mode in ("Single", "Partial"):
            _run(gpu, oracle, minmax_stages(keyed, mode, P.scan("mmpq", SCHEMA[:2]), AGGS[:2]), f"pq-{keyed}-{mode}", pyarrow_minmax(b, keyed, AGGS[:2]))


def test_minmax_over_string_expressions(timed, oracle):
    """substr() makes new views into the input; a CASE with a literal branch points results at the literal, which lives
    in the aggregate's own pipeline (U+10FFFF orders above every other string, so MAX of group 1 is the literal)"""
    gpu = timed
    b = minmax_batch(50000, 23)
    _register((gpu, oracle), "mme", b)
    sub = P.fn("substr", c("s"), P.lit_i64(2), P.lit_i64(3))
    cas = P.case([[P.binop("=", c("k"), P.lit_i32(1)), P.lit_utf8("\U0010ffff lit")]], c("s"))
    src = P.project([(c("k"), "k"), (sub, "s"), (c("u"), "u")], P.scan("mme", SCHEMA))
    src2 = P.project([(c("k"), "k"), (cas, "s"), (c("u"), "u")], P.scan("mme", SCHEMA))
    for name, s in (("substr", src), ("case", src2)):
        for keyed in (True, False):
            _run(gpu, oracle, minmax_stages(keyed, "Partial", s), f"ex-{name}-{keyed}")
    # the same expressions straight inside the aggregate, many groups (global sink)
    _register((gpu, oracle), "mme2", minmax_batch(300000, 26, n_keys=120000), parts=1)
    aggs = [P.agg("max", sub, "mx_sub"), P.agg("min", sub, "mn_sub"), P.agg("max", cas, "mx_case"), P.agg("min", cas, "mn_case")]
    st = [Stage(1, P.shuffle_writer(P.aggregate("Single", [(c("k"), "k")], aggs, P.scan("mme2", SCHEMA)), 1))]
    ks, _ = _run(gpu, oracle, st, "ex-inline")
    assert "pipeline_agg_global" in ks, ks


def _one_group(gpu, oracle, strings, job, global_sink):
    """A few million rows into one group.  Seven accumulators do not fit the register sink: the global table then takes
    every row, all of them contending for the same string cells."""
    b = pa.record_batch([strings, pc.utf8_reverse(strings)], names=["s", "r"])
    _register((gpu, oracle), "one", b, parts=1)
    sch = [P.field("s", "utf8"), P.field("r", "utf8")]
    aggs = [P.agg("max", c("s"), "mx"), P.agg("min", c("s"), "mn")]
    if global_sink:
        tail = P.fn("substr", c("s"), P.lit_i64(2), P.lit_i64(100))
        aggs += [P.agg("max", c("r"), "mxr"), P.agg("min", c("r"), "mnr"), P.agg("max", tail, "mxt"), P.agg("min", tail, "mnt")]
    st = [Stage(1, P.shuffle_writer(P.aggregate("Single", [], aggs, P.scan("one", sch)), 1))]
    ks, got = _run(gpu, oracle, st, job)
    assert ("pipeline_agg_global" if global_sink else "pipeline_agg_reg") in ks, ks
    assert got.column("mx")[0].as_py() == pc.max(strings).as_py() and got.column("mn")[0].as_py() == pc.min(strings).as_py()


@pytest.mark.parametrize("global_sink", [False, True])
def test_cas_worst_cases_at_one_group(timed, oracle, global_sink):
    n = 3_000_000
    same = pa.array(np.full(n, "the same long string, equal over its full length: " + "q" * 40, dtype=object), pa.utf8())
    _one_group(timed, oracle, same, f"same-{global_sink}", global_sink)
    ascending = pc.utf8_lpad(pc.cast(pa.array(np.arange(n)), pa.utf8()), 12, "0")   # every row improves MAX
    _one_group(timed, oracle, ascending, f"asc-{global_sink}", global_sink)


def test_results_outlive_their_input(gpu, oracle):
    """Partial stage, drop the input (and reuse its memory), then Final over the stored states: end to end, the results
    do not depend on the input once its stage has run"""
    b = minmax_batch(80000, 24)
    for keyed in (True, False):
        _register((gpu, oracle), "life", b)
        stages = minmax_stages(keyed, "Partial", P.scan("life", SCHEMA))
        job = f"life-{keyed}"
        for e in (gpu, oracle):
            q = e.create_query_stage_exec(job, 1, stages[0].json(job))
            for p in range(2):
                q.execute_query_stage(p)
            q.release()
            e.drop_table("life")
        _register((gpu,), "filler", minmax_batch(80000, 99))   # overwrite what the dropped input occupied
        st2 = stages[1]
        n2 = st2.n_tasks or 3   # keyed: one task per hash partition of stage 1
        for e in (gpu, oracle):
            q = e.create_query_stage_exec(job, 2, st2.json(job))
            for p in range(n2):
                q.execute_query_stage(p)
            q.release()
        got = pa.Table.from_batches([gpu.partition_export(job, 2, p) for p in range(n2) if gpu.partition_rows(job, 2, p) >= 0])
        want = pa.Table.from_batches([oracle.partition_export(job, 2, p) for p in range(n2) if oracle.partition_rows(job, 2, p) >= 0])
        assert_tables_equal(got, want)
        assert_tables_equal(got, pyarrow_minmax(b, keyed))
        gpu.drop_table("filler")


def test_u64_final_over_states_from_a_pyarrow_file(gpu, tmp_path):
    """UInt64 states on both sides of 2^63 written by pyarrow as a shuffle file, merged by FinalPartitioned"""
    big = [2**63 - 1, 2**63, 2**64 - 1, 0, 1, 2**63 + 5]
    rng = np.random.default_rng(25)
    n = 3000
    k = pa.array(rng.integers(0, 40, n).astype(np.int32))
    mn = pa.array([None if rng.random() < 0.1 else big[i] for i in rng.integers(0, len(big), n)], pa.uint64())
    mx = pa.array([None if rng.random() < 0.1 else big[i] for i in rng.integers(0, len(big), n)], pa.uint64())
    states = pa.record_batch([k, mn, mx], names=["k", "m[min]", "x[max]"])
    part = [P.field("k", "i32", True), P.field("m[min]", "u64", True), P.field("x[max]", "u64", True)]
    st = Stage(2, P.shuffle_writer(P.aggregate("FinalPartitioned", [(c(0), "k")], [P.agg("min", None, "m"), P.agg("max", None, "x")],
                                                P.shuffle_reader(1, part)), 2))
    job = "u64-file"
    path = os.path.join(str(tmp_path), "data-0.arrow")
    with pa.ipc.new_stream(path, states.schema, options=pa.ipc.IpcWriteOptions(compression="lz4")) as w:
        w.write_batch(states)
    gpu.shuffle_read_file(job, 1, 0, 0, path)
    q = gpu.create_query_stage_exec(job, 2, st.json(job))
    q.execute_query_stage(0)
    q.release()
    got = pa.Table.from_batches([gpu.partition_export(job, 2, 0)])
    g = pa.Table.from_batches([states]).group_by("k").aggregate([("m[min]", "min"), ("x[max]", "max")])
    want = pa.table([g["k"], g["m[min]_min"], g["x[max]_max"]], names=["k", "m", "x"])
    assert_tables_equal(got, want)
    gpu.remove_job_data(job)
