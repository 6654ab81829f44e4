"""The fixed cost of a q1 step after its stage-1 kernel: host waits and kernel launches per warm step, and the parsed-plan
cache of b200_stage_prepare (a stage plan seen before, under another job id, is not parsed again).
  * not gpu: every wait on the stream inside a task, an exchange or an export goes through the counting helper; the
    ctypes output arrays of the stage calls are reused per thread, not allocated per stage;
  * gpu: a warm q1 step at SF1 keeps to its budget of host waits and launches; jobs that share cached plans compute what
    the CPU oracle computes, store under their own job and stage ids, report the same metrics, and still fail, cancel and
    reject malformed plans as an uncached plan does."""
import ctypes as C
import os
import re
import threading

import pyarrow as pa
import pytest

from ballista_b200 import engine, tpch
from util import assert_tables_equal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENGINE_CPP = os.path.join(ROOT, "datafusion-ballista_b200", "csrc", "host", "engine.cpp")

MSF = 1000   # SF1 lineitem: 5,999,989 rows

# Per warm q1 step (3 stages, one task each, then the export of the result), measured on an H100 80GB HBM3.  Both are
# what the build before the plan cache did too (9 cudaStreamSynchronize calls and 14 launches per step under
# torch.profiler): the cache and the reused output arrays remove host work between the waits, not waits or launches.
# Among the waits: one after each aggregate kernel (its group count and status), each writer's final sync, and the
# export's single read-back.
Q1_STEP_HOST_WAITS = 9
Q1_STEP_LAUNCHES = 14


def test_task_waits_go_through_the_counting_helper():
    src = open(ENGINE_CPP).read()
    assert "inline cudaError_t host_wait(b200_engine* e, cudaStream_t st)" in src
    # Exec::sync, the waits of do_sort / the window operator / the export download / the exchange, and the unwinding of a
    # failed task all call host_wait; raw waits remain only on ingest, engine lifecycle and diagnostic paths
    sync_body = re.search(r"void sync\(\) const \{(.*?)\n  \}", src, re.S).group(1)
    assert "host_wait(e, st())" in sync_body and "cudaStreamSynchronize" not in sync_body
    for fn in ("do_sort", "exec_window", "download_batch"):
        body = re.search(r"\b" + fn + r"\(.*?\n  ?\}\n", src, re.S).group(0)
        assert "cudaStreamSynchronize" not in body, fn


def test_output_arrays_are_reused_per_thread():
    # execute_query_stage / collect_plan_metrics copy their results out of these arrays before returning, so one of each
    # per thread is enough; another thread (another task running concurrently) gets its own
    a, m = engine._partition_buffer(), engine._metrics_buffer()
    assert engine._partition_buffer() is a and engine._metrics_buffer() is m
    assert len(a) >= 4096 and len(m) == engine._METRICS_CAP
    other = []
    t = threading.Thread(target=lambda: other.append((engine._partition_buffer(), engine._metrics_buffer())))
    t.start()
    t.join()
    assert other[0][0] is not a and other[0][1] is not m


def _step(eng, stages, job):
    for st in stages:
        q = eng.create_query_stage_exec(job, st.stage_id, st.json(job))
        q.execute_query_stage(0)
        q.release()
    res = eng.partition_export(job, 3, 0)
    eng.remove_job_data(job)
    return pa.Table.from_batches([res])


@pytest.fixture()
def q1_sf1(gpu, oracle):
    n = engine.GpuExecutionEngine.tpch_table_rows("lineitem", MSF)
    gpu.drop_table("lineitem")
    for e in (gpu, oracle):
        e.tpch_generate("lineitem", MSF, 0, 0, n, tpch.Q1_COLUMNS)
    stages = tpch.q1(1)
    want = _step(oracle, stages, "tail-oracle")
    return gpu, stages, want


@pytest.mark.gpu
def test_warm_q1_step_budget(q1_sf1):
    gpu, stages, want = q1_sf1
    for w in range(3):
        _step(gpu, stages, f"tail-warm{w}")
    steps = 4
    s0, l0 = gpu.counter("host_syncs"), gpu.kernel_launches()
    for k in range(steps):
        got = _step(gpu, stages, f"tail-step{k}")
    waits, launches = (gpu.counter("host_syncs") - s0) / steps, (gpu.kernel_launches() - l0) / steps
    print(f"per warm q1 step: {waits} host waits, {launches} kernel launches")
    assert_tables_equal(got, want, sort=False)
    assert waits == Q1_STEP_HOST_WAITS
    assert launches == Q1_STEP_LAUNCHES


def _metrics(q):
    return [(m["name"], m["output_rows"], m["input_rows"], m["bytes_written"], m["kernel_launches"]) for m in q.collect_plan_metrics()]


@pytest.mark.gpu
def test_cached_plans_keep_results_ids_and_metrics(q1_sf1):
    gpu, stages, want = q1_sf1
    _step(gpu, stages, "tail-warm")   # settles the aggregate strategy (a first run also samples the keys)
    seen = []
    for job in ("tail-first", "tail-second"):   # the second job's stage plans differ from the first's only in the job id
        per_job = []
        for st in stages:
            q = gpu.create_query_stage_exec(job, st.stage_id, st.json(job))
            parts = q.execute_query_stage(0)
            per_job.append(([(p.partition_id, p.num_rows, p.num_bytes) for p in parts], _metrics(q)))
            q.release()
        got = pa.Table.from_batches([gpu.partition_export(job, 3, 0)])
        assert_tables_equal(got, want, sort=False)
        seen.append(per_job)
    assert seen[0] == seen[1]
    for name, out_rows, _, _, _ in seen[1][0][1]:
        if name == "AggregateExec":
            assert out_rows == 4
    # the first job's outputs are its own: removing them leaves the second's in place
    gpu.remove_job_data("tail-first")
    assert gpu.partition_rows("tail-first", 3, 0) < 0
    assert gpu.partition_rows("tail-second", 3, 0) == want.num_rows
    gpu.remove_job_data("tail-second")
    # the cached stage-3 plan text prepared under another stage id stores under that id
    for stage_id, st in ((1, stages[0]), (2, stages[1]), (7, stages[2])):
        q = gpu.create_query_stage_exec("tail-other", stage_id, st.json("tail-other"))
        q.execute_query_stage(0)
        q.release()
    assert gpu.partition_rows("tail-other", 7, 0) == want.num_rows
    assert gpu.partition_rows("tail-other", 3, 0) < 0
    gpu.remove_job_data("tail-other")


@pytest.mark.gpu
def test_cached_plans_fail_and_cancel_like_fresh_ones(q1_sf1):
    gpu, stages, want = q1_sf1
    _step(gpu, stages, "tail-prime")   # every stage plan of q1 is now cached
    # cancelled before it starts: B200_ERR_CANCELLED, nothing stored
    flag = C.c_int32(1)
    q = gpu.create_query_stage_exec("tail-cancel", 1, stages[0].json("tail-cancel"))
    with pytest.raises(engine.B200Error) as ex:
        q.execute_query_stage(0, cancel_flag=flag)
    q.release()
    assert ex.value.code == -6
    assert gpu.partition_rows("tail-cancel", 1, 0) < 0
    # a malformed plan is rejected on every call: failures are never cached
    bad = stages[0].json("tail-bad").replace('ShuffleWriterExec"', 'NoSuchExec"')
    for _ in range(2):
        with pytest.raises(engine.B200Error) as ex:
            gpu.create_query_stage_exec("tail-bad", 1, bad)
        assert ex.value.code == -1
    # a stage whose kernel overflows (ABS of the smallest Int64) fails with B200_ERR_EXECUTION on a cached plan too, and
    # stores nothing
    P = tpch.P
    gpu.register_batch("tail_ovf", 0, pa.record_batch([pa.array([1, -(2 ** 63), 5] * 700, type=pa.int64())], names=["v"]))
    plan = P.project([(P.fn("abs", P.col("v")), "a")], P.scan("tail_ovf", [P.field("v", "i64", True)]))
    st = P.Stage(1, P.shuffle_writer(plan, 1))
    for job in ("tail-ovf1", "tail-ovf2"):
        q = gpu.create_query_stage_exec(job, 1, st.json(job))
        with pytest.raises(engine.B200Error) as ex:
            q.execute_query_stage(0)
        q.release()
        assert ex.value.code == -3, str(ex.value)
        assert gpu.partition_rows(job, 1, 0) < 0
    gpu.drop_table("tail_ovf")
    # and the engine keeps working
    assert_tables_equal(_step(gpu, stages, "tail-after"), want, sort=False)
