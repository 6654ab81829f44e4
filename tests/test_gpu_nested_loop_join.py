"""GPU: NestedLoopJoinExec on the device (csrc/device/nlj.cu) against the CPU oracle.  The output order is deterministic
(pairs by probe row, build rows in order inside a probe row, then unmatched build rows, then unmatched probe rows), so
results are compared in order."""
import base64
import ctypes as C
import json
import os
import threading

import pyarrow as pa
import pytest

import ballista_b200 as bb
from ballista_b200 import driver, tpch
from ballista_b200 import plan as P
from test_tpch_queries import load_tables
from util import assert_tables_equal
import nlj_cases as N

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _both(gpu, oracle, left, right, jt, filt, projection=None, probe_parts=1, job="nlj"):
    for e in (gpu, oracle):
        N.register(e, left, right, probe_parts)
    got = N.run_join(gpu, job, jt, filt, projection)
    want = N.run_join(oracle, job, jt, filt, projection)
    return got, want


def _assert_same(got, want):
    assert N.same_rows(N.rows_of(got), N.rows_of(want))


@pytest.fixture(scope="module")
def tables():
    return N.make_table(300, seed=11), N.make_table(700, seed=12)


@pytest.mark.parametrize("jt", N.JOIN_TYPES)
@pytest.mark.parametrize("fname", sorted(N.FILTERS))
def test_device_matches_oracle(gpu, oracle, tables, jt, fname):
    got, want = _both(gpu, oracle, *tables, jt, N.FILTERS[fname], job=f"g-{jt}-{fname}")
    _assert_same(got, want)


@pytest.mark.parametrize("jt", N.JOIN_TYPES)
@pytest.mark.parametrize("shape", ["empty_build", "empty_probe", "one_row_build"])
def test_edge_sizes(gpu, oracle, jt, shape):
    nb, np_ = {"empty_build": (0, 900), "empty_probe": (70, 0), "one_row_build": (1, 4000)}[shape]
    for fname in ("none", "int_lt", "mixed"):
        got, want = _both(gpu, oracle, N.make_table(nb, seed=5), N.make_table(np_, seed=6), jt, N.FILTERS[fname], job=f"e-{shape}-{jt}-{fname}")
        _assert_same(got, want)


@pytest.mark.parametrize("jt", ["Inner", "Full", "LeftSemi", "RightAnti"])
def test_projection(gpu, oracle, tables, jt):
    proj = None if jt.endswith("Semi") or jt.endswith("Anti") else [N.NC + 1, 0, 6]
    got, want = _both(gpu, oracle, *tables, jt, N.FILTERS["band"], proj, job=f"p-{jt}")
    _assert_same(got, want)


def _int_tables(nb, np_, seed):
    import numpy as np
    r = np.random.default_rng(seed)
    b = pa.table({"x": pa.array(r.integers(0, 10000, nb), pa.int64())})
    p = pa.table({"y": pa.array(r.integers(0, 10000, np_), pa.int64())})
    return b, p


@pytest.mark.parametrize("sel", ["1pct", "all"])
def test_crosses_shared_memory_tiles(gpu, oracle, sel):
    """5,000 build rows (20 shared-memory tiles) x 20,000 probe rows, at about 1 % and at 100 % selectivity."""
    b, p = _int_tables(5000, 20000, 3)
    sch = [P.field("x", "i64", True)]
    psch = [P.field("y", "i64", True)]
    filt = None if sel == "all" else P.and_(P.binop(">=", P.col(1), P.col(0)), P.binop("<", P.col(1), P.binop("+", P.col(0), P.lit_i64(100))))
    plan = [P.Stage(1, P.shuffle_writer(P.nested_loop_join(P.scan("nlj_b", sch), P.scan("nlj_p", psch), "Left", filter=filt), 1))]
    for e in (gpu, oracle):
        for t, data in (("nlj_b", b), ("nlj_p", p)):
            try:
                e.drop_table(t)
            except Exception:
                pass
            e.register_batch(t, 0, data.to_batches()[0])
    gpu.set_config("b200.metrics.kernel_timing", "1")
    gpu.kernel_stats(reset=True)
    got = driver.run_stages(gpu, plan, f"tiles-{sel}")
    ks = gpu.kernel_stats(reset=True)
    gpu.set_config("b200.metrics.kernel_timing", "0")
    want = driver.run_stages(oracle, plan, f"tiles-{sel}")
    assert_tables_equal(got, want, sort=False)
    assert "nlj_count" in ks and "nlj_write" in ks and "join_probe" not in ks
    if sel == "all":
        assert got.num_rows == 5000 * 20000


def test_one_row_build_against_3m_probe_rows(gpu, oracle):
    import numpy as np
    r = np.random.default_rng(7)
    b = pa.table({"avg": pa.array([0.25], pa.float64())})
    vals = r.random(3_000_000)
    vals[::97] = np.nan
    p = pa.table({"k": pa.array(np.arange(3_000_000), pa.int64()), "v": pa.array(vals, pa.float64(), mask=(np.arange(3_000_000) % 101 == 0))})
    sch_b = [P.field("avg", "f64", True)]
    sch_p = [P.field("k", "i64", True), P.field("v", "f64", True)]
    j = P.nested_loop_join(P.scan("nlj_b", sch_b), P.scan("nlj_p", sch_p), "Inner", filter=P.binop(">", P.col(2), P.col(0)), projection=[1, 2])
    plan = [P.Stage(1, P.shuffle_writer(j, 1))]
    for e in (gpu, oracle):
        for t, data in (("nlj_b", b), ("nlj_p", p)):
            try:
                e.drop_table(t)
            except Exception:
                pass
            e.register_batch(t, 0, data.to_batches()[0])
    before = gpu.counter("nlj_pairs")
    got = driver.run_stages(gpu, plan, "scalar")
    want = driver.run_stages(oracle, plan, "scalar")
    assert_tables_equal(got, want, sort=False)
    assert gpu.counter("nlj_pairs") - before == 3_000_000


with open(os.path.join(HERE, "golden", "nlj_proto_plans.json")) as fh:
    PROTO = {c["name"]: base64.b64decode(c["proto_b64"]) for c in json.load(fh)["cases"]}


class _FromProto:
    def __init__(self, eng, query):
        self._e, self._q = eng, query

    def __getattr__(self, name):
        return getattr(self._e, name)

    def create_query_stage_exec(self, job_id, stage_id, plan_json):
        return self._e.create_query_stage_exec_proto(job_id, stage_id, PROTO[f"{self._q}_nlj/stage{stage_id}"])


@pytest.mark.parametrize("q", ["q11", "q22"])
def test_tpch_nlj_end_to_end(gpu, oracle, oracle_lib, q):
    """q11_nlj / q22_nlj over 2 partitions, twice each: from the IR text and from the protobuf plan bytes."""
    tables = tpch.union_tables([q])
    for e in (gpu, oracle):
        load_tables(e, oracle_lib, 50, tables, 2)
    want = driver.run_stages(oracle, getattr(tpch, f"{q}_nlj")(4), f"{q}-nlj")
    assert want is not None and want.num_rows > 0
    for run in range(2):
        got = driver.run_stages(gpu, getattr(tpch, f"{q}_nlj")(4), f"{q}-nlj-{run}")
        assert_tables_equal(got, want, sort=False, f64_rtol=1e-12)
        got = driver.run_stages(_FromProto(gpu, q), getattr(tpch, f"{q}_nlj")(4), f"{q}-nlj-pb-{run}")
        assert_tables_equal(got, want, sort=False, f64_rtol=1e-12)


def _refused(gpu, left, right, jt, filt, probe_parts=1, job="refuse"):
    N.register(gpu, left, right, probe_parts)
    with pytest.raises(bb.B200Error) as ei:
        N.run_join(gpu, job, jt, filt)
    return ei.value


def test_refusals_leave_the_engine_working(gpu, oracle, tables):
    left, right = tables
    L, R = N.L, N.R
    e = _refused(gpu, left, right, "Inner", P.binop(">", P.binop("+", L("i"), R("i")), P.lit_i32(3)), job="r1")
    assert e.code == -2 and "mixes both sides" in str(e) and '"bin":"+"' in str(e)
    e = _refused(gpu, left, right, "Left", N.FILTERS["int_lt"], probe_parts=2, job="r2")
    assert e.code == -2 and "more than one probe partition" in str(e)
    many = P.and_(*[P.binop("<", L("i"), P.binop("+", R("i"), P.lit_i32(k))) for k in range(9)])
    e = _refused(gpu, left, right, "Inner", many, job="r3")
    assert e.code == -2 and "more than 8" in str(e)
    e = _refused(gpu, left, right, "Inner", P.binop("<", L("m"), R("m4")), job="r4")
    assert e.code == -2 and "scales" in str(e)
    got, want = _both(gpu, oracle, left, right, "Full", N.FILTERS["mixed"], job="after")
    _assert_same(got, want)


def test_cancelled_task_stores_nothing(gpu, oracle):
    b, p = _int_tables(20000, 2_000_000, 9)
    sch = [P.field("x", "i64", True)]
    psch = [P.field("y", "i64", True)]
    filt = P.binop("=", P.col(0), P.col(1))
    j = P.nested_loop_join(P.scan("nlj_b", sch), P.scan("nlj_p", psch), "Inner", filter=filt)
    st = P.Stage(1, P.shuffle_writer(j, 1))
    for t, data in (("nlj_b", b), ("nlj_p", p)):
        try:
            gpu.drop_table(t)
        except Exception:
            pass
        gpu.register_batch(t, 0, data.to_batches()[0])
    cancelled = False
    for k, delay in enumerate((0.02, 0.005, 0.0)):
        job = f"nlj-cancel{k}"
        flag = C.c_int32(0)
        q = gpu.create_query_stage_exec(job, 1, st.json(job))
        timer = threading.Timer(delay, lambda: setattr(flag, "value", 1))
        timer.start()
        try:
            q.execute_query_stage(0, cancel_flag=flag)
        except bb.B200Error as ex:
            assert ex.code == -6
            cancelled = True
        timer.join()
        q.release()
        if cancelled:
            assert gpu.partition_rows(job, 1, 0) < 0
            break
        gpu.remove_job_data(job)
    assert cancelled
