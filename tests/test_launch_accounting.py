"""Kernel launches are counted where they are enqueued: every launch of the device module goes through
launch_kernel (csrc/device/kernels.h), which bumps a per-thread counter; the engine-wide count and every operator's
kernel_launches are differences of that counter, never hand-written numbers.
  * not gpu: the sources keep to that rule;
  * gpu: the per-operator counts of every stage add up to what the engine counted for it."""
import os
import re

import pyarrow as pa
import pytest

from ballista_b200 import driver, tpch
from test_tpch_queries import load_tables

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "datafusion-ballista_b200", "csrc")
DEVICE = os.path.join(CSRC, "device")


def _read(path):
    with open(path) as f:
        return f.read()


def test_every_launch_goes_through_the_counting_helper():
    sources = sorted(f for f in os.listdir(DEVICE) if f.endswith((".cu", ".cuh", ".h")))
    assert "kernels.cu" in sources
    raw = []
    for f in sources:
        for no, line in enumerate(_read(os.path.join(DEVICE, f)).splitlines(), 1):
            if "<<<" in line:
                raw.append((f, no, line.strip()))
    # the single launch inside launch_kernel itself
    assert len(raw) == 1 and raw[0][0] == "kernels.h" and raw[0][2].startswith("kernel<<<"), raw
    h = _read(os.path.join(DEVICE, "kernels.h"))
    assert "inline void launch_kernel(" in h
    # no launcher reports its own launch count
    assert not re.search(r"\buint64_t\*\s*launches\b", h)
    assert not re.search(r"^uint64_t\s+launch_", h, re.M)


def test_engine_states_no_launch_counts():
    src = _read(os.path.join(CSRC, "host", "engine.cpp"))
    hand = re.compile(r"\bx\.count\(|\bExec::count\b|\bvoid count\(|->launches\s*(\+\+|\+=\s*\d)")
    found = [line.strip() for line in src.splitlines() if hand.search(line)]
    assert not found, found


class _CountingEngine:
    """The engine as driver.run_stages sees it, recording by how much the engine-wide launch counter grows across
    each stage's b200_stage_execute calls."""

    def __init__(self, engine):
        self.engine = engine
        self.launches = {}

    def __getattr__(self, name):
        return getattr(self.engine, name)

    def create_query_stage_exec(self, job_id, stage_id, plan):
        qse = self.engine.create_query_stage_exec(job_id, stage_id, plan)
        run = qse.execute_query_stage

        def counted(partition, *args):
            l0 = self.engine.kernel_launches()
            out = run(partition, *args)
            self.launches[stage_id] = self.launches.get(stage_id, 0) + self.engine.kernel_launches() - l0
            return out

        qse.execute_query_stage = counted
        return qse


def _run(engine, stages, job):
    ce = _CountingEngine(engine)
    metrics = []
    driver.run_stages(ce, stages, job, collect=False, metrics_out=metrics)
    assert len(metrics) == len(stages)
    for stage_id, ops in metrics:
        assert ce.launches[stage_id] > 0
        assert sum(m["kernel_launches"] for m in ops) == ce.launches[stage_id], (stage_id, ops)
    return {stage_id: ops for stage_id, ops in metrics}


def _launches(ops, name):
    got = [m["kernel_launches"] for m in ops if m["name"] == name]
    assert got, (name, ops)
    return got


def _writer_launches(ops):
    assert ops[0]["name"].endswith("ShuffleWriterExec"), ops[0]   # the stage's root comes first (pre-order)
    return ops[0]["kernel_launches"]


@pytest.mark.gpu
def test_q1_operator_launches(gpu, oracle_lib):
    n = oracle_lib.lib().oracle_tpch_table_rows(b"lineitem", 20)
    gpu.drop_table("lineitem")
    gpu.tpch_generate("lineitem", 20, 0, 0, n // 2, tpch.Q1_COLUMNS)
    gpu.tpch_generate("lineitem", 20, 1, n // 2, n, tpch.Q1_COLUMNS)
    ops = _run(gpu, tpch.q1(4), "launches-q1")
    # stage 1: the filter and the projection run fused into the aggregate's kernel and are charged to it
    assert all(k > 0 for k in _launches(ops[1], "AggregateExec"))
    assert _writer_launches(ops[1]) > 0   # hash repartition
    for name in ("FilterExec", "ProjectionExec", "DataSourceExec"):
        assert _launches(ops[1], name) == [0]
    assert all(k > 0 for k in _launches(ops[2], "AggregateExec"))
    assert all(k > 0 for k in _launches(ops[3], "SortPreservingMergeExec"))


@pytest.mark.gpu
def test_q3_operator_launches(gpu, oracle, oracle_lib):
    load_tables(gpu, oracle_lib, 20, tpch.Q3_TABLES, 2)
    load_tables(oracle, oracle_lib, 20, {"customer": tpch.Q3_TABLES["customer"]}, 2)
    seg = pa.Table.from_batches([oracle.export_table("customer", 0)]).slice(0, 1).to_pylist()[0]["c_mktsegment"]
    ops = _run(gpu, tpch.q3(3, seg), "launches-q3")
    for stage_id in (1, 2, 3, 4, 5):   # hash repartitions
        assert _writer_launches(ops[stage_id]) > 0
    for stage_id in (3, 5):
        assert all(k > 0 for k in _launches(ops[stage_id], "HashJoinExec"))
    assert all(k > 0 for k in _launches(ops[5], "AggregateExec"))
    assert all(k > 0 for k in _launches(ops[6], "SortExec"))
    assert all(k > 0 for k in _launches(ops[7], "SortPreservingMergeExec"))
