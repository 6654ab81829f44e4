"""Minimal stand-in for the parts of Ballista that sit ABOVE the execution engine in a test or a
benchmark: it walks a list of stages in dependency order and, per stage, runs one task per input
partition -- what the scheduler's task binding (ballista/scheduler/src/cluster/mod.rs:354,438)
plus ``Executor::execute_query_stage`` (ballista/executor/src/executor.rs:186-212) amount to when
there is one executor.  It is deliberately engine-agnostic (the CPU oracle in tests/ exposes the
same Python surface) and contains no data-path logic.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import pyarrow as pa

from .plan import Stage


def _leaf_info(node: dict):
    """(scan tables, upstream stage ids) reachable from a plan node."""
    tables, readers = [], []
    op = node.get("op")
    if op in ("DataSourceExec", "MemoryScan", "Scan"):
        tables.append(node["table"])
    elif op in ("ShuffleReaderExec", "UnresolvedShuffleExec"):
        readers.append(node["stage_id"])
    for k in ("input", "left", "right"):
        if k in node:
            t, r = _leaf_info(node[k])
            tables += t
            readers += r
    return tables, readers


def _probe_side_leaf(node: dict):
    """The leaf that decides the task count: for a hash join it is the probe (right) side."""
    op = node.get("op")
    if op in ("DataSourceExec", "MemoryScan", "Scan"):
        return ("table", node["table"])
    if op in ("ShuffleReaderExec", "UnresolvedShuffleExec"):
        return ("stage", node["stage_id"])
    if op in ("HashJoinExec", "SortMergeJoinExec", "NestedLoopJoinExec"):
        return _probe_side_leaf(node["right"])
    return _probe_side_leaf(node["input"])


def register_csv_scan(engine, node: dict, partition: int, path_map: Optional[Dict[str, str]] = None) -> None:
    """What an executor-side shim does with a CSV leaf: register file group `partition` of a decoded CSV DataSourceExec
    node (plan IR as the protobuf decoder emits it: "file_groups", "file_ranges", "csv" options) through
    engine.register_csv.  The node's projection indexes the file schema, so the table is registered with the schema's
    columns up to the last projected one, in file order, and the projection applies to it unchanged.  path_map renames
    files (the plan's paths as seen by this host)."""
    schema = node["schema"]
    proj = node.get("projection", list(range(len(schema))))
    cols = [f["name"] for f in schema[:max(proj) + 1]] if proj else []
    ranges = node.get("file_ranges")
    files = []
    for i, path in enumerate(node["file_groups"][partition]):
        path = (path_map or {}).get(path, path)
        r = ranges[partition][i] if ranges else None
        files.append((path, r[0], r[1]) if r else path)
    o = node["csv"]
    engine.register_csv(node["table"], partition, files, schema, columns=cols, has_header=o["has_header"],
                        delimiter=o["delimiter"], quote=o["quote"], escape=o["escape"],
                        newlines_in_values=o["newlines_in_values"])


def run_stages(engine, stages: List[Stage], job_id: str = "job", collect: bool = True,
               metrics_out: Optional[list] = None) -> Optional[pa.Table]:
    """Execute `stages` in order on `engine`; return the last stage's output as one Table."""
    out_parts: Dict[int, int] = {}
    last_stats = []
    for st in stages:
        root = st.plan
        if st.n_tasks is not None:
            n_tasks = st.n_tasks
        else:
            kind, what = _probe_side_leaf(root["input"])
            n_tasks = engine.n_table_partitions(what) if kind == "table" else out_parts[what]
        qse = engine.create_query_stage_exec(job_id, st.stage_id, st.json(job_id))
        stats = []
        for p in range(n_tasks):
            stats += qse.execute_query_stage(p)
        if metrics_out is not None:
            metrics_out.append((st.stage_id, qse.collect_plan_metrics()))
        qse.release()
        part = root.get("partitioning")
        out_parts[st.stage_id] = part["n"] if part else n_tasks
        last_stats = stats
    if not collect:
        return None
    last = stages[-1]
    batches = []
    for p in range(out_parts[last.stage_id]):
        if engine.partition_rows(job_id, last.stage_id, p) >= 0:
            batches.append(engine.partition_export(job_id, last.stage_id, p))
    if not batches:
        return None
    return pa.Table.from_batches(batches)


# ---- one executor per GPU (gang-scheduled stages + NVLink exchange inside the library) ------------------------
REPLICATED_TABLES = {"nation", "region"}   # dimension tables every executor holds in full


def _readers_of(node: dict, stage_id: int, under_merge: bool = False):
    """(broadcast?, under a merge / coalesce?, schema) of every ShuffleReaderExec of `stage_id` below `node`."""
    out = []
    op = node.get("op")
    if op in ("ShuffleReaderExec", "UnresolvedShuffleExec") and node["stage_id"] == stage_id:
        out.append((bool(node.get("broadcast")), under_merge, node["schema"]))
    merge = under_merge or op in ("CoalescePartitionsExec", "SortPreservingMergeExec", "GlobalLimitExec")
    for k in ("input", "left", "right"):
        if k in node:
            out += _readers_of(node[k], stage_id, merge)
    return out


def _fixed_width(schema) -> bool:
    return all(str(f.get("type")).lower() not in ("utf8", "string") for f in schema)


def run_stages_distributed(engine, stages: List[Stage], job_id: str, rank: int, world: int, collect: bool = True,
                           on_stage=None, fused: bool = False) -> Optional[pa.Table]:
    """The same walk as run_stages with one executor per GPU: every rank runs the tasks whose input lives in its HBM,
    and after each stage the engines exchange the stage's output partitions (b200_exchange_stage) according to how
    the consuming stage reads them -- hash repartition (partition p -> rank p % world), merge / single-task consumer
    (everything -> rank 0) or broadcast build side (everything -> everyone).  Returns the result on rank 0."""
    from .engine import EXCHANGE_BROADCAST, EXCHANGE_GATHER, EXCHANGE_HASH
    out_parts: Dict[int, int] = {}
    placement: Dict[int, str] = {}   # stage id -> "hash" | "root" | "all"
    # tables every executor holds in full (the engine's loader says which; tiny tables are replicated whatever their name)
    REPLICATED_TABLES = set(globals()["REPLICATED_TABLES"]) | set(getattr(engine, "replicated_tables", ()))
    for si, st in enumerate(stages):
        root = st.plan
        kind, what = _probe_side_leaf(root["input"])
        if st.n_tasks == 1:
            tasks = [0] if rank == 0 else []
            n_keys = 1
        elif kind == "table":
            n_local = engine.n_table_partitions(what)
            tasks = list(range(n_local)) if (what not in REPLICATED_TABLES or rank == 0) else []
            n_keys = n_local
        else:
            n_up = out_parts[what]
            where = placement[what]
            if where == "hash":
                tasks = [p for p in range(n_up) if p % world == rank]
            elif where == "root":
                tasks = list(range(n_up)) if rank == 0 else []
            else:
                tasks = list(range(n_up)) if rank == 0 else []
            n_keys = n_up
        part = root.get("partitioning")
        n_out = part["n"] if part else n_keys
        out_parts[st.stage_id] = n_out
        # how do later stages read this one?
        readers = []
        for later in stages[si + 1:]:
            rs = _readers_of(later.plan["input"], st.stage_id)
            readers += [(b, m or later.n_tasks == 1, sch) for (b, m, sch) in rs]
        if not readers:
            placement[st.stage_id] = "root"
            last_schema = None
            mode = None
        else:
            bcast = any(r[0] for r in readers)
            merged = all(r[1] for r in readers)
            schema = readers[0][2]
            if bcast:
                mode, placement[st.stage_id] = EXCHANGE_BROADCAST, "all"
            elif part and not merged:
                mode, placement[st.stage_id] = EXCHANGE_HASH, "hash"
            else:
                mode, placement[st.stage_id] = EXCHANGE_GATHER, "root"
        # fused = writer + hash exchange as one collective per map task (b200_stage_execute_exchange): needs the same number
        # of map tasks on every executor -- true for partitioned tables loaded evenly and for hash-placed inputs whose
        # partition count is a multiple of the executor count
        symmetric = st.n_tasks != 1 and ((kind == "table" and what not in REPLICATED_TABLES) or
                                         (kind != "table" and placement.get(what) == "hash" and out_parts[what] % world == 0))
        fuse = fused and world > 1 and readers and mode == EXCHANGE_HASH and symmetric and _fixed_width(schema)
        qse = engine.create_query_stage_exec(job_id, st.stage_id, st.json(job_id))
        if fuse:
            tot = {"sent_bytes": 0, "recv_bytes": 0, "fused": True}
            for p in tasks:
                _, xs = qse.execute_query_stage_exchange(p)
                tot["sent_bytes"] += xs["sent_bytes"]
                tot["recv_bytes"] += xs["recv_bytes"]
            if on_stage is not None:
                on_stage(st.stage_id, mode, tot)
        else:
            for p in tasks:
                qse.execute_query_stage(p)
        qse.release()
        if readers and world > 1 and not fuse:
            stats = engine.exchange_stage(job_id, st.stage_id, n_out, schema, mode, 0)
            if on_stage is not None:
                on_stage(st.stage_id, mode, stats)
    if not collect or rank != 0:
        return None
    last = stages[-1]
    batches = []
    for p in range(out_parts[last.stage_id]):
        if engine.partition_rows(job_id, last.stage_id, p) >= 0:
            batches.append(engine.partition_export(job_id, last.stage_id, p))
    if not batches:
        return None
    return pa.Table.from_batches(batches)
