"""ctypes host-side mirror of the reference plug-in interface on top of ``libb200exec.so``.

    reference (Rust)                                           here
    ---------------------------------------------------------  -------------------------------------
    trait ExecutionEngine::create_query_stage_exec             GpuExecutionEngine.create_query_stage_exec
      ballista/executor/src/execution_engine.rs:50-58            -> b200_stage_prepare
    trait QueryStageExecutor::execute_query_stage              QueryStageExecutor.execute_query_stage
      ballista/executor/src/execution_engine.rs:73-77            -> b200_stage_execute
    QueryStageExecutor::collect_plan_metrics  (:80)            QueryStageExecutor.collect_plan_metrics
    message ShuffleWritePartition (ballista.proto:481-492)     ShuffleWritePartition

The CUDA library is mandatory: importing succeeds without it (so that CPU-only tests can check the
exported symbols), but constructing an engine raises if the library or a GPU is missing -- there
is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from typing import List, Optional

import pyarrow as pa

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200EXEC_LIB") or os.path.join(_PKG, "lib", "libb200exec.so")


class ShuffleWritePartition(C.Structure):
    _fields_ = [("partition_id", C.c_uint64), ("num_batches", C.c_uint64), ("num_rows", C.c_uint64),
                ("num_bytes", C.c_uint64), ("file_id", C.c_int64), ("is_sort_shuffle", C.c_int32),
                ("_pad", C.c_int32)]

    def as_tuple(self):
        return (self.partition_id, self.num_batches, self.num_rows, self.num_bytes, self.file_id, self.is_sort_shuffle)


class OperatorMetrics(C.Structure):
    _fields_ = [("name", C.c_char * 48), ("output_rows", C.c_uint64), ("input_rows", C.c_uint64),
                ("elapsed_compute_ns", C.c_uint64), ("bytes_read", C.c_uint64), ("bytes_written", C.c_uint64),
                ("kernel_launches", C.c_uint64)]


class KernelStat(C.Structure):
    _fields_ = [("name", C.c_char * 48), ("elapsed_ns", C.c_uint64), ("launches", C.c_uint64), ("algorithmic_bytes", C.c_uint64)]


class ExchangeStats(C.Structure):
    _fields_ = [("sent_bytes", C.c_uint64), ("recv_bytes", C.c_uint64)]


EXCHANGE_HASH, EXCHANGE_GATHER, EXCHANGE_BROADCAST = 0, 1, 2
NCCL_ID_BYTES = 128


class ArrowSchema(C.Structure):
    _fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64),
                ("n_children", C.c_int64), ("children", C.c_void_p), ("dictionary", C.c_void_p),
                ("release", C.c_void_p), ("private_data", C.c_void_p)]


class ArrowArray(C.Structure):
    _fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
                ("n_children", C.c_int64), ("buffers", C.c_void_p), ("children", C.c_void_p),
                ("dictionary", C.c_void_p), ("release", C.c_void_p), ("private_data", C.c_void_p)]


# every symbol include/b200exec.h declares (checked by tests/test_abi.py)
EXPORTED_SYMBOLS = [
    "b200_engine_create", "b200_engine_destroy", "b200_last_error", "b200_engine_set_stream",
    "b200_engine_synchronize", "b200_engine_kernel_launches", "b200_engine_counter", "b200_engine_set_config",
    "b200_engine_register_batch", "b200_engine_register_parquet", "b200_engine_register_csv", "b200_parquet_describe", "b200_engine_drop_table", "b200_engine_tpch_generate",
    "b200_engine_export_table", "b200_tpch_table_rows", "b200_stage_prepare", "b200_stage_execute", "b200_stage_metrics",
    "b200_stage_release", "b200_partition_export", "b200_partition_rows",
    "b200_remove_job_data", "b200_remove_stage_data", "b200_host_alloc_pinned", "b200_host_free_pinned",
    "b200_comm_unique_id", "b200_engine_comm_init", "b200_exchange_stage", "b200_stage_execute_exchange", "b200_engine_kernel_stats",
    "b200_ipc_encode", "b200_ipc_free", "b200_ipc_decode", "b200_shuffle_write_files", "b200_shuffle_read_file",
    "b200_stage_prepare_proto", "b200_stage_prepare_task", "b200_task_status_encode", "b200_plan_proto_to_json", "b200_string_free", "b200_plan_typed_json",
    "b200_version",
]

_lib = None


def load_library():
    """dlopen libb200exec.so (no CUDA call is made by loading)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `make` (or __graft_entry__.build()); "
                           "the engine has no CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, cp, i64, u64, ci = C.c_void_p, C.c_char_p, C.c_int64, C.c_uint64, C.c_int
    L.b200_engine_create.argtypes = [ci, u64, ci, ci, C.POINTER(vp)]
    L.b200_engine_destroy.argtypes = [vp]
    L.b200_engine_destroy.restype = None
    L.b200_last_error.restype = cp
    L.b200_engine_set_stream.argtypes = [vp, vp]
    L.b200_engine_synchronize.argtypes = [vp]
    L.b200_engine_kernel_launches.argtypes = [vp]
    L.b200_engine_kernel_launches.restype = u64
    L.b200_engine_counter.argtypes = [vp, cp]
    L.b200_engine_counter.restype = u64
    L.b200_engine_set_config.argtypes = [vp, cp, cp]
    L.b200_engine_register_batch.argtypes = [vp, cp, ci, vp, vp]
    L.b200_engine_register_parquet.argtypes = [vp, cp, ci, cp, cp]
    L.b200_engine_register_csv.argtypes = [vp, cp, ci, cp]
    L.b200_parquet_describe.argtypes = [cp, vp, u64]
    L.b200_engine_drop_table.argtypes = [vp, cp]
    L.b200_engine_tpch_generate.argtypes = [vp, cp, i64, ci, i64, i64, cp]
    L.b200_engine_export_table.argtypes = [vp, cp, ci, vp, vp]
    L.b200_tpch_table_rows.argtypes = [cp, i64]
    L.b200_tpch_table_rows.restype = i64
    L.b200_stage_prepare.argtypes = [vp, cp, i64, cp, u64, C.POINTER(vp)]
    L.b200_stage_execute.argtypes = [vp, ci, vp, C.POINTER(ShuffleWritePartition), ci, C.POINTER(ci)]
    L.b200_stage_prepare_proto.argtypes = [vp, cp, i64, vp, u64, C.POINTER(vp)]
    L.b200_plan_proto_to_json.argtypes = [vp, u64, cp, C.POINTER(vp)]
    L.b200_plan_typed_json.argtypes = [cp, u64, C.POINTER(vp)]
    L.b200_task_status_encode.argtypes = [cp, cp, C.POINTER(TaskResult), C.POINTER(ShuffleWritePartition), ci, C.POINTER(OperatorMetrics), ci,
                                          C.POINTER(vp), C.POINTER(u64)]
    L.b200_stage_prepare_task.argtypes = [vp, vp, u64, ci, C.POINTER(vp), C.POINTER(vp)]
    L.b200_string_free.argtypes = [vp]
    L.b200_string_free.restype = None
    L.b200_stage_metrics.argtypes = [vp, C.POINTER(OperatorMetrics), ci, C.POINTER(ci)]
    L.b200_stage_release.argtypes = [vp]
    L.b200_stage_release.restype = None
    L.b200_partition_export.argtypes = [vp, cp, i64, ci, vp, vp]
    L.b200_partition_rows.argtypes = [vp, cp, i64, ci]
    L.b200_partition_rows.restype = i64
    L.b200_remove_job_data.argtypes = [vp, cp]
    L.b200_remove_stage_data.argtypes = [vp, cp, i64]
    L.b200_engine_kernel_stats.argtypes = [vp, C.POINTER(KernelStat), ci, C.POINTER(ci), ci]
    L.b200_ipc_encode.argtypes = [vp, vp, ci, i64, C.POINTER(vp), C.POINTER(u64)]
    L.b200_ipc_free.argtypes = [vp]
    L.b200_ipc_free.restype = None
    L.b200_ipc_decode.argtypes = [vp, u64, vp, vp]
    L.b200_shuffle_write_files.argtypes = [vp, cp, i64, cp, ci, ci, C.POINTER(u64), C.POINTER(u64)]
    L.b200_shuffle_read_file.argtypes = [vp, cp, i64, ci, i64, cp, u64, u64, ci]
    L.b200_comm_unique_id.argtypes = [vp, u64]
    L.b200_engine_comm_init.argtypes = [vp, vp, u64]
    L.b200_exchange_stage.argtypes = [vp, cp, i64, ci, ci, ci, cp, C.POINTER(ExchangeStats)]
    L.b200_stage_execute_exchange.argtypes = [vp, ci, vp, C.POINTER(ShuffleWritePartition), ci, C.POINTER(ci), C.POINTER(ExchangeStats)]
    L.b200_host_alloc_pinned.argtypes = [u64]
    L.b200_host_alloc_pinned.restype = vp
    L.b200_host_free_pinned.argtypes = [vp]
    L.b200_host_free_pinned.restype = None
    L.b200_version.restype = cp
    _lib = L
    return L


class B200Error(RuntimeError):
    """Maps b200_status codes (include/b200exec.h) the way the Rust shim maps them to
    DataFusionError / BallistaError."""
    NAMES = {-1: "Plan", -2: "NotImplemented", -3: "Execution", -4: "External(CUDA)", -5: "FetchFailed",
             -6: "Cancelled", -7: "ResourcesExhausted"}

    def __init__(self, code, msg):
        super().__init__(f"{self.NAMES.get(code, code)}: {msg}")
        self.code = code


def _check(rc):
    if rc != 0:
        raise B200Error(rc, load_library().b200_last_error().decode(errors="replace"))


def ipc_encode(batch: pa.RecordBatch, compress: bool = True, max_rows_per_message: int = 0) -> bytes:
    """RecordBatch -> one Arrow IPC stream (schema, record batch message(s), end-of-stream) with LZ4_FRAME buffers: the byte
    format of the reference's shuffle files (b200_ipc_encode; host only)."""
    arr, sch = ArrowArray(), ArrowSchema()
    batch._export_to_c(C.addressof(arr), C.addressof(sch))
    out, n = C.c_void_p(), C.c_uint64(0)
    _check(load_library().b200_ipc_encode(C.addressof(arr), C.addressof(sch), 1 if compress else 0, max_rows_per_message, C.byref(out), C.byref(n)))
    try:
        return C.string_at(out.value, n.value)
    finally:
        load_library().b200_ipc_free(out)


def ipc_decode(data: bytes) -> pa.RecordBatch:
    """One or several back-to-back Arrow IPC streams (optionally LZ4_FRAME compressed) -> one RecordBatch (b200_ipc_decode)."""
    arr, sch = ArrowArray(), ArrowSchema()
    buf = C.create_string_buffer(data, len(data))
    _check(load_library().b200_ipc_decode(buf, len(data), C.addressof(arr), C.addressof(sch)))
    return pa.RecordBatch._import_from_c(C.addressof(arr), C.addressof(sch))


def parquet_describe(path: str) -> dict:
    """What the device Parquet scan's host-side metadata reader sees in `path` (b200_parquet_describe; no GPU needed)."""
    import json as _json
    cap = 1 << 20
    buf = C.create_string_buffer(cap)
    _check(load_library().b200_parquet_describe(path.encode(), buf, cap))
    return _json.loads(buf.value.decode())


# Output arrays of b200_stage_execute / b200_stage_metrics, one of each per thread and reused by every stage executor of
# that thread: the results are copied out before the call returns.  A fresh 8192-entry array per stage cost more host
# time than preparing the stage itself, and every microsecond of it leaves the GPU idle between two stages.
_out_bufs = threading.local()
_OUT_CAP = 8192   # >= the largest shuffle fan-out the engine accepts (4096)
_METRICS_CAP = 256


def _partition_buffer():
    b = getattr(_out_bufs, "partitions", None)
    if b is None:
        b = _out_bufs.partitions = (ShuffleWritePartition * _OUT_CAP)()
    return b


def _metrics_buffer():
    b = getattr(_out_bufs, "metrics", None)
    if b is None:
        b = _out_bufs.metrics = (OperatorMetrics * _METRICS_CAP)()
    return b


class QueryStageExecutor:
    def __init__(self, engine: "GpuExecutionEngine", handle, job_id: str, stage_id: int):
        self.engine, self.h, self.job_id, self.stage_id = engine, handle, job_id, stage_id

    def execute_query_stage(self, input_partition: int, cancel_flag=None) -> List[ShuffleWritePartition]:
        out = _partition_buffer()
        n = C.c_int(0)
        cf = C.addressof(cancel_flag) if cancel_flag is not None else None
        _check(load_library().b200_stage_execute(self.h, input_partition, cf, out, _OUT_CAP, C.byref(n)))
        res = [ShuffleWritePartition.from_buffer_copy(out[i]) for i in range(n.value)]
        return res

    def execute_query_stage_exchange(self, input_partition: int, cancel_flag=None):
        """Collective: this map task plus the hash exchange of its output in one call (b200_stage_execute_exchange).
        Returns (ShuffleWritePartition list, {"sent_bytes", "recv_bytes"})."""
        n = C.c_int(0)
        st = ExchangeStats()
        out = _partition_buffer()
        cf = C.addressof(cancel_flag) if cancel_flag is not None else None
        _check(load_library().b200_stage_execute_exchange(self.h, input_partition, cf, out, _OUT_CAP, C.byref(n), C.byref(st)))
        res = [ShuffleWritePartition.from_buffer_copy(out[i]) for i in range(n.value)]
        return res, {"sent_bytes": st.sent_bytes, "recv_bytes": st.recv_bytes}

    def collect_plan_metrics(self) -> List[dict]:
        out = _metrics_buffer()
        n = C.c_int(0)
        _check(load_library().b200_stage_metrics(self.h, out, _METRICS_CAP, C.byref(n)))
        return [dict(name=out[i].name.decode(), output_rows=out[i].output_rows, input_rows=out[i].input_rows,
                     elapsed_compute_ns=out[i].elapsed_compute_ns, bytes_read=out[i].bytes_read,
                     bytes_written=out[i].bytes_written, kernel_launches=out[i].kernel_launches)
                for i in range(n.value)]

    def release(self):
        if self.h:
            load_library().b200_stage_release(self.h)
            self.h = None


def plan_proto_to_json(plan_bytes: bytes, job_id: Optional[str] = None) -> str:
    """Decode a protobuf datafusion.PhysicalPlanNode (a Ballista task's plan bytes) into the stage-plan IR (JSON text).
    Host-only (b200_plan_proto_to_json): needs the library, not a GPU."""
    L = load_library()
    out = C.c_void_p()
    buf = C.create_string_buffer(plan_bytes, len(plan_bytes))
    _check(L.b200_plan_proto_to_json(C.cast(buf, C.c_void_p), len(plan_bytes), job_id.encode() if job_id else None, C.byref(out)))
    try:
        return C.string_at(out.value).decode()
    finally:
        L.b200_string_free(out)


class TaskResult(C.Structure):
    """b200_task_result (include/b200exec.h)."""
    _fields_ = [("task_id", C.c_uint32), ("stage_id", C.c_uint32), ("stage_attempt_num", C.c_uint32), ("partition_id", C.c_uint32),
                ("launch_time", C.c_uint64), ("start_exec_time", C.c_uint64), ("end_exec_time", C.c_uint64), ("status", C.c_int32),
                ("fetch_map_stage_id", C.c_uint32), ("fetch_map_partition_id", C.c_uint32), ("fetch_executor_id", C.c_char_p),
                ("error_message", C.c_char_p)]


def task_status_encode(job_id: str, executor_id: str, result: "TaskResult", partitions=(), metrics=()) -> bytes:
    """ballista.protobuf.TaskStatus bytes for a finished task (b200_task_status_encode; host only).
    partitions: ShuffleWritePartition structs (b200_stage_execute's output); metrics: OperatorMetrics structs."""
    L = load_library()
    parts = (ShuffleWritePartition * max(len(partitions), 1))(*partitions)
    mets = (OperatorMetrics * max(len(metrics), 1))(*metrics)
    out, n = C.c_void_p(), C.c_uint64(0)
    _check(L.b200_task_status_encode(job_id.encode(), executor_id.encode(), C.byref(result), parts, len(partitions), mets, len(metrics),
                                     C.byref(out), C.byref(n)))
    try:
        return C.string_at(out.value, n.value)
    finally:
        L.b200_string_free(out)


def task_definition_decode(task_bytes: bytes, multi: bool = False) -> dict:
    """Decode a ballista.protobuf.TaskDefinition / MultiTaskDefinition (identities + props; host only)."""
    import json as _json
    L = load_library()
    out = C.c_void_p()
    buf = C.create_string_buffer(task_bytes, len(task_bytes))
    _check(L.b200_stage_prepare_task(None, C.cast(buf, C.c_void_p), len(task_bytes), 1 if multi else 0, None, C.byref(out)))
    try:
        return _json.loads(C.string_at(out.value).decode())
    finally:
        L.b200_string_free(out)


def plan_typed_json(plan_json: str) -> str:
    """The typed plan the engine derives from an IR text (b200_plan_typed_json): canonical JSON, host-only."""
    L = load_library()
    out = C.c_void_p()
    _check(L.b200_plan_typed_json(plan_json.encode(), 0, C.byref(out)))
    try:
        return C.string_at(out.value).decode()
    finally:
        L.b200_string_free(out)


class GpuExecutionEngine:
    """One per executor process == one per GPU (SURVEY.md 8(b) "Threading")."""

    def __init__(self, device: int = 0, pool_bytes: int = 0, rank: int = 0, world: int = 1):
        L = load_library()
        h = C.c_void_p()
        _check(L.b200_engine_create(device, pool_bytes, rank, world, C.byref(h)))
        self.h = h
        self.device = device
        self._parts = {}

    def close(self):
        if self.h:
            load_library().b200_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- config / stream ---------------------------------------------------------------------
    def set_config(self, key: str, value) -> None:
        _check(load_library().b200_engine_set_config(self.h, key.encode(), str(value).encode()))

    def set_stream(self, cuda_stream_ptr: Optional[int]) -> None:
        _check(load_library().b200_engine_set_stream(self.h, cuda_stream_ptr))

    def synchronize(self) -> None:
        _check(load_library().b200_engine_synchronize(self.h))

    def kernel_launches(self) -> int:
        return load_library().b200_engine_kernel_launches(self.h)

    def counter(self, name: str) -> int:
        """Pipelines run per kernel family: 'fused', 'fused_static', 'vm' (b200_engine_counter)."""
        return load_library().b200_engine_counter(self.h, name.encode())

    def kernel_stats(self, reset: bool = False) -> dict:
        """{kernel family: {"ms", "launches", "bytes"}} while b200.metrics.kernel_timing is on (b200_engine_kernel_stats)."""
        cap = 128
        out = (KernelStat * cap)()
        n = C.c_int(0)
        _check(load_library().b200_engine_kernel_stats(self.h, out, cap, C.byref(n), 1 if reset else 0))
        return {out[i].name.decode(): {"ms": out[i].elapsed_ns / 1e6, "launches": out[i].launches, "bytes": out[i].algorithmic_bytes}
                for i in range(n.value)}

    # -- leaf inputs ---------------------------------------------------------------------------
    def register_batch(self, table: str, partition: int, batch: pa.RecordBatch) -> None:
        arr, sch = ArrowArray(), ArrowSchema()
        batch._export_to_c(C.addressof(arr), C.addressof(sch))
        _check(load_library().b200_engine_register_batch(self.h, table.encode(), partition, C.addressof(arr), C.addressof(sch)))
        self._parts.setdefault(table, set()).add(partition)

    def register_parquet(self, table: str, partition: int, path: str, columns: Optional[List[str]] = None) -> None:
        """Scan a Parquet file into a table partition with the page decode on the device (b200_engine_register_parquet)."""
        csv = ",".join(columns).encode() if columns else None
        _check(load_library().b200_engine_register_parquet(self.h, table.encode(), partition, path.encode(), csv))
        self._parts.setdefault(table, set()).add(partition)

    def register_csv(self, table: str, partition: int, files, schema: List[dict], columns: Optional[List[str]] = None,
                     has_header: bool = False, delimiter: str = ",", quote: str = '"', escape: Optional[str] = None,
                     newlines_in_values: bool = False) -> None:
        """Scan CSV / .tbl files into a table partition with records, fields and values found on the device
        (b200_engine_register_csv).  files: paths or (path, start, end) byte ranges; schema: the files' columns as plan-IR
        fields; columns: the ones to materialise, in this order (None: all)."""
        import json as _json
        fl = []
        for f in ([files] if isinstance(files, (str, tuple)) else files):
            fl.append({"path": f[0], "range": [int(f[1]), int(f[2])]} if isinstance(f, tuple) else {"path": f})
        spec = {"files": fl, "schema": schema, "has_header": has_header, "delimiter": delimiter, "quote": quote,
                "escape": escape, "newlines_in_values": newlines_in_values}
        if columns is not None:
            spec["columns"] = list(columns)
        self.register_csv_json(table, partition, _json.dumps(spec))

    def register_csv_json(self, table: str, partition: int, scan_json: str) -> None:
        """b200_engine_register_csv with the scan description as it crosses the C ABI."""
        _check(load_library().b200_engine_register_csv(self.h, table.encode(), partition, scan_json.encode()))
        self._parts.setdefault(table, set()).add(partition)

    def drop_table(self, table: str) -> None:
        _check(load_library().b200_engine_drop_table(self.h, table.encode()))
        self._parts.pop(table, None)

    def tpch_generate(self, table, msf, partition, row_begin, row_end, columns: Optional[List[str]] = None) -> None:
        csv = ",".join(columns).encode() if columns else None
        _check(load_library().b200_engine_tpch_generate(self.h, table.encode(), msf, partition, row_begin, row_end, csv))
        self._parts.setdefault(table, set()).add(partition)

    @staticmethod
    def tpch_table_rows(table: str, msf: int) -> int:
        return load_library().b200_tpch_table_rows(table.encode(), msf)

    def tpch_load(self, tables: dict, msf: int, rank: int = 0, world: int = 1, parts: int = 1, replicated=("nation", "region")) -> dict:
        """Generate this executor's share of the given TPC-H tables in HBM: rows [rank, rank+1) / world of every
        table, split into `parts` input partitions; the small dimension tables are replicated in full.
        Returns {table: global row count}."""
        rows = {}
        if not hasattr(self, "replicated_tables"):
            self.replicated_tables = set()   # consulted by driver.run_stages_distributed: scanned on one executor only
        for t, cols in tables.items():
            n = self.tpch_table_rows(t, msf)
            rows[t] = n
            self.drop_table(t)
            self.replicated_tables.discard(t)
            if t in replicated or n < 1000:
                self.tpch_generate(t, msf, 0, 0, n, cols)
                self.replicated_tables.add(t)
                continue
            lo, hi = n * rank // world, n * (rank + 1) // world
            step = (hi - lo + parts - 1) // parts
            for p in range(parts):
                self.tpch_generate(t, msf, p, min(hi, lo + p * step), min(hi, lo + (p + 1) * step), cols)
        return rows

    def export_table(self, table: str, partition: int) -> pa.RecordBatch:
        arr, sch = ArrowArray(), ArrowSchema()
        _check(load_library().b200_engine_export_table(self.h, table.encode(), partition, C.addressof(arr), C.addressof(sch)))
        return pa.RecordBatch._import_from_c(C.addressof(arr), C.addressof(sch))

    def n_table_partitions(self, table: str) -> int:
        return max(self._parts[table]) + 1

    # -- ExecutionEngine -------------------------------------------------------------------------
    def create_query_stage_exec(self, job_id: str, stage_id: int, plan_json: str) -> QueryStageExecutor:
        h = C.c_void_p()
        pj = plan_json.encode()
        _check(load_library().b200_stage_prepare(self.h, job_id.encode(), stage_id, pj, len(pj), C.byref(h)))
        return QueryStageExecutor(self, h, job_id, stage_id)

    def create_query_stage_exec_proto(self, job_id: str, stage_id: int, plan_bytes: bytes) -> QueryStageExecutor:
        """The same from the protobuf plan bytes of a Ballista task (b200_stage_prepare_proto)."""
        h = C.c_void_p()
        buf = C.create_string_buffer(plan_bytes, len(plan_bytes))
        _check(load_library().b200_stage_prepare_proto(self.h, job_id.encode(), stage_id, C.cast(buf, C.c_void_p), len(plan_bytes), C.byref(h)))
        return QueryStageExecutor(self, h, job_id, stage_id)

    def create_query_stage_exec_task(self, task_bytes: bytes, multi: bool = False):
        """From a whole TaskDefinition / MultiTaskDefinition (b200_stage_prepare_task): (QueryStageExecutor, task info dict)."""
        import json as _json
        h, out = C.c_void_p(), C.c_void_p()
        buf = C.create_string_buffer(task_bytes, len(task_bytes))
        _check(load_library().b200_stage_prepare_task(self.h, C.cast(buf, C.c_void_p), len(task_bytes), 1 if multi else 0, C.byref(h), C.byref(out)))
        try:
            info = _json.loads(C.string_at(out.value).decode())
        finally:
            load_library().b200_string_free(out)
        return QueryStageExecutor(self, h, info["job_id"], info["stage_id"]), info

    # -- shuffle partitions ----------------------------------------------------------------------
    def partition_export(self, job_id: str, stage_id: int, out_partition: int) -> pa.RecordBatch:
        arr, sch = ArrowArray(), ArrowSchema()
        _check(load_library().b200_partition_export(self.h, job_id.encode(), stage_id, out_partition,
                                                    C.addressof(arr), C.addressof(sch)))
        return pa.RecordBatch._import_from_c(C.addressof(arr), C.addressof(sch))

    def partition_rows(self, job_id: str, stage_id: int, out_partition: int) -> int:
        return load_library().b200_partition_rows(self.h, job_id.encode(), stage_id, out_partition)

    # -- exchange between the box's GPU executors (NCCL inside the library) -------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        """128 bytes generated by ONE executor and handed to every executor's comm_init (b200_comm_unique_id)."""
        buf = C.create_string_buffer(NCCL_ID_BYTES)
        _check(load_library().b200_comm_unique_id(buf, NCCL_ID_BYTES))
        return buf.raw

    def comm_init(self, nccl_id: bytes) -> None:
        buf = C.create_string_buffer(nccl_id, len(nccl_id))
        _check(load_library().b200_engine_comm_init(self.h, buf, len(nccl_id)))

    def exchange_stage(self, job_id: str, stage_id: int, n_out_partitions: int, schema, mode: int = EXCHANGE_HASH, root: int = 0) -> dict:
        """Collective: move every output partition of (job, stage) to the executor(s) that will read it
        (b200_exchange_stage).  `schema`: the stage's output schema (list of {"name", "type"} dicts)."""
        import json as _json
        st = ExchangeStats()
        sj = schema if isinstance(schema, str) else _json.dumps(schema)
        _check(load_library().b200_exchange_stage(self.h, job_id.encode(), stage_id, n_out_partitions, mode, root, sj.encode(), C.byref(st)))
        return {"sent_bytes": st.sent_bytes, "recv_bytes": st.recv_bytes}

    # -- the reference's shuffle files ---------------------------------------------------------------------
    def shuffle_write_files(self, job_id: str, stage_id: int, work_dir: str, n_out_partitions: int, sort_layout: bool) -> dict:
        nf, nb = C.c_uint64(0), C.c_uint64(0)
        _check(load_library().b200_shuffle_write_files(self.h, job_id.encode(), stage_id, work_dir.encode(), n_out_partitions, 1 if sort_layout else 0,
                                                       C.byref(nf), C.byref(nb)))
        return {"files": nf.value, "bytes": nb.value}

    def shuffle_read_file(self, job_id: str, stage_id: int, out_partition: int, file_id: int, path: str, byte_offset: int = 0, byte_length: int = 0,
                          use_index: bool = False) -> None:
        _check(load_library().b200_shuffle_read_file(self.h, job_id.encode(), stage_id, out_partition, file_id, path.encode(), byte_offset, byte_length,
                                                     1 if use_index else 0))

    def remove_job_data(self, job_id: str) -> None:
        _check(load_library().b200_remove_job_data(self.h, job_id.encode()))

    def remove_stage_partitions(self, job_id: str, stage_id: int) -> None:
        _check(load_library().b200_remove_stage_data(self.h, job_id.encode(), stage_id))
