"""Builders for the stage-plan IR (JSON) consumed by ``b200_stage_prepare``.

The IR is a JSON rendering of the DataFusion physical plan a Ballista task carries
(``TaskDefinition.plan``, ballista/core/proto/ballista.proto:518-529; node shapes pinned by
ballista/core/proto/datafusion.proto:716-757 and :851-901).  A Rust shim produces the same JSON
by walking ``Arc<dyn ExecutionPlan>`` (INTEGRATION.md); this module is the Python harness'
equivalent so tests read like the reference's own (`ctx.sql(...)` -> physical plan -> stages).
"""
from __future__ import annotations

import datetime as _dt
import json
from typing import Any, Dict, List, Optional, Sequence

Json = Dict[str, Any]


# ---- types ---------------------------------------------------------------------------------------
def dec(p: int, s: int) -> Json:
    return {"dec": [p, s]}


def field(name: str, typ, nullable: bool = False) -> Json:
    return {"name": name, "type": typ, "nullable": nullable}


# ---- expressions ---------------------------------------------------------------------------------
def col(i) -> Json:
    """Column by index (or by name, resolved against the input schema by the parser)."""
    return {"col": i}


def lit_i64(v: Optional[int]) -> Json:
    return {"lit": {"t": "i64", "v": v}}


def lit_i32(v: Optional[int]) -> Json:
    return {"lit": {"t": "i32", "v": v}}


def lit_f64(v: Optional[float]) -> Json:
    return {"lit": {"t": "f64", "v": v}}


def lit_bool(v: Optional[bool]) -> Json:
    return {"lit": {"t": "bool", "v": v}}


def lit_utf8(v: Optional[str]) -> Json:
    return {"lit": {"t": "utf8", "v": v}}


def lit_dec(unscaled: int, p: int, s: int) -> Json:
    return {"lit": {"t": dec(p, s), "v": str(int(unscaled))}}


def lit_date(s: str) -> Json:
    d = _dt.date.fromisoformat(s)
    return {"lit": {"t": "date32", "v": (d - _dt.date(1970, 1, 1)).days}}


def lit_null(typ) -> Json:
    return {"lit": {"t": typ, "v": None}}


def binop(op: str, l: Json, r: Json) -> Json:
    return {"bin": op, "l": l, "r": r}


def and_(*xs: Json) -> Json:
    out = xs[0]
    for x in xs[1:]:
        out = binop("and", out, x)
    return out


def or_(*xs: Json) -> Json:
    out = xs[0]
    for x in xs[1:]:
        out = binop("or", out, x)
    return out


def not_(x: Json) -> Json:
    return {"not": x}


def neg(x: Json) -> Json:
    return {"neg": x}


def is_null(x: Json) -> Json:
    return {"is_null": x}


def is_not_null(x: Json) -> Json:
    return {"is_not_null": x}


def cast(x: Json, to) -> Json:
    return {"cast": x, "to": to}


def case(whens: Sequence[Sequence[Json]], else_: Optional[Json] = None) -> Json:
    c: Json = {"when": [list(w) for w in whens]}
    if else_ is not None:
        c["else"] = else_
    return {"case": c}


def in_list(x: Json, items: Sequence[Json], negated: bool = False) -> Json:
    return {"in": x, "list": list(items), "negated": negated}


def like(x: Json, pattern: str, negated: bool = False, case_insensitive: bool = False) -> Json:
    """[NOT] LIKE, or [NOT] ILIKE with case_insensitive (arrow's LIKE-to-regex translation under the flags i and s)."""
    n: Json = {"like": x, "pattern": pattern, "negated": negated}
    if case_insensitive:
        n["case_insensitive"] = True
    return n


def regex_match(x: Json, pattern, negated: bool = False, case_insensitive: bool = False) -> Json:
    """x ~ p, x ~* p, x !~ p, x !~* p: an unanchored Rust-regex match against a Utf8 literal pattern (a str, or an
    expression such as lit_utf8(None))."""
    p = lit_utf8(pattern) if isinstance(pattern, str) else pattern
    return binop(("!~" if negated else "~") + ("*" if case_insensitive else ""), x, p)


def fn(name: str, *args: Json) -> Json:
    return {"fn": name, "args": list(args)}


def str_concat(*xs: Json) -> Json:
    """x0 || x1 || ...: Utf8 operands, NULL if any is NULL (left-associated, as DataFusion parses it)."""
    out = xs[0]
    for x in xs[1:]:
        out = binop("||", out, x)
    return out


# ---- operators -----------------------------------------------------------------------------------
def scan(table: str, schema: List[Json], projection: Optional[List[int]] = None) -> Json:
    n: Json = {"op": "DataSourceExec", "table": table, "schema": schema}
    if projection is not None:
        n["projection"] = projection
    return n


def csv_scan(table: str, schema: List[Json], projection: Optional[List[int]] = None, file_groups: Optional[List[List[str]]] = None,
             file_ranges: Optional[List[list]] = None, has_header: bool = False, delimiter: str = ",", quote: str = '"',
             escape: Optional[str] = None, newlines_in_values: bool = False) -> Json:
    """DataSourceExec over CSV files (CsvScanExecNode): `schema` is the files' columns, `projection` indexes it, and the
    reader options ride along as the protobuf decoder emits them ("format", "csv", "file_ranges")."""
    n = scan(table, schema, projection)
    if file_groups is not None:
        n["file_groups"] = file_groups
    n["format"] = "csv"
    n["csv"] = {"has_header": has_header, "delimiter": delimiter, "quote": quote, "escape": escape,
                "newlines_in_values": newlines_in_values}
    if file_ranges is not None:
        n["file_ranges"] = file_ranges
    return n


def shuffle_reader(stage_id: int, schema: List[Json], broadcast: bool = False) -> Json:
    return {"op": "ShuffleReaderExec", "stage_id": stage_id, "schema": schema, "broadcast": broadcast}


def filter_(predicate: Json, input: Json, projection: Optional[List[int]] = None) -> Json:
    n: Json = {"op": "FilterExec", "predicate": predicate, "input": input}
    if projection is not None:
        n["projection"] = projection
    return n


def project(exprs: Sequence, input: Json) -> Json:
    """exprs: list of (expr, name)."""
    return {"op": "ProjectionExec", "exprs": [{"expr": e, "name": n} for e, n in exprs], "input": input}


def agg(fn_: str, arg: Optional[Json], name: str, input_type=None, arg2: Optional[Json] = None) -> Json:
    """arg2: the second argument of covar / corr."""
    a: Json = {"fn": fn_, "name": name, "args": ([] if arg is None else [arg]) + ([] if arg2 is None else [arg2])}
    if input_type is not None:
        a["input_type"] = input_type
    return a


def aggregate(mode: str, group_by: Sequence, aggr: Sequence[Json], input: Json,
              grouping_sets: Optional[Sequence[Sequence[bool]]] = None) -> Json:
    """group_by: list of (expr, name).  grouping_sets (Partial / Single / SinglePartitioned only): one list of len(group_by)
    bools per set, True where that key is replaced by NULL; the output then holds the keys, `__grouping_id`, then the
    aggregates (DESIGN.md §6)."""
    n: Json = {"op": "AggregateExec", "mode": mode,
               "group_by": [{"expr": e, "name": n} for e, n in group_by], "aggr": list(aggr), "input": input}
    if grouping_sets is not None:
        n["grouping_sets"] = [[bool(b) for b in s] for s in grouping_sets]
    return n


def rollup_sets(n_keys: int) -> List[List[bool]]:
    """ROLLUP(k0, ..., k{n-1}): (k0..k{n-1}), (k0..k{n-2}), ..., ()."""
    return [[k >= n_keys - d for k in range(n_keys)] for d in range(n_keys + 1)]


def cube_sets(n_keys: int) -> List[List[bool]]:
    """CUBE(k0, ..., k{n-1}): every subset of the keys (the order of the sets does not change the result)."""
    return [[bool((m >> (n_keys - 1 - k)) & 1) for k in range(n_keys)] for m in range(1 << n_keys)]


def grouping_id(mask: Sequence[bool]) -> int:
    """__grouping_id of a set: the keys folded first to last, id = id << 1 | is_null [EXT]."""
    v = 0
    for b in mask:
        v = v << 1 | int(bool(b))
    return v


def hash_join(left: Json, right: Json, on: Sequence[Sequence[Json]], join_type: str = "Inner",
              mode: str = "CollectLeft", filter: Optional[Json] = None,
              projection: Optional[List[int]] = None, null_equals_null: bool = False) -> Json:
    """HashJoinExecNode (datafusion.proto:1134-1144).  `null_equals_null`: a NULL key matches a NULL key
    (NullEquality::NullEqualsNull, as DataFusion plans INTERSECT / EXCEPT and IS NOT DISTINCT FROM keys)."""
    n: Json = {"op": "HashJoinExec", "left": left, "right": right, "on": [list(p) for p in on],
               "join_type": join_type, "mode": mode}
    if filter is not None:
        n["filter"] = filter
    if projection is not None:
        n["projection"] = projection
    if null_equals_null:
        n["null_equals_null"] = True
    return n


def nested_loop_join(left: Json, right: Json, join_type: str = "Inner", filter: Optional[Json] = None,
                     projection: Optional[List[int]] = None) -> Json:
    """NestedLoopJoinExecNode (datafusion.proto:1301-1307): a join without equality keys.  The left input is the build
    side, read whole by every task; `filter` indexes left ++ right."""
    n: Json = {"op": "NestedLoopJoinExec", "left": left, "right": right, "join_type": join_type}
    if filter is not None:
        n["filter"] = filter
    if projection is not None:
        n["projection"] = projection
    return n


def sort_merge_join(left: Json, right: Json, on: Sequence[Sequence[Json]], join_type: str = "Inner",
                    filter: Optional[Json] = None, sort_options: Optional[Sequence[Json]] = None,
                    null_equals_null: bool = False) -> Json:
    """SortMergeJoinExecNode (datafusion.proto:1433): Ballista's default join strategy (extension.rs:683).
    Inputs are co-partitioned on the keys; the output is ordered by them."""
    n: Json = {"op": "SortMergeJoinExec", "left": left, "right": right, "on": [list(p) for p in on], "join_type": join_type}
    if filter is not None:
        n["filter"] = filter
    if sort_options is not None:
        n["sort_options"] = list(sort_options)
    if null_equals_null:
        n["null_equals_null"] = True
    return n


def sort_key(expr: Json, asc: bool = True, nulls_first: Optional[bool] = None) -> Json:
    return {"expr": expr, "asc": asc, "nulls_first": (not asc) if nulls_first is None else nulls_first}


def sort(keys: Sequence[Json], input: Json, fetch: Optional[int] = None, preserve_partitioning: bool = False) -> Json:
    n: Json = {"op": "SortExec", "expr": list(keys), "input": input, "preserve_partitioning": preserve_partitioning}
    if fetch is not None:
        n["fetch"] = fetch
    return n


def sort_preserving_merge(keys: Sequence[Json], input: Json, fetch: Optional[int] = None) -> Json:
    n: Json = {"op": "SortPreservingMergeExec", "expr": list(keys), "input": input}
    if fetch is not None:
        n["fetch"] = fetch
    return n


UNBOUNDED_PRECEDING: Json = {"kind": "unbounded_preceding"}
CURRENT_ROW: Json = {"kind": "current_row"}
UNBOUNDED_FOLLOWING: Json = {"kind": "unbounded_following"}


def preceding(n: int) -> Json:
    return {"kind": "preceding", "n": int(n)}


def following(n: int) -> Json:
    return {"kind": "following", "n": int(n)}


def rows(start: Json, end: Json) -> Json:
    """ROWS BETWEEN start AND end (bounds: UNBOUNDED_PRECEDING, preceding(n), CURRENT_ROW, following(n), UNBOUNDED_FOLLOWING)."""
    return {"units": "rows", "start": start, "end": end}


def range_(start: Json, end: Json) -> Json:
    """RANGE BETWEEN start AND end; the device takes UNBOUNDED and CURRENT ROW bounds (CURRENT ROW = the row's peers)."""
    return {"units": "range", "start": start, "end": end}


def win(fn_: str, name: str, args: Sequence[Json] = (), partition_by: Sequence[Json] = (), order_by: Sequence[Json] = (),
        frame: Optional[Json] = None) -> Json:
    """One window expression.  frame=None: DataFusion's default, RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW (the whole
    partition without ORDER BY).  order_by: sort_key(...) entries."""
    w: Json = {"fn": fn_, "name": name, "args": list(args), "partition_by": list(partition_by), "order_by": list(order_by)}
    if frame is not None:
        w["frame"] = frame
    return w


def window(exprs: Sequence[Json], input: Json, partition_keys: Optional[Sequence[Json]] = None, mode: Optional[str] = "sorted") -> Json:
    """WindowAggExec (mode None) / BoundedWindowAggExec (mode "sorted").  The output is the input's columns, then one column
    per expression, named by its name (DESIGN.md §6 (viii)).  partition_keys default to the first expression's."""
    pk = list(exprs[0]["partition_by"]) if partition_keys is None else list(partition_keys)
    return {"op": "WindowAggExec", "mode": mode, "partition_keys": pk, "window_expr": list(exprs), "input": input}


def coalesce_batches(input: Json) -> Json:
    return {"op": "CoalesceBatchesExec", "input": input}


def coalesce_partitions(input: Json) -> Json:
    return {"op": "CoalescePartitionsExec", "input": input}


def limit(input: Json, fetch: int, skip: int = 0, global_: bool = True) -> Json:
    return {"op": "GlobalLimitExec" if global_ else "LocalLimitExec", "input": input, "fetch": fetch, "skip": skip}


def shuffle_writer(input: Json, stage_id: int, hash_exprs: Optional[Sequence[Json]] = None,
                   n_partitions: int = 0, sort_shuffle: bool = True, job_id: str = "job") -> Json:
    """Root of every stage.  hash_exprs=None -> the un-partitioned (`None`) branch."""
    n: Json = {"op": "SortShuffleWriterExec" if (sort_shuffle and hash_exprs is not None) else "ShuffleWriterExec",
               "job_id": job_id, "stage_id": stage_id, "input": input}
    if hash_exprs is not None:
        n["partitioning"] = {"hash": list(hash_exprs), "n": int(n_partitions)}
    return n


def dumps(plan: Json) -> str:
    return json.dumps(plan, separators=(",", ":"))


# ---- helper: output schema of a plan (mirrors csrc/common/plan.hpp only for leaf wiring) ----------
class Stage:
    """One query stage: plan rooted at a shuffle writer + how many input partitions (= tasks)."""

    def __init__(self, stage_id: int, plan: Json, n_tasks: Optional[int] = None):
        self.stage_id = stage_id
        self.plan = plan
        self.n_tasks = n_tasks  # None: as many as the leaf has partitions (driver decides)
        self._json = None

    def json(self, job_id: str) -> str:
        # serialised once; the job id is patched into the cached text (a stage is prepared once per task, and the
        # harness runs the same stage plans under a fresh job id every benchmark step)
        if self._json is None:
            p = dict(self.plan)
            p["job_id"] = "\x00JOB\x00"
            p["stage_id"] = self.stage_id
            self._json = dumps(p)
        return self._json.replace("\\u0000JOB\\u0000", json.dumps(job_id)[1:-1])
