"""Generate tests/golden/proto_plans.json: stage plans as the protobuf bytes a Ballista scheduler ships to an executor.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_proto_plans.py      (commit the output)

For every stage of the 22 TPC-H queries (ballista_b200/tpch.py) and a few extra shapes, the stage-plan IR is typed by the
engine's own plan front end (b200_plan_typed_json: resolved column indices, node schemas) and then ENCODED as
datafusion.PhysicalPlanNode with message classes built at run time from the reference's .proto files
(tests/golden/protoc_lite.py over ballista/core/proto/*.proto) -- field numbers and wire types are therefore the reference's,
serialisation is google.protobuf's.  Conventions of datafusion-proto's `to_proto` [EXT, un-vendored crate] are restated here:
BinaryExpr.op = Debug name of the operator, Decimal128 literal = 16 big-endian bytes, date_part('YEAR', x) as a scalar UDF,
aggregates as PhysicalAggregateExprNode{user_defined_aggr_function}, Ballista's shuffle nodes wrapped in
PhysicalExtensionNode by BallistaPhysicalExtensionCodec (ballista/core/src/serde/mod.rs:481-640).
tests/test_plan_proto.py decodes the bytes with the C++ decoder (csrc/common/plan_proto.hpp) and requires the typed plan of
the result to equal the typed plan of the IR it was generated from.
"""
import base64
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import protoc_lite  # noqa: E402

CLS, _POOL = None, None


def C(name):
    global CLS, _POOL
    if CLS is None:
        CLS, _POOL = protoc_lite.load_ballista()
    return CLS[name]


# ---- types, schemas, literals ---------------------------------------------------------------------------------------------
_SIMPLE = {"null": "NONE", "bool": "BOOL", "i8": "INT8", "i16": "INT16", "i32": "INT32", "i64": "INT64", "u8": "UINT8",
           "u16": "UINT16", "u32": "UINT32", "u64": "UINT64", "f32": "FLOAT32", "f64": "FLOAT64", "utf8": "UTF8",
           "date32": "DATE32"}


def set_type(msg, t):
    if isinstance(t, dict):
        msg.DECIMAL128.precision, msg.DECIMAL128.scale = t["dec"]
    elif t == "ts":
        msg.TIMESTAMP.time_unit = 3
    else:
        getattr(msg, _SIMPLE[t]).SetInParent()


def set_schema(msg, fields):
    for f in fields:
        c = msg.columns.add()
        c.name = f["name"]
        set_type(c.arrow_type, f["type"])
        c.nullable = bool(f.get("nullable", True))


def set_literal(msg, lit):
    t, v = lit["t"], lit.get("v")
    if v is None:
        set_type(msg.null_value, t)
    elif isinstance(t, dict):
        msg.decimal128_value.value = int(v).to_bytes(16, "big", signed=True)
        msg.decimal128_value.p, msg.decimal128_value.s = t["dec"]
    elif t == "bool":
        msg.bool_value = bool(v)
    elif t == "utf8":
        msg.utf8_value = v
    elif t == "date32":
        msg.date_32_value = int(v)
    elif t in ("f32", "f64"):
        setattr(msg, {"f32": "float32_value", "f64": "float64_value"}[t], float(v))
    else:
        setattr(msg, {"i8": "int8_value", "i16": "int16_value", "i32": "int32_value", "i64": "int64_value", "u8": "uint8_value",
                      "u16": "uint16_value", "u32": "uint32_value", "u64": "uint64_value"}[t], int(v))


# ---- expressions (input: the typed form, every column an index) ---------------------------------------------------------------
_OPS = {"=": "Eq", "!=": "NotEq", "<": "Lt", "<=": "LtEq", ">": "Gt", ">=": "GtEq", "+": "Plus", "-": "Minus", "*": "Multiply",
        "/": "Divide", "%": "Modulo", "and": "And", "or": "Or"}


def set_expr(msg, e, remap=None, names=None):
    rec = lambda m, x: set_expr(m, x, remap, names)   # noqa: E731
    if "col" in e:
        idx = e["col"] if remap is None else remap[e["col"]]
        msg.column.index = idx
        msg.column.name = (names[idx] if names else e.get("name", "")) or f"c{idx}"
    elif "lit" in e:
        set_literal(msg.literal, e["lit"])
    elif "bin" in e:
        msg.binary_expr.op = _OPS[e["bin"]]
        rec(msg.binary_expr.l, e["l"])
        rec(msg.binary_expr.r, e["r"])
    elif "not" in e:
        rec(msg.not_expr.expr, e["not"])
    elif "neg" in e:
        rec(msg.negative.expr, e["neg"])
    elif "is_null" in e:
        rec(msg.is_null_expr.expr, e["is_null"])
    elif "is_not_null" in e:
        rec(msg.is_not_null_expr.expr, e["is_not_null"])
    elif "cast" in e:
        rec(msg.cast.expr, e["cast"])
        set_type(msg.cast.arrow_type, e["to"])
    elif "case" in e:
        c = getattr(msg, "case_")
        for w, t in e["case"]["when"]:
            wt = c.when_then_expr.add()
            rec(wt.when_expr, w)
            rec(wt.then_expr, t)
        if "else" in e["case"]:
            rec(c.else_expr, e["case"]["else"])
    elif "in" in e:
        rec(msg.in_list.expr, e["in"])
        for it in e["list"]:
            rec(msg.in_list.list.add(), it)
        msg.in_list.negated = bool(e.get("negated"))
    elif "like" in e:
        msg.like_expr.negated = bool(e.get("negated"))
        msg.like_expr.case_insensitive = False
        rec(msg.like_expr.expr, e["like"])
        msg.like_expr.pattern.literal.utf8_value = e["pattern"]
    elif "fn" in e:
        u = msg.scalar_udf
        if e["fn"] == "date_part_year":
            u.name = "date_part"
            u.args.add().literal.utf8_value = "YEAR"
            rec(u.args.add(), e["args"][0])
            set_type(u.return_type, "i32")
        elif e["fn"] == "substr":
            u.name = "substr"
            for a in e["args"]:
                rec(u.args.add(), a)
            set_type(u.return_type, "utf8")
        else:
            raise ValueError(e["fn"])
    else:
        raise ValueError(f"expression {e}")


def cols_of(e, out):
    if isinstance(e, dict):
        if "col" in e:
            if e["col"] not in out:
                out.append(e["col"])
        for v in e.values():
            cols_of(v, out)
    elif isinstance(e, list):
        for v in e:
            cols_of(v, out)
    return out


def set_sort(msgs, keys):
    for k in keys:
        s = msgs.add().sort
        set_expr(s.expr, k["expr"])
        s.asc, s.nulls_first = bool(k["asc"]), bool(k["nulls_first"])


_JOIN = {"Inner": 0, "Left": 1, "Right": 2, "Full": 3, "LeftSemi": 4, "LeftAnti": 5, "RightSemi": 6, "RightAnti": 7}
_MODE = {"Partial": 0, "Final": 1, "FinalPartitioned": 2, "Single": 3, "SinglePartitioned": 4}


def set_join_common(j, t, left_schema, right_schema):
    for l, r in t["on"]:
        on = j.on.add()
        set_expr(on.left, l)
        set_expr(on.right, r)
    j.join_type = _JOIN[t["join_type"]]
    if t.get("null_equals_null"):
        j.null_equality = 1     # NullEquality::NULL_EQUALS_NULL (datafusion_common.proto:98-101)
    if "filter" in t:
        used = cols_of(t["filter"], [])
        nl = len(left_schema)
        remap = {}
        for k, c in enumerate(used):
            remap[c] = k
            ci = j.filter.column_indices.add()
            ci.index = c if c < nl else c - nl
            ci.side = 0 if c < nl else 1
            f = (left_schema + right_schema)[c]
            fc = j.filter.schema.columns.add()
            fc.name = f["name"]
            set_type(fc.arrow_type, f["type"])
            fc.nullable = bool(f["nullable"])
        set_expr(j.filter.expression, t["filter"], remap)


def set_plan(msg, t, o):
    """t: typed node (b200_plan_typed_json), o: the original IR node (for what typing drops: scan table schemas)."""
    op = t["op"]
    if op in ("DataSourceExec", "Scan", "MemoryScan"):
        conf = msg.parquet_scan.base_conf
        conf.file_groups.add().files.add().path = f"/data/tpch/{t['table']}/part-0.parquet"
        set_schema(conf.schema, o["schema"])
        proj = o.get("projection")
        if proj is not None:
            conf.projection.extend(proj)
        conf.object_store_url = "file://"
    elif op in ("ShuffleReaderExec", "UnresolvedShuffleExec"):
        b = C("ballista.protobuf.BallistaPhysicalPlanNode")()
        if op == "ShuffleReaderExec":
            r = b.shuffle_reader
            r.stage_id = t["stage_id"]
            # two output partitions, each with the map outputs of two executors (what the scheduler resolves an
            # UnresolvedShuffleExec into, execution_graph / execution_stage)
            for out_p in range(2):
                part = r.partition.add()
                for m in range(2):
                    loc = part.location.add()
                    loc.map_partition_id = m
                    loc.partition_id.job_id, loc.partition_id.stage_id, loc.partition_id.partition_id = "job", t["stage_id"], out_p
                    loc.executor_meta.id, loc.executor_meta.host, loc.executor_meta.port = f"exec-{m}", f"10.0.0.{m + 1}", 50050 + m
                    loc.partition_stats.num_rows, loc.partition_stats.num_batches, loc.partition_stats.num_bytes = 1000 + out_p, 1, 16000 + m
                    if m == 1:
                        loc.file_id = 7
                    loc.is_sort_shuffle = bool(m)
            r.upstream_partition_count = 2
        else:
            r = b.unresolved_shuffle
            r.stage_id = t["stage_id"]
        set_schema(r.schema, t["schema"])
        r.partitioning.unknown = 1
        r.broadcast = bool(t["broadcast"])
        msg.extension.node = b.SerializeToString()
    elif op == "FilterExec":
        f = msg.filter
        set_plan(f.input, t["input"], o["input"])
        set_expr(f.expr, t["predicate"])
        f.default_filter_selectivity = 20
        if "projection" in t:
            f.projection.extend(t["projection"])
        if "fetch" in t:
            f.fetch = t["fetch"]
    elif op == "ProjectionExec":
        p = msg.projection
        set_plan(p.input, t["input"], o["input"])
        for ne in t["exprs"]:
            set_expr(p.expr.add(), ne["expr"])
            p.expr_name.append(ne["name"])
    elif op == "AggregateExec":
        a = msg.aggregate
        set_plan(a.input, t["input"], o["input"])
        a.mode = _MODE[t["mode"]]
        final = t["mode"] in ("Final", "FinalPartitioned")
        for g in t["group_by"]:
            set_expr(a.group_expr.add(), g["expr"])
            a.group_expr_name.append(g["name"])
            a.null_expr.add().literal.null_value.NONE.SetInParent()
            a.groups.append(False)
        if final:
            # the reference repeats the partial stage's argument expressions and input schema in the final node; a stage plan
            # of the IR only keeps their types, so the fixture states "column i of type input_type_i" -- the decoder types
            # whatever expression it finds against input_schema the same way
            fields = [{"name": f"__arg{i}", "type": ag["input_type"], "nullable": True} for i, ag in enumerate(t["aggr"])]
            set_schema(a.input_schema, fields)
        else:
            set_schema(a.input_schema, t["input"]["schema"])
        for i, ag in enumerate(t["aggr"]):
            ae = a.aggr_expr.add().aggregate_expr
            ae.user_defined_aggr_function = ag["fn"]
            if final:
                c = ae.expr.add().column
                c.name, c.index = f"__arg{i}", i
            elif ag["args"]:
                set_expr(ae.expr.add(), ag["args"][0])
            else:
                ae.expr.add().literal.int64_value = 1      # COUNT(*) = count(Int64(1))
            ae.human_display = ag["name"]
            a.aggr_expr_name.append(ag["name"])
            a.filter_expr.add()
    elif op in ("HashJoinExec", "SortMergeJoinExec"):
        smj = op == "SortMergeJoinExec"
        j = msg.sort_merge_join if smj else msg.hash_join
        set_plan(j.left, t["left"], o["left"])
        set_plan(j.right, t["right"], o["right"])
        set_join_common(j, t, t["left"]["schema"], t["right"]["schema"])
        if smj:
            for k in t.get("sort_keys", []):
                so = j.sort_options.add()
                so.asc, so.nulls_first = bool(k["asc"]), bool(k["nulls_first"])
        else:
            j.partition_mode = {"CollectLeft": 0, "Partitioned": 1}[t["mode"]]
            if "projection" in t:
                j.projection.extend(t["projection"])
    elif op in ("SortExec", "SortPreservingMergeExec"):
        s = msg.sort if op == "SortExec" else msg.sort_preserving_merge
        set_plan(s.input, t["input"], o["input"])
        set_sort(s.expr, t["expr"])
        s.fetch = t.get("fetch", -1)
        if op == "SortExec":
            s.preserve_partitioning = bool(t["preserve_partitioning"])
    elif op == "CoalesceBatchesExec":
        set_plan(msg.coalesce_batches.input, t["input"], o["input"])
        msg.coalesce_batches.target_batch_size = 8192
    elif op == "CoalescePartitionsExec":
        set_plan(msg.merge.input, t["input"], o["input"])
    elif op == "RepartitionExec":
        set_plan(msg.repartition.input, t["input"], o["input"])
        msg.repartition.partitioning.round_robin = 8
    elif op in ("GlobalLimitExec", "LocalLimitExec"):
        if op == "GlobalLimitExec":
            set_plan(msg.global_limit.input, t["input"], o["input"])
            msg.global_limit.skip, msg.global_limit.fetch = t["skip"], t["fetch"]
        else:
            set_plan(msg.local_limit.input, t["input"], o["input"])
            msg.local_limit.fetch = t["fetch"]
    elif op in ("ShuffleWriterExec", "SortShuffleWriterExec"):
        b = C("ballista.protobuf.BallistaPhysicalPlanNode")()
        w = b.sort_shuffle_writer if op == "SortShuffleWriterExec" else b.shuffle_writer
        w.job_id, w.stage_id = t["job_id"], t["stage_id"]
        if "partitioning" in t:
            for h in t["partitioning"]["hash"]:
                set_expr(w.output_partitioning.hash_expr.add(), h)
            w.output_partitioning.partition_count = t["partitioning"]["n"]
        if op == "SortShuffleWriterExec":
            w.batch_size = 8192
        msg.extension.node = b.SerializeToString()     # `input: None` inside; the child travels in `inputs`
        set_plan(msg.extension.inputs.add(), t["input"], o["input"])
    else:
        raise ValueError(f"operator {op}")


def encode(ir_text):
    from ballista_b200 import engine
    typed = json.loads(engine.plan_typed_json(ir_text))
    node = C("datafusion.PhysicalPlanNode")()
    set_plan(node, typed, json.loads(ir_text))
    return node.SerializeToString()


def extra_cases():
    """Shapes the TPC-H plans do not contain."""
    from ballista_b200 import plan as P
    c = P.col
    sch = [P.field("k", "i64"), P.field("g", "utf8", True), P.field("x", P.dec(15, 2), True), P.field("y", "f64", True),
           P.field("d", "date32"), P.field("b", "bool", True), P.field("n", "i32", True)]
    scan = P.scan("t", sch)
    out = {}
    # Partial and Final in one stage, the final node carrying the original expressions (the reference's own shape)
    part = P.aggregate("Partial", [(c(1), "g")], [P.agg("avg", P.binop("*", c(2), c(2)), "a"), P.agg("sum", c(3), "s"), P.agg("count", None, "n"),
                                                  P.agg("min", c(4), "lo"), P.agg("max", c(6), "hi")], scan)
    fin = P.aggregate("Final", [(c(0), "g")], [P.agg("avg", None, "a", P.dec(31, 4)), P.agg("sum", None, "s"), P.agg("count", None, "n"),
                                              P.agg("min", None, "lo"), P.agg("max", None, "hi")], part)
    out["agg_partial_final"] = P.shuffle_writer(fin, 1)
    # every expression form
    pred = P.and_(P.or_(P.binop(">=", c(4), P.lit_date("1995-01-01")), P.is_null(c(2))), P.not_(P.in_list(c(0), [P.lit_i64(1), P.lit_i64(2)])),
                  P.like(c(1), "%ab_c%"), P.is_not_null(c(5)), P.binop("<>", P.neg(c(6)), P.lit_i32(-3)),
                  P.in_list(c(1), [P.lit_utf8("x"), P.lit_utf8("y\"z")], negated=True))
    proj = P.project([(P.case([[P.binop("<", c(3), P.lit_f64(0.5)), P.lit_dec(-12345, 15, 2)]], P.lit_null(P.dec(15, 2))), "cs"),
                      (P.cast(c(0), "f64"), "kf"), (P.fn("substr", c(1), P.lit_i64(2), P.lit_i64(3)), "sub"),
                      (P.fn("date_part_year", c(4)), "yr"), (P.binop("%", c(0), P.lit_i64(7)), "m"),
                      (P.binop("/", c(2), P.lit_dec(3, 10, 0)), "q"), (P.lit_bool(True), "t"), (P.binop("-", c(3), P.lit_f64(1.25e-3)), "f")],
                     P.filter_(pred, scan, projection=[0, 1, 2, 3, 4, 5, 6]))
    out["expressions"] = P.shuffle_writer(P.sort([P.sort_key(c(1), False), P.sort_key(c(0), True, True)], proj, fetch=10), 2, [c(1), c(6)], 5)
    # limits, merges, coalesce, unpartitioned plain writer, sort-merge join with a filter, outer joins
    l = P.scan("l", [P.field("a", "i64"), P.field("b", "utf8", True)])
    r = P.scan("r", [P.field("c", "i64"), P.field("d", P.dec(10, 2), True)])
    smj = P.sort_merge_join(l, r, [[c(0), c(0)]], "Left", filter=P.binop(">", c(3), P.lit_dec(100, 10, 2)))
    out["smj_limits"] = P.shuffle_writer(P.limit(P.coalesce_partitions(P.coalesce_batches({"op": "RepartitionExec", "input": smj})), 5, 2), 3, sort_shuffle=False)
    full = P.hash_join(l, r, [[c(0), c(0)]], "Full", "Partitioned", filter=P.binop("<>", c(1), P.lit_utf8("z")), projection=[3, 1])
    out["full_join"] = P.shuffle_writer(P.sort_preserving_merge([P.sort_key(c(1))], P.limit(full, 7, global_=False), fetch=3), 4, [c(0)], 3, sort_shuffle=False)
    return out


def main():
    from ballista_b200 import tpch
    cases = []
    for q in sorted(tpch.QUERIES, key=lambda s: int(s[1:])):
        for st in tpch.QUERIES[q][1](4):
            ir = st.json("job")
            cases.append({"name": f"{q}/stage{st.stage_id}", "ir": ir, "proto_b64": base64.b64encode(encode(ir)).decode()})
    for name, plan in extra_cases().items():
        p = dict(plan)
        ir = json.dumps(p, separators=(",", ":"))
        cases.append({"name": f"extra/{name}", "ir": ir, "proto_b64": base64.b64encode(encode(ir)).decode()})
    # whole tasks as an executor receives them (ballista.proto:518-542), wrapping the q5 lineitem shuffle stage
    plan = base64.b64decode([c for c in cases if c["name"] == "q5/stage5"][0]["proto_b64"])
    td = C("ballista.protobuf.TaskDefinition")()
    td.task_id, td.task_attempt_num, td.job_id, td.stage_id, td.stage_attempt_num, td.partition_id = 17, 1, "job-a1b2", 5, 0, 3
    td.plan, td.session_id, td.launch_time = plan, "sess-9", 1726000000123
    for k, v in (("datafusion.execution.batch_size", "4096"), ("ballista.job.name", "tpch q5")):
        kv = td.props.add()
        kv.key, kv.value = k, v
    td.props.add().key = "flag.without.value"
    mt = C("ballista.protobuf.MultiTaskDefinition")()
    for tid, part in ((40, 0), (41, 1), (42, 2)):
        t = mt.task_ids.add()
        t.task_id, t.task_attempt_num, t.partition_id = tid, 0, part
    mt.job_id, mt.stage_id, mt.stage_attempt_num, mt.plan, mt.session_id, mt.launch_time = "job-a1b2", 5, 2, plan, "sess-9", 1726000000456
    kv = mt.props.add()
    kv.key, kv.value = "datafusion.execution.batch_size", "1024"
    tasks = {
        "single_b64": base64.b64encode(td.SerializeToString()).decode(),
        "single": {"job_id": "job-a1b2", "stage_id": 5, "stage_attempt_num": 0, "session_id": "sess-9", "launch_time": 1726000000123,
                   "tasks": [{"task_id": 17, "task_attempt_num": 1, "partition_id": 3}],
                   "props": {"datafusion.execution.batch_size": "4096", "ballista.job.name": "tpch q5", "flag.without.value": ""}},
        "multi_b64": base64.b64encode(mt.SerializeToString()).decode(),
        "multi": {"job_id": "job-a1b2", "stage_id": 5, "stage_attempt_num": 2, "session_id": "sess-9", "launch_time": 1726000000456,
                  "tasks": [{"task_id": 40, "task_attempt_num": 0, "partition_id": 0}, {"task_id": 41, "task_attempt_num": 0, "partition_id": 1},
                            {"task_id": 42, "task_attempt_num": 0, "partition_id": 2}],
                  "props": {"datafusion.execution.batch_size": "1024"}},
    }
    # the way back: TaskStatus messages as ballista/executor/src/lib.rs:101-152 + ballista/core/src/error.rs:205-256 build them
    statuses = []
    parts = [dict(partition_id=0, num_batches=2, num_rows=10000, num_bytes=480000, file_id=3, is_sort_shuffle=1),
             dict(partition_id=3, num_batches=1, num_rows=17, num_bytes=816, file_id=-1, is_sort_shuffle=0)]
    mets = [dict(name="SortShuffleWriterExec", output_rows=10017, input_rows=10017, elapsed_compute_ns=123456, bytes_read=480816, bytes_written=480816, kernel_launches=4),
            dict(name="FilterExec", output_rows=10017, input_rows=60000, elapsed_compute_ns=0, bytes_read=2880000, bytes_written=0, kernel_launches=1)]
    base = dict(task_id=17, stage_id=5, stage_attempt_num=1, partition_id=3, launch_time=1726000000123, start_exec_time=1726000000200, end_exec_time=1726000000950)
    for name, status, extra in (("successful", 0, {}), ("fetch_failed", -5, dict(fetch_executor_id="exec-7", fetch_map_stage_id=4, fetch_map_partition_id=9,
                                                                              error_message="partition 9 of stage 4 is gone")),
                                ("killed", -6, dict(error_message="task cancelled")), ("execution_error", -3, dict(error_message="Execution: Arithmetic overflow")),
                                ("zero_ids", 0, dict(task_id=0, partition_id=0, stage_attempt_num=0))):
        r = dict(base, status=status, **extra)
        ts = C("ballista.protobuf.TaskStatus")()
        ts.task_id, ts.job_id, ts.stage_id, ts.stage_attempt_num, ts.partition_id = r["task_id"], "job-a1b2", r["stage_id"], r["stage_attempt_num"], r["partition_id"]
        ts.launch_time, ts.start_exec_time, ts.end_exec_time = r["launch_time"], r["start_exec_time"], r["end_exec_time"]
        use_parts = parts if status == 0 else []
        if status == 0:
            ts.successful.executor_id = "exec-1"
            for p in use_parts:
                sp = ts.successful.partitions.add()
                sp.partition_id, sp.num_batches, sp.num_rows, sp.num_bytes = p["partition_id"], p["num_batches"], p["num_rows"], p["num_bytes"]
                if p["file_id"] >= 0:
                    sp.file_id = p["file_id"]
                sp.is_sort_shuffle = bool(p["is_sort_shuffle"])
        elif status == -5:
            ts.failed.error = r["error_message"]
            fe = ts.failed.fetch_partition_error
            fe.executor_id, fe.map_stage_id, fe.map_partition_id = r["fetch_executor_id"], r["fetch_map_stage_id"], r["fetch_map_partition_id"]
        elif status == -6:
            ts.failed.error = r["error_message"]
            ts.failed.task_killed.SetInParent()
        else:
            ts.failed.error = "Task failed due to runtime execution error: " + r["error_message"]
            ts.failed.execution_error.SetInParent()
        for m in mets:
            ms = ts.metrics.add()
            ms.metrics.add().output_rows = m["output_rows"]
            ms.metrics.add().elapse_time = m["elapsed_compute_ns"]
            ms.metrics.add().output_bytes = m["bytes_written"]
            for nm in ("input_rows", "bytes_read", "kernel_launches"):
                c = ms.metrics.add().count
                c.name, c.value = nm, m[nm]
        statuses.append({"name": name, "result": r, "partitions": use_parts, "metrics": mets, "executor_id": "exec-1", "job_id": "job-a1b2",
                         "expected_b64": base64.b64encode(ts.SerializeToString()).decode()})
    with open(os.path.join(HERE, "proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_proto_plans.py", "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto",
                   "cases": cases, "tasks": tasks, "statuses": statuses}, fh, indent=0)
    print(len(cases), "plans,", sum(len(c["proto_b64"]) for c in cases) * 3 // 4, "proto bytes")
    write_reference_checks(cases)
    write_random_plans()


def write_reference_checks(cases):
    """What google.protobuf, given the reference's message definitions, reports for every fixture (tests/golden/proto_plans_checked.json):
    the fixture parses completely and re-serialises byte-identically, which oneof its root and its Ballista node hold, and the field
    numbers involved, so that tests/test_plan_proto.py can check the fixtures without the .proto files."""
    import hashlib
    P, E, B = C("datafusion.PhysicalPlanNode"), C("datafusion.PhysicalExtensionNode"), C("ballista.protobuf.BallistaPhysicalPlanNode")
    checked = []
    for c in cases:
        raw = base64.b64decode(c["proto_b64"])
        m = P()
        m.ParseFromString(raw)
        b = B()
        b.ParseFromString(m.extension.node)
        checked.append({"name": c["name"], "sha256": hashlib.sha256(raw).hexdigest(), "reserialises_identically": m.SerializeToString() == raw,
                        "root_oneof": m.WhichOneof("PhysicalPlanType"), "ballista_oneof": b.WhichOneof("PhysicalPlanType"),
                        "extension_inputs": len(m.extension.inputs)})
    fields = {"PhysicalPlanNode.extension": P.DESCRIPTOR.fields_by_name["extension"].number,
              "PhysicalExtensionNode.node": E.DESCRIPTOR.fields_by_name["node"].number,
              "PhysicalExtensionNode.inputs": E.DESCRIPTOR.fields_by_name["inputs"].number,
              "BallistaPhysicalPlanNode.shuffle_writer": B.DESCRIPTOR.fields_by_name["shuffle_writer"].number,
              "BallistaPhysicalPlanNode.sort_shuffle_writer": B.DESCRIPTOR.fields_by_name["sort_shuffle_writer"].number}
    with open(os.path.join(HERE, "proto_plans_checked.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_proto_plans.py", "field_numbers": fields, "cases": checked}, fh, indent=0)


def write_random_plans():
    """The seeded random plans of tests/test_plan_proto_random.py, encoded (tests/golden/random_proto_plans.json.gz: seed -> bytes)."""
    import gzip
    sys.path.insert(0, os.path.dirname(HERE))
    import test_plan_proto_random as T
    from ballista_b200 import engine
    protos = {}
    for seed in range(T.N_SEEDS):
        ir = json.dumps(T._plan(seed), separators=(",", ":"))
        try:
            engine.plan_typed_json(ir)
        except engine.B200Error:
            continue
        protos[str(seed)] = base64.b64encode(encode(ir)).decode()
    with gzip.GzipFile(os.path.join(HERE, "random_proto_plans.json.gz"), "wb", mtime=0) as fh:
        fh.write(json.dumps({"generated_by": "tests/golden/make_proto_plans.py", "protos": protos}, separators=(",", ":")).encode())
    print(len(protos), "random plans")


if __name__ == "__main__":
    main()
