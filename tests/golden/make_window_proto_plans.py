"""Generate tests/golden/window_proto_plans.json: window plans (WindowAggExec / BoundedWindowAggExec) as the protobuf bytes a
Ballista scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_window_proto_plans.py      (commit the output)

Encoded as datafusion.PhysicalPlanNode exactly as make_proto_plans.py encodes its fixtures (message classes built from the
reference's .proto files by protoc_lite.py), plus the window node: PhysicalPlanNode.window = 15, WindowAggExecNode
{ input = 1, window_expr = 2, partition_keys = 5, sorted = 9 for BoundedWindowAggExec, no mode for WindowAggExec }.

Unpinned datafusion-proto 53 `to_proto` conventions, restated here:
  - window functions travel by name: user_defined_window_function = 10 for row_number, rank, dense_rank, percent_rank,
    cume_dist, ntile, lag, lead, first_value, last_value, nth_value; user_defined_aggr_function = 3 for the aggregates;
  - their arguments are the SQL arguments as physical expressions: ntile(Int64 n), lag / lead(x, Int64 k, default),
    nth_value(x, Int64 n), COUNT(*) as count(Int64(1));
  - every expression carries its frame (WindowFrame = 7); ROWS offsets are UInt64 scalars and an UNBOUNDED bound is a NULL
    scalar (null_value = 33, here of type UInt64) under PRECEDING / FOLLOWING.

The refused cases are encoded from a plan the typing accepts, then changed in the bytes (a flag set, the frame units or a bound
rewritten, the function renamed, the input order mode switched), since the typing refuses them.
"""
import base64
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_proto_plans as M  # noqa: E402

WINDOW_FNS = {"row_number", "rank", "dense_rank", "percent_rank", "cume_dist", "ntile", "lag", "lead", "first_value", "last_value", "nth_value"}
_BOUND = {"current_row": 0, "preceding": 1, "unbounded_preceding": 1, "following": 2, "unbounded_following": 2}
_set_plan = M.set_plan


def _i64(v):
    return {"lit": {"t": "i64", "v": int(v)}}


def _args(we):
    """The SQL arguments back from the typed expression (the typing folds the literal ones into "n" / "default")."""
    fn, a = we["fn"], we["args"]
    if fn == "ntile":
        return [_i64(we["n"])]
    if fn == "nth_value":
        return [a[0], _i64(we["n"])]
    if fn in ("lag", "lead"):
        k = we["n"] if fn == "lead" else -we["n"]
        return [a[0], _i64(k)] + ([we["default"]] if "default" in we else [])
    if fn == "count" and not a:
        return [_i64(1)]
    return a


def _set_bound(msg, b):
    msg.window_frame_bound_type = _BOUND[b["kind"]]
    if b["kind"].startswith("unbounded"):
        M.set_type(msg.bound_value.null_value, "u64")
    elif b["kind"] != "current_row":
        msg.bound_value.uint64_value = int(b["n"])


def set_plan(msg, t, o):
    if t["op"] != "WindowAggExec":
        return _set_plan(msg, t, o)
    w = msg.window
    set_plan(w.input, t["input"], o["input"])
    for k in t["partition_keys"]:
        M.set_expr(w.partition_keys.add(), k)
    if t["mode"] == "sorted":
        w.sorted.SetInParent()
    for we in t["window_expr"]:
        e = w.window_expr.add()
        if we["fn"] in WINDOW_FNS:
            e.user_defined_window_function = we["fn"]
        else:
            e.user_defined_aggr_function = we["fn"]
        for a in _args(we):
            M.set_expr(e.args.add(), a)
        for k in t["partition_keys"]:
            M.set_expr(e.partition_by.add(), k)
        for k in t["order_by"]:
            s = e.order_by.add()
            M.set_expr(s.expr, k["expr"])
            s.asc, s.nulls_first = bool(k["asc"]), bool(k["nulls_first"])
        f = we["frame"]
        e.window_frame.window_frame_units = {"rows": 0, "range": 1}[f["units"]]
        _set_bound(e.window_frame.start_bound, f["start"])
        _set_bound(e.window_frame.bound, f["end"])
        e.name = we["name"]


M.set_plan = set_plan   # children of the other operators recurse through the module's name


def _window_node(node):
    """The window node of a stage: ShuffleWriter (extension) -> [Filter ->] WindowAggExec."""
    n = node.extension.inputs[0]
    while n.WhichOneof("PhysicalPlanType") != "window":
        n = n.filter.input
    return n.window


def cases():
    from ballista_b200 import plan as P
    import window_cases as W
    c = P.col
    scan = P.scan("wt", W.SCHEMA)
    pk, ob = [c("g")], [P.sort_key(c("o"))]

    def win(exprs, input_=scan, mode="sorted", part=pk, order=ob):
        return P.window([dict(w, partition_by=part, order_by=order) for w in exprs], input_, part, mode)

    ranking = [P.win("row_number", "rn"), P.win("rank", "rk"), P.win("dense_rank", "dr"), P.win("percent_rank", "pr"),
               P.win("cume_dist", "cd"), P.win("ntile", "nt", [P.lit_i64(4)]), P.win("lag", "lg", [c("i64")]),
               P.win("lead", "ld", [c("ks"), P.lit_i64(2), P.lit_utf8("none")]), P.win("lag", "lg_neg", [c("dt"), P.lit_i64(-3)]),
               P.win("lag", "lg_cast_default", [c("i32"), P.lit_i64(1), P.lit_i64(-7)])]

    def framed(tag, f):
        return [P.win("count", f"cs_{tag}", [], frame=f), P.win("count", f"cx_{tag}", [c("ks")], frame=f),
                P.win("sum", f"si_{tag}", [c("i64")], frame=f), P.win("sum", f"sd_{tag}", [c("dec")], frame=f),
                P.win("sum", f"sf_{tag}", [c("f64")], frame=f), P.win("mean", f"ad_{tag}", [c("dec")], frame=f),
                P.win("avg", f"ai_{tag}", [c("i32")], frame=f), P.win("min", f"mn_{tag}", [c("u64")], frame=f),
                P.win("max", f"mx_{tag}", [c("f64")], frame=f), P.win("first_value", f"fv_{tag}", [c("ks")], frame=f),
                P.win("last_value", f"lv_{tag}", [c("dt")], frame=f), P.win("nth_value", f"nv_{tag}", [c("dec"), P.lit_i64(2)], frame=f)]

    frames = {"range_default": None, "range_all": P.range_(P.UNBOUNDED_PRECEDING, P.UNBOUNDED_FOLLOWING),
              "range_to_end": P.range_(P.CURRENT_ROW, P.UNBOUNDED_FOLLOWING), "range_peers": P.range_(P.CURRENT_ROW, P.CURRENT_ROW),
              "rows_2p_cur": P.rows(P.preceding(2), P.CURRENT_ROW), "rows_1p_1f": P.rows(P.preceding(1), P.following(1)),
              "rows_3p_1p": P.rows(P.preceding(3), P.preceding(1)), "rows_1f_3f": P.rows(P.following(1), P.following(3)),
              "rows_cur_end": P.rows(P.CURRENT_ROW, P.UNBOUNDED_FOLLOWING), "rows_start_2f": P.rows(P.UNBOUNDED_PRECEDING, P.following(2))}
    single = [("ranking_and_offsets/bounded", win(ranking)), ("ranking/window_agg_exec", win(ranking[:5], mode=None)),
              ("no_partition", win(ranking[:3], part=[])), ("no_order", win(ranking[:5] + framed("np", None), order=[]))]
    single += [(f"frame_{k}", win(framed(k, f))) for k, f in frames.items()]
    out = []
    for name, plan in single:
        st = P.Stage(1, P.shuffle_writer(plan, 1))
        ir = st.json("job")
        out.append({"name": name, "table": "wt",
                    "stages": [{"name": f"{name}/stage1", "ir": ir, "proto_b64": base64.b64encode(M.encode(ir)).decode()}]})
    # the reference planner's window query (scheduler/src/planner.rs:1128-1178): stage 1 repartitions lineitem by
    # l_shipmode; stage 2 is SortExec(l_shipmode ASC NULLS LAST, l_shipdate DESC) -> BoundedWindowAggExec(rank() ... RANGE
    # BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW, mode Sorted) -> FilterExec(rk <= 100)
    sch = [P.field("l_orderkey", "i64"), P.field("l_linenumber", "i32"), P.field("l_shipmode", "utf8"), P.field("l_shipdate", "date32")]
    s1 = P.Stage(1, P.shuffle_writer(P.scan("lineitem", sch), 1, [c("l_shipmode")], 2))
    srt = P.sort([P.sort_key(c("l_shipmode"), True, False), P.sort_key(c("l_shipdate"), False, True)], P.shuffle_reader(1, sch))
    wpk, wob = [c("l_shipmode")], [P.sort_key(c("l_shipdate"), False, True)]
    w = P.window([P.win("rank", "rk", [], wpk, wob, P.range_(P.UNBOUNDED_PRECEDING, P.CURRENT_ROW))], srt, wpk)
    s2 = P.Stage(2, P.shuffle_writer(P.filter_(P.binop("<=", c("rk"), P.lit_i64(100)), w), 2))
    out.append({"name": "reference_planner_stage", "table": "lineitem",
                "stages": [{"name": f"reference_planner_stage/stage{s.stage_id}", "ir": s.json("job"),
                            "proto_b64": base64.b64encode(M.encode(s.json("job"))).decode()} for s in (s1, s2)]})

    # refused: a plan the typing accepts, changed in the bytes
    def frame_groups(e):
        e.window_frame.window_frame_units = 2

    def range_offset(e):
        e.window_frame.window_frame_units = 1
        e.window_frame.start_bound.bound_value.int64_value = 7

    def start_unbounded_following(e):
        e.window_frame.start_bound.window_frame_bound_type = 2
        M.set_type(e.window_frame.start_bound.bound_value.null_value, "u64")

    def end_unbounded_preceding(e):
        e.window_frame.bound.window_frame_bound_type = 1
        M.set_type(e.window_frame.bound.bound_value.null_value, "u64")

    def rename(fn):
        def f(e):
            e.user_defined_aggr_function = fn
        return f

    def set_flag(field):
        def f(e):
            setattr(e, field, True)
        return f

    def ntile_zero(e):
        e.args[0].literal.int64_value = 0

    base_sum = win([P.win("sum", "s", [c("i64")], frame=P.rows(P.preceding(1), P.CURRENT_ROW))])
    base_ntile = win([P.win("ntile", "nt", [P.lit_i64(3)])])
    bad = [("ignore_nulls", base_sum, set_flag("ignore_nulls"), None, -2, "IGNORE NULLS"),
           ("distinct", base_sum, set_flag("distinct"), None, -2, "DISTINCT window function sum (s)"),
           ("groups_frame", base_sum, frame_groups, None, -2, "GROUPS window frame of sum (s)"),
           ("range_offset", base_sum, range_offset, None, -2, "RANGE window frame with an offset bound"),
           ("string_agg", base_sum, rename("string_agg"), None, -2, "window function string_agg (s) is not supported"),
           ("var_samp", base_sum, rename("var_samp"), None, -2, "window function var_samp (s) is not supported"),
           ("linear_mode", base_sum, None, "linear", -2, "window input order mode linear"),
           ("partially_sorted_mode", base_sum, None, "partially_sorted", -2, "window input order mode partially_sorted"),
           ("start_unbounded_following", base_sum, start_unbounded_following, None, -1, "starts at UNBOUNDED FOLLOWING"),
           ("end_unbounded_preceding", base_sum, end_unbounded_preceding, None, -1, "ends at UNBOUNDED PRECEDING"),
           ("ntile_zero", base_ntile, ntile_zero, None, -1, "needs n >= 1")]
    node_cls = M.C("datafusion.PhysicalPlanNode")
    for name, plan, change, mode, code, match in bad:
        node = node_cls.FromString(M.encode(P.Stage(1, P.shuffle_writer(plan, 1)).json("job")))
        wn = _window_node(node)
        if change:
            change(wn.window_expr[0])
        if mode == "linear":
            wn.linear.SetInParent()
        elif mode == "partially_sorted":
            wn.partially_sorted.columns.append(0)
        out.append({"name": name, "refuse": {"code": code, "match": match},
                    "stages": [{"name": f"{name}/stage1", "proto_b64": base64.b64encode(node.SerializeToString()).decode()}]})
    return out


def main():
    res = cases()
    with open(os.path.join(HERE, "window_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_window_proto_plans.py", "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto",
                   "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "cases")


if __name__ == "__main__":
    main()
