"""Generate tests/golden/first_last_proto_plans.json: first_value / last_value plans as the protobuf bytes a Ballista
scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_first_last_proto_plans.py      (commit the output)

Single and Partial -> FinalPartitioned with a key, Partial -> Final without one, a DISTINCT ON shape (one first_value per
column under one ordering), and the refused cases (too many ordering keys, ordering_req on SUM); encoded as
datafusion.PhysicalPlanNode exactly as make_proto_plans.py encodes its fixtures (message classes built from the
reference's .proto files by protoc_lite.py).  The ordering goes into PhysicalAggregateExprNode.ordering_req (bare
PhysicalSortExprNodes) and IGNORE NULLS into ignore_nulls.  A Final's ordering_req names the Final's own argument column:
the decoder takes only the directions from it.
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

_set_plan = M.set_plan


def set_plan(msg, t, o):
    _set_plan(msg, t, o)
    if t["op"] != "AggregateExec":
        return
    final = t["mode"] in ("Final", "FinalPartitioned")
    for i, ta in enumerate(t["aggr"]):
        ae = msg.aggregate.aggr_expr[i].aggregate_expr
        for k in ta.get("order_by", []):
            s = ae.ordering_req.add()
            M.set_expr(s.expr, {"col": i} if final else k["expr"])
            s.asc, s.nulls_first = bool(k["asc"]), bool(k["nulls_first"])
        if ta.get("ignore_nulls"):
            ae.ignore_nulls = True


M.set_plan = set_plan


def cases():
    from ballista_b200 import plan as P
    from first_last_cases import stages
    c = P.col
    sch = [P.field("k", "i32", True), P.field("x", "i64", True), P.field("o", "f64", True), P.field("s", "utf8", True)]
    src = P.scan("t", sch)
    out = []
    shapes = [("single", [(c("k"), "k")], [], "Single"), ("partial_final_keyed", [(c("k"), "k")], [P.field("k", "i32", True)], "Partial"),
              ("partial_final_scalar", [], [], "Partial")]
    aggsets = {
        "first_value": [("first_value", c("x"), "i64", [(c("o"), True, False)], False, "f")],
        "last_value_desc_ignore_nulls": [("last_value", c("s"), "utf8", [(c("o"), False, True), (c("x"), True, True)], True, "l")],
        "unordered": [("first_value", c("o"), "f64", [], False, "f"), ("last_value", c("x"), "i64", [], True, "l")],
    }
    for an, aggs in aggsets.items():
        for shape, keys, kf, mode in shapes:
            for st in stages(src, aggs, keys, kf, mode):
                out.append((f"{an}/{shape}/stage{st.stage_id}", st.json("job"), True))
    # SELECT DISTINCT ON (k) x, o, s ... ORDER BY k, o DESC: one first_value per column under one ordering
    don = [("first_value", c(n), t, [(c("k"), True, False), (c("o"), False, True)], False, n) for n, t in (("x", "i64"), ("o", "f64"), ("s", "utf8"))]
    for st in stages(src, don, [(c("k"), "k")], [P.field("k", "i32", True)], "Partial"):
        out.append((f"distinct_on/partial_final_keyed/stage{st.stage_id}", st.json("job"), True))
    return out


def refused():
    """(name, encoded bytes, expected message fragment): typed stand-ins encoded, then the refused part added to the
    message -- ordering_req on SUM, and a fifth ordering key on first_value"""
    from ballista_b200 import plan as P
    from ballista_b200.plan import Stage
    c = P.col
    sch = [P.field("k", "i32", True), P.field("x", "i64", True), P.field("o", "f64", True), P.field("s", "utf8", True)]
    src = P.scan("t", sch)
    out = []

    def encoded_with_key(plan):  # ShuffleWriterExec extension -> its input -> the aggregate's first expression
        node = M.C("datafusion.PhysicalPlanNode")()
        node.ParseFromString(M.encode(Stage(1, P.shuffle_writer(plan, 1)).json("job")))
        s = node.extension.inputs[0].aggregate.aggr_expr[0].aggregate_expr.ordering_req.add()
        s.expr.column.name, s.expr.column.index = "o", 2
        s.asc = True
        return node.SerializeToString()
    plan = P.aggregate("Single", [(c("k"), "k")], [P.agg("sum", c("x"), "s")], src)
    out.append(("sum_with_ordering_req", encoded_with_key(plan), "ordered aggregates are not supported"))
    four = [P.sort_key(c("o")), P.sort_key(c("x")), P.sort_key(c("k")), P.sort_key(c("s"))]
    plan = P.aggregate("Single", [(c("k"), "k")], [P.agg("first_value", c("x"), "f", order_by=four)], src)
    out.append(("five_ordering_keys", encoded_with_key(plan), "ordering keys"))
    return out


def main():
    res = []
    for name, ir, runs in cases():
        res.append({"name": name, "ir": ir, "runs": runs, "proto_b64": base64.b64encode(M.encode(ir)).decode()})
    for name, data, msg in refused():
        res.append({"name": "refused/" + name, "refusal": msg, "proto_b64": base64.b64encode(data).decode()})
    with open(os.path.join(HERE, "first_last_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_first_last_proto_plans.py",
                   "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto", "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
