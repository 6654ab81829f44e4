"""Generate tests/golden/stat_proto_plans.json: VAR / STDDEV / COVAR / CORR plans as the protobuf bytes a Ballista scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_stat_proto_plans.py      (commit the output)

Every name and alias (some spelled in upper case: the decoder lower-cases what the function registry resolves), Single and
Partial -> FinalPartitioned with a key, and Partial -> Final without one, mixed with SUM; encoded as datafusion.PhysicalPlanNode
exactly as make_proto_plans.py encodes its fixtures (message classes built from the reference's .proto files by
protoc_lite.py).  The aggregate keeps the name the plan was written with, and COVAR / CORR carry both arguments in
PhysicalAggregateExprNode.expr.
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
    for i, (ta, oa) in enumerate(zip(t["aggr"], o["aggr"])):
        ae = msg.aggregate.aggr_expr[i].aggregate_expr
        ae.user_defined_aggr_function = SPELLING.get(oa["fn"], oa["fn"])
        if not final and len(ta["args"]) > 1:
            M.set_expr(ae.expr.add(), ta["args"][1])


M.set_plan = set_plan   # children of the other operators recurse through the module's name
SPELLING = {}           # IR name (lower case) -> the spelling the protobuf carries for the case being encoded

NAMES = ["var", "VAR_SAMP", "var_sample", "var_pop", "Var_Population", "stddev", "STDDEV_SAMP", "stddev_pop",
         "covar", "covar_samp", "COVAR_POP", "corr"]


def cases():
    from ballista_b200 import plan as P
    from stat_cases import stat_stages
    c = P.col
    sch = [P.field("k", "i32", True), P.field("x", "i64", True), P.field("y", P.dec(15, 2), True), P.field("z", "f64", False)]
    out = []
    for fn in NAMES:
        two = fn.lower() in ("covar", "covar_samp", "covar_pop", "corr")
        agg = [(fn, c("x"), c("y") if two else None, "r")]
        extra = [("sum", c("z"), "s", [P.field("s[sum]", "f64", True)], None)]
        shapes = [("single", [(c("k"), "k")], [], "Single"), ("partial_final_keyed", [(c("k"), "k")], [P.field("k", "i32", True)], "Partial"),
                  ("partial_final_scalar", [], [], "Partial")]
        for shape, keys, kf, mode in shapes:
            for st in stat_stages(P.scan("t", sch), [(fn.lower(), *a[1:]) for a in agg], keys, kf, mode, extra=extra):
                out.append((f"{fn}/{shape}/stage{st.stage_id}", st.json("job"), fn))
    return out


def main():
    res = []
    for name, ir, spelled in cases():
        SPELLING.clear()
        SPELLING[spelled.lower()] = spelled
        res.append({"name": name, "ir": ir, "fn": spelled, "proto_b64": base64.b64encode(M.encode(ir)).decode()})
    with open(os.path.join(HERE, "stat_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_stat_proto_plans.py", "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto",
                   "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
