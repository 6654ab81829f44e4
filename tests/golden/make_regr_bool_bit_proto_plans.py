"""Generate tests/golden/regr_bool_bit_proto_plans.json: regr_* / bool_* / bit_* plans as the protobuf bytes a Ballista
scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_regr_bool_bit_proto_plans.py      (commit the output)

Every one of the 14 names (some spelled in upper case: the decoder lower-cases what the function registry resolves),
Single and Partial -> FinalPartitioned with a key, and Partial -> Final without one, mixed with SUM; encoded as
datafusion.PhysicalPlanNode exactly as make_stat_proto_plans.py encodes its fixtures (message classes built from the
reference's .proto files by protoc_lite.py).  regr_* carries both arguments in PhysicalAggregateExprNode.expr.
"""
import base64
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_stat_proto_plans as S  # noqa: E402  (installs the two-argument set_plan on make_proto_plans)

_stat_set_plan = S.M.set_plan


def set_plan(msg, t, o):
    """A Final that carries its aggregates' original arguments and the Partial's input schema (as Ballista ships it) is
    encoded with exactly those, both regr_* arguments included"""
    _stat_set_plan(msg, t, o)
    if t["op"] != "AggregateExec" or t["mode"] not in ("Final", "FinalPartitioned") or "input_schema" not in o:
        return
    a = msg.aggregate
    a.input_schema.Clear()
    S.M.set_schema(a.input_schema, o["input_schema"])
    names = [f["name"] for f in o["input_schema"]]

    def by_index(e):  # columns named in the IR, by position in the input schema as the protobuf has them
        if isinstance(e, dict):
            return {k: (names.index(v) if k == "col" and isinstance(v, str) else by_index(v)) for k, v in e.items()}
        return [by_index(v) for v in e] if isinstance(e, list) else e
    for i, oa in enumerate(o["aggr"]):
        ae = a.aggr_expr[i].aggregate_expr
        del ae.expr[:]
        for e in oa["args"]:
            S.M.set_expr(ae.expr.add(), by_index(e))


S.M.set_plan = set_plan

NAMES = ["regr_slope", "REGR_INTERCEPT", "regr_count", "Regr_R2", "regr_avgx", "regr_avgy", "REGR_SXX", "regr_syy", "regr_sxy",
         "bool_and", "BOOL_OR", "bit_and", "Bit_Or", "BIT_XOR"]


def cases():
    from ballista_b200 import plan as P
    from regr_bool_bit_cases import stages
    c = P.col
    sch = [P.field("k", "i32", True), P.field("x", "i64", True), P.field("y", P.dec(15, 2), True), P.field("z", "f64", False),
           P.field("b", "bool", True), P.field("u", "u16", True)]
    out = []
    for fn in NAMES:
        f = fn.lower()
        a = (f, c("y"), c("x"), "r", None) if f.startswith("regr") else (f, c("b"), None, "r", "bool") if f.startswith("bool") else (f, c("u"), None, "r", "u16")
        aggs = [a, ("sum", c("z"), None, "s", None)]
        shapes = [("single", [(c("k"), "k")], [], "Single"), ("partial_final_keyed", [(c("k"), "k")], [P.field("k", "i32", True)], "Partial"),
                  ("partial_final_scalar", [], [], "Partial")]
        for shape, keys, kf, mode in shapes:
            for st in stages(P.scan("t", sch), aggs, keys, kf, mode):
                out.append((f"{fn}/{shape}/stage{st.stage_id}", st.json("job"), fn))
    # all nine over one pair, Partial -> FinalPartitioned: one AggregateExec per stage
    nine = [(f.lower(), c("y"), c("x"), f.lower(), None) for f in NAMES[:9]]
    for st in stages(P.scan("t", sch), nine, [(c("k"), "k")], [P.field("k", "i32", True)], "Partial"):
        out.append((f"regr_all/partial_final_keyed/stage{st.stage_id}", st.json("job"), "regr_slope"))
    return out


def main():
    res = []
    for name, ir, spelled in cases():
        S.SPELLING.clear()
        S.SPELLING[spelled.lower()] = spelled
        res.append({"name": name, "ir": ir, "fn": spelled, "proto_b64": base64.b64encode(S.M.encode(ir)).decode()})
    with open(os.path.join(HERE, "regr_bool_bit_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_regr_bool_bit_proto_plans.py",
                   "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto", "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
