"""Generate tests/golden/grouping_set_proto_plans.json: ROLLUP / CUBE / GROUPING SETS plans as the protobuf bytes a Ballista
scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_grouping_set_proto_plans.py      (commit the output)

Encoded as datafusion.PhysicalPlanNode exactly as make_proto_plans.py encodes its fixtures (message classes built from the
reference's .proto files by protoc_lite.py), plus the grouping-set fields of AggregateExecNode: groups = 9 (S x n bools,
row-major, true = the key is NULL in that set), has_grouping_set = 12, and the n NULL literals of null_expr = 8 that the base
encoder already writes.  GROUPING() arrives in the form DataFusion's analyzer leaves it: CAST(... AS Int32) over
BitwiseAnd / BitwiseShiftRight of __grouping_id and UInt8 literals, in a projection above the Final aggregate.

The refused cases (a duplicate set, too many keys, a statistical aggregate, a `groups` length that is not a multiple of the
key count) are encoded from the plan without its sets, then given the sets, since the typing refuses them.
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

M._OPS.update({"&": "BitwiseAnd", "|": "BitwiseOr", "^": "BitwiseXor", "<<": "BitwiseShiftLeft", ">>": "BitwiseShiftRight"})
_set_plan = M.set_plan
GROUPS = {}  # the flattened groups to write into the (single) Partial / Single aggregate of the plan being encoded


def set_plan(msg, t, o):
    _set_plan(msg, t, o)
    if t["op"] == "AggregateExec" and t["mode"] not in ("Final", "FinalPartitioned") and "flat" in GROUPS:
        del msg.aggregate.groups[:]
        msg.aggregate.groups.extend(GROUPS["flat"])
        msg.aggregate.has_grouping_set = True


M.set_plan = set_plan   # children of the other operators recurse through the module's name


def cases():
    from ballista_b200 import plan as P
    import golden_data as G
    c = P.col
    scan = P.scan("aggregate_test_100", G.ir_schema("aggregate_test_100"))
    aggs = [P.agg("sum", c("c4"), "sum_c4"), P.agg("count", None, "cnt"), P.agg("min", c("c13"), "min_c13"),
            P.agg("max", c("c10"), "max_c10"), P.agg("avg", c("c12"), "avg_c12"), P.agg("min", c("c12"), "min_c12")]
    u8 = lambda v: {"lit": {"t": "u8", "v": v}}  # noqa: E731
    runs = [("rollup1/single", ["c1"], P.rollup_sets(1), "Single", None),
            ("rollup2/partial_final", ["c1", "c2"], P.rollup_sets(2), "Partial", None),
            ("rollup3/single", ["c1", "c2", "c3"], P.rollup_sets(3), "Single", None),
            ("cube3/partial_final", ["c1", "c2", "c13"], P.cube_sets(3), "Partial", None),
            ("one_all_false_set/single", ["c1", "c2"], [[False, False]], "Single", None),
            ("sets_with_empty/partial_final", ["c2", "c1"], [[False, True], [True, False], [True, True]], "Partial", None),
            ("grouping_fn/partial_final", ["c1", "c2"], P.rollup_sets(2), "Partial",
             [("grouping(c1)", P.cast(P.binop("&", P.binop(">>", c(2), u8(1)), u8(1)), "i32"), [0]),
              ("grouping(c1, c2)", P.cast(P.binop("&", c(2), u8(3)), "i32"), [0, 1])])]
    out = []
    for name, knames, sets, mode, gproj in runs:
        keys = [(c(k), k) for k in knames]
        partial = P.aggregate(mode, keys, aggs, scan, grouping_sets=sets)
        flat = [b for s in sets for b in s]
        if mode == "Single":
            stages = [P.Stage(1, P.shuffle_writer(partial, 1))]
        else:
            t = json.loads(__import__("ballista_b200").engine.plan_typed_json(json.dumps(partial)))
            nk = len(keys) + 1
            faggs = [P.agg(a["fn"], None, a["name"], ta["input_type"] if a["fn"] == "avg" else None) for a, ta in zip(aggs, t["aggr"])]
            final = P.aggregate("FinalPartitioned", [(c(i), t["schema"][i]["name"]) for i in range(nk)], faggs, P.shuffle_reader(1, t["schema"]))
            if gproj:
                final = P.project([(c(i), f["name"]) for i, f in enumerate(t["schema"][:nk])] + [(e, n) for n, e, _ in gproj] +
                                  [(c(nk + j), a["name"]) for j, a in enumerate(aggs)], final)
            stages = [P.Stage(1, P.shuffle_writer(partial, 1, [c(i) for i in range(nk)], 3)), P.Stage(2, P.shuffle_writer(final, 2))]
        entries = []
        for st in stages:
            ir = st.json("job")
            GROUPS.clear()
            GROUPS["flat"] = flat
            entries.append({"name": f"{name}/stage{st.stage_id}", "ir": ir, "proto_b64": base64.b64encode(M.encode(ir)).decode()})
        out.append({"name": name, "stages": entries,
                    "run": {"input_ir": json.dumps(scan), "keys": [{"expr": c(k), "name": k} for k in knames], "aggs": aggs,
                            "sets": sets, "grouping_projection": [[n, bits] for n, _, bits in gproj or []]}})
    # refused: encoded without the sets (the typing refuses them), then given the sets
    bad = [("duplicate_set", ["c1", "c2"], aggs, [[False, True], [True, True], [False, True]], -2, "duplicate grouping set"),
           ("too_many_keys", ["c1", "c2", "c3", "c4", "c5", "c6", "c7", "c8"], aggs, P.rollup_sets(8), -2, "8 keys"),
           ("stat_aggregate", ["c1"], [P.agg("var", c("c12"), "var_c12")], P.rollup_sets(1), -2, "alongside grouping sets"),
           ("bad_groups_length", ["c1", "c2"], aggs, [[True, False, True]], -1, "grouping-set entries")]
    for name, knames, baggs, sets, code, match in bad:
        plain = P.aggregate("Single", [(c(k), k) for k in knames], baggs, scan)
        ir = P.Stage(1, P.shuffle_writer(plain, 1)).json("job")
        GROUPS.clear()
        GROUPS["flat"] = [b for s in sets for b in s]
        out.append({"name": name, "refuse": {"code": code, "match": match},
                    "stages": [{"name": f"{name}/stage1", "proto_b64": base64.b64encode(M.encode(ir)).decode()}]})
    return out


def main():
    res = cases()
    with open(os.path.join(HERE, "grouping_set_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_grouping_set_proto_plans.py", "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto",
                   "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "cases")


if __name__ == "__main__":
    main()
