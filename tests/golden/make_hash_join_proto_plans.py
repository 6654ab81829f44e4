"""Generate tests/golden/hash_join_proto_plans.json: HashJoinExec and SortMergeJoinExec plans, with and without
null_equality = NULL_EQUALS_NULL, as the protobuf bytes a Ballista scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_hash_join_proto_plans.py      (commit the output)

Encoded exactly as make_proto_plans.py encodes its fixtures (message classes built from the reference's .proto files by
protoc_lite.py): the join's null_equals_null becomes HashJoinExecNode / SortMergeJoinExecNode.null_equality = 1
(datafusion.proto:1140, :1440; NullEquality, datafusion_common.proto:98-101).  The "null_aware/" plans set
HashJoinExecNode.null_aware (field 10) on an anti join, which the decoder refuses.
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

KEYS = ["k_i64", "k_utf8"]


def stage(op, jt, nen):
    from ballista_b200 import plan as P
    import hash_join_cases as H
    if op == "HashJoinExec":
        return H.collect_left_stages(KEYS, jt, null_equals_null=nen)[0]
    on = H.on_cols(KEYS)
    j = P.sort_merge_join(P.scan("hj_l", H.IR_SCHEMA), P.scan("hj_r", H.IR_SCHEMA), on, jt,
                          sort_options=[{"asc": True, "nulls_first": False}] * len(on), null_equals_null=nen)
    return P.Stage(1, P.shuffle_writer(j, 1))


def main():
    import nlj_cases as N
    res = []
    for op in ("HashJoinExec", "SortMergeJoinExec"):
        for jt in N.JOIN_TYPES:
            for nen in (False, True):
                ir = stage(op, jt, nen).json("job")
                name = f"{op}/{jt}/" + ("null_equals_null" if nen else "null_equals_nothing")
                res.append({"name": name, "ir": ir, "proto_b64": base64.b64encode(M.encode(ir)).decode()})
    for jt in ("LeftAnti", "RightAnti"):
        ir = stage("HashJoinExec", jt, False).json("job")
        node = M.C("datafusion.PhysicalPlanNode")()
        node.ParseFromString(M.encode(ir))
        node.extension.inputs[0].hash_join.null_aware = True     # the stage root is the shuffle writer
        res.append({"name": f"null_aware/{jt}", "ir": ir, "proto_b64": base64.b64encode(node.SerializeToString()).decode()})
    with open(os.path.join(HERE, "hash_join_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_hash_join_proto_plans.py", "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto",
                   "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
