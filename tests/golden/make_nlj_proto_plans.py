"""Generate tests/golden/nlj_proto_plans.json: NestedLoopJoinExec plans as the protobuf bytes a Ballista scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_nlj_proto_plans.py      (commit the output)

Every stage of tpch.q11_nlj / tpch.q22_nlj (4 shuffle partitions) and one plan per join type, with and without a filter and a
projection, encoded as datafusion.PhysicalPlanNode exactly as make_proto_plans.py encodes its fixtures (message classes built
from the reference's .proto files by protoc_lite.py); the nested-loop join becomes NestedLoopJoinExecNode
(datafusion.proto:1301-1307) with its filter as a JoinFilter over column_indices.
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
    if t["op"] != "NestedLoopJoinExec":
        return _set_plan(msg, t, o)
    j = msg.nested_loop_join
    set_plan(j.left, t["left"], o["left"])
    set_plan(j.right, t["right"], o["right"])
    M.set_join_common(j, dict(t, on=[]), t["left"]["schema"], t["right"]["schema"])
    if "projection" in t:
        j.projection.extend(t["projection"])


M.set_plan = set_plan   # children of the other operators recurse through the module's name


def cases():
    from ballista_b200 import plan as P
    from ballista_b200 import tpch
    import nlj_cases as N
    out = []
    for q in ("q11", "q22"):
        for st in getattr(tpch, f"{q}_nlj")(4):
            out.append((f"{q}_nlj/stage{st.stage_id}", st.json("job")))
    for jt in N.JOIN_TYPES:
        for fname in ("none", "mixed", "dec_cast_gt", "utf8_ge_flipped"):
            proj = None if jt.endswith("Semi") or jt.endswith("Anti") else [N.NC + 1, 0, 6]
            for pr in ((None, proj) if proj else (None,)):
                name = f"join/{jt}/{fname}" + ("/projection" if pr else "")
                out.append((name, N.join_stage(jt, N.FILTERS[fname], pr)[0].json("job")))
    return out


def main():
    res = []
    for name, ir in cases():
        res.append({"name": name, "ir": ir, "proto_b64": base64.b64encode(M.encode(ir)).decode()})
    with open(os.path.join(HERE, "nlj_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_nlj_proto_plans.py", "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto",
                   "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
