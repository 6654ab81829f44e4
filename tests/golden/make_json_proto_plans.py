"""Generate tests/golden/json_proto_plans.json: newline-delimited JSON scans (JsonScanExecNode) as the protobuf bytes a
Ballista scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_json_proto_plans.py      (commit the output)

Cases, encoded as datafusion.PhysicalPlanNode exactly as make_proto_plans.py encodes its fixtures (message classes built from
the reference's .proto files by protoc_lite.py), with every DataSourceExec leaf a JsonScanExecNode (datafusion.proto:1103-1105,
FileScanExecConf :1058-1086):
  * every stage of q1, q6 and q3 over one NDJSON file per TPC-H table: the table's schema, projection into it;
  * a ranged scan over two file groups of several files;
  * a scan whose projection travels as `projection_exprs` (FileScanExecConf field 13) rather than `projection`;
  * one refusal: a schema with a type the engine does not read, with the expected status code and the word the message
    must contain.
"""
import base64
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_proto_plans as M  # noqa: E402

_set_plan = M.set_plan


def set_plan(msg, t, o):
    if t["op"] not in ("DataSourceExec", "Scan", "MemoryScan") or o.get("format") != "json":
        return _set_plan(msg, t, o)
    conf = msg.json_scan.base_conf
    ranges = o.get("file_ranges")
    for gi, group in enumerate(o["file_groups"]):
        g = conf.file_groups.add()
        for fi, path in enumerate(group):
            f = g.files.add()
            f.path = path
            r = ranges[gi][fi] if ranges else None
            if r is not None:
                f.range.start, f.range.end = r
    M.set_schema(conf.schema, o["schema"])
    for c in conf.schema.columns:
        if c.name in o.get("_list_columns", ()):   # List<Utf8>: a nested type the plan IR cannot spell
            c.arrow_type.LIST.field_type.name = "item"
            c.arrow_type.LIST.field_type.arrow_type.UTF8.SetInParent()
    if o.get("projection") is not None:
        if o.get("_projection_exprs"):
            for i in o["projection"]:
                pe = conf.projection_exprs.projections.add()
                pe.alias = o["schema"][i]["name"]
                pe.expr.column.name = o["schema"][i]["name"]
                pe.expr.column.index = i
        else:
            conf.projection.extend(o["projection"])
    conf.object_store_url = "file://"


M.set_plan = set_plan   # children of the other operators recurse through the module's name


def json_table_scan(table, columns):
    from ballista_b200 import plan as P
    from ballista_b200 import tpch
    full = tpch.SCHEMAS[table]
    names = [f["name"] for f in full]
    return P.json_scan(table, full, projection=[names.index(c) for c in columns], file_groups=[[f"/data/tpch/{table}.json"]])


def as_json(node):
    """The stage plan with every TPC-H table scan replaced by its NDJSON scan (same output columns)."""
    if isinstance(node, list):
        return [as_json(x) for x in node]
    if not isinstance(node, dict):
        return node
    if node.get("op") == "DataSourceExec":
        sch = node["schema"]
        cols = [sch[i]["name"] for i in node["projection"]] if "projection" in node else [f["name"] for f in sch]
        return json_table_scan(node["table"], cols)
    return {k: as_json(v) for k, v in node.items()}


def cases():
    from ballista_b200 import plan as P
    from ballista_b200 import tpch
    out = []
    for q in ("q1", "q6", "q3"):
        for st in getattr(tpch, q)(4):
            out.append({"name": f"{q}/stage{st.stage_id}", "ir": P.Stage(st.stage_id, as_json(st.plan)).json("job")})
    sch = [P.field("id", "i64"), P.field("name", "utf8", True), P.field("price", P.dec(12, 2), True), P.field("day", "date32", True),
           P.field("ok", "bool", True), P.field("score", "f64", True)]
    scan = P.json_scan("events", sch, projection=[5, 0, 2],
                       file_groups=[["/data/events/part-0.json", "/data/events/part-1.json"], ["/data/events/part-1.json", "/data/events/part-2.json"]],
                       file_ranges=[[[0, 4096], [0, 1000]], [[1000, 9000], None]])
    out.append({"name": "ranges_multi_file", "ir": P.Stage(1, P.shuffle_writer(scan, 1)).json("job")})
    pe = P.json_scan("events", sch, projection=[1, 4], file_groups=[["/data/events/part-0.json"]])
    enc = dict(pe, _projection_exprs=True)
    out.append({"name": "projection_exprs", "ir": P.Stage(1, P.shuffle_writer(pe, 1)).json("job"),
                "encode_ir": P.Stage(1, P.shuffle_writer(enc, 1)).json("job")})
    bad = P.json_scan("events", [P.field("id", "i64"), P.field("tags", "utf8", True)], file_groups=[["/data/events/part-0.json"]])
    out.append({"name": "refuse/list_column", "ir": P.Stage(1, P.shuffle_writer(bad, 1)).json("job"), "code": -2, "needle": "type",
                "encode_ir": P.Stage(1, P.shuffle_writer(dict(bad, _list_columns=["tags"]), 1)).json("job")})
    return out


def main():
    res = []
    for c in cases():
        enc = c.pop("encode_ir", c["ir"])
        res.append(dict(c, proto_b64=base64.b64encode(M.encode(enc)).decode()))
    with open(os.path.join(HERE, "json_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_json_proto_plans.py", "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto",
                   "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
