"""Generate tests/golden/csv_proto_plans.json: CSV scans (CsvScanExecNode) as the protobuf bytes a Ballista scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_csv_proto_plans.py      (commit the output)

Cases, encoded as datafusion.PhysicalPlanNode exactly as make_proto_plans.py encodes its fixtures (message classes built from
the reference's .proto files by protoc_lite.py), with every DataSourceExec leaf a CsvScanExecNode (datafusion.proto:1088-1101):
  * every stage of q1, q6 and q3 over dbgen .tbl files as tpch.rs plans them for `--format tbl` (tpch.rs:653-683, schema
    :1056-1060): tbl_schema with `__placeholder`, delimiter '|', no header, projection into the full schema;
  * a scan with a header, quote, escape and byte ranges over two file groups;
  * one case per refusal (the options 'comment' and 'truncate_rows'; malformed option strings), with the expected status
    code and the word the message must contain.
"""
import base64
import copy
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
    if t["op"] not in ("DataSourceExec", "Scan", "MemoryScan") or o.get("format") != "csv":
        return _set_plan(msg, t, o)
    c = msg.csv_scan
    conf = c.base_conf
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
    if o.get("projection") is not None:
        conf.projection.extend(o["projection"])
    conf.object_store_url = "file://"
    opts = o["csv"]
    c.has_header = opts["has_header"]
    c.delimiter = opts["delimiter"]
    c.quote = opts["quote"]
    if opts.get("escape") is not None:
        c.escape = opts["escape"]
    if opts.get("comment") is not None:
        c.comment = opts["comment"]
    c.newlines_in_values = opts["newlines_in_values"]
    c.truncate_rows = bool(opts.get("truncate_rows", False))


M.set_plan = set_plan   # children of the other operators recurse through the module's name


def as_tbl(node):
    """The stage plan with every TPC-H table scan replaced by its .tbl scan (same output columns)."""
    from ballista_b200 import tpch
    if isinstance(node, list):
        return [as_tbl(x) for x in node]
    if not isinstance(node, dict):
        return node
    if node.get("op") == "DataSourceExec":
        sch = node["schema"]
        cols = [sch[i]["name"] for i in node["projection"]] if "projection" in node else [f["name"] for f in sch]
        return tpch.tbl_scan(node["table"], cols)
    return {k: as_tbl(v) for k, v in node.items()}


def cases():
    from ballista_b200 import plan as P
    from ballista_b200 import tpch
    out = []
    for q in ("q1", "q6", "q3"):
        for st in getattr(tpch, q)(4):
            p = as_tbl(st.plan)
            out.append({"name": f"{q}/stage{st.stage_id}", "ir": P.Stage(st.stage_id, p).json("job")})
    sch = [P.field("c1", "utf8"), P.field("c2", "i64"), P.field("c3", P.dec(10, 2), True), P.field("c4", "utf8", True)]
    opts = dict(has_header=True, delimiter=";", quote="'", escape="\\")
    scan = P.csv_scan("quoted", sch, projection=[3, 1], file_groups=[["/data/quoted/part-0.csv", "/data/quoted/part-1.csv"], ["/data/quoted/part-0.csv"]],
                      file_ranges=[[[0, 100], None], [[100, 250]]], **opts)
    out.append({"name": "header_quote_escape_ranges", "ir": P.Stage(1, P.shuffle_writer(scan, 1)).json("job")})
    base = P.csv_scan("plain", sch, file_groups=[["/data/plain/part-0.csv"]])
    refusals = [("comment", {"comment": "#"}, -2, "comment"), ("truncate_rows", {"truncate_rows": True}, -2, "truncate_rows"),
                ("empty_delimiter", {"delimiter": ""}, -1, "delimiter"), ("long_delimiter", {"delimiter": "||"}, -1, "delimiter"),
                ("long_quote", {"quote": "''"}, -1, "quote"), ("non_ascii_escape", {"escape": "é"}, -1, "escape")]
    for name, change, code, needle in refusals:
        node = copy.deepcopy(base)
        node["csv"].update(change)
        out.append({"name": "refuse/" + name, "ir": P.Stage(1, P.shuffle_writer(node, 1)).json("job"), "code": code, "needle": needle})
    return out


def main():
    res = []
    for c in cases():
        res.append(dict(c, proto_b64=base64.b64encode(M.encode(c["ir"])).decode()))
    with open(os.path.join(HERE, "csv_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_csv_proto_plans.py", "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto",
                   "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
