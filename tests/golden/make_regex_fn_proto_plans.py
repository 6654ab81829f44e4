"""Generate tests/golden/regex_fn_proto_plans.json: regexp_count and regexp_replace as the protobuf bytes a Ballista scheduler
ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_regex_fn_proto_plans.py      (commit the output)

Encoded exactly as make_proto_plans.py encodes its fixtures (its set_expr is wrapped, not edited; message classes built from
the reference's .proto files by protoc_lite.py): both functions are PhysicalScalarUdfNode (datafusion.proto:903-910), names
in mixed case, each in a projection and a filter predicate.  Cases with "code" are refused when the decoded plan is typed,
with that status and a message containing "needle"; they are built from an expression that types, and the refused literal
or column is put into the typed plan the encoder reads.
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

_set_expr = M.set_expr
SPELLED = {"regexp_count": "REGEXP_COUNT", "regexp_replace": "Regexp_Replace"}


def set_expr(msg, e, remap=None, names=None):
    if e.get("fn") in SPELLED:
        u = msg.scalar_udf
        u.name = SPELLED[e["fn"]]
        for a in e["args"]:
            set_expr(u.args.add(), a, remap, names)
        M.set_type(u.return_type, e["type"])
        return
    return _set_expr(msg, e, remap, names)


M.set_expr = set_expr   # every operator encodes its expressions through the module's name

PLACEHOLDER = "__P__"
COLUMN_T = '{"col":2,"name":"t","type":"utf8"}'


def lit(v):
    return '{"lit":{"t":"utf8","v":%s}}' % json.dumps(v)


def exprs():
    """(name, expression over the scan below, refusal (code, needle, {typed text: replacement}) or None)"""
    from ballista_b200 import plan as P
    c, s, i = P.col, P.lit_utf8, P.lit_i64
    X = PLACEHOLDER
    count = lambda *a: P.fn("regexp_count", c("s"), *a)    # noqa: E731
    replace = lambda *a: P.fn("regexp_replace", c("s"), *a)  # noqa: E731
    return [
        ("count", count(s("a.")), None),
        ("count_start", count(s("^[a-f]"), i(3)), None),
        ("count_start_flags", count(s("K|z"), i(2), s("is")), None),
        ("count_null_pattern", count(s(None)), None),
        ("replace", replace(s("[0-9]+"), s("#")), None),
        ("replace_global", replace(s("a|ab"), s("<€>"), s("g")), None),
        ("replace_flags_gi", replace(s("k+?"), s(""), s("gi")), None),
        ("replace_null_replacement", replace(s("a"), s(None)), None),
        ("refused_replacement_dollar", replace(s("(a)"), s(X)), (-2, "replacement", {lit(X): lit("$1")})),
        ("refused_replacement_backslash", replace(s("(a)"), s(X)), (-2, "replacement", {lit(X): lit("\\1")})),
        ("refused_count_pattern_column", count(s(X)), (-2, "literal", {lit(X): COLUMN_T})),
        ("refused_count_word", count(s(X)), (-2, "\\w", {lit(X): lit("\\w+")})),
        ("refused_replace_flag_m", replace(s("a"), s("b"), s("is")), (-2, "'m'", {lit("is"): lit("m")})),
        ("invalid_count_flag_g", count(s("a"), i(1), s("is")), (-1, "global", {lit("is"): lit("g")})),
        ("invalid_count_start_0", count(s("a"), i(7)), (-1, "start", {'{"lit":{"t":"i64","v":7}}': '{"lit":{"t":"i64","v":0}}'})),
        ("invalid_replace_syntax", replace(s(X), s("b")), (-1, "offset 1", {lit(X): lit("a(b")})),
    ]


def cases():
    from ballista_b200 import plan as P
    import queries as Q
    c = P.col
    sch = [P.field("k", "i32", True), P.field("s", "utf8", True), P.field("t", "utf8", True)]
    scan = P.scan("t", sch)
    out = []
    for name, e, refusal in exprs():
        pred = P.binop(">", e, P.lit_i64(0)) if e["fn"] == "regexp_count" else P.binop("<>", e, P.col("s"))
        proj = Q.Stage(1, P.shuffle_writer(P.project([(e, "r"), (c("k"), "k")], scan), 1))
        filt = Q.Stage(1, P.shuffle_writer(P.filter_(pred, scan, projection=[0, 1]), 1))
        for shape, st in (("projection", proj), ("filter", filt)):
            if refusal and shape == "filter":
                continue
            out.append((name, shape, st, refusal))
    return out


def main():
    from ballista_b200 import engine
    res = []
    for name, shape, st, refusal in cases():
        ir = st.json("job")
        case = {"name": f"{name}/{shape}"}
        if refusal:
            code, needle, repl = refusal
            typed = engine.plan_typed_json(ir)
            for k, v in repl.items():
                assert k in typed, (k, typed)
                typed = typed.replace(k, v)
                ir = ir.replace(k.replace(":", ": ").replace(",", ", "), v) if k not in ir else ir.replace(k, v)
            node = M.C("datafusion.PhysicalPlanNode")()
            M.set_plan(node, json.loads(typed), json.loads(st.json("job")))
            proto = node.SerializeToString()
            case["code"], case["needle"] = code, needle
        else:
            proto = M.encode(ir)
        case["ir"] = ir
        case["proto_b64"] = base64.b64encode(proto).decode()
        res.append(case)
    with open(os.path.join(HERE, "regex_fn_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_regex_fn_proto_plans.py",
                   "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto", "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
