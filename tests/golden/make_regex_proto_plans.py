"""Generate tests/golden/regex_proto_plans.json: ILIKE, the regex operators and regexp_like as the protobuf bytes a Ballista
scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_regex_proto_plans.py      (commit the output)

Encoded exactly as make_proto_plans.py encodes its fixtures (its set_expr is wrapped, not edited; message classes built from
the reference's .proto files by protoc_lite.py):
  * [NOT] ILIKE: PhysicalLikeExprNode with case_insensitive = true (datafusion.proto:969-974);
  * `~`, `~*`, `!~`, `!~*`: PhysicalBinaryExprNode with op RegexMatch, RegexIMatch, RegexNotMatch, RegexNotIMatch (the Debug
    names of datafusion_expr::Operator);
  * regexp_like(x, p [, flags]): PhysicalScalarUdfNode, name in mixed case;
each in a projection and in a filter predicate.  Cases with "code" are refused when the decoded plan is typed (or, for an
ILIKE with a non-literal pattern, when it is decoded), with that status and a message containing "needle".
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

M._OPS.update({"~": "RegexMatch", "~*": "RegexIMatch", "!~": "RegexNotMatch", "!~*": "RegexNotIMatch"})
_set_expr = M.set_expr
SPELLED = {"regexp_like": "regexp_like"}


def set_expr(msg, e, remap=None, names=None):
    if "like" in e and (e.get("case_insensitive") or e["pattern"] is None):
        msg.like_expr.negated = bool(e.get("negated"))
        msg.like_expr.case_insensitive = bool(e.get("case_insensitive"))
        set_expr(msg.like_expr.expr, e["like"], remap, names)
        if isinstance(e["pattern"], dict):
            set_expr(msg.like_expr.pattern, e["pattern"], remap, names)
        else:
            msg.like_expr.pattern.literal.utf8_value = e["pattern"]
        return
    if e.get("fn") == "regexp_like":
        u = msg.scalar_udf
        u.name = SPELLED["regexp_like"]
        for a in e["args"]:
            set_expr(u.args.add(), a, remap, names)
        M.set_type(u.return_type, e["type"])
        return
    return _set_expr(msg, e, remap, names)


M.set_expr = set_expr   # every operator encodes its expressions through the module's name

PLACEHOLDER = "__P__"
LIT_PLACEHOLDER = '{"lit":{"t":"utf8","v":"__P__"}}'
COLUMN_T = '{"col":2,"name":"t","type":"utf8"}'


def exprs():
    """(name, expression over the scan below, refusal (code, needle, replacement) or None).  A refused expression is built
    with a pattern that types ("__P__", or the flags "is"), and the replacement (the refused pattern or flags, or a column) is
    put into the typed plan the encoder reads."""
    from ballista_b200 import plan as P
    c, s = P.col, P.lit_utf8
    X = PLACEHOLDER
    lit = lambda v: '{"lit":{"t":"utf8","v":%s}}' % json.dumps(v)   # noqa: E731
    return [
        ("ilike", P.like(c("s"), "%ab_C%", case_insensitive=True), None),
        ("not_ilike", P.like(c("s"), "x\\%y%", negated=True, case_insensitive=True), None),
        ("like_plain", P.like(c("s"), "%ab%"), None),
        ("match", P.regex_match(c("s"), "^a.*z$"), None),
        ("imatch", P.regex_match(c("s"), "k[a-f]+", case_insensitive=True), None),
        ("not_match", P.regex_match(c("s"), "\\d{2,}", negated=True), None),
        ("not_imatch", P.regex_match(c("s"), "(?s)a.b|(?-i:€)", negated=True, case_insensitive=True), None),
        ("match_null_pattern", P.regex_match(c("s"), P.lit_utf8(None)), None),
        ("regexp_like", P.fn("regexp_like", c("s"), s("q.*z")), None),
        ("regexp_like_flags_i", P.fn("regexp_like", c("s"), s("^ab"), s("i")), None),
        ("regexp_like_flags_is", P.fn("regexp_like", c("s"), s("a.b"), s("is")), None),
        ("refused_word_class", P.regex_match(c("s"), X), (-2, "\\w", {LIT_PLACEHOLDER: lit("\\w+")})),
        ("refused_flag_m", P.fn("regexp_like", c("s"), s("^a"), s("is")), (-2, "'m'", {lit("is"): lit("m")})),
        ("refused_non_ascii_ilike", P.like(c("s"), X, case_insensitive=True), (-2, "U+00E9", {'"pattern":"__P__"': '"pattern":' + json.dumps("%é%")})),
        ("refused_pattern_column", P.regex_match(c("s"), X), (-2, "literal", {LIT_PLACEHOLDER: COLUMN_T})),
        ("refused_regexp_like_column", P.fn("regexp_like", c("s"), s(X)), (-2, "literal", {LIT_PLACEHOLDER: COLUMN_T})),
        ("refused_ilike_column", P.like(c("s"), X, case_insensitive=True), (-2, "non-literal", {'"pattern":"__P__"': '"pattern":' + COLUMN_T})),
        ("invalid_unclosed_group", P.regex_match(c("s"), X), (-1, "offset 1", {LIT_PLACEHOLDER: lit("a(b")})),
        ("invalid_trailing_escape", P.like(c("s"), X, case_insensitive=True), (-1, "offset 2", {'"pattern":"__P__"': '"pattern":' + json.dumps("ab\\")})),
        ("invalid_flag_g", P.fn("regexp_like", c("s"), s("a"), s("is")), (-1, "global", {lit("is"): lit("g")})),
    ]


def cases():
    from ballista_b200 import plan as P
    import queries as Q
    c = P.col
    sch = [P.field("k", "i32", True), P.field("s", "utf8", True), P.field("t", "utf8", True)]
    scan = P.scan("t", sch)
    out = []
    for name, e, refusal in exprs():
        proj = Q.Stage(1, P.shuffle_writer(P.project([(e, "r"), (c("k"), "k")], scan), 1))
        filt = Q.Stage(1, P.shuffle_writer(P.filter_(e, scan, projection=[0, 1]), 1))
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
                assert k in typed, k
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
    with open(os.path.join(HERE, "regex_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_regex_proto_plans.py",
                   "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto", "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
