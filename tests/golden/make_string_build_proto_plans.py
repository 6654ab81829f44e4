"""Generate tests/golden/string_build_proto_plans.json: concat, `||`, concat_ws, repeat, reverse and CAST / TRY_CAST to Utf8
as the protobuf bytes a Ballista scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_string_build_proto_plans.py      (commit the output)

Encoded exactly as make_proto_plans.py encodes its fixtures (its set_expr is wrapped, not edited; message classes built from
the reference's .proto files by protoc_lite.py):
  * concat / concat_ws / repeat / reverse: PhysicalScalarUdfNode (datafusion.proto:903-910), names in mixed case;
  * `||`: PhysicalBinaryExprNode with op StringConcat (the Debug name of datafusion_expr::Operator);
  * CAST(x AS Utf8): PhysicalCastNode; TRY_CAST: PhysicalTryCastNode (:999-1007);
each in a projection and a filter predicate.  Cases with "refused" spell a string function the engine does not compute
under a function that types (the decoder refuses it by name).
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

M._OPS["||"] = "StringConcat"
_set_expr = M.set_expr
SPELLED = {"concat": "CONCAT", "concat_ws": "Concat_Ws", "repeat": "repeat", "reverse": "REVERSE"}
OPTS = {"rename": None, "try_cast": False}  # the case being encoded: a refused name for its function, casts as TRY_CAST


def set_expr(msg, e, remap=None, names=None):
    if e.get("fn") in SPELLED:
        u = msg.scalar_udf
        u.name = OPTS["rename"] or SPELLED[e["fn"]]
        for a in e["args"]:
            set_expr(u.args.add(), a, remap, names)
        M.set_type(u.return_type, e["type"])
        return
    if "cast" in e and e.get("to") == "utf8" and OPTS["try_cast"]:
        set_expr(msg.try_cast.expr, e["cast"], remap, names)
        M.set_type(msg.try_cast.arrow_type, e["to"])
        return
    return _set_expr(msg, e, remap, names)


M.set_expr = set_expr   # every operator encodes its expressions through the module's name


def exprs():
    """(name, expression over the scan below, refused name or None, encode casts as TRY_CAST)"""
    from ballista_b200 import plan as P
    c, s = P.col, P.lit_utf8
    return [
        ("concat", P.fn("concat", c("s"), s("-"), P.cast(c("x"), "utf8")), None, False),
        ("concat_null_literal", P.fn("concat", c("s"), P.lit_utf8(None)), None, False),
        ("string_concat", P.str_concat(c("s"), s("/"), c("t")), None, False),
        ("concat_ws", P.fn("concat_ws", s(", "), c("s"), c("t")), None, False),
        ("concat_ws_column_separator", P.fn("concat_ws", c("t"), c("s"), s("z")), None, False),
        ("repeat", P.fn("repeat", c("s"), P.lit_i64(3)), None, False),
        ("repeat_column_count", P.fn("repeat", c("s"), c("x")), None, False),
        ("reverse", P.fn("reverse", c("s")), None, False),
        ("cast_int", P.cast(c("x"), "utf8"), None, False),
        ("cast_uint64", P.cast(c("u"), "utf8"), None, False),
        ("cast_decimal", P.cast(c("m"), "utf8"), None, False),
        ("cast_date", P.cast(c("d"), "utf8"), None, False),
        ("cast_bool", P.cast(c("b"), "utf8"), None, False),
        ("try_cast_int", P.cast(c("k"), "utf8"), None, True),
        ("refused_lpad", P.fn("concat", c("s"), s("x")), "lpad", False),
        ("refused_rpad", P.fn("concat", c("s"), s("x")), "rpad", False),
        ("refused_to_hex", P.fn("reverse", c("s")), "to_hex", False),
        ("refused_to_char", P.fn("concat", c("s"), s("x")), "to_char", False),
        ("refused_left", P.fn("repeat", c("s"), P.lit_i64(2)), "left", False),
        ("refused_right", P.fn("repeat", c("s"), P.lit_i64(2)), "right", False),
        ("refused_split_part", P.fn("concat", c("s"), s("x")), "split_part", False),
        ("refused_translate", P.fn("concat", c("s"), s("x")), "translate", False),
        ("refused_initcap", P.fn("reverse", c("s")), "initcap", False),
    ]


def cases():
    from ballista_b200 import plan as P
    import queries as Q
    c = P.col
    sch = [P.field("k", "i32", True), P.field("s", "utf8", True), P.field("t", "utf8", True), P.field("x", "i64", True),
           P.field("u", "u64", True), P.field("m", P.dec(12, 2), True), P.field("d", "date32", True), P.field("b", "bool", True)]
    scan = P.scan("t", sch)
    out = []
    for name, e, refused, try_cast in exprs():
        proj = Q.Stage(1, P.shuffle_writer(P.project([(e, "r"), (c("k"), "k")], scan), 1))
        filt = Q.Stage(1, P.shuffle_writer(P.filter_(P.binop("<>", e, P.lit_utf8("")), scan, projection=[0, 1]), 1))
        for shape, st in (("projection", proj), ("filter", filt)):
            if refused and shape == "filter":
                continue
            out.append((name, shape, st, refused, try_cast))
    return out


def main():
    res = []
    for name, shape, st, refused, try_cast in cases():
        ir = st.json("job")
        OPTS.update(rename=refused, try_cast=try_cast)
        case = {"name": f"{name}/{shape}", "ir": ir, "proto_b64": base64.b64encode(M.encode(ir)).decode()}
        if refused:
            case["refused"] = refused
        res.append(case)
    with open(os.path.join(HERE, "string_build_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_string_build_proto_plans.py",
                   "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto", "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
