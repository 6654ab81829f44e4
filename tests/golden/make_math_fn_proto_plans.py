"""Generate tests/golden/math_fn_proto_plans.json: plans calling the math functions of DESIGN.md §6 (xviii) as the protobuf
bytes a Ballista scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_math_fn_proto_plans.py      (commit the output)

Every name and alias (pow for power), in mixed case, with PhysicalScalarUdfNode.return_type set to the result type.  Each is
used in a projection, a filter predicate, and as a group key and aggregate argument over Partial -> FinalPartitioned.
Encoded exactly as make_scalar_fn_proto_plans.py encodes its fixtures (make_proto_plans.py's set_expr wrapped, message
classes built from the reference's .proto files by protoc_lite.py).  Cases with "refused" hold an argument type the engine
does not take, a non-literal trunc digit count, or random; "refused" is what the refusal names.
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
SPELLING = {}   # IR function name -> protobuf name for the case being encoded


def set_expr(msg, e, remap=None, names=None):
    if "fn" not in e:
        return _set_expr(msg, e, remap, names)
    u = msg.scalar_udf
    u.name = SPELLING.get(e["fn"], e["fn"])
    for a in e["args"]:
        set_expr(u.args.add(), a, remap, names)
    M.set_type(u.return_type, e["type"])


M.set_expr = set_expr   # every operator encodes its expressions through the module's name

UNARY = ["sqrt", "cbrt", "exp", "ln", "log2", "log10", "sin", "cos", "tan", "asin", "acos", "atan", "sinh", "cosh", "tanh",
         "asinh", "acosh", "atanh", "cot", "degrees", "radians", "signum"]


def calls():
    """(case label, IR function, protobuf spelling, scalar expression over the scan below, result type, refused)"""
    from ballista_b200 import plan as P
    c = P.col
    out = []
    for k, n in enumerate(UNARY):
        col, t = ("f", "f64") if k % 2 == 0 else ("g", "f32")
        out.append((n, n, n.upper() if k % 3 == 0 else n, P.fn(n, c(col)), t, None))
    out += [("log", "log", "Log", P.fn("log", c("f")), "f64", None),
            ("log_base", "log", "log", P.fn("log", P.lit_f64(2.0), c("f")), "f64", None),
            ("atan2", "atan2", "ATAN2", P.fn("atan2", c("g"), c("g")), "f32", None),
            ("nanvl", "nanvl", "nanvl", P.fn("nanvl", c("f"), P.lit_f64(0.0)), "f64", None),
            ("power", "power", "power", P.fn("power", c("f"), P.lit_f64(2.0)), "f64", None),
            ("pow", "power", "POW", P.fn("power", c("x"), P.lit_i64(2)), "i64", None),
            ("trunc", "trunc", "trunc", P.fn("trunc", c("f"), P.lit_i64(1)), "f64", None),
            ("trunc_f32", "trunc", "Trunc", P.fn("trunc", c("g")), "f32", None),
            ("gcd", "gcd", "gcd", P.fn("gcd", c("x"), P.lit_i64(6)), "i64", None),
            ("lcm", "lcm", "LCM", P.fn("lcm", c("x"), P.lit_i64(4)), "i64", None),
            ("factorial", "factorial", "factorial", P.fn("factorial", P.binop("%", c("x"), P.lit_i64(21))), "i64", None),
            ("isnan", "isnan", "isnan", P.fn("isnan", c("f")), "bool", None),
            ("iszero", "iszero", "IsZero", P.fn("iszero", c("g")), "bool", None),
            ("pi", "pi", "pi", P.binop("*", P.fn("pi"), c("f")), "f64", None),
            # refused: a plan the IR cannot type is encoded through a function that takes the argument, spelled as the
            # refused one (its return_type is that function's)
            ("sqrt_dec", "abs", "sqrt", P.fn("abs", c("dec")), "dec", "dec(15,2)"),
            ("ln_utf8", "btrim", "ln", P.fn("btrim", c("s")), "utf8", "utf8"),
            ("exp_i32", "abs", "exp", P.fn("abs", c("k")), "i32", "i32"),
            ("trunc_column_digits", "trunc", "trunc", P.fn("trunc", c("f"), c("x")), "f64", "literal"),
            ("random", "sqrt", "random", P.fn("sqrt", c("f")), "f64", "random")]
    return out


def predicate(e, typ):
    from ballista_b200 import plan as P
    if typ == "bool":
        return e
    if typ in ("f64", "f32"):
        return P.binop(">", e, P.lit_f64(0.0) if typ == "f64" else {"lit": {"t": "f32", "v": 0.0}})
    return P.binop(">", e, P.lit_i64(1))


def cases():
    from ballista_b200 import plan as P
    import queries as Q
    c = P.col
    sch = [P.field("k", "i32", True), P.field("x", "i64", True), P.field("f", "f64", True), P.field("g", "f32", True),
           P.field("s", "utf8", True), P.field("dec", P.dec(15, 2), True)]
    scan = P.scan("t", sch)
    out = []
    for label, fn, spelled, e, typ, refused in calls():
        proj = [Q.Stage(1, P.shuffle_writer(P.project([(e, "r"), (c("k"), "k")], scan), 1))]
        out.append((label, fn, spelled, refused, "projection", proj))
        if refused:
            continue
        filt = [Q.Stage(1, P.shuffle_writer(P.filter_(predicate(e, typ), scan, projection=[0, 2]), 1))]
        arg = P.cast(e, "i64") if typ == "bool" else e
        arg_t = {"f32": "f64", "bool": "i64"}.get(typ, typ)
        part = P.aggregate("Partial", [(e, "g")], [P.agg("sum", arg, "s"), P.agg("count", None, "n")], scan)
        st1 = Q.Stage(1, P.shuffle_writer(part, 1, [c(0)], 2))
        fields = [P.field("g", typ, True), P.field("s[sum]", arg_t, True), P.field("n[count]", "i64", True)]
        fin = P.aggregate("FinalPartitioned", [(c(0), "g")], [P.agg("sum", c(1), "s", input_type=arg_t), P.agg("count", c(2), "n")],
                          P.shuffle_reader(1, fields))
        st2 = Q.Stage(2, P.shuffle_writer(fin, 2))
        out.append((label, fn, spelled, refused, "filter", filt))
        out.append((label, fn, spelled, refused, "group_key_and_argument", [st1, st2]))
    return out


def main():
    res = []
    for label, fn, spelled, refused, shape, stages in cases():
        SPELLING.clear()
        SPELLING[fn] = spelled
        for st in stages:
            ir = st.json("job")
            res.append({"name": f"{label}/{shape}/stage{st.stage_id}", "fn": fn, "spelled": spelled, "refused": refused, "ir": ir,
                        "proto_b64": base64.b64encode(M.encode(ir)).decode()})
    with open(os.path.join(HERE, "math_fn_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_math_fn_proto_plans.py",
                   "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto", "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
