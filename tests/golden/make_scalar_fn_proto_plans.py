"""Generate tests/golden/scalar_fn_proto_plans.json: plans calling the scalar functions of DESIGN.md §3 as the protobuf bytes a
Ballista scheduler ships.

    BALLISTA_SRC=<datafusion-ballista checkout> python tests/golden/make_scalar_fn_proto_plans.py      (commit the output)

Every function and alias, names and date parts in mixed case (EXTRACT arrives as date_part with an upper-case part), with
PhysicalScalarUdfNode.return_type set to the result type.  Each is used in a projection, a filter predicate, a group key and
an aggregate argument, over Partial -> FinalPartitioned.  Encoded exactly as make_proto_plans.py encodes its fixtures (its
set_expr is wrapped, not edited; message classes built from the reference's .proto files by protoc_lite.py).  Cases with
"refused" spell a function or a date part the engine does not compute.
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
SPELLING = {}   # IR function name -> (protobuf name, date part or None) for the case being encoded


def set_expr(msg, e, remap=None, names=None):
    if "fn" not in e or e["fn"] in ("date_part_year", "substr") and e["fn"] not in SPELLING:
        return _set_expr(msg, e, remap, names)
    u = msg.scalar_udf
    default = ("date_part", e["fn"][10:]) if e["fn"].startswith("date_part_") else (e["fn"], None)
    name, part = SPELLING.get(e["fn"], default)
    u.name = name
    if part is not None:
        u.args.add().literal.utf8_value = part
    for a in e["args"]:
        set_expr(u.args.add(), a, remap, names)
    M.set_type(u.return_type, e["type"])


M.set_expr = set_expr   # every operator encodes its expressions through the module's name

# (IR function, protobuf spelling, date part spelling, refused)
SPELLINGS = [("date_part_year", "date_part", "YEAR", None), ("date_part_quarter", "DATE_PART", "quarter", None),
             ("date_part_month", "date_part", "Month", None), ("date_part_week", "datepart", "WEEK", None),
             ("date_part_day", "date_part", "DAY", None), ("date_part_doy", "Date_Part", "doy", None),
             ("date_part_dow", "date_part", "DOW", None),
             ("abs", "ABS", None, None), ("round", "round", None, None), ("round", "Round", None, None), ("floor", "floor", None, None),
             ("ceil", "CEIL", None, None), ("nullif", "NullIf", None, None), ("coalesce", "coalesce", None, None),
             ("coalesce", "COALESCE", None, None),
             ("character_length", "character_length", None, None), ("character_length", "CHAR_LENGTH", None, None),
             ("character_length", "length", None, None), ("octet_length", "Octet_Length", None, None),
             ("starts_with", "starts_with", None, None), ("ends_with", "ENDS_WITH", None, None),
             ("btrim", "btrim", None, None), ("btrim", "TRIM", None, None), ("ltrim", "ltrim", None, None), ("rtrim", "RTrim", None, None),
             ("date_part_year", "date_part", "EPOCH", "epoch"), ("date_part_year", "date_part", "hour", "hour"),
             ("date_part_year", "date_part", "isodow", "isodow"), ("character_length", "upper", None, "upper"),
             ("character_length", "lower", None, "lower"), ("btrim", "replace", None, "replace")]


def calls():
    """IR function -> (scalar expression over the scan below, result type)"""
    from ballista_b200 import plan as P
    c = P.col
    dp = {f"date_part_{p}": (P.fn(f"date_part_{p}", c("d")), "i32") for p in ("year", "quarter", "month", "week", "day", "doy", "dow")}
    return {**dp,
            "abs": (P.fn("abs", c("x")), "i64"),
            "round": (P.fn("round", c("f"), P.lit_i64(2)), "f64"),
            "floor": (P.fn("floor", c("f")), "f64"),
            "ceil": (P.fn("ceil", c("f")), "f64"),
            "nullif": (P.fn("nullif", c("x"), P.lit_i64(0)), "i64"),
            "coalesce": (P.fn("coalesce", c("s"), c("t"), P.lit_utf8("-")), "utf8"),
            "character_length": (P.fn("character_length", c("s")), "i32"),
            "octet_length": (P.fn("octet_length", c("s")), "i32"),
            "starts_with": (P.fn("starts_with", c("s"), P.lit_utf8("ab")), "bool"),
            "ends_with": (P.fn("ends_with", c("s"), c("t")), "bool"),
            "btrim": (P.fn("btrim", c("s"), P.lit_utf8("x€ ")), "utf8"),
            "ltrim": (P.fn("ltrim", c("s")), "utf8"),
            "rtrim": (P.fn("rtrim", c("s")), "utf8")}


def predicate(e, typ):
    from ballista_b200 import plan as P
    if typ == "bool":
        return e
    if typ == "utf8":
        return P.binop("!=", e, P.lit_utf8(""))
    if typ == "f64":
        return P.binop(">", e, P.lit_f64(0.0))
    return P.binop(">", e, P.lit_i64(1))


def cases():
    from ballista_b200 import plan as P
    import queries as Q
    c = P.col
    sch = [P.field("k", "i32", True), P.field("x", "i64", True), P.field("f", "f64", True), P.field("d", "date32", True),
           P.field("s", "utf8", True), P.field("t", "utf8", True)]
    scan = P.scan("t", sch)
    out = []
    for fn, (e, typ) in calls().items():
        proj = [Q.Stage(1, P.shuffle_writer(P.project([(e, "r"), (c("k"), "k")], scan), 1))]
        filt = [Q.Stage(1, P.shuffle_writer(P.filter_(predicate(e, typ), scan, projection=[0, 4]), 1))]
        # group key and aggregate argument, Partial -> hash shuffle -> FinalPartitioned
        arg = e if typ in ("i32", "i64", "f64") else P.cast(e, "i64") if typ == "bool" else P.fn("octet_length", e) if typ == "utf8" else e
        arg_t = {"i32": "i64", "i64": "i64", "f64": "f64"}.get(typ, "i64")
        part = P.aggregate("Partial", [(e, "g")], [P.agg("sum", arg, "s"), P.agg("count", None, "n")], scan)
        st1 = Q.Stage(1, P.shuffle_writer(part, 1, [c(0)], 2))
        fields = [P.field("g", typ, True), P.field("s[sum]", arg_t, True), P.field("n[count]", "i64", True)]
        fin = P.aggregate("FinalPartitioned", [(c(0), "g")], [P.agg("sum", c(1), "s", input_type=arg_t), P.agg("count", c(2), "n")],
                          P.shuffle_reader(1, fields))
        st2 = Q.Stage(2, P.shuffle_writer(fin, 2))
        out.append((fn, "projection", proj))
        out.append((fn, "filter", filt))
        out.append((fn, "group_key_and_argument", [st1, st2]))
    return out


def main():
    per_fn = {}
    for fn, shape, stages in cases():
        per_fn.setdefault(fn, []).append((shape, stages))
    res = []
    for fn_ir, spelled, part, refused in SPELLINGS:
        SPELLING.clear()
        SPELLING[fn_ir] = (spelled, part)
        label = spelled + (f"({part})" if part else "")
        for shape, stages in per_fn[fn_ir]:
            if refused and shape != "projection":
                continue
            for st in stages:
                ir = st.json("job")
                res.append({"name": f"{label}/{shape}/stage{st.stage_id}", "fn": fn_ir, "spelled": spelled, "part": part,
                            "refused": refused, "ir": ir, "proto_b64": base64.b64encode(M.encode(ir)).decode()})
    with open(os.path.join(HERE, "scalar_fn_proto_plans.json"), "w") as fh:
        json.dump({"generated_by": "tests/golden/make_scalar_fn_proto_plans.py",
                   "proto_files": "ballista/core/proto/{datafusion_common,datafusion,ballista}.proto", "cases": res}, fh, indent=0)
        fh.write("\n")
    print(len(res), "plans")


if __name__ == "__main__":
    main()
