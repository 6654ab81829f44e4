"""Shared pieces of the regr_* / bool_and / bool_or / bit_and / bit_or / bit_xor tests: the rules restated in plain Python
(sharing nothing with plan.hpp or the oracle), the plans (Single, or Partial -> shuffle -> Final / FinalPartitioned) and
the UNION ALL form of a grouping-set aggregate.

[EXT] DataFusion 53 (datafusion-functions-aggregate regr.rs, bool_and_or.rs, bit_and_or_xor.rs) is not vendored: every
rule below is a restatement and is unpinned, as DESIGN.md §6 (xvi) says.  The regr_r2 rule in particular (NULL when
syy = 0, where PostgreSQL returns 1) is written from the issue's understanding of DataFusion, not checked against it."""
from fractions import Fraction

from ballista_b200 import plan as P
from ballista_b200.plan import Stage

c = P.col

REGR = ["regr_slope", "regr_intercept", "regr_count", "regr_r2", "regr_avgx", "regr_avgy", "regr_sxx", "regr_syy", "regr_sxy"]
BOOL = ["bool_and", "bool_or"]
BIT = ["bit_and", "bit_or", "bit_xor"]
REGR_STATE = ["count", "mean_x", "mean_y", "m2_x", "m2_y", "algo_const"]
INT_TYPES = {"i8": 8, "i16": 16, "i32": 32, "i64": 64, "u8": 8, "u16": 16, "u32": 32, "u64": 64}


def state_fields(fn, name, arg_type):
    """The Partial output's state fields of one aggregate (arg_type: the IR type of bool / bit arguments; "sum" stands for
    SUM of a Float64, mixed into some plans)."""
    if fn == "sum":
        return [P.field(f"{name}[sum]", "f64", True)]
    if fn in REGR:
        return [P.field(f"{name}[{s}]", "u64" if s == "count" else "f64", True) for s in REGR_STATE]
    return [P.field(f"{name}[{fn}]", arg_type, True)]


def result_type(fn, arg_type):
    if fn == "regr_count":
        return "u64"
    return "f64" if fn in REGR else arg_type


# ---- regression: exact rational arithmetic over the Float64 values (the same coercion as stat_cases.py) ---------------
def regr_exact(fn, ys, xs):
    """regr_*(y, x) over the rows where both are non-NULL, computed exactly and rounded once; None = NULL."""
    if fn == "regr_count":
        return sum(1 for y, x in zip(ys, xs) if x is not None and y is not None)
    pairs = [(Fraction(x), Fraction(y)) for y, x in zip(ys, xs) if x is not None and y is not None]
    n = len(pairs)
    if n == 0:
        return None
    mx = sum(p[0] for p in pairs) / n
    my = sum(p[1] for p in pairs) / n
    sxx = sum((p[0] - mx) ** 2 for p in pairs)
    syy = sum((p[1] - my) ** 2 for p in pairs)
    sxy = sum((p[0] - mx) * (p[1] - my) for p in pairs)
    simple = {"regr_avgx": mx, "regr_avgy": my, "regr_sxx": sxx, "regr_syy": syy, "regr_sxy": sxy}
    if fn in simple:
        return float(simple[fn])
    if n <= 1 or sxx == 0:
        return None
    slope = sxy / sxx  # (sxy/n) / (sxx/n)
    if fn == "regr_slope":
        return float(slope)
    if fn == "regr_intercept":
        return float(my - slope * mx)
    if syy == 0:
        return None  # regr_r2: [EXT] unpinned (PostgreSQL: 1)
    return float(sxy * sxy / (sxx * syy))


def regr_state(ys, xs):
    """The exact partial state [count, mean_x, mean_y, m2_x, m2_y, algo_const] of one group (an empty group's means and
    moments are 0)."""
    pairs = [(Fraction(x), Fraction(y)) for y, x in zip(ys, xs) if x is not None and y is not None]
    n = len(pairs)
    if n == 0:
        return [0, 0.0, 0.0, 0.0, 0.0, 0.0]
    mx = sum(p[0] for p in pairs) / n
    my = sum(p[1] for p in pairs) / n
    return [n, float(mx), float(my), float(sum((p[0] - mx) ** 2 for p in pairs)), float(sum((p[1] - my) ** 2 for p in pairs)),
            float(sum((p[0] - mx) * (p[1] - my) for p in pairs))]


# ---- bool / bit folds ----------------------------------------------------------------------------------------------------
def fold(fn, vals, arg_type=None):
    """bool_and / bool_or over Python bools, bit_* over Python ints of IR type arg_type; NULLs skipped, None when no value."""
    vs = [v for v in vals if v is not None]
    if not vs:
        return None
    if fn == "bool_and":
        return all(vs)
    if fn == "bool_or":
        return any(vs)
    bits = INT_TYPES[arg_type]
    mask = (1 << bits) - 1
    acc = mask if fn == "bit_and" else 0
    for v in vs:
        w = v & mask
        acc = acc & w if fn == "bit_and" else acc | w if fn == "bit_or" else acc ^ w
    if arg_type.startswith("i") and acc >> (bits - 1):
        acc -= 1 << bits  # back to the signed value
    return acc


def grouped(rows, key_idx, aggs):
    """{key tuple: {name: value}} over rows (tuples); aggs: [(fn, arg index, arg2 index or None, name, arg IR type)]."""
    groups = {}
    for r in rows:
        groups.setdefault(tuple(r[k] for k in key_idx), []).append(r)
    if not key_idx:
        groups.setdefault((), [])
    out = {}
    for g, rs in groups.items():
        d = {}
        for fn, a, b, name, t in aggs:
            if fn in REGR:
                d[name] = regr_exact(fn, [r[a] for r in rs], [r[b] for r in rs])
            else:
                d[name] = fold(fn, [r[a] for r in rs], t)
        out[g] = d
    return out


def union_all(rows, key_idx, sets, aggs):
    """The UNION ALL form of a grouping-set aggregate: {(keys with NULL where masked..., __grouping_id): {name: value}}."""
    out = {}
    for mask in sets:
        present = [k for k, m in zip(key_idx, mask) if not m]
        gid = P.grouping_id(mask)
        groups = grouped(rows, present, aggs) if rows else {}
        for g, vals in groups.items():
            it = iter(g)
            full = tuple(None if m else next(it) for m in mask)
            out[full + (gid,)] = vals
    return out


# ---- plans ----------------------------------------------------------------------------------------------------------------
def stages(src, aggs, keys=(), key_fields=(), mode="Single", n_out=3, grouping_sets=None, final_args=True):
    """aggs: [(fn, arg expr, arg2 expr or None, name, arg IR type)]; keys: [(expr, name)]; key_fields: their IR fields.
    mode "Single" / "SinglePartitioned": one stage; "Partial": Partial -> shuffle -> FinalPartitioned (with keys) or Final
    (without).  final_args: the Final's aggregates carry their original arguments and the node the Partial's input schema,
    as a Ballista plan does (AggregateExecNode.input_schema), so that regr_* over one pair merge their states once."""
    pagg = [P.agg(fn, a, name, arg2=b) for fn, a, b, name, _ in aggs]
    gb = list(keys)
    if mode in ("Single", "SinglePartitioned"):
        return [Stage(1, P.shuffle_writer(P.aggregate(mode, gb, pagg, src, grouping_sets=grouping_sets), 1))]
    s1 = P.aggregate("Partial", gb, pagg, src, grouping_sets=grouping_sets)
    part = list(key_fields) + [f for fn, _, _, name, t in aggs for f in state_fields(fn, name, t)]
    fagg = [P.agg(fn, a if final_args else None, name, arg2=b if final_args else None) for fn, a, b, name, _ in aggs]
    nk = len(gb)

    def final(node):
        if final_args:
            node["input_schema"] = src["schema"]
        return node
    if nk:
        return [Stage(1, P.shuffle_writer(s1, 1, [c(i) for i in range(nk)], n_out)),
                Stage(2, P.shuffle_writer(final(P.aggregate("FinalPartitioned", [(c(i), n) for i, (_, n) in enumerate(gb)], fagg,
                                                            P.shuffle_reader(1, part))), 2))]
    return [Stage(1, P.shuffle_writer(s1, 1)),
            Stage(2, P.shuffle_writer(final(P.aggregate("Final", [], fagg, P.coalesce_partitions(P.shuffle_reader(1, part)))), 2), n_tasks=1)]


def partial_only(src, aggs, keys=()):
    """One stage: the Partial aggregate, so that its state columns come back as the result."""
    pagg = [P.agg(fn, a, name, arg2=b) for fn, a, b, name, _ in aggs]
    return [Stage(1, P.shuffle_writer(P.aggregate("Partial", list(keys), pagg, src), 1))]
