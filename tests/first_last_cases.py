"""Shared pieces of the first_value / last_value tests: the rules of DESIGN.md §6 (xvii) restated in plain Python (sharing
nothing with plan.hpp or the device code), the partial state and its Final merge, and the plans (Single, or Partial ->
shuffle -> Final / FinalPartitioned).

- The candidates of a group are its rows (with IGNORE NULLS: those whose value is not NULL).
- They are sorted stably, in input order, by the ordering; first_value takes the first, last_value the last.  Ties keep
  input order, so the earliest tied row wins for first_value and the latest for last_value.  No candidate: NULL.
- The ordering follows the device sort: floats in the IEEE total order (-0.0 before +0.0, NaN greatest), strings
  bytewise with a proper prefix first, each key with its own direction and NULL placement.
- A Final merges the states whose is_set is true, in the order it reads them, under the same rule.

[EXT-unverified] DataFusion 53 does not define tie-breaking; these rules are the engine's, and no test compares ties with
DataFusion."""
import functools
import struct

from ballista_b200 import plan as P
from ballista_b200.plan import Stage

c = P.col


def f64_total(x):
    """the IEEE total-order rank of a float (as a signed integer)"""
    b = struct.unpack("<q", struct.pack("<d", x))[0]
    return b ^ ((b >> 63) & 0x7FFFFFFFFFFFFFFF)


def value_rank(v):
    if isinstance(v, float):
        return f64_total(v)
    if isinstance(v, str):
        return v.encode()
    if isinstance(v, bool):
        return int(v)
    return v


def compare(a, b, order):
    """three-way compare of two ordering tuples; order: [(asc, nulls_first)]"""
    for x, y, (asc, nulls_first) in zip(a, b, order):
        if x is None or y is None:
            if x is None and y is None:
                continue
            return (-1 if nulls_first else 1) if x is None else (1 if nulls_first else -1)
        rx, ry = value_rank(x), value_rank(y)
        if rx != ry:
            cmp = -1 if rx < ry else 1
            return cmp if asc else -cmp
    return 0


def pick(fn, cands, order):
    """cands: [(x, ordering tuple)] in input order -> the winner (x, ordering tuple), or None without candidates"""
    if not cands:
        return None
    ranked = sorted(cands, key=functools.cmp_to_key(lambda p, q: compare(p[1], q[1], order)))  # stable
    return ranked[0] if fn == "first_value" else ranked[-1]


def first_last(fn, rows, x, keys, order, ignore_nulls=False):
    """rows in input order; x / keys: functions of a row (value and ordering values); -> the result (None = NULL)"""
    cands = [(x(r), tuple(k(r) for k in keys)) for r in rows if not (ignore_nulls and x(r) is None)]
    w = pick(fn, cands, order)
    return None if w is None else w[0]


def partial_state(fn, rows, x, keys, order, ignore_nulls=False):
    """the partial state: (x, ordering values..., is_set)"""
    cands = [(x(r), tuple(k(r) for k in keys)) for r in rows if not (ignore_nulls and x(r) is None)]
    w = pick(fn, cands, order)
    if w is None:
        return (None,) + (None,) * len(keys) + (False,)
    return (w[0],) + w[1] + (True,)


def final_merge(fn, states, order):
    """states in the order the Final reads them -> the result"""
    cands = [(s[0], tuple(s[1:-1])) for s in states if s[-1]]
    w = pick(fn, cands, order)
    return None if w is None else w[0]


def grouped(rows, key_idx, aggs):
    """{key tuple: {name: value}}; aggs: [(fn, x index, [(key index, asc, nulls_first)], ignore_nulls, name)]"""
    groups = {}
    for r in rows:
        groups.setdefault(tuple(r[k] for k in key_idx), []).append(r)
    if not key_idx:
        groups.setdefault((), [])
    out = {}
    for g, rs in groups.items():
        out[g] = {name: first_last(fn, rs, lambda r, i=xi: r[i], [lambda r, i=k: r[i] for k, _, _ in ob], [(a, n) for _, a, n in ob], ign)
                  for fn, xi, ob, ign, name in aggs}
    return out


# ---- plans ----------------------------------------------------------------------------------------------------------------
def sort_keys(ob):
    """[(expr, asc, nulls_first)] -> sort_key entries"""
    return [P.sort_key(e, a, n) for e, a, n in ob]


def state_fields(name, fn, x_type, ob_fields):
    """the Partial output's state fields of one aggregate: ob_fields = [(column name, column index, type)]"""
    return [P.field(f"{name}[{fn}]", x_type, True)] + [P.field(f"{n}@{i}", t, True) for n, i, t in ob_fields] + [P.field("is_set", "bool", True)]


def stages(src, aggs, keys=(), key_fields=(), mode="Single", n_out=3):
    """aggs: [(fn, x expr, x IR type, [(expr, asc, nulls_first)], ignore_nulls, name)] with column expressions in the
    ordering (their state fields are named "<col>@<index>"); keys: [(expr, name)]; key_fields: their IR fields.  mode
    "Single" / "SinglePartitioned": one stage; "Partial": Partial -> shuffle -> FinalPartitioned (with keys) or Final."""
    names = [f["name"] for f in src["schema"]]
    pagg = [P.agg(fn, x, name, order_by=sort_keys(ob), ignore_nulls=ign) for fn, x, _, ob, ign, name in aggs]
    gb = list(keys)
    if mode in ("Single", "SinglePartitioned"):
        return [Stage(1, P.shuffle_writer(P.aggregate(mode, gb, pagg, src), 1))]
    s1 = P.aggregate("Partial", gb, pagg, src)
    part = list(key_fields)
    for fn, x, xt, ob, ign, name in aggs:
        obf = [(e["col"], names.index(e["col"]), next(f["type"] for f in src["schema"] if f["name"] == e["col"])) for e, _, _ in ob]
        part += state_fields(name, fn, xt, obf)
    fagg = [P.agg(fn, None, name, order_by=sort_keys(ob), ignore_nulls=ign) for fn, x, _, ob, ign, name in aggs]
    nk = len(gb)
    if nk:
        return [Stage(1, P.shuffle_writer(s1, 1, [c(i) for i in range(nk)], n_out)),
                Stage(2, P.shuffle_writer(P.aggregate("FinalPartitioned", [(c(i), n) for i, (_, n) in enumerate(gb)], fagg,
                                                      P.shuffle_reader(1, part)), 2))]
    return [Stage(1, P.shuffle_writer(s1, 1)),
            Stage(2, P.shuffle_writer(P.aggregate("Final", [], fagg, P.coalesce_partitions(P.shuffle_reader(1, part))), 2), n_tasks=1)]


def partial_only(src, aggs, keys=()):
    """One stage: the Partial aggregate, so that its state columns come back as the result."""
    pagg = [P.agg(fn, x, name, order_by=sort_keys(ob), ignore_nulls=ign) for fn, x, _, ob, ign, name in aggs]
    return [Stage(1, P.shuffle_writer(P.aggregate("Partial", list(keys), pagg, src), 1))]
