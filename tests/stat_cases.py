"""Shared pieces of the VAR / STDDEV / COVAR / CORR tests: the plans (Single, or Partial -> shuffle -> Final) and the
expected values computed in exact rational arithmetic (fractions.Fraction over the Float64 values the arguments are
coerced to), with the NULL rules of the engine."""
import math
from fractions import Fraction

import pyarrow as pa

from ballista_b200 import plan as P
from ballista_b200.plan import Stage

c = P.col

# canonical name -> (arguments, partial state suffixes)
STATE = {
    "var": ["count", "mean", "m2"], "var_samp": ["count", "mean", "m2"], "var_sample": ["count", "mean", "m2"],
    "var_pop": ["count", "mean", "m2"], "var_population": ["count", "mean", "m2"],
    "stddev": ["count", "mean", "m2"], "stddev_samp": ["count", "mean", "m2"], "stddev_pop": ["count", "mean", "m2"],
    "covar": ["count", "mean1", "mean2", "algo_const"], "covar_samp": ["count", "mean1", "mean2", "algo_const"],
    "covar_pop": ["count", "mean1", "mean2", "algo_const"],
    "corr": ["count", "mean1", "m2_1", "mean2", "m2_2", "algo_const"],
}
BIVARIATE = {"covar", "covar_samp", "covar_pop", "corr"}


def part_fields(aggs):
    """The Partial output's state fields of `aggs` [(fn, x, y, name)]."""
    return [P.field(f"{name}[{s}]", "u64" if s == "count" else "f64", True) for fn, _, _, name in aggs for s in STATE[fn]]


def stat_stages(src, aggs, keys=(), key_fields=(), mode="Single", n_out=3, extra=()):
    """aggs: [(fn, x expr, y expr or None, name)]; keys: [(expr, name)]; key_fields: their IR fields (for the shuffle).
    extra: further (fn, expr, name, state fields, Final input_type or None) aggregates mixed into the same AggregateExec."""
    pagg = [P.agg(fn, x, name, arg2=y) for fn, x, y, name in aggs] + [P.agg(fn, x, name) for fn, x, name, _, _ in extra]
    gb = list(keys)
    if mode == "Single":
        return [Stage(1, P.shuffle_writer(P.aggregate("Single", gb, pagg, src), 1))]
    s1 = P.aggregate("Partial", gb, pagg, src)
    part = list(key_fields) + part_fields(aggs) + [f for _, _, _, fs, _ in extra for f in fs]
    fagg = [P.agg(fn, None, name) for fn, _, _, name in aggs] + [P.agg(fn, None, name, input_type=it) for fn, _, name, _, it in extra]
    nk = len(gb)
    if nk:
        return [Stage(1, P.shuffle_writer(s1, 1, [c(i) for i in range(nk)], n_out)),
                Stage(2, P.shuffle_writer(P.aggregate("FinalPartitioned", [(c(i), n) for i, (_, n) in enumerate(gb)], fagg,
                                                      P.shuffle_reader(1, part)), 2))]
    return [Stage(1, P.shuffle_writer(s1, 1)),
            Stage(2, P.shuffle_writer(P.aggregate("Final", [], fagg, P.coalesce_partitions(P.shuffle_reader(1, part))), 2), n_tasks=1)]


def _f(v):
    return None if v is None else float(v)


def exact(fn, xs, ys=None):
    """The value of `fn` over the Float64 values xs (and ys), exactly rounded from rational arithmetic; None = NULL.
    NaN / Inf in the input make the result NaN, as IEEE arithmetic propagates them."""
    if fn in BIVARIATE:
        pairs = [(x, y) for x, y in zip(xs, ys) if x is not None and y is not None]
    else:
        pairs = [(x, x) for x in xs if x is not None]
    n = len(pairs)
    samp = fn in ("var", "var_samp", "var_sample", "stddev", "stddev_samp", "covar", "covar_samp")
    if n == 0 or (samp and n <= 1) or (fn == "corr" and n < 2):
        return None
    if any(not math.isfinite(v) for p in pairs for v in p):
        return math.nan
    X = [Fraction(x) for x, _ in pairs]
    Y = [Fraction(y) for _, y in pairs]
    mx, my = sum(X) / n, sum(Y) / n
    co = sum((x - mx) * (y - my) for x, y in zip(X, Y))
    if fn == "corr":
        vx = sum((x - mx) ** 2 for x in X)
        vy = sum((y - my) ** 2 for y in Y)
        if vx == 0 or vy == 0:
            return None  # [EXT] the engine's rule (unpinned)
        return _corr(co, vx, vy)
    v = co / (n - 1 if samp else n)
    if fn.startswith("stddev"):
        return _sqrt(v)
    return float(v)


def _sqrt(q: Fraction) -> float:
    """sqrt of a non-negative rational, correctly rounded to within an ulp"""
    return math.sqrt(q.numerator) / math.sqrt(q.denominator) if q.denominator < 2**1000 and q.numerator < 2**1000 else math.sqrt(float(q))


def _corr(co: Fraction, vx: Fraction, vy: Fraction) -> float:
    r2 = co * co / (vx * vy)
    r = _sqrt(r2)
    return r if co >= 0 else -r


def rel_close(got, want, rtol):
    if want is None or got is None:
        return got is None and want is None
    if math.isnan(want) or math.isnan(got):
        return math.isnan(want) and math.isnan(got)
    if want == 0:
        return abs(got) <= rtol
    return abs(got - want) <= rtol * abs(want)


def grouped_exact(table: pa.Table, key_names, aggs, f=None):
    """{key tuple: {name: exact value}} for aggs [(fn, xcol, ycol, name)] over the columns of `table` as Float64
    (f: another per-group function with the signature of `exact`, e.g. `welford`)."""
    f = f or exact
    keys = [table.column(k).to_pylist() for k in key_names]
    cols = {}
    for _, x, y, _ in aggs:
        for col in (x, y):
            if col is not None and col not in cols:
                cols[col] = [_f(v) for v in table.column(col).to_pylist()]
    groups = {}
    for i in range(table.num_rows):
        groups.setdefault(tuple(k[i] for k in keys), []).append(i)
    if not key_names:
        groups.setdefault((), [])
    out = {}
    for g, rows in groups.items():
        out[g] = {name: f(fn, [cols[x][i] for i in rows], [cols[y][i] for i in rows] if y else None) for fn, x, y, name in aggs}
    return out


def check_result(got: pa.Table, key_names, want, names, rtol):
    """every group of `want` exactly once in `got`, each value within rtol (relative) of the exact one"""
    assert got.num_rows == len(want), (got.num_rows, len(want))
    rows = got.to_pylist()
    for r in rows:
        g = tuple(r[k] for k in key_names)
        assert g in want, g
        for nm in names:
            assert rel_close(r[nm], want[g][nm], rtol), (g, nm, r[nm], want[g][nm])


def welford(fn, xs, ys=None, parts=1):
    """DataFusion's own computation, restated: a Welford update per row (variance.rs / covariance.rs update_batch) in
    `parts` contiguous partitions, whose states are then combined with its merge_batch (Chan's formula).  The device is
    checked against this within 1e-10 and against `exact` within 1e-12; the reference's goldens are this function's
    roundings."""
    if fn in BIVARIATE:
        pairs = [(x, y) for x, y in zip(xs, ys) if x is not None and y is not None]
    else:
        pairs = [(x, x) for x in xs if x is not None]
    step = max((len(pairs) + parts - 1) // parts, 1)
    states = []
    for p in range(parts):
        n = 0
        m1 = m2 = s11 = s22 = s12 = 0.0
        for x, y in pairs[p * step:(p + 1) * step]:
            n += 1
            d1 = x - m1
            m1 = d1 / n + m1
            d2 = y - m2
            m2 = d2 / n + m2
            s11 += d1 * (x - m1)
            s22 += d2 * (y - m2)
            s12 += d1 * (y - m2)
        states.append((n, m1, m2, s11, s22, s12))
    n, m1, m2, s11, s22, s12 = states[0]
    for c, a1, a2, t11, t22, t12 in states[1:]:
        if c == 0:
            continue
        nn = n + c
        e1, e2 = m1 - a1, m2 - a2
        s11 += t11 + e1 * e1 * n * c / nn
        s22 += t22 + e2 * e2 * n * c / nn
        s12 += t12 + e1 * e2 * n * c / nn
        m1 = m1 * n / nn + a1 * c / nn
        m2 = m2 * n / nn + a2 * c / nn
        n = nn
    samp = fn in ("var", "var_samp", "var_sample", "stddev", "stddev_samp", "covar", "covar_samp")
    if n == 0 or (samp and n <= 1) or (fn == "corr" and n < 2):
        return None
    if fn == "corr":
        if s11 == 0 or s22 == 0:
            return None if all(math.isfinite(v) for p in pairs for v in p) else math.nan
        return s12 / (math.sqrt(s11) * math.sqrt(s22))
    v = (s12 if fn in BIVARIATE else s11) / (n - 1 if samp else n)
    return math.sqrt(v) if fn.startswith("stddev") else v
