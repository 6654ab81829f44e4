"""GPU: the math functions of DESIGN.md §6 (xviii) on the device, against the per-row restatement in math_fn_cases.py (itself
pinned against libm and mpmath by test_math_functions.py).  The exact functions and every special value bit for bit; the
transcendental functions within the tabulated ulp bound of the correctly rounded value; each function in a projection, a
FilterExec predicate, a group key and a SUM argument; the execution errors; the protobuf fixtures; a lineitem query."""
import base64
import collections
import json
import math
import os

import numpy as np
import pyarrow as pa
import pytest

import golden_data as G
import math_fn_cases as M
import queries as Q
from ballista_b200 import driver, engine
from ballista_b200 import plan as P

pytestmark = pytest.mark.gpu
c = P.col
HERE = os.path.dirname(os.path.abspath(__file__))
EXECUTION, UNSUPPORTED = -3, -2
N = 3500  # three full 1024-row tiles and a partial one


def _f64_col(vals, nulls_every=0):
    """a Float64 column from Python floats, bits kept; every nulls_every-th row NULL"""
    data = np.array([M.bits(v) for v in vals], dtype=np.uint64).view(np.float64)
    mask = None if not nulls_every else np.array([(r % nulls_every) == 3 for r in range(len(vals))])
    return pa.array(data, pa.float64(), mask=mask)


def _f32_col(vals, nulls_every=0):
    data = np.array([M.f64_to_f32_bits(M.bits(v)) for v in vals], dtype=np.uint32).view(np.float32)
    mask = None if not nulls_every else np.array([(r % nulls_every) == 3 for r in range(len(vals))])
    return pa.array(data, pa.float32(), mask=mask)


def _values(arr):
    """the column's values as the engine holds them: floats with their bits (Float32 widened), None for NULL"""
    arr = arr.combine_chunks() if isinstance(arr, pa.ChunkedArray) else arr
    valid = arr.is_valid().to_pylist()
    if pa.types.is_float64(arr.type):
        raw = np.frombuffer(arr.buffers()[1], dtype=np.uint64, count=len(arr) + arr.offset)[arr.offset:]
        return [M.from_bits(int(u)) if v else None for u, v in zip(raw, valid)]
    if pa.types.is_float32(arr.type):
        raw = np.frombuffer(arr.buffers()[1], dtype=np.uint32, count=len(arr) + arr.offset)[arr.offset:]
        return [M.from_bits(M.f32_to_f64_bits(int(u))) if v else None for u, v in zip(raw, valid)]
    return arr.to_pylist()


def _spread(vals, n, seed):
    """n values: every edge value at least twice (in different tiles), the rest drawn from them"""
    rng = np.random.default_rng(seed)
    out = list(vals) + [vals[int(i)] for i in rng.integers(0, len(vals), n - 2 * len(vals))] + list(vals)
    return out[:n]


@pytest.fixture(scope="module")
def edge():
    x64 = _spread(M.EDGE64, N, 1)
    y64 = _spread(M.EDGE64, N, 2)
    x32 = _spread(M.EDGE32, N, 3)
    y32 = _spread(M.EDGE32, N, 4)
    cols = {"a": _f64_col(x64), "an": _f64_col(x64), "az": _f64_col(x64, 7), "y": _f64_col(y64),
            "b": _f32_col(x32), "bn": _f32_col(x32), "bz": _f32_col(x32, 7), "y32": _f32_col(y32)}
    return pa.table(cols)


EDGE_SCHEMA = [P.field("a", "f64", False), P.field("an", "f64", True), P.field("az", "f64", True), P.field("y", "f64", False),
               P.field("b", "f32", False), P.field("bn", "f32", True), P.field("bz", "f32", True), P.field("y32", "f32", False)]


def _project(exprs, table, schema):
    return [Q.Stage(1, P.shuffle_writer(P.project([(e, n) for n, e in exprs], P.scan(table, schema)), 1))]


def _run(gpu, exprs, table, schema, tag):
    out = []
    for i in range(0, len(exprs), 8):
        res = driver.run_stages(gpu, _project(exprs[i:i + 8], table, schema), f"{tag}-{i}")
        out += [(n, _values(res.column(n))) for n, _ in exprs[i:i + 8]]
    return dict(out)


def _float_cases():
    """(output name, IR, reference over (x, y), transcendental name or None, is32, x column, y column or None)"""
    out = []
    for is32, cols in ((False, ("a", "an", "az", "y")), (True, ("b", "bn", "bz", "y32"))):
        t = "f32" if is32 else "f64"
        for col in cols[:3]:
            for n in M.UNARY + ["isnan", "iszero"]:
                out.append((f"{n}_{col}", P.fn(n, c(col)), lambda x, y, n=n, is32=is32: M.unary(n, x, is32),
                            n if n in M.TRANSCENDENTAL else None, is32, col, None))
            out.append((f"log_{col}", P.fn("log", c(col)), lambda x, y, is32=is32: M.unary("log10", x, is32), "log10", is32, col, None))
            out.append((f"logb_{col}", P.fn("log", c(cols[3]), c(col)), lambda x, y, is32=is32: M.log_base(y, x, is32), "log_base",
                        is32, col, cols[3]))
            out.append((f"atan2_{col}", P.fn("atan2", c(col), c(cols[3])), lambda x, y, is32=is32: M.atan2(x, y, is32), "atan2",
                        is32, col, cols[3]))
            out.append((f"nanvl_{col}", P.fn("nanvl", c(col), c(cols[3])), lambda x, y: M.nanvl(x, y), None, is32, col, cols[3]))
            for d in (0, 2, -1, 22):
                out.append((f"trunc{d}_{col}".replace("-", "m"), P.fn("trunc", c(col), P.lit_i64(d)),
                            lambda x, y, d=d, is32=is32: M.trunc(x, d, is32), None, is32, col, None))
            if not is32:
                out.append((f"power_{col}", P.fn("power", c(col), c("y")), lambda x, y: M.power(x, y), "power", False, col, "y"))
        del t
    return out


FLOAT_CASES = _float_cases()


def _check(name, got, xs, ys, ref, trans, is32, worst, bad):
    for r, g in enumerate(got):
        x = xs[r]
        y = None if ys is None else ys[r]
        w = ref(x, y) if x is not None else None
        if x is None:
            if g is not None:
                bad.append((name, r, "not NULL"))
            continue
        if isinstance(w, bool):
            if g != w:
                bad.append((name, r, x, g, w))
            continue
        if trans is None or M.special([x] + ([] if y is None else [y]), w):
            if M.bits(g) != M.bits(w):
                bad.append((name, r, hex(M.bits(x)), y, hex(M.bits(g)), hex(M.bits(w))))
            continue
        args = (y, x) if trans == "log_base" else (x, y) if y is not None else (x,)
        err = M.ulp_error(g, M.exact(trans, *args), is32)
        key = (trans, "f32" if is32 else "f64")
        worst[key] = max(worst.get(key, 0.0), err)
        if err > M.ULP_BOUND[key[1]][trans] + 0.5:
            bad.append((name, r, x, y, g, w, err))


def test_edge_table_bit_for_bit(gpu, edge):
    """the exact functions and every special value equal the restatement bit for bit; the rest stay within their bound"""
    G.register(gpu, "mx", edge, 3)
    vm0 = gpu.counter("vm")
    got = _run(gpu, [(n, e) for n, e, *_ in FLOAT_CASES], "mx", EDGE_SCHEMA, "math-edge")
    assert gpu.counter("vm") > vm0
    cols = {k: _values(edge.column(k)) for k in edge.column_names}
    worst, bad = {}, []
    for name, _, ref, trans, is32, xc, yc in FLOAT_CASES:
        _check(name, got[name], cols[xc], None if yc is None else cols[yc], ref, trans, is32, worst, bad)
    assert not bad, (collections.Counter(b[0] for b in bad), bad[:20])


def test_transcendental_functions_within_their_ulp_bound(gpu):
    """>= 4096 seeded values per function and type, log-uniform magnitudes, both signs; the largest error is printed"""
    n = 4096
    cols, cases = {}, []
    for k, name in enumerate(M.TRANSCENDENTAL):
        for is32 in (False, True):
            if name == "power" and is32:
                continue
            col = f"{name}_{'f32' if is32 else 'f64'}"
            base = name if name not in ("log_base", "atan2", "power") else "ln" if name == "log_base" else "atan"
            xs = M.sample(base, n, is32, 1000 + 2 * k + is32)
            if name == "power":
                xs = [abs(v) for v in M.sample("exp", n, False, 77)]
                xs = [math.exp(v / 100) for v in xs]
            cols[col] = (_f32_col if is32 else _f64_col)(xs)
            if name in ("log_base", "atan2", "power"):
                ys = M.sample("exp" if name == "power" else base, n, is32, 5000 + k + is32)
                if name == "log_base":
                    ys = [abs(v) for v in ys]
                cols[col + "_y"] = (_f32_col if is32 else _f64_col)(ys)
            cases.append((name, is32, col))
    t = pa.table(cols)
    sch = [P.field(k, "f32" if k.split("_y")[0].endswith("f32") else "f64", False) for k in t.column_names]
    G.register(gpu, "mt", t, 2)
    exprs = []
    for name, is32, col in cases:
        if name == "log_base":
            e = P.fn("log", c(col + "_y"), c(col))
        elif name in ("atan2", "power"):
            e = P.fn(name, c(col), c(col + "_y"))
        else:
            e = P.fn("ln" if name == "ln" else name, c(col))
        exprs.append((col + "_r", e))
    got = _run(gpu, exprs, "mt", sch, "math-ulp")
    vals = {k: _values(t.column(k)) for k in t.column_names}
    worst, bad = {}, []
    for name, is32, col in cases:
        xs, ys = vals[col], vals.get(col + "_y")
        if name == "log_base":
            ref = lambda x, y, is32=is32: M.log_base(y, x, is32)  # noqa: E731
        elif name in ("atan2", "power"):
            ref = (lambda x, y, is32=is32: M.atan2(x, y, is32)) if name == "atan2" else (lambda x, y: M.power(x, y))
        else:
            ref = lambda x, y, name=name, is32=is32: M.unary(name, x, is32)  # noqa: E731
        _check(col, got[col + "_r"], xs, ys, ref, name, is32, worst, bad)
    print("largest ulp error observed:", json.dumps({f"{k[0]}/{k[1]}": round(v, 3) for k, v in sorted(worst.items())}))
    assert not bad, (collections.Counter(b[0] for b in bad), bad[:20])
    assert len(worst) == 2 * len(M.TRANSCENDENTAL) - 1


def test_integer_functions_exact(gpu):
    """gcd / lcm over every pair of Int64 edge values that does not fail, factorial over -3..20; NULLs in every position"""
    pairs = []
    for x in M.INT_EDGE:
        for y in M.INT_EDGE:
            try:
                M.gcd(x, y), M.lcm(x, y)
            except M.Overflow:
                continue
            pairs.append((x, y))
    rows = (pairs * (N // len(pairs) + 1))[:N]
    a, b = [x for x, _ in rows], [y for _, y in rows]
    f = [r % 24 - 3 for r in range(N)]
    az = [None if r % 5 == 1 else x for r, x in enumerate(a)]
    t = pa.table({"a": pa.array(a, pa.int64()), "b": pa.array(b, pa.int64()), "f": pa.array(f, pa.int64()), "az": pa.array(az, pa.int64())})
    G.register(gpu, "mi", t, 2)
    sch = [P.field("a", "i64", False), P.field("b", "i64", False), P.field("f", "i64", False), P.field("az", "i64", True)]
    exprs = [("gcd", P.fn("gcd", c("a"), c("b"))), ("lcm", P.fn("lcm", c("a"), c("b"))), ("fact", P.fn("factorial", c("f"))),
             ("gcdz", P.fn("gcd", c("az"), c("b"))), ("lcmz", P.fn("lcm", c("b"), c("az")))]
    got = _run(gpu, exprs, "mi", sch, "math-int")
    assert got["gcd"] == [M.gcd(x, y) for x, y in rows]
    assert got["lcm"] == [M.lcm(x, y) for x, y in rows]
    assert got["fact"] == [M.factorial(v) for v in f]
    assert got["gcdz"] == [M.gcd(z, y) for z, y in zip(az, b)]
    assert got["lcmz"] == [M.lcm(y, z) for z, y in zip(az, b)]


def test_integer_functions_exact_over_rows_that_fit(gpu):
    """the rows above are chosen so that nothing fails; here power over each edge base with every exponent that fits"""
    xs, es, want = [], [], []
    for x in M.INT_EDGE:
        for e in range(0, 66):
            try:
                w = M.power(x, e)
            except M.Overflow:
                continue
            xs.append(x)
            es.append(e)
            want.append(w)
    t = pa.table({"x": pa.array(xs, pa.int64()), "e": pa.array(es, pa.int64())})
    G.register(gpu, "mp", t, 1)
    got = _run(gpu, [("p", P.fn("power", c("x"), c("e")))], "mp", [P.field("x", "i64", False), P.field("e", "i64", False)], "math-pow")
    assert got["p"] == want


ERRORS = [
    ("factorial", lambda v: P.fn("factorial", v), 21, 5, "overflow"),
    ("power_negative", lambda v: P.fn("power", P.lit_i64(2), v), -1, 3, "exponent"),
    ("power_overflow", lambda v: P.fn("power", P.lit_i64(2), v), 63, 3, "overflow"),
    ("gcd", lambda v: P.fn("gcd", v, P.lit_i64(0)), M.INT64_MIN, 4, "overflow"),
    ("lcm", lambda v: P.fn("lcm", v, P.lit_i64(3)), M.INT64_MIN, 4, "overflow"),
]


@pytest.mark.parametrize("name,mk,bad,good,word", ERRORS, ids=[e[0] for e in ERRORS])
def test_execution_errors(gpu, name, mk, bad, good, word):
    """raised at the first row, the last row and a later tile's row; not when that row is NULL, filtered out, or not
    selected by a CASE"""
    sch = [P.field("v", "i64", True), P.field("k", "i64", False)]
    for at in (0, N - 1, 2500):
        vals = [good] * N
        vals[at] = bad
        keep = [1] * N
        t = pa.table({"v": pa.array(vals, pa.int64()), "k": pa.array(keep, pa.int64())})
        G.register(gpu, "me", t, 1)
        with pytest.raises(engine.B200Error) as ei:
            driver.run_stages(gpu, _project([("r", mk(c("v")))], "me", sch), f"me-{name}-{at}")
        assert ei.value.code == EXECUTION and word in str(ei.value).lower(), str(ei.value)
        # NULL there: no error
        nulled = pa.table({"v": pa.array([None if r == at else v for r, v in enumerate(vals)], pa.int64()), "k": t.column("k")})
        G.register(gpu, "me", nulled, 1)
        out = driver.run_stages(gpu, _project([("r", mk(c("v")))], "me", sch), f"me-null-{name}-{at}")
        assert out.column("r")[at].as_py() is None
        # filtered out: no error
        kk = pa.array([0 if r == at else 1 for r in range(N)], pa.int64())
        G.register(gpu, "me", pa.table({"v": t.column("v"), "k": kk}), 1)
        filt = P.filter_(P.binop("=", c("k"), P.lit_i64(1)), P.scan("me", sch))
        st = [Q.Stage(1, P.shuffle_writer(P.project([(mk(c(0)), "r")], filt), 1))]
        out = driver.run_stages(gpu, st, f"me-filt-{name}-{at}")
        assert out.num_rows == N - 1
        # a CASE that does not select the row: no error
        e = P.case([(P.binop("=", c("k"), P.lit_i64(1)), mk(c("v")))], P.lit_i64(-7))
        out = driver.run_stages(gpu, _project([("r", e)], "me", sch), f"me-case-{name}-{at}")
        assert out.column("r")[at].as_py() == -7


POSITION_FNS = [n for n in M.UNARY] + ["isnan", "iszero", "log", "log_base", "atan2", "nanvl", "power", "trunc", "gcd", "lcm",
                                        "factorial", "power_i64", "pi"]


def _position_expr(name):
    if name == "log_base":
        return P.fn("log", c("y"), c("a")), "f64"
    if name in ("atan2", "nanvl", "power"):
        return P.fn(name, c("a"), c("y")), "f64"
    if name == "trunc":
        return P.fn("trunc", c("a"), P.lit_i64(1)), "f64"
    if name in ("gcd", "lcm"):
        return P.fn(name, c("i"), P.lit_i64(12)), "i64"
    if name == "factorial":
        return P.fn("factorial", c("i")), "i64"
    if name == "power_i64":
        return P.fn("power", c("i"), P.lit_i64(3)), "i64"
    if name == "pi":
        return P.binop("*", P.fn("pi"), c("a")), "f64"
    return P.fn(name, c("a")), "bool" if name in ("isnan", "iszero") else "f64"


@pytest.mark.parametrize("name", POSITION_FNS)
def test_plan_positions(gpu, name):
    """each function as a projection, inside a FilterExec predicate, as a group key and as a SUM argument; the filter and the
    aggregate agree with the projection's values, and the VM (not the fused / group-by / fast-filter kernels) ran them"""
    rng = np.random.default_rng(21)
    a = [float(v) for v in rng.choice([0.5, 2.0, -1.0, 0.0, 3.0, 10.0, -0.25], N)]
    y = [float(v) for v in rng.choice([2.0, 0.5, 3.0, 10.0], N)]
    i = [int(v) for v in rng.integers(0, 15, N)]
    t = pa.table({"a": pa.array(a, pa.float64()), "y": pa.array(y, pa.float64()), "i": pa.array(i, pa.int64()),
                  "row": pa.array(range(N), pa.int64())})
    G.register(gpu, "mpos", t, 2)
    sch = [P.field("a", "f64", False), P.field("y", "f64", False), P.field("i", "i64", False), P.field("row", "i64", False)]
    e, typ = _position_expr(name)
    proj = _values(driver.run_stages(gpu, _project([("r", e)], "mpos", sch), f"mpos-p-{name}").column("r"))
    counters = {k: gpu.counter(k) for k in ("vm", "fastfilter", "fused", "groupby")}
    pred = e if typ == "bool" else P.binop(">", e, P.lit_f64(1.0) if typ == "f64" else P.lit_i64(1))
    st = [Q.Stage(1, P.shuffle_writer(P.filter_(pred, P.scan("mpos", sch), projection=[3]), 1))]
    out = driver.run_stages(gpu, st, f"mpos-f-{name}")
    got_rows = [] if out is None else out.column("row").to_pylist()

    def gt(v):
        if typ == "bool":
            return v is True
        if v != v:
            return not math.copysign(1, v) < 0  # total order: a positive NaN sorts above everything, a negative one below
        return v > 1
    assert got_rows == [r for r, v in enumerate(proj) if gt(v)]
    arg = P.cast(e, "i64") if typ == "bool" else e
    arg_t = "i64" if typ in ("bool", "i64") else "f64"
    # keyed on (f, CAST(i AS DOUBLE)): more than 4 groups and a float key, so the Final stage (which reads the key as a
    # column) is not small enough for the fused kernel nor integer-keyed for the group-by kernel
    part = P.aggregate("Partial", [(e, "g"), (P.cast(c("i"), "f64"), "i")], [P.agg("sum", arg, "s"), P.agg("count", None, "n")],
                       P.scan("mpos", sch))
    st1 = Q.Stage(1, P.shuffle_writer(part, 1, [c(0), c(1)], 2))
    fields = [P.field("g", typ, True), P.field("i", "f64", False), P.field("s[sum]", arg_t, True), P.field("n[count]", "i64", True)]
    fin = P.aggregate("FinalPartitioned", [(c(0), "g"), (c(1), "i")],
                      [P.agg("sum", c(2), "s", input_type=arg_t), P.agg("count", c(3), "n")], P.shuffle_reader(1, fields))
    res = driver.run_stages(gpu, [st1, Q.Stage(2, P.shuffle_writer(fin, 2))], f"mpos-g-{name}")
    want = {}
    for v, k in zip(proj, i):
        key = (M.bits(v) if isinstance(v, float) else v, float(k))
        want.setdefault(key, []).append(v)
    gk = _values(res.column("g"))
    got = {((M.bits(k) if isinstance(k, float) else k), ki): (s, n)
           for k, ki, s, n in zip(gk, res.column("i").to_pylist(), res.column("s").to_pylist(), res.column("n").to_pylist())}
    assert set(got) == set(want)
    for k, vs in want.items():
        s, n = got[k]
        assert n == len(vs)
        if typ == "f64":
            w = math.fsum(vs)
            assert (s != s and w != w) or s == w or abs(s - w) <= 1e-12 * abs(w), (k, s, w)
        else:
            assert s == sum(int(v) for v in vs)
    assert gpu.counter("vm") > counters["vm"]
    if name != "pi":  # pi() is folded into a literal: its plans hold no math op and may take any kernel
        for k in ("fastfilter", "fused", "groupby"):
            assert gpu.counter(k) == counters[k], k


with open(os.path.join(HERE, "golden", "math_fn_proto_plans.json")) as _fh:
    PROTO_CASES = json.load(_fh)["cases"]


class _FromProto:
    def __init__(self, eng, cases):
        self._e, self._c = eng, cases

    def __getattr__(self, name):
        return getattr(self._e, name)

    def create_query_stage_exec(self, job_id, stage_id, plan_json):
        return self._e.create_query_stage_exec_proto(job_id, stage_id, base64.b64decode(self._c[stage_id]["proto_b64"]))


def test_every_fixture_runs_from_its_bytes(gpu):
    rng = np.random.default_rng(5)
    n = 2500
    t = pa.table({"k": pa.array(rng.integers(0, 5, n), pa.int32()), "x": pa.array(rng.integers(-30, 30, n), pa.int64()),
                  "f": pa.array(rng.choice([0.5, 2.0, -1.5, 0.0, 7.25, float("nan")], n), pa.float64()),
                  "g": pa.array(rng.choice([0.5, 2.0, -1.5, 0.0, 7.25], n), pa.float32()),
                  "s": pa.array(["a"] * n, pa.string()), "dec": pa.array([None] * n, pa.decimal128(15, 2))})
    G.register(gpu, "t", t, 2)
    groups = {}
    for case in PROTO_CASES:
        if not case["refused"]:
            groups.setdefault(case["name"].rsplit("/", 1)[0], {})[int(case["name"].rsplit("stage", 1)[1])] = case
    assert len(groups) >= 3 * 35
    for j, (name, cases) in enumerate(sorted(groups.items())):
        stages = [Q.Stage(i, json.loads(cases[i]["ir"])) for i in sorted(cases)]
        got = driver.run_stages(_FromProto(gpu, cases), stages, f"mf-proto-{j}")
        want = driver.run_stages(gpu, stages, f"mf-ir-{j}")
        if want is None:
            assert got is None or got.num_rows == 0, name
            continue
        ordered = "/projection" in name or "/filter" in name
        a = got.to_pylist() if ordered else sorted(got.to_pylist(), key=repr)
        b = want.to_pylist() if ordered else sorted(want.to_pylist(), key=repr)
        assert repr(a) == repr(b), name
    # a non-literal trunc digit count decodes and types, and is refused when the stage is lowered
    lit = [x for x in PROTO_CASES if x["refused"] == "literal"]
    assert lit
    with pytest.raises(engine.B200Error) as ei:
        driver.run_stages(_FromProto(gpu, {1: lit[0]}), [Q.Stage(1, json.loads(lit[0]["ir"]))], "mf-proto-lit")
    assert ei.value.code == UNSUPPORTED and "literal" in str(ei.value), str(ei.value)


def test_lineitem_aggregate(gpu):
    """l_returnflag, l_linestatus, SUM(ln(price)), AVG(sqrt(quantity)), MAX(power(discount, 2.0)) over generated lineitem,
    against the restatement over the exported columns (1e-12 relative; math.fsum for the sums)"""
    import oracle_ffi
    cols = ["l_returnflag", "l_linestatus", "l_quantity", "l_extendedprice", "l_discount"]
    msf, parts = 200, 2
    n = oracle_ffi.lib().oracle_tpch_table_rows(b"lineitem", msf)
    gpu.drop_table("lineitem")
    step = (n + parts - 1) // parts
    for p in range(parts):
        gpu.tpch_generate("lineitem", msf, p, p * step, min(n, (p + 1) * step), cols)
    data = pa.Table.from_batches([gpu.export_table("lineitem", p) for p in range(parts)])
    sch = [P.field("l_returnflag", "utf8", False), P.field("l_linestatus", "utf8", False), P.field("l_quantity", P.dec(15, 2), False),
           P.field("l_extendedprice", P.dec(15, 2), False), P.field("l_discount", P.dec(15, 2), False)]
    scan = P.scan("lineitem", sch)
    lnp = P.fn("ln", P.cast(c("l_extendedprice"), "f64"))
    sq = P.fn("sqrt", P.cast(c("l_quantity"), "f64"))
    pw = P.fn("power", P.cast(c("l_discount"), "f64"), P.lit_f64(2.0))
    part = P.aggregate("Partial", [(c("l_returnflag"), "rf"), (c("l_linestatus"), "ls")],
                       [P.agg("sum", lnp, "s"), P.agg("avg", sq, "a"), P.agg("max", pw, "m")], scan)
    st1 = Q.Stage(1, P.shuffle_writer(part, 1, [c(0), c(1)], 2))
    fields = json.loads(engine.plan_typed_json(st1.json("j")))["input"]["schema"]
    fin = P.aggregate("FinalPartitioned", [(c(0), "rf"), (c(1), "ls")],
                      [P.agg("sum", c(2), "s", input_type="f64"), P.agg("avg", c(3), "a", input_type="f64"),
                       P.agg("max", c(5), "m", input_type="f64")], P.shuffle_reader(1, fields))
    got = driver.run_stages(gpu, [st1, Q.Stage(2, P.shuffle_writer(fin, 2))], "math-lineitem")
    rf, ls = data.column("l_returnflag").to_pylist(), data.column("l_linestatus").to_pylist()
    q = [float(v) for v in data.column("l_quantity").to_pylist()]
    ep = [float(v) for v in data.column("l_extendedprice").to_pylist()]
    di = [float(v) for v in data.column("l_discount").to_pylist()]
    want = {}
    for r in range(data.num_rows):
        w = want.setdefault((rf[r], ls[r]), ([], [], []))
        w[0].append(M.unary("ln", ep[r]))
        w[1].append(M.unary("sqrt", q[r]))
        w[2].append(M.power(di[r], 2.0))
    g = {(r["rf"], r["ls"]): r for r in got.to_pylist()}
    assert set(g) == set(want) and len(want) >= 3
    for k, (s, a, m) in want.items():
        assert abs(g[k]["s"] - math.fsum(s)) <= 1e-12 * abs(math.fsum(s)), k
        assert abs(g[k]["a"] - math.fsum(a) / len(a)) <= 1e-12 * abs(math.fsum(a) / len(a)), k
        assert abs(g[k]["m"] - max(m)) <= 1e-12 * max(m), k
