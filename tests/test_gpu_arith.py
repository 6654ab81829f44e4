"""GPU: the tile VM's scalar core -- `+ - * / %`, negation, the six comparisons, the numeric casts and CASE -- bit-exact
against the per-row restatement in arith_cases.py (itself pinned by test_arith.py), over the edge table of every integer,
float and Decimal128 type in its three nullability forms (so the micro-op fast paths and the NULL-aware path both run,
and all three Decimal image widths), 3 full 1024-row tiles plus a partial one, in 1 and 3 partitions."""
import json

import pyarrow as pa
import pytest

import arith_cases as A
import golden_data as G
import queries as Q
from ballista_b200 import driver, engine
from ballista_b200 import plan as P

pytestmark = pytest.mark.gpu
c = P.col
EXECUTION = -3


@pytest.mark.parametrize("parts", [1, 3])
@pytest.mark.parametrize("t", A.TYPES)
def test_operator_matrix(gpu, t, parts):
    """every operator x type, operands column-column, column-literal, literal-column and nested (a register operand), in
    each nullability form, through ProjectionExec"""
    vm0 = gpu.counter("vm")
    bad = []
    for op in A.OPS:
        vals = A.safe_operands(op, t)
        tbl, sch = A.edge_table(t, vals)
        G.register(gpu, "ar", tbl, parts)
        cases = [s for form in A.FORMS for s in A.shapes(op, t, form)]
        bad += [(op,) + b for b in A.check_projection(gpu, f"ar-{t}-{op}-{parts}", "ar", sch, A.rows_of(vals), cases)]
    assert not bad, bad
    assert gpu.counter("vm") > vm0


@pytest.mark.parametrize("t", A.TYPES)
def test_comparisons_and_negation(gpu, t):
    vals = A.operands(t)
    tbl, sch = A.edge_table(t, vals)
    G.register(gpu, "ar", tbl, 2)
    cases = []
    for form in A.FORMS:
        for op in A.CMPS:
            cases.append((f"{op}_{form}", P.binop(op, c(f"a_{form}"), c(f"b_{form}")),
                          lambda r, op=op, form=form: A.compare(op, r[f"a_{form}"], r[f"b_{form}"], t), "bool"))
            cases.append((f"{op}_lit_{form}", P.binop(op, c(f"a_{form}"), A.literal(t, A.edges(t)[1])),
                          lambda r, op=op, form=form: A.compare(op, r[f"a_{form}"], A.edges(t)[1], t), "bool"))
        if t in A.INTS and not A.INTS[t][1]:
            continue
        cases.append((f"neg_{form}", P.neg(c(f"a_{form}")), lambda r, form=form: A.neg(r[f"a_{form}"], t), t))
        if t == "f64":  # the sign of a negated NaN decides a comparison in the total order
            cases.append((f"negcmp_{form}", P.binop("<", P.neg(c(f"a_{form}")), P.lit_f64(0.0)),
                          lambda r, form=form: A.compare("<", A.neg(r[f"a_{form}"], t), 0.0, t), "bool"))
    bad = A.check_projection(gpu, f"ar-cmp-{t}", "ar", sch, A.rows_of(vals), cases)
    assert not bad, bad


FF_TYPES = [t for t in A.TYPES if t not in A.FLOATS]


@pytest.mark.parametrize("t", A.TYPES)
def test_comparisons_as_filters_keep_row_order(gpu, t):
    """each comparison as a FilterExec predicate: on the fast filter kernel where it takes the shape (integer and decimal
    columns without NULLs), and on the tile VM when an arithmetic operand forces it there"""
    vals = A.operands(t)
    rows = A.rows_of(vals)
    tbl, sch = A.edge_table(t, vals)
    G.register(gpu, "ar", tbl, 1)
    row_idx = len(sch) - 1
    z = A.literal(t, A.zero_one(t)[0])
    for op in A.CMPS:
        for form in A.FORMS:
            a, b = c(f"a_{form}"), c(f"b_{form}")
            want = [i for i, r in enumerate(rows) if A.compare(op, r[f"a_{form}"], r[f"b_{form}"], t) is True]
            # a nullable column without NULLs has no validity buffer: the fast filter takes it as a non-nullable one
            preds = [(P.binop(op, a, b), form != "nl" and t in FF_TYPES)]
            if t not in A.FLOATS:  # floats compare on the VM anyway (and float arithmetic may not keep a NaN's bits)
                preds.append((P.binop(op, P.binop("-", a, z), b), False))
            for pred, on_ff in preds:
                ff0, vm0 = gpu.counter("fastfilter"), gpu.counter("vm")
                st = [Q.Stage(1, P.shuffle_writer(P.filter_(pred, P.scan("ar", sch), projection=[row_idx]), 1))]
                out = driver.run_stages(gpu, st, f"ar-f-{t}-{op}-{form}")
                got = [] if out is None else out.column("row").to_pylist()
                assert got == want, (op, form, on_ff)
                if on_ff:
                    assert gpu.counter("fastfilter") > ff0, (op, form)
                else:
                    assert gpu.counter("fastfilter") == ff0 and gpu.counter("vm") > vm0, (op, form)


def _sum_min_max(rows, f):
    vals = [v for v in (f(r) for r in rows) if v is not None]
    return sum(vals), min(vals), max(vals)


@pytest.mark.parametrize("t,expr,ref", [
    ("i32", lambda a, b: P.binop("-", a, b), lambda x, y: A.arith("-", x, y, "i32")),
    ("i64", lambda a, b: P.binop("%", a, P.lit_i64(1000)), lambda x, y: A.arith("%", x, 1000, "i64")),
    ("d15_2", lambda a, b: P.binop("+", a, b), lambda x, y: A.arith("+", x, y, "d15_2")),
    ("d28_6", lambda a, b: P.binop("-", a, b), lambda x, y: A.arith("-", x, y, "d28_6")),
    ("i32", lambda a, b: P.binop("*", P.cast(a, "f64"), P.lit_f64(2.0)), lambda x, y: None if x is None else float(x) * 2.0),
])
def test_aggregate_arguments(gpu, t, expr, ref):
    """SUM / MIN / MAX of an arithmetic argument through Partial -> hash shuffle -> FinalPartitioned; the sums are exact
    (integers, decimals, integer-valued doubles)"""
    vals = A.safe_operands("-", t)
    rows = A.rows_of(vals)
    tbl, sch = A.edge_table(t, vals)
    G.register(gpu, "ar", tbl, 3)
    arg = expr(c("a_nl"), c("b_nl"))
    key = P.binop("%", c("row"), P.lit_i32(3))
    part = P.aggregate("Partial", [(key, "k")], [P.agg("sum", arg, "s"), P.agg("min", arg, "lo"), P.agg("max", arg, "hi")], P.scan("ar", sch))
    st1 = Q.Stage(1, P.shuffle_writer(part, 1, [c(0)], 2))
    fields = json.loads(engine.plan_typed_json(st1.json("j")))["input"]["schema"]
    fin = P.aggregate("FinalPartitioned", [(c(0), "k")], [P.agg("sum", c(1), "s", input_type=_type_of(arg, sch, "ar")),
                                                          P.agg("min", c(2), "lo"), P.agg("max", c(3), "hi")],
                      P.shuffle_reader(1, fields))
    got = driver.run_stages(gpu, [st1, Q.Stage(2, P.shuffle_writer(fin, 2))], f"ar-agg-{t}")
    unscaled = {n: got.column(n).to_pylist() if not pa.types.is_decimal(got.column(n).type) else
                A.to_python(got.column(n), A.dec_name(got.column(n).type.precision, got.column(n).type.scale)) for n in ("s", "lo", "hi")}
    res = {k: (unscaled["s"][i], unscaled["lo"][i], unscaled["hi"][i]) for i, k in enumerate(got.column("k").to_pylist())}
    assert sorted(res) == [0, 1, 2]
    for k in range(3):
        want = _sum_min_max([r for i, r in enumerate(rows) if i % 3 == k], lambda r: ref(r["a_nl"], r["b_nl"]))
        assert res[k] == want, k


# ---- errors: each failing row on its own, at the start, the end and inside a later tile -----------------------------------
N = A.N_ROWS
ERRORS = [
    ("i64_div0", "i64", (5, 0), P.binop("/", c("a"), c("b"))),
    ("i64_mod0", "i64", (5, 0), P.binop("%", c("a"), c("b"))),
    ("i64_min_div", "i64", (-(1 << 63), -1), P.binop("/", c("a"), c("b"))),
    ("i32_min_div", "i32", (-(1 << 31), -1), P.binop("/", c("a"), c("b"))),
    ("i16_min_div", "i16", (-(1 << 15), -1), P.binop("/", c("a"), c("b"))),
    ("u64_div0", "u64", (A.U64_MAX, 0), P.binop("/", c("a"), c("b"))),
    ("dec_div0", "d15_2", (500, 0), P.binop("/", c("a"), c("b"))),
    ("dec_mod0", "d15_2", (500, 0), P.binop("%", c("a"), c("b"))),
    ("dec_mul_overflow", "d38_0", (10 ** 38 - 1, 10 ** 38 - 1), P.binop("*", c("a"), c("b"))),
    ("dec_add_overflow", "d38_0", (10 ** 38 - 1, 10 ** 38 - 1), P.binop("+", c("a"), c("b"))),
    ("dec_div_scale_overflow", "d38_0", (10 ** 38 - 1, 3), P.binop("/", c("a"), c("b"))),
    ("int_to_dec_precision", "i64", (100000, 1), P.cast(c("a"), P.dec(5, 0))),
]


def _error_table(t, bad_pair, at, null_a=False):
    """rows a = 7, b = 1 (each fine for every operation above), with the failing pair at row `at`"""
    z7, one = (7 * 10 ** A.parse_dec(t)[1], 10 ** A.parse_dec(t)[1]) if A.is_dec(t) else (7, 1)
    a, b = [z7] * N, [one] * N
    a[at], b[at] = bad_pair
    if null_a:
        a[at] = None
    tbl = pa.table({"a": A.arrow_array(t, a), "b": A.arrow_array(t, b), "row": pa.array(range(N), pa.int32())})
    return tbl, [P.field("a", A.plan_type(t), True), P.field("b", A.plan_type(t), True), P.field("row", "i32", False)]


@pytest.mark.parametrize("name,t,pair,expr", ERRORS, ids=[e[0] for e in ERRORS])
def test_errors(gpu, name, t, pair, expr):
    for at in (0, N - 1, 2 * 1024 + 77):
        tbl, sch = _error_table(t, pair, at)
        G.register(gpu, "ae", tbl, 1)
        with pytest.raises(engine.B200Error) as ei:
            driver.run_stages(gpu, A.project([("r", expr)], "ae", sch), f"ae-{name}-{at}")
        assert ei.value.code == EXECUTION, (at, str(ei.value))
        # the engine runs the next plan correctly
        tbl, sch = _error_table(t, pair, at, null_a=True)
        G.register(gpu, "ae", tbl, 1)
        out = driver.run_stages(gpu, A.project([("r", expr)], "ae", sch), f"ae-{name}-{at}-next")
        assert out.num_rows == N and out.column("r").null_count >= 1


@pytest.mark.parametrize("name,t,pair,expr", ERRORS, ids=[e[0] for e in ERRORS])
def test_rows_that_must_not_raise(gpu, name, t, pair, expr):
    """the failing pair on a NULL row, on a row a filter dropped, and under a CASE branch that does not select it"""
    at = 2 * 1024 + 77
    tbl, sch = _error_table(t, pair, at, null_a=True)
    G.register(gpu, "ae", tbl, 2)
    out = driver.run_stages(gpu, A.project([("r", expr)], "ae", sch), f"an-{name}-null")
    assert out.column("r")[at].as_py() is None
    tbl, sch = _error_table(t, pair, at)
    G.register(gpu, "ae", tbl, 2)
    not_at = P.binop("<>", c("row"), P.lit_i32(at))
    st = [Q.Stage(1, P.shuffle_writer(P.project([(expr, "r"), (c("row"), "row")], P.filter_(not_at, P.scan("ae", sch))), 1))]
    out = driver.run_stages(gpu, st, f"an-{name}-filter")
    assert out.num_rows == N - 1 and at not in out.column("row").to_pylist()
    for case in (P.case([(not_at, expr)]), P.case([(P.not_(not_at), P.lit_null(_type_of(expr, sch, "ae")))], expr)):
        out = driver.run_stages(gpu, A.project([("r", case)], "ae", sch), f"an-{name}-case")
        assert out.column("r")[at].as_py() is None and out.column("r")[0].as_py() is not None


def _type_of(expr, sch, table):
    st = A.project([("r", expr)], table, sch)[0]
    return json.loads(engine.plan_typed_json(st.json("j")))["input"]["schema"][0]["type"]


@pytest.mark.parametrize("case", A.defect_cases(), ids=[d[0] for d in A.defect_cases()])
def test_defect_cases(gpu, case):
    name, cols, expr, want = case
    assert A.run_defect(gpu, name, cols, expr, want) is None


@pytest.mark.parametrize("frm", A.TYPES)
def test_casts(gpu, frm):
    """every cast between two of the edge types, in the three forms (int -> decimal targets some edge overflows are left to
    the error tests)"""
    vals = A.operands(frm)
    rows = A.rows_of(vals)
    tbl, sch = A.edge_table(frm, vals)
    G.register(gpu, "ar", tbl, 3)
    cases = A.cast_cases(frm, [t for t in A.TYPES if t != frm], rows)
    ulp = 1 if A.is_dec(frm) and A.parse_dec(frm)[1] > 22 else 0  # 10.0**s is exact only up to s = 22
    bad = A.check_projection(gpu, f"ar-cast-{frm}", "ar", sch, rows, cases, ulp=ulp)
    assert not bad, bad
