"""The arithmetic core on the host: the per-row restatement in arith_cases.py pinned against independent computations
(Python's decimal at 80 digits, pyarrow.compute's checked kernels and safe casts, struct bit patterns), then the CPU
oracle -- the checker of the rest of the suite -- against the restatement on the operator matrix, the comparisons, the
casts, CASE and each defect the restatement was written for."""
import math
import struct
from decimal import ROUND_DOWN, ROUND_HALF_UP, Context, Decimal, localcontext
from fractions import Fraction

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import arith_cases as A
import golden_data as G
from ballista_b200 import plan as P

c = P.col


# ---- the restatement against independent computations ---------------------------------------------------------------------
@pytest.mark.parametrize("t", list(A.INTS))
def test_integer_ops_against_pyarrow_checked_kernels(t):
    """+ - * agree with pyarrow's wrapping kernels, / with its checked kernel (errors included), % with Python's math"""
    vals = A.operands(t)
    a, b = vals["a_nn"][:400], vals["b_nn"][:400]
    pa_a, pa_b = pa.array(a, A.arrow_type(t)), pa.array(b, A.arrow_type(t))
    for op, fn in (("+", pc.add), ("-", pc.subtract), ("*", pc.multiply)):
        assert fn(pa_a, pa_b).to_pylist() == [A.arith(op, x, y, t) for x, y in zip(a, b)], op
    for x, y in zip(a, b):
        try:
            want = pc.divide_checked(pa.scalar(x, A.arrow_type(t)), pa.scalar(y, A.arrow_type(t))).as_py()
        except (pa.ArrowInvalid, ZeroDivisionError):
            want = A.Raise
        try:
            got = A.arith("/", x, y, t)
        except A.Raise:
            got = A.Raise
        assert got == want, (x, y)
        if y != 0:
            with localcontext(A.CTX):
                assert A.arith("%", x, y, t) == int(Decimal(x) % Decimal(y))  # Decimal's % takes the dividend's sign
    lo, _ = A.int_range(t)
    if lo < 0:
        assert A.arith("%", lo, -1, t) == 0  # [EXT]: both engines give 0 where arrow's mod_checked may raise


@pytest.mark.parametrize("t", list(A.FLOATS))
def test_float_ops_against_struct_and_pyarrow(t):
    vals = A.edges(t)
    pa_t = A.arrow_type(t)
    for x in vals:
        for y in vals:
            for op, fn in (("+", pc.add), ("-", pc.subtract), ("*", pc.multiply), ("/", pc.divide)):
                want = fn(pa.scalar(x, pa_t), pa.scalar(y, pa_t)).as_py()
                assert A.same(A.arith(op, x, y, t), want), (op, x, y)
            r = A.arith("%", x, y, t)
            if math.isfinite(x) and math.isfinite(y) and y != 0:
                assert Fraction(r) == Fraction(x) - Fraction(y) * math.trunc(Fraction(x) / Fraction(y))  # fmod is exact
    # negation flips the sign bit of every value, NaNs included
    for bits in A.NAN_BITS + (0, 1 << 63, 0x7FF0000000000000):
        x = A.f64_from_bits(bits)
        assert struct.unpack("<Q", struct.pack("<d", A.neg(x, "f64")))[0] == bits ^ (1 << 63)


def test_total_order_of_floats():
    ordered = [A.f64_from_bits(0xFFF8000000000000), -math.inf, -1.0, -5e-324, -0.0, 0.0, 5e-324, 1.0, math.inf,
               A.f64_from_bits(0x7FF0000000000123), A.f64_from_bits(0x7FF8000000000000)]
    for i, x in enumerate(ordered):
        for j, y in enumerate(ordered):
            assert A.compare("<", x, y, "f64") == (i < j) and A.compare("=", x, y, "f64") == (i == j), (x, y)


@pytest.mark.parametrize("p,s", A.DECS)
def test_decimal_ops_against_python_decimal(p, s):
    """every pair of edges of one Decimal128 type: the unscaled result, and the result type from arrow's rules, against
    Python's decimal at 80 digits"""
    t = A.dec_name(p, s)
    e = A.edges(t)
    ctx = Context(prec=80)
    for op in A.OPS:
        rp, rs = A.dec_result(op, (p, s), (p, s))
        assert rp <= 38 and rs <= 38
        for x in e:
            for y in e:
                dx, dy = Decimal(x).scaleb(-s, ctx), Decimal(y).scaleb(-s, ctx)
                with localcontext(ctx):
                    if op in "+-*":
                        exact = dx + dy if op == "+" else dx - dy if op == "-" else dx * dy
                    elif dy == 0:
                        exact = None
                    elif op == "/":
                        exact = (dx / dy).quantize(Decimal(1).scaleb(-rs), rounding=ROUND_DOWN)
                    else:
                        exact = dx % dy  # Python's Decimal % takes the dividend's sign
                    want = None if exact is None else int(exact.scaleb(rs))
                if want is None:
                    with pytest.raises(A.Raise):
                        A.arith(op, x, y, t)
                    continue
                if not A.I128_MIN <= want <= A.I128_MAX:
                    with pytest.raises(A.Raise):
                        A.arith(op, x, y, t)
                    continue
                try:
                    got = A.arith(op, x, y, t)
                except A.Raise:
                    # only an intermediate (a rescaled operand or the scaled dividend) may overflow where the result fits
                    assert op in "/%" or (op in "+-" and rs > s), (op, x, y)
                    continue
                assert got == want, (op, x, y)


def test_casts_against_pyarrow_safe_casts():
    """int <-> int, int -> float, float -> int and decimal -> decimal against pyarrow.compute.cast (safe=True gives an error
    where the engine gives NULL: each value is cast on its own)"""
    def pa_cast(v, frm, to):
        try:
            return pc.cast(pa.array([v], A.arrow_type(frm)), A.arrow_type(to), safe=True)[0].as_py()
        except pa.ArrowInvalid:
            return None

    for frm in A.INTS:
        for to in list(A.INTS) + ["f64"]:
            for v in A.edges(frm):
                if to == "f64" and abs(v) > 2 ** 53:
                    continue  # pyarrow's safe cast refuses an integer a double may not hold exactly
                assert A.cast(v, frm, to) == pa_cast(v, frm, to), (frm, to, v)
    for frm in A.FLOATS:
        for to in A.INTS:
            for v in A.edges(frm):
                want = None if not math.isfinite(v) else pa_cast(float(math.trunc(v)), frm, to)
                assert A.cast(v, frm, to) == want, (frm, to, v)
    for (p1, s1) in A.DECS:
        for (p2, s2) in A.DECS:
            if s2 < s1:
                continue  # pyarrow truncates when it scales down; the engine rounds half away (checked below)
            for v in A.edges(A.dec_name(p1, s1)):
                d = Decimal(v).scaleb(-s1, A.CTX)
                want = pa_cast(d, A.dec_name(p1, s1), A.dec_name(p2, s2))
                want = None if want is None else int(want.scaleb(s2, A.CTX))
                try:
                    got = A.cast(v, A.dec_name(p1, s1), A.dec_name(p2, s2))
                except A.Raise:
                    got = None
                assert got == want, ((p1, s1), (p2, s2), v)


def test_cast_rounding_rules():
    # decimal down-scaling rounds half away from zero (Python's round would give 2 and -2)
    assert A.cast(250, "d5_2", "d5_0") == 3 and A.cast(-250, "d5_2", "d5_0") == -3 and A.cast(249, "d5_2", "d5_0") == 2
    for v in (12345, -12345, 5, -5, 99999):
        want = int(Decimal(v).scaleb(-2).quantize(Decimal(1), rounding=ROUND_HALF_UP))
        assert A.cast(v, "d5_2", "d5_0") == want
    # float -> decimal rounds the double x * 10**s half away from zero
    assert A.cast(2.5, "f64", "d5_0") == 3 and A.cast(-0.5, "f64", "d5_0") == -1 and A.cast(0.125, "f64", "d5_2") == 13
    assert A.cast(1e10, "f64", "d5_2") is None and A.cast(999.994, "f64", "d5_2") == 99999
    # int -> Float32 once from the integer: 2^62 + 2^38 + 1 is above the halfway point 2^62 + 2^38 between two binary32
    # neighbours, so it rounds up; through a double (2^62 + 2^38, a tie) it would round to even, down to 2^62
    big = (1 << 62) + (1 << 38) + 1
    assert A.int_to_f32(big) == float((1 << 62) + (1 << 39))
    assert A.to_f32(float(big)) == float(1 << 62)
    rng = np.random.default_rng(5)
    for v in [int(x) for x in rng.integers(-(1 << 63), (1 << 63) - 1, 2000, dtype=np.int64)] + list(range(-70000, 70000, 999)):
        f = A.int_to_f32(v)
        assert f == float(np.float32(f)), v  # a binary32 value
        up = np.nextafter(np.float32(f), np.float32(math.inf))
        dn = np.nextafter(np.float32(f), np.float32(-math.inf))
        assert abs(Fraction(f) - v) <= min(abs(Fraction(float(up)) - v), abs(Fraction(float(dn)) - v)), v
    # int -> decimal beyond the precision is an error, not NULL
    with pytest.raises(A.Raise):
        A.cast(100000, "i32", "d5_0")


def test_case_restatement_is_lazy():
    f = A.case_rows([lambda r: r["b"] != 0], [lambda r: A.arith("/", r["l"], r["b"], "i64")])
    assert [f({"l": 10, "b": b}) for b in (2, 0)] == [5, None]


# ---- the oracle against the restatement -----------------------------------------------------------------------------------
@pytest.mark.parametrize("t", A.TYPES)
def test_oracle_operator_matrix(oracle, t):
    for op in A.OPS:
        vals = A.safe_operands(op, t)
        tbl, sch = A.edge_table(t, vals)
        G.register(oracle, "ar", tbl, 1)
        cases = [s for form in A.FORMS for s in A.shapes(op, t, form)]
        bad = A.check_projection(oracle, f"ar-{t}-{op}", "ar", sch, A.rows_of(vals), cases)
        assert not bad, (op, bad)


@pytest.mark.parametrize("t", A.TYPES)
def test_oracle_comparisons_and_negation(oracle, t):
    vals = A.operands(t)
    tbl, sch = A.edge_table(t, vals)
    G.register(oracle, "ar", tbl, 1)
    cases = []
    for form in A.FORMS:
        for op in A.CMPS:
            cases.append((f"{op}_{form}", P.binop(op, c(f"a_{form}"), c(f"b_{form}")),
                          lambda r, op=op, form=form: A.compare(op, r[f"a_{form}"], r[f"b_{form}"], t), "bool"))
        if t in A.INTS and not A.INTS[t][1]:
            continue  # DataFusion refuses the negation of an unsigned integer
        cases.append((f"neg_{form}", P.neg(c(f"a_{form}")), lambda r, form=form: A.neg(r[f"a_{form}"], t), t))
    bad = A.check_projection(oracle, "ar-cmp", "ar", sch, A.rows_of(vals), cases)
    assert not bad, bad


@pytest.mark.parametrize("frm", A.TYPES)
def test_oracle_casts(oracle, frm):
    vals = A.operands(frm)
    rows = A.rows_of(vals)
    tbl, sch = A.edge_table(frm, vals)
    G.register(oracle, "ar", tbl, 1)
    cases = A.cast_cases(frm, [t for t in A.TYPES if t != frm], rows)
    assert cases
    # 10.0**s is exact only up to s = 22: DataFusion's 10_f64.powi(s) may differ from the nearest double by an ulp above
    ulp = 1 if A.is_dec(frm) and A.parse_dec(frm)[1] > 22 else 0
    bad = A.check_projection(oracle, f"ar-cast-{frm}", "ar", sch, rows, cases, ulp=ulp)
    assert not bad, bad


@pytest.mark.parametrize("case", A.defect_cases(), ids=[d[0] for d in A.defect_cases()])
def test_oracle_defect_cases(oracle, case):
    name, cols, expr, want = case
    assert A.run_defect(oracle, name, cols, expr, want) is None
