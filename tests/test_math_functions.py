"""Math functions (DESIGN.md §6 (xviii)) on the host: result types and nullability, the refusals (each naming its function and
type), the protobuf fixtures decoding to the plans they were generated from, the CPU oracle's refusal, and the restatement
in math_fn_cases.py pinned against libm (NaN bits and special values) and mpmath (libm within 3 ulp on a sample)."""
import base64
import json
import math
import os

import mpmath
import pytest

import golden_data as G
import math_fn_cases as M
import queries as Q
from ballista_b200 import driver, engine
from ballista_b200 import plan as P

c = P.col
UNSUPPORTED = -2  # B200_ERR_UNSUPPORTED (include/b200exec.h)
HERE = os.path.dirname(os.path.abspath(__file__))
SCHEMA = [P.field("a", "f64", False), P.field("an", "f64", True), P.field("b", "f32", False), P.field("bn", "f32", True),
          P.field("i", "i64", False), P.field("iz", "i64", True), P.field("i32", "i32", True), P.field("dec", P.dec(15, 2), True),
          P.field("s", "utf8", True)]


def _typed(e):
    st = Q.Stage(1, P.shuffle_writer(P.project([(e, "r")], P.scan("x", SCHEMA)), 1))
    return json.loads(engine.plan_typed_json(st.json("j")))["input"]["schema"][0]


# ---- result types -----------------------------------------------------------------------------------------------------------
def _type_cases():
    out = []
    for name in M.UNARY + ["log"]:
        out += [(P.fn(name, c("a")), "f64", False), (P.fn(name, c("an")), "f64", True), (P.fn(name, c("b")), "f32", False),
                (P.fn(name, c("bn")), "f32", True)]
    for name in ("isnan", "iszero"):
        out += [(P.fn(name, c("a")), "bool", False), (P.fn(name, c("bn")), "bool", True)]
    for name in ("log", "atan2", "nanvl"):
        out += [(P.fn(name, c("a"), c("an")), "f64", True), (P.fn(name, c("b"), c("b")), "f32", False)]
    out += [(P.fn("power", c("a"), c("a")), "f64", False), (P.fn("power", c("i"), c("iz")), "i64", True),
            (P.fn("trunc", c("a")), "f64", False), (P.fn("trunc", c("bn"), P.lit_i64(2)), "f32", True),
            (P.fn("trunc", c("b"), P.lit_i64(-22)), "f32", False),
            (P.fn("gcd", c("i"), c("i")), "i64", False), (P.fn("lcm", c("iz"), c("i")), "i64", True),
            (P.fn("factorial", c("i")), "i64", False), (P.fn("factorial", c("iz")), "i64", True), (P.fn("pi"), "f64", False)]
    return out


TYPE_CASES = _type_cases()


@pytest.mark.parametrize("i", range(len(TYPE_CASES)))
def test_result_types(i):
    e, typ, nullable = TYPE_CASES[i]
    f = _typed(e)
    assert (f["type"], f["nullable"]) == (typ, nullable), e


# ---- refusals ---------------------------------------------------------------------------------------------------------------
REFUSALS = [(P.fn(n, c(col)), n, t) for n in ("sqrt", "ln", "cot", "signum", "isnan", "log", "exp") for col, t in
            (("dec", "dec(15,2)"), ("i32", "i32"), ("i", "i64"), ("s", "utf8"))]
REFUSALS += [
    (P.fn("power", c("b"), c("b")), "power", "f32"), (P.fn("power", c("a"), c("i")), "power", "i64"),
    (P.fn("power", c("i32"), c("i32")), "power", "i32"), (P.fn("power", c("dec"), c("i")), "power", "dec(15,2)"),
    (P.fn("atan2", c("a"), c("b")), "atan2", "f32"), (P.fn("nanvl", c("s"), c("a")), "nanvl", "utf8"),
    (P.fn("log", c("b"), c("a")), "log", "f64"), (P.fn("gcd", c("i"), c("i32")), "gcd", "i32"),
    (P.fn("lcm", c("a"), c("i")), "lcm", "f64"), (P.fn("factorial", c("dec")), "factorial", "dec(15,2)"),
    (P.fn("trunc", c("dec")), "trunc", "dec(15,2)"), (P.fn("trunc", c("i32")), "trunc", "i32"),
    (P.fn("trunc", c("a"), P.lit_i64(23)), "trunc", "23"), (P.fn("trunc", c("b"), P.lit_i64(-40)), "trunc", "-40"),
]


@pytest.mark.parametrize("e,fn,culprit", REFUSALS, ids=[f"{f}-{t}" for _, f, t in REFUSALS])
def test_refusals_name_the_function_and_type(e, fn, culprit):
    with pytest.raises(engine.B200Error) as ei:
        _typed(e)
    assert ei.value.code == UNSUPPORTED and fn in str(ei.value) and culprit in str(ei.value), str(ei.value)


@pytest.mark.parametrize("e", [P.fn("sqrt"), P.fn("sqrt", c("a"), c("a")), P.fn("atan2", c("a")), P.fn("pi", c("a")),
                               P.fn("log", c("a"), c("a"), c("a")), P.fn("trunc", c("a"), P.lit_i64(1), P.lit_i64(1))])
def test_wrong_argument_counts_are_malformed(e):
    with pytest.raises(engine.B200Error) as ei:
        _typed(e)
    assert "argument" in str(ei.value), str(ei.value)


# ---- protobuf fixtures ------------------------------------------------------------------------------------------------------
with open(os.path.join(HERE, "golden", "math_fn_proto_plans.json")) as _fh:
    PROTO_CASES = json.load(_fh)["cases"]


def _fns(node, out):
    if isinstance(node, dict):
        if "fn" in node and "args" in node and "type" in node:
            out.append((node["fn"], json.dumps(node["type"])))
        for v in node.values():
            _fns(v, out)
    elif isinstance(node, list):
        for v in node:
            _fns(v, out)
    return out


def test_fixtures_cover_every_name_and_alias():
    spelled = {x["spelled"].lower() for x in PROTO_CASES if not x["refused"]}
    assert set(M.UNARY) | {"log", "atan2", "nanvl", "power", "pow", "trunc", "gcd", "lcm", "factorial", "isnan", "iszero", "pi"} <= spelled
    shapes = {x["name"].split("/")[1] for x in PROTO_CASES if not x["refused"]}
    assert shapes == {"projection", "filter", "group_key_and_argument"}
    assert {x["refused"] for x in PROTO_CASES if x["refused"]} >= {"random", "dec(15,2)", "utf8", "i32", "literal"}


@pytest.mark.parametrize("case", [x for x in PROTO_CASES if not x["refused"]], ids=lambda x: x["name"])
def test_protobuf_plans_decode_to_the_same_typed_plan(case):
    decoded = engine.plan_typed_json(engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]), "job"))
    want = engine.plan_typed_json(case["ir"])
    assert _fns(json.loads(decoded), []) == _fns(json.loads(want), [])
    assert json.loads(decoded)["input"]["schema"] == json.loads(want)["input"]["schema"]


@pytest.mark.parametrize("case", [x for x in PROTO_CASES if x["refused"] not in (None, "literal")], ids=lambda x: x["name"])
def test_protobuf_refusals(case):
    """random stays unknown to the decoder; the others decode and are refused when typed (a non-literal trunc digit count
    types, and is refused when the stage is lowered: test_gpu_math_functions.py)"""
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]), "job"))
    assert ei.value.code == UNSUPPORTED and case["refused"] in str(ei.value).lower(), str(ei.value)


# ---- the CPU oracle ---------------------------------------------------------------------------------------------------------
def test_cpu_oracle_refuses_every_math_function(oracle):
    import pyarrow as pa
    from oracle_ffi import OracleError
    t = pa.table({"a": pa.array([1.0, 2.0], pa.float64()), "i": pa.array([3, 4], pa.int64())})
    G.register(oracle, "m", t, 1)
    sch = [P.field("a", "f64", False), P.field("i", "i64", False)]
    calls = [P.fn(n, c("a")) for n in M.UNARY + ["log", "isnan", "iszero", "trunc"]]
    calls += [P.fn(n, c("a"), c("a")) for n in ("log", "atan2", "nanvl", "power")]
    calls += [P.fn(n, c("i"), c("i")) for n in ("gcd", "lcm", "power")] + [P.fn("factorial", c("i")), P.fn("pi")]
    for k, e in enumerate(calls):
        st = [Q.Stage(1, P.shuffle_writer(P.project([(e, "r")], P.scan("m", sch)), 1))]
        with pytest.raises(OracleError) as ei:
            driver.run_stages(oracle, st, f"o-math-{k}")
        assert "scalar function" in str(ei.value), str(ei.value)


# ---- the restatement against libm and mpmath --------------------------------------------------------------------------------
def test_nan_rules_equal_libm():
    """a NaN argument comes back with its own bits, quieted; a NaN a function makes has the sign glibc gives it"""
    for name in ["sqrt", "cbrt", "exp", "ln", "log2", "log10", "sin", "cos", "tan", "asin", "acos", "atan", "sinh", "cosh",
                 "tanh", "asinh", "acosh", "atanh"]:
        for u in M.NAN_BITS64:
            assert M.bits(M.unary(name, M.from_bits(u))) == u | 0x0008000000000000, (name, hex(u))
        for u in M.NAN_BITS32:
            got = M.f64_to_f32_bits(M.bits(M.unary(name, M.f32(u), True)))
            assert got == u | 0x00400000, (name, hex(u))
    neg, pos = M.bits(M.X86_NAN), M.bits(M.RUST_NAN)
    for name, x, want in (("sqrt", -1.0, neg), ("ln", -1.0, neg), ("log2", -1.0, neg), ("log10", -1.0, pos), ("sin", math.inf, neg),
                          ("cos", -math.inf, neg), ("tan", math.inf, neg), ("asin", 2.0, pos), ("acos", 2.0, pos),
                          ("acos", -math.inf, pos), ("acosh", 0.5, neg), ("atanh", 2.0, neg), ("cot", math.inf, neg)):
        assert M.bits(M.unary(name, x)) == want, name
        assert M.bits(M.unary(name, M.to_f32(x), True)) == want, name + "f"
    assert M.bits(M.power(-2.0, 0.5)) == neg
    assert M.bits(M.unary("signum", M.from_bits(0xFFF8000000000123))) == pos
    assert M.bits(M.log_base(1.0, 1.0)) == neg                   # 0 / 0 in divsd
    # two NaNs: pow and log return the first operand's, atan2(y, x) x's
    a, b = M.from_bits(0x7FF8000000000001), M.from_bits(0xFFF8000000000123)
    assert M.bits(M.power(a, b)) == M.bits(a) and M.bits(M.atan2(a, b)) == M.bits(b) and M.bits(M.atan2(a, 1.0)) == M.bits(a)
    assert M.power(a, 0.0) == 1.0 and M.power(1.0, b) == 1.0 and M.power(-1.0, math.inf) == 1.0
    snan = M.from_bits(0x7FF0000000000005)   # glibc: a signalling NaN is not caught by pow(x, 0) = 1 or pow(1, y) = 1
    assert M.bits(M.power(snan, 0.0)) == M.bits(M.power(1.0, snan)) == 0x7FF8000000000005
    for y in (1.0, 3.0, -1.0):                # a NaN x to an odd integer power loses its sign; to another keeps it
        assert M.bits(M.power(b, y)) == M.bits(b) & ~(1 << 63), y
    for y in (2.0, 0.5, -2.0):
        assert M.bits(M.power(b, y)) == M.bits(b), y
    assert M.bits(M.nanvl(a, b)) == M.bits(b) and M.nanvl(1.0, b) == 1.0


def test_special_values_equal_libm():
    cases = [("ln", 0.0, -math.inf), ("ln", -0.0, -math.inf), ("sqrt", -0.0, -0.0), ("acosh", 1.0, 0.0), ("atanh", 1.0, math.inf),
             ("atanh", -1.0, -math.inf), ("exp", 710.0, math.inf), ("exp", -746.0, 0.0), ("exp", -math.inf, 0.0),
             ("tanh", -math.inf, -1.0), ("sin", -0.0, -0.0), ("cot", -0.0, -math.inf), ("signum", -0.0, 0.0),
             ("degrees", -0.0, -0.0), ("cbrt", -math.inf, -math.inf), ("log10", 1.0, 0.0)]
    for name, x, want in cases:
        for is32 in (False, True):
            got = M.unary(name, M.to_f32(x) if is32 else x, is32)
            assert M.bits(got) == M.bits(want), (name, x, is32)
    assert M.trunc(-0.25, 0) == 0.0 and math.copysign(1, M.trunc(-0.25)) < 0 and M.trunc(1e300, 22) == math.inf
    assert M.trunc(1.239, 2) == 1.23 and M.trunc(-1234.5, -2) == -1200.0


def test_integer_rules():
    assert M.gcd(0, 0) == 0 and M.gcd(-12, 18) == 6 and M.gcd(M.INT64_MIN, 3) == 1
    for a, b in ((M.INT64_MIN, 0), (M.INT64_MIN, M.INT64_MIN)):
        with pytest.raises(M.Overflow):
            M.gcd(a, b)
    assert M.lcm(0, M.INT64_MIN) == 0 and M.lcm(-4, 6) == 12
    with pytest.raises(M.Overflow):
        M.lcm(M.INT64_MIN, 1)
    with pytest.raises(M.Overflow):
        M.lcm(3037000500, 3037000501)
    assert M.factorial(-5) == 1 and M.factorial(20) == 2432902008176640000
    with pytest.raises(M.Overflow):
        M.factorial(21)
    assert M.power(-2, 63) == M.INT64_MIN and M.power(0, 0) == 1 and M.power(-1, 2**32 - 1) == -1
    with pytest.raises(M.Overflow):
        M.power(2, 63)
    with pytest.raises(M.NegativeExponent):
        M.power(2, -1)


def test_libm_is_within_three_ulp_of_mpmath():
    """the reference is sound: glibc is within 3 ulp of the exact value on the sample (under 1 for most functions; glibc's
    own tables allow cbrt, sinh, tanh and atanh more)"""
    worst = 0.0
    for k, name in enumerate(["cbrt", "exp", "ln", "log2", "log10", "sin", "cos", "tan", "asin", "acos", "atan", "sinh", "cosh",
                              "tanh", "asinh", "acosh", "atanh"]):
        for is32 in (False, True):
            for x in M.sample(name, 200, is32, 100 + k):
                got = M.unary(name, x, is32)
                if M.special([x], got):
                    continue
                worst = max(worst, M.ulp_error(got, M.exact(name, x), is32))
    assert worst <= 3.0, worst
