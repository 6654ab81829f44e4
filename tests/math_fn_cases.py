"""The math functions of DESIGN.md §6 (xviii) restated per row: the float results are glibc's (libm.so.6 through ctypes,
which is what Rust's f64::exp / f32::exp call on Linux), the formulas DataFusion writes in Rust (signum, degrees, radians,
trunc, cot, two-argument log) are spelled out in IEEE arithmetic with x86's NaN rules, and the integer functions use exact
Python ints.  Also: the correctly rounded reference (mpmath at 80 digits), the tabulated ulp bounds, and the edge values.

Floats travel as Python floats.  A Float32 value is held widened to binary64 exactly as the engine holds it (its NaN
payload shifted along), so one bit comparison serves both types."""
import ctypes
import math
import struct

import mpmath
import numpy as np

LIBM = ctypes.CDLL("libm.so.6")

UNARY = ["sqrt", "cbrt", "exp", "ln", "log2", "log10", "sin", "cos", "tan", "asin", "acos", "atan", "sinh", "cosh", "tanh",
         "asinh", "acosh", "atanh", "cot", "degrees", "radians", "signum"]
LIBM_NAME = {"ln": "log"}
TRANSCENDENTAL = ["cbrt", "exp", "ln", "log2", "log10", "sin", "cos", "tan", "asin", "acos", "atan", "sinh", "cosh", "tanh",
                  "asinh", "acosh", "atanh", "cot", "log_base", "power", "atan2"]
# maximum ulp error of CUDA 12.9's library functions (Programming Guide, Mathematical Functions), against the correctly
# rounded result; cot and log_base derived in DESIGN.md §6 (xviii)
ULP_BOUND = {
    "f64": {"cbrt": 1, "exp": 1, "ln": 1, "log2": 1, "log10": 1, "sin": 2, "cos": 2, "tan": 2, "asin": 2, "acos": 2, "atan": 2,
            "sinh": 2, "cosh": 1, "tanh": 1, "asinh": 3, "acosh": 3, "atanh": 2, "power": 2, "atan2": 2, "cot": 5, "log_base": 5},
    "f32": {"cbrt": 1, "exp": 2, "ln": 1, "log2": 1, "log10": 2, "sin": 2, "cos": 2, "tan": 4, "asin": 2, "acos": 2, "atan": 2,
            "sinh": 3, "cosh": 2, "tanh": 2, "asinh": 3, "acosh": 4, "atanh": 3, "atan2": 3, "cot": 9, "log_base": 5},
}
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1


class Overflow(Exception):
    pass


class NegativeExponent(Exception):
    pass


# ---- bits ----------------------------------------------------------------------------------------------------------------
def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def from_bits(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


def f32_to_f64_bits(u):
    """a Float32's bits widened to binary64, NaN payload shifted along (the engine's f32_bits_to_f64_bits)"""
    s, e, m = u >> 31, (u >> 23) & 0xFF, u & 0x7FFFFF
    if e == 0xFF:
        return (s << 63) | (0x7FF << 52) | (m << 29)
    return bits(float(np.frombuffer(struct.pack("<I", u), np.float32)[0]))


def f64_to_f32_bits(u):
    """the inverse for a value that came from a Float32 (or a NaN): mantissa truncated"""
    s, e, m = u >> 63, (u >> 52) & 0x7FF, u & ((1 << 52) - 1)
    if e == 0x7FF:
        return (s << 31) | (0xFF << 23) | (m >> 29)
    return struct.unpack("<I", struct.pack("<f", from_bits(u)))[0]


def f32(u32):
    """a Float32 given by its bits, as the engine holds it"""
    return from_bits(f32_to_f64_bits(u32))


def to_f32(x):
    """round a binary64 to Float32 (round to nearest) and hold it widened"""
    if x != x:
        return from_bits(f32_to_f64_bits(f64_to_f32_bits(bits(x))))
    return float(np.float32(x))


def quiet(x):
    return from_bits(bits(x) | 0x0008000000000000)


def isnan(x):
    return x != x


X86_NAN = from_bits(0xFFF8000000000000)   # x86 SSE's default NaN
RUST_NAN = from_bits(0x7FF8000000000000)  # f64::NAN (and f32::NAN widened)


def same_bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    return bits(a) == bits(b)


# ---- libm ------------------------------------------------------------------------------------------------------------------
def _libm(name, f32_, nargs):
    fn = getattr(LIBM, name + ("f" if f32_ else ""))
    t = ctypes.c_float if f32_ else ctypes.c_double
    fn.restype, fn.argtypes = t, [t] * nargs
    return fn


_FN = {}


def libm(name, is32, *args):
    """glibc's name(args) (name + 'f' in f32); a NaN argument or result keeps its bits across ctypes (quiet NaNs only: a
    signalling one is quieted on the way, as the call itself would)"""
    key = (name, is32, len(args))
    if key not in _FN:
        _FN[key] = _libm(name, is32, len(args))
    if not is32:
        return _FN[key](*args)
    # a Float32 NaN crosses ctypes as a double -> float conversion, which keeps a quiet NaN's payload
    r = _FN[key](*[from_bits(f32_to_f64_bits(f64_to_f32_bits(bits(a)))) if a != a else a for a in args])
    return to_f32(r)


def _mul(x, c, is32):
    if is32:
        return float(np.float32(x) * np.float32(c))
    return x * c


def _div(a, b, is32):
    """x86 divsd / divss: a NaN dividend quieted, else a NaN divisor quieted, else the quotient (0/0 etc: default NaN)"""
    if isnan(a):
        return quiet(a)
    if isnan(b):
        return quiet(b)
    if is32:
        with np.errstate(all="ignore"):
            q = float(np.float32(a) / np.float32(b))
    else:
        if b == 0:
            q = X86_NAN if a == 0 else math.copysign(math.inf, a) * math.copysign(1.0, b)
        elif math.isinf(a) and math.isinf(b):
            q = X86_NAN
        else:
            q = a / b
    return X86_NAN if isnan(q) else q


DEG = {False: 180.0 / math.pi, True: f32(0x42652EE1)}          # Rust's to_degrees factors
RAD = {False: math.pi / 180.0, True: f32(0x3C8EFA35)}          # and to_radians: (PI as f32) / 180.0f32 in f32


# ---- per-row rules ---------------------------------------------------------------------------------------------------------
def unary(name, x, is32=False):
    if x is None:
        return None
    if name == "isnan":
        return isnan(x)
    if name == "iszero":
        return x == 0.0
    if name == "signum":
        if isnan(x):
            return RUST_NAN
        return 0.0 if x == 0.0 else math.copysign(1.0, x)
    if name in ("degrees", "radians"):
        if isnan(x):
            return quiet(x)
        return _mul(x, (DEG if name == "degrees" else RAD)[is32], is32)
    if name == "cot":
        return _div(1.0, libm("tan", is32, x), is32)
    if name == "log":
        name = "log10"
    return libm(LIBM_NAME.get(name, name), is32, x)


def log_base(base, x, is32=False):
    """Rust's x.log(base) = x.ln() / base.ln()"""
    if base is None or x is None:
        return None
    return _div(libm("log", is32, x), libm("log", is32, base), is32)


def atan2(y, x, is32=False):
    if y is None or x is None:
        return None
    return libm("atan2", is32, y, x)


def power(x, y):
    if x is None or y is None:
        return None
    if isinstance(x, int):
        if y < 0 or y > 0xFFFFFFFF:
            raise NegativeExponent(y)
        if x in (0, 1) or y == 0:
            return 1 if y == 0 or x == 1 else 0
        if x == -1:
            return -1 if y & 1 else 1
        if y > 64:
            raise Overflow(x)
        r = x ** y
        if not INT64_MIN <= r <= INT64_MAX:
            raise Overflow(x)
        return r
    return libm("pow", False, x, y)


def nanvl(x, y):
    if x is None or y is None:
        return None
    return y if isnan(x) else x


def trunc(x, n=0, is32=False):
    """DataFusion: (x * f).trunc() / f with round's f = 10^n (1 / 10^-n for n < 0), each step rounded once"""
    if x is None or n is None:
        return None
    if isnan(x):
        return quiet(x)
    p = float(10 ** abs(n))
    if is32:
        f = float(np.float32(p)) if n >= 0 else float(np.float32(1.0) / np.float32(p))
        with np.errstate(all="ignore"):
            y = np.float32(x) * np.float32(f)
            t = np.trunc(y)
            return float(t / np.float32(f))
    f = p if n >= 0 else 1.0 / p
    y = x * f
    t = y if math.isinf(y) else math.copysign(float(math.trunc(y)), y)
    return t / f


def gcd(a, b):
    if a is None or b is None:
        return None
    r = math.gcd(a, b)
    if r > INT64_MAX:
        raise Overflow((a, b))
    return r


def lcm(a, b):
    if a is None or b is None:
        return None
    if a == 0 or b == 0:
        return 0
    r = abs(a) // math.gcd(a, b) * abs(b)
    if r > INT64_MAX:
        raise Overflow((a, b))
    return r


def factorial(n):
    if n is None:
        return None
    if n > 20:
        raise Overflow(n)
    return math.factorial(n) if n >= 2 else 1


# ---- the correctly rounded reference -------------------------------------------------------------------------------------
mpmath.mp.dps = 80
_MP = {"cbrt": lambda v: mpmath.sign(v) * mpmath.cbrt(abs(v)), "exp": mpmath.exp, "ln": mpmath.ln, "log2": lambda v: mpmath.log(v, 2), "log10": mpmath.log10,
       "sin": mpmath.sin, "cos": mpmath.cos, "tan": mpmath.tan, "asin": mpmath.asin, "acos": mpmath.acos, "atan": mpmath.atan,
       "sinh": mpmath.sinh, "cosh": mpmath.cosh, "tanh": mpmath.tanh, "asinh": mpmath.asinh, "acosh": mpmath.acosh,
       "atanh": mpmath.atanh, "cot": mpmath.cot}


def exact(name, *args):
    """the exact value (80 digits) of a transcendental function at finite arguments inside its domain"""
    a = [mpmath.mpf(v) for v in args]
    if name == "log_base":
        return mpmath.ln(a[1]) / mpmath.ln(a[0])
    if name == "atan2":
        return mpmath.atan2(a[0], a[1])
    if name == "power":
        return mpmath.power(a[0], a[1])
    return _MP[name](a[0])


def ulp_error(got, ref, is32):
    """|got - ref| in units of the last place at ref (subnormal spacing below the normal range)"""
    p, emin = (24, -126) if is32 else (53, -1022)
    if ref == 0:
        e = emin
    else:
        e = max(int(mpmath.floor(mpmath.log(abs(ref), 2))), emin)
        if mpmath.mpf(2) ** e > abs(ref):  # log2 rounding at an exact power of two
            e = max(e - 1, emin)
        if mpmath.mpf(2) ** (e + 1) <= abs(ref):
            e += 1
    return float(abs(mpmath.mpf(got) - ref) / mpmath.mpf(2) ** (e - p + 1))


def special(x_args, result):
    """rows the exact rule covers: a non-finite or zero argument, or a non-finite or zero result"""
    return any(not math.isfinite(v) or v == 0.0 for v in x_args) or not math.isfinite(result) or result == 0.0


# ---- edge values -------------------------------------------------------------------------------------------------------------
NAN_BITS64 = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000000000123, 0xFFF80000DEADBEEF, 0x7FF0000000000005]
NAN_BITS32 = [0x7FC00000, 0xFFC00000, 0x7FC00123, 0xFFC0BEEF, 0x7F800005]
EDGE64 = ([0.0, -0.0, math.inf, -math.inf, 5e-324, -5e-324, 2.2250738585072014e-308, -1e-310, 1.0, -1.0, 0.5, -0.5, 2.0, -2.0,
           1e22, -1e22, 2.0 ** 1000, -(2.0 ** 1000), 1e300, -1e300, 709.782712893384, 709.7827128933841, 710.0, -708.3964185322641,
           -745.1332191019411, -745.1332191019412, -746.0, math.pi, math.pi / 2, -math.pi / 4, 1e-300, 0.9999999999999999,
           1.0000000000000002, 3.0, 100.0, -100.0, 1e-8, 1.7976931348623157e308, -1.7976931348623157e308, 0.1, 123.456]
          + [from_bits(u) for u in NAN_BITS64])
EDGE32 = [to_f32(v) for v in (0.0, -0.0, math.inf, -math.inf, 1e-45, -1e-45, 1e-40, 1.1754943508222875e-38, 1.0, -1.0, 0.5, -0.5,
                              2.0, -2.0, 1e22, -1e22, 2.0 ** 100, -(2.0 ** 100), 3.4028234663852886e38, -3.4028234663852886e38,
                              88.72283, 88.72284, 89.0, -87.33654, -103.97208, -103.97209, -105.0, math.pi, math.pi / 2, 0.1,
                              0.99999994, 1.0000001, 3.0, 100.0, -100.0, 1e-8, 123.456)] + [f32(u) for u in NAN_BITS32]
INT_EDGE = [0, 1, -1, 2, -2, 3, 7, -12, 20, 21, 62, 63, 64, 2**31, -2**31, 2**32, 3037000499, 3037000500, 2**62, -2**62,
            INT64_MAX, INT64_MIN + 1, INT64_MIN, 6, 10, 1000000007]


def sample(name, n, is32, seed):
    """n arguments, log-uniform magnitudes over the function's useful range, both signs"""
    lo, hi = {"exp": (-6, 2.85), "sinh": (-6, 2.85), "cosh": (-6, 2.85), "asin": (-12, 0), "acos": (-12, 0),
              "atanh": (-12, 0), "acosh": (0, 30), "tanh": (-8, 1.5)}.get(name, (-30, 30))
    if is32 and name in ("exp", "sinh", "cosh"):
        hi = 1.9
    rng = np.random.default_rng(seed)
    mags = 10.0 ** rng.uniform(lo, hi, n)
    signs = np.where(rng.integers(0, 2, n) == 1, 1.0, -1.0)
    vals = [float(m * s) for m, s in zip(mags, signs)]
    if name == "acosh":
        vals = [abs(v) + 1.0 for v in vals]
    return [to_f32(v) for v in vals] if is32 else vals
