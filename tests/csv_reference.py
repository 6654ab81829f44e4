"""Reference reader for the CSV scan tests: pyarrow.csv configured to the scan's rules (DESIGN.md §6 (ix)) plus exact Python
arithmetic for floats, and the hand-written expectations of the edge-shape files.  Host only."""
import datetime as dt
import struct
from decimal import Decimal
from fractions import Fraction

import pyarrow as pa
import pyarrow.csv as pacsv

_PA = {"bool": pa.bool_(), "i8": pa.int8(), "i16": pa.int16(), "i32": pa.int32(), "i64": pa.int64(), "u8": pa.uint8(),
       "u16": pa.uint16(), "u32": pa.uint32(), "u64": pa.uint64(), "f32": pa.float32(), "f64": pa.float64(),
       "date32": pa.date32(), "utf8": pa.string()}


def pa_type(t):
    return pa.decimal128(t["dec"][0], t["dec"][1]) if isinstance(t, dict) else _PA[t]


def read(path, schema, delimiter=",", quote='"', escape=None, has_header=False) -> pa.Table:
    """pyarrow.csv with the scan's rules: the schema's names and types, every empty field (quoted or not) NULL."""
    names = [f["name"] for f in schema]
    ro = pacsv.ReadOptions(column_names=names, skip_rows=1 if has_header else 0)
    po = pacsv.ParseOptions(delimiter=delimiter, quote_char=quote, escape_char=escape or False, double_quote=True,
                            newlines_in_values=True, ignore_empty_lines=True)
    co = pacsv.ConvertOptions(column_types={f["name"]: pa_type(f["type"]) for f in schema}, null_values=[""],
                              strings_can_be_null=True, quoted_strings_can_be_null=True)
    return pacsv.read_csv(path, read_options=ro, parse_options=po, convert_options=co)


def write_tbl(table: pa.Table, path: str) -> None:
    """dbgen's .tbl shape: '|'-delimited, no header, no quoting, and an empty last field (a NULL `__placeholder`) that
    leaves the trailing '|' on every line."""
    t = table.append_column("__placeholder", pa.nulls(table.num_rows, pa.string()))
    pacsv.write_csv(t, path, write_options=pacsv.WriteOptions(include_header=False, delimiter="|", quoting_style="none"))


def b64(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def b32(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


def canon_values(col):
    """Column values for exact comparison: floats as their IEEE bits."""
    vals = col.to_pylist()
    if pa.types.is_float64(col.type):
        return [None if v is None else b64(v) for v in vals]
    if pa.types.is_float32(col.type):
        return [None if v is None else b32(v) for v in vals]
    return vals


def is_nan64(b: int) -> bool:
    return (b >> 52) & 0x7FF == 0x7FF and b & ((1 << 52) - 1) != 0


def is_nan32(b: int) -> bool:
    return (b >> 23) & 0xFF == 0xFF and b & ((1 << 23) - 1) != 0


def f64_bits(s: str) -> int:
    """Float64 of a field: Python's float() rounds correctly (nearest, ties to even)."""
    return b64(float(s))


def _special(s: str):
    t = s.strip().lower().lstrip("+-")
    if t in ("inf", "infinity"):
        return "inf"
    if t == "nan":
        return "nan"
    return None


def f32_bits(s: str) -> int:
    """Float32 of a field, rounded once from the exact decimal value (never through a double)."""
    neg = s.strip().startswith("-")
    sign = 0x80000000 if neg else 0
    sp = _special(s)
    if sp == "nan":
        return 0x7FC00000
    if sp == "inf":
        return sign | 0x7F800000
    a = abs(Fraction(s.strip()))
    if a == 0:
        return sign
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    q = max(e, -126) - 23
    n = round(a / Fraction(2) ** q)   # half to even
    if n == 1 << 24:
        n, q = 1 << 23, q + 1
    if q + 23 > 127:
        return sign | 0x7F800000
    if n < 1 << 23:
        return sign | n
    return sign | ((q + 23 + 127) << 23) | (n - (1 << 23))


def fraction_to_decimal(fr: Fraction) -> str:
    """Exact decimal text of a dyadic fraction."""
    num, den = fr.numerator, fr.denominator
    k = den.bit_length() - 1
    assert den == 1 << k
    digits = str(num * 5 ** k)
    if k == 0:
        return digits
    digits = digits.rjust(k + 1, "0")
    return digits[:-k] + "." + digits[-k:]


_D = dt.date
_EDGE = {
    "quoted": {"k": ["a", "b", "c", "d"], "v": ["x,y", "line1\nline2", 'he said "hi"', None]},
    "escaped": {"k": [1, 2, 3], "v": ['a"b', "c\\d", 'e"f']},
    "newlines": {"k": [1, 2], "v": ["a\r\nb", "c\rd"]},
    "crlf_cr_blank": {"k": [1, 2, 3, 4], "v": ["x", "y", "z", "w"]},
    "header_only": {"k": [], "v": []},
    "empty": {"k": [], "v": []},
    "one_column": {"k": [5, 6, 7]},
    "nulls": {"i": [None, 1, None], "f": [None, b64(2.5), None], "g": [None, b32(3.5), None],
              "d": [None, Decimal("1.25"), None], "t": [None, _D(2020, 1, 1), None], "b": [None, True, None],
              "s": [None, "s", None], "q": [None, "x", None]},
    "utf8": {"a": ["é", "😀"], "b": ["日本語", "a,ü"]},
    "ints": {"a": [-128, 127, 1], "b": [255, 0, 2], "c": [-32768, 32767, 3], "d": [65535, 0, 4], "e": [-2147483648, 2147483647, 5],
             "f": [4294967295, 0, 6], "g": [-9223372036854775808, 9223372036854775807, 7], "h": [18446744073709551615, 0, 8]},
    "decimals": {"a": [Decimal("9" * 38), Decimal("-" + "9" * 38), Decimal(0)], "b": [Decimal("-1.5"), Decimal(2), Decimal(0)],
                 "c": [Decimal("0.25"), Decimal("-0.5"), Decimal(0)]},
    "dates": {"d": [_D(1, 1, 1), _D(1970, 1, 1), _D(2000, 2, 29), _D(9999, 12, 31), _D(1969, 12, 31)]},
    "bools": {"b": [True, False, True, False]},
    "tab_delim_quote": {"k": [1, 2], "v": ["a\tb", "c'd"]},
}


def expected_edge(name: str) -> dict:
    return _EDGE[name]
