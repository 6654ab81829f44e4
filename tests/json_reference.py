"""Reference reader for the newline-delimited JSON scan tests (DESIGN.md §6 (xv)): Python's json module with duplicate keys
kept (object_pairs_hook), NaN / Infinity refused (parse_constant) and numbers kept as their text, then converted with exact
arithmetic; the scan's stricter line and token rules are applied on top.  Host only.

read() returns {column: [values]} (floats as their IEEE bits, as csv_reference.canon_values gives them) or raises Refused
with what the device must report: the status code, the 1-based record (blank lines not counted), its byte offset in the
file and the column where one applies."""
import datetime as dt
import json
import re
from decimal import Decimal

import csv_reference as CR

INVALID, UNSUPPORTED = -1, -2
MAX_DEPTH = 64
_INT_RANGE = {"i8": (-2 ** 7, 2 ** 7 - 1), "i16": (-2 ** 15, 2 ** 15 - 1), "i32": (-2 ** 31, 2 ** 31 - 1), "i64": (-2 ** 63, 2 ** 63 - 1),
              "u8": (0, 2 ** 8 - 1), "u16": (0, 2 ** 16 - 1), "u32": (0, 2 ** 32 - 1), "u64": (0, 2 ** 64 - 1)}
_DATE = re.compile(r"[0-9]{4}-[0-9]{2}-[0-9]{2}\Z")
_WS = b" \t\r"


class Refused(Exception):
    def __init__(self, code, record, offset, column=None, why=""):
        super().__init__(f"{why}: record {record} (byte offset {offset}), column {column}")
        self.code, self.record, self.offset, self.column, self.why = code, record, offset, column, why


class Num(str):
    """A JSON number, kept as its text."""


class _Bad(Exception):
    def __init__(self, code, why):
        super().__init__(why)
        self.code, self.why = code, why


def _no_constant(name):
    raise ValueError("not a JSON literal: " + name)


def _check_string(v):
    """Lone surrogates, which Python's json accepts from \\u escapes."""
    if isinstance(v, str) and not isinstance(v, Num) and any(0xD800 <= ord(c) <= 0xDFFF for c in v):
        raise _Bad(INVALID, "lone surrogate")


class _Obj(list):
    """An object: its (key, value) pairs in order, duplicates kept."""


def parse_line(line: bytes):
    """The pairs of a line's top-level object, or _Bad."""
    try:
        text = line.decode("utf-8")
    except UnicodeDecodeError:
        raise _Bad(INVALID, "invalid UTF-8")
    try:
        v = json.loads(text, object_pairs_hook=_Obj, parse_float=Num, parse_int=Num, parse_constant=_no_constant)
    except (ValueError, RecursionError) as e:
        raise _Bad(INVALID, str(e))
    if not isinstance(v, _Obj):
        raise _Bad(INVALID, "not an object")
    # the depth limit applies to every value below the top-level object; strings are checked everywhere
    for k, x in v:
        _check_string(k)
        _check_value(x, 0)
    return list(v)


def _check_value(x, depth):
    if isinstance(x, list):   # an array, or an object's pairs
        if depth >= MAX_DEPTH:
            raise _Bad(UNSUPPORTED, "nested deeper than 64 levels")
        for y in x:
            if isinstance(x, _Obj):
                _check_string(y[0])
                y = y[1]
            _check_value(y, depth + 1)
    else:
        _check_string(x)


def _type_name(t):
    return "dec" if isinstance(t, dict) else t


def convert(v, t):
    """The column value of JSON value v in a column of plan-IR type t (None: NULL), or _Bad."""
    if v is None:
        return None
    tn = _type_name(t)
    if tn in _INT_RANGE:
        if not isinstance(v, Num) or any(c in v for c in ".eE"):
            raise _Bad(INVALID, "not an integer")
        if tn.startswith("u") and v.startswith("-"):
            raise _Bad(INVALID, "not an integer")
        lo, hi = _INT_RANGE[tn]
        n = int(v)
        if not lo <= n <= hi:
            raise _Bad(INVALID, "integer out of range")
        return n
    if tn == "dec":
        if not isinstance(v, Num) or any(c in v for c in "eE"):
            raise _Bad(INVALID, "not a decimal")
        p, s = t["dec"]
        frac = len(v.split(".")[1]) if "." in v else 0
        if frac > s:
            raise _Bad(INVALID, "decimal scale")
        d = Decimal(v)
        if abs(d.scaleb(s)) >= 10 ** p:
            raise _Bad(INVALID, "decimal precision")
        return d
    if tn == "f64":
        if not isinstance(v, Num):
            raise _Bad(INVALID, "not a number")
        return CR.f64_bits(v)
    if tn == "f32":
        if not isinstance(v, Num):
            raise _Bad(INVALID, "not a number")
        return CR.f32_bits(v)
    if tn == "bool":
        if not isinstance(v, bool):
            raise _Bad(INVALID, "not a boolean")
        return v
    if tn in ("utf8", "date32"):
        if not isinstance(v, str) or isinstance(v, Num):
            raise _Bad(INVALID, "not a string")
        if tn == "utf8":
            return v
        if not _DATE.match(v):
            raise _Bad(INVALID, "not a date")
        try:
            return dt.date(int(v[:4]), int(v[5:7]), int(v[8:]))
        except ValueError:
            raise _Bad(INVALID, "not a date")
    raise _Bad(UNSUPPORTED, "type")


def records(data: bytes):
    """(byte offset, line) of every non-blank line."""
    out, pos = [], 0
    for line in data.split(b"\n"):
        if line.strip(_WS):
            out.append((pos, line))
        pos += len(line) + 1
    return out


def read(data: bytes, schema, columns=None, base_record=0):
    """The scan of one file's bytes: {column: [values]} in `columns` order (None: every schema column)."""
    by_name = {f["name"]: f for f in schema}
    cols = [f["name"] for f in schema] if columns is None else list(columns)
    out = {c: [] for c in cols}
    want = set(cols)
    for r, (off, line) in enumerate(records(data)):
        rec = base_record + r + 1
        try:
            pairs = parse_line(line)
        except _Bad as b:
            raise Refused(b.code, rec, off, None, b.why)
        seen = {}
        for k, v in pairs:
            if k in want:
                if k in seen:
                    raise Refused(INVALID, rec, off, k, "duplicate key")
                seen[k] = v
        vals = {}
        for c in cols:
            v = seen.get(c)
            if isinstance(v, (list, tuple)):
                raise Refused(INVALID, rec, off, c, "not a scalar")
            try:
                x = convert(v, by_name[c]["type"])
            except _Bad as b:
                raise Refused(b.code, rec, off, c, b.why)
            if x is None and not by_name[c].get("nullable", False):
                raise Refused(INVALID, rec, off, c, "NULL in a non-nullable column")
            vals[c] = x
        for c in cols:
            out[c].append(vals[c])
    return out


def dumps_record(obj: dict) -> str:
    """One NDJSON line: json.dumps with numbers given as Num written as their text."""
    parts = []
    for k, v in obj.items():
        if isinstance(v, Num):
            parts.append(json.dumps(k) + ":" + str(v))
        else:
            parts.append(json.dumps(k) + ":" + json.dumps(v, ensure_ascii=False))
    return "{" + ",".join(parts) + "}"
