"""The regex corpus shared by tests/test_regex.py (host compiler and walk, tests/native/regex_check.cpp) and
tests/test_gpu_regex.py (the same patterns as device stages): seeded random patterns in the accepted Rust-regex subset, each
rendered twice -- in Rust syntax for the engine and in Python syntax for the reference answer (re.search) -- and subject
strings covering ASCII, 2- to 4-byte UTF-8, the empty string, strings ending in a newline, strings over 4 KB and the two
non-ASCII code points that fold onto ASCII letters (U+212A KELVIN SIGN, U+017F LATIN SMALL LETTER LONG S).

Python's re agrees with Rust on this subset once three spellings are mapped: Rust's `$` and `\\z` (end of text only) are
Python's `\\Z`, a POSIX class is written out as ranges, and an inline flag group (?i) in the middle of a group becomes a
scoped group running to the group's end.  Subjects avoid the code points where the two differ outside the subset: U+001C..
U+001F (Python's \\s, not White_Space), U+0130 / U+0131 (Python's per-character lower / upper case)."""
import random
import re
import subprocess
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

META = set("\\.+*?()|[]{}^$#&-~")
NON_ASCII = ["é", "ж", "€", "中", "😀", "K", "ſ", "٣", " ", " ", "　", "ß", "Ω"]
ASCII_LIT = list("abcdefkqsz") + list("ABKSZ") + list("019") + [" ", "-", ".", "%", "_", "/", "\n", "\t"]
POSIX = {"alpha": "A-Za-z", "digit": "0-9", "lower": "a-z", "upper": "A-Z", "space": "\\t\\n\\x0b\\f\\r ", "xdigit": "0-9A-Fa-f",
         "alnum": "0-9A-Za-z", "punct": "!-/:-@\\[-`{-~", "word": "0-9A-Za-z_", "blank": "\\t "}


def _esc(ch):
    if ch == "\n":
        return "\\n"
    if ch == "\t":
        return "\\t"
    return "\\" + ch if ch in META or ch == " " and False else ch


class Gen:
    """Random pattern generator.  pattern() -> (rust, python, n_unbounded)"""

    def __init__(self, rnd):
        self.r = rnd
        self.names = 0
        self.unbounded = 0

    def lit(self, ci):
        pool = ASCII_LIT if ci or self.r.random() < 0.8 else NON_ASCII
        ch = self.r.choice(pool)
        e = _esc(ch)
        return e, e

    def cls_item(self, ci):
        k = self.r.random()
        if k < 0.15:
            e = self.r.choice(["\\d", "\\s", "\\D", "\\S"])
            return e, e
        if k < 0.25:
            name = self.r.choice(sorted(POSIX))
            return f"[:{name}:]", POSIX[name]
        pool = "abcdefkqsxyzKS019"
        if k < 0.55:
            a, b = sorted(self.r.sample(pool, 2))
            return f"{a}-{b}", f"{a}-{b}"
        ch = self.r.choice(list(pool) + ["-", ".", "^", "[", "]", "&", "~"] + ([] if ci else ["é", "€", "😀", "K"]))
        e = "\\" + ch if ch in META else ch
        return e, e

    def cls(self, ci):
        neg = self.r.random() < 0.3
        items = [self.cls_item(ci) for _ in range(self.r.randint(1, 3))]
        h = "^" if neg else ""
        return "[" + h + "".join(i[0] for i in items) + "]", "[" + h + "".join(i[1] for i in items) + "]"

    def atom(self, depth, ci, dotall):
        k = self.r.random()
        if k < 0.45:
            return self.lit(ci), True
        if k < 0.55:
            return (".", "."), True
        if k < 0.68:
            return self.cls(ci), True
        if k < 0.74:
            e = self.r.choice(["\\d", "\\s", "\\D", "\\S"])
            return (e, e), True
        if k < 0.80:
            a = self.r.choice([("^", "^"), ("$", "\\Z"), ("\\A", "\\A"), ("\\z", "\\Z")])
            return a, False
        if depth >= 2:
            return self.lit(ci), True
        return self.group(depth + 1, ci, dotall), True

    def group(self, depth, ci, dotall):
        kind = self.r.choice(["cap", "noncap", "named", "flags", "flags"])
        if kind == "flags":
            f = self.r.choice(["i", "-i", "s", "-s", "is"])
            ci2 = ("i" in f and "-i" not in f) or (ci and "-i" not in f)
            ds2 = ("s" in f and "-s" not in f) or (dotall and "-s" not in f)
            body = self.alt(depth, ci2, ds2)
            return f"(?{f}:" + body[0] + ")", f"(?{f}:" + body[1] + ")"
        body = self.alt(depth, ci, dotall)
        if kind == "cap":
            return "(" + body[0] + ")", "(" + body[1] + ")"
        if kind == "noncap":
            return "(?:" + body[0] + ")", "(?:" + body[1] + ")"
        self.names += 1
        n = f"g{self.names}"
        return f"(?P<{n}>" + body[0] + ")", f"(?P<{n}>" + body[1] + ")"

    def rep(self, is_single):
        k = self.r.random()
        lazy = "?" if self.r.random() < 0.2 else ""
        if k < 0.5:
            return "", False
        if is_single and k < 0.75:
            return self.r.choice(["*", "+"]) + lazy, True
        if is_single and k < 0.8:
            return "{%d,}" % self.r.randint(0, 2) + lazy, True
        if k < 0.88:
            return "?" + lazy, False
        if k < 0.94:
            return "{%d}" % self.r.randint(0, 3) + lazy, False
        a = self.r.randint(0, 2)
        return "{%d,%d}" % (a, a + self.r.randint(0, 2)) + lazy, False

    def concat(self, depth, ci, dotall, allow_flags):
        rs, ps = "", ""
        n = self.r.randint(1, 4)
        for i in range(n):
            if allow_flags and i > 0 and self.r.random() < 0.1:
                # Rust (?i) mid-group runs to the group's end: Python spells it as a scoped group
                f = self.r.choice(["i", "-i", "s"])
                ci2 = (f == "i") or (ci and f != "-i")
                ds2 = (f == "s") or dotall
                rest = self.concat(depth, ci2, ds2, False)
                return rs + f"(?{f})" + rest[0], ps + f"(?{f}:" + rest[1] + ")"
            (ra, pa), repeatable = self.atom(depth, ci, dotall)
            if repeatable:
                single = not ra.startswith("(")
                q, unb = self.rep(single)
                if unb:
                    self.unbounded += 1
                ra, pa = ra + q, pa + q
            rs, ps = rs + ra, ps + pa
        return rs, ps

    def alt(self, depth, ci, dotall):
        n = 1 if self.r.random() < 0.7 else self.r.randint(2, 3)
        if n == 1:
            return self.concat(depth, ci, dotall, True)
        parts = [self.concat(depth, ci, dotall, False) for _ in range(n)]
        return "|".join(p[0] for p in parts), "|".join(p[1] for p in parts)

    def pattern(self, ci, dotall):
        self.names = 0
        self.unbounded = 0
        rs, ps = self.alt(0, ci, dotall)
        return rs, ps, self.unbounded


def corpus(n_patterns=240, seed=20261017):
    """[(rust pattern, flags, python pattern, long_ok)]"""
    r = random.Random(seed)
    g = Gen(r)
    out = []
    for i in range(n_patterns):
        flags = r.choice(["", "", "", "i", "s", "is"])
        rs, ps, unb = g.pattern("i" in flags, "s" in flags)
        out.append((rs, flags, ps, unb <= 1))
    return out


def subjects(n=2000, seed=7):
    r = random.Random(seed)
    alpha = list("abcdefkqsz") * 3 + list("ABKSZ") + list("0123456789") + [" ", " ", "-", ".", "%", "_", "/", "\n", "\t", "&", "~"] + NON_ASCII
    out = ["", "\n", "a", "a\n", "K", "ſ", "K", "S", "k", "s", "é", "😀"]
    while len(out) < n - 6:
        s = "".join(r.choice(alpha) for _ in range(r.choice([1, 2, 3, 5, 8, 13, 21])))
        if r.random() < 0.1:
            s += "\n"
        out.append(s)
    for _ in range(6):  # over 4 KB
        out.append("".join(r.choice(alpha) for _ in range(4200 + r.randrange(300))))
    return out


def python_flags(flags):
    return (re.I if "i" in flags else 0) | (re.S if "s" in flags else 0)


def expected(pattern_py, flags, subs, long_ok=True):
    """re.search over subs; None for subjects skipped for backtracking cost"""
    rx = re.compile(pattern_py, python_flags(flags))
    return [None if (len(s) > 300 and not long_ok) else rx.search(s) is not None for s in subs]


def like_to_python(like):
    """arrow-rs's LIKE -> regex translation (applied with the flags i and s), written in Python's syntax"""
    out, i = ["^"], 0
    while i < len(like):
        c = like[i]
        if c == "\\":
            i += 1
            out.append(re.escape(like[i]))
        elif c == "%":
            out.append(".*")
        elif c == "_":
            out.append(".")
        else:
            out.append(re.escape(c))
        i += 1
    out.append("\\Z")
    return "".join(out)


def run_native(exe, subs, patterns, tmp):
    """patterns: [(kind 'r' | 'l', flags, pattern)] -> [(status, n_states, bits) | (status, message)]"""
    path = os.path.join(tmp, "regex_in.txt")
    with open(path, "w") as fh:
        fh.write(f"{len(subs)}\n")
        for s in subs:
            fh.write((s.encode().hex() or "-") + "\n")
        for kind, flags, p in patterns:
            fh.write(f"{kind} {flags or '-'} {p.encode().hex() or '-'}\n")
    out = subprocess.run([exe, path], check=True, capture_output=True, text=True, timeout=600).stdout.splitlines()
    assert len(out) == len(patterns)
    res = []
    for line in out:
        parts = line.split(" ")
        if parts[0] == "0":
            res.append((0, int(parts[1]), parts[2] if parts[2] != "-" else ""))
        else:
            res.append((int(parts[0]), bytes.fromhex(parts[1]).decode()))
    return res


def build_native(tmp):
    exe = os.path.join(tmp, "regex_check")
    subprocess.run(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "native", "regex_check.cpp"), "-o", exe], check=True)
    return exe
