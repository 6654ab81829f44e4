"""CPU: regexp_count and regexp_replace.  The span DFAs of csrc/common/regex_dfa.hpp (driven through
tests/native/regex_span_check.cpp: the forward / reverse walks and the find_iter step the device operations run) against a
Python reference on the regex corpus, hand-pinned iteration rules, the plan IR typing and its refusals, the protobuf
decoding, and a check that the is_match DFAs are byte-for-byte what they were before the span DFAs existed.

The reference applies the Rust regex crate's find_iter rules (DESIGN.md §6 (xiii)) around Python's `compiled.search(s, pos)`,
not `re.finditer` / `re.sub`, whose empty-match rule differs (`a*` over `baaac`: Python reports an extra empty match).
Python's backtracker and Rust's automata also disagree on which match wins when a repeated sub-expression can match the
empty string (`(|a)*` over `aa`); corpus patterns holding such a repetition are left out of the span comparison (they are
still compiled and walked)."""
import base64
import hashlib
import json
import os
import re
import re._constants as RCON
import re._parser as RPARSE
import subprocess
import zlib

import pytest

import regex_cases as RC
from ballista_b200 import driver, engine
from ballista_b200 import plan as P

HERE = os.path.dirname(os.path.abspath(__file__))
REPL = "<€>"


@pytest.fixture(scope="module")
def native(tmp_path_factory):
    exe = os.path.join(str(tmp_path_factory.mktemp("regex_fn")), "regex_span_check")
    subprocess.run(["g++", "-O2", "-std=c++17", os.path.join(HERE, "native", "regex_span_check.cpp"), "-o", exe], check=True)
    return exe


@pytest.fixture(scope="module")
def tmp(tmp_path_factory):
    return str(tmp_path_factory.mktemp("regex_fn_io"))


def run_native(exe, subs, patterns, tmp, mode="span"):
    """patterns: [(flags, pattern)] -> per pattern (0, [per subject tuple]) | (status, message)"""
    path = os.path.join(tmp, "span_in.txt")
    with open(path, "w") as fh:
        fh.write(f"{len(subs)}\n")
        for s in subs:
            fh.write((s.encode().hex() or "-") + "\n")
        for flags, p in patterns:
            fh.write(f"r {flags or '-'} {p.encode().hex() or '-'}\n")
    args = [exe, path, mode] + ([REPL.encode().hex()] if mode == "span" else [])
    out = subprocess.run(args, check=True, capture_output=True, text=True, timeout=900).stdout.splitlines()
    assert len(out) == len(patterns)
    res = []
    for line in out:
        parts = line.split(" ")
        if parts[0] != "0":
            res.append((int(parts[0]), bytes.fromhex(parts[1]).decode()))
        elif mode == "blob":
            res.append((0, parts[1], parts[2]))
        else:
            res.append((0, [tuple(int(v) for v in p.split(",")) for p in parts[1:]]))
    return res


# ---- the reference ----------------------------------------------------------------------------------------------------
def spans(rx, s):
    """find_iter over s (code point offsets): search from pos; an empty match ending where the last reported one ended is
    skipped and the search restarts one code point on; after another empty match the next search starts one code point
    past it, after a non-empty one at its end"""
    out, pos, last = [], 0, None
    while pos <= len(s):
        m = rx.search(s, pos)
        if m is None:
            break
        a, b = m.span()
        if a == b and b == last:
            pos = b + 1
            continue
        out.append((a, b))
        last = b
        pos = b + 1 if a == b else b
    return out


def replaced(s, sp, repl, glob):
    if not glob:
        sp = sp[:1]
    out, done = [], 0
    for a, b in sp:
        out.append(s[done:a])
        out.append(repl)
        done = b
    out.append(s[done:])
    return "".join(out)


def expected_row(rx, s):
    """(fs, fe, c1, c2, cp, crc_g, len_g, crc_1, len_1) as regex_span_check prints it (byte offsets)"""
    sp = spans(rx, s)
    if sp:
        a, b = sp[0]
        first = (len(s[:a].encode()), len(s[:b].encode()))
    else:
        first = (-1, -1)
    reps = []
    for glob in (True, False):
        r = replaced(s, sp, REPL, glob).encode()
        reps += [zlib.crc32(r), len(r)]
    # regexp_count: an empty str counts 0 before start applies; from start 2 the haystack loses one code point, past the
    # end it is '' (where a pattern that matches empty counts 1)
    counts = (0, 0, 0) if s == "" else (len(sp), len(spans(rx, s[1:])), len(spans(rx, "")))
    return first + counts + tuple(reps)


def empty_repetition(pattern_py, flags):
    """does the pattern repeat (more than once) a sub-expression that can match the empty string?"""
    def walk(items):
        for op, av in items:
            if op in (RCON.MAX_REPEAT, RCON.MIN_REPEAT, getattr(RCON, "POSSESSIVE_REPEAT", None)):
                lo, hi, sub = av
                if hi > 1 and sub.getwidth()[0] == 0:
                    return True
                if walk(sub):
                    return True
            elif op == RCON.SUBPATTERN:
                if walk(av[-1]):
                    return True
            elif op == RCON.BRANCH:
                if any(walk(b) for b in av[1]):
                    return True
        return False
    return walk(RPARSE.parse(pattern_py, RC.python_flags(flags)))


def test_corpus_spans_match_the_reference(native, tmp):
    pats = RC.corpus()
    subs = RC.subjects()
    assert len(subs) >= 2000 and any(len(s) > 4096 for s in subs) and "" in subs
    assert any("K" in s for s in subs) and any("ſ" in s for s in subs)
    assert {f for _r, f, _p, _l in pats} >= {"", "i", "s", "is"}
    res = run_native(native, subs, [(f, rs) for rs, f, _ps, _l in pats], tmp)
    compared = excluded = 0
    for (rs, flags, ps, long_ok), r in zip(pats, res):
        assert r[0] in (0, -2), (rs, r)
        if r[0] != 0:
            assert "DFA" in r[1], (rs, r)  # only the size caps may refuse a generated pattern
            continue
        assert len(r[1]) == len(subs)
        if empty_repetition(ps, flags):
            excluded += 1
            continue
        compared += 1
        rx = re.compile(ps, RC.python_flags(flags))
        for s, got in zip(subs, r[1]):
            if len(s) > 300 and not long_ok:
                continue  # backtracking cost of the reference
            assert got == expected_row(rx, s), (rs, flags, s[:60], got, expected_row(rx, s))
    assert compared >= 190 and excluded < 40, (compared, excluded)


def test_is_match_dfas_are_unchanged(native, tmp):
    with open(os.path.join(HERE, "golden", "regex_is_match_sha256.json")) as fh:
        want = json.load(fh)["dfas"]
    pats = RC.corpus()
    assert [(w["pattern"], w["flags"]) for w in want] == [(rs, f) for rs, f, _p, _l in pats]
    res = run_native(native, [], [(f, rs) for rs, f, _ps, _l in pats], tmp, mode="blob")
    got = [hashlib.sha256(bytes.fromhex(r[1]) + b"|" + r[2].encode()).hexdigest() if r[0] == 0 else None for r in res]
    assert got == [w["sha256"] for w in want]
    assert sum(g is not None for g in got) >= 200


# (flags, pattern, subject, all spans as byte offsets, count, regexp_replace(s, p, 'X', 'g'), regexp_replace(s, p, 'X'))
PINNED = [
    ("", "a*", "baaac", [(0, 0), (1, 4), (5, 5)], "XbXcX", "Xbaaac"),
    ("", "", "abc", [(0, 0), (1, 1), (2, 2), (3, 3)], "XaXbXcX", "Xabc"),
    ("", "", "", [(0, 0)], "X", "X"),
    ("", "a|ab", "abab", [(0, 1), (2, 3)], "XbXb", "Xbab"),
    ("", "ab|a", "abab", [(0, 2), (2, 4)], "XX", "Xab"),
    ("", "a+?", "aaa", [(0, 1), (1, 2), (2, 3)], "XXX", "Xaa"),
    ("", "a+", "aaa", [(0, 3)], "X", "X"),
    ("", "a*?", "aa", [(0, 0), (1, 1), (2, 2)], "XaXaX", "Xaa"),
    ("", "a{2,3}?", "aaaaa", [(0, 2), (2, 4)], "XXa", "Xaaa"),
    ("", "a??b", "ab", [(0, 2)], "X", "X"),
    ("", "^a", "aaa", [(0, 1)], "Xaa", "Xaa"),
    ("", "\\Aa|b", "abab", [(0, 1), (1, 2), (3, 4)], "XXaX", "Xbab"),
    ("", "^", "ab", [(0, 0)], "Xab", "Xab"),
    ("", "a$", "a\n", [], "a\n", "a\n"),
    ("", "a\\n$", "a\n", [(0, 2)], "X", "X"),
    ("", "$", "a\n", [(2, 2)], "a\nX", "a\nX"),
    ("", "x*$", "ax", [(1, 2)], "aX", "aX"),
    ("", "b*", "aé", [(0, 0), (1, 1), (3, 3)], "XaXéX", "Xaé"),
    ("", ".", "é😀", [(0, 2), (2, 6)], "XX", "X😀"),
    ("i", "k", "\u212a k", [(0, 3), (4, 5)], "X X", "X k"),
    ("s", "a.", "a\nb", [(0, 2)], "Xb", "Xb"),
    ("", "a.", "a\nb", [], "a\nb", "a\nb"),
]


def test_pinned_iteration_rules(native, tmp):
    subs = sorted({c[2] for c in PINNED})
    # the replacement 'X' of the table is REPL here: compare through the reference functions, which the table pins too
    res = run_native(native, subs, [(f, p) for f, p, *_ in PINNED], tmp)
    for (flags, p, s, sp, rg, r1), r in zip(PINNED, res):
        assert r[0] == 0, (p, r)
        b = s.encode()
        # the table itself, in code points, against the reference
        cps = [(len(b[:x].decode()), len(b[:y].decode())) for x, y in sp]
        rx = None if (flags, p) == ("i", "k") else re.compile(p.replace("$", "\\Z"), RC.python_flags(flags))
        if rx is not None:
            assert spans(rx, s) == cps, (p, s)
        assert replaced(s, cps, "X", True) == rg and replaced(s, cps, "X", False) == r1, (p, s)
        got = r[1][subs.index(s)]
        first = sp[0] if sp else (-1, -1)
        assert got[:3] == first + (len(sp) if s else 0,), (p, s, got)  # regexp_count of '' is 0
        for glob, k in ((True, 5), (False, 7)):
            want = replaced(s, cps, REPL, glob).encode()
            assert got[k:k + 2] == (zlib.crc32(want), len(want)), (p, s, glob)


def test_count_from_start(native, tmp):
    # the haystack loses its first start - 1 code points, so ^ holds at the new beginning; past the end it is ''
    (r,) = run_native(native, ["éab", "ab", ""], [("", "^a")], tmp)
    assert [g[2:5] for g in r[1]] == [(0, 1, 0), (1, 0, 0), (0, 0, 0)]
    # an empty str counts 0 whatever the start, though '' past the end of a non-empty str counts the empty match
    (r,) = run_native(native, ["éab", ""], [("", "x*")], tmp)
    assert [g[2:5] for g in r[1]] == [(4, 3, 1), (0, 0, 0)]
    for r in run_native(native, [""], [("", "a*"), ("", "x?"), ("", "^$")], tmp):
        assert r[0] == 0 and r[1][0][2:5] == (0, 0, 0), r


def test_span_dfas_share_the_refusals_and_caps(native, tmp):
    cases = [("", "\\w", -2, "\\w"), ("", "(?m)^a", -2, "'m'"), ("", "a(b", -1, "offset 1"), ("", "(a|b)*a.{20}", -2, "DFA"),
             ("i", "é", -2, "U+00E9"), ("g", "a", -1, "regexp_count does not support the \"global\" option")]
    res = run_native(native, ["a"], [(f, p) for f, p, _c, _n in cases], tmp)
    for (f, p, code, needle), r in zip(cases, res):
        assert r[0] == code and needle in r[1], (p, r)


# ---- the plan IR ------------------------------------------------------------------------------------------------------
SCH = [P.field("k", "i32", True), P.field("s", "utf8", True), P.field("t", "utf8", True), P.field("n", "i64", True)]


def _stage(e):
    return P.Stage(1, P.shuffle_writer(P.project([(e, "r")], P.scan("t", SCH)), 1)).json("job")


def _typed_expr(e):
    typed = json.loads(engine.plan_typed_json(_stage(e)))
    node = typed
    while "exprs" not in node:
        node = node["input"]
    return node["exprs"][0]["expr"], node["schema"][0]


def test_ir_typing():
    c, s = P.col, P.lit_utf8
    for args in ([c("s"), s("a")], [c("s"), s("a"), P.lit_i64(2)], [c("s"), s("a"), P.lit_i64(1), s("is")],
                 [c("s"), s(None)], [c("s"), s("")], [P.lit_utf8(None), s("a")]):
        e, f = _typed_expr(P.fn("regexp_count", *args))
        assert e["fn"] == "regexp_count" and f["type"] == "i64" and f["nullable"] is True, (args, f)
    for args in ([c("s"), s("a"), s("b")], [c("s"), s("a"), s("b"), s("gi")], [c("s"), s("a"), s(None)], [c("s"), s("a"), s(""), s("")]):
        e, f = _typed_expr(P.fn("regexp_replace", *args))
        assert e["fn"] == "regexp_replace" and f["type"] == "utf8" and f["nullable"] is True, (args, f)


@pytest.mark.parametrize("e,code,needle", [
    (lambda c: P.fn("regexp_count", c("s"), c("t")), -2, "literal"),
    (lambda c: P.fn("regexp_count", c("s"), P.lit_utf8("\\w")), -2, "\\w"),
    (lambda c: P.fn("regexp_count", c("s"), P.lit_utf8("a(b")), -1, "offset 1"),
    (lambda c: P.fn("regexp_count", c("k"), P.lit_utf8("a")), -2, "i32"),
    (lambda c: P.fn("regexp_count", c("s"), P.lit_utf8("a"), P.lit_i64(0)), -1, "start"),
    (lambda c: P.fn("regexp_count", c("s"), P.lit_utf8("a"), c("n")), -2, "start"),
    (lambda c: P.fn("regexp_count", c("s"), P.lit_utf8("a"), P.lit_i64(None)), -2, "start"),
    (lambda c: P.fn("regexp_count", c("s"), P.lit_utf8("a"), P.lit_i64(1), c("t")), -2, "flags"),
    (lambda c: P.fn("regexp_count", c("s"), P.lit_utf8("a"), P.lit_i64(1), P.lit_utf8(None)), -2, "flags"),
    (lambda c: P.fn("regexp_count", c("s"), P.lit_utf8(None), P.lit_i64(1), P.lit_utf8(None)), -2, "flags"),
    (lambda c: P.fn("regexp_count", c("s"), P.lit_utf8(None), P.lit_i64(1), P.lit_utf8("zz")), -1, "unrecognized flag"),
    (lambda c: P.fn("regexp_replace", c("s"), P.lit_utf8(None), P.lit_utf8("x"), P.lit_utf8("m")), -2, "'m'"),
    (lambda c: P.fn("regexp_count", c("s"), P.lit_utf8("a"), P.lit_i64(1), P.lit_utf8("g")), -1, "global"),
    (lambda c: P.fn("regexp_count", c("s"), P.lit_utf8("a"), P.lit_i64(1), P.lit_utf8("m")), -2, "'m'"),
    (lambda c: P.fn("regexp_count", c("s")), -1, "argument"),
    (lambda c: P.fn("regexp_replace", c("s"), P.lit_utf8("a"), c("t")), -2, "replacement"),
    (lambda c: P.fn("regexp_replace", c("s"), P.lit_utf8("a"), P.lit_utf8("$1")), -2, "replacement '$1'"),
    (lambda c: P.fn("regexp_replace", c("s"), P.lit_utf8("a"), P.lit_utf8("x\\1")), -2, "replacement"),
    (lambda c: P.fn("regexp_replace", c("s"), c("t"), P.lit_utf8("x")), -2, "literal"),
    (lambda c: P.fn("regexp_replace", c("s"), P.lit_utf8("a"), P.lit_utf8("x"), c("t")), -2, "flags"),
    (lambda c: P.fn("regexp_replace", c("s"), P.lit_utf8("a"), P.lit_utf8("x"), P.lit_utf8("x")), -2, "'x'"),
    (lambda c: P.fn("regexp_replace", c("s"), P.lit_utf8("\\b"), P.lit_utf8("x")), -2, "\\b"),
    (lambda c: P.fn("regexp_replace", c("s"), P.lit_utf8("a")), -1, "argument"),
], ids=["count_column_pattern", "count_word", "count_syntax", "count_non_utf8", "count_start_0", "count_start_column",
        "count_start_null", "count_flags_column", "count_flags_null", "count_null_pattern_null_flags",
        "count_null_pattern_bad_flags", "replace_null_pattern_flag_m", "count_flag_g", "count_flag_m", "count_arity", "replace_column_replacement",
        "replace_dollar", "replace_backslash", "replace_column_pattern", "replace_flags_column", "replace_flag_x",
        "replace_word_boundary", "replace_arity"])
def test_ir_refusals(e, code, needle):
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(_stage(e(P.col)))
    assert ei.value.code == code and needle in str(ei.value), str(ei.value)


def test_oracle_refuses_regex_functions(oracle):
    import pyarrow as pa
    t = pa.table({"k": pa.array([1], pa.int32()), "s": pa.array(["a"]), "t": pa.array(["b"]), "n": pa.array([1], pa.int64())})
    oracle.register_batch("t", 0, t.to_batches()[0])
    for e in (P.fn("regexp_count", P.col("s"), P.lit_utf8("a")), P.fn("regexp_replace", P.col("s"), P.lit_utf8("a"), P.lit_utf8("b"))):
        with pytest.raises(Exception) as ei:
            driver.run_stages(oracle, [P.Stage(1, P.shuffle_writer(P.project([(e, "r")], P.scan("t", SCH)), 1))], "refuse")
        assert "not computed by this consumer" in str(ei.value)


# ---- protobuf ---------------------------------------------------------------------------------------------------------
with open(os.path.join(HERE, "golden", "regex_fn_proto_plans.json")) as fh:
    PROTO = json.load(fh)["cases"]
PROTO_GOOD = [c for c in PROTO if "code" not in c]
PROTO_REFUSED = [c for c in PROTO if "code" in c]


def test_proto_fixtures_cover_both_functions():
    names = {c["name"].split("/")[0] for c in PROTO}
    assert {"count", "count_start", "count_start_flags", "replace", "replace_global", "replace_flags_gi", "refused_replacement_dollar",
            "invalid_count_flag_g", "invalid_count_start_0"} <= names


@pytest.mark.parametrize("case", PROTO_GOOD, ids=[c["name"] for c in PROTO_GOOD])
def test_proto_decodes_like_the_source_ir(case):
    got_ir = engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]))
    assert json.loads(engine.plan_typed_json(got_ir)) == json.loads(engine.plan_typed_json(case["ir"]))


def _outcome(f):
    try:
        f()
    except engine.B200Error as e:
        return e.code, str(e)
    return 0, ""


@pytest.mark.parametrize("case", PROTO_REFUSED, ids=[c["name"] for c in PROTO_REFUSED])
def test_proto_refusals_equal_the_ir_refusals(case):
    code, msg = _outcome(lambda: engine.plan_typed_json(engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]))))
    assert code == case["code"] and case["needle"] in msg, msg
    want = _outcome(lambda: engine.plan_typed_json(case["ir"]))
    assert (code, msg.split(": ", 1)[1]) == (want[0], want[1].split(": ", 1)[1])
