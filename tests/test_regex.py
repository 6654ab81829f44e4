"""CPU: the regex compiler and DFA walk of csrc/common/regex_dfa.hpp (driven through tests/native/regex_check.cpp, the walk the
OP_REGEX device operation runs) against Python's re on a seeded corpus, hand-pinned folding and anchor rules, refusals by
name, syntax errors by offset, the DFA size cap, arrow's ILIKE translation, and the plan IR / typing surface (host-only
library calls; the CPU oracle refuses these predicates)."""
import json
import random

import pytest

import regex_cases as RC
from ballista_b200 import driver, engine
from ballista_b200 import plan as P


@pytest.fixture(scope="module")
def native(tmp_path_factory):
    return RC.build_native(str(tmp_path_factory.mktemp("regex")))


@pytest.fixture(scope="module")
def tmp(tmp_path_factory):
    return str(tmp_path_factory.mktemp("regex_io"))


def test_corpus_matches_python_re(native, tmp):
    pats = RC.corpus()
    subs = RC.subjects()
    assert len(subs) >= 2000 and any(len(s) > 4096 for s in subs) and "" in subs
    assert any(s.endswith("\n") for s in subs) and any("K" in s for s in subs) and any("ſ" in s for s in subs)
    assert all(any(len(c.encode()) == k for s in subs for c in s) for k in (1, 2, 3, 4))
    res = RC.run_native(native, subs, [("r", f, rs) for rs, f, _ps, _l in pats], tmp)
    compiled = 0
    for (rs, flags, ps, long_ok), r in zip(pats, res):
        assert r[0] in (0, -2), (rs, r)
        if r[0] != 0:
            assert "DFA" in r[1], (rs, r)  # only the size cap may refuse a generated pattern
            continue
        compiled += 1
        want = RC.expected(ps, flags, subs, long_ok)
        bad = [(subs[i], w) for i, w in enumerate(want) if w is not None and w != (r[2][i] == "1")]
        assert not bad, (rs, flags, ps, bad[:3])
    assert compiled >= 200


# (kind, flags, pattern, subject, expected): each folding and anchor rule, written out by hand
PINNED = [
    # case-insensitive: ASCII letters, KELVIN SIGN and LONG S, negated classes folded before negation
    ("r", "i", "k", "K", True), ("r", "i", "K", "K", True), ("r", "i", "s", "ſ", True), ("r", "i", "S", "ſ", True),
    ("r", "", "k", "K", False), ("r", "", "s", "ſ", False), ("r", "i", "[^k]", "K", False), ("r", "i", "[^k]", "K", False),
    ("r", "i", "[^s]", "ſ", False), ("r", "i", "^[a-z]+$", "ABC", True), ("r", "i", "[[:upper:]]", "k", True),
    ("r", "", "(?i)abc", "AbC", True), ("r", "", "(?i:a)b", "Ab", True), ("r", "", "(?i:a)b", "AB", False),
    ("r", "i", "(?-i)a", "A", False), ("r", "", "a(?i)b|c", "C", True), ("r", "i", "é", "É", None),
    ("r", "", "é", "é", True), ("r", "", "(?-i:é)", "é", True),
    # a negated POSIX class is folded before it is negated, like every class
    ("r", "i", "^[[:^lower:]]$", "a", False), ("r", "i", "[[:^lower:]]", "z", False), ("r", "i", "[[:^lower:]]", "A", False),
    ("r", "i", "[^[:lower:]]", "a", False), ("r", "i", "[[:^alpha:]]", "k", False), ("r", "i", "[[:^alpha:]]", "K", False),
    ("r", "i", "[[:^alpha:]]", "K", False), ("r", "i", "[[:^alpha:]]", "ſ", False), ("r", "i", "[[:^lower:]]", "1", True),
    ("r", "", "[[:^lower:]]", "A", True), ("r", "", "[[:^lower:]]", "a", False),
    # anchors: Rust's $ and \z are the end of the text only; ^ and \A its start
    ("r", "", "a$", "a\n", False), ("r", "", "a\\z", "a\n", False), ("r", "", "a\\n$", "a\n", True), ("r", "", "a$", "ba", True),
    ("r", "", "^a", "ba", False), ("r", "", "\\Aa", "ab", True), ("r", "", "^$", "", True), ("r", "", "$", "abc", True),
    ("r", "", "a^", "a", False), ("r", "", "$^", "", True), ("r", "", "^", "", True), ("r", "", "^$", "\n", False),
    # . is one scalar value, not \n unless s
    ("r", "", ".", "\n", False), ("r", "s", ".", "\n", True), ("r", "", "(?s).", "\n", True), ("r", "", "^.$", "é", True),
    ("r", "", "^.$", "😀", True), ("r", "", "^..$", "é", False), ("r", "", "^[^a]$", "中", True),
    # Unicode \d (Nd) and \s (White_Space)
    ("r", "", "^\\d$", "٣", True), ("r", "", "^\\s$", "　", True), ("r", "", "\\s", "\x1c", False), ("r", "", "^\\D$", "٣", False),
    # escapes and repetition
    ("r", "", "^\\x{1F600}$", "😀", True), ("r", "", "^\\xe9$", "é", True), ("r", "", "^\\x{000000041}$", "A", True), ("r", "", "^a{2,3}$", "aaaa", False), ("r", "", "^a{2,}?$", "aaaa", True),
    # ILIKE: anchored, % and _ (one scalar value, newlines included), \ escapes, case folding
    ("l", "", "%ab_c%", "xABéCx", True), ("l", "", "ab", "AB", True), ("l", "", "ab", "xab", False), ("l", "", "a%", "a\nb", True),
    ("l", "", "a_b", "a\nb", True), ("l", "", "a\\%b", "a%b", True), ("l", "", "a\\%b", "axb", False), ("l", "", "a\\_b", "a_b", True),
    ("l", "", "a\\_b", "axb", False), ("l", "", "k", "K", True), ("l", "", "a.c", "abc", False), ("l", "", "a\\\\b", "a\\b", True),
    ("l", "", "(x)*", "(X)*", True), ("l", "", "%", "", True), ("l", "", "_", "", False),
]


def test_pinned_rules(native, tmp):
    subs = sorted({p[3] for p in PINNED})
    res = RC.run_native(native, subs, [(k, f, p) for k, f, p, _s, _w in PINNED], tmp)
    for (k, f, p, s, want), r in zip(PINNED, res):
        if want is None:
            assert r[0] == -2 and "U+00E9" in r[1], (p, r)
            continue
        assert r[0] == 0, (p, r)
        assert (r[2][subs.index(s)] == "1") == want, (k, f, p, s)


REFUSED = [
    ("r", "", "\\w", "\\w"), ("r", "", "a\\W", "\\W"), ("r", "", "\\bfoo", "\\b"), ("r", "", "x\\B", "\\B"), ("r", "", "\\p{L}", "\\p"),
    ("r", "", "\\P{L}", "\\P"), ("r", "", "\\<a", "\\<"), ("r", "", "(?m)^a", "'m'"), ("r", "", "(?x)a b", "'x'"),
    ("r", "", "(?U)a+", "'U'"), ("r", "", "(?-u)a", "'u'"), ("r", "", "(?R)a", "'R'"), ("r", "", "[a-z&&b]", "&&"),
    ("r", "", "[a-z--b]", "--"), ("r", "", "[a~~b]", "~~"), ("r", "m", "a", "'m'"), ("r", "x", "a", "'x'"), ("r", "U", "a", "'U'"),
    ("r", "u", "a", "'u'"), ("r", "R", "a", "'R'"), ("r", "i", "é", "U+00E9"), ("r", "", "(?i)[é]", "U+00E9"),
    ("l", "", "%é%", "U+00E9"), ("r", "", "(a|b)*a.{20}", "DFA"), ("r", "", "a**", "repetition"),
]


@pytest.mark.parametrize("case", REFUSED, ids=[f"{c[0]}:{c[2]}/{c[1]}" for c in REFUSED])
def test_refused_constructs_are_named(native, tmp, case):
    kind, flags, pat, needle = case
    (r,) = RC.run_native(native, [], [(kind, flags, pat)], tmp)
    assert r[0] == -2 and needle in r[1], r
    if kind == "r" and not flags:
        assert pat in r[1]  # the message names the pattern too


INVALID = [
    ("r", "", "a(b", 1), ("r", "", "a)b", 1), ("r", "", "*a", 0), ("r", "", "a|+", 2), ("r", "", "a{2,1}", 1), ("r", "", "[a", 0),
    ("r", "", "a{", 1), ("r", "", "a{x}", 1), ("r", "", "\\", 0), ("r", "", "(?z)", 2), ("r", "", "[z-a]", 1), ("r", "", "(?i)*", 4),
    ("r", "", "\\1", 0), ("r", "", "(?=a)", 0), ("r", "", "\\x{110000}", 0), ("r", "", "(?P<1a>x)", 4), ("r", "", "\\q", 0),
    ("l", "", "ab\\", 2), ("r", "", "[\\d-z]", 1), ("r", "", "[a\\s-z]", 2),
]


@pytest.mark.parametrize("case", INVALID, ids=[f"{c[0]}:{c[2]}" for c in INVALID])
def test_syntax_errors_give_the_offset(native, tmp, case):
    kind, flags, pat, off = case
    (r,) = RC.run_native(native, [], [(kind, flags, pat)], tmp)
    assert r[0] == -1 and f"offset {off}:" in r[1] + ":", r


def test_dfa_size_cap_is_a_refusal_not_a_truncation(native, tmp):
    pats = [("r", "", "(a|b)*a.{20}"), ("r", "", "[ab]*a[ab]{10}"), ("r", "", "[ab]*a[ab]{14}")]
    res = RC.run_native(native, ["b" * 40 + "a" + "b" * 12, "b" * 40], pats, tmp)
    assert res[0][0] == -2 and "DFA" in res[0][1]
    assert res[1][0] == 0 and res[1][2] == "10"       # below the cap: exact
    assert res[2][0] == 0 and res[2][1] > 16000        # a large DFA that still fits
    assert res[2][2] == "00"


def test_ilike_agrees_with_arrows_translation(native, tmp):
    r = random.Random(5)
    alpha = list("abkKsSxy%_\\") + ["%", "_"]
    likes = set()
    while len(likes) < 150:
        p = "".join(r.choice(alpha) for _ in range(r.randint(0, 6)))
        if not p.endswith("\\") or p.endswith("\\\\"):
            likes.add(p)
    likes = sorted(likes)
    subs = ["", "\n"] + ["".join(r.choice(list("abkKsSxy%_\\\nKſé")) for _ in range(r.randint(0, 7))) for _ in range(600)]
    res = RC.run_native(native, subs, [("l", "", p) for p in likes], tmp)
    import re
    for p, got in zip(likes, res):
        if got[0] != 0:  # a trailing lone backslash after an escaped one, e.g. "a\\\\\\"
            assert got[0] == -1, (p, got)
            continue
        rx = re.compile(RC.like_to_python(p), re.I | re.S)
        want = "".join("1" if rx.search(s) else "0" for s in subs)
        assert got[2] == want, p


# ---- the plan IR ------------------------------------------------------------------------------------------------------
SCH = [P.field("k", "i32", True), P.field("s", "utf8", True), P.field("t", "utf8", True)]


def _stage(e):
    return P.Stage(1, P.shuffle_writer(P.project([(e, "r")], P.scan("t", SCH)), 1)).json("job")


def _typed_expr(e):
    typed = json.loads(engine.plan_typed_json(_stage(e)))
    node = typed
    while "exprs" not in node:
        node = node["input"]
    return node["exprs"][0]["expr"], node["schema"][0]


def test_ir_typing_and_dump():
    c = P.col
    e, f = _typed_expr(P.like(c("s"), "%a_%", case_insensitive=True))
    assert e.get("case_insensitive") is True and f["type"] == "bool" and f["nullable"] is True
    e, _ = _typed_expr(P.like(c("s"), "%a_%"))
    assert "case_insensitive" not in e  # plain LIKE dumps as before
    for neg in (False, True):
        for ci in (False, True):
            e, f = _typed_expr(P.regex_match(c("s"), "a+", negated=neg, case_insensitive=ci))
            assert e["bin"] == ("!~" if neg else "~") + ("*" if ci else "") and f["type"] == "bool"
    e, f = _typed_expr(P.fn("regexp_like", c("s"), P.lit_utf8("a"), P.lit_utf8("is")))
    assert e["fn"] == "regexp_like" and f["type"] == "bool" and f["nullable"] is True
    # NULL patterns and flags type (the result is NULL)
    _typed_expr(P.regex_match(c("s"), P.lit_utf8(None)))
    _typed_expr(P.fn("regexp_like", c("s"), P.lit_utf8("a"), P.lit_utf8(None)))


@pytest.mark.parametrize("e,code,needle", [
    (lambda c: P.regex_match(c("s"), "\\w"), -2, "\\w"),
    (lambda c: P.regex_match(c("s"), "a(b"), -1, "offset 1"),
    (lambda c: P.regex_match(c("s"), c("t")), -2, "literal"),
    (lambda c: P.regex_match(c("k"), "a"), -2, "i32"),
    (lambda c: P.fn("regexp_like", c("s"), c("t")), -2, "literal"),
    (lambda c: P.fn("regexp_like", c("s"), P.lit_utf8("a"), c("t")), -2, "literal"),
    (lambda c: P.fn("regexp_like", c("s"), P.lit_utf8("a"), P.lit_utf8("g")), -1, "global"),
    (lambda c: P.fn("regexp_like", c("s"), P.lit_utf8("a"), P.lit_utf8("m")), -2, "'m'"),
    (lambda c: P.fn("regexp_like", c("s")), -1, "argument"),
    (lambda c: P.like(c("s"), "é%", case_insensitive=True), -2, "U+00E9"),
    (lambda c: P.like(c("s"), "a\\", case_insensitive=True), -1, "offset 1"),
], ids=["word", "syntax", "column_pattern", "non_utf8", "regexp_like_column", "flags_column", "flag_g", "flag_m", "arity",
        "ilike_non_ascii", "ilike_trailing_escape"])
def test_ir_refusals(e, code, needle):
    with pytest.raises(engine.B200Error) as ei:
        engine.plan_typed_json(_stage(e(P.col)))
    assert ei.value.code == code and needle in str(ei.value), str(ei.value)


def test_oracle_refuses_regex_plans(oracle):
    import pyarrow as pa
    t = pa.table({"k": pa.array([1], pa.int32()), "s": pa.array(["a"]), "t": pa.array(["b"])})
    oracle.register_batch("t", 0, t.to_batches()[0])
    for e in (P.like(P.col("s"), "a", case_insensitive=True), P.regex_match(P.col("s"), "a"), P.fn("regexp_like", P.col("s"), P.lit_utf8("a"))):
        with pytest.raises(Exception) as ei:
            driver.run_stages(oracle, [P.Stage(1, P.shuffle_writer(P.project([(e, "r")], P.scan("t", SCH)), 1))], "refuse")
        assert "not computed by this consumer" in str(ei.value)


def test_pattern_above_the_bmp_survives_the_plan_text():
    # JSON writers send U+1F600 as a surrogate pair; the pattern must reach the compiler as one 4-byte character
    e, _ = _typed_expr(P.regex_match(P.col("s"), "z[😀\\s]"))
    assert e["r"]["lit"]["v"] == "z[😀\\s]"
    e, _ = _typed_expr(P.like(P.col("s"), "%😀_"))
    assert e["pattern"] == "%😀_"


@pytest.mark.parametrize("pat", ["[" * 20000 + "a" + "]" * 20000, "(" * 20000 + "a" + ")" * 20000, "[" * 251 + "a" + "]" * 251,
                                 "(?:" * 126 + "[" * 126 + "a" + "]" * 126 + ")" * 126],
                         ids=["classes_20000", "groups_20000", "classes_251", "groups_and_classes_252"])
def test_deep_nesting_is_refused_not_a_crash(native, tmp, pat):
    (r,) = RC.run_native(native, [], [("r", "", pat)], tmp)
    assert r[0] == -2 and "nesting" in r[1], r[:1]


def test_nesting_at_the_limit_compiles(native, tmp):
    (r,) = RC.run_native(native, ["a", "b"], [("r", "", "[" * 250 + "a" + "]" * 250)], tmp)
    assert r[0] == 0 and r[2] == "10"


def test_empty_repetitions_compile_at_once(native, tmp):
    import time
    pats = [("r", "", "(?:" * k + "(?:)" + "){1000}" * k) for k in (3, 5, 8)] + [("r", "", "x(?:(?:){1000}a{0}){1000}y")]
    t0 = time.monotonic()
    res = RC.run_native(native, ["xy", "x", ""], pats, tmp)
    assert time.monotonic() - t0 < 10
    assert [r[0] for r in res] == [0, 0, 0, 0]
    assert [r[2] for r in res] == ["111", "111", "111", "100"]


def test_dfa_construction_work_is_bounded(native, tmp):
    import time
    # few states, but each closes over thousands of NFA states: refused by the work bound, not left to run for long
    pat = "(?:(?:.?){1000}){4}[ab]*a[ab]{8}x"
    t0 = time.monotonic()
    (r,) = RC.run_native(native, ["ab"], [("r", "", pat)], tmp)
    assert time.monotonic() - t0 < 10
    assert r[0] == -2 and "expensive" in r[1], r
