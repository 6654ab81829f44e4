"""GPU: regexp_count and regexp_replace as device stages (the count op and the arena builder over the span DFAs the host
compiled).  The corpus of tests/regex_cases.py runs as ProjectionExec stages over a two-partition table with NULLs, 70 KB
strings and multi-byte UTF-8, and must equal the find_iter reference of tests/test_regex_fn.py bit for bit (patterns that
reference leaves out are compared with the host walk of tests/native/regex_span_check.cpp); a count is a filter; a
replacement that outgrows the first arena is re-run; the protobuf fixtures give the results of their IR; TPC-H q13 with its
NOT LIKE rewritten as regexp_count(...) = 0 gives the oracle's q13."""
import base64
import json
import os
import random
import re
import zlib

import pyarrow as pa
import pytest

import regex_cases as RC
import test_regex_fn as TF
from ballista_b200 import driver, tpch
from ballista_b200 import plan as P
from util import assert_tables_equal

HERE = os.path.dirname(os.path.abspath(__file__))
SCH = [P.field("k", "i32", False), P.field("s", "utf8", True), P.field("t", "utf8", True)]
REPL = TF.REPL


def _values(long_rows=True):
    r = random.Random(11)
    alpha = list("abcdefkqsz") * 3 + list("ABKSZ") + list("0123456789 \n") + RC.NON_ASCII
    long = []
    for _ in range(2):   # 70 KB each in UTF-8
        chars, n = [], 0
        while n < 70 * 1024:
            chars.append(r.choice(alpha))
            n += len(chars[-1].encode())
        long.append("".join(chars))
    subs = RC.subjects() + (long if long_rows else [])
    return [None if i % 97 == 5 else s for i, s in enumerate(subs)]


def _table(vals):
    return pa.table({"k": pa.array(range(len(vals)), pa.int32()), "s": pa.array(vals, pa.string()),
                     "t": pa.array(["x"] * len(vals), pa.string())})


def _register(e, t, parts=2):
    e.drop_table("t")
    step = (t.num_rows + parts - 1) // parts
    for p in range(parts):
        e.register_batch("t", p, t.slice(p * step, step).combine_chunks().to_batches()[0])


def _run(gpu, stages, job):
    out = driver.run_stages(gpu, stages, job)
    gpu.remove_job_data(job)
    return out


def _project(exprs):
    scan = P.scan("t", SCH)
    return [P.Stage(1, P.shuffle_writer(P.project([(P.col("k"), "k")] + [(e, f"r{j}") for j, e in enumerate(exprs)], scan), 1))]


def _rows(tbl, n):
    d = tbl.to_pydict()
    return {k: tuple(d[f"r{j}"][i] for j in range(n)) for i, k in enumerate(d["k"])}


def _forms(rs, flags, start):
    s, lit = P.col("s"), P.lit_utf8
    count = P.fn("regexp_count", s, lit(rs), P.lit_i64(1), lit(flags)) if flags else P.fn("regexp_count", s, lit(rs))
    count_from = P.fn("regexp_count", s, lit(rs), P.lit_i64(start), lit(flags)) if flags else P.fn("regexp_count", s, lit(rs), P.lit_i64(start))
    rep_g = P.fn("regexp_replace", s, lit(rs), lit(REPL), lit(flags + "g"))
    rep_1 = P.fn("regexp_replace", s, lit(rs), lit(REPL), lit(flags)) if flags else P.fn("regexp_replace", s, lit(rs), lit(REPL))
    return [count, count_from, rep_g, rep_1]


def _reference(rx, s, start):
    sp = TF.spans(rx, s)
    counts = (0, 0) if s == "" else (len(sp), len(TF.spans(rx, s[start - 1:])))   # regexp_count of '' is 0
    return counts + (TF.replaced(s, sp, REPL, True), TF.replaced(s, sp, REPL, False))


@pytest.mark.gpu
def test_corpus_on_device_matches_the_reference(gpu, tmp_path):
    # the corpus subjects go up to 4.5 KB; 70 KB rows are test_long_rows' (a forward walk runs until its DFA dies, so a
    # pattern such as `.*x` costs O(n) per match: quadratic in the row over many matches, on the host reference too)
    vals = _values(long_rows=False)
    _register(gpu, _table(vals))
    native = os.path.join(str(tmp_path), "span_check")
    import subprocess
    subprocess.run(["g++", "-O2", "-std=c++17", os.path.join(HERE, "native", "regex_span_check.cpp"), "-o", native], check=True)
    pats = RC.corpus()
    subs = [v or "" for v in vals]
    host = TF.run_native(native, subs, [(f, rs) for rs, f, _p, _l in pats], str(tmp_path))
    ran = by_host = 0
    for i, ((rs, flags, ps, long_ok), h) in enumerate(zip(pats, host)):
        if h[0] != 0:
            continue
        start = 2 + i % 2
        got = _rows(_run(gpu, _project(_forms(rs, flags, start)), f"rfn{i}"), 4)
        excluded = TF.empty_repetition(ps, flags)
        rx = re.compile(ps, RC.python_flags(flags))
        for k, v in enumerate(vals):
            g = got[k]
            if v is None:
                assert g == (0, 0, None, None), (rs, g)
                continue
            if excluded or (len(v) > 300 and not long_ok):
                # the host walk, which tests/test_regex_fn.py holds to the reference (the reference leaves these patterns
                # out, or would backtrack for long over a long row): counts and the replaced strings' CRC-32 and length
                hr = h[1][k]
                assert g[0] == hr[2], (rs, flags, v[:40], g[0], hr)
                for j, (crc, ln) in ((2, hr[5:7]), (3, hr[7:9])):
                    b = g[j].encode()
                    assert (zlib.crc32(b), len(b)) == (crc, ln), (rs, flags, v[:40], j)
                if start == 2:
                    assert g[1] == hr[3], (rs, flags, v[:40])
                by_host += 1
                continue
            assert g == _reference(rx, v, start), (rs, flags, v[:60], g, _reference(rx, v, start))
        ran += 1
    assert ran >= 200 and by_host > 0


@pytest.mark.gpu
def test_long_rows(gpu):
    vals = _values()
    assert sum(len(v.encode()) >= 70 * 1024 for v in vals if v) == 2
    _register(gpu, _table(vals))
    for i, (p, flags) in enumerate([("a", ""), ("[0-9]+", ""), ("é|ж", ""), ("k+?", "i"), ("^a", ""), ("x*", ""), ("z$", ""),
                                    ("(ab|a)c?", ""), (".", "s"), ("[^a-z]{2}", "")]):
        got = _rows(_run(gpu, _project(_forms(p, flags, 3)), f"long{i}"), 4)
        rx = re.compile(p.replace("$", "\\Z"), RC.python_flags(flags))
        for k, v in enumerate(vals):
            assert got[k] == ((0, 0, None, None) if v is None else _reference(rx, v, 3)), (p, k)


@pytest.mark.gpu
def test_pinned_cases_on_device(gpu):
    subs = sorted({c[2] for c in TF.PINNED}) + [None]
    _register(gpu, _table(subs), parts=1)
    for j, (flags, p, s, sp, rg, r1) in enumerate(TF.PINNED):
        lit = P.lit_utf8
        exprs = [P.fn("regexp_count", P.col("s"), lit(p), P.lit_i64(1), lit(flags or "")),
                 P.fn("regexp_replace", P.col("s"), lit(p), lit("X"), lit(flags + "g")),
                 P.fn("regexp_replace", P.col("s"), lit(p), lit("X"), lit(flags))]
        got = _rows(_run(gpu, _project(exprs), f"pin{j}"), 3)
        # regexp_count of an empty pattern or an empty str is 0 (§6 (xiii)); the spans of the table are regexp_replace's
        assert got[subs.index(s)] == (len(sp) if p and s else 0, rg, r1), (p, s, got[subs.index(s)])
        assert got[len(subs) - 1] == (0, None, None)


@pytest.mark.gpu
def test_null_and_empty_arguments(gpu):
    vals = ["", "abc", None, "aaa"]
    _register(gpu, _table(vals), parts=1)
    s, lit = P.col("s"), P.lit_utf8
    exprs = [P.fn("regexp_count", s, lit("")), P.fn("regexp_count", s, lit(None)), P.fn("regexp_count", s, lit("a*")),
             P.fn("regexp_count", s, lit("a"), P.lit_i64(100)), P.fn("regexp_count", s, lit("x*"), P.lit_i64(100)),
             P.fn("regexp_replace", s, lit(""), lit("X"), lit("g")), P.fn("regexp_replace", s, lit(None), lit("X")),
             P.fn("regexp_replace", s, lit("a"), lit(None)), P.fn("regexp_replace", s, lit("a"), lit("X"), lit(None)),
             P.fn("regexp_count", lit(None), lit("a")), P.fn("regexp_replace", s, lit("a"), lit(""), lit("g"))]
    got = _rows(_run(gpu, _project(exprs), "nulls"), len(exprs))
    assert got[0] == (0, 0, 0, 0, 0, "X", None, None, None, 0, "")   # an empty str counts 0, whatever the start
    assert got[1] == (0, 0, 3, 0, 1, "XaXbXcX", None, None, None, 0, "bc")
    assert got[2] == (0, 0, 0, 0, 0, None, None, None, None, 0, None)
    assert got[3] == (0, 0, 1, 0, 1, "XaXaXaX", None, None, None, 0, "")


@pytest.mark.gpu
def test_count_as_a_filter(gpu):
    vals = _values()
    _register(gpu, _table(vals))
    for j, (p, flags) in enumerate([("a", ""), ("[0-9]+", ""), ("k.", "i"), ("^.", "s")]):
        args = [P.col("s"), P.lit_utf8(p)] + ([P.lit_i64(1), P.lit_utf8(flags)] if flags else [])
        pred = P.binop(">", P.fn("regexp_count", *args), P.lit_i64(1))
        st = [P.Stage(1, P.shuffle_writer(P.filter_(pred, P.scan("t", SCH), projection=[0]), 1))]
        out = _run(gpu, st, f"cf{j}")
        got = set(out.to_pydict()["k"]) if out is not None else set()
        rx = re.compile(p, RC.python_flags(flags))
        assert got == {k for k, v in enumerate(vals) if v is not None and len(TF.spans(rx, v)) > 1}, p


@pytest.mark.gpu
def test_replacement_outgrowing_the_first_arena_is_rerun(gpu):
    vals = _values()
    _register(gpu, _table(vals))
    big = "R" * 1500   # the bound len + (len + 1) * 1500 is far above the first arena, so the launch starts from a guess
    r0 = gpu.counter("string_arena_retries")
    got = _rows(_run(gpu, _project([P.fn("regexp_replace", P.col("s"), P.lit_utf8("a|é"), P.lit_utf8(big), P.lit_utf8("g"))]), "grow"), 1)
    assert gpu.counter("string_arena_retries") > r0
    rx = re.compile("a|é")
    for k, v in enumerate(vals):
        assert got[k][0] == (None if v is None else TF.replaced(v, TF.spans(rx, v), big, True)), k


@pytest.mark.gpu
def test_protobuf_stages_give_the_ir_results(gpu):
    with open(os.path.join(HERE, "golden", "regex_fn_proto_plans.json")) as fh:
        cases = [c for c in json.load(fh)["cases"] if "code" not in c]
    _register(gpu, _table(_values()[:3000]), parts=1)   # the decoded scan has one file group: one input partition
    for j, c in enumerate(cases):
        want_stage = json.loads(c["ir"])
        qse = gpu.create_query_stage_exec_proto(f"pb{j}", 1, base64.b64decode(c["proto_b64"]))
        qse.execute_query_stage(0)
        qse.release()
        got = pa.Table.from_batches([gpu.partition_export(f"pb{j}", 1, 0)]) if gpu.partition_rows(f"pb{j}", 1, 0) >= 0 else None
        gpu.remove_job_data(f"pb{j}")
        want = _run(gpu, [P.Stage(1, want_stage)], f"ir{j}")
        if want is None or got is None:
            assert (got is None or got.num_rows == 0) and (want is None or want.num_rows == 0), c["name"]
        else:
            assert_tables_equal(got, want, sort=True, check_names=False)


def _rewrite_like(node, fn):
    if isinstance(node, list):
        return [_rewrite_like(x, fn) for x in node]
    if not isinstance(node, dict):
        return node
    if "like" in node and "pattern" in node:
        return fn(node)
    return {k: _rewrite_like(v, fn) for k, v in node.items()}


@pytest.mark.gpu
def test_tpch_q13_with_regexp_count_equals_the_oracle(gpu, oracle, oracle_lib):
    msf = 100
    for e in (gpu, oracle):
        for table, cols in tpch.Q13_TABLES.items():
            n = oracle_lib.lib().oracle_tpch_table_rows(table.encode(), msf)
            step = (n + 2) // 3
            for p in range(3):
                e.tpch_generate(table, msf, p, min(n, p * step), min(n, (p + 1) * step), cols)
    base = tpch.q13(4)
    want = driver.run_stages(oracle, base, "q13o")
    assert want.num_rows > 1
    seen = []

    def to_count(n):
        assert n["pattern"] == "%special%requests%" and n["negated"]
        seen.append(1)
        return P.binop("=", P.fn("regexp_count", n["like"], P.lit_utf8("special.*requests")), P.lit_i64(0))
    stages = [P.Stage(st.stage_id, _rewrite_like(st.plan, to_count), st.n_tasks) for st in base]
    got = driver.run_stages(gpu, stages, "q13count")
    assert seen
    assert_tables_equal(got, want, sort=False)
