"""GPU: ILIKE, the regex operators and regexp_like as device stages (OP_REGEX over the DFA the host compiled).  The corpus of
tests/regex_cases.py runs as ProjectionExec stages (the Bool with its NULLs) and FilterExec stages and must equal Python's
re.search bit for bit; the protobuf fixtures give the results of their IR; TPC-H q13 / q9 with the LIKE node rewritten into
the equivalent regex or ILIKE give the LIKE results; warm stages compile nothing; refused patterns store nothing."""
import base64
import json
import os

import pyarrow as pa
import pytest

import regex_cases as RC
from ballista_b200 import driver, engine, tpch
from ballista_b200 import plan as P
from util import assert_tables_equal

HERE = os.path.dirname(os.path.abspath(__file__))
SCH = [P.field("k", "i32", False), P.field("s", "utf8", True), P.field("t", "utf8", True)]


def _table():
    subs = RC.subjects()
    vals = [None if i % 97 == 5 else s for i, s in enumerate(subs)]   # NULL rows
    return vals, pa.table({"k": pa.array(range(len(vals)), pa.int32()), "s": pa.array(vals, pa.string()),
                           "t": pa.array(["x"] * len(vals), pa.string())})


def _register(e, t, parts=2):
    e.drop_table("t")
    step = (t.num_rows + parts - 1) // parts
    for p in range(parts):
        e.register_batch("t", p, t.slice(p * step, step).combine_chunks().to_batches()[0])


def _stage(pred, filt):
    scan = P.scan("t", SCH)
    node = P.filter_(pred, scan, projection=[0]) if filt else P.project([(P.col("k"), "k"), (pred, "r")], scan)
    return [P.Stage(1, P.shuffle_writer(node, 1))]


def _run(gpu, stages, job):
    out = driver.run_stages(gpu, stages, job)
    gpu.remove_job_data(job)
    return out


def _by_k(tbl):
    if tbl is None:   # a filter that kept nothing
        return set()
    d = tbl.to_pydict()
    return dict(zip(d["k"], d["r"])) if "r" in d else set(d["k"])


def _expr(i, rs, flags):
    """the i-th pattern as one of the regex forms (flags through regexp_like or ~*)"""
    s = P.col("s")
    if flags == "i" and i % 2:
        return P.regex_match(s, rs, case_insensitive=True), False
    if flags:
        return P.fn("regexp_like", s, P.lit_utf8(rs), P.lit_utf8(flags)), False
    if i % 3 == 0:
        return P.fn("regexp_like", s, P.lit_utf8(rs)), False
    if i % 3 == 1:
        return P.regex_match(s, rs, negated=True), True
    return P.regex_match(s, rs), False


@pytest.mark.gpu
def test_corpus_on_device_matches_python_re(gpu, tmp_path):
    vals, t = _table()
    _register(gpu, t)
    native = RC.build_native(str(tmp_path))
    pats = RC.corpus()
    res = RC.run_native(native, [], [("r", f, rs) for rs, f, _p, _l in pats], str(tmp_path))
    ran = 0
    for i, ((rs, flags, ps, long_ok), r) in enumerate(zip(pats, res)):
        if r[0] != 0:
            continue
        e, neg = _expr(i, rs, flags)
        want = RC.expected(ps, flags, [v or "" for v in vals], long_ok)
        want = [None if v is None else (w if w is None else w != neg) for v, w in zip(vals, want)]
        got = _by_k(_run(gpu, _stage(e, False), f"rxp{i}"))
        for k, w in enumerate(want):
            if w is None and vals[k] is not None:
                continue   # a long subject the Python reference skips (backtracking cost)
            assert got[k] == w, (rs, flags, neg, vals[k], got[k], w)
        kept = _by_k(_run(gpu, _stage(e, True), f"rxf{i}"))
        assert {k for k in kept if want[k] is not None} == {k for k, w in enumerate(want) if w}, rs
        ran += 1
    assert ran >= 200


@pytest.mark.gpu
def test_ilike_and_pinned_rules_on_device(gpu):
    import test_regex as TR
    subs = sorted({p[3] for p in TR.PINNED if p[4] is not None})
    t = pa.table({"k": pa.array(range(len(subs)), pa.int32()), "s": pa.array(subs), "t": pa.array(subs)})
    _register(gpu, t, parts=1)
    for j, (kind, flags, p, s, want) in enumerate(TR.PINNED):
        if want is None:
            continue
        s_col = P.col("s")
        e = P.like(s_col, p, case_insensitive=True) if kind == "l" else P.fn("regexp_like", s_col, P.lit_utf8(p), P.lit_utf8(flags)) if flags else P.regex_match(s_col, p)
        got = _by_k(_run(gpu, _stage(e, False), f"pin{j}"))
        assert got[subs.index(s)] == want, (kind, flags, p, s)


@pytest.mark.gpu
def test_null_pattern_and_null_rows(gpu):
    vals, t = _table()
    _register(gpu, t)
    for j, e in enumerate([P.regex_match(P.col("s"), P.lit_utf8(None)), P.fn("regexp_like", P.col("s"), P.lit_utf8("a"), P.lit_utf8(None)),
                           P.like(P.col("s"), "%a%", negated=True, case_insensitive=True)]):
        got = _by_k(_run(gpu, _stage(e, False), f"null{j}"))
        for k, v in enumerate(vals):
            if v is None or j < 2:
                assert got[k] is None
            else:
                assert got[k] == ("a" not in v.lower())
        assert _by_k(_run(gpu, _stage(e, True), f"nullf{j}")) == ({k for k, v in enumerate(vals) if v is not None and "a" not in v.lower()} if j == 2 else set())


@pytest.mark.gpu
def test_protobuf_stages_give_the_ir_results(gpu):
    with open(os.path.join(HERE, "golden", "regex_proto_plans.json")) as fh:
        cases = [c for c in json.load(fh)["cases"] if "code" not in c]
    _vals, t = _table()
    _register(gpu, t, parts=1)   # the decoded scan has one file group: one input partition
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


def _rewritten(stages, fn):
    return [P.Stage(st.stage_id, _rewrite_like(st.plan, fn), st.n_tasks) for st in stages]


@pytest.mark.gpu
def test_tpch_q13_with_a_regex_equals_not_like(gpu):
    gpu.tpch_load(tpch.Q13_TABLES, 100, parts=3)
    base = tpch.q13(4, "%q%z%")
    want = driver.run_stages(gpu, base, "q13like")
    assert want.num_rows > 1
    seen = []

    def to_regex(n):
        assert n["pattern"] == "%q%z%" and n["negated"]
        seen.append(1)
        return P.regex_match(n["like"], "q.*z", negated=True)
    got = driver.run_stages(gpu, _rewritten(base, to_regex), "q13rx")
    assert seen
    assert_tables_equal(got, want, sort=False)


@pytest.mark.gpu
def test_tpch_q9_with_ilike_and_regex_equals_like(gpu):
    gpu.tpch_load(tpch.Q9_TABLES, 50, parts=2)
    base = tpch.q9(3, "%z%")
    want = driver.run_stages(gpu, base, "q9like")
    assert want.num_rows > 5
    ilike = _rewritten(base, lambda n: P.like(n["like"], "%Z%", negated=n["negated"], case_insensitive=True))
    regex = _rewritten(base, lambda n: P.regex_match(n["like"], "z", negated=n["negated"]))
    assert "case_insensitive" in json.dumps([s.plan for s in ilike])
    assert_tables_equal(driver.run_stages(gpu, ilike, "q9ilike"), want, sort=False)
    assert_tables_equal(driver.run_stages(gpu, regex, "q9rx"), want, sort=False)


@pytest.mark.gpu
def test_warm_stage_compiles_nothing(gpu):
    _vals, t = _table()
    _register(gpu, t)
    pat = "^[a-f]{2}(ab|cd)+ unique-to-this-test"
    st = _stage(P.regex_match(P.col("s"), pat), False)
    c0 = gpu.counter("regex_compiles")
    first = _run(gpu, st, "warm1")
    c1 = gpu.counter("regex_compiles")
    assert c1 == c0 + 1
    qse = gpu.create_query_stage_exec("warm2", 1, st[0].json("warm2"))
    for p in range(2):
        qse.execute_query_stage(p)
    for p in range(2):
        qse.execute_query_stage(p)   # a second execution of the prepared stage
    qse.release()
    gpu.remove_job_data("warm2")
    assert gpu.counter("regex_compiles") == c1
    again = _run(gpu, st, "warm3")
    assert gpu.counter("regex_compiles") == c1
    assert_tables_equal(first, again, sort=True)


@pytest.mark.gpu
def test_refused_pattern_fails_at_prepare_and_stores_nothing(gpu):
    _vals, t = _table()
    _register(gpu, t)
    for j, (e, code) in enumerate([(P.regex_match(P.col("s"), "\\bx"), -2), (P.regex_match(P.col("s"), "(a"), -1),
                                   (P.like(P.col("s"), "%ü%", case_insensitive=True), -2)]):
        c0 = gpu.counter("regex_compiles")
        st = _stage(e, False)
        with pytest.raises(engine.B200Error) as ei:
            gpu.create_query_stage_exec(f"bad{j}", 1, st[0].json(f"bad{j}"))
        assert ei.value.code == code
        assert gpu.partition_rows(f"bad{j}", 1, 0) == -1
        assert gpu.counter("regex_compiles") == c0
