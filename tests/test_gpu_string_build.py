"""GPU: the string builders (concat, ||, concat_ws, repeat, reverse, CAST(x AS Utf8)) writing into the launch's character
arena.  Every expression of tests/string_build_cases.py must equal the restatement byte for byte after export as a
projection, a filter, a group key, a MIN / MAX argument, a hash-join key, a sort key and the output of a hash shuffle writer
(P = 4) read back by a second stage.  A repeat whose column count defeats the first arena is re-run (string_arena_retries)
with the same results; a row over 2^31 - 1 bytes fails naming repeat; TPC-H customer / orders projections match the
restatement and, for the signed-integer casts, the CPU oracle; the fused and group-by fast paths never take these programs.
Also: a builder behind CASE over an arena-overflowing repeat converges on re-runs, a bound far above the need behind a
filter starts small, invalid UTF-8 reverses without touching its neighbours, and a sound bound adds no host wait."""
import collections

import pyarrow as pa
import pytest

import string_build_cases as S
from ballista_b200 import driver
from ballista_b200 import plan as P

pytestmark = pytest.mark.gpu
c = P.col
EXECUTION, UNSUPPORTED = -3, -2


def _register(e, t, name="x", parts=2):
    e.drop_table(name)
    step = (t.num_rows + parts - 1) // parts
    for p in range(parts):
        e.register_batch(name, p, t.slice(p * step, step).combine_chunks().to_batches()[0])


def _run(gpu, stages, job):
    out = driver.run_stages(gpu, stages, job)
    gpu.remove_job_data(job)
    return out


def _by_k(tbl, col="r"):
    d = tbl.to_pydict()
    return dict(zip(d["k"], d[col]))


@pytest.fixture()
def edge(gpu):
    t = S.edge_table()
    _register(gpu, t)
    return t


def _cases():
    return [(name, e, rule) for name, e, rule in S.projections()]


@pytest.mark.parametrize("name,e,rule", _cases(), ids=[x[0] for x in _cases()])
def test_projection_and_filter(gpu, edge, name, e, rule):
    want = S.expected(edge, rule)
    scan = P.scan("x", S.SCHEMA)
    f0, g0 = gpu.counter("fused"), gpu.counter("groupby")
    got = _by_k(_run(gpu, [P.Stage(1, P.shuffle_writer(P.project([(c("k"), "k"), (e, "r")], scan), 1))], f"p-{name}"))
    assert [got[k] for k in range(edge.num_rows)] == want, name
    pred = P.binop("<>", e, P.lit_utf8(""))
    kept = _run(gpu, [P.Stage(1, P.shuffle_writer(P.filter_(pred, scan, projection=[0]), 1))], f"f-{name}")
    kept = set() if kept is None else set(kept.column("k").to_pylist())
    assert kept == {k for k, w in enumerate(want) if w}, name
    assert (gpu.counter("fused"), gpu.counter("groupby")) == (f0, g0)


@pytest.mark.parametrize("name", ["concat_ab", "pipe3", "concat_ws", "repeat_col", "reverse", "cast_dec", "cast_u64", "cast_date"])
def test_group_key_min_max_and_shuffle(gpu, edge, name):
    e, rule = next((x[1], x[2]) for x in _cases() if x[0] == name)
    want = S.expected(edge, rule)
    scan = P.scan("x", S.SCHEMA)
    # group key: Partial -> hash shuffle (P = 4) -> FinalPartitioned
    part = P.aggregate("Partial", [(e, "g")], [P.agg("count", None, "n")], scan)
    fields = [P.field("g", "utf8", True), P.field("n[count]", "i64", True)]
    fin = P.aggregate("FinalPartitioned", [(c(0), "g")], [P.agg("count", c(1), "n")], P.shuffle_reader(1, fields))
    got = _run(gpu, [P.Stage(1, P.shuffle_writer(part, 1, [c(0)], 4)), P.Stage(2, P.shuffle_writer(fin, 2))], f"g-{name}").to_pydict()
    assert dict(zip(got["g"], got["n"])) == dict(collections.Counter(want))
    # MIN / MAX arguments, grouped
    _register(gpu, edge, parts=1)
    mm = P.aggregate("Single", [(P.binop("%", c("k"), P.lit_i32(3)), "m")], [P.agg("min", e, "lo"), P.agg("max", e, "hi")], scan)
    got = _run(gpu, [P.Stage(1, P.shuffle_writer(mm, 1))], f"mm-{name}").to_pydict()
    for m, lo, hi in zip(got["m"], got["lo"], got["hi"]):
        vals = [w for k, w in enumerate(want) if k % 3 == m and w is not None]
        assert (lo, hi) == ((min(vals), max(vals)) if vals else (None, None)), m
    # the output of a hash shuffle writer (P = 4), read back by a second stage
    st1 = P.Stage(1, P.shuffle_writer(P.project([(c("k"), "k"), (e, "r")], scan), 1, [c(1)], 4))
    st2 = P.Stage(2, P.shuffle_writer(P.shuffle_reader(1, [P.field("k", "i32", False), P.field("r", "utf8", True)]), 2))
    got = _by_k(_run(gpu, [st1, st2], f"s-{name}"))
    assert [got[k] for k in range(edge.num_rows)] == want


@pytest.mark.parametrize("name", ["concat_lits", "pipe", "concat_ws_lit", "repeat_lit", "cast_i64", "cast_date", "cast_bool"])
def test_join_and_sort_keys(gpu, edge, name):
    e, rule = next((x[1], x[2]) for x in _cases() if x[0] == name)
    want = S.expected(edge, rule)
    uniq = sorted({w for w in want if w is not None})
    _register(gpu, pa.table({"s": pa.array(uniq, pa.string()), "i": pa.array(range(len(uniq)), pa.int32())}), "y", parts=1)
    scan = P.scan("x", S.SCHEMA)
    right = P.scan("y", [P.field("s", "utf8", False), P.field("i", "i32", False)])
    j = P.hash_join(P.project([(c("k"), "k"), (e, "r")], scan), right, [[c(1), c(0)]])
    got = _run(gpu, [P.Stage(1, P.shuffle_writer(j, 1))], f"j-{name}").to_pydict()
    assert sorted(zip(got["k"], got["i"])) == sorted((k, uniq.index(w)) for k, w in enumerate(want) if w is not None)
    srt = P.sort([P.sort_key(e, True, True), P.sort_key(c("k"))], scan)
    st = P.Stage(1, P.shuffle_writer(P.project([(c("k"), "k"), (e, "r")], srt), 1), n_tasks=1)
    _register(gpu, edge, parts=1)
    got = _run(gpu, [st], f"o-{name}").column("r").to_pylist()
    assert got == [None] * sum(w is None for w in want) + sorted(w for w in want if w is not None)


def test_column_repeat_count_defeats_the_first_arena(gpu):
    n = 3000
    t = pa.table({"k": pa.array(range(n), pa.int32()), "s": pa.array(["abc" if i % 7 else None for i in range(n)], pa.string()),
                  "n": pa.array([500 + i % 5 for i in range(n)], pa.int64())})
    _register(gpu, t, parts=1)
    sch = [P.field("k", "i32", False), P.field("s", "utf8", True), P.field("n", "i64", False)]
    e = P.fn("concat", P.fn("repeat", c("s"), c("n")), P.lit_utf8("|"))
    r0 = gpu.counter("string_arena_retries")
    got = _by_k(_run(gpu, [P.Stage(1, P.shuffle_writer(P.project([(c("k"), "k"), (e, "r")], P.scan("x", sch)), 1))], "retry"))
    assert gpu.counter("string_arena_retries") > r0
    assert [got[k] for k in range(n)] == [S.concat(S.repeat(s, m), "|") for s, m in zip(t.column("s").to_pylist(), t.column("n").to_pylist())]
    # the same as a group key: the aggregate is re-run on a fresh table
    r1 = gpu.counter("string_arena_retries")
    part = P.aggregate("Single", [(e, "g")], [P.agg("count", None, "c")], P.scan("x", sch))
    got = _run(gpu, [P.Stage(1, P.shuffle_writer(part, 1))], "retry-agg").to_pydict()
    assert gpu.counter("string_arena_retries") > r1
    want = collections.Counter(S.concat(S.repeat(s, m), "|") for s, m in zip(t.column("s").to_pylist(), t.column("n").to_pylist()))
    assert dict(zip(got["g"], got["c"])) == dict(want)


def test_row_longer_than_2_pow_31_fails_naming_repeat(gpu):
    import ballista_b200 as bb
    t = pa.table({"k": pa.array([0, 1], pa.int32()), "s": pa.array(["ab", "c"]), "n": pa.array([2**30, 1], pa.int64())})
    _register(gpu, t, parts=1)
    sch = [P.field("k", "i32", False), P.field("s", "utf8", False), P.field("n", "i64", False)]
    st = [P.Stage(1, P.shuffle_writer(P.project([(P.fn("repeat", c("s"), c("n")), "r")], P.scan("x", sch)), 1))]
    with pytest.raises(bb.engine.B200Error) as ei:
        _run(gpu, st, "toolong")
    assert ei.value.code == EXECUTION and "repeat" in str(ei.value)


@pytest.mark.parametrize("typ,culprit", [("f64", "f64"), ("f32", "f32"), ("ts", "ts"), (P.dec(10, -2), "-2")])
def test_cast_refusals_name_the_source_type(gpu, typ, culprit):
    import ballista_b200 as bb
    t = pa.table({"k": pa.array([0, 1], pa.int64())})
    _register(gpu, t, parts=1)
    sch = [P.field("k", "i64", False)]
    st = [P.Stage(1, P.shuffle_writer(P.project([(P.cast(P.cast(c("k"), typ), "utf8"), "r")], P.scan("x", sch)), 1))]
    with pytest.raises(bb.engine.B200Error) as ei:
        _run(gpu, st, "refuse")
    assert ei.value.code == UNSUPPORTED and culprit in str(ei.value) and "Utf8" in str(ei.value), str(ei.value)


def test_tpch_customer_and_orders(gpu, oracle, oracle_lib):
    from ballista_b200 import tpch
    msf = 10
    for e in (gpu, oracle):
        for tname, cols in (("customer", ["c_custkey", "c_name"]), ("orders", ["o_orderkey", "o_totalprice", "o_orderdate"])):
            e.drop_table(tname)
            n = oracle_lib.lib().oracle_tpch_table_rows(tname.encode(), msf)
            for p in range(2):
                e.tpch_generate(tname, msf, p, min(n, p * ((n + 1) // 2)), min(n, (p + 1) * ((n + 1) // 2)), cols)
    cust = tpch.table_scan("customer", ["c_custkey", "c_name"])
    e = P.fn("concat", c("c_name"), P.lit_utf8("-"), P.cast(c("c_custkey"), "utf8"))
    st = [P.Stage(1, P.shuffle_writer(P.project([(c("c_custkey"), "k"), (e, "r"), (P.cast(c("c_custkey"), "utf8"), "ks")], cust), 1))]
    got = _run(gpu, st, "tpch-c").to_pydict()
    src = {}
    for p in range(2):
        b = gpu.export_table("customer", p).to_pydict()
        src.update(zip(b["c_custkey"], b["c_name"]))
    assert len(got["k"]) == len(src) > 0
    for k, r in zip(got["k"], got["r"]):
        assert r == S.concat(src[k], "-", str(k))
    want = driver.run_stages(oracle, [P.Stage(1, P.shuffle_writer(P.project([(c("c_custkey"), "k"), (P.cast(c("c_custkey"), "utf8"), "ks")], cust), 1))], "tpch-co")
    assert dict(zip(got["k"], got["ks"])) == dict(zip(want.column("k").to_pylist(), want.column("ks").to_pylist()))
    orders = tpch.table_scan("orders", ["o_orderkey", "o_totalprice", "o_orderdate"])
    st = [P.Stage(1, P.shuffle_writer(P.project([(c("o_orderkey"), "k"), (P.cast(c("o_totalprice"), "utf8"), "r"),
                                                 (P.cast(c("o_orderdate"), "utf8"), "d")], orders), 1))]
    got = _run(gpu, st, "tpch-o").to_pydict()
    src = {}
    for p in range(2):
        b = gpu.export_table("orders", p)
        scale = b.schema.field("o_totalprice").type.scale
        d = b.to_pydict()
        for k, v, dt in zip(d["o_orderkey"], d["o_totalprice"], d["o_orderdate"]):
            src[k] = (S.cast_decimal(S._unscaled(v, scale), scale), S.cast_date(S._days(dt)))
    assert len(got["k"]) == len(src) > 0
    for k, r, d in zip(got["k"], got["r"], got["d"]):
        assert (r, d) == src[k]


def _reverse_bytes(b):
    """the device's reverse over arbitrary bytes: UTF-8 sequences kept whole, a sequence cut short by the end as it is"""
    out, i = [], 0
    while i < len(b):
        c0 = b[i]
        k = 1 if c0 < 0x80 else 2 if c0 >> 5 == 6 else 3 if c0 >> 4 == 14 else 4
        k = min(k, len(b) - i)
        out.insert(0, b[i:i + k])
        i += k
    return b"".join(out)


def test_reverse_of_invalid_utf8_stays_in_its_row(gpu):
    raw = [b"abc", b"\x80", b"ab\xe2", b"\xf0\x9d", b"\xc3", b"xy\xe2\x82", "日本".encode(), b"\x80\x80z", b"tail"] * 40
    t = pa.table({"k": pa.array(range(len(raw)), pa.int32()), "s": pa.array(raw, pa.binary()).view(pa.string())})
    _register(gpu, t, parts=1)
    sch = [P.field("k", "i32", False), P.field("s", "utf8", False)]
    e = P.fn("concat", P.lit_utf8("<"), P.fn("reverse", c("s")), P.lit_utf8(">"))
    got = _run(gpu, [P.Stage(1, P.shuffle_writer(P.project([(c("k"), "k"), (e, "r")], P.scan("x", sch)), 1))], "rev-invalid")
    got = dict(zip(got.column("k").to_pylist(), got.column("r").cast(pa.binary()).to_pylist()))
    assert [got[k] for k in range(len(raw))] == [b"<" + _reverse_bytes(b) + b">" for b in raw]


def test_case_over_an_overflowing_builder_converges(gpu):
    n = 2000
    t = pa.table({"k": pa.array(range(n), pa.int32()), "s": pa.array(["xyz" if i % 5 else None for i in range(n)], pa.string()),
                  "n": pa.array([300 + i % 7 for i in range(n)], pa.int64())})
    _register(gpu, t, parts=1)
    sch = [P.field("k", "i32", False), P.field("s", "utf8", True), P.field("n", "i64", False)]
    even = P.binop("=", P.binop("%", c("k"), P.lit_i32(2)), P.lit_i32(0))
    e = P.fn("concat", P.case([[even, P.fn("repeat", c("s"), c("n"))]]), P.lit_utf8("|"))
    r0 = gpu.counter("string_arena_retries")
    got = _by_k(_run(gpu, [P.Stage(1, P.shuffle_writer(P.project([(c("k"), "k"), (e, "r")], P.scan("x", sch)), 1))], "case-retry"))
    assert gpu.counter("string_arena_retries") > r0
    rows = zip(t.column("k").to_pylist(), t.column("s").to_pylist(), t.column("n").to_pylist())
    assert [got[k] for k in range(n)] == [S.concat(S.repeat(s, m) if k % 2 == 0 else None, "|") for k, s, m in rows]


def test_bound_far_above_the_need_starts_small(gpu, edge):
    """repeat(a, 100000) over every row would be gigabytes; the filter keeps one row of 'a', so 100 kB are needed"""
    e = P.fn("repeat", c("a"), P.lit_i64(100000))
    pred = P.binop("=", c("k"), P.lit_i32(2))
    node = P.project([(c("k"), "k"), (e, "r")], P.filter_(pred, P.scan("x", S.SCHEMA)))
    got = _run(gpu, [P.Stage(1, P.shuffle_writer(node, 1))], "big-bound").to_pydict()
    assert got == {"k": [2], "r": ["a" * 100000]}


def test_sound_bound_adds_no_host_wait(gpu, edge):
    """an unfiltered projection whose builders have a sound bound waits no more than one that makes string views without
    building bytes (btrim); one with a column repeat count (no bound) waits for the arena's need"""
    scan = P.scan("x", S.SCHEMA)

    def waits(e, job):
        st = [P.Stage(1, P.shuffle_writer(P.project([(c("k"), "k"), (e, "r")], scan), 1))]
        _run(gpu, st, job + "-warm")
        s0 = gpu.counter("host_syncs")
        _run(gpu, st, job)
        return gpu.counter("host_syncs") - s0

    sound = waits(P.fn("concat", P.cast(c("i64"), "utf8"), P.lit_utf8("-"), c("a")), "w-sound")
    assert sound <= waits(P.fn("btrim", c("a")), "w-plain")
    assert waits(P.fn("repeat", c("a"), c("n")), "w-unbounded") > sound
