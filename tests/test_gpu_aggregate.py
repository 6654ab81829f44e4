"""GPU: AggregateExec on the device against the plain-Python reference of aggregate_cases, not the oracle.  Keys,
integers, decimals and float MIN / MAX are compared bit for bit (NaN payloads and the sign of zero included); float SUM
and AVG within the order-independent bound of aggregate_cases.Approx.

Every case runs in the four modes (Partial -> hash shuffle -> FinalPartitioned with more partitions than groups,
Partial -> Final, Single, SinglePartitioned) and twice, so that the second run starts from the strategy the first one
taught the engine.  The path tests steer run_aggregate onto each of its strategies and prove which one ran with the
engine's counters and kernel statistics."""
import numpy as np
import pyarrow as pa
import pytest

import ballista_b200 as bb
from ballista_b200 import driver
from ballista_b200 import plan as P
import aggregate_cases as A

pytestmark = pytest.mark.gpu
EXECUTION = -3


@pytest.fixture(scope="module")
def arg_table():
    return A.arg_table(4097)


def _twice(gpu, table, mode, keys, aggs, job, **kw):
    for i in range(2):
        A.check(gpu, table, mode, keys, aggs, f"{job}-{i}", **kw)


@pytest.mark.parametrize("mode", A.MODES)
@pytest.mark.parametrize("typ", list(A.TYPES))
def test_arguments(gpu, arg_table, typ, mode):
    """Every argument type in its three forms, 4 groups (the register sink, or the fused kernel for non-nullable
    integer and decimal SUM / COUNT) and the same aggregates without keys."""
    for form in A.FORMS:
        for fns in A.fn_groups(typ):
            aggs = A.arg_aggs(typ, form, fns)
            _twice(gpu, arg_table, mode, ["g"], aggs, f"a-{typ}-{form}-{mode}")
            if mode in ("final", "single"):
                _twice(gpu, arg_table, mode, [], aggs, f"as-{typ}-{form}-{mode}")


@pytest.mark.parametrize("mode", A.MODES)
@pytest.mark.parametrize("typ", ["i64", "u64", "d38_0", "f32", "f64", "utf8", "bool"])
def test_minmax_on_the_global_table(gpu, typ, mode):
    """MIN / MAX over 40 groups: past the register sink's 4, on the global table's per-row atomics (UInt64 operands
    zero-extended into the 128-bit cells)."""
    n = 4097
    table = A.make_table([typ], n, 11, {"g": ("i64", [(i * 7) % 40 for i in range(n)])})
    for form in A.FORMS:
        A.check(gpu, table, mode, ["g"], A.arg_aggs(typ, form, ["count_star", "min", "max"]), f"mm-{typ}-{form}-{mode}")


@pytest.mark.parametrize("n", [0, 1, 1023, 1024, 1025, 4097])
@pytest.mark.parametrize("typ", ["i64", "u64", "f32", "f64", "d20_3", "d38_10", "utf8"])
def test_row_counts(gpu, arg_table, typ, n):
    t = arg_table.slice(0, n)
    for mode in A.MODES:
        for fns in A.fn_groups(typ):
            for form in ("nn", "n"):
                A.check(gpu, t, mode, ["g"], A.arg_aggs(typ, form, fns), f"n-{typ}-{n}-{mode}")
                if mode in ("final", "single"):
                    A.check(gpu, t, mode, [], A.arg_aggs(typ, form, fns), f"ns-{typ}-{n}-{mode}")


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("mode", A.MODES)
@pytest.mark.parametrize("shape", sorted(A.KEY_SHAPES))
def test_keys(gpu, shape, mode, nullable):
    """Keys at their types' edges, alone and in pairs (pack_mode 2 squeezes two narrow keys into 32 bits each, around a
    +2^31 shift), with and without NULLs."""
    table, keys = A.key_table(shape, 3000, seed=len(shape), nullable=nullable)
    _twice(gpu, table, mode, keys, A.KEY_AGGS, f"k-{shape}-{mode}-{nullable}")


@pytest.mark.parametrize("t", ["f32", "f64"])
@pytest.mark.parametrize("groups", [3, 40])
def test_float_keys_group_by_bits(gpu, t, groups):
    """-0.0 and 0.0 are two groups and keep their signs; every NaN payload is a group of its own and comes back with
    its payload -- on the register sink (3 distinct keys) and the global table."""
    dom = (A.F32_EDGES if t == "f32" else A.F64_EDGES)
    zero, neg0 = (0, 0x80000000) if t == "f32" else (0, 1 << 63)
    dom = [zero, neg0, dom[-4]] if groups == 3 else dom
    vals = [dom[i % len(dom)] for i in range(2500)]
    table = A.make_table(["i64"], len(vals), 1, {f"k_{t}": (t, vals)})
    for mode in A.MODES:
        got = A.check(gpu, table, mode, [f"k_{t}"], [("count_star", None, "cnt"), ("sum", "v_i64_nn", "s")], f"fk-{t}-{groups}-{mode}")
        assert sorted(A.raw_values(got.column(0))) == sorted(dom)


def test_float32_signalling_nan(gpu):
    """A Float32 signalling NaN decides MIN or MAX and comes back with its bits; as a key it is not the quiet NaN of the
    same payload."""
    table = A.snan_table()
    for mode in A.MODES:
        A.check(gpu, table, mode, ["g"], A.SNAN_AGGS, f"sn-{mode}")
        got = A.check(gpu, table, mode, ["kf"], [("count_star", None, "c")], f"snk-{mode}")
        assert sorted(A.raw_values(got.column(0))) == [0x7F800001, 0x7FC00001]


def test_colliding_key_hashes(gpu):
    """Two distinct Int64 key pairs with the same 64-bit row hash stay two groups."""
    import hash_join_cases as H
    (a1, b1), (a2, b2) = H.colliding_keys()
    rows = [(a1, b1), (a2, b2), (5, 6)] * 700
    table = A.make_table(["i64"], len(rows), 2, {"a": ("i64", [r[0] for r in rows]), "b": ("i64", [r[1] for r in rows])})
    for mode in A.MODES:
        got = A.check(gpu, table, mode, ["a", "b"], [("count_star", None, "cnt"), ("min", "v_i64_n", "mn")], f"hc-{mode}")
        assert got.num_rows == 3


# ---- paths ----------------------------------------------------------------------------------------------------------
def _paths(gpu, fn):
    """Runs fn(); returns (counter deltas, kernel families launched)."""
    names = ("fused", "vm", "groupby", "groupby_partition_first")
    before = {n: gpu.counter(n) for n in names}
    gpu.set_config("b200.metrics.kernel_timing", "1")
    gpu.kernel_stats(reset=True)
    try:
        fn()
        ks = gpu.kernel_stats(reset=True)
    finally:
        gpu.set_config("b200.metrics.kernel_timing", "0")
    return {n: gpu.counter(n) - before[n] for n in names}, {k for k, v in ks.items() if v["launches"]}


def _big_table(n, groups, seed, last_tile_key=None):
    """n rows: a non-nullable Int64 key with `groups` values (the last row's key replaced by last_tile_key) and a
    non-nullable Int64 value."""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, groups, n).astype(np.int64) * 7919 - 3
    if last_tile_key is not None:
        k[-1] = last_tile_key
    v = rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64)
    return pa.table({"k": pa.array(k), "v": pa.array(v)}), k, v


BIG_SCHEMA = [P.field("k", "i64"), P.field("v", "i64")]
# COUNT and SUM only: the group-by kernel (and the sampling probe that runs on it) takes no MIN / MAX
BIG_AGGS = [("count_star", None, "cnt"), ("sum", "v", "s")]


def _big_reference(k, v):
    """Vectorised reference of BIG_AGGS (wrapping Int64 sums) for millions of rows."""
    u, inv = np.unique(k, return_inverse=True)
    cnt = np.bincount(inv)
    s = np.zeros(len(u), np.int64)
    np.add.at(s, inv, v)
    return {(int(u[i]),): [int(cnt[i]), int(s[i])] for i in range(len(u))}


def _run_big(gpu, table, want, mode, job, parts=1):
    A.register(gpu, table, parts)
    got = driver.run_stages(gpu, A.stages(mode, BIG_SCHEMA, ["k"], BIG_AGGS), job)
    bad = A.mismatches(A.results_of(got, 1), want, [a[2] for a in BIG_AGGS])
    assert not bad, bad


def test_path_fused_and_register_sink(gpu, monkeypatch):
    table = A.arg_table(4097)
    aggs = A.arg_aggs("d15_2", "nn", ["count_star", "count", "sum", "avg"])
    d, fam = _paths(gpu, lambda: A.check(gpu, table, "single", ["g"], aggs, "p-fused"))
    assert d["fused"] >= 1 and "pipeline_fused_agg" in fam, (d, fam)
    monkeypatch.setenv("B200_NO_FUSED", "1")
    d, fam = _paths(gpu, lambda: A.check(gpu, table, "single", ["g"], aggs, "p-reg"))
    assert d["fused"] == 0 and d["vm"] >= 1 and "pipeline_agg_reg" in fam, (d, fam)


def test_path_fifth_group_in_the_last_tile(gpu, monkeypatch):
    """Four groups, then a fifth in the input's last row: the register sink gives up and the global table runs."""
    monkeypatch.setenv("B200_NO_FUSED", "1")
    table, k, v = _big_table(20000, 4, 3, last_tile_key=10 ** 15)
    d, fam = _paths(gpu, lambda: _run_big(gpu, table, _big_reference(k, v), "single", "p-fifth"))
    assert {"pipeline_agg_reg", "pipeline_agg_global"} <= fam or {"pipeline_agg_reg", "groupby_hash_agg"} <= fam, fam
    monkeypatch.setenv("B200_NO_GROUPBY", "1")
    gpu.set_config("b200.agg.reset_hints", "1")
    d, fam = _paths(gpu, lambda: _run_big(gpu, table, _big_reference(k, v), "single", "p-fifth-vm"))
    assert {"pipeline_agg_reg", "pipeline_agg_global"} <= fam, fam


def test_path_groupby_kernel_and_partition_first(gpu, monkeypatch):
    table, k, v = _big_table(300000, 50000, 4)
    want = _big_reference(k, v)
    d, fam = _paths(gpu, lambda: _run_big(gpu, table, want, "single", "p-gb"))
    assert d["groupby"] >= 1 and "groupby_hash_agg" in fam, (d, fam)
    gpu.set_config("b200.agg.partition_first.min_rows", "1000")
    gpu.set_config("b200.agg.partition_first.bucket_slots", "4096")
    try:
        d, fam = _paths(gpu, lambda: _run_big(gpu, table, want, "single", "p-pf"))
        assert d["groupby_partition_first"] >= 1, d
    finally:
        gpu.set_config("b200.agg.partition_first.bucket_slots", str(1 << 19))
        gpu.set_config("b200.agg.partition_first.min_rows", str(1 << 22))
    monkeypatch.setenv("B200_NO_GROUPBY", "1")
    d, fam = _paths(gpu, lambda: _run_big(gpu, table, want, "single", "p-global"))
    assert d["groupby"] == 0 and "pipeline_agg_global" in fam, (d, fam)


@pytest.mark.parametrize("n,groups", [((1 << 20) + 4096, 3), ((1 << 20) + 4096, 200000), ((1 << 22) + 4096, 1500000)])
def test_path_large_inputs(gpu, monkeypatch, n, groups):
    """Over 2^20 rows with no hint the group-by kernel samples 16 K rows first; over 2^22 rows the global table climbs
    its capacity ladder and re-runs on overflow.  Each plan runs twice: the second run starts from the hint."""
    table, k, v = _big_table(n, groups, 5)
    want = _big_reference(k, v)
    d, _fam = _paths(gpu, lambda: _run_big(gpu, table, want, "single", f"big-{n}-{groups}-0"))
    assert d["groupby"] >= 1, d   # the sampling probe (and, for many groups, the group-by kernel after it)
    _run_big(gpu, table, want, "single", f"big-{n}-{groups}-1")
    if groups > 1000:
        monkeypatch.setenv("B200_NO_GROUPBY", "1")
        gpu.set_config("b200.agg.reset_hints", "1")
        d, fam = _paths(gpu, lambda: _run_big(gpu, table, want, "single", f"big-vm-{n}"))
        assert d["groupby"] == 0 and "pipeline_agg_global" in fam, (d, fam)


def test_path_capacity_ladder_reruns(gpu, monkeypatch):
    """> 2^22 rows on the global table (group-by kernel off): the table starts small, overflows and grows."""
    monkeypatch.setenv("B200_NO_GROUPBY", "1")
    monkeypatch.setenv("B200_NO_FUSED", "1")
    table, k, v = _big_table((1 << 22) + 1000, 400000, 6)
    want = _big_reference(k, v)
    gpu.set_config("b200.metrics.kernel_timing", "1")
    gpu.kernel_stats(reset=True)
    try:
        _run_big(gpu, table, want, "single", "ladder")
        ks = gpu.kernel_stats(reset=True)
    finally:
        gpu.set_config("b200.metrics.kernel_timing", "0")
    assert ks["pipeline_agg_global"]["launches"] >= 2, ks   # at least one overflowed table and the re-run


AGG_FAMILIES = ("pipeline_fused_agg", "pipeline_agg_reg", "pipeline_agg_global", "groupby_hash_agg")


def _agg_launches(gpu, fn):
    """Runs fn(); returns how many aggregate kernels it launched."""
    gpu.set_config("b200.metrics.kernel_timing", "1")
    gpu.kernel_stats(reset=True)
    try:
        fn()
        ks = gpu.kernel_stats(reset=True)
    finally:
        gpu.set_config("b200.metrics.kernel_timing", "0")
    return sum(ks.get(f, {}).get("launches", 0) for f in AGG_FAMILIES)


def test_path_pack_overflow_in_the_last_tile(gpu, monkeypatch):
    """String keys of at most 7 bytes pack into an Int64 -- until one of 8 bytes shows up in the last tile.  The packed
    run is abandoned and the aggregate is lowered again with plain string keys: one aggregate launch more than over the
    same keys without the long one."""
    n = 5000
    keys = [("", "a", "a\0", "abc", "abcdefg")[i % 5] for i in range(n)]
    short = A.make_table(["i64", "d15_2"], n, 8, {"s": ("utf8", keys)})
    keys[-1] = "abcdefgh"
    table = A.make_table(["i64", "d15_2"], n, 8, {"s": ("utf8", keys)})
    aggs = [("count_star", None, "cnt"), ("sum", "v_d15_2_nn", "s"), ("max", "v_i64_n", "mx")]
    for prepack in ("", "1"):
        if prepack:
            monkeypatch.setenv("B200_NO_PREPACK", "1")
        gpu.set_config("b200.agg.reset_hints", "1")
        base = _agg_launches(gpu, lambda: A.check(gpu, short, "single", ["s"], aggs, f"pack-short-{prepack}"))
        gpu.set_config("b200.agg.reset_hints", "1")
        relowered = _agg_launches(gpu, lambda: A.check(gpu, table, "single", ["s"], aggs, f"pack-long-{prepack}"))
        assert relowered > base, (base, relowered)
        for mode in A.MODES:
            _twice(gpu, table, mode, ["s"], aggs, f"pack-{mode}-{prepack}")


def test_sibling_task_with_more_groups_than_the_hint(gpu):
    """A plan first run over 3 groups learns a small table; the same plan then runs over a partition of 3 groups and one
    of 50,000, and the second task starts from that hint, overflows it and grows."""
    t0, k0, v0 = _big_table(5000, 3, 9)
    t1, k1, v1 = _big_table(200000, 50000, 10)
    for mode in ("final_partitioned", "final"):
        st = A.stages(mode, BIG_SCHEMA, ["k"], BIG_AGGS)
        gpu.set_config("b200.agg.reset_hints", "1")
        A.register(gpu, t0, 1)
        _run_big(gpu, t0, _big_reference(k0, v0), mode, f"sib-small-{mode}")
        gpu.register_batch("agg_t", 1, t1.combine_chunks().to_batches()[0])
        out = []
        launches = _agg_launches(gpu, lambda: out.append(driver.run_stages(gpu, st[:1], f"sib-partial-{mode}")))
        assert launches >= 3, launches   # task 0 once; task 1 at the hinted size, then again on a larger table
        part = out[0]
        assert sum(part.column(1).to_pylist()) == 205000
        want = _big_reference(np.concatenate([k0, k1]), np.concatenate([v0, v1]))
        got = driver.run_stages(gpu, st, f"sib-{mode}")
        assert not A.mismatches(A.results_of(got, 1), want, [a[2] for a in BIG_AGGS])


# ---- errors ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", A.MODES)
def test_decimal_avg_overflow(gpu, mode):
    """AVG over Decimal(38, 0) -> Decimal(38, 4): 9e33 fits (it was refused by a proxy bound before); 1.5e34 is beyond
    38 digits and 2e34 * 10^4 beyond i128, both execution errors, after which the engine still works."""
    for v in (9 * 10 ** 33, -9 * 10 ** 33, 15 * 10 ** 33, -2 * 10 ** 34):
        for rows in ([v], [v, 0, 0, 1]):
            table = A.make_table([], len(rows), 1, {"k": ("i64", [1] * len(rows)), "x": ("d38_0", rows)})
            aggs = [("avg", "x", "a"), ("count_star", None, "c")]
            try:
                A.reference(table, ["k"], aggs)
            except A.AggOverflow:
                with pytest.raises(bb.B200Error) as e:
                    A.run(gpu, table, mode, ["k"], aggs, f"avgerr-{mode}")
                assert e.value.code == EXECUTION, str(e.value)
                continue
            A.check(gpu, table, mode, ["k"], aggs, f"avgok-{mode}")
    table = A.arg_table(300)
    A.check(gpu, table, mode, ["g"], A.arg_aggs("d38_10", "n", ["count_star", "count", "sum", "avg"]), f"after-{mode}")


def test_window_decimal_avg_overflow(gpu):
    """The window AVG shares the grouped AVG's rule: over Decimal(38, 0), a partition of one 9e33 row averages to 9e33
    as Decimal(38, 4); 1.5e34 is beyond 38 digits and 2e34 * 10^4 beyond i128."""
    sch = [P.field("k", "i64"), P.field("x", P.dec(38, 0))]
    plan = P.window([P.win("avg", "a", [P.col(1)], [P.col(0)])], P.scan("agg_t", sch), [P.col(0)])
    for v in (9 * 10 ** 33, -9 * 10 ** 33, 15 * 10 ** 33, -2 * 10 ** 34):
        for rows in ([v], [v, 0, 0, 1]):
            table = A.make_table([], len(rows), 1, {"k": ("i64", [1] * len(rows)), "x": ("d38_0", rows)})
            A.register(gpu, table, 1)
            try:
                want = A.aggregate_values("avg", "d38_0", rows)
            except A.AggOverflow:
                with pytest.raises(bb.B200Error) as e:
                    driver.run_stages(gpu, [P.Stage(1, P.shuffle_writer(plan, 1))], "wavgerr")
                assert e.value.code == EXECUTION, str(e.value)
                continue
            got = driver.run_stages(gpu, [P.Stage(1, P.shuffle_writer(plan, 1))], "wavg")
            assert got.schema.field(2).type == pa.decimal128(38, 4)
            assert A.raw_values(got.column(2)) == [want] * len(rows), (v, rows)
