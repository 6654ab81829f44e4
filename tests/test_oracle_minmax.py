"""The CPU oracle's MIN / MAX over Utf8 and UInt64 -- the reference the device's string and unsigned accumulators are
checked against -- pinned against pyarrow's hash aggregation: NULLs and all-NULL groups, empty strings, strings that are
prefixes of each other or differ only after byte 40, non-ASCII UTF-8 (bytes >= 0x80, which order as unsigned bytes) and
UInt64 values on both sides of 2^63."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

from ballista_b200 import driver
from ballista_b200 import plan as P
from ballista_b200.plan import Stage
from util import assert_tables_equal

SCHEMA = [P.field("k", "i32", True), P.field("s", "utf8", True), P.field("u", "u64", True)]
WORDS = ["", "a", "ab", "abc", "abd", "b", "Z", "zz", "é", "éa", "ÿ", "中文", "x" * 41 + "a", "x" * 41 + "b",
         "x" * 41, "x" * 60 + "é", "A longer sentence that runs past forty bytes, then ends."]
U64 = [0, 1, 2**63 - 1, 2**63, 2**63 + 1, 2**64 - 1, 12345, 2**62]


def minmax_batch(n, seed, n_keys=5, p_null=0.15):
    """Rows of (k, s, u).  Key n_keys - 1 holds only NULL values (its MIN / MAX are NULL); a NULL key is a group too."""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, n_keys, n)
    key = [None if rng.random() < 0.05 else int(v) for v in k]
    s = [None if (kk == n_keys - 1 or rng.random() < p_null) else WORDS[w] for kk, w in zip(k, rng.integers(0, len(WORDS), n))]
    u = [None if (kk == n_keys - 1 or rng.random() < p_null) else U64[w] for kk, w in zip(k, rng.integers(0, len(U64), n))]
    return pa.record_batch([pa.array(key, pa.int32()), pa.array(s, pa.utf8()), pa.array(u, pa.uint64())], names=["k", "s", "u"])


AGGS = [("min", "s", "mn_s"), ("max", "s", "mx_s"), ("min", "u", "mn_u"), ("max", "u", "mx_u")]


def pyarrow_minmax(table, keyed, aggs=AGGS):
    """What the aggregate computes, by pyarrow: (k,) and the `aggs` columns (default mn_s, mx_s, mn_u, mx_u)."""
    if isinstance(table, pa.RecordBatch):
        table = pa.Table.from_batches([table])
    if keyed:
        g = table.group_by("k").aggregate([(col, fn) for fn, col, _ in aggs])
        return pa.table([g["k"]] + [g[f"{col}_{fn}"] for fn, col, _ in aggs], names=["k"] + [n for _, _, n in aggs])
    cols = [pa.array([getattr(pc, fn)(table[col]).as_py()], table.schema.field(col).type) for fn, col, _ in aggs]
    return pa.table(cols, names=[n for _, _, n in aggs])


def minmax_stages(keyed, mode, src, aggs=AGGS, n_out=3):
    """Stages computing `aggs` over `src` (columns k, s, u): one Single stage, or Partial -> shuffle -> Final(Partitioned)."""
    c = P.col
    gb = [(c("k"), "k")] if keyed else []
    pagg = [P.agg(fn, c(col), name) for fn, col, name in aggs]
    if mode == "Single":
        return [Stage(1, P.shuffle_writer(P.aggregate("Single", gb, pagg, src), 1))]
    s1 = P.aggregate("Partial", gb, pagg, src)
    part = ([P.field("k", "i32", True)] if keyed else []) + \
        [P.field(f"{name}[{fn}]", "utf8" if col == "s" else "u64", True) for fn, col, name in aggs]
    faggs = [P.agg(fn, None, name) for fn, _, name in aggs]
    if keyed:
        return [Stage(1, P.shuffle_writer(s1, 1, [c(0)], n_out)),
                Stage(2, P.shuffle_writer(P.aggregate("FinalPartitioned", [(c(0), "k")], faggs, P.shuffle_reader(1, part)), 2))]
    return [Stage(1, P.shuffle_writer(s1, 1)),
            Stage(2, P.shuffle_writer(P.aggregate("Final", [], faggs, P.coalesce_partitions(P.shuffle_reader(1, part))), 2), n_tasks=1)]


def test_oracle_string_and_u64_minmax_match_pyarrow(oracle):
    b = minmax_batch(6000, 5)
    oracle.register_batch("mm", 0, b.slice(0, 2500))   # two partitions: Partial -> Final
    oracle.register_batch("mm", 1, b.slice(2500))
    oracle.register_batch("mm1", 0, b)                 # one partition: Single
    for keyed in (True, False):
        want = pyarrow_minmax(b, keyed)
        for mode, table in (("Single", "mm1"), ("Partial", "mm")):
            got = driver.run_stages(oracle, minmax_stages(keyed, mode, P.scan(table, SCHEMA)), f"omm-{keyed}-{mode}")
            assert_tables_equal(got, want)


def test_oracle_all_null_input(oracle):
    """No value at all: every MIN / MAX is NULL, the scalar aggregate still emits its one row."""
    b = minmax_batch(50, 6, p_null=1.0)
    oracle.register_batch("mmn", 0, b)
    for keyed in (True, False):
        got = driver.run_stages(oracle, minmax_stages(keyed, "Single", P.scan("mmn", SCHEMA)), f"omn-{keyed}")
        assert_tables_equal(got, pyarrow_minmax(b, keyed))
        assert got.column("mx_s").null_count == got.num_rows
