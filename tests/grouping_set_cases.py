"""Grouping sets (ROLLUP / CUBE / GROUPING SETS) for the tests: input tables with a key of every type the engine carries
and real NULLs, the stage plans that run them, and the expected result.

The expected result restates the definition: a grouping-set aggregate is the UNION ALL over its sets of an ordinary
GROUP BY of the set's keys, with NULL in place of the other keys and the set's __grouping_id as a literal.  Each of those
ordinary aggregates runs on the CPU oracle, which has no grouping-set code of its own (it refuses such plans).  On an
empty input every set gives no rows (hash-aggregate behaviour), the () set included."""
from __future__ import annotations

import json
from typing import List, Sequence

import numpy as np
import pyarrow as pa

from ballista_b200 import driver, engine
from ballista_b200 import plan as P

c = P.col

SCHEMA = [P.field("ks", "utf8", True), P.field("ki", "i32", True), P.field("kd", P.dec(12, 2), True),
          P.field("kt", "date32", True), P.field("kf", "f64", True), P.field("kb", "bool", True),
          P.field("v", "f64", True), P.field("q", P.dec(12, 2), True), P.field("n", "i64", True),
          P.field("s", "utf8", True), P.field("u", "u64", True)]

# every accumulator kind of the global sink: COUNT / COUNT(*), SUM, AVG, MIN / MAX (Utf8 and UInt64 included)
AGGS = [P.agg("sum", c("q"), "sum_q"), P.agg("sum", c("v"), "sum_v"), P.agg("count", None, "cnt"),
        P.agg("count", c("n"), "cnt_n"), P.agg("avg", c("q"), "avg_q"), P.agg("avg", c("v"), "avg_v"),
        P.agg("min", c("s"), "min_s"), P.agg("max", c("s"), "max_s"), P.agg("min", c("n"), "min_n"),
        P.agg("max", c("u"), "max_u"), P.agg("min", c("kt"), "min_kt"), P.agg("max", c("v"), "max_v")]


def make_table(n: int, seed: int, null_frac: float = 0.1, card: int = 5) -> pa.Table:
    """n rows; every key column has about `card` distinct values and real NULLs."""
    rng = np.random.default_rng(seed)

    def nulls():
        return rng.random(n) < null_frac

    def arr(values, typ):
        m = nulls()
        return pa.array([None if m[i] else values[i] for i in range(n)], type=typ)

    words = ["", "a", "AIR", "MAIL", "TRUCK", "R", "longer than seven", "é"]
    ks = [words[i] for i in rng.integers(0, min(card, len(words)), n)]
    ki = [int(x) for x in rng.integers(-card // 2, card - card // 2, n)]
    kd = [int(x) * 125 for x in rng.integers(-2, card - 2, n)]
    kt = [int(x) for x in rng.integers(9000, 9000 + card, n)]
    kf = [float(x) / 4 for x in rng.integers(-2, card - 2, n)]
    kb = [bool(x) for x in rng.integers(0, 2, n)]
    v = [float(x) for x in rng.normal(0, 1000, n)]
    q = [int(x) for x in rng.integers(-10 ** 6, 10 ** 6, n)]
    nn = [int(x) for x in rng.integers(-10 ** 12, 10 ** 12, n)]
    s = ["".join(chr(97 + int(k)) for k in rng.integers(0, 26, int(rng.integers(0, 9)))) for _ in range(n)]
    u = [int(x) for x in rng.integers(0, 2 ** 63, n, dtype=np.uint64)]
    import decimal
    cols = [arr(ks, pa.string()), arr(ki, pa.int32()),
            arr([decimal.Decimal(x).scaleb(-2) for x in kd], pa.decimal128(12, 2)),
            arr(kt, pa.int32()).cast(pa.date32()), arr(kf, pa.float64()), arr(kb, pa.bool_()),
            arr(v, pa.float64()), arr([decimal.Decimal(x).scaleb(-2) for x in q], pa.decimal128(12, 2)),
            arr(nn, pa.int64()), arr(s, pa.string()), arr(u, pa.uint64())]
    return pa.Table.from_arrays(cols, names=[f["name"] for f in SCHEMA])


def register(e, name: str, table: pa.Table, parts: int) -> None:
    e.drop_table(name)
    step = max((table.num_rows + parts - 1) // parts, 1)
    for p in range(parts):
        sl = table.slice(min(table.num_rows, p * step), step).combine_chunks()
        e.register_batch(name, p, sl.to_batches()[0] if sl.num_rows else
                         pa.RecordBatch.from_arrays([pa.array([], type=f.type) for f in table.schema], schema=table.schema))


def typed(node: dict) -> dict:
    return json.loads(engine.plan_typed_json(json.dumps(node)))


def single_stages(input_plan: dict, keys, aggs, sets) -> List[P.Stage]:
    """One stage: a Single aggregate with the grouping sets (run it over one input partition)."""
    return [P.Stage(1, P.shuffle_writer(P.aggregate("Single", keys, aggs, input_plan, grouping_sets=sets), 1))]


def two_stages(input_plan: dict, keys, aggs, sets, n_out: int = 3) -> List[P.Stage]:
    """Partial with the grouping sets -> hash shuffle on the keys and __grouping_id -> FinalPartitioned over n + 1 plain keys."""
    partial = P.aggregate("Partial", keys, aggs, input_plan, grouping_sets=sets)
    t = typed(partial)
    nk = len(keys) + 1
    st1 = P.Stage(1, P.shuffle_writer(partial, 1, [c(i) for i in range(nk)], n_out))
    faggs = [P.agg(a["fn"], None, a["name"], ta["input_type"] if a["fn"] == "avg" else None) for a, ta in zip(aggs, t["aggr"])]
    final = P.aggregate("FinalPartitioned", [(c(i), t["schema"][i]["name"]) for i in range(nk)], faggs,
                        P.shuffle_reader(1, t["schema"]))
    return [st1, P.Stage(2, P.shuffle_writer(final, 2))]


def id_arrow_type(n_keys: int) -> pa.DataType:
    return pa.uint8() if n_keys <= 8 else pa.uint16() if n_keys <= 16 else pa.uint32() if n_keys <= 32 else pa.uint64()


def expected(oracle, input_plan: dict, keys, aggs, sets: Sequence[Sequence[bool]], job: str, mode: str = "Single") -> pa.Table:
    """The UNION ALL form on the oracle (the input's tables registered there as one partition each).  mode "Partial": the
    partial state columns after the keys and the id instead of the results."""
    full = driver.run_stages(oracle, [P.Stage(1, P.shuffle_writer(P.aggregate(mode, keys, aggs, input_plan), 1))], job + "-all")
    key_types = [full.schema.field(i).type for i in range(len(keys))]
    agg_fields = [full.schema.field(j) for j in range(len(keys), full.num_columns)]
    names = [n for _, n in keys] + ["__grouping_id"] + [f.name for f in agg_fields]
    parts = []
    empty_input = full.num_rows == 0
    for si, mask in enumerate(sets):
        present = [k for k, m in zip(keys, mask) if not m]
        got = driver.run_stages(oracle, [P.Stage(1, P.shuffle_writer(P.aggregate(mode, present, aggs, input_plan), 1))], f"{job}-{si}")
        if empty_input:
            got = got.slice(0, 0)  # no rows for any set on an empty input, () included
        n = got.num_rows
        cols, j = [], 0
        for i, m in enumerate(mask):
            if m:
                cols.append(pa.nulls(n, key_types[i]))
            else:
                cols.append(got.column(j).combine_chunks().cast(key_types[i]))
                j += 1
        cols.append(pa.array([P.grouping_id(mask)] * n, id_arrow_type(len(keys))))
        cols += [got.column(len(present) + a).combine_chunks().cast(agg_fields[a].type) for a in range(len(agg_fields))]
        parts.append(pa.Table.from_arrays(cols, names=names))
    return pa.concat_tables(parts)
