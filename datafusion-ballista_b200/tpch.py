"""TPC-H schemas (benchmarks/src/bin/tpch.rs:960-1049) and hand-lowered distributed stage plans for
the benchmark queries (benchmarks/queries/q*.sql), in the shape Ballista's planner produces
(ballista/scheduler/src/planner.rs:126-263; example stage shapes :655-670): every stage is rooted
at a shuffle writer, cut at hash repartitions / SortPreservingMerge.

Joins are lowered as HashJoinExec (``datafusion.optimizer.prefer_hash_join=true``, the opt-in
setting the north_star names; Ballista's default is sort-merge join, extension.rs:683).
"""
from __future__ import annotations

from typing import Dict, List

from . import plan as P
from .plan import Stage

D152 = P.dec(15, 2)

SCHEMAS: Dict[str, List[dict]] = {
    "part": [P.field("p_partkey", "i64"), P.field("p_name", "utf8"), P.field("p_mfgr", "utf8"),
             P.field("p_brand", "utf8"), P.field("p_type", "utf8"), P.field("p_size", "i32"),
             P.field("p_container", "utf8"), P.field("p_retailprice", D152), P.field("p_comment", "utf8")],
    "supplier": [P.field("s_suppkey", "i64"), P.field("s_name", "utf8"), P.field("s_address", "utf8"),
                 P.field("s_nationkey", "i64"), P.field("s_phone", "utf8"), P.field("s_acctbal", D152),
                 P.field("s_comment", "utf8")],
    "partsupp": [P.field("ps_partkey", "i64"), P.field("ps_suppkey", "i64"), P.field("ps_availqty", "i32"),
                 P.field("ps_supplycost", D152), P.field("ps_comment", "utf8")],
    "customer": [P.field("c_custkey", "i64"), P.field("c_name", "utf8"), P.field("c_address", "utf8"),
                 P.field("c_nationkey", "i64"), P.field("c_phone", "utf8"), P.field("c_acctbal", D152),
                 P.field("c_mktsegment", "utf8"), P.field("c_comment", "utf8")],
    "orders": [P.field("o_orderkey", "i64"), P.field("o_custkey", "i64"), P.field("o_orderstatus", "utf8"),
               P.field("o_totalprice", D152), P.field("o_orderdate", "date32"), P.field("o_orderpriority", "utf8"),
               P.field("o_clerk", "utf8"), P.field("o_shippriority", "i32"), P.field("o_comment", "utf8")],
    "lineitem": [P.field("l_orderkey", "i64"), P.field("l_partkey", "i64"), P.field("l_suppkey", "i64"),
                 P.field("l_linenumber", "i32"), P.field("l_quantity", D152), P.field("l_extendedprice", D152),
                 P.field("l_discount", D152), P.field("l_tax", D152), P.field("l_returnflag", "utf8"),
                 P.field("l_linestatus", "utf8"), P.field("l_shipdate", "date32"), P.field("l_commitdate", "date32"),
                 P.field("l_receiptdate", "date32"), P.field("l_shipinstruct", "utf8"), P.field("l_shipmode", "utf8"),
                 P.field("l_comment", "utf8")],
    "nation": [P.field("n_nationkey", "i64"), P.field("n_name", "utf8"), P.field("n_regionkey", "i64"),
               P.field("n_comment", "utf8")],
    "region": [P.field("r_regionkey", "i64"), P.field("r_name", "utf8"), P.field("r_comment", "utf8")],
}


def tbl_schema(table: str) -> List[dict]:
    """The schema a dbgen .tbl file is read with (tpch.rs:1056-1060 `get_tbl_tpch_table_schema`): the table's columns and
    a non-nullable Utf8 `__placeholder` that absorbs the empty field after each line's trailing '|'."""
    return SCHEMAS[table] + [P.field("__placeholder", "utf8")]


def tbl_scan(table: str, columns: List[str], path: str = None) -> dict:
    """The CSV variant of table_scan: DataSourceExec over the table's dbgen .tbl file ('|', no header), schema tbl_schema,
    projection into it -- what tpch.rs plans for `--format tbl`."""
    full = tbl_schema(table)
    names = [f["name"] for f in full]
    return P.csv_scan(table, full, projection=[names.index(c) for c in columns],
                      file_groups=[[path or f"/data/tpch/{table}.tbl"]], delimiter="|")


def col_index(table: str, name: str) -> int:
    for i, f in enumerate(SCHEMAS[table]):
        if f["name"] == name:
            return i
    raise KeyError(name)


# table -> the columns it is registered with, when that is a superset of what a query references (None: exactly the
# query's columns, the projection is the identity)
TABLE_LAYOUT: dict = {}


def table_scan(table: str, columns: List[str]) -> dict:
    """DataSourceExec with projection push-down.  By default the table is registered with exactly `columns`
    (the harness generates only the referenced columns); with TABLE_LAYOUT[table] set, the scan carries the
    projection indices into the registered layout."""
    sch = [f for name in columns for f in SCHEMAS[table] if f["name"] == name]
    layout = TABLE_LAYOUT.get(table)
    if layout is not None:
        full = [f for name in layout for f in SCHEMAS[table] if f["name"] == name]
        return P.scan(table, full, projection=[layout.index(name) for name in columns])
    return P.scan(table, sch)


def one_minus(x):  # `1 - x` with the Int64 literal already coerced to Decimal128(20,0) [EXT]
    return P.binop("-", P.lit_dec(1, 20, 0), x)


def one_plus(x):
    return P.binop("+", P.lit_dec(1, 20, 0), x)


Q1_COLUMNS = ["l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag", "l_linestatus", "l_shipdate"]


def q1(n_partitions: int = 16) -> List[Stage]:
    """benchmarks/queries/q1.sql -- scan + filter + projection + hash aggregate (low cardinality)."""
    c = P.col
    s1 = table_scan("lineitem", Q1_COLUMNS)
    s1 = P.filter_(P.binop("<=", c("l_shipdate"), P.lit_date("1998-09-02")), s1, projection=[0, 1, 2, 3, 4, 5])
    # DataFusion common-subexpression elimination: disc_price is computed once
    s1 = P.project([(P.binop("*", c("l_extendedprice"), one_minus(c("l_discount"))), "__common_expr_1"),
                    (c("l_quantity"), "l_quantity"), (c("l_extendedprice"), "l_extendedprice"),
                    (c("l_discount"), "l_discount"), (c("l_tax"), "l_tax"),
                    (c("l_returnflag"), "l_returnflag"), (c("l_linestatus"), "l_linestatus")], s1)
    aggs = [P.agg("sum", c("l_quantity"), "sum_qty"),
            P.agg("sum", c("l_extendedprice"), "sum_base_price"),
            P.agg("sum", c("__common_expr_1"), "sum_disc_price"),
            P.agg("sum", P.binop("*", c("__common_expr_1"), one_plus(c("l_tax"))), "sum_charge"),
            P.agg("avg", c("l_quantity"), "avg_qty"),
            P.agg("avg", c("l_extendedprice"), "avg_price"),
            P.agg("avg", c("l_discount"), "avg_disc"),
            P.agg("count", None, "count_order")]
    s1 = P.aggregate("Partial", [(c("l_returnflag"), "l_returnflag"), (c("l_linestatus"), "l_linestatus")], aggs, s1)
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0), c(1)], n_partitions))

    partial_schema = [P.field("l_returnflag", "utf8"), P.field("l_linestatus", "utf8"),
                      P.field("sum_qty[sum]", P.dec(25, 2), True), P.field("sum_base_price[sum]", P.dec(25, 2), True),
                      P.field("sum_disc_price[sum]", P.dec(38, 4), True), P.field("sum_charge[sum]", P.dec(38, 6), True),
                      P.field("avg_qty[count]", "u64", True), P.field("avg_qty[sum]", P.dec(25, 2), True),
                      P.field("avg_price[count]", "u64", True), P.field("avg_price[sum]", P.dec(25, 2), True),
                      P.field("avg_disc[count]", "u64", True), P.field("avg_disc[sum]", P.dec(25, 2), True),
                      P.field("count_order[count]", "i64")]
    faggs = [P.agg("sum", None, "sum_qty"), P.agg("sum", None, "sum_base_price"),
             P.agg("sum", None, "sum_disc_price"), P.agg("sum", None, "sum_charge"),
             P.agg("avg", None, "avg_qty", D152), P.agg("avg", None, "avg_price", D152),
             P.agg("avg", None, "avg_disc", D152), P.agg("count", None, "count_order")]
    s2 = P.aggregate("FinalPartitioned", [(c(0), "l_returnflag"), (c(1), "l_linestatus")], faggs,
                     P.shuffle_reader(1, partial_schema))
    keys = [P.sort_key(c(0)), P.sort_key(c(1))]
    s2 = P.sort(keys, s2, preserve_partitioning=True)
    st2 = Stage(2, P.shuffle_writer(s2, 2))

    final_schema = [P.field("l_returnflag", "utf8"), P.field("l_linestatus", "utf8"),
                    P.field("sum_qty", P.dec(25, 2), True), P.field("sum_base_price", P.dec(25, 2), True),
                    P.field("sum_disc_price", P.dec(38, 4), True), P.field("sum_charge", P.dec(38, 6), True),
                    P.field("avg_qty", P.dec(19, 6), True), P.field("avg_price", P.dec(19, 6), True),
                    P.field("avg_disc", P.dec(19, 6), True), P.field("count_order", "i64")]
    s3 = P.sort_preserving_merge(keys, P.shuffle_reader(2, final_schema))
    st3 = Stage(3, P.shuffle_writer(s3, 3), n_tasks=1)
    return [st1, st2, st3]


Q6_COLUMNS = ["l_quantity", "l_extendedprice", "l_discount", "l_shipdate"]


def q6(n_partitions: int = 16) -> List[Stage]:
    """benchmarks/queries/q6.sql -- multi-conjunct range filter + scalar aggregate."""
    c = P.col
    s1 = table_scan("lineitem", Q6_COLUMNS)
    pred = P.and_(P.binop(">=", c("l_shipdate"), P.lit_date("1994-01-01")),
                  P.binop("<", c("l_shipdate"), P.lit_date("1995-01-01")),
                  P.binop(">=", c("l_discount"), P.lit_dec(5, 15, 2)),
                  P.binop("<=", c("l_discount"), P.lit_dec(7, 15, 2)),
                  P.binop("<", c("l_quantity"), P.lit_dec(2400, 15, 2)))
    s1 = P.filter_(pred, s1, projection=[1, 2])
    s1 = P.aggregate("Partial", [], [P.agg("sum", P.binop("*", c("l_extendedprice"), c("l_discount")), "revenue")], s1)
    st1 = Stage(1, P.shuffle_writer(s1, 1))
    partial_schema = [P.field("revenue[sum]", P.dec(38, 4), True)]
    s2 = P.aggregate("Final", [], [P.agg("sum", None, "revenue")],
                     P.coalesce_partitions(P.shuffle_reader(1, partial_schema)))
    st2 = Stage(2, P.shuffle_writer(s2, 2), n_tasks=1)
    return [st1, st2]


def _sch(table, cols):
    return [f for name in cols for f in SCHEMAS[table] if f["name"] == name]


Q5_TABLES = {"region": ["r_regionkey", "r_name"], "nation": ["n_nationkey", "n_name", "n_regionkey"],
             "customer": ["c_custkey", "c_nationkey"], "orders": ["o_orderkey", "o_custkey", "o_orderdate"],
             "lineitem": ["l_orderkey", "l_suppkey", "l_extendedprice", "l_discount"], "supplier": ["s_suppkey", "s_nationkey"]}


def q5(n_partitions: int = 4) -> List[Stage]:
    """benchmarks/queries/q5.sql -- 6-way join (HashJoinExec, Partitioned + CollectLeft) with hash shuffles on
    the join keys, then a low-cardinality aggregate and ORDER BY revenue DESC (BASELINE.json configs[2])."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    # S1: nation |x| region(r_name = 'ASIA')  (both tiny: CollectLeft inside one task)
    reg = P.filter_(P.binop("=", c("r_name"), P.lit_utf8("ASIA")), table_scan("region", Q5_TABLES["region"]), projection=[0])
    s1 = P.hash_join(reg, table_scan("nation", Q5_TABLES["nation"]), [[c(0), c("n_regionkey")]], "Inner", "CollectLeft", projection=[1, 2])
    st1 = Stage(1, P.shuffle_writer(s1, 1), n_tasks=1)
    nat = [P.field("n_nationkey", i64, True), P.field("n_name", "utf8", True)]
    # S2: customer |x| nation (broadcast build side)
    s2 = P.hash_join(P.shuffle_reader(1, nat, broadcast=True), table_scan("customer", Q5_TABLES["customer"]),
                     [[c(0), c("c_nationkey")]], "Inner", "CollectLeft", projection=[2, 3, 1])
    st2 = Stage(2, P.shuffle_writer(s2, 2, [c(0)], Pn))
    cust = [P.field("c_custkey", i64, True), P.field("c_nationkey", i64, True), P.field("n_name", "utf8", True)]
    # S3: orders filtered by date
    s3 = P.filter_(P.and_(P.binop(">=", c("o_orderdate"), P.lit_date("1994-01-01")), P.binop("<", c("o_orderdate"), P.lit_date("1995-01-01"))),
                   table_scan("orders", Q5_TABLES["orders"]), projection=[0, 1])
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(1)], Pn))
    ords = [P.field("o_orderkey", i64, True), P.field("o_custkey", i64, True)]
    # S4: customer' |x| orders' on custkey
    s4 = P.hash_join(P.shuffle_reader(2, cust), P.shuffle_reader(3, ords), [[c(0), c(1)]], "Inner", "Partitioned", projection=[3, 1, 2])
    st4 = Stage(4, P.shuffle_writer(s4, 4, [c(0)], Pn))
    co = [P.field("o_orderkey", i64, True), P.field("c_nationkey", i64, True), P.field("n_name", "utf8", True)]
    # S5: lineitem by orderkey
    st5 = Stage(5, P.shuffle_writer(table_scan("lineitem", Q5_TABLES["lineitem"]), 5, [c(0)], Pn))
    li = _sch("lineitem", Q5_TABLES["lineitem"])
    li = [dict(f, nullable=True) for f in li]
    # S6: (customer, orders) |x| lineitem on orderkey
    s6 = P.hash_join(P.shuffle_reader(4, co), P.shuffle_reader(5, li), [[c(0), c(0)]], "Inner", "Partitioned", projection=[4, 1, 2, 5, 6])
    st6 = Stage(6, P.shuffle_writer(s6, 6, [c(0)], Pn))
    col6 = [P.field("l_suppkey", i64, True), P.field("c_nationkey", i64, True), P.field("n_name", "utf8", True),
            P.field("l_extendedprice", D152, True), P.field("l_discount", D152, True)]
    # S7: supplier by suppkey
    st7 = Stage(7, P.shuffle_writer(table_scan("supplier", Q5_TABLES["supplier"]), 7, [c(0)], Pn))
    sup = [P.field("s_suppkey", i64, True), P.field("s_nationkey", i64, True)]
    # S8: supplier |x| ... on (suppkey, nationkey) -> partial aggregate by n_name
    s8 = P.hash_join(P.shuffle_reader(7, sup), P.shuffle_reader(6, col6), [[c(0), c(0)], [c(1), c(1)]], "Inner", "Partitioned", projection=[4, 5, 6])
    s8 = P.project([(c(0), "n_name"), (P.binop("*", c(1), one_minus(c(2))), "rev")], s8)
    s8 = P.aggregate("Partial", [(c(0), "n_name")], [P.agg("sum", c(1), "revenue")], s8)
    st8 = Stage(8, P.shuffle_writer(s8, 8, [c(0)], Pn))
    part = [P.field("n_name", "utf8", True), P.field("revenue[sum]", P.dec(38, 4), True)]
    s9 = P.aggregate("FinalPartitioned", [(c(0), "n_name")], [P.agg("sum", None, "revenue")], P.shuffle_reader(8, part))
    keys = [P.sort_key(c(1), asc=False)]
    s9 = P.sort(keys, s9, preserve_partitioning=True)
    st9 = Stage(9, P.shuffle_writer(s9, 9))
    fin = [P.field("n_name", "utf8", True), P.field("revenue", P.dec(38, 4), True)]
    st10 = Stage(10, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(9, fin)), 10), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7, st8, st9, st10]


Q17_TABLES = {"lineitem": ["l_partkey", "l_quantity", "l_extendedprice"], "part": ["p_partkey", "p_brand", "p_container"]}


def q17(n_partitions: int = 4, brand: str = "Brand#23", container: str = "MED BOX") -> List[Stage]:
    """benchmarks/queries/q17.sql after decorrelation: high-cardinality AVG per l_partkey joined back to the
    filtered parts and lineitems (`l_quantity < 0.2 * avg`, fp64), final `sum(l_extendedprice) / 7.0` (configs[3])."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    li = table_scan("lineitem", Q17_TABLES["lineitem"])
    s1 = P.aggregate("Partial", [(c("l_partkey"), "l_partkey")], [P.agg("avg", c("l_quantity"), "avg_qty")], li)
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    st_avg = [P.field("l_partkey", i64, True), P.field("avg_qty[count]", "u64", True), P.field("avg_qty[sum]", P.dec(25, 2), True)]
    prt = P.filter_(P.and_(P.binop("=", c("p_brand"), P.lit_utf8(brand)), P.binop("=", c("p_container"), P.lit_utf8(container))),
                    table_scan("part", Q17_TABLES["part"]), projection=[0])
    st2 = Stage(2, P.shuffle_writer(prt, 2, [c(0)], Pn))
    st3 = Stage(3, P.shuffle_writer(table_scan("lineitem", Q17_TABLES["lineitem"]), 3, [c(0)], Pn))
    lis = [dict(f, nullable=True) for f in _sch("lineitem", Q17_TABLES["lineitem"])]
    avg = P.aggregate("FinalPartitioned", [(c(0), "l_partkey")], [P.agg("avg", None, "avg_qty", D152)], P.shuffle_reader(1, st_avg))
    thr = P.project([(c(0), "pk"), (P.binop("*", P.lit_f64(0.2), P.cast(c(1), "f64")), "thr")], avg)
    pl = P.hash_join(P.shuffle_reader(2, [P.field("p_partkey", i64, True)]), P.shuffle_reader(3, lis), [[c(0), c(0)]], "Inner", "Partitioned",
                     projection=[1, 2, 3])
    # residual filter over concat(thr(pk, thr), pl(l_partkey, l_quantity, l_extendedprice))
    j = P.hash_join(thr, pl, [[c(0), c(0)]], "Inner", "Partitioned", filter=P.binop("<", P.cast(c(3), "f64"), c(1)), projection=[4])
    s4 = P.aggregate("Partial", [], [P.agg("sum", c(0), "s")], j)
    st4 = Stage(4, P.shuffle_writer(s4, 4))
    s5 = P.aggregate("Final", [], [P.agg("sum", None, "s")], P.coalesce_partitions(P.shuffle_reader(4, [P.field("s[sum]", P.dec(25, 2), True)])))
    s5 = P.project([(P.binop("/", P.cast(c(0), "f64"), P.lit_f64(7.0)), "avg_yearly")], s5)
    return [st1, st2, st3, st4 if False else Stage(4, P.shuffle_writer(s4, 4)), Stage(5, P.shuffle_writer(s5, 5), n_tasks=1)]


Q3_TABLES = {"customer": ["c_custkey", "c_mktsegment"], "orders": ["o_orderkey", "o_custkey", "o_orderdate", "o_shippriority"],
             "lineitem": ["l_orderkey", "l_extendedprice", "l_discount", "l_shipdate"]}


def q3(n_partitions: int = 4, segment: str = "BUILDING", date: str = "1995-03-15") -> List[Stage]:
    """benchmarks/queries/q3.sql -- customer |x| orders |x| lineitem (Partitioned hash joins on hash-shuffled
    inputs), aggregate on (l_orderkey, o_orderdate, o_shippriority), top-10 by revenue (SortExec fetch +
    SortPreservingMergeExec fetch, the cut the planner makes at `planner.rs:214-230`)."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    s1 = P.filter_(P.binop("=", c("c_mktsegment"), P.lit_utf8(segment)), table_scan("customer", Q3_TABLES["customer"]), projection=[0])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    s2 = P.filter_(P.binop("<", c("o_orderdate"), P.lit_date(date)), table_scan("orders", Q3_TABLES["orders"]))
    st2 = Stage(2, P.shuffle_writer(s2, 2, [c(1)], Pn))
    ords = [dict(f, nullable=True) for f in _sch("orders", Q3_TABLES["orders"])]
    # S3: customer' |x| orders' on custkey -> (o_orderkey, o_orderdate, o_shippriority), re-shuffled on orderkey
    s3 = P.hash_join(P.shuffle_reader(1, [P.field("c_custkey", i64, True)]), P.shuffle_reader(2, ords), [[c(0), c(1)]], "Inner", "Partitioned",
                     projection=[1, 3, 4])
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(0)], Pn))
    co = [P.field("o_orderkey", i64, True), P.field("o_orderdate", "date32", True), P.field("o_shippriority", "i32", True)]
    s4 = P.filter_(P.binop(">", c("l_shipdate"), P.lit_date(date)), table_scan("lineitem", Q3_TABLES["lineitem"]), projection=[0, 1, 2])
    st4 = Stage(4, P.shuffle_writer(s4, 4, [c(0)], Pn))
    li = [P.field("l_orderkey", i64, True), P.field("l_extendedprice", D152, True), P.field("l_discount", D152, True)]
    # S5: (customer, orders) |x| lineitem' on orderkey -> partial aggregate
    s5 = P.hash_join(P.shuffle_reader(3, co), P.shuffle_reader(4, li), [[c(0), c(0)]], "Inner", "Partitioned", projection=[3, 1, 2, 4, 5])
    s5 = P.project([(c(0), "l_orderkey"), (c(1), "o_orderdate"), (c(2), "o_shippriority"),
                    (P.binop("*", c(3), one_minus(c(4))), "rev")], s5)
    gb = [(c(0), "l_orderkey"), (c(1), "o_orderdate"), (c(2), "o_shippriority")]
    s5 = P.aggregate("Partial", gb, [P.agg("sum", c(3), "revenue")], s5)
    st5 = Stage(5, P.shuffle_writer(s5, 5, [c(0), c(1), c(2)], Pn))
    part = [P.field("l_orderkey", i64, True), P.field("o_orderdate", "date32", True), P.field("o_shippriority", "i32", True),
            P.field("revenue[sum]", P.dec(38, 4), True)]
    s6 = P.aggregate("FinalPartitioned", gb, [P.agg("sum", None, "revenue")], P.shuffle_reader(5, part))
    s6 = P.project([(c(0), "l_orderkey"), (c(3), "revenue"), (c(1), "o_orderdate"), (c(2), "o_shippriority")], s6)
    keys = [P.sort_key(c(1), asc=False), P.sort_key(c(2))]
    s6 = P.sort(keys, s6, fetch=10, preserve_partitioning=True)
    st6 = Stage(6, P.shuffle_writer(s6, 6))
    fin = [P.field("l_orderkey", i64, True), P.field("revenue", P.dec(38, 4), True), P.field("o_orderdate", "date32", True),
           P.field("o_shippriority", "i32", True)]
    st7 = Stage(7, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(6, fin), fetch=10), 7), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7]


Q12_TABLES = {"lineitem": ["l_orderkey", "l_shipdate", "l_commitdate", "l_receiptdate", "l_shipmode"],
              "orders": ["o_orderkey", "o_orderpriority"]}


def q12(n_partitions: int = 4, modes=("MAIL", "SHIP"), year: int = 1994) -> List[Stage]:
    """benchmarks/queries/q12.sql -- IN list, column-vs-column date compares, join, SUM(CASE WHEN ... THEN 1 ELSE 0 END)
    (Int64 sums), GROUP BY l_shipmode ORDER BY l_shipmode."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    pred = P.and_(P.in_list(c("l_shipmode"), [P.lit_utf8(m) for m in modes]),
                  P.binop("<", c("l_commitdate"), c("l_receiptdate")),
                  P.binop("<", c("l_shipdate"), c("l_commitdate")),
                  P.binop(">=", c("l_receiptdate"), P.lit_date(f"{year}-01-01")),
                  P.binop("<", c("l_receiptdate"), P.lit_date(f"{year + 1}-01-01")))
    s1 = P.filter_(pred, table_scan("lineitem", Q12_TABLES["lineitem"]), projection=[0, 4])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    st2 = Stage(2, P.shuffle_writer(table_scan("orders", Q12_TABLES["orders"]), 2, [c(0)], Pn))
    li = [P.field("l_orderkey", i64, True), P.field("l_shipmode", "utf8", True)]
    od = [P.field("o_orderkey", i64, True), P.field("o_orderpriority", "utf8", True)]
    j = P.hash_join(P.shuffle_reader(1, li), P.shuffle_reader(2, od), [[c(0), c(0)]], "Inner", "Partitioned", projection=[1, 3])
    urgent = P.or_(P.binop("=", c(1), P.lit_utf8("1-URGENT")), P.binop("=", c(1), P.lit_utf8("2-HIGH")))
    other = P.and_(P.binop("<>", c(1), P.lit_utf8("1-URGENT")), P.binop("<>", c(1), P.lit_utf8("2-HIGH")))
    one, zero = P.lit_i64(1), P.lit_i64(0)
    s3 = P.project([(c(0), "l_shipmode"), (P.case([[urgent, one]], zero), "hi"), (P.case([[other, one]], zero), "lo")], j)
    s3 = P.aggregate("Partial", [(c(0), "l_shipmode")], [P.agg("sum", c(1), "high_line_count"), P.agg("sum", c(2), "low_line_count")], s3)
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(0)], Pn))
    part = [P.field("l_shipmode", "utf8", True), P.field("high_line_count[sum]", i64, True), P.field("low_line_count[sum]", i64, True)]
    s4 = P.aggregate("FinalPartitioned", [(c(0), "l_shipmode")], [P.agg("sum", None, "high_line_count"), P.agg("sum", None, "low_line_count")],
                     P.shuffle_reader(3, part))
    keys = [P.sort_key(c(0))]
    s4 = P.sort(keys, s4, preserve_partitioning=True)
    st4 = Stage(4, P.shuffle_writer(s4, 4))
    fin = [P.field("l_shipmode", "utf8", True), P.field("high_line_count", i64, True), P.field("low_line_count", i64, True)]
    st5 = Stage(5, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(4, fin)), 5), n_tasks=1)
    return [st1, st2, st3, st4, st5]


Q4_TABLES = {"orders": ["o_orderkey", "o_orderdate", "o_orderpriority"], "lineitem": ["l_orderkey", "l_commitdate", "l_receiptdate"]}


def q4(n_partitions: int = 4, date_from: str = "1993-07-01", date_to: str = "1993-10-01") -> List[Stage]:
    """benchmarks/queries/q4.sql -- EXISTS subquery decorrelated into a semi join (orders LEFT SEMI lineitem on
    orderkey), COUNT(*) GROUP BY o_orderpriority ORDER BY o_orderpriority."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    s1 = P.filter_(P.and_(P.binop(">=", c("o_orderdate"), P.lit_date(date_from)), P.binop("<", c("o_orderdate"), P.lit_date(date_to))),
                   table_scan("orders", Q4_TABLES["orders"]), projection=[0, 2])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    s2 = P.filter_(P.binop("<", c("l_commitdate"), c("l_receiptdate")), table_scan("lineitem", Q4_TABLES["lineitem"]), projection=[0])
    st2 = Stage(2, P.shuffle_writer(s2, 2, [c(0)], Pn))
    od = [P.field("o_orderkey", i64, True), P.field("o_orderpriority", "utf8", True)]
    # build = lineitem keys, probe = orders: RightSemi keeps every probe-side order that has a match
    j = P.hash_join(P.shuffle_reader(2, [P.field("l_orderkey", i64, True)]), P.shuffle_reader(1, od), [[c(0), c(0)]], "RightSemi", "Partitioned")
    s3 = P.aggregate("Partial", [(c(1), "o_orderpriority")], [P.agg("count", None, "order_count")], j)
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(0)], Pn))
    part = [P.field("o_orderpriority", "utf8", True), P.field("order_count[count]", i64)]
    s4 = P.aggregate("FinalPartitioned", [(c(0), "o_orderpriority")], [P.agg("count", None, "order_count")], P.shuffle_reader(3, part))
    keys = [P.sort_key(c(0))]
    s4 = P.sort(keys, s4, preserve_partitioning=True)
    st4 = Stage(4, P.shuffle_writer(s4, 4))
    fin = [P.field("o_orderpriority", "utf8", True), P.field("order_count", i64)]
    st5 = Stage(5, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(4, fin)), 5), n_tasks=1)
    return [st1, st2, st3, st4, st5]


Q13_TABLES = {"customer": ["c_custkey"], "orders": ["o_orderkey", "o_custkey", "o_comment"]}


def q13(n_partitions: int = 4, pattern: str = "%special%requests%") -> List[Stage]:
    """benchmarks/queries/q13.sql -- customer LEFT OUTER JOIN orders (NOT LIKE filter pushed below the join),
    COUNT(o_orderkey) per customer (SinglePartitioned: the join output is already partitioned on c_custkey), then the
    distribution of that count: GROUP BY c_count ORDER BY custdist DESC, c_count DESC."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    st1 = Stage(1, P.shuffle_writer(table_scan("customer", Q13_TABLES["customer"]), 1, [c(0)], Pn))
    s2 = P.filter_(P.like(c("o_comment"), pattern, negated=True), table_scan("orders", Q13_TABLES["orders"]), projection=[0, 1])
    st2 = Stage(2, P.shuffle_writer(s2, 2, [c(1)], Pn))
    od = [P.field("o_orderkey", i64, True), P.field("o_custkey", i64, True)]
    # build = orders, probe = customer: Right join keeps every probe-side customer, NULL orders where none match
    j = P.hash_join(P.shuffle_reader(2, od), P.shuffle_reader(1, [P.field("c_custkey", i64, True)]), [[c(1), c(0)]], "Right", "Partitioned",
                    projection=[2, 0])
    s3 = P.aggregate("SinglePartitioned", [(c(0), "c_custkey")], [P.agg("count", c(1), "c_count")], j)
    s3 = P.project([(c(1), "c_count")], s3)
    s3 = P.aggregate("Partial", [(c(0), "c_count")], [P.agg("count", None, "custdist")], s3)
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(0)], Pn))
    part = [P.field("c_count", i64, True), P.field("custdist[count]", i64)]
    s4 = P.aggregate("FinalPartitioned", [(c(0), "c_count")], [P.agg("count", None, "custdist")], P.shuffle_reader(3, part))
    keys = [P.sort_key(c(1), asc=False), P.sort_key(c(0), asc=False)]
    s4 = P.sort(keys, s4, preserve_partitioning=True)
    st4 = Stage(4, P.shuffle_writer(s4, 4))
    fin = [P.field("c_count", i64, True), P.field("custdist", i64)]
    st5 = Stage(5, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(4, fin)), 5), n_tasks=1)
    return [st1, st2, st3, st4, st5]


Q10_TABLES = {"nation": ["n_nationkey", "n_name"],
              "customer": ["c_custkey", "c_name", "c_address", "c_nationkey", "c_phone", "c_acctbal", "c_comment"],
              "orders": ["o_orderkey", "o_custkey", "o_orderdate"],
              "lineitem": ["l_orderkey", "l_extendedprice", "l_discount", "l_returnflag"]}


def q10(n_partitions: int = 4, date_from: str = "1993-10-01", date_to: str = "1994-01-01", flag: str = "R") -> List[Stage]:
    """benchmarks/queries/q10.sql -- customer |x| nation (broadcast), |x| orders, |x| lineitem; seven group keys (integer,
    strings, decimal) through the hash-table aggregate; top-20 by revenue."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    st1 = Stage(1, P.shuffle_writer(table_scan("nation", Q10_TABLES["nation"]), 1), n_tasks=1)
    nat = [P.field("n_nationkey", i64, True), P.field("n_name", "utf8", True)]
    # S2: nation (broadcast build side) |x| customer -> c_custkey, c_name, c_address, c_phone, c_acctbal, c_comment, n_name
    s2 = P.hash_join(P.shuffle_reader(1, nat, broadcast=True), table_scan("customer", Q10_TABLES["customer"]), [[c(0), c("c_nationkey")]],
                     "Inner", "CollectLeft", projection=[2, 3, 4, 6, 7, 8, 1])
    st2 = Stage(2, P.shuffle_writer(s2, 2, [c(0)], Pn))
    cust = [P.field("c_custkey", i64, True), P.field("c_name", "utf8", True), P.field("c_address", "utf8", True), P.field("c_phone", "utf8", True),
            P.field("c_acctbal", D152, True), P.field("c_comment", "utf8", True), P.field("n_name", "utf8", True)]
    s3 = P.filter_(P.and_(P.binop(">=", c("o_orderdate"), P.lit_date(date_from)), P.binop("<", c("o_orderdate"), P.lit_date(date_to))),
                   table_scan("orders", Q10_TABLES["orders"]), projection=[0, 1])
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(1)], Pn))
    ords = [P.field("o_orderkey", i64, True), P.field("o_custkey", i64, True)]
    # S4: customer' |x| orders' on custkey -> (o_orderkey, customer columns...), re-shuffled on orderkey
    s4 = P.hash_join(P.shuffle_reader(2, cust), P.shuffle_reader(3, ords), [[c(0), c(1)]], "Inner", "Partitioned",
                     projection=[7, 0, 1, 2, 3, 4, 5, 6])
    st4 = Stage(4, P.shuffle_writer(s4, 4, [c(0)], Pn))
    co = [P.field("o_orderkey", i64, True)] + cust
    s5 = P.filter_(P.binop("=", c("l_returnflag"), P.lit_utf8(flag)), table_scan("lineitem", Q10_TABLES["lineitem"]), projection=[0, 1, 2])
    st5 = Stage(5, P.shuffle_writer(s5, 5, [c(0)], Pn))
    li = [P.field("l_orderkey", i64, True), P.field("l_extendedprice", D152, True), P.field("l_discount", D152, True)]
    # S6: (customer, orders) |x| lineitem' on orderkey -> partial aggregate on the seven keys
    s6 = P.hash_join(P.shuffle_reader(4, co), P.shuffle_reader(5, li), [[c(0), c(0)]], "Inner", "Partitioned",
                     projection=[1, 2, 5, 4, 7, 3, 6, 9, 10])
    # columns now: c_custkey, c_name, c_acctbal, c_phone, n_name, c_address, c_comment, l_extendedprice, l_discount
    gb_names = ["c_custkey", "c_name", "c_acctbal", "c_phone", "n_name", "c_address", "c_comment"]
    s6 = P.project([(c(i), nme) for i, nme in enumerate(gb_names)] + [(P.binop("*", c(7), one_minus(c(8))), "rev")], s6)
    gb = [(c(i), nme) for i, nme in enumerate(gb_names)]
    s6 = P.aggregate("Partial", gb, [P.agg("sum", c(7), "revenue")], s6)
    st6 = Stage(6, P.shuffle_writer(s6, 6, [c(i) for i in range(7)], Pn))
    ktypes = [i64, "utf8", D152, "utf8", "utf8", "utf8", "utf8"]
    part = [P.field(nme, t, True) for nme, t in zip(gb_names, ktypes)] + [P.field("revenue[sum]", P.dec(38, 4), True)]
    s7 = P.aggregate("FinalPartitioned", gb, [P.agg("sum", None, "revenue")], P.shuffle_reader(6, part))
    # select list order: c_custkey, c_name, revenue, c_acctbal, n_name, c_address, c_phone, c_comment
    s7 = P.project([(c(0), "c_custkey"), (c(1), "c_name"), (c(7), "revenue"), (c(2), "c_acctbal"), (c(4), "n_name"), (c(5), "c_address"),
                    (c(3), "c_phone"), (c(6), "c_comment")], s7)
    keys = [P.sort_key(c(2), asc=False)]
    s7 = P.sort(keys, s7, fetch=20, preserve_partitioning=True)
    st7 = Stage(7, P.shuffle_writer(s7, 7))
    fin = [P.field("c_custkey", i64, True), P.field("c_name", "utf8", True), P.field("revenue", P.dec(38, 4), True), P.field("c_acctbal", D152, True),
           P.field("n_name", "utf8", True), P.field("c_address", "utf8", True), P.field("c_phone", "utf8", True), P.field("c_comment", "utf8", True)]
    st8 = Stage(8, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(7, fin), fetch=20), 8), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7, st8]


Q19_TABLES = {"part": ["p_partkey", "p_brand", "p_size", "p_container"],
              "lineitem": ["l_partkey", "l_quantity", "l_extendedprice", "l_discount", "l_shipinstruct", "l_shipmode"]}
Q19_GROUPS = [("Brand#12", ["SM CASE", "SM BOX", "SM PACK", "SM PKG"], 1, 11, 5),
              ("Brand#23", ["MED BAG", "MED BOX", "MED PKG", "MED PACK"], 10, 20, 10),
              ("Brand#34", ["LG CASE", "LG BOX", "LG PACK", "LG PKG"], 20, 30, 15)]


def q19(n_partitions: int = 4, groups=None, modes=("AIR", "AIR REG"), instruct: str = "DELIVER IN PERSON") -> List[Stage]:
    """benchmarks/queries/q19.sql -- lineitem |x| part on partkey with the three-way OR of conjunctions as the join's
    residual filter (IN lists, BETWEEN, decimal compares across both sides); the common factors (ship mode / instruction,
    p_size >= 1) are pushed below the join as DataFusion does.  groups: [(brand, containers, qty_lo, qty_hi, size_hi)]."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    groups = groups or Q19_GROUPS
    qty = lambda v: P.lit_dec(int(v) * 100, 15, 2)
    s1 = P.filter_(P.binop(">=", c("p_size"), P.lit_i32(1)), table_scan("part", Q19_TABLES["part"]))
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    pred = P.and_(P.in_list(c("l_shipmode"), [P.lit_utf8(m) for m in modes]), P.binop("=", c("l_shipinstruct"), P.lit_utf8(instruct)))
    s2 = P.filter_(pred, table_scan("lineitem", Q19_TABLES["lineitem"]), projection=[0, 1, 2, 3])
    st2 = Stage(2, P.shuffle_writer(s2, 2, [c(0)], Pn))
    pt = [P.field("p_partkey", i64, True), P.field("p_brand", "utf8", True), P.field("p_size", "i32", True), P.field("p_container", "utf8", True)]
    li = [P.field("l_partkey", i64, True), P.field("l_quantity", D152, True), P.field("l_extendedprice", D152, True), P.field("l_discount", D152, True)]
    # residual filter over concat(part[0..3], lineitem[4..7])
    ors = []
    for brand, conts, q_lo, q_hi, size_hi in groups:
        ors.append(P.and_(P.binop("=", c(1), P.lit_utf8(brand)), P.in_list(c(3), [P.lit_utf8(x) for x in conts]),
                          P.binop(">=", c(5), qty(q_lo)), P.binop("<=", c(5), qty(q_hi)),
                          P.binop("<=", c(2), P.lit_i32(size_hi))))
    j = P.hash_join(P.shuffle_reader(1, pt), P.shuffle_reader(2, li), [[c(0), c(0)]], "Inner", "Partitioned", filter=P.or_(*ors), projection=[6, 7])
    s3 = P.project([(P.binop("*", c(0), one_minus(c(1))), "rev")], j)
    s3 = P.aggregate("Partial", [], [P.agg("sum", c(0), "revenue")], s3)
    st3 = Stage(3, P.shuffle_writer(s3, 3))
    s4 = P.aggregate("Final", [], [P.agg("sum", None, "revenue")], P.coalesce_partitions(P.shuffle_reader(3, [P.field("revenue[sum]", P.dec(38, 4), True)])))
    return [st1, st2, st3, Stage(4, P.shuffle_writer(s4, 4), n_tasks=1)]


Q18_TABLES = {"customer": ["c_custkey", "c_name"], "orders": ["o_orderkey", "o_custkey", "o_totalprice", "o_orderdate"],
              "lineitem": ["l_orderkey", "l_quantity"]}


def q18(n_partitions: int = 4, threshold: int = 300) -> List[Stage]:
    """benchmarks/queries/q18.sql -- IN (subquery with GROUP BY ... HAVING sum(l_quantity) > t) as a semi join against a
    high-cardinality aggregate that is filtered after the aggregation, joined back to customer/orders/lineitem,
    five group keys, ORDER BY o_totalprice DESC, o_orderdate LIMIT 100."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    # S1: lineitem by orderkey (feeds both the HAVING subquery and the final join)
    st1 = Stage(1, P.shuffle_writer(table_scan("lineitem", Q18_TABLES["lineitem"]), 1, [c(0)], Pn))
    li = [P.field("l_orderkey", i64, True), P.field("l_quantity", D152, True)]
    st2 = Stage(2, P.shuffle_writer(table_scan("customer", Q18_TABLES["customer"]), 2, [c(0)], Pn))
    cu = [P.field("c_custkey", i64, True), P.field("c_name", "utf8", True)]
    st3 = Stage(3, P.shuffle_writer(table_scan("orders", Q18_TABLES["orders"]), 3, [c(1)], Pn))
    od = [P.field("o_orderkey", i64, True), P.field("o_custkey", i64, True), P.field("o_totalprice", D152, True), P.field("o_orderdate", "date32", True)]
    # S4: customer |x| orders on custkey -> (c_name, c_custkey, o_orderkey, o_orderdate, o_totalprice), re-shuffled on orderkey
    s4 = P.hash_join(P.shuffle_reader(2, cu), P.shuffle_reader(3, od), [[c(0), c(1)]], "Inner", "Partitioned", projection=[1, 0, 2, 5, 4])
    st4 = Stage(4, P.shuffle_writer(s4, 4, [c(2)], Pn))
    co = [P.field("c_name", "utf8", True), P.field("c_custkey", i64, True), P.field("o_orderkey", i64, True), P.field("o_orderdate", "date32", True),
          P.field("o_totalprice", D152, True)]
    # S5 (co-partitioned on orderkey): big orders = HAVING sum(l_quantity) > t; semi join; join lineitem back; partial aggregate
    big = P.aggregate("SinglePartitioned", [(c(0), "l_orderkey")], [P.agg("sum", c(1), "q")], P.shuffle_reader(1, li))
    big = P.filter_(P.binop(">", c(1), P.lit_dec(int(threshold) * 100, 25, 2)), big, projection=[0])
    semi = P.hash_join(big, P.shuffle_reader(4, co), [[c(0), c(2)]], "RightSemi", "Partitioned")
    j = P.hash_join(semi, P.shuffle_reader(1, li), [[c(2), c(0)]], "Inner", "Partitioned", projection=[0, 1, 2, 3, 4, 6])
    gb_names = ["c_name", "c_custkey", "o_orderkey", "o_orderdate", "o_totalprice"]
    gb = [(c(i), nme) for i, nme in enumerate(gb_names)]
    s5 = P.aggregate("Partial", gb, [P.agg("sum", c(5), "sum_qty")], j)
    st5 = Stage(5, P.shuffle_writer(s5, 5, [c(i) for i in range(5)], Pn))
    ktypes = ["utf8", i64, i64, "date32", D152]
    part = [P.field(nme, t, True) for nme, t in zip(gb_names, ktypes)] + [P.field("sum_qty[sum]", P.dec(25, 2), True)]
    s6 = P.aggregate("FinalPartitioned", gb, [P.agg("sum", None, "sum_qty")], P.shuffle_reader(5, part))
    keys = [P.sort_key(c(4), asc=False), P.sort_key(c(3))]
    s6 = P.sort(keys, s6, fetch=100, preserve_partitioning=True)
    st6 = Stage(6, P.shuffle_writer(s6, 6))
    fin = [P.field(nme, t, True) for nme, t in zip(gb_names, ktypes)] + [P.field("sum_qty", P.dec(25, 2), True)]
    st7 = Stage(7, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(6, fin), fetch=100), 7), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7]


Q9_TABLES = {"part": ["p_partkey", "p_name"], "supplier": ["s_suppkey", "s_nationkey"], "nation": ["n_nationkey", "n_name"],
             "partsupp": ["ps_partkey", "ps_suppkey", "ps_supplycost"], "orders": ["o_orderkey", "o_orderdate"],
             "lineitem": ["l_orderkey", "l_partkey", "l_suppkey", "l_quantity", "l_extendedprice", "l_discount"]}


def q9(n_partitions: int = 4, pattern: str = "%green%") -> List[Stage]:
    """benchmarks/queries/q9.sql -- six-table join (a two-column key on partsupp), LIKE on p_name, EXTRACT(YEAR ...),
    amount = price*(1-discount) - supplycost*quantity (signed Decimal128(38,4)), GROUP BY nation, o_year
    ORDER BY nation, o_year DESC."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    s1 = P.filter_(P.like(c("p_name"), pattern), table_scan("part", Q9_TABLES["part"]), projection=[0])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    st2 = Stage(2, P.shuffle_writer(table_scan("lineitem", Q9_TABLES["lineitem"]), 2, [c(1)], Pn))
    li = [dict(f, nullable=True) for f in _sch("lineitem", Q9_TABLES["lineitem"])]
    # S3: part' |x| lineitem on partkey -> l_orderkey, l_partkey, l_suppkey, l_quantity, l_extendedprice, l_discount; by (suppkey, partkey)
    s3 = P.hash_join(P.shuffle_reader(1, [P.field("p_partkey", i64, True)]), P.shuffle_reader(2, li), [[c(0), c(1)]], "Inner", "Partitioned",
                     projection=[1, 2, 3, 4, 5, 6])
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(2), c(1)], Pn))
    st4 = Stage(4, P.shuffle_writer(table_scan("partsupp", Q9_TABLES["partsupp"]), 4, [c(1), c(0)], Pn))
    ps = [dict(f, nullable=True) for f in _sch("partsupp", Q9_TABLES["partsupp"])]
    # S5: partsupp |x| (part, lineitem) on (suppkey, partkey) -> l_orderkey, l_suppkey, l_quantity, l_extendedprice, l_discount, ps_supplycost
    s5 = P.hash_join(P.shuffle_reader(4, ps), P.shuffle_reader(3, li), [[c(1), c(2)], [c(0), c(1)]], "Inner", "Partitioned",
                     projection=[3, 5, 6, 7, 8, 2])
    st5 = Stage(5, P.shuffle_writer(s5, 5, [c(1)], Pn))
    pl = [P.field("l_orderkey", i64, True), P.field("l_suppkey", i64, True), P.field("l_quantity", D152, True),
          P.field("l_extendedprice", D152, True), P.field("l_discount", D152, True), P.field("ps_supplycost", D152, True)]
    # S6: nation |x| supplier (tiny, one task) -> s_suppkey, n_name; by suppkey
    s6 = P.hash_join(table_scan("nation", Q9_TABLES["nation"]), table_scan("supplier", Q9_TABLES["supplier"]), [[c(0), c("s_nationkey")]],
                     "Inner", "CollectLeft", projection=[2, 1])
    st6 = Stage(6, P.shuffle_writer(s6, 6, [c(0)], Pn))
    sn = [P.field("s_suppkey", i64, True), P.field("n_name", "utf8", True)]
    # S7: (supplier, nation) |x| ... on suppkey -> l_orderkey, amount inputs, n_name; by orderkey
    s7 = P.hash_join(P.shuffle_reader(6, sn), P.shuffle_reader(5, pl), [[c(0), c(1)]], "Inner", "Partitioned", projection=[2, 4, 5, 6, 7, 1])
    st7 = Stage(7, P.shuffle_writer(s7, 7, [c(0)], Pn))
    sl = [P.field("l_orderkey", i64, True), P.field("l_quantity", D152, True), P.field("l_extendedprice", D152, True), P.field("l_discount", D152, True),
          P.field("ps_supplycost", D152, True), P.field("n_name", "utf8", True)]
    st8 = Stage(8, P.shuffle_writer(table_scan("orders", Q9_TABLES["orders"]), 8, [c(0)], Pn))
    od = [P.field("o_orderkey", i64, True), P.field("o_orderdate", "date32", True)]
    # S9: orders |x| ... on orderkey -> nation, o_year, amount -> partial aggregate
    s9 = P.hash_join(P.shuffle_reader(8, od), P.shuffle_reader(7, sl), [[c(0), c(0)]], "Inner", "Partitioned", projection=[7, 1, 3, 4, 5, 6])
    amount = P.binop("-", P.binop("*", c(3), one_minus(c(4))), P.binop("*", c(5), c(2)))
    s9 = P.project([(c(0), "nation"), (P.fn("date_part_year", c(1)), "o_year"), (amount, "amount")], s9)
    gb = [(c(0), "nation"), (c(1), "o_year")]
    s9 = P.aggregate("Partial", gb, [P.agg("sum", c(2), "sum_profit")], s9)
    st9 = Stage(9, P.shuffle_writer(s9, 9, [c(0), c(1)], Pn))
    part = [P.field("nation", "utf8", True), P.field("o_year", "i32", True), P.field("sum_profit[sum]", P.dec(38, 4), True)]
    s10 = P.aggregate("FinalPartitioned", gb, [P.agg("sum", None, "sum_profit")], P.shuffle_reader(9, part))
    keys = [P.sort_key(c(0)), P.sort_key(c(1), asc=False)]
    s10 = P.sort(keys, s10, preserve_partitioning=True)
    st10 = Stage(10, P.shuffle_writer(s10, 10))
    fin = [P.field("nation", "utf8", True), P.field("o_year", "i32", True), P.field("sum_profit", P.dec(38, 4), True)]
    st11 = Stage(11, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(10, fin)), 11), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7, st8, st9, st10, st11]


Q7_TABLES = {"supplier": ["s_suppkey", "s_nationkey"], "nation": ["n_nationkey", "n_name"], "customer": ["c_custkey", "c_nationkey"],
             "orders": ["o_orderkey", "o_custkey"], "lineitem": ["l_orderkey", "l_suppkey", "l_extendedprice", "l_discount", "l_shipdate"]}


def q7(n_partitions: int = 4, nation_a: str = "FRANCE", nation_b: str = "GERMANY", date_from: str = "1995-01-01", date_to: str = "1996-12-31") -> List[Stage]:
    """benchmarks/queries/q7.sql -- nation joined twice (supplier side, customer side; the IN-lists DataFusion infers from the
    OR are pushed to both scans), the OR of nation pairs as the last join's residual filter, EXTRACT(YEAR FROM l_shipdate),
    GROUP BY supp_nation, cust_nation, l_year ORDER BY the same."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    two = lambda x: P.in_list(x, [P.lit_utf8(nation_a), P.lit_utf8(nation_b)])
    # S1: nation(a|b) |x| supplier -> s_suppkey, n_name ; by suppkey
    n1 = P.filter_(two(c("n_name")), table_scan("nation", Q7_TABLES["nation"]))
    s1 = P.hash_join(n1, table_scan("supplier", Q7_TABLES["supplier"]), [[c(0), c("s_nationkey")]], "Inner", "CollectLeft", projection=[2, 1])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    sn = [P.field("s_suppkey", i64, True), P.field("supp_nation", "utf8", True)]
    # S2: lineitem in the date range ; by suppkey
    s2 = P.filter_(P.and_(P.binop(">=", c("l_shipdate"), P.lit_date(date_from)), P.binop("<=", c("l_shipdate"), P.lit_date(date_to))),
                   table_scan("lineitem", Q7_TABLES["lineitem"]))
    st2 = Stage(2, P.shuffle_writer(s2, 2, [c(1)], Pn))
    li = [dict(f, nullable=True) for f in _sch("lineitem", Q7_TABLES["lineitem"])]
    # S3: supplier' |x| lineitem' -> l_orderkey, l_extendedprice, l_discount, l_shipdate, supp_nation ; by orderkey
    s3 = P.hash_join(P.shuffle_reader(1, sn), P.shuffle_reader(2, li), [[c(0), c(1)]], "Inner", "Partitioned", projection=[2, 4, 5, 6, 1])
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(0)], Pn))
    sl = [P.field("l_orderkey", i64, True), P.field("l_extendedprice", D152, True), P.field("l_discount", D152, True), P.field("l_shipdate", "date32", True),
          P.field("supp_nation", "utf8", True)]
    # S4: nation(a|b) |x| customer -> c_custkey, n_name ; by custkey
    n2 = P.filter_(two(c("n_name")), table_scan("nation", Q7_TABLES["nation"]))
    s4 = P.hash_join(n2, table_scan("customer", Q7_TABLES["customer"]), [[c(0), c("c_nationkey")]], "Inner", "CollectLeft", projection=[2, 1])
    st4 = Stage(4, P.shuffle_writer(s4, 4, [c(0)], Pn))
    cn = [P.field("c_custkey", i64, True), P.field("cust_nation", "utf8", True)]
    st5 = Stage(5, P.shuffle_writer(table_scan("orders", Q7_TABLES["orders"]), 5, [c(1)], Pn))
    od = [P.field("o_orderkey", i64, True), P.field("o_custkey", i64, True)]
    # S6: customer' |x| orders -> o_orderkey, cust_nation ; by orderkey
    s6 = P.hash_join(P.shuffle_reader(4, cn), P.shuffle_reader(5, od), [[c(0), c(1)]], "Inner", "Partitioned", projection=[2, 1])
    st6 = Stage(6, P.shuffle_writer(s6, 6, [c(0)], Pn))
    oc = [P.field("o_orderkey", i64, True), P.field("cust_nation", "utf8", True)]
    # S7: (orders, customer) |x| (supplier, lineitem) on orderkey, residual = the two nation pairs
    pair = P.or_(P.and_(P.binop("=", c(6), P.lit_utf8(nation_a)), P.binop("=", c(1), P.lit_utf8(nation_b))),
                 P.and_(P.binop("=", c(6), P.lit_utf8(nation_b)), P.binop("=", c(1), P.lit_utf8(nation_a))))
    j = P.hash_join(P.shuffle_reader(6, oc), P.shuffle_reader(3, sl), [[c(0), c(0)]], "Inner", "Partitioned", filter=pair, projection=[6, 1, 5, 3, 4])
    s7 = P.project([(c(0), "supp_nation"), (c(1), "cust_nation"), (P.fn("date_part_year", c(2)), "l_year"),
                    (P.binop("*", c(3), one_minus(c(4))), "volume")], j)
    gb = [(c(0), "supp_nation"), (c(1), "cust_nation"), (c(2), "l_year")]
    s7 = P.aggregate("Partial", gb, [P.agg("sum", c(3), "revenue")], s7)
    st7 = Stage(7, P.shuffle_writer(s7, 7, [c(0), c(1), c(2)], Pn))
    part = [P.field("supp_nation", "utf8", True), P.field("cust_nation", "utf8", True), P.field("l_year", "i32", True), P.field("revenue[sum]", P.dec(38, 4), True)]
    s8 = P.aggregate("FinalPartitioned", gb, [P.agg("sum", None, "revenue")], P.shuffle_reader(7, part))
    keys = [P.sort_key(c(0)), P.sort_key(c(1)), P.sort_key(c(2))]
    s8 = P.sort(keys, s8, preserve_partitioning=True)
    st8 = Stage(8, P.shuffle_writer(s8, 8))
    fin = [P.field("supp_nation", "utf8", True), P.field("cust_nation", "utf8", True), P.field("l_year", "i32", True), P.field("revenue", P.dec(38, 4), True)]
    st9 = Stage(9, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(8, fin)), 9), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7, st8, st9]


Q16_TABLES = {"part": ["p_partkey", "p_brand", "p_type", "p_size"], "partsupp": ["ps_partkey", "ps_suppkey"], "supplier": ["s_suppkey", "s_comment"]}


def q16(n_partitions: int = 4, brand: str = "Brand#45", type_prefix: str = "MEDIUM POLISHED%", sizes=(49, 14, 23, 45, 19, 3, 36, 9),
        complaint: str = "%Customer%Complaints%") -> List[Stage]:
    """benchmarks/queries/q16.sql -- NOT IN (subquery) as an anti join, <> / NOT LIKE / IN filters, and COUNT(DISTINCT ps_suppkey)
    in the two-level form DataFusion's SingleDistinctToGroupBy rule produces (group by keys + the distinct column, then count)."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    s1 = P.filter_(P.like(c("s_comment"), complaint), table_scan("supplier", Q16_TABLES["supplier"]), projection=[0])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    pred = P.and_(P.binop("<>", c("p_brand"), P.lit_utf8(brand)), P.like(c("p_type"), type_prefix, negated=True),
                  P.in_list(c("p_size"), [P.lit_i32(int(v)) for v in sizes]))
    st2 = Stage(2, P.shuffle_writer(P.filter_(pred, table_scan("part", Q16_TABLES["part"])), 2, [c(0)], Pn))
    pt = [P.field("p_partkey", i64, True), P.field("p_brand", "utf8", True), P.field("p_type", "utf8", True), P.field("p_size", "i32", True)]
    st3 = Stage(3, P.shuffle_writer(table_scan("partsupp", Q16_TABLES["partsupp"]), 3, [c(0)], Pn))
    ps = [P.field("ps_partkey", i64, True), P.field("ps_suppkey", i64, True)]
    # S4: part' |x| partsupp -> ps_suppkey, p_brand, p_type, p_size ; by suppkey
    s4 = P.hash_join(P.shuffle_reader(2, pt), P.shuffle_reader(3, ps), [[c(0), c(0)]], "Inner", "Partitioned", projection=[5, 1, 2, 3])
    st4 = Stage(4, P.shuffle_writer(s4, 4, [c(0)], Pn))
    pp = [P.field("ps_suppkey", i64, True), P.field("p_brand", "utf8", True), P.field("p_type", "utf8", True), P.field("p_size", "i32", True)]
    # S5: NOT IN complaints: keep probe rows without a match (RightAnti), then the inner level of the distinct count
    anti = P.hash_join(P.shuffle_reader(1, [P.field("s_suppkey", i64, True)]), P.shuffle_reader(4, pp), [[c(0), c(0)]], "RightAnti", "Partitioned")
    gb4 = [(c(1), "p_brand"), (c(2), "p_type"), (c(3), "p_size"), (c(0), "ps_suppkey")]
    s5 = P.aggregate("Partial", gb4, [], anti)
    st5 = Stage(5, P.shuffle_writer(s5, 5, [c(0), c(1), c(2), c(3)], Pn))
    d4 = [P.field("p_brand", "utf8", True), P.field("p_type", "utf8", True), P.field("p_size", "i32", True), P.field("ps_suppkey", i64, True)]
    s6 = P.aggregate("FinalPartitioned", [(c(0), "p_brand"), (c(1), "p_type"), (c(2), "p_size"), (c(3), "ps_suppkey")], [], P.shuffle_reader(5, d4))
    gb3 = [(c(0), "p_brand"), (c(1), "p_type"), (c(2), "p_size")]
    s6 = P.aggregate("Partial", gb3, [P.agg("count", c(3), "supplier_cnt")], s6)
    st6 = Stage(6, P.shuffle_writer(s6, 6, [c(0), c(1), c(2)], Pn))
    part = [P.field("p_brand", "utf8", True), P.field("p_type", "utf8", True), P.field("p_size", "i32", True), P.field("supplier_cnt[count]", i64)]
    s7 = P.aggregate("FinalPartitioned", gb3, [P.agg("count", None, "supplier_cnt")], P.shuffle_reader(6, part))
    keys = [P.sort_key(c(3), asc=False), P.sort_key(c(0)), P.sort_key(c(1)), P.sort_key(c(2))]
    s7 = P.sort(keys, s7, preserve_partitioning=True)
    st7 = Stage(7, P.shuffle_writer(s7, 7))
    fin = [P.field("p_brand", "utf8", True), P.field("p_type", "utf8", True), P.field("p_size", "i32", True), P.field("supplier_cnt", i64)]
    st8 = Stage(8, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(7, fin)), 8), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7, st8]


Q21_TABLES = {"supplier": ["s_suppkey", "s_name", "s_nationkey"], "nation": ["n_nationkey", "n_name"], "orders": ["o_orderkey", "o_orderstatus"],
              "lineitem": ["l_orderkey", "l_suppkey", "l_commitdate", "l_receiptdate"]}


def q21(n_partitions: int = 4, nation: str = "SAUDI ARABIA", status: str = "F") -> List[Stage]:
    """benchmarks/queries/q21.sql -- EXISTS / NOT EXISTS with inequality correlation (`l2.l_suppkey <> l1.l_suppkey`) as semi /
    anti joins with residual filters over three readings of lineitem; COUNT(*) GROUP BY s_name, top-100."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    late = P.binop(">", c("l_receiptdate"), c("l_commitdate"))
    nat = P.filter_(P.binop("=", c("n_name"), P.lit_utf8(nation)), table_scan("nation", Q21_TABLES["nation"]), projection=[0])
    s1 = P.hash_join(nat, table_scan("supplier", Q21_TABLES["supplier"]), [[c(0), c("s_nationkey")]], "Inner", "CollectLeft", projection=[1, 2])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    sup = [P.field("s_suppkey", i64, True), P.field("s_name", "utf8", True)]
    st2 = Stage(2, P.shuffle_writer(P.filter_(late, table_scan("lineitem", Q21_TABLES["lineitem"]), projection=[0, 1]), 2, [c(1)], Pn))
    lk = [P.field("l_orderkey", i64, True), P.field("l_suppkey", i64, True)]
    # S3: supplier' |x| l1 -> s_name, l_orderkey, l_suppkey ; by orderkey
    s3 = P.hash_join(P.shuffle_reader(1, sup), P.shuffle_reader(2, lk), [[c(0), c(1)]], "Inner", "Partitioned", projection=[1, 2, 3])
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(1)], Pn))
    t1 = [P.field("s_name", "utf8", True), P.field("l_orderkey", i64, True), P.field("l_suppkey", i64, True)]
    st4 = Stage(4, P.shuffle_writer(P.filter_(P.binop("=", c("o_orderstatus"), P.lit_utf8(status)), table_scan("orders", Q21_TABLES["orders"]), projection=[0]),
                                    4, [c(0)], Pn))
    st5 = Stage(5, P.shuffle_writer(P.project([(c("l_orderkey"), "l_orderkey"), (c("l_suppkey"), "l_suppkey")], table_scan("lineitem", Q21_TABLES["lineitem"])),
                                    5, [c(0)], Pn))
    st6 = Stage(6, P.shuffle_writer(P.filter_(late, table_scan("lineitem", Q21_TABLES["lineitem"]), projection=[0, 1]), 6, [c(0)], Pn))
    # S7, everything co-partitioned on the order key
    t = P.hash_join(P.shuffle_reader(4, [P.field("o_orderkey", i64, True)]), P.shuffle_reader(3, t1), [[c(0), c(1)]], "Inner", "Partitioned", projection=[1, 2, 3])
    # EXISTS l2: another supplier has a line in the same order   (filter columns: l2 = 0..1, t = 2..4)
    other = P.binop("<>", c(1), c(4))
    t = P.hash_join(P.shuffle_reader(5, lk), t, [[c(0), c(1)]], "RightSemi", "Partitioned", filter=other)
    # NOT EXISTS l3: no other supplier was late on that order
    t = P.hash_join(P.shuffle_reader(6, lk), t, [[c(0), c(1)]], "RightAnti", "Partitioned", filter=other)
    s7 = P.aggregate("Partial", [(c(0), "s_name")], [P.agg("count", None, "numwait")], t)
    st7 = Stage(7, P.shuffle_writer(s7, 7, [c(0)], Pn))
    part = [P.field("s_name", "utf8", True), P.field("numwait[count]", i64)]
    s8 = P.aggregate("FinalPartitioned", [(c(0), "s_name")], [P.agg("count", None, "numwait")], P.shuffle_reader(7, part))
    keys = [P.sort_key(c(1), asc=False), P.sort_key(c(0))]
    s8 = P.sort(keys, s8, fetch=100, preserve_partitioning=True)
    st8 = Stage(8, P.shuffle_writer(s8, 8))
    fin = [P.field("s_name", "utf8", True), P.field("numwait", i64)]
    st9 = Stage(9, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(8, fin), fetch=100), 9), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7, st8, st9]


# ---- q14: join + SUM(CASE WHEN p_type LIKE 'PROMO%' ...) / SUM(...) in fp64 (the 100.00 literal is a Float64) ----------
Q14_TABLES = {"lineitem": ["l_partkey", "l_extendedprice", "l_discount", "l_shipdate"], "part": ["p_partkey", "p_type"]}
D384 = P.dec(38, 4)


def q14(n_partitions: int = 4, date_from: str = "1995-09-01", date_to: str = "1995-10-01", prefix: str = "PROMO%") -> List[Stage]:
    """benchmarks/queries/q14.sql."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    s1 = P.filter_(P.and_(P.binop(">=", c("l_shipdate"), P.lit_date(date_from)), P.binop("<", c("l_shipdate"), P.lit_date(date_to))),
                   table_scan("lineitem", Q14_TABLES["lineitem"]), projection=[0, 1, 2])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    st2 = Stage(2, P.shuffle_writer(table_scan("part", Q14_TABLES["part"]), 2, [c(0)], Pn))
    li = [P.field("l_partkey", i64, True), P.field("l_extendedprice", D152, True), P.field("l_discount", D152, True)]
    pt = [P.field("p_partkey", i64, True), P.field("p_type", "utf8", True)]
    j = P.hash_join(P.shuffle_reader(2, pt), P.shuffle_reader(1, li), [[c(0), c(0)]], "Inner", "Partitioned", projection=[1, 3, 4])
    vol = P.binop("*", c(1), one_minus(c(2)))
    s3 = P.project([(P.case([[P.like(c(0), prefix), vol]], P.lit_dec(0, 38, 4)), "promo"), (vol, "rev")], j)
    s3 = P.aggregate("Partial", [], [P.agg("sum", c(0), "promo"), P.agg("sum", c(1), "rev")], s3)
    st3 = Stage(3, P.shuffle_writer(s3, 3))
    part = [P.field("promo[sum]", D384, True), P.field("rev[sum]", D384, True)]
    s4 = P.aggregate("Final", [], [P.agg("sum", None, "promo"), P.agg("sum", None, "rev")], P.coalesce_partitions(P.shuffle_reader(3, part)))
    s4 = P.project([(P.binop("/", P.binop("*", P.lit_f64(100.0), P.cast(c(0), "f64")), P.cast(c(1), "f64")), "promo_revenue")], s4)
    return [st1, st2, st3, Stage(4, P.shuffle_writer(s4, 4), n_tasks=1)]


# ---- q8: eight-table join, CASE inside SUM, decimal division ------------------------------------------------------
Q8_TABLES = {"part": ["p_partkey", "p_type"], "supplier": ["s_suppkey", "s_nationkey"],
             "lineitem": ["l_orderkey", "l_partkey", "l_suppkey", "l_extendedprice", "l_discount"],
             "orders": ["o_orderkey", "o_custkey", "o_orderdate"], "customer": ["c_custkey", "c_nationkey"],
             "nation": ["n_nationkey", "n_name", "n_regionkey"], "region": ["r_regionkey", "r_name"]}


def q8(n_partitions: int = 4, nation: str = "BRAZIL", region: str = "AMERICA", ptype: str = "ECONOMY ANODIZED STEEL",
       date_from: str = "1995-01-01", date_to: str = "1996-12-31") -> List[Stage]:
    """benchmarks/queries/q8.sql -- market share: SUM(CASE WHEN nation = X THEN volume ELSE 0 END) / SUM(volume) per o_year
    (Decimal128(38,4) / Decimal128(38,4) -> Decimal128(38,8) [EXT])."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    s1 = P.filter_(P.binop("=", c("p_type"), P.lit_utf8(ptype)), table_scan("part", Q8_TABLES["part"]), projection=[0])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    st2 = Stage(2, P.shuffle_writer(table_scan("lineitem", Q8_TABLES["lineitem"]), 2, [c(1)], Pn))
    li = [dict(f, nullable=True) for f in _sch("lineitem", Q8_TABLES["lineitem"])]
    # S3: part' |x| lineitem -> l_orderkey, l_suppkey, l_extendedprice, l_discount ; by orderkey
    s3 = P.hash_join(P.shuffle_reader(1, [P.field("p_partkey", i64, True)]), P.shuffle_reader(2, li), [[c(0), c(1)]], "Inner", "Partitioned", projection=[1, 3, 4, 5])
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(0)], Pn))
    pl = [P.field("l_orderkey", i64, True), P.field("l_suppkey", i64, True), P.field("l_extendedprice", D152, True), P.field("l_discount", D152, True)]
    s4 = P.filter_(P.and_(P.binop(">=", c("o_orderdate"), P.lit_date(date_from)), P.binop("<=", c("o_orderdate"), P.lit_date(date_to))),
                   table_scan("orders", Q8_TABLES["orders"]))
    st4 = Stage(4, P.shuffle_writer(s4, 4, [c(0)], Pn))
    od = [P.field("o_orderkey", i64, True), P.field("o_custkey", i64, True), P.field("o_orderdate", "date32", True)]
    # S5: orders' |x| (part, lineitem) on orderkey -> o_custkey, o_orderdate, l_suppkey, l_extendedprice, l_discount ; by custkey
    s5 = P.hash_join(P.shuffle_reader(4, od), P.shuffle_reader(3, pl), [[c(0), c(0)]], "Inner", "Partitioned", projection=[1, 2, 4, 5, 6])
    st5 = Stage(5, P.shuffle_writer(s5, 5, [c(0)], Pn))
    ol = [P.field("o_custkey", i64, True), P.field("o_orderdate", "date32", True), P.field("l_suppkey", i64, True),
          P.field("l_extendedprice", D152, True), P.field("l_discount", D152, True)]
    # S6: customers of the region: region' |x| nation |x| customer -> c_custkey ; by custkey
    reg = P.filter_(P.binop("=", c("r_name"), P.lit_utf8(region)), table_scan("region", Q8_TABLES["region"]), projection=[0])
    n1 = P.hash_join(reg, table_scan("nation", Q8_TABLES["nation"]), [[c(0), c("n_regionkey")]], "Inner", "CollectLeft", projection=[1])
    s6 = P.hash_join(n1, table_scan("customer", Q8_TABLES["customer"]), [[c(0), c("c_nationkey")]], "Inner", "CollectLeft", projection=[1])
    st6 = Stage(6, P.shuffle_writer(s6, 6, [c(0)], Pn))
    # S7: customers' |x| ... on custkey -> o_orderdate, l_suppkey, l_extendedprice, l_discount ; by suppkey
    s7 = P.hash_join(P.shuffle_reader(6, [P.field("c_custkey", i64, True)]), P.shuffle_reader(5, ol), [[c(0), c(0)]], "Inner", "Partitioned", projection=[2, 3, 4, 5])
    st7 = Stage(7, P.shuffle_writer(s7, 7, [c(1)], Pn))
    t7 = [P.field("o_orderdate", "date32", True), P.field("l_suppkey", i64, True), P.field("l_extendedprice", D152, True), P.field("l_discount", D152, True)]
    # S8: nation n2 |x| supplier -> s_suppkey, n_name ; by suppkey
    n2 = P.project([(c("n_nationkey"), "n_nationkey"), (c("n_name"), "n_name")], table_scan("nation", Q8_TABLES["nation"]))
    s8 = P.hash_join(n2, table_scan("supplier", Q8_TABLES["supplier"]), [[c(0), c("s_nationkey")]], "Inner", "CollectLeft", projection=[2, 1])
    st8 = Stage(8, P.shuffle_writer(s8, 8, [c(0)], Pn))
    sn = [P.field("s_suppkey", i64, True), P.field("n_name", "utf8", True)]
    # S9: -> o_year, volume, nation -> partial aggregate
    s9 = P.hash_join(P.shuffle_reader(8, sn), P.shuffle_reader(7, t7), [[c(0), c(1)]], "Inner", "Partitioned", projection=[1, 2, 4, 5])
    vol = P.binop("*", c(2), one_minus(c(3)))
    s9 = P.project([(P.fn("date_part_year", c(1)), "o_year"), (P.case([[P.binop("=", c(0), P.lit_utf8(nation)), vol]], P.lit_dec(0, 38, 4)), "nat_volume"),
                    (vol, "volume")], s9)
    gb = [(c(0), "o_year")]
    s9 = P.aggregate("Partial", gb, [P.agg("sum", c(1), "nat"), P.agg("sum", c(2), "tot")], s9)
    st9 = Stage(9, P.shuffle_writer(s9, 9, [c(0)], Pn))
    part = [P.field("o_year", "i32", True), P.field("nat[sum]", D384, True), P.field("tot[sum]", D384, True)]
    s10 = P.aggregate("FinalPartitioned", gb, [P.agg("sum", None, "nat"), P.agg("sum", None, "tot")], P.shuffle_reader(9, part))
    s10 = P.project([(c(0), "o_year"), (P.binop("/", c(1), c(2)), "mkt_share")], s10)
    keys = [P.sort_key(c(0))]
    s10 = P.sort(keys, s10, preserve_partitioning=True)
    st10 = Stage(10, P.shuffle_writer(s10, 10))
    fin = [P.field("o_year", "i32", True), P.field("mkt_share", P.dec(38, 8), True)]
    st11 = Stage(11, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(10, fin)), 11), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7, st8, st9, st10, st11]


def _with_const_key(plan, n_cols: int):
    """plan + a constant Int64 column: a scalar subquery's single row joins every row through it."""
    return P.project([(P.col(i), f"c{i}") for i in range(n_cols)] + [(P.lit_i64(1), "__one")], plan)


# ---- q11: HAVING sum > (scalar subquery) * 0.0001 -- the scalar joins as a broadcast one-row build side ---------------
Q11_TABLES = {"partsupp": ["ps_partkey", "ps_suppkey", "ps_availqty", "ps_supplycost"], "supplier": ["s_suppkey", "s_nationkey"],
              "nation": ["n_nationkey", "n_name"]}


def q11(n_partitions: int = 4, nation: str = "GERMANY", fraction: float = 0.0001) -> List[Stage]:
    """benchmarks/queries/q11.sql -- value = SUM(ps_supplycost * ps_availqty) per part (Decimal128(15,2) x Int32->Decimal128(10,0)
    = Decimal128(26,2), SUM -> (36,2)); the threshold is fp64 because 0.0001 is a Float64 literal."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    nat = P.filter_(P.binop("=", c("n_name"), P.lit_utf8(nation)), table_scan("nation", Q11_TABLES["nation"]), projection=[0])
    s1 = P.hash_join(nat, table_scan("supplier", Q11_TABLES["supplier"]), [[c(0), c("s_nationkey")]], "Inner", "CollectLeft", projection=[1])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    st2 = Stage(2, P.shuffle_writer(table_scan("partsupp", Q11_TABLES["partsupp"]), 2, [c(1)], Pn))
    ps = [dict(f, nullable=True) for f in _sch("partsupp", Q11_TABLES["partsupp"])]
    s3 = P.hash_join(P.shuffle_reader(1, [P.field("s_suppkey", i64, True)]), P.shuffle_reader(2, ps), [[c(0), c(1)]], "Inner", "Partitioned", projection=[1, 3, 4])
    s3 = P.project([(c(0), "ps_partkey"), (P.binop("*", c(2), P.cast(c(1), P.dec(10, 0))), "v")], s3)
    gb = [(c(0), "ps_partkey")]
    s3 = P.aggregate("Partial", gb, [P.agg("sum", c(1), "value")], s3)
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(0)], Pn))
    D362 = P.dec(36, 2)
    part = [P.field("ps_partkey", i64, True), P.field("value[sum]", D362, True)]
    s4 = P.aggregate("FinalPartitioned", gb, [P.agg("sum", None, "value")], P.shuffle_reader(3, part))
    st4 = Stage(4, P.shuffle_writer(s4, 4))
    pv = [P.field("ps_partkey", i64, True), P.field("value", D362, True)]
    s5 = P.aggregate("Partial", [], [P.agg("sum", c(1), "total")], P.shuffle_reader(4, pv))
    st5 = Stage(5, P.shuffle_writer(s5, 5))
    s6 = P.aggregate("Final", [], [P.agg("sum", None, "total")], P.coalesce_partitions(P.shuffle_reader(5, [P.field("total[sum]", P.dec(38, 2), True)])))
    s6 = P.project([(P.binop("*", P.cast(c(0), "f64"), P.lit_f64(fraction)), "thr"), (P.lit_i64(1), "__one")], s6)
    st6 = Stage(6, P.shuffle_writer(s6, 6), n_tasks=1)
    thr = [P.field("thr", "f64", True), P.field("__one", i64, True)]
    probe = _with_const_key(P.shuffle_reader(4, pv), 2)
    # filter columns: thr, __one | c0 (ps_partkey), c1 (value), __one
    j = P.hash_join(P.shuffle_reader(6, thr, broadcast=True), probe, [[c(1), c(2)]], "Inner", "CollectLeft",
                    filter=P.binop(">", P.cast(c(3), "f64"), c(0)), projection=[2, 3])
    j = P.project([(c(0), "ps_partkey"), (c(1), "value")], j)
    keys = [P.sort_key(c(1), asc=False)]
    st7 = Stage(7, P.shuffle_writer(P.sort(keys, j, preserve_partitioning=True), 7))
    st8 = Stage(8, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(7, pv)), 8), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7, st8]


# ---- q15: the revenue0 view evaluated once, its MAX joined back as a one-row build side --------------------------
Q15_TABLES = {"lineitem": ["l_suppkey", "l_extendedprice", "l_discount", "l_shipdate"], "supplier": ["s_suppkey", "s_name", "s_address", "s_phone"]}


def q15(n_partitions: int = 4, date_from: str = "1996-01-01", date_to: str = "1996-04-01") -> List[Stage]:
    """benchmarks/queries/q15.sql (CREATE VIEW revenue0 ...; SELECT ...; DROP VIEW -- benchmarks/src/bin/tpch.rs:720-749 runs the
    three statements; the view is inlined here)."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    s1 = P.filter_(P.and_(P.binop(">=", c("l_shipdate"), P.lit_date(date_from)), P.binop("<", c("l_shipdate"), P.lit_date(date_to))),
                   table_scan("lineitem", Q15_TABLES["lineitem"]), projection=[0, 1, 2])
    s1 = P.project([(c(0), "supplier_no"), (P.binop("*", c(1), one_minus(c(2))), "rev")], s1)
    gb = [(c(0), "supplier_no")]
    s1 = P.aggregate("Partial", gb, [P.agg("sum", c(1), "total_revenue")], s1)
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    part = [P.field("supplier_no", i64, True), P.field("total_revenue[sum]", D384, True)]
    s2 = P.aggregate("FinalPartitioned", gb, [P.agg("sum", None, "total_revenue")], P.shuffle_reader(1, part))
    st2 = Stage(2, P.shuffle_writer(s2, 2))
    rv = [P.field("supplier_no", i64, True), P.field("total_revenue", D384, True)]
    st3 = Stage(3, P.shuffle_writer(P.aggregate("Partial", [], [P.agg("max", c(1), "m")], P.shuffle_reader(2, rv)), 3))
    s4 = P.aggregate("Final", [], [P.agg("max", None, "m")], P.coalesce_partitions(P.shuffle_reader(3, [P.field("m[max]", D384, True)])))
    s4 = P.project([(c(0), "m"), (P.lit_i64(1), "__one")], s4)
    st4 = Stage(4, P.shuffle_writer(s4, 4), n_tasks=1)
    mx = [P.field("m", D384, True), P.field("__one", i64, True)]
    # filter columns: m, __one | c0 (supplier_no), c1 (total_revenue), __one
    j = P.hash_join(P.shuffle_reader(4, mx, broadcast=True), _with_const_key(P.shuffle_reader(2, rv), 2), [[c(1), c(2)]], "Inner", "CollectLeft",
                    filter=P.binop("=", c(3), c(0)), projection=[2, 3])
    st5 = Stage(5, P.shuffle_writer(j, 5, [c(0)], Pn))
    st6 = Stage(6, P.shuffle_writer(table_scan("supplier", Q15_TABLES["supplier"]), 6, [c(0)], Pn))
    sp = [dict(f, nullable=True) for f in _sch("supplier", Q15_TABLES["supplier"])]
    rj = [P.field("c0", i64, True), P.field("c1", D384, True)]
    s7 = P.hash_join(P.shuffle_reader(5, rj), P.shuffle_reader(6, sp), [[c(0), c(0)]], "Inner", "Partitioned", projection=[2, 3, 4, 5, 1])
    s7 = P.project([(c(0), "s_suppkey"), (c(1), "s_name"), (c(2), "s_address"), (c(3), "s_phone"), (c(4), "total_revenue")], s7)
    keys = [P.sort_key(c(0))]
    st7 = Stage(7, P.shuffle_writer(P.sort(keys, s7, preserve_partitioning=True), 7))
    fin = [P.field("s_suppkey", i64, True), P.field("s_name", "utf8", True), P.field("s_address", "utf8", True), P.field("s_phone", "utf8", True),
           P.field("total_revenue", D384, True)]
    st8 = Stage(8, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(7, fin)), 8), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7, st8]


# ---- q2: correlated MIN subquery decorrelated into a per-part aggregate joined back -------------------------------
Q2_TABLES = {"part": ["p_partkey", "p_mfgr", "p_type", "p_size"],
             "supplier": ["s_suppkey", "s_name", "s_address", "s_nationkey", "s_phone", "s_acctbal", "s_comment"],
             "partsupp": ["ps_partkey", "ps_suppkey", "ps_supplycost"], "nation": ["n_nationkey", "n_name", "n_regionkey"],
             "region": ["r_regionkey", "r_name"]}


def q2(n_partitions: int = 4, size: int = 15, type_suffix: str = "%BRASS", region: str = "EUROPE") -> List[Stage]:
    """benchmarks/queries/q2.sql -- minimum-cost supplier of the region per part, top 100 by s_acctbal DESC, n_name, s_name, p_partkey."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    reg = P.filter_(P.binop("=", c("r_name"), P.lit_utf8(region)), table_scan("region", Q2_TABLES["region"]), projection=[0])
    nat = P.hash_join(reg, table_scan("nation", Q2_TABLES["nation"]), [[c(0), c("n_regionkey")]], "Inner", "CollectLeft", projection=[1, 2])
    # nation'(n_nationkey, n_name) |x| supplier -> s_suppkey, s_name, s_address, s_phone, s_acctbal, s_comment, n_name ; by suppkey
    s1 = P.hash_join(nat, table_scan("supplier", Q2_TABLES["supplier"]), [[c(0), c("s_nationkey")]], "Inner", "CollectLeft", projection=[2, 3, 4, 6, 7, 8, 1])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    sup = [P.field("s_suppkey", i64, True), P.field("s_name", "utf8", True), P.field("s_address", "utf8", True), P.field("s_phone", "utf8", True),
           P.field("s_acctbal", D152, True), P.field("s_comment", "utf8", True), P.field("n_name", "utf8", True)]
    st2 = Stage(2, P.shuffle_writer(table_scan("partsupp", Q2_TABLES["partsupp"]), 2, [c(1)], Pn))
    ps = [dict(f, nullable=True) for f in _sch("partsupp", Q2_TABLES["partsupp"])]
    # S3: suppliers of the region |x| partsupp -> ps_partkey, ps_supplycost, s_acctbal, s_name, n_name, s_address, s_phone, s_comment ; by partkey
    s3 = P.hash_join(P.shuffle_reader(1, sup), P.shuffle_reader(2, ps), [[c(0), c(1)]], "Inner", "Partitioned", projection=[7, 9, 4, 1, 6, 2, 3, 5])
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(0)], Pn))
    e = [P.field("ps_partkey", i64, True), P.field("ps_supplycost", D152, True), P.field("s_acctbal", D152, True), P.field("s_name", "utf8", True),
         P.field("n_name", "utf8", True), P.field("s_address", "utf8", True), P.field("s_phone", "utf8", True), P.field("s_comment", "utf8", True)]
    s4 = P.filter_(P.and_(P.binop("=", c("p_size"), P.lit_i32(size)), P.like(c("p_type"), type_suffix)), table_scan("part", Q2_TABLES["part"]), projection=[0, 1])
    st4 = Stage(4, P.shuffle_writer(s4, 4, [c(0)], Pn))
    pt = [P.field("p_partkey", i64, True), P.field("p_mfgr", "utf8", True)]
    # S5 (everything co-partitioned on the part key): min cost per part, joined back with `cost = min`
    m = P.aggregate("SinglePartitioned", [(c(0), "ps_partkey")], [P.agg("min", c(1), "min_cost")], P.shuffle_reader(3, e))
    j1 = P.hash_join(P.shuffle_reader(4, pt), P.shuffle_reader(3, e), [[c(0), c(0)]], "Inner", "Partitioned", projection=[0, 1, 3, 4, 5, 6, 7, 8, 9])
    # filter columns: ps_partkey, min_cost | p_partkey, p_mfgr, cost, s_acctbal, s_name, n_name, s_address, s_phone, s_comment
    j2 = P.hash_join(m, j1, [[c(0), c(0)]], "Inner", "Partitioned", filter=P.binop("=", c(4), c(1)), projection=[5, 6, 7, 2, 3, 8, 9, 10])
    s5 = P.project([(c(0), "s_acctbal"), (c(1), "s_name"), (c(2), "n_name"), (c(3), "p_partkey"), (c(4), "p_mfgr"), (c(5), "s_address"),
                    (c(6), "s_phone"), (c(7), "s_comment")], j2)
    keys = [P.sort_key(c(0), asc=False), P.sort_key(c(2)), P.sort_key(c(1)), P.sort_key(c(3))]
    st5 = Stage(5, P.shuffle_writer(P.sort(keys, s5, fetch=100, preserve_partitioning=True), 5))
    fin = [P.field("s_acctbal", D152, True), P.field("s_name", "utf8", True), P.field("n_name", "utf8", True), P.field("p_partkey", i64, True),
           P.field("p_mfgr", "utf8", True), P.field("s_address", "utf8", True), P.field("s_phone", "utf8", True), P.field("s_comment", "utf8", True)]
    st6 = Stage(6, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(5, fin), fetch=100), 6), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6]


# ---- q20: nested IN subqueries as semi joins, correlated SUM as a two-key aggregate joined with an fp64 residual ----
Q20_TABLES = {"supplier": ["s_suppkey", "s_name", "s_address", "s_nationkey"], "nation": ["n_nationkey", "n_name"],
              "partsupp": ["ps_partkey", "ps_suppkey", "ps_availqty"], "part": ["p_partkey", "p_name"],
              "lineitem": ["l_partkey", "l_suppkey", "l_quantity", "l_shipdate"]}


def q20(n_partitions: int = 4, pattern: str = "forest%", nation: str = "CANADA", date_from: str = "1994-01-01", date_to: str = "1995-01-01") -> List[Stage]:
    """benchmarks/queries/q20.sql -- `ps_availqty > 0.5 * SUM(l_quantity)`: 0.5 is a Float64 literal, so both sides compare as fp64."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    s1 = P.filter_(P.like(c("p_name"), pattern), table_scan("part", Q20_TABLES["part"]), projection=[0])
    st1 = Stage(1, P.shuffle_writer(s1, 1, [c(0)], Pn))
    st2 = Stage(2, P.shuffle_writer(table_scan("partsupp", Q20_TABLES["partsupp"]), 2, [c(0)], Pn))
    ps = [dict(f, nullable=True) for f in _sch("partsupp", Q20_TABLES["partsupp"])]
    s3 = P.hash_join(P.shuffle_reader(1, [P.field("p_partkey", i64, True)]), P.shuffle_reader(2, ps), [[c(0), c(0)]], "RightSemi", "Partitioned")
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(0), c(1)], Pn))
    s4 = P.filter_(P.and_(P.binop(">=", c("l_shipdate"), P.lit_date(date_from)), P.binop("<", c("l_shipdate"), P.lit_date(date_to))),
                   table_scan("lineitem", Q20_TABLES["lineitem"]), projection=[0, 1, 2])
    gb = [(c(0), "l_partkey"), (c(1), "l_suppkey")]
    s4 = P.aggregate("Partial", gb, [P.agg("sum", c(2), "q")], s4)
    st4 = Stage(4, P.shuffle_writer(s4, 4, [c(0), c(1)], Pn))
    part = [P.field("l_partkey", i64, True), P.field("l_suppkey", i64, True), P.field("q[sum]", P.dec(25, 2), True)]
    agg = P.aggregate("FinalPartitioned", gb, [P.agg("sum", None, "q")], P.shuffle_reader(4, part))
    # filter columns: l_partkey, l_suppkey, q | ps_partkey, ps_suppkey, ps_availqty
    j = P.hash_join(agg, P.shuffle_reader(3, ps), [[c(0), c(0)], [c(1), c(1)]], "Inner", "Partitioned",
                    filter=P.binop(">", P.cast(c(5), "f64"), P.binop("*", P.lit_f64(0.5), P.cast(c(2), "f64"))), projection=[4])
    st5 = Stage(5, P.shuffle_writer(j, 5, [c(0)], Pn))
    nat = P.filter_(P.binop("=", c("n_name"), P.lit_utf8(nation)), table_scan("nation", Q20_TABLES["nation"]), projection=[0])
    s6 = P.hash_join(nat, table_scan("supplier", Q20_TABLES["supplier"]), [[c(0), c("s_nationkey")]], "Inner", "CollectLeft", projection=[1, 2, 3])
    st6 = Stage(6, P.shuffle_writer(s6, 6, [c(0)], Pn))
    sp = [P.field("s_suppkey", i64, True), P.field("s_name", "utf8", True), P.field("s_address", "utf8", True)]
    s7 = P.hash_join(P.shuffle_reader(5, [P.field("ps_suppkey", i64, True)]), P.shuffle_reader(6, sp), [[c(0), c(0)]], "RightSemi", "Partitioned")
    s7 = P.project([(c(1), "s_name"), (c(2), "s_address")], s7)
    keys = [P.sort_key(c(0))]
    st7 = Stage(7, P.shuffle_writer(P.sort(keys, s7, preserve_partitioning=True), 7))
    fin = [P.field("s_name", "utf8", True), P.field("s_address", "utf8", True)]
    st8 = Stage(8, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(7, fin)), 8), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7, st8]


# ---- q22: substring, uncorrelated scalar AVG (one-row build side), NOT EXISTS as an anti join -----------------------
Q22_TABLES = {"customer": ["c_custkey", "c_phone", "c_acctbal"], "orders": ["o_custkey"]}


def q22(n_partitions: int = 4, codes=("13", "31", "23", "29", "30", "18", "17")) -> List[Stage]:
    """benchmarks/queries/q22.sql."""
    c, Pn = P.col, n_partitions
    i64 = "i64"
    code = P.fn("substr", c("c_phone"), P.lit_i64(1), P.lit_i64(2))
    in_codes = P.in_list(code, [P.lit_utf8(v) for v in codes])
    cust = table_scan("customer", Q22_TABLES["customer"])
    s1 = P.filter_(P.and_(in_codes, P.binop(">", c("c_acctbal"), P.lit_dec(0, 15, 2))), cust, projection=[2])
    st1 = Stage(1, P.shuffle_writer(P.aggregate("Partial", [], [P.agg("avg", c(0), "a")], s1), 1))
    st_avg = [P.field("a[count]", "u64", True), P.field("a[sum]", P.dec(25, 2), True)]
    s2 = P.aggregate("Final", [], [P.agg("avg", None, "a", D152)], P.coalesce_partitions(P.shuffle_reader(1, st_avg)))
    s2 = P.project([(c(0), "a"), (P.lit_i64(1), "__one")], s2)
    st2 = Stage(2, P.shuffle_writer(s2, 2), n_tasks=1)
    av = [P.field("a", P.dec(19, 6), True), P.field("__one", i64, True)]
    s3 = P.filter_(in_codes, cust)
    s3 = P.project([(c(0), "c_custkey"), (P.fn("substr", c(1), P.lit_i64(1), P.lit_i64(2)), "cntrycode"), (c(2), "c_acctbal"), (P.lit_i64(1), "__one")], s3)
    # filter columns: a, __one | c_custkey, cntrycode, c_acctbal, __one
    s3 = P.hash_join(P.shuffle_reader(2, av, broadcast=True), s3, [[c(1), c(3)]], "Inner", "CollectLeft", filter=P.binop(">", c(4), c(0)), projection=[2, 3, 4])
    st3 = Stage(3, P.shuffle_writer(s3, 3, [c(0)], Pn))
    cu = [P.field("c_custkey", i64, True), P.field("cntrycode", "utf8", True), P.field("c_acctbal", D152, True)]
    st4 = Stage(4, P.shuffle_writer(table_scan("orders", Q22_TABLES["orders"]), 4, [c(0)], Pn))
    s5 = P.hash_join(P.shuffle_reader(4, [P.field("o_custkey", i64, True)]), P.shuffle_reader(3, cu), [[c(0), c(0)]], "RightAnti", "Partitioned")
    gb = [(c(1), "cntrycode")]
    s5 = P.aggregate("Partial", gb, [P.agg("count", None, "numcust"), P.agg("sum", c(2), "totacctbal")], s5)
    st5 = Stage(5, P.shuffle_writer(s5, 5, [c(0)], Pn))
    part = [P.field("cntrycode", "utf8", True), P.field("numcust[count]", i64), P.field("totacctbal[sum]", P.dec(25, 2), True)]
    s6 = P.aggregate("FinalPartitioned", [(c(0), "cntrycode")], [P.agg("count", None, "numcust"), P.agg("sum", None, "totacctbal")], P.shuffle_reader(5, part))
    keys = [P.sort_key(c(0))]
    st6 = Stage(6, P.shuffle_writer(P.sort(keys, s6, preserve_partitioning=True), 6))
    fin = [P.field("cntrycode", "utf8", True), P.field("numcust", i64), P.field("totacctbal", P.dec(25, 2), True)]
    st7 = Stage(7, P.shuffle_writer(P.sort_preserving_merge(keys, P.shuffle_reader(6, fin)), 7), n_tasks=1)
    return [st1, st2, st3, st4, st5, st6, st7]


# ---- q11 / q22 as DataFusion plans them: the scalar subquery's one row is the build side of a NestedLoopJoinExec ----
# whose filter is the comparison (q11 / q22 above join it through an invented constant key instead)
def q11_nlj(n_partitions: int = 4, nation: str = "GERMANY", fraction: float = 0.0001) -> List[Stage]:
    c = P.col
    stages = q11(n_partitions, nation, fraction)
    s6 = P.aggregate("Final", [], [P.agg("sum", None, "total")], P.coalesce_partitions(P.shuffle_reader(5, [P.field("total[sum]", P.dec(38, 2), True)])))
    s6 = P.project([(P.binop("*", P.cast(c(0), "f64"), P.lit_f64(fraction)), "thr")], s6)
    pv = [P.field("ps_partkey", "i64", True), P.field("value", P.dec(36, 2), True)]
    # filter columns: thr | ps_partkey, value
    j = P.nested_loop_join(P.shuffle_reader(6, [P.field("thr", "f64", True)], broadcast=True), P.shuffle_reader(4, pv), "Inner",
                           filter=P.binop(">", P.cast(c(2), "f64"), c(0)), projection=[1, 2])
    keys = [P.sort_key(c(1), asc=False)]
    stages[5] = Stage(6, P.shuffle_writer(s6, 6), n_tasks=1)
    stages[6] = Stage(7, P.shuffle_writer(P.sort(keys, j, preserve_partitioning=True), 7))
    return stages


def q22_nlj(n_partitions: int = 4, codes=("13", "31", "23", "29", "30", "18", "17")) -> List[Stage]:
    c, Pn = P.col, n_partitions
    stages = q22(n_partitions, codes)
    st_avg = [P.field("a[count]", "u64", True), P.field("a[sum]", P.dec(25, 2), True)]
    s2 = P.aggregate("Final", [], [P.agg("avg", None, "a", D152)], P.coalesce_partitions(P.shuffle_reader(1, st_avg)))
    code = P.fn("substr", c("c_phone"), P.lit_i64(1), P.lit_i64(2))
    s3 = P.filter_(P.in_list(code, [P.lit_utf8(v) for v in codes]), table_scan("customer", Q22_TABLES["customer"]))
    s3 = P.project([(c(0), "c_custkey"), (P.fn("substr", c(1), P.lit_i64(1), P.lit_i64(2)), "cntrycode"), (c(2), "c_acctbal")], s3)
    # filter columns: a | c_custkey, cntrycode, c_acctbal ; c_acctbal > a compares as Decimal128(19, 6), AVG's result type
    s3 = P.nested_loop_join(P.shuffle_reader(2, [P.field("a", P.dec(19, 6), True)], broadcast=True), s3, "Inner",
                            filter=P.binop(">", P.cast(c(3), P.dec(19, 6)), c(0)), projection=[1, 2, 3])
    stages[1] = Stage(2, P.shuffle_writer(s2, 2), n_tasks=1)
    stages[2] = Stage(3, P.shuffle_writer(s3, 3, [c(0)], Pn))
    return stages


# ---- registry: query name -> (tables it scans with the columns it references, stage-plan builder) -------------
QUERIES = {
    "q1": ({"lineitem": Q1_COLUMNS}, q1), "q3": (Q3_TABLES, q3), "q4": (Q4_TABLES, q4), "q5": (Q5_TABLES, q5),
    "q6": ({"lineitem": Q6_COLUMNS}, q6), "q7": (Q7_TABLES, q7), "q9": (Q9_TABLES, q9), "q10": (Q10_TABLES, q10),
    "q12": (Q12_TABLES, q12), "q13": (Q13_TABLES, q13), "q16": (Q16_TABLES, q16), "q17": (Q17_TABLES, q17),
    "q18": (Q18_TABLES, q18), "q19": (Q19_TABLES, q19), "q21": (Q21_TABLES, q21),
    "q2": (Q2_TABLES, q2), "q8": (Q8_TABLES, q8), "q11": (Q11_TABLES, q11), "q14": (Q14_TABLES, q14), "q15": (Q15_TABLES, q15),
    "q20": (Q20_TABLES, q20), "q22": (Q22_TABLES, q22),
}


def union_tables(names) -> dict:
    """{table: [columns]} covering every query in `names` (each table registered once, scans carry projections)."""
    out: dict = {}
    for n in names:
        for t, cols in QUERIES[n][0].items():
            out.setdefault(t, [])
            out[t] += [c for c in cols if c not in out[t]]
    return out


def base_rows(name: str, rows_of: dict) -> int:
    """Base-table rows a query scans (the numerator of the rows/s metric, SURVEY.md 8(d))."""
    return sum(rows_of[t] for t in QUERIES[name][0])
