"""NestedLoopJoinExec without a GPU: the CPU oracle against independent computations (a pure-Python cross product + filter
in three-valued logic, and sqlite3), the typed plan of the node, and the protobuf decoder's variant 22."""
import json
import sqlite3

import pytest

from ballista_b200 import engine
from ballista_b200 import plan as P
import nlj_cases as N


@pytest.fixture(scope="module")
def tables():
    return N.make_table(23, seed=1), N.make_table(31, seed=2)


@pytest.mark.parametrize("jt", N.JOIN_TYPES)
@pytest.mark.parametrize("fname", sorted(N.FILTERS))
def test_oracle_matches_cross_product(oracle, tables, jt, fname):
    """Every join type x every filter shape, in the output order the device reproduces: pairs by probe row, build rows in
    order inside a probe row, then unmatched build rows, then unmatched probe rows."""
    left, right = tables
    N.register(oracle, left, right)
    got = N.rows_of(N.run_join(oracle, f"o-{jt}-{fname}", jt, N.FILTERS[fname]))
    want = N.reference_join(left, right, jt, N.FILTERS[fname])
    assert N.same_rows(got, want)


def test_not_with_null_operand_drops_the_pair(oracle):
    """NOT (a < b) with a NULL a is NULL, not TRUE: a two-valued evaluation would keep the pair."""
    left = N.make_table(3, seed=3, null_every=1)     # every nullable column NULL
    right = N.make_table(4, seed=4, null_every=1000)
    N.register(oracle, left, right)
    got = N.rows_of(N.run_join(oracle, "o-not", "Inner", N.FILTERS["not_lt"]))
    assert got == []
    anti = N.rows_of(N.run_join(oracle, "o-not-anti", "LeftAnti", N.FILTERS["not_lt"]))
    assert len(anti) == 3


@pytest.mark.parametrize("shape", ["empty_build", "empty_probe", "one_row_build"])
@pytest.mark.parametrize("jt", N.JOIN_TYPES)
def test_oracle_edge_sizes(oracle, shape, jt):
    nb, np_ = {"empty_build": (0, 9), "empty_probe": (7, 0), "one_row_build": (1, 40)}[shape]
    left, right = N.make_table(nb, seed=5), N.make_table(np_, seed=6)
    N.register(oracle, left, right)
    for fname in ("none", "int_lt"):
        got = N.rows_of(N.run_join(oracle, f"o-{shape}-{jt}-{fname}", jt, N.FILTERS[fname]))
        assert N.same_rows(got, N.reference_join(left, right, jt, N.FILTERS[fname]))


_SQL_JOIN = {"Inner": "JOIN", "Left": "LEFT JOIN", "Right": "RIGHT JOIN", "Full": "FULL JOIN"}
_SQL_FILTERS = {"int_lt": "l.i < r.i", "date_ge": "l.dt >= r.dt", "utf8_lt": "l.s < r.s", "band": "r.i >= l.i AND r.i <= l.i + 2",
                "not_lt": "NOT (l.i < r.i)", "or_nulls": "l.i = r.i OR NOT (l.dt > r.dt)", "none": "1"}


@pytest.mark.parametrize("jt", N.JOIN_TYPES)
@pytest.mark.parametrize("fname", sorted(_SQL_FILTERS))
def test_oracle_matches_sqlite(oracle, tables, jt, fname):
    """The same joins in sqlite3 (integer, date and string columns; sqlite compares TEXT bytewise), as multisets."""
    left, right = tables
    N.register(oracle, left, right)
    got = N.rows_of(N.run_join(oracle, f"s-{jt}-{fname}", jt, N.FILTERS[fname]))
    db = sqlite3.connect(":memory:")
    cols = ["k", "i", "dt", "s"]
    for name, t in (("l", left), ("r", right)):
        db.execute(f"CREATE TABLE {name} (k INTEGER, i INTEGER, dt INTEGER, s TEXT)")
        d = t.select(cols).to_pydict()
        days = [None if v is None else (v - v.__class__(1970, 1, 1)).days for v in d["dt"]]
        db.executemany(f"INSERT INTO {name} VALUES (?,?,?,?)", list(zip(d["k"], d["i"], days, d["s"])))
    cond = _SQL_FILTERS[fname]
    if jt in _SQL_JOIN:
        sql = f"SELECT l.k, r.k FROM l {_SQL_JOIN[jt]} r ON {cond}"
        want = [tuple(r) for r in db.execute(sql)]
        have = [(r[N.COL["k"]], r[N.NC + N.COL["k"]]) for r in got]
    else:
        keep, other = ("l", "r") if jt.startswith("Left") else ("r", "l")
        neg = "" if jt.endswith("Semi") else "NOT "
        sql = f"SELECT {keep}.k FROM {keep} WHERE {neg}EXISTS (SELECT 1 FROM {other} AS {other} WHERE {cond})"
        want = [tuple(r) for r in db.execute(sql)]
        have = [(r[N.COL["k"]],) for r in got]
    key = lambda r: tuple(-1 if v is None else v for v in r)  # noqa: E731
    assert sorted(have, key=key) == sorted(want, key=key)


@pytest.mark.parametrize("jt", N.JOIN_TYPES)
def test_typed_plan_schema_and_projection(jt):
    """Output schema and nullability per join type follow the hash join's rules; a projection picks columns."""
    stage = N.join_stage(jt, N.FILTERS["int_lt"])[0]
    typed = json.loads(engine.plan_typed_json(stage.json("j")))
    j = typed["input"]
    assert j["op"] == "NestedLoopJoinExec" and j["join_type"] == jt and "on" not in j and "mode" not in j
    assert j["filter"]["bin"] == "<"
    names = [f["name"] for f in j["schema"]]
    nulls = [f["nullable"] for f in j["schema"]]
    base = [f["name"] for f in N.IR_SCHEMA]
    if jt in ("LeftSemi", "LeftAnti", "RightSemi", "RightAnti"):
        assert names == base
    else:
        assert names == base + base
        assert all(nulls)   # every input column is nullable here
    lf = [dict(f, nullable=False) for f in N.IR_SCHEMA]
    sch = json.loads(engine.plan_typed_json(N.join_stage(jt, None, schema=lf)[0].json("j")))["input"]["schema"]
    nn = [f["nullable"] for f in sch]
    if jt == "Inner" or jt.endswith("Semi") or jt.endswith("Anti"):
        assert not any(nn)
    elif jt == "Left":
        assert nn == [False] * N.NC + [True] * N.NC
    elif jt == "Right":
        assert nn == [True] * N.NC + [False] * N.NC
    else:
        assert all(nn)
    if not (jt.endswith("Semi") or jt.endswith("Anti")):
        proj = json.loads(engine.plan_typed_json(N.join_stage(jt, None, projection=[N.NC + 1, 0])[0].json("j")))["input"]
        assert [f["name"] for f in proj["schema"]] == ["i", "k"] and proj["projection"] == [N.NC + 1, 0]


def test_projection_on_the_oracle(oracle, tables):
    left, right = tables
    N.register(oracle, left, right)
    proj = [N.NC + 1, 0, 6]
    got = N.rows_of(N.run_join(oracle, "o-proj", "Full", N.FILTERS["band"], proj))
    assert N.same_rows(got, N.reference_join(left, right, "Full", N.FILTERS["band"], proj))


def test_hash_join_without_keys_is_still_a_hash_join():
    """HashJoinExec with an empty `on` keeps its own typed form (mode, on); only NestedLoopJoinExec is a nested-loop join."""
    j = P.hash_join(P.scan("nlj_l", N.IR_SCHEMA), P.scan("nlj_r", N.IR_SCHEMA), [], "Inner", "CollectLeft", filter=N.FILTERS["int_lt"])
    typed = json.loads(engine.plan_typed_json(P.Stage(1, P.shuffle_writer(j, 1)).json("j")))["input"]
    assert typed["op"] == "HashJoinExec" and typed["mode"] == "CollectLeft" and typed["on"] == []


def test_nested_loop_join_rejects_keys():
    j = P.nested_loop_join(P.scan("nlj_l", N.IR_SCHEMA), P.scan("nlj_r", N.IR_SCHEMA))
    j["on"] = [[P.col(0), P.col(0)]]
    with pytest.raises(engine.B200Error):
        engine.plan_typed_json(P.Stage(1, P.shuffle_writer(j, 1)).json("j"))


@pytest.mark.parametrize("q", ["q11", "q22"])
def test_tpch_scalar_subquery_as_nested_loop_join(oracle, oracle_lib, q):
    """q11 / q22 as DataFusion plans them (the scalar subquery's row as a nested-loop join's build side) return what the
    constant-key plans return, whose answers tests/test_tpch_queries*.py pin independently."""
    from ballista_b200 import driver, tpch
    from test_tpch_queries import load_tables
    from util import assert_tables_equal
    load_tables(oracle, oracle_lib, 20, tpch.union_tables([q]), 2)
    want = driver.run_stages(oracle, tpch.QUERIES[q][1](4), f"{q}-key")
    got = driver.run_stages(oracle, getattr(tpch, f"{q}_nlj")(4), f"{q}-nlj")
    assert want is not None and want.num_rows > 0
    assert_tables_equal(got, want, sort=False)


with open(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "nlj_proto_plans.json")) as _fh:
    PROTO_CASES = json.load(_fh)["cases"]


def _strip_cosmetic(t):
    if isinstance(t, dict):
        return {k: _strip_cosmetic(v) for k, v in t.items() if not (k == "name" and "col" in t)}
    if isinstance(t, list):
        return [_strip_cosmetic(v) for v in t]
    return t


@pytest.mark.parametrize("case", PROTO_CASES, ids=[c["name"] for c in PROTO_CASES])
def test_proto_plan_decodes_to_its_source(case):
    """NestedLoopJoinExecNode bytes (variant 22, built from the reference's .proto files) type exactly like the IR they encode."""
    import base64
    ir = engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]))
    assert _strip_cosmetic(json.loads(engine.plan_typed_json(ir))) == _strip_cosmetic(json.loads(engine.plan_typed_json(case["ir"])))


def test_proto_damaged_bytes_raise():
    import base64
    import random
    rnd = random.Random(22)
    raws = [base64.b64decode(c["proto_b64"]) for c in PROTO_CASES if c["name"] in ("q11_nlj/stage7", "join/Full/mixed/projection")]
    assert len(raws) == 2
    errors = 0
    for raw in raws:
        for _ in range(200):
            b = bytearray(raw)
            if rnd.randrange(2):
                b = b[:rnd.randrange(len(b))]
            else:
                b[rnd.randrange(len(b))] ^= 1 << rnd.randrange(8)
            try:
                json.loads(engine.plan_typed_json(engine.plan_proto_to_json(bytes(b))))
            except engine.B200Error:
                errors += 1
    assert errors > 50


@pytest.mark.parametrize("q", ["q11", "q22"])
def test_tpch_nlj_from_proto_bytes(oracle, oracle_lib, q):
    """q11_nlj / q22_nlj run on the oracle from the decoded plan bytes equal the constant-key plans."""
    import base64
    from ballista_b200 import driver, tpch
    from test_tpch_queries import load_tables
    from util import assert_tables_equal
    byname = {c["name"]: c for c in PROTO_CASES}

    class Decoded:
        def __init__(self, e):
            self._e = e

        def __getattr__(self, k):
            return getattr(self._e, k)

        def create_query_stage_exec(self, job_id, stage_id, plan_json):
            ir = engine.plan_proto_to_json(base64.b64decode(byname[f"{q}_nlj/stage{stage_id}"]["proto_b64"]), job_id)
            return self._e.create_query_stage_exec(job_id, stage_id, ir)
    load_tables(oracle, oracle_lib, 20, tpch.union_tables([q]), 2)
    want = driver.run_stages(oracle, tpch.QUERIES[q][1](4), f"{q}-key")
    got = driver.run_stages(Decoded(oracle), getattr(tpch, f"{q}_nlj")(4), f"{q}-pb")
    assert_tables_equal(got, want, sort=False)
