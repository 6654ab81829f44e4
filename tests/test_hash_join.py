"""HashJoinExec without a GPU: the CPU oracle against the plain-Python reference of hash_join_cases (every join type, one
key of every type, mixed and nullable multi-column keys, with and without a residual filter, with NULL = NULL on and off),
and the protobuf decoder's null_equality / null_aware fields of HashJoinExecNode and SortMergeJoinExecNode."""
import base64
import json
import os

import pytest

from ballista_b200 import engine
from ballista_b200 import plan as P
import hash_join_cases as H

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def tables():
    return H.make_table(60, seed=21), H.make_table(80, seed=22)


@pytest.mark.parametrize("jt", H.JOIN_TYPES)
@pytest.mark.parametrize("shape", sorted(H.SHAPES))
def test_oracle_matches_reference(oracle, tables, jt, shape):
    left, right = tables
    keys = H.SHAPES[shape]
    H.register(oracle, left, right)
    for fname, filt in H.FILTERS.items():
        for nen in (False, True):
            got = H.run(oracle, H.collect_left_stages(keys, jt, filt, null_equals_null=nen), f"o-{jt}-{shape}-{fname}-{nen}")
            want = H.reference_hash_join(left, right, [(k, k) for k in keys], jt, filt, null_equals_null=nen)
            assert H.same_multiset(got, want), (fname, nen)


@pytest.mark.parametrize("t", ["f32", "f64"])
def test_oracle_float_keys_match_by_bits(oracle, t):
    """-0.0 does not join 0.0; NaN joins NaN only with the same payload: the engine's `=`, as the nested-loop join has it."""
    left = H.make_table(4, seed=1, null_every=10 ** 9, domains={t: [0x80000000 if t == "f32" else 1 << 63]})
    right = H.make_table(3, seed=2, null_every=10 ** 9, domains={t: [0]})
    H.register(oracle, left, right)
    assert H.run(oracle, H.collect_left_stages([f"k_{t}"], "Inner"), f"neg0-{t}") == []
    nan_a, nan_b = (0x7FC00000, 0x7FC00001) if t == "f32" else (0x7FF8000000000000, 0x7FF8000000000001)
    left = H.make_table(12, seed=3, null_every=10 ** 9, domains={t: [nan_a, nan_b]})
    right = H.make_table(5, seed=4, null_every=10 ** 9, domains={t: [nan_a]})
    H.register(oracle, left, right)
    got = H.run(oracle, H.collect_left_stages([f"k_{t}"], "Inner"), f"nan-{t}")
    want = H.reference_hash_join(left, right, [(f"k_{t}",) * 2], "Inner")
    n_a = sum(1 for k in H.key_values(left, f"k_{t}") if k == ("f", nan_a))
    assert 0 < n_a < 12 and len(want) == n_a * 5
    assert H.same_multiset(got, want)


def test_reference_collision_keys():
    """The two keys of hash_join_cases.colliding_keys differ and have one row hash (checked with test_hash's restatement)."""
    import test_hash as T
    (a1, b1), (a2, b2) = H.colliding_keys()
    assert (a1, b1) != (a2, b2)

    def row_hash(a, b):
        return T.combine(T.hash_i64(b & T.M), T.hash_i64(a & T.M))
    assert row_hash(a1, b1) == row_hash(a2, b2)
    assert H.unmix64(T.mix64(12345)) == 12345


def test_oracle_row_hash_of_collision_keys(oracle):
    import pyarrow as pa
    (a1, b1), (a2, b2) = H.colliding_keys()
    batch = pa.RecordBatch.from_arrays([pa.array([a1, a2], pa.int64()), pa.array([b1, b2], pa.int64())], names=["a", "b"])
    h, _ = oracle.hash_partition_ids(batch, [0, 1], 7)
    assert int(h[0]) == int(h[1])


# ---- protobuf: null_equality and null_aware ------------------------------------------------------------------------
with open(os.path.join(HERE, "golden", "hash_join_proto_plans.json")) as _fh:
    PROTO_CASES = json.load(_fh)["cases"]


def _strip_cosmetic(t):
    if isinstance(t, dict):
        return {k: _strip_cosmetic(v) for k, v in t.items() if not (k == "name" and "col" in t)}
    if isinstance(t, list):
        return [_strip_cosmetic(v) for v in t]
    return t


def _join_node(t):
    while t["op"] not in ("HashJoinExec", "SortMergeJoinExec"):
        t = t["input"]
    return t


DECODED = [c for c in PROTO_CASES if not c["name"].startswith("null_aware/")]


@pytest.mark.parametrize("case", DECODED, ids=[c["name"] for c in DECODED])
def test_proto_plan_decodes_to_its_source(case):
    ir = engine.plan_proto_to_json(base64.b64decode(case["proto_b64"]))
    got = json.loads(engine.plan_typed_json(ir))
    assert _strip_cosmetic(got) == _strip_cosmetic(json.loads(engine.plan_typed_json(case["ir"])))
    nen = "/null_equals_null" in case["name"]
    assert bool(_join_node(json.loads(ir)).get("null_equals_null")) == nen
    assert bool(_join_node(got).get("null_equals_null")) == nen


def test_proto_null_aware_is_refused():
    cases = [c for c in PROTO_CASES if c["name"].startswith("null_aware/")]
    assert cases
    for c in cases:
        with pytest.raises(engine.B200Error) as e:
            engine.plan_proto_to_json(base64.b64decode(c["proto_b64"]))
        assert e.value.code == -2 and "null-aware" in str(e.value)


@pytest.mark.parametrize("op", ["HashJoinExec", "SortMergeJoinExec"])
def test_proto_null_equals_null_runs_on_the_oracle(oracle, op):
    """A two-key LeftSemi join with (NULL, NULL) on both sides: decoded from the plan bytes, NULL matches NULL."""
    c = [c for c in PROTO_CASES if c["name"] == f"{op}/LeftSemi/null_equals_null"][0]
    left = H.make_table(30, seed=31, null_every=3)
    right = H.make_table(30, seed=32, null_every=3)
    H.register(oracle, left, right)
    keys = [("k_i64", "k_i64"), ("k_utf8", "k_utf8")]
    want = H.reference_hash_join(left, right, keys, "LeftSemi", null_equals_null=True)
    assert len(want) > len(H.reference_hash_join(left, right, keys, "LeftSemi"))

    class FromProto:
        def __init__(self, e):
            self._e = e

        def __getattr__(self, k):
            return getattr(self._e, k)

        def create_query_stage_exec(self, job_id, stage_id, plan_json):
            return self._e.create_query_stage_exec(job_id, stage_id, engine.plan_proto_to_json(base64.b64decode(c["proto_b64"]), job_id))
    from ballista_b200 import driver
    import nlj_cases as N
    got = N.rows_of(driver.run_stages(FromProto(oracle), [P.Stage(1, json.loads(c["ir"]))], f"pb-{op}"))
    assert H.same_multiset(got, want)
