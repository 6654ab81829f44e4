"""GPU: HashJoinExec on the device (csrc/device/join.cu, exec_join / join_output in engine.cpp) against the plain-Python
reference of hash_join_cases and, where it runs the case too, the CPU oracle.  The pair order of the device join depends
on its atomics, so rows are compared as multisets."""
import numpy as np
import pyarrow as pa
import pytest

import ballista_b200 as bb
from ballista_b200 import driver, engine
from ballista_b200 import plan as P
import hash_join_cases as H

pytestmark = pytest.mark.gpu
JT = H.JOIN_TYPES
EMITS_BUILD = ("Left", "Full", "LeftSemi", "LeftAnti")


@pytest.fixture(scope="module")
def tables():
    return H.make_table(150, seed=41), H.make_table(250, seed=42)


def _check(gpu, oracle, left, right, stages, on, jt, filt=None, projection=None, nen=False, build_parts=1, probe_parts=1, job="hj"):
    want = H.reference_hash_join(left, right, on, jt, filt, projection, nen)
    H.register(gpu, left, right, build_parts, probe_parts)
    got = H.run(gpu, stages, job)
    assert H.same_multiset(got, want), f"device: {len(got)} rows, reference: {len(want)} rows"
    if oracle is not None:
        H.register(oracle, left, right, build_parts, probe_parts)
        assert H.same_multiset(H.run(oracle, stages, job), want)
    return got


@pytest.mark.parametrize("jt", JT)
@pytest.mark.parametrize("shape", sorted(H.SHAPES))
def test_matrix(gpu, oracle, tables, jt, shape):
    """Every join type x one key of every type (single integer-like keys: the exact-key table; the rest: the hash-tagged
    table) and two mixed / three nullable keys, without and with a residual filter."""
    keys = H.SHAPES[shape]
    for fname, filt in H.FILTERS.items():
        _check(gpu, oracle, *tables, H.collect_left_stages(keys, jt, filt), [(k, k) for k in keys], jt, filt, job=f"m-{jt}-{shape}-{fname}")


@pytest.mark.parametrize("jt", JT)
@pytest.mark.parametrize("shape", ["i64", "u8", "date32", "utf8", "f64", "i32_utf8", "i16_dec_date32"])
def test_null_equals_null(gpu, oracle, tables, jt, shape):
    """NULL matches NULL: a single nullable integer key leaves the exact-key table (which keeps NULLs out) for the
    hash-tagged one; multi-column keys match NULL with NULL column by column."""
    keys = H.SHAPES[shape]
    for fname, filt in H.FILTERS.items():
        _check(gpu, oracle, *tables, H.collect_left_stages(keys, jt, filt, null_equals_null=True), [(k, k) for k in keys], jt, filt, nen=True,
               job=f"n-{jt}-{shape}-{fname}")


_AB = [P.field("a", "i64", True), P.field("b", "i64", True), P.field("id", "i64", True)]


def _ab_table(rows):
    return pa.table({"a": pa.array([r[0] for r in rows], pa.int64()), "b": pa.array([r[1] for r in rows], pa.int64()),
                     "id": pa.array(list(range(len(rows))), pa.int64())})


@pytest.mark.parametrize("jt", JT)
def test_forced_tag_collision_produces_no_pair(gpu, oracle, jt):
    """Build and probe keys that differ but share their 64-bit row hash (the hash-tagged table's tag): only the check of
    the key columns keeps them apart."""
    k1, k2 = H.colliding_keys()
    left = _ab_table([k1, k1, (5, 6), k1, (None, 1)])
    right = _ab_table([k2, (5, 6), k2, (7, None)])
    on = [("a", "a"), ("b", "b")]
    stages = H.collect_left_stages(["a", "b"], jt, ir_schema=_AB)
    want = H.reference_hash_join(left, right, on, jt, ir_schema=_AB)
    for e in (gpu, oracle):
        H.register(e, left, right)
        assert H.same_multiset(H.run(e, stages, f"c-{jt}"), want)
    if jt == "Inner":
        assert len(want) == 1


@pytest.mark.parametrize("jt", JT)
@pytest.mark.parametrize("t", ["f32", "f64"])
def test_float_keys_match_the_nested_loop_join(gpu, oracle, t, jt):
    """+-0.0, NaN payloads, +-inf: the hash join returns the rows of a NestedLoopJoinExec with filter l.f = r.f over the
    same data (the nested-loop join has its own reference), and both equal the reference."""
    left, right = H.make_table(90, seed=50, null_every=8), H.make_table(120, seed=51, null_every=8)
    k = f"k_{t}"
    hj = _check(gpu, oracle, left, right, H.collect_left_stages([k], jt), [(k, k)], jt, job=f"f-{t}-{jt}")
    nlj = [P.Stage(1, P.shuffle_writer(P.nested_loop_join(P.scan("hj_l", H.IR_SCHEMA), P.scan("hj_r", H.IR_SCHEMA), jt,
                                                          filter=P.binop("=", H.L(k), H.R(k))), 1))]
    got_nlj = H.run(gpu, nlj, f"fn-{t}-{jt}")
    assert H.same_multiset(got_nlj, hj)


@pytest.mark.parametrize("jt", JT)
@pytest.mark.parametrize("size", ["empty_build", "empty_probe", "one_row_build", "all_null_build"])
def test_edge_sizes(gpu, oracle, jt, size):
    nb, np_ = {"empty_build": (0, 90), "empty_probe": (70, 0), "one_row_build": (1, 400), "all_null_build": (50, 60)}[size]
    left = H.make_table(nb, seed=5, null_every=1 if size == "all_null_build" else 6)
    right = H.make_table(np_, seed=6)
    for shape in ("i64", "i32_utf8"):
        keys = H.SHAPES[shape]
        for nen in (False, True):
            _check(gpu, oracle, left, right, H.collect_left_stages(keys, jt, null_equals_null=nen), [(k, k) for k in keys], jt, nen=nen,
                   job=f"e-{jt}-{size}-{shape}-{nen}")


_IK = [P.field("id", "i64", False), P.field("k", "i64", True)]


def _ik(ids, keys):
    return pa.table({"id": pa.array(ids, pa.int64()), "k": pa.array(keys, pa.int64())})


def _ik_join(gpu, left, right, jt, job, projection=None):
    H._register(gpu, "hj_l", left, 1)
    H._register(gpu, "hj_r", right, 1)
    return driver.run_stages(gpu, H.collect_left_stages(["k"], jt, projection=projection, ir_schema=_IK), job)


def test_all_keys_equal_reruns_the_probe(gpu):
    """5,000 x 4,000 rows with one key: 20M pairs overflow the first pair buffer and the probe runs again at the exact size."""
    nb, np_ = 5000, 4000
    gpu.set_config("b200.metrics.kernel_timing", "1")
    gpu.kernel_stats(reset=True)
    try:
        out = _ik_join(gpu, _ik(np.arange(nb), np.full(nb, 7)), _ik(np.arange(np_), np.full(np_, 7)), "Inner", "rerun", projection=[0, 2])
        ks = gpu.kernel_stats(reset=True)
    finally:
        gpu.set_config("b200.metrics.kernel_timing", "0")
    assert ks["join_probe"]["launches"] == 2
    assert out.num_rows == nb * np_
    code = out.column(0).to_numpy() * np_ + out.column(1).to_numpy()
    assert np.array_equal(np.sort(code), np.arange(nb * np_))


def test_one_probe_row_matching_1000_build_rows(gpu, oracle):
    """One probe row walks a chain of 1,000 matching build rows: the warp's staged pairs are flushed inside the chain."""
    rng = np.random.default_rng(3)
    bk = np.where(np.arange(3000) % 3 == 0, 42, rng.integers(100, 10 ** 6, 3000))
    left = _ik(np.arange(3000), bk)
    right = _ik(np.arange(40), np.where(np.arange(40) == 17, 42, -np.arange(40) - 1))
    for jt in JT:
        want = H.reference_hash_join(left, right, [("k", "k")], jt, ir_schema=_IK)
        for e in (gpu, oracle):
            H.register(e, left, right)
            assert H.same_multiset(H.run(e, H.collect_left_stages(["k"], jt, ir_schema=_IK), f"chain-{jt}"), want)
    assert len(H.reference_hash_join(left, right, [("k", "k")], "Inner", ir_schema=_IK)) == 1000


def test_large_probe_carries_staged_pairs_across_iterations(gpu):
    """2M probe rows x 1M build rows at about 10 % matches: more probe rows than one pass of the grid (132 * 16 blocks of
    256 threads), so warps carry staged pairs from one grid-stride iteration to the next."""
    rng = np.random.default_rng(11)
    nb, np_ = 1_000_000, 2_000_000
    perm = rng.permutation(nb)
    bkeys = perm.astype(np.int64) * 10                      # build row i has key 10 * perm[i]
    pkeys = rng.integers(0, 10 * nb, np_).astype(np.int64)  # matches iff divisible by 10
    left, right = _ik(np.arange(nb), bkeys), _ik(np.arange(np_), pkeys)
    hit = pkeys % 10 == 0
    inv = np.empty(nb, np.int64)
    inv[perm] = np.arange(nb)
    want = np.sort(inv[pkeys[hit] // 10] * np_ + np.nonzero(hit)[0])
    out = _ik_join(gpu, left, right, "Inner", "large", projection=[0, 2])
    got = np.sort(out.column(0).to_numpy() * np_ + out.column(1).to_numpy())
    assert 0.09 * np_ < len(want) < 0.11 * np_
    assert np.array_equal(got, want)
    semi = _ik_join(gpu, left, right, "RightAnti", "large-anti")
    assert np.array_equal(np.sort(semi.column(0).to_numpy()), np.nonzero(~hit)[0])


@pytest.mark.parametrize("jt,probe_parts", [(jt, 1) for jt in JT] + [(jt, 4) for jt in JT if jt not in EMITS_BUILD])
def test_collect_left_build_in_three_partitions(gpu, oracle, tables, jt, probe_parts):
    """The build side in 3 partitions, read whole by every task; the probe side in 1 or 4 (join types that emit build
    rows only with 1: see the refusal below)."""
    for shape in ("i64", "i32_utf8"):
        keys = H.SHAPES[shape]
        _check(gpu, oracle, *tables, H.collect_left_stages(keys, jt), [(k, k) for k in keys], jt, build_parts=3, probe_parts=probe_parts,
               job=f"cl-{jt}-{probe_parts}-{shape}")


def test_build_emitting_join_over_many_probe_partitions_is_refused(gpu, oracle, tables):
    left, right = tables
    for jt in EMITS_BUILD:
        H.register(gpu, left, right, 1, 4)
        with pytest.raises(bb.B200Error) as e:
            H.run(gpu, H.collect_left_stages(["k_i64"], jt), f"refuse-{jt}")
        assert e.value.code == -2 and "more than one probe partition" in str(e.value)
    _check(gpu, oracle, left, right, H.collect_left_stages(["k_utf8"], "Full"), [("k_utf8", "k_utf8")], "Full", job="after-refusal")


@pytest.mark.parametrize("jt", JT)
@pytest.mark.parametrize("shape", ["i64", "bool", "utf8", "f64", "i32_utf8"])
def test_partitioned_two_stage(gpu, oracle, tables, jt, shape):
    """Both sides hash-repartitioned on the key into 4 partitions (Bool keys leave at least one empty), then joined
    partition by partition."""
    keys = H.SHAPES[shape]
    for nen in (False, True):
        _check(gpu, oracle, *tables, H.partitioned_stages(keys, jt, null_equals_null=nen), [(k, k) for k in keys], jt, nen=nen,
               build_parts=2, probe_parts=2, job=f"pt-{jt}-{shape}-{nen}")


@pytest.mark.parametrize("jt", JT)
def test_computed_keys(gpu, oracle, tables, jt):
    """Keys that are expressions take the materialising branch of materialize_mixed: cast(i32 -> i64) = i64, btrim(s) = s,
    and a probe side behind a filter."""
    left, right = tables
    on = [[P.cast(H.L("k_i32"), "i64"), P.col(H.COL["k_i64"])]]
    j = P.hash_join(P.scan("hj_l", H.IR_SCHEMA), P.scan("hj_r", H.IR_SCHEMA), on, jt, "CollectLeft")
    _check(gpu, oracle, left, right, [P.Stage(1, P.shuffle_writer(j, 1))], [("k_i32", "k_i64")], jt, job=f"cast-{jt}")

    padded = left.set_column(H.COL["k_utf8"], "k_utf8", pa.array([None if v is None else f"  {v} " for v in left.column("k_utf8").to_pylist()]))
    on = [[P.fn("btrim", H.L("k_utf8")), P.col(H.COL["k_utf8"])]]
    j = P.hash_join(P.scan("hj_l", H.IR_SCHEMA), P.scan("hj_r", H.IR_SCHEMA), on, jt, "CollectLeft")
    # the oracle has no btrim: the device against the reference only
    _check(gpu, None, padded, right, [P.Stage(1, P.shuffle_writer(j, 1))], [(H.key_values(left, "k_utf8"), "k_utf8")], jt, job=f"trim-{jt}")

    cut = 200
    probe = P.filter_(P.binop(">=", P.col(0), P.lit_i64(cut)), P.scan("hj_r", H.IR_SCHEMA))
    stages = H.collect_left_stages(["k_i64"], jt, right=probe)
    want = H.reference_hash_join(left, right.slice(cut), [("k_i64", "k_i64")], jt)
    for e in (gpu, oracle):
        H.register(e, left, right)
        assert H.same_multiset(H.run(e, stages, f"pf-{jt}"), want)
    assert want


_NN = [P.field(n, f["type"], False) for n, f in zip(H.NAMES, H.IR_SCHEMA)]


@pytest.mark.parametrize("jt", ["Inner", "Left", "Right", "Full"])
def test_outer_join_projection_and_nullability(gpu, oracle, jt):
    """Non-nullable inputs: the side an outer join pads with NULLs becomes nullable in the output schema, and every type
    gathers its NULL fill for index -1."""
    left = H.make_table(120, seed=61, null_every=10 ** 9)
    right = H.make_table(150, seed=62, null_every=10 ** 9)
    proj = [0] + [H.NC + c for c in range(1, H.NC)] + list(range(1, H.NC))
    stages = H.collect_left_stages(["k_utf8"], jt, projection=proj, ir_schema=_NN)
    typed = __import__("json").loads(engine.plan_typed_json(stages[0].json("job")))
    sch = typed["input"]["schema"]
    lnull, rnull = jt in ("Right", "Full"), jt in ("Left", "Full")
    assert [f["nullable"] for f in sch] == [lnull] + [rnull] * (H.NC - 1) + [lnull] * (H.NC - 1)
    _check(gpu, oracle, left, right, stages, [("k_utf8", "k_utf8")], jt, projection=proj, job=f"proj-{jt}")


@pytest.mark.parametrize("jt", JT)
@pytest.mark.parametrize("shape", ["i64", "utf8", "f32"])
def test_sort_merge_join(gpu, oracle, tables, jt, shape):
    """SortMergeJoinExec over the same inputs: the hash join's rows, ordered by the key (ascending, NULLs last; the order
    is checked for the integer and string keys)."""
    left, right = tables
    keys = H.SHAPES[shape]
    j = P.sort_merge_join(P.scan("hj_l", H.IR_SCHEMA), P.scan("hj_r", H.IR_SCHEMA), H.on_cols(keys), jt, sort_options=[{"asc": True, "nulls_first": False}])
    got = _check(gpu, oracle, left, right, [P.Stage(1, P.shuffle_writer(j, 1))], [(k, k) for k in keys], jt, job=f"smj-{jt}-{shape}")
    if shape == "f32":
        return
    c = H.COL[keys[0]] + (H.NC if jt == "Right" else 0)
    key = [(v is None, b"" if v is None else v.encode() if isinstance(v, str) else v) for v in (r[c] for r in got)]
    assert key == sorted(key)
