"""Decimal128 columns of registered tables carry a 4-byte companion image (the value as int32) when every value fits 32 bits,
and the fused aggregate kernel streams it instead of the 16-byte values: q1 then reads 28 bytes per row, q6 16.  What was
streamed is read from the kernel timer of the fused family (pipeline_fused_agg); every result is checked against the CPU
oracle, bit-exact."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from ballista_b200 import driver, tpch
from test_gpu_fused_edge import _lineitem
from util import assert_tables_equal

pytestmark = pytest.mark.gpu

Q1_BYTES = 7 * 4    # 4 decimal images + 2 key images + the date
Q6_BYTES = 4 * 4    # 3 decimal images + the date
INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1


@pytest.fixture()
def timed(gpu):
    gpu.set_config("b200.metrics.kernel_timing", "on")
    yield gpu
    gpu.set_config("b200.metrics.kernel_timing", "off")


def _load_tpch(engines, oracle_lib, msf, columns, parts):
    n = oracle_lib.lib().oracle_tpch_table_rows(b"lineitem", msf)
    step = (n + parts - 1) // parts
    for e in engines:
        e.drop_table("lineitem")
        for p in range(parts):
            e.tpch_generate("lineitem", msf, p, min(n, p * step), min(n, (p + 1) * step), columns)
    return n


def _batch(n, seed, **kw):
    """a q1 lineitem batch with TPC-H's four (l_returnflag, l_linestatus) groups, so that the register sink holds them"""
    groups = np.random.default_rng(seed + 1000).choice(["AF", "NF", "NO", "RF"], n)
    return _lineitem(n, seed, flags=[g[0] for g in groups], status=[g[1] for g in groups], **kw)


def _same_arrow(got, want):
    assert got.schema.names == want.schema.names
    for i in range(want.num_columns):
        assert got.column(i).type == want.column(i).type
        assert got.column(i).equals(want.column(i)), want.schema.names[i]


def _register(engines, batches):
    for e in engines:
        e.drop_table("lineitem")
        for p, b in enumerate(batches):
            e.register_batch("lineitem", p, b)


def _streamed(gpu, stages, job):
    """(bytes the fused kernel streamed, fused launches, shape-specialised fused launches) of stage 1 alone"""
    f0, s0 = gpu.counter("fused"), gpu.counter("fused_static")
    gpu.kernel_stats(reset=True)
    driver.run_stages(gpu, stages[:1], job + "-s1", collect=False)
    ks = gpu.kernel_stats(reset=True)
    return ks.get("pipeline_fused_agg", {}).get("bytes", 0), gpu.counter("fused") - f0, gpu.counter("fused_static") - s0


def _check(gpu, oracle, stages, job):
    got = driver.run_stages(gpu, stages, job)
    want = driver.run_stages(oracle, stages, job)
    assert_tables_equal(got, want, sort=False)
    return got


@pytest.mark.parametrize("msf,parts,P", [(10, 1, 2), (50, 3, 4), (200, 2, 16)])
def test_q1_streams_28_bytes_per_row(timed, oracle, oracle_lib, msf, parts, P):
    n = _load_tpch((timed, oracle), oracle_lib, msf, tpch.Q1_COLUMNS, parts)
    nbytes, fused, static = _streamed(timed, tpch.q1(P), f"img-q1-{msf}")
    assert (nbytes, fused, static) == (Q1_BYTES * n, parts, parts)
    got = _check(timed, oracle, tpch.q1(P), f"img-q1-{msf}-{parts}-{P}")
    assert got.num_rows == 4


@pytest.mark.parametrize("msf,parts", [(10, 1), (100, 3)])
def test_q6_streams_16_bytes_per_row(timed, oracle, oracle_lib, msf, parts):
    n = _load_tpch((timed, oracle), oracle_lib, msf, tpch.Q6_COLUMNS, parts)
    nbytes, fused, static = _streamed(timed, tpch.q6(4), f"img-q6-{msf}")
    assert (nbytes, fused, static) == (Q6_BYTES * n, parts, parts)
    _check(timed, oracle, tpch.q6(4), f"img-q6-{msf}-{parts}")


def test_without_images_streams_arrow_widths(timed, oracle, oracle_lib, monkeypatch):
    """B200_NO_PREPACK switches off the key images and the decimal images alike: 4 x 16 B of decimals, offsets for keys"""
    monkeypatch.setenv("B200_NO_PREPACK", "1")
    n = _load_tpch((timed, oracle), oracle_lib, 20, tpch.Q1_COLUMNS, 1)
    nbytes, fused, static = _streamed(timed, tpch.q1(2), "img-noprepack")
    assert (nbytes, fused, static) == ((4 * 16 + 3 * 4) * n, 1, 1)
    _check(timed, oracle, tpch.q1(2), "img-noprepack")


def test_int32_limits_keep_the_image(timed, oracle):
    """INT32_MIN and INT32_MAX are representable: every column keeps its image, the narrow path hands these tiles to the
    exact path"""
    n = 5000
    rng = np.random.default_rng(21)
    qty = rng.integers(100, 5001, n).astype(object)
    tax = rng.integers(0, 9, n).astype(object)
    qty[0], qty[n // 2], tax[7], tax[n - 1] = INT32_MIN, INT32_MAX, INT32_MAX, INT32_MIN
    _register((timed, oracle), [_batch(n, 22, qty=qty, tax=tax)])
    nbytes, fused, static = _streamed(timed, tpch.q1(2), "img-limits")
    assert (nbytes, fused, static) == (Q1_BYTES * n, 1, 1)
    _check(timed, oracle, tpch.q1(2), "img-limits")


@pytest.mark.parametrize("column,value", [("price", 2 ** 31), ("disc", -2 ** 31 - 1), ("qty", 2 ** 31), ("tax", -2 ** 31 - 1)])
def test_one_value_past_int32_drops_that_image_only(timed, oracle, column, value):
    """the column with the out-of-range value streams its 16-byte values, the others their images: a mixed shape that
    runs on the run-time-described variant of the kernel"""
    n = 7000
    vals = np.random.default_rng(23).integers(0, 9, n).astype(object)
    if column in ("price", "qty"):
        vals = np.random.default_rng(24).integers(100, 5001, n).astype(object)
    vals[n // 3] = value
    _register((timed, oracle), [_batch(n, 25, **{column: vals})])
    nbytes, fused, static = _streamed(timed, tpch.q1(2), f"img-wide-{column}")
    assert (nbytes, fused, static) == ((Q1_BYTES + 12) * n, 1, 0)
    _check(timed, oracle, tpch.q1(2), f"img-wide-{column}")


def test_negative_and_mixed_sign_values(timed, oracle):
    n = 40000
    rng = np.random.default_rng(26)
    price = -rng.integers(90000, 10495001, n)             # every price negative
    qty = rng.integers(-5000, 5001, n)                    # mixed signs
    disc = rng.integers(-10, 11, n)
    _register((timed, oracle), [_batch(n, 27, qty=qty, price=price, disc=disc)])
    nbytes, fused, static = _streamed(timed, tpch.q1(3), "img-neg")
    assert (nbytes, fused, static) == (Q1_BYTES * n, 1, 1)
    _check(timed, oracle, tpch.q1(3), "img-neg")


def test_appended_table_keeps_images(timed, oracle):
    """two register_batch calls into one partition: the concatenated table gets its images too"""
    a, b = _batch(30001, 28), _batch(20011, 29)
    for e in (timed, oracle):
        e.drop_table("lineitem")
        e.register_batch("lineitem", 0, a)
        e.register_batch("lineitem", 0, b)
    nbytes, fused, static = _streamed(timed, tpch.q1(2), "img-append")
    assert (nbytes, fused, static) == (Q1_BYTES * (a.num_rows + b.num_rows), 1, 1)
    _check(timed, oracle, tpch.q1(2), "img-append")
    _same_arrow(timed.export_table("lineitem", 0), pa.Table.from_batches([a, b]).combine_chunks().to_batches()[0])


def test_parquet_registered_lineitem(timed, oracle, oracle_lib, tmp_path):
    n = _load_tpch((oracle,), oracle_lib, 20, tpch.Q1_COLUMNS, 1)
    b = oracle.export_table("lineitem", 0)
    path = str(tmp_path / "lineitem.parquet")
    pq.write_table(pa.Table.from_batches([b]), path, row_group_size=50000)
    timed.drop_table("lineitem")
    timed.register_parquet("lineitem", 0, path)
    nbytes, fused, static = _streamed(timed, tpch.q1(2), "img-parquet")
    assert (nbytes, fused, static) == (Q1_BYTES * n, 1, 1)
    _check(timed, oracle, tpch.q1(2), "img-parquet")


def test_export_is_unchanged(gpu):
    """the images are companions: the exported table is the registered Arrow data"""
    b = _batch(10007, 30)
    gpu.drop_table("lineitem")
    gpu.register_batch("lineitem", 0, b)
    _same_arrow(gpu.export_table("lineitem", 0), b)


@pytest.mark.parametrize("n", [0, 1, 37])
def test_small_and_empty_tables(timed, oracle, n):
    _register((timed, oracle), [_batch(n, 31 + n)])
    nbytes, fused, static = _streamed(timed, tpch.q1(2), f"img-small-{n}")
    if n:
        assert (nbytes, fused, static) == (Q1_BYTES * n, 1, 1)
    _check(timed, oracle, tpch.q1(2), f"img-small-{n}")
