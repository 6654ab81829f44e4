"""Device Parquet scan of GZIP and LZ4_RAW compressed pages.

CPU: the hand-built files (parquet_codec_pages.py) read back through pyarrow to their values, and every malformed page
(except an LZ4 offset of 0, which liblz4 accepts) is refused by pyarrow too; b200_parquet_describe's `codec` and `codecs`
agree with pyarrow's metadata.  GPU: pyarrow-written gzip and lz4 files in the layouts of test_parquet_scan's VARIANTS and in
every encoding set of test_parquet_encodings, with gzip levels 1 and 9, and the hand-built pages (stored, fixed-Huffman, RLE
and Huffman-only deflate, zlib and multi-member wrappers, optional gzip header fields, LZ4 continuation lengths, offsets 1 and
65535, a column mixing four codecs) decode bit-exactly as pyarrow reads them; malformed pages are refused with
B200_ERR_INVALID naming the column; brotli is still refused; TPC-H q1 / q6 run from a gzip and an lz4 lineitem."""
import gzip
import os
import random
import struct
import zlib

import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import ballista_b200 as bb
import parquet_codec_pages as C
import parquet_handmade as H
from ballista_b200 import driver, tpch
from test_parquet_encodings import ENCODING_SETS, _encoded_table, _write_encoded
from test_parquet_scan import VARIANTS, _table
from util import assert_tables_equal

# pyarrow's ColumnChunkMetaData.compression names -> parquet codec ids (it names LZ4_RAW, codec 7, "LZ4")
CODEC_IDS = {"UNCOMPRESSED": 0, "SNAPPY": 1, "GZIP": 2, "BROTLI": 4, "ZSTD": 6, "LZ4": 7}


def _pa(name):
    codec = pa.Codec(name)
    return lambda b: bytes(codec.compress(b))


# ---- hand-built files -------------------------------------------------------------------------------------------------------
def _ints(rnd, n):
    """Values with long runs of zero bytes and repeats: every deflate strategy finds matches."""
    return [rnd.randrange(0, 1000) * 7 for _ in range(n)]


def _one_chunk(path, codec, compress, values, page_rows=2000, kind=H.DATA_PAGE):
    pages = C.plain_pages(kind, H.INT64, values, page_rows, compress)
    return C.write_file(path, "v", H.INT64, [(codec, pages, len(values))])


def _shape_gzip_stored(path, rnd):
    v = _ints(rnd, 20000)   # 80 KB pages at level 0: two stored blocks each
    return _one_chunk(path, C.GZIP, lambda b: gzip.compress(b, compresslevel=0, mtime=0), v, 10000), v


def _shape_gzip_fixed(path, rnd):
    v = _ints(rnd, 6000)
    return _one_chunk(path, C.GZIP, lambda b: C.gzip_member(b, 9, zlib.Z_FIXED), v), v


def _shape_gzip_rle(path, rnd):
    v = [rnd.choice([0, 0, 0, 5, 2**40]) for _ in range(6000)]   # distance-1 copies over the zero bytes
    return _one_chunk(path, C.GZIP, lambda b: C.gzip_member(b, 9, zlib.Z_RLE), v), v


def _shape_gzip_huffman_only(path, rnd):
    v = _ints(rnd, 6000)
    return _one_chunk(path, C.GZIP, lambda b: C.gzip_member(b, 9, zlib.Z_HUFFMAN_ONLY), v), v


def _shape_zlib_wrapped(path, rnd):
    v = _ints(rnd, 6000)
    return _one_chunk(path, C.GZIP, lambda b: zlib.compress(b, 6), v), v


def _shape_two_members(path, rnd):
    v = _ints(rnd, 6000)
    return _one_chunk(path, C.GZIP, lambda b: C.gzip_member(b[:5000], 1) + C.gzip_member(b[5000:], 9), v), v


def _shape_gzip_header_fields(path, rnd):
    v = _ints(rnd, 6000)
    member = lambda b: C.gzip_member(b, 6, extra=b"AB\x04\x00xyzw" * 30, name=b"lineitem.tbl", comment=b"a comment", hcrc=True)
    return _one_chunk(path, C.GZIP, member, v), v


def _v2_all_null_and_uncompressed(path, rnd, codec, compress):
    # an optional column in V2 pages: an all-NULL page whose compressed values section is empty (as parquet-java writes
    # it), a page stored with is_compressed = false inside the compressed chunk, and a page compressed as usual
    a = [None] * 700
    b = [None if rnd.random() < 0.2 else x for x in _ints(rnd, 900)]
    c = [None if rnd.random() < 0.2 else x for x in _ints(rnd, 800)]
    pages = []
    for chunk, comp, flag in ((a, lambda _: b"", True), (b, compress, False), (c, compress, True)):
        present = [x for x in chunk if x is not None]
        defs = [0 if x is None else 1 for x in chunk]
        pages.append(C.page(H.DATA_PAGE_V2, H.PLAIN, H.plain(present, H.INT64), len(chunk), comp, defs, v2_compressed=flag))
    v = a + b + c
    return C.write_file(path, "v", H.INT64, [(codec, pages, len(v))], optional=True), v


def _shape_v2_all_null_and_uncompressed(path, rnd):
    return _v2_all_null_and_uncompressed(path, rnd, C.GZIP, gzip.compress)


def _shape_v2_all_null_and_uncompressed_lz4(path, rnd):
    return _v2_all_null_and_uncompressed(path, rnd, C.LZ4_RAW, _pa("lz4_raw"))


def _lz4_sequences(rnd):
    lit = bytes(rnd.randrange(256) for _ in range(70000))      # literal length continuation: 274 bytes of 255
    seqs = [(lit, 65535, 600),                                  # the farthest offset, match length continuation
            (b"\x07", 1, 1000),                                 # offset 1: a run
            (b"", 8, 19)]                                       # match length 4 + 15: a continuation byte of 0
    return C.lz4_block(seqs, bytes(rnd.randrange(256) for _ in range(20)))


def _shape_lz4_sequences(path, rnd):
    block, data = _lz4_sequences(rnd)
    assert len(data) % 8 == 0
    v = list(struct.unpack("<%dq" % (len(data) // 8), data))
    pg = C.page(H.DATA_PAGE, H.PLAIN, data, len(v), lambda _: block)
    return C.write_file(path, "v", H.INT64, [(C.LZ4_RAW, [pg], len(v))]), v


def _shape_mixed_codecs(path, rnd):
    v = [None if rnd.random() < 0.1 else x for x in _ints(rnd, 8000)]
    chunks = []
    for k, (codec, comp) in enumerate(((C.UNCOMPRESSED, C._identity), (C.SNAPPY, _pa("snappy")), (C.GZIP, gzip.compress),
                                       (C.LZ4_RAW, _pa("lz4_raw")))):
        part = v[2000 * k:2000 * (k + 1)]
        chunks.append((codec, C.plain_pages(H.DATA_PAGE, H.INT64, part, 700, comp, optional=True), len(part)))
    return C.write_file(path, "v", H.INT64, chunks, optional=True), v


SHAPES = {f.__name__[len("_shape_"):]: f for f in (
    _shape_gzip_stored, _shape_gzip_fixed, _shape_gzip_rle, _shape_gzip_huffman_only, _shape_zlib_wrapped, _shape_two_members,
    _shape_gzip_header_fields, _shape_v2_all_null_and_uncompressed, _shape_v2_all_null_and_uncompressed_lz4, _shape_lz4_sequences,
    _shape_mixed_codecs)}
SHAPE_CODECS = {name: [2] for name in SHAPES}
SHAPE_CODECS.update(lz4_sequences=[7], v2_all_null_and_uncompressed_lz4=[7], mixed_codecs=[0, 1, 2, 7])


def _build_shape(tmp_path, name):
    return SHAPES[name](os.path.join(str(tmp_path), name + ".parquet"), random.Random(name))


# malformed pages: one INT64 column "v"; (codec, stored page payload, its claimed uncompressed bytes)
def _bad_crc(data):
    g = bytearray(gzip.compress(data, mtime=0))
    g[-8] ^= 1
    return bytes(g)


def _bad_nlen(data):
    g = bytearray(gzip.compress(data, compresslevel=0, mtime=0))
    g[13] ^= 1   # header 10 bytes, block header byte, LEN, NLEN
    return bytes(g)


# Two gzip members: the second is a single match 5 bytes back, into the first member's output.  Lengths and CRCs are
# consistent with copying those bytes, so only the rule that a member's distances stay inside its own output (zlib's
# "invalid distance too far back") refuses the page.
_FIRST = b"0123456789abc"
_CROSSING = _FIRST + _FIRST[8:11]


def _distance_before_member(_):
    second = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\xff" + C.fixed_block([(3, 5)])
    second += struct.pack("<II", zlib.crc32(_CROSSING[13:]), 3)
    return C.gzip_member(_FIRST) + second


MALFORMED = {
    "gzip_crc32_flipped": (C.GZIP, _bad_crc),
    "gzip_raw_deflate": (C.GZIP, lambda d: C.deflate_raw(d)),
    "gzip_truncated": (C.GZIP, lambda d: gzip.compress(d, mtime=0)[:-12]),
    "gzip_stored_nlen": (C.GZIP, _bad_nlen),
    "gzip_distance_before_member": (C.GZIP, _distance_before_member),
    "lz4_offset_too_far": (C.LZ4_RAW, lambda _: C.lz4_block([(b"abc", 10, 4)], b"123456789")[0]),
    "lz4_offset_zero": (C.LZ4_RAW, lambda _: C.lz4_block([(b"abc", 0, 4)], b"123456789")[0]),
}
DEVICE_ONLY = {"lz4_offset_zero"}   # liblz4 (pyarrow) accepts offset 0; the block format forbids it


def _v2_stored_sizes_differ(tmp_path):
    """A gzip chunk with an is_compressed = false V2 page whose header claims 16 stored bytes but 8 uncompressed ones.
    pyarrow reads it by its stored size; the device refuses it rather than copy 16 bytes into an 8-byte payload."""
    body = H.plain([1, 2], H.INT64)
    sub = H.Struct().i32(1, 2).i32(2, 0).i32(3, 2).i32(4, H.PLAIN).i32(5, 0).i32(6, 0).boolean(7, False)
    pg = H.Struct().i32(1, H.DATA_PAGE_V2).i32(2, 8).i32(3, len(body)).struct(8, sub).bytes() + body
    return C.write_file(os.path.join(str(tmp_path), "sizes.parquet"), "v", H.INT64, [(C.GZIP, [pg], 2)])


def _build_malformed(tmp_path, name):
    codec, make = MALFORMED[name]
    data = H.plain([1, 2], H.INT64)
    if name == "gzip_distance_before_member":
        data = _CROSSING
    elif name.startswith("lz4"):
        data = b"abc" + b"\x00" * 4 + b"123456789"
    pg = C.page(H.DATA_PAGE, H.PLAIN, data, len(data) // 8, lambda _: make(data))
    return C.write_file(os.path.join(str(tmp_path), name + ".parquet"), "v", H.INT64, [(codec, [pg], len(data) // 8)])


# ---- CPU ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_handmade_files_read_back_through_pyarrow(tmp_path, name):
    path, values = _build_shape(tmp_path, name)
    assert pq.read_table(path).column(0).to_pylist() == values


@pytest.mark.parametrize("name", sorted(set(MALFORMED) - DEVICE_ONLY))
def test_malformed_pages_are_refused_by_pyarrow(tmp_path, name):
    path = _build_malformed(tmp_path, name)
    with pytest.raises(Exception):
        pq.read_table(path)


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_describe_codecs_of_handmade_files(tmp_path, name):
    path, _ = _build_shape(tmp_path, name)
    (c,) = bb.engine.parquet_describe(path)["columns"]
    md = pq.ParquetFile(path).metadata
    assert c["codecs"] == SHAPE_CODECS[name]
    assert c["codecs"] == sorted({CODEC_IDS[md.row_group(g).column(0).compression] for g in range(md.num_row_groups)})
    assert c["codec"] == CODEC_IDS[md.row_group(md.num_row_groups - 1).column(0).compression]


@pytest.mark.parametrize("compression", ["gzip", "lz4"])
def test_describe_codecs_of_pyarrow_files(tmp_path, compression):
    path = os.path.join(str(tmp_path), "c.parquet")
    pq.write_table(_table(3000), path, compression=compression, row_group_size=1000)
    md = pq.ParquetFile(path).metadata
    for i, c in enumerate(bb.engine.parquet_describe(path)["columns"]):
        ids = {CODEC_IDS[md.row_group(g).column(i).compression] for g in range(md.num_row_groups)}
        assert c["codecs"] == sorted(ids) == [2 if compression == "gzip" else 7]
        assert c["codec"] == c["codecs"][0]


def test_member_crossing_fixture_is_consistent():
    # read with the first member as its window, the second member inflates to the bytes its CRC32 and ISIZE describe, so
    # the crossing distance is the only thing wrong with gzip_distance_before_member
    d = zlib.decompressobj(wbits=-15, zdict=_FIRST)
    assert d.decompress(C.fixed_block([(3, 5)])) == _CROSSING[13:]


# ---- GPU ---------------------------------------------------------------------------------------------------------------------
def _scan(gpu, table, path, columns=None, partition=0):
    gpu.drop_table(table)
    gpu.register_parquet(table, partition, path, columns)
    return pa.Table.from_batches([gpu.export_table(table, partition)])


@pytest.mark.gpu
@pytest.mark.parametrize("nulls", [True, False])
@pytest.mark.parametrize("kw", VARIANTS)
@pytest.mark.parametrize("compression", ["gzip", "lz4"])
def test_pyarrow_compressed_files_match(gpu, tmp_path, compression, kw, nulls):
    t = _table(20000, nulls=nulls, seed=5)
    path = os.path.join(str(tmp_path), "c.parquet")
    pq.write_table(t, path, compression=compression, **kw)
    want = pq.read_table(path)
    assert_tables_equal(_scan(gpu, "pqc", path), want, sort=False)
    assert_tables_equal(_scan(gpu, "pqc", path, ["s", "d152", "i64"], 1), want.select(["s", "d152", "i64"]), sort=False)


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 9])
def test_gzip_levels_match(gpu, tmp_path, level):
    t = _table(30000, nulls=True, seed=level)
    path = os.path.join(str(tmp_path), "g.parquet")
    pq.write_table(t, path, compression="gzip", compression_level=level, row_group_size=10000, data_page_size=8192)
    assert_tables_equal(_scan(gpu, "pqg", path), pq.read_table(path), sort=False)


@pytest.mark.gpu
@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("which", sorted(ENCODING_SETS))
@pytest.mark.parametrize("compression", ["gzip", "lz4"])
def test_pyarrow_encoded_compressed_columns_match(gpu, tmp_path, compression, which, version):
    t = _encoded_table(20000, True, 13)
    path = _write_encoded(os.path.join(str(tmp_path), "e.parquet"), t, which, version, compression, row_group_size=7000, data_page_size=16384)
    assert_tables_equal(_scan(gpu, "pqe", path), pq.read_table(path), sort=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_handmade_shapes_decode(gpu, tmp_path, name):
    path, values = _build_shape(tmp_path, name)
    got = _scan(gpu, "pqh", path)
    assert_tables_equal(got, pq.read_table(path), sort=False)
    assert got.column(0).to_pylist() == values


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MALFORMED))
def test_malformed_pages_are_refused(gpu, tmp_path, name):
    path = _build_malformed(tmp_path, name)
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_parquet("pqbad", 0, path)
    assert ei.value.code == -1
    assert "column v" in str(ei.value)
    assert ("GZIP" if MALFORMED[name][0] == C.GZIP else "LZ4_RAW") in str(ei.value)
    ok_path, values = _build_shape(tmp_path, "mixed_codecs")   # the engine keeps working
    assert _scan(gpu, "pqh", ok_path).column(0).to_pylist() == values


@pytest.mark.gpu
def test_stored_v2_page_with_differing_sizes_is_refused(gpu, tmp_path):
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_parquet("pqbad", 0, _v2_stored_sizes_differ(tmp_path))
    assert ei.value.code == -1
    assert "column v" in str(ei.value)


@pytest.mark.gpu
def test_brotli_is_refused(gpu, tmp_path):
    path = os.path.join(str(tmp_path), "b.parquet")
    pq.write_table(_table(100), path, compression="brotli")
    with pytest.raises(bb.B200Error) as ei:
        gpu.register_parquet("pqb", 0, path)
    assert ei.value.code == -2


@pytest.mark.gpu
@pytest.mark.parametrize("compression", ["gzip", "lz4"])
def test_q1_q6_from_compressed_parquet(gpu, oracle, oracle_lib, tmp_path, compression):
    msf = 20
    cols = list(dict.fromkeys(tpch.Q1_COLUMNS + tpch.Q6_COLUMNS))
    n = oracle_lib.lib().oracle_tpch_table_rows(b"lineitem", msf)
    oracle.drop_table("lineitem")
    oracle.tpch_generate("lineitem", msf, 0, 0, n, cols)
    host = pa.Table.from_batches([oracle.export_table("lineitem", 0)])
    path = os.path.join(str(tmp_path), "lineitem.parquet")
    pq.write_table(host, path, compression=compression, row_group_size=50000)
    tpch.TABLE_LAYOUT["lineitem"] = cols
    try:
        gpu.drop_table("lineitem")
        gpu.register_parquet("lineitem", 0, path, cols)
        for name, st in (("q1", tpch.q1(4)), ("q6", tpch.q6(4))):
            got = driver.run_stages(gpu, st, f"pqc-{name}")
            want = driver.run_stages(oracle, st, f"pqc-{name}")
            assert_tables_equal(got, want, sort=False)
    finally:
        tpch.TABLE_LAYOUT.clear()
