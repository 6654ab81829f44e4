"""Hand-built compressed Parquet files for the GZIP and LZ4_RAW page decoders: one column, one row group per chunk, each
chunk with its own codec, pages compressed by whatever callable the test passes (Python's zlib / gzip in any strategy or
wrapper, pyarrow's Snappy and LZ4_RAW codecs, or the explicit LZ4 block writer below).  Formats restated from parquet.thrift
(PageHeader, ColumnMetaData), RFC 1950 / 1951 / 1952 and the LZ4 block format description."""
import struct
import zlib

import parquet_handmade as H

UNCOMPRESSED, SNAPPY, GZIP, LZ4_RAW = 0, 1, 2, 7


def _identity(b):
    return b


def page(kind, encoding, payload, num_values, compress=_identity, defs=None, v2_compressed=True):
    """One page whose `payload` (the encoded values) is stored as compress(...).  V1 pages compress the levels with the
    values; V2 pages keep the levels raw and compress only the values (not at all when v2_compressed is False)."""
    h = H.Struct().i32(1, kind)
    if kind == H.DICTIONARY_PAGE:
        stored = compress(payload)
        sub = H.Struct().i32(1, num_values).i32(2, encoding)
        return h.i32(2, len(payload)).i32(3, len(stored)).struct(7, sub).bytes() + stored
    if kind == H.DATA_PAGE:
        body = payload
        if defs is not None:
            lv = H.hybrid(defs, 1)
            body = struct.pack("<I", len(lv)) + lv + payload
        stored = compress(body)
        sub = H.Struct().i32(1, num_values).i32(2, encoding).i32(3, H.RLE).i32(4, H.RLE)
        return h.i32(2, len(body)).i32(3, len(stored)).struct(5, sub).bytes() + stored
    lv = H.hybrid(defs, 1) if defs is not None else b""
    vals = compress(payload) if v2_compressed else payload
    nulls = defs.count(0) if defs is not None else 0
    sub = (H.Struct().i32(1, num_values).i32(2, nulls).i32(3, num_values).i32(4, encoding).i32(5, len(lv)).i32(6, 0)
           .boolean(7, v2_compressed))
    return h.i32(2, len(lv) + len(payload)).i32(3, len(lv) + len(vals)).struct(8, sub).bytes() + lv + vals


def plain_pages(kind, phys, values, page_rows, compress, optional=False):
    """PLAIN data pages of `page_rows` rows (None = NULL when optional)."""
    out = []
    for r0 in range(0, len(values), page_rows):
        chunk = values[r0:r0 + page_rows]
        present = [v for v in chunk if v is not None]
        defs = [0 if v is None else 1 for v in chunk] if optional else None
        out.append(page(kind, H.PLAIN, H.plain(present, phys), len(chunk), compress, defs))
    return out


def write_file(path, name, phys, chunks, *, optional=False, string=False):
    """chunks: [(codec, [page bytes], rows)], one row group each."""
    col = bytearray()
    rgs = []
    for codec, pages, rows in chunks:
        start = 4 + len(col)
        body = b"".join(pages)
        col += body
        encodings = sorted({H.PLAIN, H.RLE})
        md = (H.Struct().i32(1, phys).list(2, H._I32, encodings).list(3, H._BINARY, [name.encode()]).i32(4, codec).i64(5, rows)
              .i64(6, len(body)).i64(7, len(body)).i64(9, start))
        chunk = H.Struct().i64(2, start).struct(3, md)
        rgs.append(H.Struct().list(1, H._STRUCT, [chunk]).i64(2, len(body)).i64(3, rows))
    leaf = H.Struct().i32(1, phys).i32(3, 1 if optional else 0).binary(4, name.encode())
    if string:
        leaf.i32(6, 0)
    root = H.Struct().binary(4, b"schema").i32(5, 1)
    n = sum(r for _, _, r in chunks)
    fmd = H.Struct().i32(1, 1).list(2, H._STRUCT, [root, leaf]).i64(3, n).list(4, H._STRUCT, rgs).bytes()
    with open(path, "wb") as f:
        f.write(b"PAR1" + bytes(col) + fmd + struct.pack("<I", len(fmd)) + b"PAR1")
    return path


# ---- DEFLATE wrappers ------------------------------------------------------------------------------------------------------
def deflate_raw(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    return c.compress(data) + c.flush()


def gzip_member(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, extra=None, name=None, comment=None, hcrc=False):
    """RFC 1952 member with the optional header fields asked for."""
    flg = (2 if hcrc else 0) | (4 if extra is not None else 0) | (8 if name is not None else 0) | (16 if comment is not None else 0)
    h = bytearray(b"\x1f\x8b\x08" + bytes([flg]) + b"\x00\x00\x00\x00\x00\xff")
    if extra is not None:
        h += struct.pack("<H", len(extra)) + extra
    if name is not None:
        h += name + b"\x00"
    if comment is not None:
        h += comment + b"\x00"
    if hcrc:
        h += struct.pack("<H", zlib.crc32(bytes(h)) & 0xFFFF)
    return bytes(h) + deflate_raw(data, level, strategy) + struct.pack("<II", zlib.crc32(data), len(data) & 0xFFFFFFFF)


def fixed_block(tokens):
    """One final fixed-Huffman deflate block: tokens are literal byte values or (length, distance) with length 3 and a
    distance of 5-6 (distance code 4, one extra bit)."""
    acc, n = 0, 0

    def put(v, k):
        nonlocal acc, n
        acc |= v << n
        n += k

    def code(c, k):  # Huffman codes go most significant bit first
        put(int(format(c, "0%db" % k)[::-1], 2), k)
    put(1, 1)
    put(1, 2)
    for t in tokens:
        if isinstance(t, tuple):
            length, dist = t
            assert length == 3 and dist in (5, 6)
            code(1, 7)          # symbol 257: length 3
            code(4, 5)          # distance code 4: 5 + one extra bit
            put(dist - 5, 1)
        else:
            code(0x30 + t, 8)   # literals 0-143
    code(0, 7)                  # end of block
    return acc.to_bytes((n + 7) // 8, "little")


# ---- LZ4 block format ------------------------------------------------------------------------------------------------------
def _lz4_len(v):
    out = bytearray()
    while v >= 255:
        out.append(255)
        v -= 255
    out.append(v)
    return bytes(out)


def lz4_block(seqs, last):
    """(block, decoded bytes) for sequences [(literals, offset, match length)] followed by the final literals `last`.
    Offsets are written as given (0 and out-of-range offsets too); decoding stops at the first one that is not valid."""
    out, data, valid = bytearray(), bytearray(), True
    for lit, off, ml in seqs + [(last, None, None)]:
        ln = len(lit)
        m = 0 if ml is None else ml - 4
        out.append((min(ln, 15) << 4) | min(m, 15))
        if ln >= 15:
            out += _lz4_len(ln - 15)
        out += lit
        data += lit
        if ml is None:
            break
        out += struct.pack("<H", off)
        if m >= 15:
            out += _lz4_len(m - 15)
        valid = valid and 0 < off <= len(data)
        if valid:
            for _ in range(ml):
                data.append(data[-off])
    return bytes(out), bytes(data)
