// Parquet footer + page-header reader (host side of the device Parquet scan).
//
// Stands behind DataSourceExec + ParquetSource (ballista/core/proto/datafusion.proto:1058-1077; registration path
// benchmarks/src/bin/tpch.rs:684-693): the reference decodes pages on CPU threads (parquet 58.1 [EXT]); here the host only
// parses METADATA -- the Thrift-compact FileMetaData at the end of the file and the PageHeader in front of every page --
// and ships the raw column-chunk bytes to HBM, where csrc/device/parquet.cu decodes levels, dictionaries and values.
// Format facts restated from the Apache Parquet specification (parquet-format: Thrift definitions `FileMetaData`,
// `SchemaElement`, `RowGroup`, `ColumnChunk`, `ColumnMetaData`, `PageHeader`, `DataPageHeader[V2]`, `DictionaryPageHeader`;
// Encodings.md: PLAIN, RLE/bit-packed hybrid, RLE_DICTIONARY, DELTA_*, BYTE_STREAM_SPLIT).  Supported: flat schemas, physical
// types BOOLEAN / INT32 / INT64 / DOUBLE / BYTE_ARRAY / FIXED_LEN_BYTE_ARRAY, logical DECIMAL / DATE / STRING, encodings PLAIN,
// [PLAIN|RLE]_DICTIONARY, DELTA_BINARY_PACKED, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY and BYTE_STREAM_SPLIT, data pages V1
// and V2, codecs UNCOMPRESSED, SNAPPY, GZIP and LZ4_RAW (a column may use a different codec in each row group).  Everything else,
// including BROTLI, LZO, ZSTD and the deprecated Hadoop-framed LZ4, is reported as unsupported.
#pragma once
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace b200 {
namespace pq {

enum PhysType : int32_t { T_BOOLEAN = 0, T_INT32 = 1, T_INT64 = 2, T_INT96 = 3, T_FLOAT = 4, T_DOUBLE = 5, T_BYTE_ARRAY = 6, T_FLBA = 7 };
enum Encoding : int32_t {
  E_PLAIN = 0, E_PLAIN_DICTIONARY = 2, E_RLE = 3, E_BIT_PACKED = 4, E_DELTA_BINARY_PACKED = 5, E_DELTA_LENGTH_BYTE_ARRAY = 6, E_DELTA_BYTE_ARRAY = 7,
  E_RLE_DICTIONARY = 8, E_BYTE_STREAM_SPLIT = 9
};
enum PageType : int32_t { P_DATA = 0, P_INDEX = 1, P_DICTIONARY = 2, P_DATA_V2 = 3 };
enum Codec : int32_t { C_UNCOMPRESSED = 0, C_SNAPPY = 1, C_GZIP = 2, C_LZO = 3, C_BROTLI = 4, C_LZ4 = 5, C_ZSTD = 6, C_LZ4_RAW = 7 };

struct ThriftReader {
  const uint8_t* p;
  const uint8_t* end;
  ThriftReader(const uint8_t* b, const uint8_t* e) : p(b), end(e) {}
  uint8_t byte() {
    if (p >= end) throw std::runtime_error("parquet: truncated thrift data");
    return *p++;
  }
  uint64_t varint() {
    uint64_t v = 0;
    for (int shift = 0; shift < 64; shift += 7) {
      const uint8_t b = byte();
      v |= (uint64_t)(b & 0x7F) << shift;
      if (!(b & 0x80)) return v;
    }
    throw std::runtime_error("parquet: bad varint");
  }
  int64_t zigzag() {
    const uint64_t v = varint();
    return (int64_t)(v >> 1) ^ -(int64_t)(v & 1);
  }
  std::string binary() {
    const uint64_t n = varint();
    if ((uint64_t)(end - p) < n) throw std::runtime_error("parquet: truncated thrift binary");
    std::string s((const char*)p, (size_t)n);
    p += n;
    return s;
  }
  // field header: returns false at STOP; *type in thrift compact type codes, *id the field id
  bool field(int* type, int* id, int* last_id) {
    const uint8_t h = byte();
    if (h == 0) return false;
    *type = h & 0x0F;
    const int delta = h >> 4;
    *id = delta ? *last_id + delta : (int)zigzag();
    *last_id = *id;
    return true;
  }
  void list_header(int* elem_type, uint64_t* n) {
    const uint8_t h = byte();
    *elem_type = h & 0x0F;
    *n = h >> 4;
    if (*n == 15) *n = varint();
  }
  void skip(int type) {
    switch (type) {
      case 1: case 2: break;  // bool true / false carried by the type
      case 3: byte(); break;
      case 4: case 5: case 6: zigzag(); break;
      case 7:
        if (end - p < 8) throw std::runtime_error("parquet: truncated double");
        p += 8;
        break;
      case 8: binary(); break;
      case 9: case 10: {
        int et;
        uint64_t n;
        list_header(&et, &n);
        for (uint64_t i = 0; i < n; i++) {
          if (et == 1 || et == 2) byte();  // bools inside a list take one byte each
          else skip(et);
        }
        break;
      }
      case 11: {
        const uint64_t n = varint();
        if (n) {
          const uint8_t kv = byte();
          for (uint64_t i = 0; i < n; i++) {
            skip(kv >> 4);
            skip(kv & 0x0F);
          }
        }
        break;
      }
      case 12: {
        int t, id, last = 0;
        while (field(&t, &id, &last)) skip(t);
        break;
      }
      default: throw std::runtime_error("parquet: unknown thrift type");
    }
  }
};

struct SchemaElement {
  std::string name;
  int32_t type = -1, type_length = 0, repetition = 0, num_children = 0, converted = -1, scale = 0, precision = 0;
  int logical = 0;  // 1 STRING, 5 DECIMAL, 6 DATE (LogicalType union field ids), 0 none
};
struct ColumnChunkMeta {
  int32_t type = -1, codec = 0;
  std::vector<std::string> path;
  int64_t num_values = 0, total_compressed = 0, total_uncompressed = 0, data_page_offset = 0, dictionary_page_offset = -1;
};
struct RowGroupMeta {
  std::vector<ColumnChunkMeta> columns;
  int64_t num_rows = 0;
};
struct FileMeta {
  std::vector<SchemaElement> schema;  // [0] is the root
  std::vector<RowGroupMeta> row_groups;
  int64_t num_rows = 0;
};

inline SchemaElement read_schema_element(ThriftReader& r) {
  SchemaElement e;
  int t, id, last = 0;
  while (r.field(&t, &id, &last)) {
    switch (id) {
      case 1: e.type = (int32_t)r.zigzag(); break;
      case 2: e.type_length = (int32_t)r.zigzag(); break;
      case 3: e.repetition = (int32_t)r.zigzag(); break;
      case 4: e.name = r.binary(); break;
      case 5: e.num_children = (int32_t)r.zigzag(); break;
      case 6: e.converted = (int32_t)r.zigzag(); break;
      case 7: e.scale = (int32_t)r.zigzag(); break;
      case 8: e.precision = (int32_t)r.zigzag(); break;
      case 10: {  // LogicalType union: the set field id names the type
        int t2, id2, last2 = 0;
        while (r.field(&t2, &id2, &last2)) {
          e.logical = id2;
          if (id2 == 5 && t2 == 12) {  // DecimalType {1: scale, 2: precision}
            int t3, id3, last3 = 0;
            while (r.field(&t3, &id3, &last3)) {
              if (id3 == 1) e.scale = (int32_t)r.zigzag();
              else if (id3 == 2) e.precision = (int32_t)r.zigzag();
              else r.skip(t3);
            }
          } else {
            r.skip(t2);
          }
        }
        break;
      }
      default: r.skip(t);
    }
  }
  return e;
}

inline ColumnChunkMeta read_column_meta(ThriftReader& r) {
  ColumnChunkMeta m;
  int t, id, last = 0;
  while (r.field(&t, &id, &last)) {
    switch (id) {
      case 1: m.type = (int32_t)r.zigzag(); break;
      case 3: {
        int et;
        uint64_t n;
        r.list_header(&et, &n);
        for (uint64_t i = 0; i < n; i++) m.path.push_back(r.binary());
        break;
      }
      case 4: m.codec = (int32_t)r.zigzag(); break;
      case 5: m.num_values = r.zigzag(); break;
      case 6: m.total_uncompressed = r.zigzag(); break;
      case 7: m.total_compressed = r.zigzag(); break;
      case 9: m.data_page_offset = r.zigzag(); break;
      case 11: m.dictionary_page_offset = r.zigzag(); break;
      default: r.skip(t);
    }
  }
  return m;
}

inline FileMeta read_file_meta(const uint8_t* file, size_t size) {
  if (size < 12 || memcmp(file, "PAR1", 4) != 0 || memcmp(file + size - 4, "PAR1", 4) != 0) throw std::runtime_error("parquet: not a Parquet file (magic)");
  uint32_t flen;
  memcpy(&flen, file + size - 8, 4);
  if ((size_t)flen + 12 > size) throw std::runtime_error("parquet: bad footer length");
  ThriftReader r(file + size - 8 - flen, file + size - 8);
  FileMeta fm;
  int t, id, last = 0;
  while (r.field(&t, &id, &last)) {
    if (id == 2 && t == 9) {
      int et;
      uint64_t n;
      r.list_header(&et, &n);
      for (uint64_t i = 0; i < n; i++) fm.schema.push_back(read_schema_element(r));
    } else if (id == 3) {
      fm.num_rows = r.zigzag();
    } else if (id == 4 && t == 9) {
      int et;
      uint64_t n;
      r.list_header(&et, &n);
      for (uint64_t i = 0; i < n; i++) {
        RowGroupMeta rg;
        int t2, id2, last2 = 0;
        while (r.field(&t2, &id2, &last2)) {
          if (id2 == 1 && t2 == 9) {
            int et2;
            uint64_t n2;
            r.list_header(&et2, &n2);
            for (uint64_t c = 0; c < n2; c++) {
              ColumnChunkMeta cm;
              int t3, id3, last3 = 0;
              while (r.field(&t3, &id3, &last3)) {
                if (id3 == 3 && t3 == 12) cm = read_column_meta(r);
                else r.skip(t3);
              }
              rg.columns.push_back(cm);
            }
          } else if (id2 == 3) {
            rg.num_rows = r.zigzag();
          } else {
            r.skip(t2);
          }
        }
        fm.row_groups.push_back(rg);
      }
    } else {
      r.skip(t);
    }
  }
  return fm;
}

struct PageHeader {
  int32_t type = -1, uncompressed_size = 0, compressed_size = 0;
  int32_t num_values = 0, encoding = 0, def_encoding = E_RLE;
  int32_t num_nulls = -1, def_bytes = 0, rep_bytes = 0;  // V2
  bool v2_compressed = true;
  size_t header_bytes = 0;
};

inline PageHeader read_page_header(const uint8_t* p, const uint8_t* end) {
  ThriftReader r(p, end);
  PageHeader h;
  int t, id, last = 0;
  while (r.field(&t, &id, &last)) {
    switch (id) {
      case 1: h.type = (int32_t)r.zigzag(); break;
      case 2: h.uncompressed_size = (int32_t)r.zigzag(); break;
      case 3: h.compressed_size = (int32_t)r.zigzag(); break;
      case 5: {  // DataPageHeader
        int t2, id2, last2 = 0;
        while (r.field(&t2, &id2, &last2)) {
          if (id2 == 1) h.num_values = (int32_t)r.zigzag();
          else if (id2 == 2) h.encoding = (int32_t)r.zigzag();
          else if (id2 == 3) h.def_encoding = (int32_t)r.zigzag();
          else r.skip(t2);
        }
        break;
      }
      case 7: {  // DictionaryPageHeader
        int t2, id2, last2 = 0;
        while (r.field(&t2, &id2, &last2)) {
          if (id2 == 1) h.num_values = (int32_t)r.zigzag();
          else if (id2 == 2) h.encoding = (int32_t)r.zigzag();
          else r.skip(t2);
        }
        break;
      }
      case 8: {  // DataPageHeaderV2
        int t2, id2, last2 = 0;
        while (r.field(&t2, &id2, &last2)) {
          if (id2 == 1) h.num_values = (int32_t)r.zigzag();
          else if (id2 == 2) h.num_nulls = (int32_t)r.zigzag();
          else if (id2 == 4) h.encoding = (int32_t)r.zigzag();
          else if (id2 == 5) h.def_bytes = (int32_t)r.zigzag();
          else if (id2 == 6) h.rep_bytes = (int32_t)r.zigzag();
          else if (id2 == 7) h.v2_compressed = (t2 == 1);
          else r.skip(t2);
        }
        break;
      }
      default: r.skip(t);
    }
  }
  h.header_bytes = (size_t)(r.p - p);
  return h;
}

}  // namespace pq
}  // namespace b200
