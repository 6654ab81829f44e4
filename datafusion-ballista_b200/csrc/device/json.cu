// Newline-delimited JSON scan on the GPU (sm_90a): record boundaries, an RFC 8259 tokenizer per record and per-type
// conversion into the engine's HBM column layout (Arrow fixed-width values, one validity byte per row, 16-byte views).
//
// Reference path: DataSourceExec + JsonSource (JsonScanExecNode, ballista/core/proto/datafusion.proto:1103-1105) ->
// arrow-json [EXT] on CPU threads.  Here the host only copies the file bytes to HBM; every pass below runs on the device:
//   1. json_tiles_kernel: one thread per JSON_TILE bytes counts the records that start in its tile.  A raw '\n' cannot occur
//      inside a valid JSON value, so a record starts at every line start whose line holds more than whitespace (space, tab,
//      '\r'); no string state is needed.  Each block sums its tiles.
//   2. json_block_scan_kernel: one block turns the block counts into every block's first record (and the record count).
//   3. json_record_starts_kernel: every tile with a record start re-scans its bytes and writes its record starts.
//   4. json_fields_kernel: one thread per record walks the line as RFC 8259 JSON (one object per line), looks every
//      top-level key up, after unescaping it, in a shared-memory table of the materialised names (hash, then a byte
//      compare) and keeps a {pointer, length | kind << 32} view of each materialised value.  Strings holding a '\' are
//      unescaped into a side buffer at the same offset (the escaped form is never shorter).  Unknown keys' values are
//      skipped with the nesting tracked in a 64-level bit stack, so every token of the line is checked.
//   5. json_convert_kernel<family>: the CSV scan's converters (text_convert.cuh) with JSON's NULL (a null pointer) and kinds.
// Errors never stop a kernel: each column and the structure keep one 64-bit word, atomicMin of
// (row << 24 | reason << 16 | detail), so the host reports the first failing record after one read-back.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "text_convert.cuh"

namespace b200 {

__device__ __forceinline__ bool json_ws(uint8_t b) { return b == ' ' || b == '\t' || b == '\r'; }  // '\n' ends a record

// the line that starts at data[i] with the whitespace byte data[i] holds more than whitespace
__device__ bool json_line_has_value(const uint8_t* data, int64_t i, int64_t bytes) {
  for (; i < bytes; i++) {
    const uint8_t b = data[i];
    if (b == '\n') return false;
    if (!json_ws(b)) return true;
  }
  return false;
}

// a record starts at i (which starts a line) unless its line is blank
__device__ __forceinline__ bool json_record_at(const uint8_t* data, int64_t i, int64_t bytes, uint8_t b) {
  return b != '\n' && (!json_ws(b) || json_line_has_value(data, i, bytes));
}

// ---- record boundaries -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(JSON_BLOCK) json_tiles_kernel(const uint8_t* data, int64_t bytes, uint32_t* tile_cnt, unsigned long long* blk_cnt,
                                                                unsigned int* has_backslash) {
  __shared__ uint32_t sh[JSON_BLOCK];
  const int64_t t = (int64_t)blockIdx.x * JSON_BLOCK + threadIdx.x;
  const int64_t lo = t * JSON_TILE, hi = lo + JSON_TILE < bytes ? lo + JSON_TILE : bytes;
  uint32_t c = 0;
  if (lo < bytes) {
    bool bs = false;
    uint8_t prev = lo ? data[lo - 1] : (uint8_t)'\n';
    for (int64_t i = lo; i < hi; i++) {
      const uint8_t b = data[i];
      bs |= b == '\\';
      if (prev == '\n' && json_record_at(data, i, bytes, b)) c++;
      prev = b;
    }
    tile_cnt[t] = c;
    // any '\' at all: the host then provides the unescaping side buffer
    if (bs) atomicOr(has_backslash, 1u);
  }
  sh[threadIdx.x] = c;
  __syncthreads();
  for (int w = 1; w < JSON_BLOCK; w <<= 1) {
    if ((threadIdx.x & (2 * w - 1)) == 0) sh[threadIdx.x] += sh[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = sh[0];
}

// in place: blk[b] = the records of the blocks before b
__global__ void __launch_bounds__(1024) json_block_scan_kernel(unsigned long long* blk, int64_t n_blocks, unsigned long long* n_records) {
  __shared__ unsigned long long base[1024];
  const int64_t per = (n_blocks + 1023) / 1024;
  const int64_t b0 = threadIdx.x * per, b1 = b0 + per < n_blocks ? b0 + per : n_blocks;
  unsigned long long s = 0;
  for (int64_t b = b0; b < b1; b++) s += blk[b];
  base[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long n = 0;
    for (int k = 0; k < 1024; k++) {
      const unsigned long long v = base[k];
      base[k] = n;
      n += v;
    }
    *n_records = n;
  }
  __syncthreads();
  unsigned long long n = base[threadIdx.x];
  for (int64_t b = b0; b < b1; b++) {
    const unsigned long long v = blk[b];
    blk[b] = n;
    n += v;
  }
}

__global__ void __launch_bounds__(JSON_BLOCK) json_record_starts_kernel(const uint8_t* data, int64_t bytes, const uint32_t* tile_cnt,
                                                                        const unsigned long long* blk_base, uint64_t* rec_start) {
  __shared__ unsigned long long base[JSON_BLOCK];
  const int64_t t0 = (int64_t)blockIdx.x * JSON_BLOCK;
  const int64_t n_tiles = (bytes + JSON_TILE - 1) / JSON_TILE;
  if (threadIdx.x == 0) {
    unsigned long long n = blk_base[blockIdx.x];
    for (int k = 0; k < JSON_BLOCK && t0 + k < n_tiles; k++) {
      base[k] = n;
      n += tile_cnt[t0 + k];
    }
  }
  __syncthreads();
  const int64_t t = t0 + threadIdx.x;
  if (t >= n_tiles || tile_cnt[t] == 0) return;
  const int64_t lo = t * JSON_TILE, hi = lo + JSON_TILE < bytes ? lo + JSON_TILE : bytes;
  unsigned long long n = base[threadIdx.x];
  uint8_t prev = lo ? data[lo - 1] : (uint8_t)'\n';
  for (int64_t i = lo; i < hi; i++) {
    const uint8_t b = data[i];
    if (prev == '\n' && json_record_at(data, i, bytes, b)) rec_start[n++] = (uint64_t)i;
    prev = b;
  }
}

int64_t json_tile_count(int64_t bytes) { return (bytes + JSON_TILE - 1) / JSON_TILE; }
int64_t json_block_count(int64_t bytes) { return (json_tile_count(bytes) + JSON_BLOCK - 1) / JSON_BLOCK; }

void launch_json_records_count(const uint8_t* data, int64_t bytes, uint32_t* tile_cnt, unsigned long long* blk_base, unsigned int* has_backslash,
                               unsigned long long* n_records, cudaStream_t st) {
  const int64_t nb = json_block_count(bytes);
  launch_kernel(json_tiles_kernel, dim3((unsigned)nb), dim3(JSON_BLOCK), 0, st, data, bytes, tile_cnt, blk_base, has_backslash);
  launch_kernel(json_block_scan_kernel, dim3(1), dim3(1024), 0, st, blk_base, nb, n_records);
}

void launch_json_record_starts(const uint8_t* data, int64_t bytes, const uint32_t* tile_cnt, const unsigned long long* blk_base, uint64_t* rec_start,
                               cudaStream_t st) {
  const int64_t nb = json_block_count(bytes);
  launch_kernel(json_record_starts_kernel, dim3((unsigned)nb), dim3(JSON_BLOCK), 0, st, data, bytes, tile_cnt, blk_base, rec_start);
}

// ---- tokens ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int json_hex4(const uint8_t* d, int64_t at, int64_t end, uint32_t& cp) {
  if (at + 4 > end) return JSON_E_ESCAPE;
  cp = 0;
  for (int k = 0; k < 4; k++) {
    const uint8_t b = d[at + k];
    const int v = (b >= '0' && b <= '9') ? b - '0' : (b >= 'a' && b <= 'f') ? b - 'a' + 10 : (b >= 'A' && b <= 'F') ? b - 'A' + 10 : -1;
    if (v < 0) return JSON_E_ESCAPE;
    cp = cp * 16 + (uint32_t)v;
  }
  return 0;
}

// the string whose opening quote is at d[i]: on success i is past the closing quote, the content starts at c0 and is ulen
// bytes long once unescaped (in side + c0 when esc), hash is its FNV-1a hash.  Raw bytes below 0x20, invalid UTF-8, unknown
// escapes and lone surrogates are refused.
__device__ int json_string(const uint8_t* d, int64_t& i, int64_t end, uint8_t* side, int64_t& c0, uint32_t& ulen, bool& esc, uint32_t& hash) {
  c0 = ++i;
  esc = false;
  uint32_t h = JSON_HASH_SEED;
  int64_t o = c0;  // next output byte (equal to i until the first escape)
  for (;;) {
    if (i >= end) return JSON_E_UNTERMINATED;
    const uint8_t b = d[i];
    if (b == '"') {
      i++;
      break;
    }
    if (b < 0x20) return b == '\n' ? JSON_E_UNTERMINATED : JSON_E_CONTROL;
    if (b == '\\') {
      if (!esc) {
        for (int64_t k = c0; k < i; k++) side[k] = d[k];
        esc = true;
      }
      if (i + 1 >= end) return JSON_E_UNTERMINATED;
      const uint8_t e = d[i + 1];
      uint32_t cp;
      i += 2;
      switch (e) {
        case '"': case '\\': case '/': cp = e; break;
        case 'b': cp = 8; break;
        case 'f': cp = 12; break;
        case 'n': cp = 10; break;
        case 'r': cp = 13; break;
        case 't': cp = 9; break;
        case 'u': {
          if (json_hex4(d, i, end, cp)) return JSON_E_ESCAPE;
          i += 4;
          if (cp >= 0xDC00 && cp <= 0xDFFF) return JSON_E_SURROGATE;
          if (cp >= 0xD800 && cp <= 0xDBFF) {
            uint32_t lo;
            if (i + 1 >= end || d[i] != '\\' || d[i + 1] != 'u') return JSON_E_SURROGATE;
            if (json_hex4(d, i + 2, end, lo)) return JSON_E_ESCAPE;
            if (lo < 0xDC00 || lo > 0xDFFF) return JSON_E_SURROGATE;
            cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
            i += 6;
          }
          break;
        }
        default: return JSON_E_ESCAPE;
      }
      uint8_t u[4];
      int n;
      if (cp < 0x80) {
        u[0] = (uint8_t)cp;
        n = 1;
      } else if (cp < 0x800) {
        u[0] = (uint8_t)(0xC0 | (cp >> 6));
        u[1] = (uint8_t)(0x80 | (cp & 0x3F));
        n = 2;
      } else if (cp < 0x10000) {
        u[0] = (uint8_t)(0xE0 | (cp >> 12));
        u[1] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F));
        u[2] = (uint8_t)(0x80 | (cp & 0x3F));
        n = 3;
      } else {
        u[0] = (uint8_t)(0xF0 | (cp >> 18));
        u[1] = (uint8_t)(0x80 | ((cp >> 12) & 0x3F));
        u[2] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F));
        u[3] = (uint8_t)(0x80 | (cp & 0x3F));
        n = 4;
      }
      for (int k = 0; k < n; k++) {
        side[o++] = u[k];
        h = json_hash_step(h, u[k]);
      }
      continue;
    }
    int len = 1;
    if (b >= 0x80) {
      uint32_t cp;
      if (b >= 0xC2 && b <= 0xDF) {
        len = 2;
        cp = b & 0x1F;
      } else if (b >= 0xE0 && b <= 0xEF) {
        len = 3;
        cp = b & 0x0F;
      } else if (b >= 0xF0 && b <= 0xF4) {
        len = 4;
        cp = b & 0x07;
      } else {
        return JSON_E_UTF8;
      }
      if (i + len > end) return JSON_E_UTF8;
      for (int j = 1; j < len; j++) {
        const uint8_t c = d[i + j];
        if ((c & 0xC0) != 0x80) return JSON_E_UTF8;
        cp = (cp << 6) | (c & 0x3F);
      }
      if ((len == 3 && (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF))) || (len == 4 && (cp < 0x10000 || cp > 0x10FFFF))) return JSON_E_UTF8;
    }
    for (int k = 0; k < len; k++) {
      const uint8_t c = d[i + k];
      h = json_hash_step(h, c);
      if (esc) side[o] = c;
      o++;
    }
    i += len;
  }
  ulen = (uint32_t)(o - c0);
  hash = h;
  return 0;
}

__device__ __forceinline__ bool json_digit(uint8_t b) { return b >= '0' && b <= '9'; }

// -?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)? starting at d[i]; i ends past it
__device__ int json_number(const uint8_t* d, int64_t& i, int64_t end) {
  if (d[i] == '-') i++;
  if (i >= end || !json_digit(d[i])) return JSON_E_NUMBER;
  if (d[i] == '0') i++;
  else
    while (i < end && json_digit(d[i])) i++;
  if (i < end && d[i] == '.') {
    i++;
    if (i >= end || !json_digit(d[i])) return JSON_E_NUMBER;
    while (i < end && json_digit(d[i])) i++;
  }
  if (i < end && (d[i] == 'e' || d[i] == 'E')) {
    i++;
    if (i < end && (d[i] == '+' || d[i] == '-')) i++;
    if (i >= end || !json_digit(d[i])) return JSON_E_NUMBER;
    while (i < end && json_digit(d[i])) i++;
  }
  return 0;
}

__device__ __forceinline__ bool json_lit(const uint8_t* d, int64_t i, int64_t end, const char* lit) {
  for (int k = 0; lit[k]; k++)
    if (i + k >= end || d[i + k] != (uint8_t)lit[k]) return false;
  return true;
}

__device__ __forceinline__ int json_lookup(const JsonKey* keys, int n_keys, const uint8_t* names, const uint8_t* p, uint32_t n, uint32_t hash) {
  const uint32_t m = (uint32_t)n_keys - 1;
  for (uint32_t k = hash & m;; k = (k + 1) & m) {
    const JsonKey e = keys[k];
    if (e.slot < 0) return -1;
    if (e.hash == hash && e.len == n) {
      uint32_t j = 0;
      while (j < n && names[e.off + j] == p[j]) j++;
      if (j == n) return e.slot;
    }
  }
}

// ---- fields --------------------------------------------------------------------------------------------------------------
enum JsonExpect : int { JX_KEY_OR_CLOSE = 0, JX_KEY, JX_VALUE, JX_VALUE_OR_CLOSE, JX_AFTER };

// one record: the line starting at data[i] (a non-blank line); returns 0 or the first error (detail: *detail)
__device__ int json_record(const JsonFieldArgs& A, const JsonKey* keys, const uint8_t* names, int64_t row, int64_t i, uint32_t* detail) {
  const uint8_t* d = A.data;
  const int64_t end = A.bytes;
  while (i < end && json_ws(d[i])) i++;
  if (d[i] != '{') return JSON_E_NOT_OBJECT;
  i++;
  uint64_t stack = 0;  // bit k - 1: nesting level k (below the top-level object) is an object
  int depth = 0;
  int s = JX_KEY_OR_CLOSE;
  int slot = -1;       // output slot of the current top-level member
  int64_t v0 = 0;      // first byte of a materialised nested value
  auto put = [&](const uint8_t* p, uint64_t len, int kind) -> int {
    unsigned long long* v = A.views + ((size_t)slot * (size_t)A.n_total + (size_t)row) * 2;
    if (v[0] | v[1]) {
      *detail = (uint32_t)slot;
      return JSON_E_DUPLICATE;
    }
    v[0] = (unsigned long long)p;
    v[1] = len | ((unsigned long long)kind << 32);
    return 0;
  };
  for (;;) {
    while (i < end && json_ws(d[i])) i++;
    if (i >= end || d[i] == '\n') return JSON_E_UNTERMINATED;
    const uint8_t b = d[i];
    const bool obj = depth == 0 || ((stack >> (depth - 1)) & 1);
    bool close = false;
    if (s == JX_KEY_OR_CLOSE || s == JX_VALUE_OR_CLOSE) {
      if (b == (s == JX_KEY_OR_CLOSE ? '}' : ']')) close = true;
      else s = s == JX_KEY_OR_CLOSE ? JX_KEY : JX_VALUE;
    }
    if (!close && s == JX_KEY) {
      if (b != '"') return JSON_E_SYNTAX;
      int64_t c0;
      uint32_t n, h;
      bool esc;
      const int rc = json_string(d, i, end, A.side, c0, n, esc, h);
      if (rc) return rc;
      while (i < end && json_ws(d[i])) i++;
      if (i >= end || d[i] == '\n') return JSON_E_UNTERMINATED;
      if (d[i] != ':') return JSON_E_SYNTAX;
      i++;
      if (depth == 0) slot = A.n_keys ? json_lookup(keys, A.n_keys, names, esc ? A.side + c0 : d + c0, n, h) : -1;
      s = JX_VALUE;
      continue;
    }
    if (!close && s == JX_VALUE) {
      if (b == '{' || b == '[') {
        if (depth == JSON_MAX_DEPTH) return JSON_E_DEPTH;
        if (depth == 0) v0 = i;
        if (b == '{') stack |= 1ull << depth;
        else stack &= ~(1ull << depth);
        depth++;
        i++;
        s = b == '{' ? JX_KEY_OR_CLOSE : JX_VALUE_OR_CLOSE;
        continue;
      }
      const int64_t at = i;
      const uint8_t* p = d + at;
      uint64_t len;
      int kind;
      if (b == '"') {
        int64_t c0;
        uint32_t n, h;
        bool esc;
        const int rc = json_string(d, i, end, A.side, c0, n, esc, h);
        if (rc) return rc;
        p = esc ? A.side + c0 : d + c0;
        len = n;
        kind = JK_STRING;
      } else if (b == '-' || json_digit(b)) {
        const int rc = json_number(d, i, end);
        if (rc) return rc;
        len = (uint64_t)(i - at);
        kind = JK_NUMBER;
      } else if (json_lit(d, i, end, "true")) {
        i += 4;
        len = 4;
        kind = JK_TRUE;
      } else if (json_lit(d, i, end, "false")) {
        i += 5;
        len = 5;
        kind = JK_FALSE;
      } else if (json_lit(d, i, end, "null")) {
        i += 4;
        p = nullptr;
        len = 0;
        kind = JK_NULL;
      } else {
        return (b >= 'a' && b <= 'z') || (b >= 'A' && b <= 'Z') ? JSON_E_LITERAL : JSON_E_SYNTAX;
      }
      if (depth == 0 && slot >= 0) {
        const int rc = put(p, len, kind);
        if (rc) return rc;
      }
      s = JX_AFTER;
      continue;
    }
    if (!close) {  // JX_AFTER: ',' or the close of the current container
      if (b == ',') {
        i++;
        s = obj ? JX_KEY : JX_VALUE;
        continue;
      }
      if (b != (obj ? '}' : ']')) return JSON_E_SYNTAX;
    }
    i++;
    if (depth == 0) break;  // the top-level object is complete
    depth--;
    if (depth == 0 && slot >= 0) {
      const int rc = put(d + v0, (uint64_t)(i - v0), JK_NESTED);
      if (rc) return rc;
    }
    s = JX_AFTER;
  }
  while (i < end && json_ws(d[i])) i++;
  if (i < end && d[i] != '\n') return JSON_E_TRAILING;
  return 0;
}

__global__ void __launch_bounds__(256) json_fields_kernel(JsonFieldArgs A) {
  extern __shared__ __align__(16) uint8_t smem[];
  JsonKey* keys = (JsonKey*)smem;
  uint8_t* names = smem + (size_t)A.n_keys * sizeof(JsonKey);
  for (int k = threadIdx.x; k < A.n_keys; k += blockDim.x) keys[k] = A.keys[k];
  for (int k = threadIdx.x; k < A.names_bytes; k += blockDim.x) names[k] = A.names[k];
  __syncthreads();
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < A.n_records; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = A.row_base + r;
    uint32_t detail = 0;
    const int rc = json_record(A, keys, names, row, (int64_t)A.rec_start[r], &detail);
    if (rc) csv_error(A.err, row, rc, detail);
  }
}

static size_t json_fields_smem(const JsonFieldArgs& A) { return (size_t)A.n_keys * sizeof(JsonKey) + (size_t)A.names_bytes; }

void launch_json_fields(const JsonFieldArgs& A, cudaStream_t st) {
  if (A.n_records <= 0) return;
  int64_t g = (A.n_records + 255) / 256;
  if (g > 65535) g = 65535;
  launch_kernel(json_fields_kernel, dim3((unsigned)g), dim3(256), json_fields_smem(A), st, A);
}

// ---- conversion: text_convert.cuh ------------------------------------------------------------------------------------------
template <int FAM>
__global__ void json_convert_kernel(CsvConvertArgs A) { text_convert<FAM, true>(A); }

void launch_json_convert(const CsvConvertArgs& A, int family, cudaStream_t st) {
  if (A.n <= 0) return;
  int64_t g = (A.n + 255) / 256;
  if (g > 65535) g = 65535;
  const dim3 grid((unsigned)g), block(256);
  switch (family) {
    case CSV_FAM_INT: launch_kernel(json_convert_kernel<CSV_FAM_INT>, grid, block, 0, st, A); break;
    case CSV_FAM_DEC: launch_kernel(json_convert_kernel<CSV_FAM_DEC>, grid, block, 0, st, A); break;
    case CSV_FAM_F64: launch_kernel(json_convert_kernel<CSV_FAM_F64>, grid, block, 0, st, A); break;
    case CSV_FAM_F32: launch_kernel(json_convert_kernel<CSV_FAM_F32>, grid, block, 0, st, A); break;
    case CSV_FAM_DATE: launch_kernel(json_convert_kernel<CSV_FAM_DATE>, grid, block, 0, st, A); break;
    case CSV_FAM_BOOL: launch_kernel(json_convert_kernel<CSV_FAM_BOOL>, grid, block, 0, st, A); break;
    default: launch_kernel(json_convert_kernel<CSV_FAM_UTF8>, grid, block, 0, st, A); break;
  }
}

}  // namespace b200
