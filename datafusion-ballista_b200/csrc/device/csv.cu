// CSV / TPC-H .tbl scan on the GPU (sm_90a): record boundaries under quoting, field splitting and per-type conversion
// into the engine's HBM column layout (Arrow fixed-width values, one validity byte per row, 16-byte string views).
//
// Reference path: DataSourceExec + CsvSource (CsvScanExecNode, ballista/core/proto/datafusion.proto:1088-1101) -> arrow-csv
// [EXT] on CPU threads.  Here the host only copies the file bytes to HBM; every pass below runs on the device:
//   1. csv_tiles_kernel: one thread per CSV_TILE bytes computes, for each of the CSV_STATES entry states of the quote state
//      machine, the exit state and the number of record starts in its tile (a tile without quote / escape bytes takes a
//      one-state fast path); each block composes its tiles' transitions into one.
//   2. csv_block_scan_kernel: one block composes the block transitions in file order from the start state and gives every
//      block its entry state and first record index (and the record count).
//   3. csv_record_starts_kernel: every tile is re-scanned from its now known entry state and writes its record starts.
//   4. csv_fields_kernel: one thread per record splits it into fields outside quotes, checks the field count and keeps a
//      {pointer, length} view of every materialised field (fields with escaped / doubled quotes are unquoted into a side
//      buffer at the same offset first).
//   5. csv_convert_kernel<family>: one thread per row and column parses the field: integers, Decimal128 (exact 128-bit),
//      Float32 / Float64 (correctly rounded: Clinger's exact fast path, else an exact big-integer comparison with the
//      halfway points), Date32, Bool, Utf8 (UTF-8 validated; the views are compacted into Arrow Utf8 afterwards).
// Errors never stop a kernel: each column (and the field pass) keeps one 64-bit word, atomicMin of
// (row << 24 | reason << 16 | detail), so the host reports the first failing record after one read-back.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace b200 {

// ---- quote state machine ---------------------------------------------------------------------------------------------
// states: CS_R record start pending (after a terminator, or at the start), CS_F field start (after a delimiter),
// CS_U inside an unquoted field, CS_Q inside a quoted field, CS_QQ a quote seen inside a quoted field (closing, or the
// first of a doubled quote), CS_E after the escape byte inside a quoted field.
enum CsvState : int { CS_R = 0, CS_F, CS_U, CS_Q, CS_QQ, CS_E };
// byte classes
enum CsvClass : int { CC_OTHER = 0, CC_TERM, CC_DELIM, CC_QUOTE, CC_ESC };

__device__ __forceinline__ int csv_class(uint8_t b, const CsvDialect& d) {
  if (b == '\n' || b == '\r') return CC_TERM;
  if (b == d.delim) return CC_DELIM;
  if (b == d.quote) return CC_QUOTE;
  if (d.has_escape && b == d.escape) return CC_ESC;
  return CC_OTHER;
}

__host__ __device__ __forceinline__ int csv_next(int s, int c) {
  switch (s) {
    case CS_R:
    case CS_F: return c == CC_TERM ? CS_R : c == CC_DELIM ? CS_F : c == CC_QUOTE ? CS_Q : CS_U;
    case CS_U: return c == CC_TERM ? CS_R : c == CC_DELIM ? CS_F : CS_U;
    case CS_Q: return c == CC_ESC ? CS_E : c == CC_QUOTE ? CS_QQ : CS_Q;
    case CS_QQ: return c == CC_QUOTE ? CS_Q : c == CC_TERM ? CS_R : c == CC_DELIM ? CS_F : CS_U;
    default: return CS_Q;  // CS_E: the escaped byte is taken literally
  }
}

// transition table packed per byte class: 4 bits per state (next state in bits 0-2, "a record starts here" in bit 3)
struct CsvTable {
  uint32_t t[5];
};
__device__ __forceinline__ CsvTable csv_table() {
  CsvTable T;
#pragma unroll
  for (int c = 0; c < 5; c++) {
    uint32_t w = 0;
#pragma unroll
    for (int s = 0; s < CSV_STATES; s++) {
      uint32_t v = (uint32_t)csv_next(s, c);
      if (s == CS_R && c != CC_TERM) v |= 8;
      w |= v << (4 * s);
    }
    T.t[c] = w;
  }
  return T;
}

__device__ __forceinline__ CsvTrans csv_compose(const CsvTrans& a, const CsvTrans& b) {
  CsvTrans r;
#pragma unroll
  for (int s = 0; s < CSV_STATES; s++) {
    const int m = a.exit[s];
    r.exit[s] = b.exit[m];
    r.cnt[s] = a.cnt[s] + b.cnt[m];
  }
  return r;
}

// the transition of bytes [lo, hi) of the span
__device__ CsvTrans csv_tile_trans(const uint8_t* data, int64_t lo, int64_t hi, const CsvDialect& d, const CsvTable& T, bool& special) {
  special = false;
  for (int64_t i = lo; i < hi; i++) {
    const uint8_t b = data[i];
    if (b == d.quote || (d.has_escape && b == d.escape)) {
      special = true;
      break;
    }
  }
  CsvTrans r;
  if (!special) {
    // no quote can open in this tile: every entry state outside quotes behaves alike, quoted entries stay quoted
    uint32_t inner = 0;
    bool prev_term = false;
    int last = CC_OTHER;
    for (int64_t i = lo; i < hi; i++) {
      const int c = csv_class(data[i], d);
      if (i > lo && prev_term && c != CC_TERM) inner++;
      prev_term = c == CC_TERM;
      last = c;
    }
    const int out = hi == lo ? -1 : last == CC_TERM ? CS_R : last == CC_DELIM ? CS_F : CS_U;
    const bool first_starts = hi > lo && csv_class(data[lo], d) != CC_TERM;
#pragma unroll
    for (int s = 0; s < CSV_STATES; s++) {
      if (s == CS_Q || s == CS_E) {
        r.exit[s] = (hi == lo && s == CS_E) ? CS_E : CS_Q;
        r.cnt[s] = 0;
      } else {
        r.exit[s] = out < 0 ? s : out;
        r.cnt[s] = inner + ((s == CS_R && first_starts) ? 1u : 0u);
      }
    }
    return r;
  }
  int st[CSV_STATES];
  uint32_t cn[CSV_STATES];
#pragma unroll
  for (int s = 0; s < CSV_STATES; s++) {
    st[s] = s;
    cn[s] = 0;
  }
  for (int64_t i = lo; i < hi; i++) {
    const uint32_t w = T.t[csv_class(data[i], d)];
#pragma unroll
    for (int s = 0; s < CSV_STATES; s++) {
      const uint32_t v = (w >> (4 * st[s])) & 15u;
      cn[s] += v >> 3;
      st[s] = (int)(v & 7u);
    }
  }
#pragma unroll
  for (int s = 0; s < CSV_STATES; s++) {
    r.exit[s] = (uint8_t)st[s];
    r.cnt[s] = cn[s];
  }
  return r;
}

__global__ void __launch_bounds__(CSV_BLOCK) csv_tiles_kernel(const uint8_t* data, int64_t bytes, CsvDialect d, CsvTrans* tiles, CsvTrans* blocks,
                                                              unsigned int* has_quote) {
  __shared__ CsvTrans sh[CSV_BLOCK];
  const CsvTable T = csv_table();
  const int64_t t = (int64_t)blockIdx.x * CSV_BLOCK + threadIdx.x;
  const int64_t lo = t * CSV_TILE, hi = lo + CSV_TILE < bytes ? lo + CSV_TILE : bytes;
  CsvTrans r;
  if (lo < bytes) {
    bool special;
    r = csv_tile_trans(data, lo, hi, d, T, special);
    tiles[t] = r;
    // any quote / escape byte at all: the host then provides the unquoting side buffer
    if (special) atomicOr(has_quote, 1u);
  } else {
#pragma unroll
    for (int s = 0; s < CSV_STATES; s++) {
      r.exit[s] = (uint8_t)s;
      r.cnt[s] = 0;
    }
  }
  sh[threadIdx.x] = r;
  __syncthreads();
  for (int w = 1; w < CSV_BLOCK; w <<= 1) {
    if ((threadIdx.x & (2 * w - 1)) == 0) sh[threadIdx.x] = csv_compose(sh[threadIdx.x], sh[threadIdx.x + w]);
    __syncthreads();
  }
  if (threadIdx.x == 0) blocks[blockIdx.x] = sh[0];
}

__global__ void __launch_bounds__(1024) csv_block_scan_kernel(const CsvTrans* blocks, int64_t n_blocks, uint8_t* blk_state, unsigned long long* blk_base,
                                                              unsigned long long* n_records) {
  __shared__ CsvTrans chunk[1024];
  __shared__ uint8_t entry[1024];
  __shared__ unsigned long long base[1024];
  const int64_t per = (n_blocks + 1023) / 1024;
  const int64_t b0 = threadIdx.x * per, b1 = b0 + per < n_blocks ? b0 + per : n_blocks;
  CsvTrans f;
#pragma unroll
  for (int s = 0; s < CSV_STATES; s++) {
    f.exit[s] = (uint8_t)s;
    f.cnt[s] = 0;
  }
  for (int64_t b = b0; b < b1; b++) f = csv_compose(f, blocks[b]);
  chunk[threadIdx.x] = f;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = CS_R;
    unsigned long long n = 0;
    for (int k = 0; k < 1024; k++) {
      entry[k] = (uint8_t)s;
      base[k] = n;
      n += chunk[k].cnt[s];
      s = chunk[k].exit[s];
    }
    *n_records = n;
  }
  __syncthreads();
  int s = entry[threadIdx.x];
  unsigned long long n = base[threadIdx.x];
  for (int64_t b = b0; b < b1; b++) {
    blk_state[b] = (uint8_t)s;
    blk_base[b] = n;
    n += blocks[b].cnt[s];
    s = blocks[b].exit[s];
  }
}

__global__ void __launch_bounds__(CSV_BLOCK) csv_record_starts_kernel(const uint8_t* data, int64_t bytes, CsvDialect d, const CsvTrans* tiles,
                                                                      const uint8_t* blk_state, const unsigned long long* blk_base, uint64_t* rec_start) {
  __shared__ uint8_t entry[CSV_BLOCK];
  __shared__ unsigned long long base[CSV_BLOCK];
  const int64_t t0 = (int64_t)blockIdx.x * CSV_BLOCK;
  const int64_t n_tiles = (bytes + CSV_TILE - 1) / CSV_TILE;
  if (threadIdx.x == 0) {
    int s = blk_state[blockIdx.x];
    unsigned long long n = blk_base[blockIdx.x];
    for (int k = 0; k < CSV_BLOCK && t0 + k < n_tiles; k++) {
      entry[k] = (uint8_t)s;
      base[k] = n;
      const CsvTrans& r = tiles[t0 + k];
      n += r.cnt[s];
      s = r.exit[s];
    }
  }
  __syncthreads();
  const int64_t t = t0 + threadIdx.x;
  if (t >= n_tiles) return;
  const int64_t lo = t * CSV_TILE, hi = lo + CSV_TILE < bytes ? lo + CSV_TILE : bytes;
  int s = entry[threadIdx.x];
  unsigned long long n = base[threadIdx.x];
  if (tiles[t].cnt[s] == 0) return;
  for (int64_t i = lo; i < hi; i++) {
    const int c = csv_class(data[i], d);
    if (s == CS_R && c != CC_TERM) rec_start[n++] = (uint64_t)i;
    s = csv_next(s, c);
  }
}

int64_t csv_tile_count(int64_t bytes) { return (bytes + CSV_TILE - 1) / CSV_TILE; }
int64_t csv_block_count(int64_t bytes) { return (csv_tile_count(bytes) + CSV_BLOCK - 1) / CSV_BLOCK; }

void launch_csv_records_count(const uint8_t* data, int64_t bytes, const CsvDialect& d, CsvTrans* tiles, CsvTrans* blocks, uint8_t* blk_state,
                              unsigned long long* blk_base, unsigned int* has_quote, unsigned long long* n_records, cudaStream_t st) {
  const int64_t nb = csv_block_count(bytes);
  launch_kernel(csv_tiles_kernel, dim3((unsigned)nb), dim3(CSV_BLOCK), 0, st, data, bytes, d, tiles, blocks, has_quote);
  launch_kernel(csv_block_scan_kernel, dim3(1), dim3(1024), 0, st, (const CsvTrans*)blocks, nb, blk_state, blk_base, n_records);
}

void launch_csv_record_starts(const uint8_t* data, int64_t bytes, const CsvDialect& d, const CsvTrans* tiles, const uint8_t* blk_state,
                              const unsigned long long* blk_base, uint64_t* rec_start, cudaStream_t st) {
  const int64_t nb = csv_block_count(bytes);
  launch_kernel(csv_record_starts_kernel, dim3((unsigned)nb), dim3(CSV_BLOCK), 0, st, data, bytes, d, tiles, blk_state, blk_base, rec_start);
}

// ---- fields --------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void csv_error(unsigned long long* err, int64_t row, int reason, uint32_t detail) {
  const unsigned long long w = ((unsigned long long)row << 24) | ((unsigned long long)reason << 16) | (detail & 0xFFFFu);
  if (w < *(volatile unsigned long long*)err) atomicMin(err, w);
}

// unquotes the quoted field whose opening quote is at data[q0] and which ends before data[end] into out; returns its length
__device__ uint32_t csv_unquote(const uint8_t* data, int64_t q0, int64_t end, const CsvDialect& d, uint8_t* out) {
  uint32_t n = 0;
  int s = CS_Q;
  for (int64_t i = q0 + 1; i < end; i++) {
    const uint8_t b = data[i];
    const int c = csv_class(b, d);
    if (s == CS_Q) {
      if (c == CC_ESC) s = CS_E;
      else if (c == CC_QUOTE) s = CS_QQ;
      else out[n++] = b;
    } else if (s == CS_E) {
      out[n++] = b;
      s = CS_Q;
    } else if (s == CS_QQ) {
      out[n++] = b;  // a doubled quote, or bytes after the closing quote (kept, as arrow-csv keeps them)
      s = c == CC_QUOTE ? CS_Q : CS_U;
    } else {
      out[n++] = b;
    }
  }
  return n;
}

__global__ void csv_fields_kernel(CsvFieldArgs A) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x + A.skip; r < A.n_records; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = A.row_base + (r - A.skip);
    const int64_t lo = (int64_t)A.rec_start[r];
    const int64_t hi = r + 1 < A.n_records ? (int64_t)A.rec_start[r + 1] : A.bytes;
    int field = 0;
    int64_t f0 = lo;          // first byte of the current field
    bool quoted = false, complex = false;
    int s = CS_F;
    int64_t i = lo;
    for (;; i++) {
      const int c = i < hi ? csv_class(A.data[i], A.d) : CC_TERM;
      const bool in_quotes = s == CS_Q || s == CS_E;
      if (!in_quotes && (c == CC_DELIM || c == CC_TERM)) {
        // field [f0, i) ends
        if (field < A.n_fields) {
          const int slot = A.slot_of_field[field];
          if (slot >= 0) {
            unsigned long long* v = A.views + ((size_t)slot * (size_t)A.n_total + (size_t)row) * 2;
            const uint8_t* p;
            uint32_t len;
            if (!quoted) {
              p = A.data + f0;
              len = (uint32_t)(i - f0);
            } else if (!complex && s == CS_QQ) {
              p = A.data + f0 + 1;
              len = (uint32_t)(i - f0 - 2);
            } else {
              len = csv_unquote(A.data, f0, i, A.d, A.side + f0);
              p = A.side + f0;
            }
            v[0] = (unsigned long long)p;
            v[1] = len;
          }
        }
        field++;
        if (c == CC_TERM) break;
        f0 = i + 1;
        quoted = complex = false;
        s = CS_F;
        continue;
      }
      if (i >= hi) break;  // unterminated quoted field at the end of the span: ends with it
      const int n = csv_next(s, c);
      if (s == CS_F && n == CS_Q) quoted = true;
      if (s == CS_Q && n == CS_E) complex = true;
      if (s == CS_QQ && n != CS_R && n != CS_F) complex = true;  // doubled quote, or bytes after the closing quote
      s = n;
    }
    if (i >= hi && (s == CS_Q || s == CS_E)) {
      // the span ended inside quotes: the last field still counts
      if (field < A.n_fields) {
        const int slot = A.slot_of_field[field];
        if (slot >= 0) {
          unsigned long long* v = A.views + ((size_t)slot * (size_t)A.n_total + (size_t)row) * 2;
          const uint32_t len = csv_unquote(A.data, f0, hi, A.d, A.side + f0);
          v[0] = (unsigned long long)(A.side + f0);
          v[1] = len;
        }
      }
      field++;
    }
    if (field != A.n_fields) {
      csv_error(A.err, row, CSV_E_FIELDS, (uint32_t)(field < 0xFFFF ? field : 0xFFFF));
      // keep the row's views defined for the conversion kernels
      for (int k = field; k < A.n_fields; k++) {
        const int slot = A.slot_of_field[k];
        if (slot >= 0) {
          unsigned long long* v = A.views + ((size_t)slot * (size_t)A.n_total + (size_t)row) * 2;
          v[0] = (unsigned long long)A.data;
          v[1] = 0;
        }
      }
    }
  }
}

void launch_csv_fields(const CsvFieldArgs& A, cudaStream_t st) {
  const int64_t n = A.n_records - A.skip;
  if (n <= 0) return;
  int64_t g = (n + 255) / 256;
  if (g > 65535) g = 65535;
  launch_kernel(csv_fields_kernel, dim3((unsigned)g), dim3(256), 0, st, A);
}

// ---- conversion --------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool csv_digit(uint8_t b) { return b >= '0' && b <= '9'; }
__device__ __forceinline__ uint8_t csv_lower(uint8_t b) { return (b >= 'A' && b <= 'Z') ? (uint8_t)(b + 32) : b; }
__device__ __forceinline__ bool csv_ieq(const uint8_t* p, uint32_t n, const char* lit) {
  uint32_t k = 0;
  for (; lit[k]; k++)
    if (k >= n || csv_lower(p[k]) != (uint8_t)lit[k]) return false;
  return k == n;
}

// integers: [+-]?digits, '-' only for signed types; range [lo, hi] as i128
__device__ int csv_parse_int(const uint8_t* p, uint32_t n, bool is_signed, __int128 lo, __int128 hi, __int128* out) {
  uint32_t k = 0;
  bool neg = false;
  if (k < n && (p[k] == '+' || (is_signed && p[k] == '-'))) neg = p[k++] == '-';
  if (k >= n) return CSV_E_INT;
  unsigned __int128 v = 0;
  for (; k < n; k++) {
    if (!csv_digit(p[k])) return CSV_E_INT;
    v = v * 10 + (p[k] - '0');
    if (v > ((unsigned __int128)1 << 65)) return CSV_E_INT_RANGE;
  }
  const __int128 s = neg ? -(__int128)v : (__int128)v;
  if (s < lo || s > hi) return CSV_E_INT_RANGE;
  *out = s;
  return 0;
}

__device__ int csv_parse_decimal(const uint8_t* p, uint32_t n, int precision, int scale, __int128* out) {
  uint32_t k = 0;
  bool neg = false;
  if (k < n && (p[k] == '+' || p[k] == '-')) neg = p[k++] == '-';
  unsigned __int128 v = 0;
  int int_digits = 0, frac_digits = 0, sig = 0;
  for (; k < n && csv_digit(p[k]); k++) {
    int_digits++;
    if (sig || p[k] != '0') sig++;
    if (sig > 38) return CSV_E_DEC_RANGE;
    v = v * 10 + (p[k] - '0');
  }
  if (k < n && p[k] == '.') {
    k++;
    for (; k < n && csv_digit(p[k]); k++) {
      frac_digits++;
      if (frac_digits > scale) return CSV_E_DEC_SCALE;
      if (sig || p[k] != '0') sig++;
      if (sig > 38) return CSV_E_DEC_RANGE;
      v = v * 10 + (p[k] - '0');
    }
    if (frac_digits == 0) return CSV_E_DEC;
  }
  if (k < n && (p[k] == 'e' || p[k] == 'E')) return CSV_E_DEC_EXP;
  if (k != n || int_digits + frac_digits == 0) return CSV_E_DEC;
  // the value has sig + (scale - frac_digits) digits once scaled: it fits the precision when that is at most p
  if (v != 0 && sig + (scale - frac_digits) > precision) return CSV_E_DEC_RANGE;
  for (int f = frac_digits; f < scale; f++) v *= 10;
  *out = neg ? -(__int128)v : (__int128)v;
  return 0;
}

// exact Date32: YYYY-MM-DD, proleptic Gregorian, days since 1970-01-01
__device__ int csv_parse_date(const uint8_t* p, uint32_t n, int32_t* out) {
  if (n != 10 || p[4] != '-' || p[7] != '-') return CSV_E_DATE;
  int v[3] = {0, 0, 0};
  const int at[3] = {0, 5, 8}, len[3] = {4, 2, 2};
  for (int f = 0; f < 3; f++)
    for (int k = 0; k < len[f]; k++) {
      const uint8_t b = p[at[f] + k];
      if (!csv_digit(b)) return CSV_E_DATE;
      v[f] = v[f] * 10 + (b - '0');
    }
  const int y = v[0], m = v[1], dd = v[2];
  if (m < 1 || m > 12 || dd < 1) return CSV_E_DATE;
  const bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
  const int mdays[12] = {31, leap ? 29 : 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
  if (dd > mdays[m - 1]) return CSV_E_DATE;
  const int yy = y - (m <= 2);
  const int era = (yy >= 0 ? yy : yy - 399) / 400;
  const int yoe = yy - era * 400;
  const int doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + dd - 1;
  const int doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  *out = era * 146097 + doe - 719468;
  return 0;
}

__device__ bool csv_valid_utf8(const uint8_t* p, uint32_t n) {
  uint32_t k = 0;
  while (k < n) {
    const uint8_t b = p[k];
    if (b < 0x80) {
      k++;
      continue;
    }
    int len;
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
      return false;
    }
    if (k + len > n) return false;
    for (int j = 1; j < len; j++) {
      const uint8_t c = p[k + j];
      if ((c & 0xC0) != 0x80) return false;
      cp = (cp << 6) | (c & 0x3F);
    }
    if ((len == 3 && (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF))) || (len == 4 && (cp < 0x10000 || cp > 0x10FFFF))) return false;
    k += len;
  }
  return true;
}

// ---- floats: exact decimal -> binary ------------------------------------------------------------------------------------
// Big unsigned integers for the exact comparison; CSV_BIG_WORDS x 32 bits holds 5^1100 times a 55-bit mantissa.
static const int CSV_BIG_WORDS = 88;
static const int CSV_MAX_DIGITS = 800;  // significant digits kept; any further non-zero digit is a sticky bit
struct CsvBig {
  uint32_t w[CSV_BIG_WORDS];
  int n;
};
__device__ __forceinline__ void big_set(CsvBig& a, uint64_t v) {
  a.w[0] = (uint32_t)v;
  a.w[1] = (uint32_t)(v >> 32);
  a.n = a.w[1] ? 2 : a.w[0] ? 1 : 0;
}
__device__ void big_muladd(CsvBig& a, uint32_t m, uint32_t add) {
  uint64_t carry = add;
  for (int i = 0; i < a.n; i++) {
    const uint64_t t = (uint64_t)a.w[i] * m + carry;
    a.w[i] = (uint32_t)t;
    carry = t >> 32;
  }
  if (carry && a.n < CSV_BIG_WORDS) a.w[a.n++] = (uint32_t)carry;
}
__device__ void big_mul_pow5(CsvBig& a, int e) {
  while (e >= 13) {
    big_muladd(a, 1220703125u, 0);  // 5^13
    e -= 13;
  }
  uint32_t m = 1;
  for (int k = 0; k < e; k++) m *= 5;
  if (m > 1) big_muladd(a, m, 0);
}
// r = a * v (v < 2^64)
__device__ void big_mul_u64(const CsvBig& a, uint64_t v, CsvBig& r) {
  const uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
  for (int i = 0; i < CSV_BIG_WORDS; i++) r.w[i] = 0;
  r.n = 0;
  for (int pass = 0; pass < 2; pass++) {
    const uint32_t m = pass ? hi : lo;
    if (!m) continue;
    uint64_t carry = 0;
    int i = 0;
    for (; i < a.n; i++) {
      const int j = i + pass;
      if (j >= CSV_BIG_WORDS) break;
      const uint64_t t = (uint64_t)a.w[i] * m + r.w[j] + carry;
      r.w[j] = (uint32_t)t;
      carry = t >> 32;
    }
    for (int j = i + pass; carry && j < CSV_BIG_WORDS; j++) {
      const uint64_t t = (uint64_t)r.w[j] + carry;
      r.w[j] = (uint32_t)t;
      carry = t >> 32;
    }
  }
  r.n = CSV_BIG_WORDS;
  while (r.n > 0 && r.w[r.n - 1] == 0) r.n--;
}
// word i of (a << s)
__device__ __forceinline__ uint32_t big_word_shl(const CsvBig& a, int s, int i) {
  const int ws = s >> 5, bs = s & 31;
  const int j = i - ws;
  const uint32_t hi = (j >= 0 && j < a.n) ? a.w[j] : 0u;
  if (!bs) return hi;
  const uint32_t lo = (j - 1 >= 0 && j - 1 < a.n) ? a.w[j - 1] : 0u;
  return (hi << bs) | (lo >> (32 - bs));
}
// sign of (a << sa) - (b << sb)
__device__ int big_cmp_shl(const CsvBig& a, int sa, const CsvBig& b, int sb) {
  const int na = a.n + (sa >> 5) + 1, nb = b.n + (sb >> 5) + 1;
  for (int i = (na > nb ? na : nb) - 1; i >= 0; i--) {
    const uint32_t x = big_word_shl(a, sa, i), y = big_word_shl(b, sb, i);
    if (x != y) return x < y ? -1 : 1;
  }
  return 0;
}

struct CsvDec {
  bool neg, special_inf, special_nan, sticky;
  int nd;        // significant digits kept
  int e10;       // value = D * 10^e10, D = the kept digits as an integer
  uint64_t w;    // the first (up to) 19 kept digits
  int nw;        // how many digits w holds
};

__device__ int csv_scan_float(const uint8_t* p, uint32_t n, CsvDec& o) {
  o.neg = o.special_inf = o.special_nan = o.sticky = false;
  o.nd = o.e10 = o.nw = 0;
  o.w = 0;
  uint32_t k = 0;
  if (k < n && (p[k] == '+' || p[k] == '-')) o.neg = p[k++] == '-';
  if (k < n && !csv_digit(p[k]) && p[k] != '.') {
    if (csv_ieq(p + k, n - k, "inf") || csv_ieq(p + k, n - k, "infinity")) {
      o.special_inf = true;
      return 0;
    }
    if (csv_ieq(p + k, n - k, "nan")) {
      o.special_nan = true;
      return 0;
    }
    return CSV_E_FLOAT;
  }
  int digits = 0;
  bool frac = false;
  for (; k < n; k++) {
    const uint8_t b = p[k];
    if (b == '.') {
      if (frac) return CSV_E_FLOAT;
      frac = true;
      continue;
    }
    if (!csv_digit(b)) break;
    digits++;
    const int dv = b - '0';
    if (o.nd == 0 && dv == 0) {
      if (frac) o.e10--;
      continue;
    }
    if (o.nd < CSV_MAX_DIGITS) {
      o.nd++;
      if (frac) o.e10--;
      if (o.nw < 19) {
        o.w = o.w * 10 + (uint64_t)dv;
        o.nw++;
      }
    } else {
      if (dv) o.sticky = true;
      if (!frac) o.e10++;
    }
  }
  if (digits == 0) return CSV_E_FLOAT;
  if (k < n && (p[k] == 'e' || p[k] == 'E')) {
    k++;
    bool eneg = false;
    if (k < n && (p[k] == '+' || p[k] == '-')) eneg = p[k++] == '-';
    if (k >= n) return CSV_E_FLOAT;
    int ev = 0;
    for (; k < n; k++) {
      if (!csv_digit(p[k])) return CSV_E_FLOAT;
      if (ev < 100000) ev = ev * 10 + (p[k] - '0');
    }
    o.e10 += eneg ? -ev : ev;
  }
  if (k != n) return CSV_E_FLOAT;
  return 0;
}

// the kept significant digits of the field as a big integer
__device__ void csv_digits_big(const uint8_t* p, uint32_t n, int nd, CsvBig& D) {
  big_set(D, 0);
  int got = 0;
  uint32_t chunk = 0, mul = 1;
  for (uint32_t k = 0; k < n && got < nd; k++) {
    const uint8_t b = p[k];
    if (b == 'e' || b == 'E') break;
    if (!csv_digit(b)) continue;
    if (got == 0 && b == '0') continue;
    chunk = chunk * 10 + (b - '0');
    mul *= 10;
    got++;
    if (mul == 1000000000u) {
      big_muladd(D, mul, chunk);
      chunk = 0;
      mul = 1;
    }
  }
  if (mul > 1) big_muladd(D, mul, chunk);
}

// correctly rounded (nearest, ties to even) value of the decimal with P mantissa bits (53 / 24); returns the IEEE bits
// of the magnitude
template <int P>
__device__ uint64_t csv_exact_float(const uint8_t* p, uint32_t n, const CsvDec& dd) {
  const int kmin = P == 53 ? -1074 : -149;
  const int kmax = P == 53 ? 971 : 104;
  const uint64_t top = 1ull << (P - 1);
  const uint64_t inf_bits = P == 53 ? 0x7FF0000000000000ull : 0x7F800000ull;
  const int mag = dd.nd + dd.e10;
  if (mag > (P == 53 ? 310 : 40)) return inf_bits;
  if (mag < (P == 53 ? -324 : -46)) return 0;
  // starting point: w * 10^(e10 + nd - nw) with a double kept normalised by frexp (a few ulps off at most)
  int K = 0;
  double a = frexp((double)dd.w, &K);
  int e = dd.e10 + dd.nd - dd.nw;
  while (e != 0) {
    const int step = e > 0 ? (e > 22 ? 22 : e) : (e < -22 ? -22 : e);
    double pw = 1.0;
    for (int q = 0; q < (step > 0 ? step : -step); q++) pw *= 10.0;
    a = step > 0 ? a * pw : a / pw;
    int ex = 0;
    a = frexp(a, &ex);
    K += ex;
    e -= step;
  }
  // a in [0.5, 1): value ~ a * 2^K = m * 2^k with m in [2^(P-1), 2^P)
  uint64_t m = (uint64_t)ldexp(a, P);
  int k = K - P;
  if (m >= (1ull << P)) {
    m >>= 1;
    k++;
  }
  if (k < kmin) {
    const int sh = kmin - k;
    m = sh >= 64 ? 0 : m >> sh;
    k = kmin;
  }
  if (k > kmax) {
    m = top;
    k = kmax + 1;
  }
  CsvBig L, P5, R;
  csv_digits_big(p, n, dd.nd, L);
  int lexp = 0;
  if (dd.e10 >= 0) {
    big_mul_pow5(L, dd.e10);
    lexp = dd.e10;
  } else {
    lexp = dd.e10;
    big_set(P5, 1);
    big_mul_pow5(P5, -dd.e10);
  }
  // sign of value - H * 2^h
  auto cmp = [&](uint64_t H, int h) -> int {
    int c;
    if (dd.e10 >= 0) {
      big_set(R, H);
      const int d = lexp - h;
      c = d >= 0 ? big_cmp_shl(L, d, R, 0) : big_cmp_shl(L, 0, R, -d);
    } else {
      big_mul_u64(P5, H, R);
      const int d = lexp - h;
      c = d >= 0 ? big_cmp_shl(L, d, R, 0) : big_cmp_shl(L, 0, R, -d);
    }
    if (c == 0 && dd.sticky) c = 1;
    return c;
  };
  for (int it = 0; it < 4096; it++) {
    const bool is_inf = k > kmax;
    if (!is_inf) {
      const int c = cmp(2 * m + 1, k - 1);
      if (c > 0 || (c == 0 && (m & 1))) {
        m++;
        if (m == (1ull << P)) {
          m = top;
          k++;
        }
        continue;
      }
    }
    if (m > 0) {
      const bool edge = m == top && k > kmin;
      const int c = edge ? cmp(4 * m - 1, k - 2) : cmp(2 * m - 1, k - 1);
      if (c < 0 || (c == 0 && (m & 1))) {
        if (edge) {
          m = (1ull << P) - 1;
          k--;
        } else {
          m--;
        }
        continue;
      }
    }
    break;
  }
  if (k > kmax) return inf_bits;
  if (m < top) return m;  // subnormal (k == kmin) or zero
  return ((uint64_t)(k - kmin + 1) << (P - 1)) | (m - top);
}

template <int P>
__device__ int csv_parse_float(const uint8_t* p, uint32_t n, uint64_t* bits) {
  CsvDec dd;
  const int rc = csv_scan_float(p, n, dd);
  if (rc) return rc;
  const uint64_t sign = dd.neg ? (P == 53 ? 0x8000000000000000ull : 0x80000000ull) : 0;
  if (dd.special_nan) {
    *bits = P == 53 ? 0x7FF8000000000000ull : 0x7FC00000ull;
    return 0;
  }
  if (dd.special_inf) {
    *bits = sign | (P == 53 ? 0x7FF0000000000000ull : 0x7F800000ull);
    return 0;
  }
  if (dd.nd == 0) {
    *bits = sign;
    return 0;
  }
  // Clinger: an exact mantissa and an exact power of ten, one correctly rounded IEEE operation
  if (P == 53 && !dd.sticky && dd.nd <= 15 && dd.e10 >= -22 && dd.e10 <= 22) {
    double pw = 1.0;
    for (int q = 0; q < (dd.e10 >= 0 ? dd.e10 : -dd.e10); q++) pw *= 10.0;
    const double v = dd.e10 >= 0 ? (double)dd.w * pw : (double)dd.w / pw;
    *bits = sign | (uint64_t)__double_as_longlong(v);
    return 0;
  }
  if (P == 24 && !dd.sticky && dd.nd <= 7 && dd.e10 >= -10 && dd.e10 <= 10) {
    float pw = 1.0f;
    for (int q = 0; q < (dd.e10 >= 0 ? dd.e10 : -dd.e10); q++) pw *= 10.0f;
    const float v = dd.e10 >= 0 ? __fmul_rn((float)dd.w, pw) : __fdiv_rn((float)dd.w, pw);
    *bits = sign | (uint64_t)__float_as_uint(v);
    return 0;
  }
  *bits = sign | csv_exact_float<P>(p, n, dd);
  return 0;
}

template <int FAM>
__global__ void csv_convert_kernel(CsvConvertArgs A) {
  unsigned long long nulls = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < A.n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t* p = (const uint8_t*)A.views[2 * i];
    const uint32_t len = (uint32_t)A.views[2 * i + 1];
    if (len == 0) {
      // empty or "" : NULL for every type
      A.valid[i] = 0;
      nulls++;
      if (!A.nullable) csv_error(A.err, i, CSV_E_NULL, 0);
      if (FAM == CSV_FAM_UTF8) {
        unsigned long long* o = (unsigned long long*)A.out + 2 * i;
        o[0] = (unsigned long long)p;
        o[1] = 0;
      } else {
        uint8_t* o = (uint8_t*)A.out + (size_t)i * A.width;
        for (int b = 0; b < A.width; b++) o[b] = 0;
      }
      continue;
    }
    A.valid[i] = 1;
    int rc = 0;
    if (FAM == CSV_FAM_INT) {
      __int128 v = 0;
      rc = csv_parse_int(p, len, A.is_signed, A.lo, A.hi, &v);
      const uint64_t u = (uint64_t)v;
      uint8_t* o = (uint8_t*)A.out + (size_t)i * A.width;
      if (A.width == 1) *o = (uint8_t)u;
      else if (A.width == 2) *(uint16_t*)o = (uint16_t)u;
      else if (A.width == 4) *(uint32_t*)o = (uint32_t)u;
      else *(uint64_t*)o = u;
    } else if (FAM == CSV_FAM_DEC) {
      __int128 v = 0;
      rc = csv_parse_decimal(p, len, A.precision, A.scale, &v);
      ((__int128*)A.out)[i] = v;
    } else if (FAM == CSV_FAM_F64) {
      uint64_t b = 0;
      rc = csv_parse_float<53>(p, len, &b);
      ((uint64_t*)A.out)[i] = b;
    } else if (FAM == CSV_FAM_F32) {
      uint64_t b = 0;
      rc = csv_parse_float<24>(p, len, &b);
      ((uint32_t*)A.out)[i] = (uint32_t)b;
    } else if (FAM == CSV_FAM_DATE) {
      int32_t v = 0;
      rc = csv_parse_date(p, len, &v);
      ((int32_t*)A.out)[i] = v;
    } else if (FAM == CSV_FAM_BOOL) {
      uint8_t v = 0;
      if (csv_ieq(p, len, "true")) v = 1;
      else if (!csv_ieq(p, len, "false")) rc = CSV_E_BOOL;
      ((uint8_t*)A.out)[i] = v;
    } else {
      if (!csv_valid_utf8(p, len)) rc = CSV_E_UTF8;
      unsigned long long* o = (unsigned long long*)A.out + 2 * i;
      o[0] = (unsigned long long)p;
      o[1] = len;
    }
    if (rc) csv_error(A.err, i, rc, 0);
  }
  if (nulls) atomicAdd(A.null_count, nulls);
}

void launch_csv_convert(const CsvConvertArgs& A, int family, cudaStream_t st) {
  if (A.n <= 0) return;
  int64_t g = (A.n + 255) / 256;
  if (g > 65535) g = 65535;
  const dim3 grid((unsigned)g), block(256);
  switch (family) {
    case CSV_FAM_INT: launch_kernel(csv_convert_kernel<CSV_FAM_INT>, grid, block, 0, st, A); break;
    case CSV_FAM_DEC: launch_kernel(csv_convert_kernel<CSV_FAM_DEC>, grid, block, 0, st, A); break;
    case CSV_FAM_F64: launch_kernel(csv_convert_kernel<CSV_FAM_F64>, grid, block, 0, st, A); break;
    case CSV_FAM_F32: launch_kernel(csv_convert_kernel<CSV_FAM_F32>, grid, block, 0, st, A); break;
    case CSV_FAM_DATE: launch_kernel(csv_convert_kernel<CSV_FAM_DATE>, grid, block, 0, st, A); break;
    case CSV_FAM_BOOL: launch_kernel(csv_convert_kernel<CSV_FAM_BOOL>, grid, block, 0, st, A); break;
    default: launch_kernel(csv_convert_kernel<CSV_FAM_UTF8>, grid, block, 0, st, A); break;
  }
}

}  // namespace b200
