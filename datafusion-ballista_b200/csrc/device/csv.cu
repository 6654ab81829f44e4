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
#include "text_convert.cuh"

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

// ---- conversion: text_convert.cuh --------------------------------------------------------------------------------------
template <int FAM>
__global__ void csv_convert_kernel(CsvConvertArgs A) { text_convert<FAM, false>(A); }

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
