// Parquet page decode on the GPU (sm_90a): definition levels, dictionaries, PLAIN, RLE_DICTIONARY, DELTA_BINARY_PACKED,
// DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY and BYTE_STREAM_SPLIT values ->
// the engine's HBM column layout (Arrow fixed-width values, 16-byte string views into the raw page bytes, validity bytes).
//
// Reference path: DataSourceExec + ParquetSource (ballista/core/proto/datafusion.proto:1058-1077) -> parquet 58.1 [EXT]
// column readers on CPU threads: "page decode, dictionary/RLE/PLAIN decode to Arrow" (SURVEY.md R9f), the dominant CPU cost
// of scan-heavy queries.  Here the host only walks page headers (csrc/host/parquet_meta.hpp); every page is decoded by one
// warp, all pages of all requested columns in flight at once:
//   * RLE / bit-packed hybrid runs (definition levels, dictionary indices): lane 0 reads the run header, the 32 lanes
//     expand the run (bit-packed groups: each lane extracts its own values with unaligned bit reads);
//   * PLAIN fixed-width values: coalesced copies (INT32 / INT64 / DOUBLE), FIXED_LEN_BYTE_ARRAY decimals are byte-reversed
//     into little-endian Decimal128; BYTE_ARRAY values become {pointer, length} views INTO the page bytes (no copy: the
//     engine's intermediate string layout is exactly that);
//   * DELTA_* and BYTE_STREAM_SPLIT pages: validated first, then decoded by pq_values_delta_kernel (see that section);
//   * nullable columns: values are stored densely, a second pass spreads them to their rows using the validity bytes.
// Compressed pages (SNAPPY, GZIP, LZ4_RAW) are first rebuilt uncompressed in HBM by one warp per page (end of this file).
// Integer/byte work, HBM bound: algorithmic bytes = encoded page bytes read + decoded column bytes written.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace b200 {

__device__ __forceinline__ uint64_t pq_load_bits(const uint8_t* p, const uint8_t* end, uint64_t bit_off, int bw) {
  const uint8_t* q = p + (bit_off >> 3);
  uint64_t w = 0;
#pragma unroll
  for (int k = 0; k < 6; k++)
    if (q + k < end) w |= (uint64_t)q[k] << (8 * k);
  return (w >> (bit_off & 7)) & ((bw >= 64) ? ~0ull : ((1ull << bw) - 1ull));
}

// Walks an RLE / bit-packed hybrid stream with one warp; calls emit(index, value) for the first `n` values.
template <class Emit>
__device__ __forceinline__ void pq_hybrid_decode(const uint8_t* p, const uint8_t* end, int bw, uint32_t n, int lane, Emit emit) {
  uint32_t out = 0;
  const int vbytes = (bw + 7) >> 3;
  while (out < n && p < end) {
    // run header (ULEB128), read by every lane redundantly: a handful of bytes, all lanes agree
    uint64_t h = 0;
    for (int shift = 0; shift < 35 && p < end; shift += 7) {
      const uint8_t b = *p++;
      h |= (uint64_t)(b & 0x7F) << shift;
      if (!(b & 0x80)) break;
    }
    if (h & 1) {
      const uint64_t groups = h >> 1;
      const uint64_t count = groups * 8;
      const uint32_t take = (uint32_t)((count < (uint64_t)(n - out)) ? count : (uint64_t)(n - out));
      for (uint32_t k = lane; k < take; k += 32) emit(out + k, (uint32_t)pq_load_bits(p, end, (uint64_t)k * bw, bw));
      p += groups * (uint64_t)bw;
      out += take;
    } else {
      const uint32_t run = (uint32_t)(h >> 1);
      uint32_t v = 0;
      for (int k = 0; k < vbytes && p + k < end; k++) v |= (uint32_t)p[k] << (8 * k);
      p += vbytes;
      const uint32_t take = run < (n - out) ? run : (n - out);
      for (uint32_t k = lane; k < take; k += 32) emit(out + k, v);
      out += take;
    }
  }
}

// where the definition levels and the values of a page are (V1 pages of nullable columns carry the levels' length in-band)
__device__ __forceinline__ void pq_sections(const PqPage& pg, uint32_t& def_off, uint32_t& def_len, uint32_t& val_off, uint32_t& val_len) {
  if (pg.v1_levels) {
    uint32_t len = 0;
    for (int k = 0; k < 4; k++) len |= (uint32_t)pg.data[k] << (8 * k);
    if (len > pg.val_len - 4) len = pg.val_len - 4;  // corrupt length: stay inside the page
    def_off = 4;
    def_len = len;
    val_off = 4 + len;
    val_len = pg.val_len - 4 - len;
  } else {
    def_off = pg.def_off;
    def_len = pg.def_len;
    val_off = pg.val_off;
    val_len = pg.val_len;
  }
}

// ---- definition levels -> validity bytes + non-null count per page ---------------------------------------------------------
__global__ void __launch_bounds__(128) pq_levels_kernel(const PqPage* __restrict__ pages, int n_pages, uint8_t* __restrict__ valid, uint32_t* __restrict__ nonnull,
                                                        unsigned long long* __restrict__ total_nonnull) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_pages) return;
  const PqPage pg = pages[warp];
  uint8_t* v = valid + pg.row0;
  uint32_t cnt = 0;
  uint32_t def_off, def_len, val_off, val_len;
  pq_sections(pg, def_off, def_len, val_off, val_len);
  if (def_len == 0) {
    for (uint32_t k = lane; k < pg.n_values; k += 32) v[k] = 1;
    cnt = pg.n_values;
  } else {
    const uint8_t* p = pg.data + def_off;
    uint32_t mine = 0;
    pq_hybrid_decode(p, p + def_len, 1, pg.n_values, lane, [&](uint32_t i, uint32_t lvl) {
      v[i] = (uint8_t)(lvl & 1);
      mine += lvl & 1;
    });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xFFFFFFFFu, mine, o);
    cnt = mine;
  }
  if (lane == 0) {
    nonnull[warp] = cnt;
    atomicAdd(total_nonnull, (unsigned long long)cnt);
  }
}

// dense_base[p] = number of non-null values in earlier pages (single block; n_pages is small)
__global__ void __launch_bounds__(1024) pq_page_scan_kernel(const uint32_t* __restrict__ nonnull, int n_pages, unsigned long long* __restrict__ dense_base) {
  __shared__ unsigned long long carry;
  __shared__ unsigned long long wsum[32];
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n_pages; base += 1024) {
    const int i = base + threadIdx.x;
    const unsigned long long v = i < n_pages ? nonnull[i] : 0;
    unsigned long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long t = __shfl_up_sync(0xFFFFFFFFu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    unsigned long long off = carry;
    for (int w = 0; w < warp; w++) off += wsum[w];
    if (i < n_pages) dense_base[i] = off + inc - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry = off + inc;
    __syncthreads();
  }
}

// ---- value decode ------------------------------------------------------------------------------------------------------------
// FIXED_LEN_BYTE_ARRAY decimal: big-endian two's complement of L <= 16 bytes (byte(k) = byte k) -> little-endian Decimal128
template <class Byte>
__device__ __forceinline__ ulonglong2 pq_be_dec128(Byte byte, int L) {
  const bool neg = byte(0) & 0x80;
  unsigned long long ulo = neg ? ~0ull : 0ull, uhi = neg ? ~0ull : 0ull;
  for (int k = 0; k < L; k++) {
    uhi = (uhi << 8) | (ulo >> 56);
    ulo = (ulo << 8) | byte(k);
  }
  return make_ulonglong2(ulo, uhi);
}

__device__ __forceinline__ void pq_store_fixed(const PqColumn& C, void* out, uint64_t i, const uint8_t* src) {
  // src: one PLAIN value of the column's physical type
  switch (C.out_kind) {
    case PQ_OUT_I32: {  // page payloads are not aligned: byte-wise loads
      int v;
      memcpy(&v, src, 4);
      ((int32_t*)out)[i] = v;
      break;
    }
    case PQ_OUT_I64: {
      long long v;
      memcpy(&v, src, 8);
      ((long long*)out)[i] = v;
      break;
    }
    case PQ_OUT_F64: {
      double v;
      memcpy(&v, src, 8);
      ((double*)out)[i] = v;
      break;
    }
    case PQ_OUT_DEC128: {
      long long lo, hi;
      if (C.phys == 1) {  // INT32
        int v;
        memcpy(&v, src, 4);
        lo = v;
        hi = lo >> 63;
      } else if (C.phys == 2) {  // INT64
        memcpy(&lo, src, 8);
        hi = lo >> 63;
      } else {  // FIXED_LEN_BYTE_ARRAY: big-endian two's complement of type_length bytes
        const ulonglong2 v = pq_be_dec128([&](int k) { return src[k]; }, C.type_length);
        lo = (long long)v.x;
        hi = (long long)v.y;
      }
      ((ulonglong2*)out)[i] = make_ulonglong2((unsigned long long)lo, (unsigned long long)hi);
      break;
    }
    default: break;
  }
}

__device__ __forceinline__ int pq_plain_width(const PqColumn& C) {
  switch (C.phys) {
    case 1: return 4;
    case 2: return 8;
    case 5: return 8;
    case 7: return C.type_length;
    default: return 0;
  }
}

// Dictionary pages: PLAIN values -> dictionary entries (fixed-width values converted to the output type, byte arrays as views)
__global__ void __launch_bounds__(128) pq_dict_kernel(const PqColumn C, const PqPage* __restrict__ dict_pages, int n_dicts) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_dicts) return;
  const PqPage pg = dict_pages[warp];
  const uint8_t* p = pg.data + pg.val_off;
  const uint8_t* end = p + pg.val_len;
  if (C.phys == 6) {  // BYTE_ARRAY: [u32 length][bytes] ...: a serial walk (lane 0)
    if (lane == 0) {
      unsigned long long* views = (unsigned long long*)C.dict + 2 * (uint64_t)pg.row0;
      for (uint32_t k = 0; k < pg.n_values && p + 4 <= end; k++) {
        uint32_t len;
        memcpy(&len, p, 4);
        views[2 * k] = (unsigned long long)(p + 4);
        views[2 * k + 1] = len;
        p += 4 + len;
      }
    }
    return;
  }
  if (C.phys == 0) return;  // BOOLEAN is never dictionary encoded
  const int w = pq_plain_width(C);
  for (uint32_t k = lane; k < pg.n_values; k += 32) pq_store_fixed(C, C.dict, (uint64_t)pg.row0 + k, p + (uint64_t)k * w);
}

__device__ __forceinline__ void pq_store_from_dict(const PqColumn& C, void* out, uint64_t i, uint64_t d) {
  switch (C.out_kind) {
    case PQ_OUT_I32: ((int32_t*)out)[i] = ((const int32_t*)C.dict)[d]; break;
    case PQ_OUT_I64: ((long long*)out)[i] = ((const long long*)C.dict)[d]; break;
    case PQ_OUT_F64: ((double*)out)[i] = ((const double*)C.dict)[d]; break;
    case PQ_OUT_DEC128:
    case PQ_OUT_STRVIEW: ((ulonglong2*)out)[i] = ((const ulonglong2*)C.dict)[d]; break;
    default: break;
  }
}

// One warp per data page; values land densely at `dense_base[page]` (== the page's first row when the column has no NULLs)
__global__ void __launch_bounds__(128) pq_values_kernel(const PqColumn C, const PqPage* __restrict__ pages, int n_pages, const unsigned long long* __restrict__ dense_base,
                                                        const uint32_t* __restrict__ nonnull, void* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_pages) return;
  const PqPage pg = pages[warp];
  const uint64_t base = dense_base ? dense_base[warp] : (uint64_t)pg.row0;
  const uint32_t n = nonnull ? nonnull[warp] : pg.n_values;
  uint32_t def_off, def_len, val_off, val_len;
  pq_sections(pg, def_off, def_len, val_off, val_len);
  const uint8_t* p = pg.data + val_off;
  const uint8_t* end = p + val_len;
  if (pg.encoding >= PQ_ENC_DBP) return;  // pq_values_delta_kernel's pages
  if (pg.encoding == 1) {  // [PLAIN|RLE]_DICTIONARY: one byte of bit width, then hybrid runs of dictionary indices
    if (p >= end) return;
    const int bw = *p++;
    const uint64_t dbase = (uint64_t)pg.dict_base;
    pq_hybrid_decode(p, end, bw, n, lane, [&](uint32_t i, uint32_t idx) { pq_store_from_dict(C, out, base + i, dbase + idx); });
    return;
  }
  if (pg.encoding == 2) {  // RLE-encoded BOOLEAN values (data page V2 writers): 4-byte length, then hybrid runs of width 1
    if (p + 4 > end) return;
    p += 4;
    pq_hybrid_decode(p, end, 1, n, lane, [&](uint32_t i, uint32_t v) { ((uint8_t*)out)[base + i] = (uint8_t)(v & 1); });
    return;
  }
  if (C.phys == 6) {  // PLAIN BYTE_ARRAY
    if (lane == 0) {
      unsigned long long* views = (unsigned long long*)out + 2 * base;
      for (uint32_t k = 0; k < n && p + 4 <= end; k++) {
        uint32_t len;
        memcpy(&len, p, 4);
        views[2 * k] = (unsigned long long)(p + 4);
        views[2 * k + 1] = len;
        p += 4 + len;
      }
    }
    return;
  }
  if (C.phys == 0) {  // PLAIN BOOLEAN: bit-packed, LSB first
    for (uint32_t k = lane; k < n; k += 32) ((uint8_t*)out)[base + k] = (p[k >> 3] >> (k & 7)) & 1;
    return;
  }
  const int w = pq_plain_width(C);
  for (uint32_t k = lane; k < n; k += 32) pq_store_fixed(C, out, base + k, p + (uint64_t)k * w);
}

// nullable column with NULLs: out[row] = valid[row] ? dense[dense_base + rank of the row among the page's valid rows] : 0
__global__ void __launch_bounds__(128) pq_expand_kernel(const PqPage* __restrict__ pages, int n_pages, const unsigned long long* __restrict__ dense_base,
                                                        const uint8_t* __restrict__ valid, const void* __restrict__ dense, void* __restrict__ out, int width) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_pages) return;
  const PqPage pg = pages[warp];
  uint64_t next = dense_base[warp];
  for (uint32_t k0 = 0; k0 < pg.n_values; k0 += 32) {
    const uint32_t k = k0 + lane;
    const bool v = k < pg.n_values && valid[pg.row0 + k];
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, v);
    if (k < pg.n_values) {
      const uint64_t row = (uint64_t)pg.row0 + k;
      const uint64_t src = next + __popc(m & ((1u << lane) - 1u));
      switch (width) {
        case 1: ((uint8_t*)out)[row] = v ? ((const uint8_t*)dense)[src] : 0; break;
        case 4: ((uint32_t*)out)[row] = v ? ((const uint32_t*)dense)[src] : 0u; break;
        case 8: ((uint64_t*)out)[row] = v ? ((const uint64_t*)dense)[src] : 0ull; break;
        default: ((ulonglong2*)out)[row] = v ? ((const ulonglong2*)dense)[src] : make_ulonglong2(0ull, 0ull); break;
      }
    }
    next += __popc(m);
  }
}

// ---- DELTA_BINARY_PACKED, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY, BYTE_STREAM_SPLIT: one warp per page ----------------------
// Formats (parquet-format Encodings.md):
//   DELTA_BINARY_PACKED: a header of ULEB128 fields <block size in values> <miniblocks per block> <value count> <first value,
//     zigzag>; the block size is a multiple of 128 and the values per miniblock a multiple of 32.  Blocks follow:
//     <min delta, zigzag ULEB128> <one bit-width byte per miniblock> <miniblocks>, a miniblock holding (delta - min delta) of
//     its values bit-packed LSB first, always (values per miniblock * bit width / 8) bytes long.  Miniblocks after the last
//     value keep their width byte (any value) but have no body.  value[i] = value[i-1] + delta[i], wrapping in the physical
//     width (INT32 / INT64): decoded with unsigned 64-bit adds, INT32 truncated.
//   DELTA_LENGTH_BYTE_ARRAY: the lengths as DELTA_BINARY_PACKED, then all the bytes back to back.
//   DELTA_BYTE_ARRAY: the prefix lengths as DELTA_BINARY_PACKED, then the suffixes as DELTA_LENGTH_BYTE_ARRAY; value i is
//     the first prefix[i] bytes of value i-1 followed by suffix i.
//   BYTE_STREAM_SPLIT: byte k of value i at p[k * n + i] for n values of `width` bytes.
// pq_delta_prepare_kernel validates every such page before any value is decoded (a malformed page sets the error word and
// the host refuses the file), so pq_values_delta_kernel runs on streams known to be consistent with their page.
__device__ __forceinline__ bool pq_uleb(const uint8_t*& p, const uint8_t* end, uint64_t& v) {
  v = 0;
  for (int shift = 0; shift < 64; shift += 7) {
    if (p >= end) return false;
    const uint8_t b = *p++;
    v |= (uint64_t)(b & 0x7F) << shift;
    if (!(b & 0x80)) return true;
  }
  return false;
}
__device__ __forceinline__ uint64_t pq_unzigzag(uint64_t v) { return (v >> 1) ^ (0ull - (v & 1)); }

// `bw` <= 64 bits at bit `bit_off` of p: up to 9 bytes (pq_load_bits' 6-byte window covers widths up to ~40 only)
__device__ __forceinline__ uint64_t pq_load_bits64(const uint8_t* p, const uint8_t* end, uint64_t bit_off, int bw) {
  if (bw == 0) return 0;
  const uint8_t* q = p + (bit_off >> 3);
  const int s = (int)(bit_off & 7);
  const int nb = (s + bw + 7) >> 3;
  uint64_t lo = 0, hi = 0;
#pragma unroll
  for (int k = 0; k < 8; k++)
    if (k < nb && q + k < end) lo |= (uint64_t)q[k] << (8 * k);
  if (nb > 8 && q + 8 < end) hi = q[8];
  uint64_t v = lo >> s;
  if (s) v |= hi << (64 - s);
  return bw >= 64 ? v : (v & ((1ull << bw) - 1ull));
}

__device__ __forceinline__ uint64_t pq_warp_inclusive(uint64_t v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t t = __shfl_up_sync(0xFFFFFFFFu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// Walks one DELTA_BINARY_PACKED stream that must hold exactly `n` values, with one warp; every lane reads the headers
// redundantly (a few bytes per block).  DECODE: emit(i, value, ok) is called by all 32 lanes together, once for value 0 (lane 0
// ok) and then once per 32 deltas (lane l: value i0 + l), so an emitter may use warp collectives.  Returns the first byte after
// the stream, or nullptr if it is malformed: a header past `end`, a block / miniblock size the specification does not allow,
// a value count other than `n`, or a miniblock holding values that is wider than `max_bw` bits or runs past `end`.
template <bool DECODE, class Emit>
__device__ __forceinline__ const uint8_t* pq_dbp(const uint8_t* p, const uint8_t* end, int max_bw, uint32_t n, int lane, Emit emit) {
  uint64_t block, mbs, total, first;
  if (!pq_uleb(p, end, block) || !pq_uleb(p, end, mbs) || !pq_uleb(p, end, total) || !pq_uleb(p, end, first)) return nullptr;
  if (block == 0 || (block & 127) != 0 || block > (1ull << 31) || mbs == 0 || block % mbs != 0 || ((block / mbs) & 31) != 0 || total != n) return nullptr;
  const uint64_t vpm = block / mbs;
  uint64_t acc = pq_unzigzag(first);
  if (DECODE && total) emit(0u, acc, lane == 0);
  uint64_t left = total ? total - 1 : 0;  // deltas still to read
  uint32_t i0 = 1;
  while (left) {
    uint64_t mdz;
    if (!pq_uleb(p, end, mdz) || (uint64_t)(end - p) < mbs) return nullptr;
    const uint64_t min_delta = pq_unzigzag(mdz);
    const uint8_t* widths = p;
    p += mbs;
    for (uint64_t m = 0; m < mbs && left; m++) {
      const int bw = widths[m];
      if (bw > max_bw) return nullptr;
      const uint64_t bytes = vpm * (uint64_t)bw / 8;
      if ((uint64_t)(end - p) < bytes) return nullptr;
      const uint32_t take = (uint32_t)(left < vpm ? left : vpm);
      if (DECODE) {
        for (uint32_t k0 = 0; k0 < take; k0 += 32) {
          const uint32_t k = k0 + lane;
          const bool ok = k < take;
          const uint64_t d = ok ? min_delta + pq_load_bits64(p, p + bytes, (uint64_t)k * bw, bw) : 0ull;
          const uint64_t v = acc + pq_warp_inclusive(d, lane);
          emit(i0 + k, v, ok);
          acc = __shfl_sync(0xFFFFFFFFu, v, 31);  // lanes past `take` added 0
        }
      }
      p += bytes;
      left -= take;
      i0 += take;
    }
  }
  return p;
}

// a value of the column's 4- or 8-byte physical type (INT32 in the low 32 bits) -> the column's output type
__device__ __forceinline__ void pq_store_word(const PqColumn& C, void* out, uint64_t i, uint64_t v) {
  const long long s = C.phys == 1 ? (long long)(int32_t)(uint32_t)v : (long long)v;
  switch (C.out_kind) {
    case PQ_OUT_I32: ((int32_t*)out)[i] = (int32_t)s; break;
    case PQ_OUT_I64: ((long long*)out)[i] = s; break;
    case PQ_OUT_F64: ((unsigned long long*)out)[i] = v; break;  // DOUBLE: the bits as they are
    case PQ_OUT_DEC128: ((ulonglong2*)out)[i] = make_ulonglong2((unsigned long long)s, (unsigned long long)(s >> 63)); break;
    default: break;
  }
}

struct PqNoEmit {
  __device__ void operator()(uint32_t, uint64_t, bool) const {}
};

__global__ void __launch_bounds__(128) pq_delta_prepare_kernel(const PqColumn C, const PqPage* __restrict__ pages, int n_pages, const unsigned long long* __restrict__ dense_base,
                                                               const uint32_t* __restrict__ nonnull, const PqDeltaAux A) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_pages) return;
  const PqPage pg = pages[warp];
  if (pg.encoding < PQ_ENC_DBP) {
    if (lane == 0 && A.page_bytes) A.page_bytes[warp] = 0;
    return;
  }
  const uint64_t base = dense_base ? dense_base[warp] : (uint64_t)pg.row0;
  const uint32_t n = nonnull ? nonnull[warp] : pg.n_values;
  uint32_t def_off, def_len, val_off, val_len;
  pq_sections(pg, def_off, def_len, val_off, val_len);
  const uint8_t* p = pg.data + val_off;
  const uint8_t* end = p + val_len;
  bool ok = true;
  uint64_t chars = 0;
  switch (pg.encoding) {
    case PQ_ENC_DBP: ok = pq_dbp<false>(p, end, C.phys == 1 ? 32 : 64, n, lane, PqNoEmit()) != nullptr; break;
    case PQ_ENC_DLBA: {  // lengths >= 0 whose sum fits in the bytes after them
      const uint8_t* bytes = pq_dbp<false>(p, end, 32, n, lane, PqNoEmit());
      uint64_t sum = 0;
      if (bytes) pq_dbp<true>(p, end, 32, n, lane, [&](uint32_t, uint64_t len, bool on) { sum += on ? (uint64_t)(uint32_t)len : 0ull; });
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
      ok = bytes && sum <= (uint64_t)(end - bytes);
      break;
    }
    case PQ_ENC_DBA: {
      uint32_t* pre = A.pre + base;
      uint32_t* sfx = A.sfx + base;
      const uint8_t* q = pq_dbp<true>(p, end, 32, n, lane, [&](uint32_t i, uint64_t v, bool on) { if (on) pre[i] = (uint32_t)v; });
      const uint8_t* bytes = q ? pq_dbp<false>(q, end, 32, n, lane, PqNoEmit()) : nullptr;
      if (!bytes) {
        ok = false;
        break;
      }
      pq_dbp<true>(q, end, 32, n, lane, [&](uint32_t i, uint64_t v, bool on) { if (on) sfx[i] = (uint32_t)v; });
      __syncwarp();
      // value i: prefix <= length of value i-1 (0 for the first), lengths fit 31 bits, FIXED_LEN_BYTE_ARRAY: length == type_length
      uint64_t sum_sfx = 0;
      bool good = true;
      for (uint32_t i = lane; i < n; i += 32) {
        const uint64_t pr = pre[i], sx = sfx[i];
        const uint64_t prev = i ? (uint64_t)pre[i - 1] + sfx[i - 1] : 0ull;
        good &= pr <= prev && sx < (1u << 31) && pr + sx < (1u << 31);
        if (C.phys == 7) good &= pr + sx == (uint64_t)C.type_length;
        sum_sfx += sx;
        chars += pr + sx;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        sum_sfx += __shfl_xor_sync(0xFFFFFFFFu, sum_sfx, o);
        chars += __shfl_xor_sync(0xFFFFFFFFu, chars, o);
      }
      ok = __all_sync(0xFFFFFFFFu, good) && sum_sfx <= (uint64_t)(end - bytes) && chars <= 0xFFFFFFFFull;
      if (C.phys == 7) chars = 0;  // decimals are rebuilt in registers
      break;
    }
    case PQ_ENC_BSS: {
      const int w = pq_plain_width(C);
      ok = w > 0 && (uint64_t)(end - p) == (uint64_t)n * (uint64_t)w;
      break;
    }
    default: ok = false;
  }
  if (lane == 0) {
    if (!ok) {
      atomicExch(A.error, 1u);
      chars = 0;
    }
    if (A.page_bytes) A.page_bytes[warp] = (uint32_t)chars;
    if (chars) atomicAdd(A.char_total, (unsigned long long)chars);
  }
}

// One warp per page of a new encoding (other pages are pq_values_kernel's); same output contract as pq_values_kernel
__global__ void __launch_bounds__(128) pq_values_delta_kernel(const PqColumn C, const PqPage* __restrict__ pages, int n_pages, const unsigned long long* __restrict__ dense_base,
                                                              const uint32_t* __restrict__ nonnull, void* __restrict__ out, const PqDeltaAux A) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_pages) return;
  const PqPage pg = pages[warp];
  if (pg.encoding < PQ_ENC_DBP) return;
  const uint64_t base = dense_base ? dense_base[warp] : (uint64_t)pg.row0;
  const uint32_t n = nonnull ? nonnull[warp] : pg.n_values;
  uint32_t def_off, def_len, val_off, val_len;
  pq_sections(pg, def_off, def_len, val_off, val_len);
  const uint8_t* p = pg.data + val_off;
  const uint8_t* end = p + val_len;
  if (pg.encoding == PQ_ENC_DBP) {
    pq_dbp<true>(p, end, 64, n, lane, [&](uint32_t i, uint64_t v, bool on) { if (on) pq_store_word(C, out, base + i, v); });
    return;
  }
  if (pg.encoding == PQ_ENC_BSS) {
    const int w = pq_plain_width(C);
    for (uint32_t i = lane; i < n; i += 32) {
      const uint8_t* b = p + i;
      if (C.phys == 7) {
        ((ulonglong2*)out)[base + i] = pq_be_dec128([&](int k) { return b[(uint64_t)k * n]; }, w);
      } else {
        uint64_t v = 0;
        for (int k = 0; k < w; k++) v |= (uint64_t)b[(uint64_t)k * n] << (8 * k);
        pq_store_word(C, out, base + i, v);
      }
    }
    return;
  }
  unsigned long long* views = (unsigned long long*)out + 2 * base;
  if (pg.encoding == PQ_ENC_DLBA) {  // views into the page: offset = exclusive scan of the lengths
    const uint8_t* bytes = pq_dbp<false>(p, end, 32, n, lane, PqNoEmit());
    if (!bytes) return;
    uint64_t off = 0;
    pq_dbp<true>(p, end, 32, n, lane, [&](uint32_t i, uint64_t len, bool on) {
      const uint64_t l = on ? (uint64_t)(uint32_t)len : 0ull;
      const uint64_t inc = pq_warp_inclusive(l, lane);
      if (on) {
        views[2 * (uint64_t)i] = (unsigned long long)(bytes + off + inc - l);
        views[2 * (uint64_t)i + 1] = l;
      }
      off += __shfl_sync(0xFFFFFFFFu, inc, 31);
    });
    return;
  }
  // DELTA_BYTE_ARRAY: prefix / suffix lengths come from pq_delta_prepare_kernel; values are rebuilt in order
  const uint8_t* q = pq_dbp<false>(p, end, 32, n, lane, PqNoEmit());
  const uint8_t* sbytes = q ? pq_dbp<false>(q, end, 32, n, lane, PqNoEmit()) : nullptr;
  if (!sbytes) return;
  const uint32_t* pre = A.pre + base;
  const uint32_t* sfx = A.sfx + base;
  if (C.phys == 7) {  // decimal: lane k < type_length holds byte k of the current value
    const int L = C.type_length;
    uint32_t mine = 0;
    uint64_t so = 0;
    for (uint32_t i = 0; i < n; i++) {
      const uint32_t pr = pre[i], sx = sfx[i];
      if (lane < L && (uint32_t)lane >= pr) mine = sbytes[so + lane - pr];
      so += sx;
      const ulonglong2 v = pq_be_dec128([&](int k) { return (uint8_t)__shfl_sync(0xFFFFFFFFu, mine, k); }, L);
      if (lane == 0) ((ulonglong2*)out)[base + i] = v;
    }
    return;
  }
  // strings: page's bytes at chars + char_base[page]; value i at the exclusive scan of (prefix + suffix) lengths
  uint8_t* dst = A.chars + A.char_base[warp];
  uint64_t off = 0, soff = 0, prev = 0;
  for (uint32_t c0 = 0; c0 < n; c0 += 32) {
    const uint32_t i = c0 + lane;
    const bool on = i < n;
    const uint64_t pr = on ? pre[i] : 0ull, sx = on ? sfx[i] : 0ull, len = pr + sx;
    const uint64_t oinc = pq_warp_inclusive(len, lane), sinc = pq_warp_inclusive(sx, lane);
    const uint64_t my_off = off + oinc - len, my_soff = soff + sinc - sx;
    if (on) {
      views[2 * (uint64_t)i] = (unsigned long long)(dst + my_off);
      views[2 * (uint64_t)i + 1] = len;
    }
    const uint32_t m = (n - c0) < 32u ? (n - c0) : 32u;
    for (uint32_t j = 0; j < m; j++) {  // value by value: the prefix is copied from the value before, already written
      const uint64_t o = __shfl_sync(0xFFFFFFFFu, my_off, j), so = __shfl_sync(0xFFFFFFFFu, my_soff, j);
      const uint32_t pj = (uint32_t)__shfl_sync(0xFFFFFFFFu, pr, j), sj = (uint32_t)__shfl_sync(0xFFFFFFFFu, sx, j);
      for (uint32_t k = lane; k < pj; k += 32) dst[o + k] = dst[prev + k];
      for (uint32_t k = lane; k < sj; k += 32) dst[o + pj + k] = sbytes[so + k];
      __syncwarp();
      prev = o;
    }
    off += __shfl_sync(0xFFFFFFFFu, oinc, 31);
    soff += __shfl_sync(0xFFFFFFFFu, sinc, 31);
  }
}

// ---- Snappy (raw format) page decompression: one warp per page -----------------------------------------------------------------
// Format (google/snappy format_description.txt): varint uncompressed length, then elements tagged in their low two bits:
// 00 literal (length in the upper six bits, 60..63 = 1..4 following length bytes), 01 copy with 11-bit offset and length
// 4..11, 10 copy with 16-bit offset, 11 copy with 32-bit offset.  Lane 0 parses the element, all lanes move its bytes; a copy
// whose offset is shorter than its length (a repeating pattern) is moved in offset-sized steps.
__global__ void __launch_bounds__(128) pq_snappy_kernel(const PqDecompJob* __restrict__ jobs, int n_jobs, unsigned int* __restrict__ error) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_jobs) return;
  const PqDecompJob J = jobs[warp];
  if (J.raw_copy) {  // stored section (V2 levels, uncompressed V2 pages)
    for (uint32_t k = lane; k < J.src_len; k += 32) J.dst[k] = J.src[k];
    return;
  }
  const uint8_t* ip = J.src;
  const uint8_t* iend = J.src + J.src_len;
  uint8_t* out = J.dst;
  // preamble
  uint32_t ulen = 0;
  for (int shift = 0; shift < 35 && ip < iend; shift += 7) {
    const uint8_t b = *ip++;
    ulen |= (uint32_t)(b & 0x7F) << shift;
    if (!(b & 0x80)) break;
  }
  if (ulen != J.dst_len) {
    if (lane == 0) atomicExch(error, 1u);
    return;
  }
  uint32_t op = 0;
  while (ip < iend && op < ulen) {
    const uint8_t tag = *ip;  // every lane reads the same bytes: broadcast loads
    uint32_t len, off = 0;
    const uint8_t* lit = nullptr;
    switch (tag & 3) {
      case 0: {
        uint32_t l = tag >> 2;
        ip++;
        if (l >= 60) {
          const int nb = (int)l - 59;
          l = 0;
          for (int k = 0; k < nb; k++) l |= (uint32_t)ip[k] << (8 * k);
          ip += nb;
        }
        len = l + 1;
        lit = ip;
        ip += len;
        break;
      }
      case 1:
        len = 4 + ((tag >> 2) & 7);
        off = ((uint32_t)(tag >> 5) << 8) | ip[1];
        ip += 2;
        break;
      case 2:
        len = 1 + (tag >> 2);
        off = (uint32_t)ip[1] | ((uint32_t)ip[2] << 8);
        ip += 3;
        break;
      default:
        len = 1 + (tag >> 2);
        off = (uint32_t)ip[1] | ((uint32_t)ip[2] << 8) | ((uint32_t)ip[3] << 16) | ((uint32_t)ip[4] << 24);
        ip += 5;
        break;
    }
    if (op + len > ulen || (lit == nullptr && (off == 0 || off > op)) || (lit && lit + len > iend)) {
      if (lane == 0) atomicExch(error, 1u);
      return;
    }
    if (lit) {
      for (uint32_t k = lane; k < len; k += 32) out[op + k] = lit[k];
    } else {
      // pattern copy: bytes further than `off` ahead depend on bytes this same copy writes
      for (uint32_t done = 0; done < len; done += off) {
        const uint32_t step = (len - done) < off ? (len - done) : off;
        for (uint32_t k = lane; k < step; k += 32) out[op + done + k] = out[op + done + k - off];
        __syncwarp();
      }
    }
    __syncwarp();
    op += len;
  }
  if (op != ulen && lane == 0) atomicExch(error, 1u);
}

// ---- shared by the GZIP and LZ4_RAW kernels ---------------------------------------------------------------------------------------
// out[P, P+L) = the L bytes starting D bytes back (1 <= D <= P).  When D < L the source overlaps the destination and the
// bytes repeat with period D, so byte k is out[P - D + k mod D]: every source byte lies before P, all lanes copy at once.
__device__ __forceinline__ void pq_copy_match(uint8_t* out, uint64_t P, uint32_t L, uint32_t D, int lane) {
  for (uint32_t k = lane; k < L; k += 32) out[P + k] = out[P - D + (k < D ? k : k % D)];
}

// ---- DEFLATE (RFC 1951) page decompression: one warp per job ---------------------------------------------------------------------
// A GZIP page payload is what zlib's inflate accepts with header auto-detection (which pyarrow's reader uses): one or more
// members back to back, each a gzip member (RFC 1952: header with optional FEXTRA / FNAME / FCOMMENT / FHCRC, deflate data,
// CRC32 and ISIZE) or a zlib stream (RFC 1950: CMF/FLG header, deflate data, big-endian Adler-32); the outputs concatenate.
// Raw deflate without a wrapper is refused, as zlib refuses it ("incorrect header check").
//
// Every lane runs the same bit reader and Huffman decode (broadcast loads from shared memory and the page), lane t keeping
// token t of a batch of up to 32 (a literal byte, or a length / distance pair).  A batch is then executed by the warp: an
// inclusive scan of the token lengths places every token, the literals are stored in parallel, and the matches run in order
// (pq_copy_match).  A match reads only bytes before its own position, written by earlier tokens, so storing the batch's
// literals first is safe.  Match distances reach back inside the member's own output, which is in HBM already: no window.
//
// Huffman tables (per warp, shared memory): a primary lookup on the next PQ_LIT_BITS / PQ_DIST_BITS bits giving
// (symbol << 4 | code length); a code longer than that (or a bit pattern no code has) finds entry 0 and is decoded
// canonically from the per-length counts and the symbols ordered by (length, symbol), as RFC 1951 §3.2.2 defines them.
//
// Validated, each failure refusing the page (error bit 2): CM = 8, reserved gzip flags, the zlib header check, window size
// and FDICT, the FHCRC header CRC16; block type 3; stored LEN / NLEN; HLIT <= 286, HDIST <= 30, a repeat code with nothing
// to repeat or running past the lengths, a literal/length code without end-of-block; over-subscribed code sets and
// incomplete ones except a single code of length 1 (zlib's rules; a set without codes is legal until a symbol is read from
// it); literal/length symbols 286-287 and distance symbols 30-31; a distance before the member's first output byte; the
// CRC32 and ISIZE, or the Adler-32; output not exactly dst_len; input not consumed exactly.  Reads stay inside
// [src, src+src_len) and writes inside [dst, dst+dst_len) whatever the bytes say.
constexpr int PQ_LIT_BITS = 10, PQ_DIST_BITS = 8;
struct PqHuff {
  uint16_t lit[1 << PQ_LIT_BITS];   // literal/length primary lookup
  uint16_t dist[1 << PQ_DIST_BITS];  // distance primary lookup (and the code-length code while the lengths are read)
  uint16_t lit_sym[288], dist_sym[32];  // symbols ordered by (code length, symbol)
  uint32_t lit_cnt[16], dist_cnt[16];   // codes per length
  uint32_t first[16], offs[16], next[16];  // table build: first canonical code / first sorted index / running index per length
  uint8_t lens[320];                // literal/length then distance code lengths
  uint8_t clens[20];                // code-length code lengths
};

__constant__ uint16_t pq_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t pq_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t pq_dist_base[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                          193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t pq_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t pq_clen_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// LSB-first bit reader over [s, s+len).  Bytes past the end read as zero and still advance `pos`, so after byte alignment
// `pos - cnt / 8` is the next unread byte and a value above `len` means the stream was truncated.
struct PqBits {
  const uint8_t* s;
  uint32_t len, pos;
  uint64_t buf;
  int cnt;
  __device__ __forceinline__ void fill() {
    while (cnt <= 56) {
      buf |= (uint64_t)(pos < len ? s[pos] : 0) << cnt;
      pos++;
      cnt += 8;
    }
  }
  __device__ __forceinline__ uint32_t peek(int n) const { return (uint32_t)(buf & ((1ull << n) - 1ull)); }
  __device__ __forceinline__ void drop(int n) {
    buf >>= n;
    cnt -= n;
  }
  __device__ __forceinline__ uint32_t get(int n) {
    const uint32_t v = peek(n);
    drop(n);
    return v;
  }
  __device__ __forceinline__ uint32_t align() {  // skip to the next byte boundary; returns that byte's offset, buffer emptied
    drop(cnt & 7);
    const uint32_t p = pos - (uint32_t)(cnt >> 3);
    buf = 0;
    cnt = 0;
    pos = p;
    return p;
  }
};

// Needs >= 15 buffered bits.  Returns the symbol, or -1 for a bit pattern no code has.
__device__ __forceinline__ int pq_huff_decode(PqBits& b, const uint16_t* table, int P, const uint16_t* sym, const uint32_t* cnt) {
  const uint16_t e = table[b.peek(P)];
  if (e & 15) {
    b.drop(e & 15);
    return e >> 4;
  }
  int code = 0, first = 0, index = 0;  // canonical decode, one bit at a time (the code's first bit is its most significant)
  for (int l = 1; l <= 15; l++) {
    code |= (int)((b.buf >> (l - 1)) & 1);
    const int count = (int)cnt[l];
    if (code - first < count) {
      b.drop(l);
      return sym[index + code - first];
    }
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  return -1;
}

// Builds the lookup for `n` code lengths with the whole warp.  `codes`: the code-length code, which zlib never accepts
// incomplete.  Returns false for a set zlib refuses.
__device__ bool pq_huff_build(PqHuff& H, const uint8_t* lens, int n, int P, uint16_t* table, uint16_t* sym, uint32_t* cnt, bool codes, int lane) {
  if (lane < 16) cnt[lane] = 0;
  for (int k = lane; k < (1 << P); k += 32) table[k] = 0;
  __syncwarp();
  for (int s = lane; s < n; s += 32)
    if (lens[s]) atomicAdd(&cnt[lens[s]], 1u);
  __syncwarp();
  int left = 1, maxl = 0;
  bool over = false;
  for (int l = 1; l <= 15; l++) {
    left = (left << 1) - (int)cnt[l];
    over |= left < 0;
    if (cnt[l]) maxl = l;
    if (over) break;
  }
  if (maxl == 0) return true;  // no codes: every lookup misses, a symbol read from it is an error
  if (over || (left > 0 && (codes || maxl != 1))) return false;
  if (lane == 0) {
    uint32_t code = 0, o = 0;
    for (int l = 1; l <= 15; l++) {
      code = (code + cnt[l - 1]) << 1;  // cnt[0] == 0
      H.first[l] = code;
      H.offs[l] = H.next[l] = o;
      o += cnt[l];
    }
  }
  __syncwarp();
  for (int s0 = 0; s0 < n; s0 += 32) {
    const int s = s0 + lane;
    const int L = s < n ? lens[s] : 0;
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, L);
    const unsigned below = peers & ((1u << lane) - 1u);
    const uint32_t idx = L ? H.next[L] + __popc(below) : 0;
    __syncwarp();
    if (L && below == 0) H.next[L] += __popc(peers);
    __syncwarp();
    if (L) {
      sym[idx] = (uint16_t)s;
      if (L <= P) {
        const uint32_t rev = __brev(H.first[L] + (idx - H.offs[L])) >> (32 - L);
        const uint16_t e = (uint16_t)((s << 4) | L);
        for (uint32_t k = rev; k < (1u << P); k += (1u << L)) table[k] = e;
      }
    }
  }
  __syncwarp();
  return true;
}

// Executes a batch of `nt` tokens (lane t holds token t: bit 31 match, bits 16-24 length, bits 0-15 distance or the literal)
// at out + op.  False if the batch would write past dst_len or a match reaches before `mstart`.
__device__ __forceinline__ bool pq_inflate_flush(uint8_t* out, uint32_t& op, uint32_t mstart, uint32_t dst_len, uint32_t tok, int nt, int lane) {
  const bool on = lane < nt;
  const uint32_t len = on ? (tok >> 16) & 0x1FF : 0;
  uint32_t inc = len;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, inc, o);
    if (lane >= o) inc += t;
  }
  const uint32_t total = __shfl_sync(0xFFFFFFFFu, inc, 31);
  if ((uint64_t)op + total > dst_len) return false;
  const uint32_t pos = op + inc - len;
  const bool match = on && (tok >> 31);
  const uint32_t dist = tok & 0xFFFF;
  if (__any_sync(0xFFFFFFFFu, match && dist > pos - mstart)) return false;
  if (on && !match) out[pos] = (uint8_t)tok;
  __syncwarp();
  for (unsigned m = __ballot_sync(0xFFFFFFFFu, match); m; m &= m - 1) {
    const int j = __ffs(m) - 1;
    pq_copy_match(out, __shfl_sync(0xFFFFFFFFu, pos, j), __shfl_sync(0xFFFFFFFFu, len, j), __shfl_sync(0xFFFFFFFFu, dist, j), lane);
    __syncwarp();
  }
  op += total;
  return true;
}

// CRC-32 (gzip's, reflected polynomial 0xEDB88320) over the 2^k-th powers of x: crc32_combine's shift operator.
__device__ uint32_t pq_multmodp(uint32_t a, uint32_t b) {  // a * b modulo the CRC polynomial (a != 0)
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ 0xEDB88320u : b >> 1;
  }
  return p;
}
__device__ uint32_t pq_x8nmodp(uint64_t n, const uint32_t* x2n) {  // x^(8n) modulo the polynomial
  uint32_t p = 1u << 31;
  for (int k = 3; n; n >>= 1, k++)
    if (n & 1) p = pq_multmodp(x2n[k & 31], p);
  return p;
}

// CRC-32 of p[0, n) by the warp: each lane checksums a 1/32 slice, then the slices are combined in a tree.
__device__ uint32_t pq_warp_crc32(const uint8_t* p, uint32_t n, const uint32_t* T, const uint32_t* x2n, int lane) {
  const uint32_t a = (uint32_t)((uint64_t)n * lane / 32), e = (uint32_t)((uint64_t)n * (lane + 1) / 32);
  uint32_t c = 0xFFFFFFFFu;
  for (uint32_t k = a; k < e; k++) c = T[(c ^ p[k]) & 0xFF] ^ (c >> 8);
  c = ~c;
  uint32_t len = e - a;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t c2 = __shfl_down_sync(0xFFFFFFFFu, c, o), l2 = __shfl_down_sync(0xFFFFFFFFu, len, o);
    if ((lane & (2 * o - 1)) == 0) {
      c = pq_multmodp(pq_x8nmodp(l2, x2n), c) ^ c2;
      len += l2;
    }
  }
  return __shfl_sync(0xFFFFFFFFu, c, 0);
}

// Adler-32 of p[0, n) by the warp: per-lane slice sums (a = sum of bytes, b = sum of running sums) combined in a tree.
__device__ uint32_t pq_warp_adler32(const uint8_t* p, uint32_t n, int lane) {
  const uint64_t M = 65521;
  const uint32_t s = (uint32_t)((uint64_t)n * lane / 32), e = (uint32_t)((uint64_t)n * (lane + 1) / 32);
  uint64_t a = 0, b = 0;
  for (uint32_t k = s; k < e; k++) {
    a += p[k];
    b += a;
    if (((k - s) & 4095) == 4095) {
      a %= M;
      b %= M;
    }
  }
  a %= M;
  b %= M;
  uint64_t len = e - s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t a2 = __shfl_down_sync(0xFFFFFFFFu, a, o), b2 = __shfl_down_sync(0xFFFFFFFFu, b, o), l2 = __shfl_down_sync(0xFFFFFFFFu, len, o);
    if ((lane & (2 * o - 1)) == 0) {
      b = (b + b2 + (l2 % M) * a) % M;
      a = (a + a2) % M;
      len += l2;
    }
  }
  a = __shfl_sync(0xFFFFFFFFu, a, 0);
  b = __shfl_sync(0xFFFFFFFFu, b, 0);
  return (uint32_t)((((b + (uint64_t)n) % M) << 16) | ((1 + a) % M));
}

// Parses a gzip or zlib member header at s[pos]; advances pos past it.
__device__ bool pq_member_header(const uint8_t* s, uint32_t len, uint32_t& pos, bool& gz, const uint32_t* T, const uint32_t* x2n, int lane) {
  if (len - pos < 2) return false;
  const uint32_t b0 = s[pos], b1 = s[pos + 1];
  gz = b0 == 0x1F && b1 == 0x8B;
  if (!gz) {  // zlib: CM 8, window <= 32 KiB, (CMF*256 + FLG) % 31 == 0, no preset dictionary
    if (((b0 << 8) | b1) % 31 != 0 || (b0 & 15) != 8 || (b0 >> 4) > 7 || (b1 & 0x20)) return false;
    pos += 2;
    return true;
  }
  const uint32_t h0 = pos;
  if (len - pos < 10) return false;
  const uint32_t flg = s[pos + 3];
  if (s[pos + 2] != 8 || (flg & 0xE0)) return false;
  pos += 10;
  if (flg & 4) {  // FEXTRA
    if (len - pos < 2) return false;
    const uint32_t xlen = s[pos] | ((uint32_t)s[pos + 1] << 8);
    pos += 2;
    if (len - pos < xlen) return false;
    pos += xlen;
  }
  for (uint32_t f = 8; f <= 16; f <<= 1) {  // FNAME, FCOMMENT: zero-terminated
    if (!(flg & f)) continue;
    while (pos < len && s[pos]) pos++;
    if (pos >= len) return false;
    pos++;
  }
  if (flg & 2) {  // FHCRC: the low 16 bits of the header's CRC-32
    if (len - pos < 2) return false;
    const uint32_t want = s[pos] | ((uint32_t)s[pos + 1] << 8);
    if ((pq_warp_crc32(s + h0, pos - h0, T, x2n, lane) & 0xFFFF) != want) return false;
    pos += 2;
  }
  return true;
}

// The deflate blocks of one member, starting at byte b.pos; on return b is aligned after the final block.
__device__ bool pq_inflate_blocks(PqHuff& H, PqBits& b, uint8_t* out, uint32_t& op, uint32_t dst_len, int lane) {
  const uint32_t mstart = op;
  bool last = false;
  while (!last) {
    b.fill();
    if (b.pos > b.len + 8) return false;  // reading past the end of the input
    last = b.get(1);
    const uint32_t type = b.get(2);
    if (type == 0) {  // stored
      uint32_t p = b.align();
      if (p > b.len || b.len - p < 4) return false;
      const uint32_t n = b.s[p] | ((uint32_t)b.s[p + 1] << 8), nn = b.s[p + 2] | ((uint32_t)b.s[p + 3] << 8);
      p += 4;
      if (n != (~nn & 0xFFFFu) || b.len - p < n || dst_len - op < n) return false;
      for (uint32_t k = lane; k < n; k += 32) out[op + k] = b.s[p + k];
      __syncwarp();
      op += n;
      b.pos = p + n;
      continue;
    }
    if (type == 3) return false;
    if (type == 1) {  // fixed Huffman codes
      for (int s = lane; s < 320; s += 32) H.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
      __syncwarp();
      pq_huff_build(H, H.lens, 288, PQ_LIT_BITS, H.lit, H.lit_sym, H.lit_cnt, false, lane);
      pq_huff_build(H, H.lens + 288, 32, PQ_DIST_BITS, H.dist, H.dist_sym, H.dist_cnt, false, lane);
    } else {  // dynamic: the code lengths, themselves Huffman coded
      const int hlit = (int)b.get(5) + 257, hdist = (int)b.get(5) + 1, hclen = (int)b.get(4) + 4;
      if (hlit > 286 || hdist > 30) return false;
      for (int k = 0; k < 19; k++) {
        b.fill();
        const uint8_t l = k < hclen ? (uint8_t)b.get(3) : 0;
        if (lane == 0) H.clens[pq_clen_order[k]] = l;
      }
      __syncwarp();
      if (!pq_huff_build(H, H.clens, 19, PQ_DIST_BITS, H.dist, H.dist_sym, H.dist_cnt, true, lane)) return false;
      int i = 0;
      uint8_t prev = 0;
      while (i < hlit + hdist) {
        b.fill();
        const int sym = pq_huff_decode(b, H.dist, PQ_DIST_BITS, H.dist_sym, H.dist_cnt);
        if (sym < 0) return false;
        if (sym < 16) {
          if (lane == 0) H.lens[i] = (uint8_t)sym;
          prev = (uint8_t)sym;
          i++;
          continue;
        }
        int rep;
        uint8_t v = 0;
        if (sym == 16) {
          if (i == 0) return false;
          v = prev;
          rep = 3 + (int)b.get(2);
        } else {
          rep = sym == 17 ? 3 + (int)b.get(3) : 11 + (int)b.get(7);
        }
        if (i + rep > hlit + hdist) return false;
        if (lane == 0)
          for (int k = 0; k < rep; k++) H.lens[i + k] = v;
        prev = v;
        i += rep;
      }
      __syncwarp();
      if (H.lens[256] == 0) return false;  // no end-of-block code
      if (!pq_huff_build(H, H.lens, hlit, PQ_LIT_BITS, H.lit, H.lit_sym, H.lit_cnt, false, lane)) return false;
      if (!pq_huff_build(H, H.lens + hlit, hdist, PQ_DIST_BITS, H.dist, H.dist_sym, H.dist_cnt, false, lane)) return false;
    }
    int nt = 0;
    uint32_t mytok = 0;
    for (;;) {
      b.fill();  // >= 57 bits: a token takes at most 15 + 5 + 15 + 13
      if (b.pos > b.len + 8) return false;
      const int sym = pq_huff_decode(b, H.lit, PQ_LIT_BITS, H.lit_sym, H.lit_cnt);
      if (sym < 0 || sym > 285) return false;
      if (sym == 256) break;
      uint32_t tok;
      if (sym < 256) {
        tok = (1u << 16) | (uint32_t)sym;
      } else {
        const uint32_t len = pq_len_base[sym - 257] + b.get(pq_len_extra[sym - 257]);
        const int ds = pq_huff_decode(b, H.dist, PQ_DIST_BITS, H.dist_sym, H.dist_cnt);
        if (ds < 0 || ds > 29) return false;
        tok = 0x80000000u | (len << 16) | (pq_dist_base[ds] + b.get(pq_dist_extra[ds]));
      }
      if (lane == nt) mytok = tok;
      if (++nt == 32) {
        if (!pq_inflate_flush(out, op, mstart, dst_len, mytok, nt, lane)) return false;
        nt = 0;
      }
    }
    if (nt && !pq_inflate_flush(out, op, mstart, dst_len, mytok, nt, lane)) return false;
  }
  b.align();
  return b.pos <= b.len;
}

__global__ void __launch_bounds__(128) pq_inflate_kernel(const PqDecompJob* __restrict__ jobs, int n_jobs, unsigned int* __restrict__ error) {
  __shared__ uint32_t crc_table[256], x2n[32];
  __shared__ PqHuff huff[4];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    uint32_t c = (uint32_t)i;
    for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
    crc_table[i] = c;
  }
  if (threadIdx.x == 0) {
    uint32_t p = 1u << 30;  // x^1
    x2n[0] = p;
    for (int k = 1; k < 32; k++) x2n[k] = p = pq_multmodp(p, p);
  }
  __syncthreads();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_jobs) return;
  const PqDecompJob J = jobs[warp];
  if (J.raw_copy) {  // stored section: the host refuses one whose two sizes differ; never write past dst_len regardless
    if (J.src_len != J.dst_len && lane == 0) atomicOr(error, 2u);
    for (uint32_t k = lane; k < J.src_len && k < J.dst_len; k += 32) J.dst[k] = J.src[k];
    return;
  }
  if (J.dst_len == 0) return;  // zlib's callers return an empty output without reading the input; so does pyarrow
  PqHuff& H = huff[threadIdx.x >> 5];
  uint32_t pos = 0, op = 0;
  bool ok = J.src_len > 0;
  while (ok && pos < J.src_len) {
    bool gz;
    ok = pq_member_header(J.src, J.src_len, pos, gz, crc_table, x2n, lane);
    if (!ok) break;
    const uint32_t mstart = op;
    PqBits b{J.src, J.src_len, pos, 0ull, 0};
    ok = pq_inflate_blocks(H, b, J.dst, op, J.dst_len, lane);
    if (!ok) break;
    pos = b.pos;
    const uint8_t* t = J.src + pos;
    if (gz) {
      ok = J.src_len - pos >= 8;
      if (!ok) break;
      const uint32_t crc = t[0] | ((uint32_t)t[1] << 8) | ((uint32_t)t[2] << 16) | ((uint32_t)t[3] << 24);
      const uint32_t isize = t[4] | ((uint32_t)t[5] << 8) | ((uint32_t)t[6] << 16) | ((uint32_t)t[7] << 24);
      ok = isize == op - mstart && pq_warp_crc32(J.dst + mstart, op - mstart, crc_table, x2n, lane) == crc;
      pos += 8;
    } else {
      ok = J.src_len - pos >= 4;
      if (!ok) break;
      const uint32_t adler = ((uint32_t)t[0] << 24) | ((uint32_t)t[1] << 16) | ((uint32_t)t[2] << 8) | t[3];
      ok = pq_warp_adler32(J.dst + mstart, op - mstart, lane) == adler;
      pos += 4;
    }
  }
  if ((!ok || op != J.dst_len) && lane == 0) atomicOr(error, 2u);
}

// ---- LZ4 block format (LZ4_RAW) page decompression: one warp per job -----------------------------------------------------------
// Format (lz4 Block_format.md): sequences of a token (high nibble literal length, low nibble match length - 4, 15 = more
// bytes follow: each adds 0-255, 255 = continue), the literals, a 16-bit little-endian offset and the match length
// continuation.  The final sequence ends after its literals.  Lane 0's parse is every lane's (broadcast loads); the warp moves
// the bytes.  An empty input with an empty output is accepted (pyarrow reads such V2 values sections).  Refused (error bit 4): a field past the end of the input, offset 0 (which the format forbids; liblz4 accepts it
// and writes unspecified bytes), an offset before the first output byte, output past dst_len or short of it.
__global__ void __launch_bounds__(128) pq_lz4_kernel(const PqDecompJob* __restrict__ jobs, int n_jobs, unsigned int* __restrict__ error) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n_jobs) return;
  const PqDecompJob J = jobs[warp];
  if (J.raw_copy) {  // stored section: the host refuses one whose two sizes differ; never write past dst_len regardless
    if (J.src_len != J.dst_len && lane == 0) atomicOr(error, 4u);
    for (uint32_t k = lane; k < J.src_len && k < J.dst_len; k += 32) J.dst[k] = J.src[k];
    return;
  }
  const uint8_t* s = J.src;
  const uint64_t n = J.src_len, cap = J.dst_len;
  uint64_t ip = 0, op = 0;
  bool ok = n == 0 && cap == 0;  // an empty section (the values of an all-NULL V2 page): nothing to decode
  while (ip < n) {
    const uint32_t token = s[ip++];
    uint64_t lit = token >> 4;
    if (lit == 15) {
      uint32_t more;
      do {
        if (ip >= n) goto done;
        more = s[ip++];
        lit += more;
      } while (more == 255);
    }
    if (lit > n - ip || lit > cap - op) break;
    for (uint32_t k = lane; k < lit; k += 32) J.dst[op + k] = s[ip + k];
    ip += lit;
    op += lit;
    if (ip == n) {  // the final sequence: literals only
      ok = op == cap;
      break;
    }
    if (n - ip < 2) break;
    const uint32_t off = s[ip] | ((uint32_t)s[ip + 1] << 8);
    ip += 2;
    uint64_t ml = token & 15;
    if (ml == 15) {
      uint32_t more;
      do {
        if (ip >= n) goto done;
        more = s[ip++];
        ml += more;
      } while (more == 255);
    }
    ml += 4;
    if (off == 0 || off > op || ml > cap - op) break;
    __syncwarp();
    pq_copy_match(J.dst, op, (uint32_t)ml, off, lane);
    __syncwarp();
    op += ml;
  }
done:
  if (!ok && lane == 0) atomicOr(error, 4u);
}

static inline unsigned pq_grid(int n_warps) { return (unsigned)((n_warps * 32 + 127) / 128); }
void launch_pq_snappy(const PqDecompJob* jobs, int n_jobs, unsigned int* error, cudaStream_t st) {
  if (n_jobs > 0) launch_kernel(pq_snappy_kernel, pq_grid(n_jobs), 128, 0, st, jobs, n_jobs, error);
}
void launch_pq_inflate(const PqDecompJob* jobs, int n_jobs, unsigned int* error, cudaStream_t st) {
  if (n_jobs > 0) launch_kernel(pq_inflate_kernel, pq_grid(n_jobs), 128, 0, st, jobs, n_jobs, error);
}
void launch_pq_lz4(const PqDecompJob* jobs, int n_jobs, unsigned int* error, cudaStream_t st) {
  if (n_jobs > 0) launch_kernel(pq_lz4_kernel, pq_grid(n_jobs), 128, 0, st, jobs, n_jobs, error);
}

void launch_pq_levels(const PqPage* pages, int n_pages, uint8_t* valid, uint32_t* nonnull, unsigned long long* total_nonnull, cudaStream_t st) {
  if (n_pages > 0) launch_kernel(pq_levels_kernel, pq_grid(n_pages), 128, 0, st, pages, n_pages, valid, nonnull, total_nonnull);
}
void launch_pq_page_scan(const uint32_t* nonnull, int n_pages, unsigned long long* dense_base, cudaStream_t st) {
  if (n_pages > 0) launch_kernel(pq_page_scan_kernel, 1, 1024, 0, st, nonnull, n_pages, dense_base);
}
void launch_pq_dict(const PqColumn& C, const PqPage* dict_pages, int n_dicts, cudaStream_t st) {
  if (n_dicts > 0) launch_kernel(pq_dict_kernel, pq_grid(n_dicts), 128, 0, st, C, dict_pages, n_dicts);
}
void launch_pq_values(const PqColumn& C, const PqPage* pages, int n_pages, const unsigned long long* dense_base, const uint32_t* nonnull, void* out, cudaStream_t st) {
  if (n_pages > 0) launch_kernel(pq_values_kernel, pq_grid(n_pages), 128, 0, st, C, pages, n_pages, dense_base, nonnull, out);
}
void launch_pq_expand(const PqPage* pages, int n_pages, const unsigned long long* dense_base, const uint8_t* valid, const void* dense, void* out, int width,
                      cudaStream_t st) {
  if (n_pages > 0) launch_kernel(pq_expand_kernel, pq_grid(n_pages), 128, 0, st, pages, n_pages, dense_base, valid, dense, out, width);
}
void launch_pq_delta_prepare(const PqColumn& C, const PqPage* pages, int n_pages, const unsigned long long* dense_base, const uint32_t* nonnull, const PqDeltaAux& A,
                             cudaStream_t st) {
  if (n_pages > 0) launch_kernel(pq_delta_prepare_kernel, pq_grid(n_pages), 128, 0, st, C, pages, n_pages, dense_base, nonnull, A);
}
void launch_pq_values_delta(const PqColumn& C, const PqPage* pages, int n_pages, const unsigned long long* dense_base, const uint32_t* nonnull, void* out,
                            const PqDeltaAux& A, cudaStream_t st) {
  if (n_pages > 0) launch_kernel(pq_values_delta_kernel, pq_grid(n_pages), 128, 0, st, C, pages, n_pages, dense_base, nonnull, out, A);
}

}  // namespace b200
