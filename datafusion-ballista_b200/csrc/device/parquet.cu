// Parquet page decode on the GPU (sm_90a): definition levels, dictionaries, PLAIN and RLE_DICTIONARY values ->
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
//   * nullable columns: values are stored densely, a second pass spreads them to their rows using the validity bytes.
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
        const int L = C.type_length;
        unsigned long long ulo = 0, uhi = (src[0] & 0x80) ? ~0ull : 0ull;
        if (src[0] & 0x80) ulo = ~0ull;
        for (int k = 0; k < L; k++) {
          uhi = (uhi << 8) | (ulo >> 56);
          ulo = (ulo << 8) | src[k];
        }
        lo = (long long)ulo;
        hi = (long long)uhi;
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

static inline unsigned pq_grid(int n_warps) { return (unsigned)((n_warps * 32 + 127) / 128); }
void launch_pq_snappy(const PqDecompJob* jobs, int n_jobs, unsigned int* error, cudaStream_t st) {
  if (n_jobs > 0) pq_snappy_kernel<<<pq_grid(n_jobs), 128, 0, st>>>(jobs, n_jobs, error);
}

void launch_pq_levels(const PqPage* pages, int n_pages, uint8_t* valid, uint32_t* nonnull, unsigned long long* total_nonnull, cudaStream_t st) {
  if (n_pages > 0) pq_levels_kernel<<<pq_grid(n_pages), 128, 0, st>>>(pages, n_pages, valid, nonnull, total_nonnull);
}
void launch_pq_page_scan(const uint32_t* nonnull, int n_pages, unsigned long long* dense_base, cudaStream_t st) {
  if (n_pages > 0) pq_page_scan_kernel<<<1, 1024, 0, st>>>(nonnull, n_pages, dense_base);
}
void launch_pq_dict(const PqColumn& C, const PqPage* dict_pages, int n_dicts, cudaStream_t st) {
  if (n_dicts > 0) pq_dict_kernel<<<pq_grid(n_dicts), 128, 0, st>>>(C, dict_pages, n_dicts);
}
void launch_pq_values(const PqColumn& C, const PqPage* pages, int n_pages, const unsigned long long* dense_base, const uint32_t* nonnull, void* out, cudaStream_t st) {
  if (n_pages > 0) pq_values_kernel<<<pq_grid(n_pages), 128, 0, st>>>(C, pages, n_pages, dense_base, nonnull, out);
}
void launch_pq_expand(const PqPage* pages, int n_pages, const unsigned long long* dense_base, const uint8_t* valid, const void* dense, void* out, int width,
                      cudaStream_t st) {
  if (n_pages > 0) pq_expand_kernel<<<pq_grid(n_pages), 128, 0, st>>>(pages, n_pages, dense_base, valid, dense, out, width);
}

}  // namespace b200
