// Window functions (sm_90a): WindowAggExec / BoundedWindowAggExec over an input in (partition keys, order keys) order.
//
// The host hands every kernel the sort permutation `perm` (sorted position i -> input row perm[i]; nullptr when the input
// already is in that order).  Kernels work in sorted positions and write results to input rows, so no row moves.
//
//   window_flags      row i starts a partition / a peer group (its keys differ from row i - 1's; NULL equals NULL)
//   window_segments   from the exclusive scans of those flags: partition and peer-group ids per row, their start rows
//   window_load       an aggregate's argument in sorted order, as the accumulator type
//   window_scan_*     segmented inclusive scan (forward or backward) of (value, non-NULL count); segments are partitions,
//                     peer groups, or blocks of w rows from each partition's start (the van Herk / Gil-Werman split)
//   window_eval       per row: the frame, then the ranking arithmetic, an input-row index (offset / value functions,
//                     gathered by the host) or the frame's aggregate read from at most two scan results
//
// Every part of a frame aggregate sums only rows inside that frame: no difference of partition-wide prefix sums, which
// would lose a small frame's digits after a large value.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "kernels.h"

namespace b200 {

typedef __int128 i128;
typedef unsigned __int128 u128;

static inline int win_grid(int64_t n, int block) {
  int64_t g = (n + block - 1) / block;
  if (g < 1) g = 1;
  if (g > 132 * 16) g = 132 * 16;  // grid-stride loops
  return (int)g;
}

__device__ __forceinline__ int64_t win_row(const int64_t* perm, int64_t i) { return perm ? perm[i] : i; }

// ---- partition and peer boundaries -------------------------------------------------------------------------------
__device__ bool win_key_eq(const KeyCol& k, int64_t a, int64_t b) {
  const bool va = !k.valid || k.valid[a], vb = !k.valid || k.valid[b];
  if (!va || !vb) return va == vb;
  switch (k.width) {
    case 1: return ((const uint8_t*)k.data)[a] == ((const uint8_t*)k.data)[b];
    case 2: return ((const uint16_t*)k.data)[a] == ((const uint16_t*)k.data)[b];
    case 4: return ((const uint32_t*)k.data)[a] == ((const uint32_t*)k.data)[b];
    case 8: return ((const unsigned long long*)k.data)[a] == ((const unsigned long long*)k.data)[b];
    default: break;
  }
  const ulonglong2 x = ((const ulonglong2*)k.data)[a], y = ((const ulonglong2*)k.data)[b];
  if (k.phys != PH_STRVIEW) return x.x == y.x && x.y == y.y;  // Decimal128
  if (x.y != y.y) return false;                                // view {characters, length}
  const uint8_t *p = (const uint8_t*)x.x, *q = (const uint8_t*)y.x;
  for (unsigned long long i = 0; i < x.y; i++)
    if (p[i] != q[i]) return false;
  return true;
}

__global__ void window_flags_kernel(const WinKeys K, const int64_t* perm, int64_t n, uint32_t* part_flag, uint32_t* peer_flag) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    bool p = i == 0, q = p;
    if (i > 0) {
      const int64_t r = win_row(perm, i), s = win_row(perm, i - 1);
      for (int k = 0; k < K.n_part && !p; k++) p = !win_key_eq(K.k[k], r, s);
      q = p;
      for (int k = K.n_part; k < K.n_part + K.n_order && !q; k++) q = !win_key_eq(K.k[k], r, s);
    }
    part_flag[i] = p ? 1u : 0u;
    peer_flag[i] = q ? 1u : 0u;
  }
}
void launch_window_flags(const WinKeys& K, const int64_t* perm, int64_t n, uint32_t* part_flag, uint32_t* peer_flag, cudaStream_t st) {
  if (n <= 0) return;
  launch_kernel(window_flags_kernel, win_grid(n, 256), 256, 0, st, K, perm, n, part_flag, peer_flag);
}

__global__ void window_segments_kernel(const uint32_t* part_flag, const uint32_t* peer_flag, const uint64_t* part_ex, const uint64_t* peer_ex, int64_t n,
                                       WinBounds B) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t p = (uint32_t)(part_ex[i] + part_flag[i] - 1), g = (uint32_t)(peer_ex[i] + peer_flag[i] - 1);
    B.pid[i] = p;
    B.gid[i] = g;
    if (part_flag[i]) {
      B.part_start[p] = (uint32_t)i;
      B.part_first_peer[p] = g;
    }
    if (peer_flag[i]) B.peer_start[g] = (uint32_t)i;
    if (i == n - 1) {
      B.part_start[p + 1] = (uint32_t)n;
      B.peer_start[g + 1] = (uint32_t)n;
    }
  }
}
void launch_window_segments(const uint32_t* part_flag, const uint32_t* peer_flag, const uint64_t* part_ex, const uint64_t* peer_ex, int64_t n,
                            const WinBounds& B, cudaStream_t st) {
  if (n <= 0) return;
  launch_kernel(window_segments_kernel, win_grid(n, 256), 256, 0, st, part_flag, peer_flag, part_ex, peer_ex, n, B);
}

// ---- argument load ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ long long win_ld_int(const void* d, uint8_t phys, int64_t r) {
  switch (phys) {
    case PH_I8: return ((const int8_t*)d)[r];
    case PH_I16: return ((const int16_t*)d)[r];
    case PH_I32: return ((const int32_t*)d)[r];
    case PH_U8:
    case PH_BOOL8: return ((const uint8_t*)d)[r];
    case PH_U16: return ((const uint16_t*)d)[r];
    case PH_U32: return ((const uint32_t*)d)[r];
    default: return ((const long long*)d)[r];  // PH_I64 / PH_U64 (bits)
  }
}
__device__ __forceinline__ double win_ld_f64(const void* d, uint8_t phys, int64_t r) {
  switch (phys) {
    case PH_F32: return (double)((const float*)d)[r];
    case PH_F64: return ((const double*)d)[r];
    case PH_U64: return (double)((const unsigned long long*)d)[r];
    default: return (double)win_ld_int(d, phys, r);
  }
}
// IEEE total order as a signed 64-bit key (the grouped MIN / MAX order): -0.0 < +0.0, NaN above +inf
__device__ __forceinline__ long long win_f64_key(double v) {
  const long long b = __double_as_longlong(v);
  return b ^ (long long)((unsigned long long)(b >> 63) >> 1);
}
__device__ __forceinline__ double win_key_f64(long long k) { return __longlong_as_double(k ^ (long long)((unsigned long long)(k >> 63) >> 1)); }

__global__ void window_load_kernel(const WinLoad L, const int64_t* perm, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = win_row(perm, i);
    const bool ok = L.conv == WCV_ONE || !L.valid || L.valid[r];
    L.out_valid[i] = ok ? 1 : 0;
    switch (L.conv) {
      case WCV_I64: ((long long*)L.out)[i] = ok ? win_ld_int(L.data, L.phys, r) : 0; break;
      case WCV_U64_KEY: ((long long*)L.out)[i] = ok ? (long long)(((const unsigned long long*)L.data)[r] ^ 0x8000000000000000ull) : 0; break;
      case WCV_F64: ((double*)L.out)[i] = ok ? win_ld_f64(L.data, L.phys, r) : 0.0; break;
      case WCV_F64_KEY: ((long long*)L.out)[i] = ok ? win_f64_key(win_ld_f64(L.data, L.phys, r)) : 0; break;
      case WCV_I128: ((ulonglong2*)L.out)[i] = ok ? ((const ulonglong2*)L.data)[r] : make_ulonglong2(0, 0); break;
      default: ((long long*)L.out)[i] = 0; break;  // WCV_VALID / WCV_ONE: COUNT reads the non-NULL count only
    }
  }
}
void launch_window_load(const WinLoad& L, const int64_t* perm, int64_t n, cudaStream_t st) {
  if (n <= 0) return;
  launch_kernel(window_load_kernel, win_grid(n, 256), 256, 0, st, L, perm, n);
}

// ---- segmented scans -------------------------------------------------------------------------------------------------
template <typename T>
struct WElem {
  T v;
  uint32_t c;  // non-NULL values
  uint32_t h;  // segment head inside the span
};
__device__ __forceinline__ long long wsum(long long a, long long b) { return (long long)((unsigned long long)a + (unsigned long long)b); }  // wraps, as SUM(Int64)
__device__ __forceinline__ i128 wsum(i128 a, i128 b) { return (i128)((u128)a + (u128)b); }
__device__ __forceinline__ double wsum(double a, double b) { return a + b; }

// a followed by b, both inside one segment
template <typename T>
__device__ __forceinline__ WElem<T> wmerge(const WElem<T>& a, const WElem<T>& b, int op) {
  WElem<T> r;
  r.c = a.c + b.c;
  r.h = a.h | b.h;
  if (!a.c) r.v = b.v;
  else if (!b.c) r.v = a.v;
  else if (op == WOP_SUM) r.v = wsum(a.v, b.v);
  else if (op == WOP_MIN) r.v = b.v < a.v ? b.v : a.v;
  else r.v = b.v > a.v ? b.v : a.v;
  return r;
}
// segmented scan operator: b restarts when it holds a segment head
template <typename T>
__device__ __forceinline__ WElem<T> wcomb(const WElem<T>& a, const WElem<T>& b, int op) {
  return b.h ? b : wmerge(a, b, op);
}

static const int WSCAN_BLOCK = 256, WSCAN_ITEMS = 8, WSCAN_TILE = WSCAN_BLOCK * WSCAN_ITEMS;

// the element at logical scan position l (backward scans run from the last row to the first)
template <typename T>
__device__ __forceinline__ WElem<T> wload(const WinScan& S, const WinBounds& B, int64_t l) {
  const int64_t i = S.dir ? S.n - 1 - l : l;
  WElem<T> e;
  e.v = ((const T*)S.vals)[i];
  e.c = S.valid[i];
  int64_t s0, s1;
  if (S.seg == WSEG_PEER) {
    const uint32_t g = B.gid[i];
    s0 = B.peer_start[g];
    s1 = B.peer_start[g + 1];
  } else {
    const uint32_t p = B.pid[i];
    s0 = B.part_start[p];
    s1 = B.part_start[p + 1];
    if (S.seg == WSEG_BLOCK) {
      const int64_t b0 = s0 + (i - s0) / S.w * S.w;
      s1 = b0 + S.w < s1 ? b0 + S.w : s1;
      s0 = b0;
    }
  }
  e.h = (S.dir ? i + 1 == s1 : i == s0) ? 1u : 0u;
  return e;
}

// inclusive scan of one value per thread across the block (Hillis-Steele; the operator is not commutative)
template <typename T>
__device__ WElem<T> wblock_inclusive(WElem<T> x, WElem<T>* sh, int op) {
  const int t = threadIdx.x;
  sh[t] = x;
  __syncthreads();
  for (int o = 1; o < WSCAN_BLOCK; o <<= 1) {
    WElem<T> y = x;
    if (t >= o) y = sh[t - o];
    __syncthreads();
    if (t >= o) x = wcomb(y, x, op);
    sh[t] = x;
    __syncthreads();
  }
  return x;
}

template <typename T>
__device__ __forceinline__ WElem<T> wident() {
  WElem<T> e;
  e.v = T(0);
  e.c = 0;
  e.h = 0;
  return e;
}

template <typename T>
__global__ void __launch_bounds__(WSCAN_BLOCK) window_scan_reduce_kernel(const WinScan S, const WinBounds B) {
  __shared__ WElem<T> sh[WSCAN_BLOCK];
  const int64_t base = (int64_t)blockIdx.x * WSCAN_TILE + (int64_t)threadIdx.x * WSCAN_ITEMS;
  WElem<T> acc = wident<T>();
  for (int k = 0; k < WSCAN_ITEMS; k++)
    if (base + k < S.n) acc = wcomb(acc, wload<T>(S, B, base + k), S.op);
  acc = wblock_inclusive(acc, sh, S.op);
  if (threadIdx.x == WSCAN_BLOCK - 1) ((WElem<T>*)S.tiles)[blockIdx.x] = acc;
}

// exclusive scan of the tile aggregates, in place, by one block
template <typename T>
__global__ void __launch_bounds__(WSCAN_BLOCK) window_scan_tiles_kernel(const WinScan S, int64_t n_tiles) {
  __shared__ WElem<T> sh[WSCAN_BLOCK];
  __shared__ WElem<T> carry_sh;
  WElem<T>* tiles = (WElem<T>*)S.tiles;
  if (threadIdx.x == 0) carry_sh = wident<T>();
  __syncthreads();
  for (int64_t c0 = 0; c0 < n_tiles; c0 += WSCAN_BLOCK) {
    const int64_t t = c0 + threadIdx.x;
    const WElem<T> mine = t < n_tiles ? tiles[t] : wident<T>();
    const WElem<T> inc = wblock_inclusive(mine, sh, S.op);
    const WElem<T> carry = carry_sh;
    const WElem<T> ex = threadIdx.x ? wcomb(carry, sh[threadIdx.x - 1], S.op) : carry;
    __syncthreads();
    if (t < n_tiles) tiles[t] = ex;
    if (threadIdx.x == WSCAN_BLOCK - 1) carry_sh = wcomb(carry, inc, S.op);
    __syncthreads();
  }
}

template <typename T>
__global__ void __launch_bounds__(WSCAN_BLOCK) window_scan_apply_kernel(const WinScan S, const WinBounds B) {
  __shared__ WElem<T> sh[WSCAN_BLOCK];
  const int64_t base = (int64_t)blockIdx.x * WSCAN_TILE + (int64_t)threadIdx.x * WSCAN_ITEMS;
  WElem<T> items[WSCAN_ITEMS];
  WElem<T> acc = wident<T>();
  for (int k = 0; k < WSCAN_ITEMS; k++) {
    items[k] = base + k < S.n ? wload<T>(S, B, base + k) : wident<T>();
    acc = wcomb(acc, items[k], S.op);
  }
  wblock_inclusive(acc, sh, S.op);
  const WElem<T> tile_ex = ((const WElem<T>*)S.tiles)[blockIdx.x];
  WElem<T> run = threadIdx.x ? wcomb(tile_ex, sh[threadIdx.x - 1], S.op) : tile_ex;
  for (int k = 0; k < WSCAN_ITEMS; k++) {
    const int64_t l = base + k;
    if (l >= S.n) break;
    run = wcomb(run, items[k], S.op);
    const int64_t i = S.dir ? S.n - 1 - l : l;
    ((T*)S.out_v)[i] = run.v;
    S.out_c[i] = run.c;
  }
}

template <typename T>
static void scan_t(const WinScan& S, const WinBounds& B, cudaStream_t st) {
  const int64_t n_tiles = (S.n + WSCAN_TILE - 1) / WSCAN_TILE;
  launch_kernel(window_scan_reduce_kernel<T>, (unsigned)n_tiles, WSCAN_BLOCK, 0, st, S, B);
  launch_kernel(window_scan_tiles_kernel<T>, 1, WSCAN_BLOCK, 0, st, S, n_tiles);
  launch_kernel(window_scan_apply_kernel<T>, (unsigned)n_tiles, WSCAN_BLOCK, 0, st, S, B);
}
int64_t window_scan_tile_bytes(int64_t n) { return ((n + WSCAN_TILE - 1) / WSCAN_TILE + 1) * (int64_t)sizeof(WElem<i128>); }
void launch_window_scan(const WinScan& S, const WinBounds& B, cudaStream_t st) {
  if (S.n <= 0) return;
  switch (S.acc) {
    case WACC_I128: scan_t<i128>(S, B, st); break;
    case WACC_F64: scan_t<double>(S, B, st); break;
    default: scan_t<long long>(S, B, st); break;
  }
}

// ---- per-row evaluation ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int64_t wclamp(int64_t v, int64_t lo, int64_t hi) { return v < lo ? lo : v > hi ? hi : v; }

// the frame [fs, fe) of sorted row i, clipped to its partition [ps, pe); empty when its end falls before its start
__device__ void win_frame(const WinEval& E, int64_t i, int64_t ps, int64_t pe, int64_t qs, int64_t qe, int64_t& fs, int64_t& fe) {
  const bool rows = E.units == WUNITS_ROWS;
  switch (E.s_kind) {
    case WB_UNBOUNDED_PRECEDING: fs = ps; break;
    case WB_PRECEDING: fs = i - E.s_off; break;
    case WB_CURRENT_ROW: fs = rows ? i : qs; break;
    default: fs = i + E.s_off; break;  // WB_FOLLOWING
  }
  switch (E.e_kind) {
    case WB_UNBOUNDED_FOLLOWING: fe = pe; break;
    case WB_PRECEDING: fe = i - E.e_off + 1; break;
    case WB_CURRENT_ROW: fe = rows ? i + 1 : qe; break;
    default: fe = i + E.e_off + 1; break;  // WB_FOLLOWING
  }
  fs = wclamp(fs, ps, pe);
  fe = wclamp(fe, ps, pe);
  if (fe < fs) fe = fs;
}

template <typename T>
__device__ __forceinline__ WElem<T> wat(const void* v, const uint32_t* c, int64_t i) {
  WElem<T> e;
  e.v = ((const T*)v)[i];
  e.c = c[i];
  e.h = 0;
  return e;
}

__device__ __forceinline__ void win_store_int(void* d, uint8_t phys, int64_t o, long long v) {
  switch (phys) {
    case PH_I8:
    case PH_U8:
    case PH_BOOL8: ((int8_t*)d)[o] = (int8_t)v; break;
    case PH_I16:
    case PH_U16: ((int16_t*)d)[o] = (int16_t)v; break;
    case PH_I32:
    case PH_U32: ((int32_t*)d)[o] = (int32_t)v; break;
    default: ((long long*)d)[o] = v;
  }
}

template <typename T>
__device__ void win_finish(const WinEval& E, const WElem<T>& r, int64_t o);
template <>
__device__ void win_finish<long long>(const WinEval& E, const WElem<long long>& r, int64_t o) {
  bool ok = r.c > 0;
  switch (E.fin) {
    case WFIN_COUNT:
      ((long long*)E.out)[o] = (long long)r.c;
      ok = true;
      break;
    case WFIN_MINMAX_U64: ((unsigned long long*)E.out)[o] = (unsigned long long)r.v ^ 0x8000000000000000ull; break;
    case WFIN_MINMAX_F64:
      if (E.out_phys == PH_F32) ((float*)E.out)[o] = (float)win_key_f64(r.v);
      else ((double*)E.out)[o] = win_key_f64(r.v);
      break;
    default: win_store_int(E.out, E.out_phys, o, r.v); break;  // WFIN_VALUE: SUM (wrapping), integer MIN / MAX
  }
  if (E.out_valid) E.out_valid[o] = ok ? 1 : 0;
}
template <>
__device__ void win_finish<double>(const WinEval& E, const WElem<double>& r, int64_t o) {
  const bool ok = r.c > 0;
  ((double*)E.out)[o] = !ok ? 0.0 : E.fin == WFIN_AVG ? r.v / (double)r.c : r.v;
  E.out_valid[o] = ok ? 1 : 0;
}
template <>
__device__ void win_finish<i128>(const WinEval& E, const WElem<i128>& r, int64_t o) {
  const bool ok = r.c > 0;
  i128 v = ok ? r.v : 0;
  if (ok && E.fin == WFIN_AVG && !avg_decimal(r.v, (unsigned long long)r.c, E.imm, E.prec, &v)) atomicMax(E.error, 1u);
  ((ulonglong2*)E.out)[o] = make_ulonglong2((unsigned long long)v, (unsigned long long)((u128)v >> 64));
  E.out_valid[o] = ok ? 1 : 0;
}

template <typename T>
__global__ void window_eval_kernel(const WinEval E, const WinBounds B, const int64_t* perm, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t p = B.pid[i], g = B.gid[i];
    const int64_t ps = B.part_start[p], pe = B.part_start[p + 1], qs = B.peer_start[g], qe = B.peer_start[g + 1];
    const int64_t o = win_row(perm, i);
    const int64_t rows = pe - ps;
    switch (E.fn) {
      case WF_ROW_NUMBER: ((unsigned long long*)E.out)[o] = (unsigned long long)(i - ps + 1); break;
      case WF_RANK: ((unsigned long long*)E.out)[o] = (unsigned long long)(qs - ps + 1); break;
      case WF_DENSE_RANK: ((unsigned long long*)E.out)[o] = (unsigned long long)(g - B.part_first_peer[p] + 1); break;
      case WF_PERCENT_RANK: ((double*)E.out)[o] = rows > 1 ? (double)(qs - ps) / (double)(rows - 1) : 0.0; break;
      case WF_CUME_DIST: ((double*)E.out)[o] = (double)(qe - ps) / (double)rows; break;
      case WF_NTILE: {
        // SQL standard: the first rows % n buckets hold one row more; with n > rows the buckets are 1..rows
        const int64_t r = i - ps, q = rows / E.arg, rem = rows % E.arg, big = rem * (q + 1);
        const int64_t b = r < big ? r / (q + 1) : rem + (r - big) / q;
        ((unsigned long long*)E.out)[o] = (unsigned long long)(b + 1);
        break;
      }
      case WF_OFFSET: {
        const int64_t j = i + E.arg;
        E.idx_out[o] = j >= ps && j < pe ? win_row(perm, j) : -1;
        break;
      }
      default: {
        int64_t fs, fe;
        win_frame(E, i, ps, pe, qs, qe, fs, fe);
        if (E.fn == WF_FIRST) {
          E.idx_out[o] = fe > fs ? win_row(perm, fs) : -1;
        } else if (E.fn == WF_LAST) {
          E.idx_out[o] = fe > fs ? win_row(perm, fe - 1) : -1;
        } else if (E.fn == WF_NTH) {
          E.idx_out[o] = E.arg <= fe - fs ? win_row(perm, fs + E.arg - 1) : -1;  // n >= 1: a position inside the frame
        } else {  // WF_AGG
          WElem<T> r = wident<T>();
          if (fe > fs) {
            if (E.read == WRD_FWD) {
              r = wat<T>(E.fwd_v, E.fwd_c, fe - 1);
            } else if (E.read == WRD_BWD) {
              r = wat<T>(E.bwd_v, E.bwd_c, fs);
            } else {
              // blocks of w rows from the partition start: a frame of at most w rows is a suffix of one block plus at most a
              // prefix of the next; inside one block it starts at the block's first row or ends at its last
              const int64_t bs = (fs - ps) / E.w, be = (fe - 1 - ps) / E.w;
              if (bs != be) r = wmerge(wat<T>(E.bwd_v, E.bwd_c, fs), wat<T>(E.fwd_v, E.fwd_c, fe - 1), E.op);
              else if (fs == ps + bs * E.w) r = wat<T>(E.fwd_v, E.fwd_c, fe - 1);
              else r = wat<T>(E.bwd_v, E.bwd_c, fs);
            }
          }
          win_finish<T>(E, r, o);
        }
      }
    }
  }
}
void launch_window_eval(const WinEval& E, const WinBounds& B, const int64_t* perm, int64_t n, cudaStream_t st) {
  if (n <= 0) return;
  switch (E.acc) {
    case WACC_I128: launch_kernel(window_eval_kernel<i128>, win_grid(n, 256), 256, 0, st, E, B, perm, n); break;
    case WACC_F64: launch_kernel(window_eval_kernel<double>, win_grid(n, 256), 256, 0, st, E, B, perm, n); break;
    default: launch_kernel(window_eval_kernel<long long>, win_grid(n, 256), 256, 0, st, E, B, perm, n); break;
  }
}

// rows whose index is -1 (outside the partition) get the default value of LAG / LEAD
__global__ void window_fill_kernel(const int64_t* idx, int64_t n, void* out, uint8_t* valid, int width, ulonglong2 lit) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (idx[i] >= 0) continue;
    uint8_t* d = (uint8_t*)out + i * width;
    const uint8_t* s = (const uint8_t*)&lit;
    for (int b = 0; b < width; b++) d[b] = s[b];
    valid[i] = 1;
  }
}
void launch_window_fill(const int64_t* idx, int64_t n, void* out, uint8_t* valid, int width, const void* lit16, cudaStream_t st) {
  if (n <= 0) return;
  ulonglong2 lit;
  memcpy(&lit, lit16, 16);
  launch_kernel(window_fill_kernel, win_grid(n, 256), 256, 0, st, idx, n, out, valid, width, lit);
}

}  // namespace b200
