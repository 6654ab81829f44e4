// High-cardinality GROUP BY kernel (sm_90a): AggregateExec(Partial | Final*) whose keys are one or two integer-like
// columns and whose aggregates are COUNT / SUM (AVG = SUM + COUNT) over plain columns or decimal products.
//
// Reference operator: AggregateExec + GroupsAccumulator [EXT, DataFusion 53.1] (wire surface
// ballista/core/proto/datafusion.proto:1257-1271): rows are grouped through a hash table keyed by the group values and
// every accumulator state is updated per row; q17's inner aggregate (GROUP BY l_partkey, 20 M groups at SF100), q18's
// (l_orderkey), q15's (l_suppkey), q20's ((l_partkey, l_suppkey)) and every FinalPartitioned merge of such states.
//
// One pass, no tile VM: each thread streams R rows per step straight from the Arrow columns (coalesced, the byte count per
// row is the algorithmic figure of SURVEY.md 8(d): N * (w_keys + w_args)), resolves its group in the open-addressing table
// (the slot word holds mix64(key image), a bijection, so ONE 8-byte compare identifies the group exactly) and updates
// the accumulators with L2 atomics: COUNT is a fire-and-forget reduction, a 128-bit SUM is one 64-bit atomic add plus a
// second one only when a carry or a non-zero high word exists.  Table traffic is random access: while the table fits the
// 50 MB L2 the kernel runs at the column-scan rate, beyond that it is bound by 32-byte-sector DRAM accesses.
// Anything outside the pattern (wide decimal operands, keys that do not fit the image) raises `bail` and the host
// re-runs the aggregate on the general tile-VM sink: same results by construction.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../common/hash.hpp"
#include "kernels.h"

namespace b200 {

typedef __int128 gi128;

static const int GB_BLOCK = 256;
static const int GB_R = 4;
static const int GB_MAX_PROBE = 512;

__device__ __forceinline__ bool gb_ld(const FusedCol& c, int64_t i, uint64_t& lo, uint64_t& hi) {
  // value of row i as a sign-extended 128-bit integer; false for an unsupported width
  if (c.width == 16) {
    const ulonglong2 v = ((const ulonglong2*)c.data)[i];
    lo = v.x;
    hi = v.y;
  } else if (c.width == 8) {
    const int64_t v = ((const int64_t*)c.data)[i];
    lo = (uint64_t)v;
    hi = (uint64_t)(v >> 63);
  } else {
    const int64_t v = (int64_t)((const int32_t*)c.data)[i];
    lo = (uint64_t)v;
    hi = (uint64_t)(v >> 63);
  }
  return true;
}
__device__ __forceinline__ bool gb_fits64(uint64_t lo, uint64_t hi) { return hi == (uint64_t)((int64_t)lo >> 63); }

__device__ __forceinline__ bool gb_cmp(int op, int64_t v, int64_t imm) {
  switch (op) {
    case 0: return v == imm;
    case 1: return v != imm;
    case 2: return v < imm;
    case 3: return v <= imm;
    case 4: return v > imm;
    default: return v >= imm;
  }
}

__global__ void __launch_bounds__(GB_BLOCK) groupby_kernel(const GroupBySpec S) {
  __shared__ unsigned int new_groups;
  if (threadIdx.x == 0) new_groups = 0;
  __syncthreads();
  const AggTable& T = S.table;
  unsigned long long mask = T.cap - 1, slot_base = 0;
  int64_t n = S.n_rows;
  int64_t first = (int64_t)blockIdx.x * (GB_BLOCK * GB_R), stride = (int64_t)gridDim.x * (GB_BLOCK * GB_R);
  if (S.pf_K > 0) {
    // partition-first: which bucket does this CTA serve?  (largest b with cta_start[b] <= blockIdx.x)
    int lo = 0, hi = S.pf_K;
    if (blockIdx.x >= S.pf_cta_start[S.pf_K]) return;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (S.pf_cta_start[mid] <= blockIdx.x) lo = mid;
      else hi = mid;
    }
    mask = S.pf_slots - 1;
    slot_base = (unsigned long long)lo * S.pf_slots;
    first = (int64_t)S.pf_row_start[lo] + (int64_t)(blockIdx.x - S.pf_cta_start[lo]) * (GB_BLOCK * GB_R);
    n = (int64_t)S.pf_row_start[lo + 1];
    stride = (int64_t)1 << 60;  // exactly one tile per CTA
  }
  unsigned int inserted = 0;
  bool stop = false;
  for (int64_t base = first; base < n && !stop; base += stride) {
    // another thread found the table full or met a row outside the pattern: the launch is void, leave early
    if (*(volatile unsigned int*)&S.status->overflow || *(volatile unsigned int*)&S.status->pack_overflow) break;
    unsigned long long slot[GB_R];
    uint32_t live = 0;
    // ---- keys, filters, group resolution: GB_R independent probe chains in flight ---------------------------------
#pragma unroll
    for (int r = 0; r < GB_R; r++) {
      const int64_t i = base + (int64_t)r * GB_BLOCK + threadIdx.x;
      slot[r] = 0;
      if (i >= n) continue;
      bool pass = true;
      for (int f = 0; f < S.n_filters && pass; f++) {
        uint64_t lo, hi;
        gb_ld(S.cols[S.f_col[f]], i, lo, hi);
        if (!gb_fits64(lo, hi)) {
          atomicExch(&S.status->pack_overflow, 1u);  // wide decimal in a filter: general path
          pass = false;
          stop = true;
        }
        pass = pass && gb_cmp(S.f_op[f], (int64_t)lo, S.f_imm[f]);
      }
      if (!pass) continue;
      uint64_t img = 0;
      if (S.n_keys >= 1) {
        uint64_t lo, hi;
        gb_ld(S.cols[S.key_col[0]], i, lo, hi);
        img = lo;
        if (S.n_keys == 2) {
          uint64_t lo2, hi2;
          gb_ld(S.cols[S.key_col[1]], i, lo2, hi2);
          if ((lo >> 32) || (lo2 >> 32)) {  // the two-key image needs both keys in [0, 2^32)
            atomicExch(&S.status->pack_overflow, 1u);
            stop = true;
            continue;
          }
          img = lo | (lo2 << 32);
        }
      }
      const unsigned long long h = S.n_keys ? mix64(img) : 1ull;
      if (h == 0) {  // the one key image whose hash collides with the "empty" word
        atomicExch(&S.status->pack_overflow, 1u);
        stop = true;
        continue;
      }
      unsigned long long s = slot_base + (h & mask);
      bool found = false;
      for (int probe = 0; probe < GB_MAX_PROBE; probe++) {
        unsigned long long cur = *(volatile unsigned long long*)&T.hash[s];
        if (cur == 0) {
          cur = atomicCAS(&T.hash[s], 0ull, h);
          if (cur == 0) {
            // new group: publish its key columns for the extraction kernel (read after this kernel)
            if (S.n_keys >= 1) {
              uint64_t lo, hi;
              gb_ld(S.cols[S.key_col[0]], i, lo, hi);
              T.keys[(0ull * T.cap + s) * 2 + 0] = lo;
              T.keys[(0ull * T.cap + s) * 2 + 1] = hi;
              T.key_valid[0ull * T.cap + s] = 1;
            }
            if (S.n_keys == 2) {
              uint64_t lo, hi;
              gb_ld(S.cols[S.key_col[1]], i, lo, hi);
              T.keys[(1ull * T.cap + s) * 2 + 0] = lo;
              T.keys[(1ull * T.cap + s) * 2 + 1] = hi;
              T.key_valid[1ull * T.cap + s] = 1;
            }
            T.state[s] = 2u;
            inserted++;
            found = true;
            break;
          }
        }
        if (cur == h) {
          found = true;
          break;
        }
        s = slot_base + ((s + 1) & mask);
      }
      if (!found) {
        atomicExch(&S.status->overflow, 1u);  // table (nearly) full: the host retries with a larger one
        stop = true;
        continue;
      }
      slot[r] = s;
      live |= 1u << r;
    }
    // ---- accumulate -------------------------------------------------------------------------------------------------
#pragma unroll
    for (int r = 0; r < GB_R; r++) {
      if (!((live >> r) & 1)) continue;
      const int64_t i = base + (int64_t)r * GB_BLOCK + threadIdx.x;
      gi128 prod[2] = {0, 0};
      bool ok = true;
      for (int j = 0; j < S.n_prod; j++) {
        gi128 a;
        if (S.p_a_src[j] == 1) {
          a = prod[0];
        } else {
          uint64_t lo, hi;
          gb_ld(S.cols[S.p_a_col[j]], i, lo, hi);
          ok = ok && gb_fits64(lo, hi);
          a = (gi128)(int64_t)lo;
        }
        uint64_t blo, bhi;
        gb_ld(S.cols[S.p_b_col[j]], i, blo, bhi);
        ok = ok && gb_fits64(blo, bhi);
        gi128 b = (gi128)(int64_t)blo;
        if (S.p_kind[j] == 0) b = (gi128)S.p_lit[j] - b;
        else if (S.p_kind[j] == 1) b = (gi128)S.p_lit[j] + b;
        // exact while |a| < 2^63 (first product) / < 2^95 (chained) and |b| < 2^31: checked below
        const gi128 lim = (gi128)1 << 31;
        ok = ok && b > -lim && b < lim;
        if (S.p_a_src[j] == 1) {
          const gi128 lim_a = (gi128)1 << 95;
          ok = ok && a > -lim_a && a < lim_a;
        }
        prod[j] = a * b;
      }
      if (!ok) {
        atomicExch(&S.status->pack_overflow, 1u);  // operands outside the fast ranges: general (checked 128-bit) path
        stop = true;
        continue;
      }
      const unsigned long long s = slot[r];
      for (int a = 0; a < S.n_acc; a++) {
        unsigned long long* cell = T.acc + ((unsigned long long)a * T.cap + s) * 2;
        const int src = S.a_src[a];
        if (src == 3) {
          atomicAdd(&cell[0], 1ull);
          continue;
        }
        uint64_t lo, hi;
        if (src == 0) {
          gb_ld(S.cols[S.a_col[a]], i, lo, hi);
        } else {
          const gi128 v = prod[src - 1];
          lo = (uint64_t)v;
          hi = (uint64_t)(v >> 64);
        }
        const unsigned long long old = atomicAdd(&cell[0], (unsigned long long)lo);
        const unsigned long long h2 = hi + ((old + lo) < old ? 1ull : 0ull);
        if (h2) atomicAdd(&cell[1], h2);
      }
    }
  }
  if (inserted) atomicAdd(&new_groups, inserted);
  __syncthreads();
  if (threadIdx.x == 0 && new_groups) atomicAdd(T.n_groups, new_groups);
}

// One warp: exclusive prefix sums of the bucket sizes (rows) and of the CTAs each bucket needs.
__global__ void groupby_plan_kernel(const unsigned long long* __restrict__ counts, int K, unsigned long long* __restrict__ row_start,
                                    unsigned int* __restrict__ cta_start) {
  const int lane = threadIdx.x;
  unsigned long long rows_run = 0;
  unsigned int ctas_run = 0;
  for (int b0 = 0; b0 < K; b0 += 32) {
    const int b = b0 + lane;
    const unsigned long long c = b < K ? counts[b] : 0ull;
    const unsigned int t = (unsigned int)((c + GROUPBY_ROWS_PER_CTA - 1) / GROUPBY_ROWS_PER_CTA);
    unsigned long long ri = c;
    unsigned int ti = t;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long ro = __shfl_up_sync(0xFFFFFFFFu, ri, d);
      const unsigned int to = __shfl_up_sync(0xFFFFFFFFu, ti, d);
      if (lane >= d) {
        ri += ro;
        ti += to;
      }
    }
    if (b < K) {
      row_start[b] = rows_run + ri - c;
      cta_start[b] = ctas_run + ti - t;
    }
    rows_run += __shfl_sync(0xFFFFFFFFu, ri, 31);
    ctas_run += __shfl_sync(0xFFFFFFFFu, ti, 31);
  }
  if (lane == 0) {
    row_start[K] = rows_run;
    cta_start[K] = ctas_run;
  }
}

cudaError_t launch_groupby_plan(const unsigned long long* counts, int K, unsigned long long* row_start, unsigned int* cta_start, cudaStream_t st) {
  static_assert(GROUPBY_ROWS_PER_CTA == GB_BLOCK * GB_R, "one tile per CTA in partition-first mode");
  launch_kernel(groupby_plan_kernel, 1, 32, 0, st, counts, K, row_start, cta_start);
  return cudaGetLastError();
}

cudaError_t launch_groupby(const GroupBySpec& S, int sm_count, cudaStream_t st) {
  if (S.pf_K > 0) {
    // upper bound of sum_b ceil(rows_b / tile): the CTAs past cta_start[K] exit at once
    const int64_t g = (S.n_rows + GROUPBY_ROWS_PER_CTA - 1) / GROUPBY_ROWS_PER_CTA + S.pf_K;
    launch_kernel(groupby_kernel, (unsigned)g, GB_BLOCK, 0, st, S);
    return cudaGetLastError();
  }
  int64_t g = (S.n_rows + (int64_t)GB_BLOCK * GB_R - 1) / ((int64_t)GB_BLOCK * GB_R);
  if (g < 1) g = 1;
  if (g > (int64_t)sm_count * 8) g = (int64_t)sm_count * 8;  // 8 resident CTAs of 256 threads per SM
  launch_kernel(groupby_kernel, (unsigned)g, GB_BLOCK, 0, st, S);
  return cudaGetLastError();
}

}  // namespace b200
