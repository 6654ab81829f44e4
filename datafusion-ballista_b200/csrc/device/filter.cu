// FilterExec (+ column projection) without the tile VM (sm_90a): predicates that are boolean combinations of comparisons
// between plain columns and literals -- every TPC-H scan filter except LIKE -- evaluated per row in registers, the
// surviving rows of the forwarded columns compacted in input order.
//
// Reference operator: FilterExec (ballista/core/proto/datafusion.proto:1027-1034: expr, optional projection):
// `mask = expr.evaluate(batch)`, `filter_record_batch` compacts every projected column.  Here one kernel does both:
//   * the lowered predicate (comparison / AND / OR / NOT instructions over bool registers, csrc/host/lower.hpp) is run on a
//     64-bit register file per row: bit k = bool register k -- no shared-memory VM registers, no per-instruction decode;
//   * integer / date / decimal operands are compared as 64- or 128-bit integers, strings by length + bytes (equality only);
//   * the kept rows of a 1024-row tile are ranked with ballots, the tile's output base comes from the same decoupled
//     look-back as the VM's materialising sink (input order is preserved across tiles: FilterExec is order preserving);
//   * Utf8 columns leave as 16-byte views {pointer, length} into the source characters.
// HBM bound: N * (w_pred + w_pass) read + s * N * w_pass written (SURVEY.md 8(d) "Filter").
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace b200 {

static const int FF_BLOCK = 256;
static const int FF_R = 4;
static const int FF_TILE = FF_BLOCK * FF_R;

__device__ __forceinline__ unsigned long long ff_ld_acquire(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void ff_st_release(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ void ff_load_int(const FfCol& c, int64_t i, int64_t& lo, int64_t& hi) {
  switch (c.phys) {
    case PH_DEC128: {
      const ulonglong2 v = ((const ulonglong2*)c.data)[i];
      lo = (int64_t)v.x;
      hi = (int64_t)v.y;
      return;
    }
    case PH_I64: lo = ((const int64_t*)c.data)[i]; break;
    case PH_U64: lo = ((const int64_t*)c.data)[i]; hi = 0; return;
    case PH_I32: lo = ((const int32_t*)c.data)[i]; break;
    case PH_U32: lo = ((const uint32_t*)c.data)[i]; break;
    case PH_I16: lo = ((const int16_t*)c.data)[i]; break;
    case PH_U16: lo = ((const uint16_t*)c.data)[i]; break;
    case PH_I8: lo = ((const int8_t*)c.data)[i]; break;
    default: lo = ((const uint8_t*)c.data)[i]; break;
  }
  hi = lo >> 63;
}
__device__ __forceinline__ void ff_load_str(const FfCol& c, int64_t i, const uint8_t*& p, uint32_t& len) {
  if (c.phys == PH_STRVIEW) {
    const ulonglong2 v = ((const ulonglong2*)c.data)[i];
    p = (const uint8_t*)v.x;
    len = (uint32_t)v.y;
  } else {
    const int32_t o0 = ((const int32_t*)c.data)[i], o1 = ((const int32_t*)c.data)[i + 1];
    p = c.chars + o0;
    len = (uint32_t)(o1 - o0);
  }
}
__device__ __forceinline__ bool ff_cmp(int op, int c) {  // c: -1 / 0 / +1
  switch (op) {
    case 0: return c == 0;
    case 1: return c != 0;
    case 2: return c < 0;
    case 3: return c <= 0;
    case 4: return c > 0;
    default: return c >= 0;
  }
}

// The predicate program for FF_R rows in lockstep: every instruction first loads its operands for all rows (independent
// loads in flight together), then computes; rows are predicated, nothing branches on data.  Returns the pass bits.
__device__ __forceinline__ uint32_t ff_eval_rows(const FastFilterSpec& S, const int64_t (&row)[FF_R], uint32_t live) {
  unsigned long long regs[FF_R];
#pragma unroll
  for (int r = 0; r < FF_R; r++) regs[r] = 0;
  uint32_t pass = live;
  for (int k = 0; k < S.n_ops; k++) {
    const FfOp op = S.ops[k];
    uint32_t res = 0;
    if (op.kind == FF_CMP) {
      if (op.vt == 2) {
#pragma unroll
        for (int r = 0; r < FF_R; r++) {
          if (!(((op.filter ? pass : live) >> r) & 1)) continue;  // string compares walk bytes: skip rows that cannot matter
          const uint8_t *pa, *pb;
          uint32_t la, lb;
          if (op.a_imm) {
            pa = (const uint8_t*)S.imms[op.a].lo;
            la = (uint32_t)S.imms[op.a].hi;
          } else {
            ff_load_str(S.cols[op.a], row[r], pa, la);
          }
          if (op.b_imm) {
            pb = (const uint8_t*)S.imms[op.b].lo;
            lb = (uint32_t)S.imms[op.b].hi;
          } else {
            ff_load_str(S.cols[op.b], row[r], pb, lb);
          }
          bool eq = la == lb;
          for (uint32_t q = 0; eq && q < la; q++) eq = pa[q] == pb[q];
          res |= (uint32_t)((op.cmp == 0) ? eq : !eq) << r;
        }
      } else {
        int64_t alo[FF_R], ahi[FF_R], blo[FF_R], bhi[FF_R];
#pragma unroll
        for (int r = 0; r < FF_R; r++) {
          const int64_t i = ((live >> r) & 1) ? row[r] : row[0];
          if (op.a_imm) {
            alo[r] = (int64_t)S.imms[op.a].lo;
            ahi[r] = (int64_t)S.imms[op.a].hi;
          } else {
            ff_load_int(S.cols[op.a], i, alo[r], ahi[r]);
          }
          if (op.b_imm) {
            blo[r] = (int64_t)S.imms[op.b].lo;
            bhi[r] = (int64_t)S.imms[op.b].hi;
          } else {
            ff_load_int(S.cols[op.b], i, blo[r], bhi[r]);
          }
        }
#pragma unroll
        for (int r = 0; r < FF_R; r++) {
          int c;
          if (op.vt == 0) c = alo[r] < blo[r] ? -1 : (alo[r] > blo[r] ? 1 : 0);
          else if (op.vt == 3) c = (uint64_t)alo[r] < (uint64_t)blo[r] ? -1 : ((uint64_t)alo[r] > (uint64_t)blo[r] ? 1 : 0);
          else c = ahi[r] != bhi[r] ? (ahi[r] < bhi[r] ? -1 : 1) : ((uint64_t)alo[r] < (uint64_t)blo[r] ? -1 : ((uint64_t)alo[r] > (uint64_t)blo[r] ? 1 : 0));
          res |= (uint32_t)ff_cmp(op.cmp, c) << r;
        }
      }
    } else {
#pragma unroll
      for (int r = 0; r < FF_R; r++) {
        const bool x = (regs[r] >> op.a) & 1, y = (regs[r] >> op.b) & 1;
        const bool v = op.kind == FF_AND ? (x && y) : op.kind == FF_OR ? (x || y) : op.kind == FF_NOT ? !x : x;
        res |= (uint32_t)v << r;
      }
    }
    if (op.filter) {
      pass &= res;
    } else {
#pragma unroll
      for (int r = 0; r < FF_R; r++) regs[r] = (regs[r] & ~(1ull << op.dst)) | ((unsigned long long)((res >> r) & 1) << op.dst);
    }
  }
  return pass;
}

__global__ void __launch_bounds__(FF_BLOCK, 4) fast_filter_kernel(const FastFilterSpec S) {
  __shared__ uint32_t warp_tot[FF_R][FF_BLOCK / 32];
  __shared__ unsigned long long tile_base_sh;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t n = S.n_rows;
  const int64_t n_tiles = (n + FF_TILE - 1) / FF_TILE;
  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int64_t t0 = t * FF_TILE;
    uint32_t lane_pre[FF_R], live = 0;
    int64_t row[FF_R];
#pragma unroll
    for (int r = 0; r < FF_R; r++) {
      row[r] = t0 + r * FF_BLOCK + tid;
      live |= (uint32_t)(row[r] < n) << r;
    }
    const uint32_t pass = live ? ff_eval_rows(S, row, live) : 0u;
#pragma unroll
    for (int r = 0; r < FF_R; r++) {
      const uint32_t m = __ballot_sync(0xFFFFFFFFu, (pass >> r) & 1);
      lane_pre[r] = __popc(m & ((1u << lane) - 1u));
      if (lane == 0) warp_tot[r][warp] = __popc(m);
    }
    __syncthreads();
    // rank of row (r, warp, lane) == its row index order inside the tile
    uint32_t pos[FF_R], run = 0;
#pragma unroll
    for (int r = 0; r < FF_R; r++) {
      uint32_t mine = 0;
      for (int w = 0; w < FF_BLOCK / 32; w++) {
        if (w == warp) mine = run;
        run += warp_tot[r][w];
      }
      pos[r] = mine + lane_pre[r];
    }
    if (warp == 0) {
      const unsigned long long F_AGG = 1ull << 62, F_PFX = 2ull << 62, CNT = (1ull << 62) - 1;
      unsigned long long* ts = S.tile_state;
      if (lane == 0 && t > 0) ff_st_release(&ts[t], F_AGG | (unsigned long long)run);
      unsigned long long excl = 0;
      for (int64_t p = t - 1; p >= 0; p -= 32) {
        const int64_t q = p - lane;
        unsigned long long v = F_PFX;
        if (q >= 0) {
          do {
            v = ff_ld_acquire(&ts[q]);
          } while ((v >> 62) == 0);
        }
        const uint32_t pf = __ballot_sync(0xFFFFFFFFu, (v >> 62) == 2);
        const int first = pf ? __ffs(pf) - 1 : 32;
        unsigned long long c = (lane <= first) ? (v & CNT) : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, o);
        excl += c;
        if (pf) break;
      }
      if (lane == 0) {
        ff_st_release(&ts[t], F_PFX | (excl + (unsigned long long)run));
        tile_base_sh = excl;
        if (t == n_tiles - 1) S.status->out_rows = excl + (unsigned long long)run;
      }
    }
    __syncthreads();
    const unsigned long long base = tile_base_sh;
    if (run) {
      for (int j = 0; j < S.n_out; j++) {
        const FfCol c = S.cols[S.out_col[j]];
        void* out = S.out_data[j];
#pragma unroll
        for (int r = 0; r < FF_R; r++) {
          if (!((pass >> r) & 1)) continue;
          const int64_t i = t0 + r * FF_BLOCK + tid;
          const unsigned long long o = base + pos[r];
          if (c.phys == PH_UTF8 || c.phys == PH_STRVIEW) {
            const uint8_t* p;
            uint32_t len;
            ff_load_str(c, i, p, len);
            ((ulonglong2*)out)[o] = make_ulonglong2((unsigned long long)p, (unsigned long long)len);
          } else {
            switch (c.width) {
              case 1: ((uint8_t*)out)[o] = ((const uint8_t*)c.data)[i]; break;
              case 2: ((uint16_t*)out)[o] = ((const uint16_t*)c.data)[i]; break;
              case 4: ((uint32_t*)out)[o] = ((const uint32_t*)c.data)[i]; break;
              case 8: ((uint64_t*)out)[o] = ((const uint64_t*)c.data)[i]; break;
              default: ((ulonglong2*)out)[o] = ((const ulonglong2*)c.data)[i]; break;
            }
          }
        }
      }
    }
    __syncthreads();  // warp_tot / tile_base_sh are reused by the next tile
  }
}

cudaError_t launch_fast_filter(const FastFilterSpec& S, int sm_count, cudaStream_t st) {
  const int64_t n_tiles = (S.n_rows + FF_TILE - 1) / FF_TILE;
  if (n_tiles <= 0) return cudaSuccess;
  // the look-back needs every CTA co-resident: ask the runtime how many fit (launch bounds ask for 4 per SM)
  static int per_sm = 0;
  if (per_sm == 0) {
    int v = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, fast_filter_kernel, FF_BLOCK, 0) != cudaSuccess || v < 1) v = 1;
    per_sm = v > 4 ? 4 : v;
  }
  int64_t g = n_tiles < (int64_t)sm_count * per_sm ? n_tiles : (int64_t)sm_count * per_sm;
  launch_kernel(fast_filter_kernel, (unsigned)g, FF_BLOCK, 0, st, S);
  return cudaGetLastError();
}

}  // namespace b200
