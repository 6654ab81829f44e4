// Nested-loop join kernels (sm_90a): NestedLoopJoinExec (wire surface ballista/core/proto/datafusion.proto:1301-1307).
//
// The cross product of the build side (left, read whole by every task) and the probe side is walked without being
// materialised.  Each CTA owns 256 probe rows, one per thread; the thread keeps its probe row's operands in registers.
// Build rows go through shared memory one 256-row tile at a time: the staging pass turns every build operand into its
// comparison image once, so the inner loop is one broadcast shared-memory load and one compare per atom and pair.
// The filter is the boolean program of NljSpec (kernels.h), evaluated in Kleene logic on two bit words per pair.
//
// Two launches with a scan between them, so the output is exact and deterministic:
//   nlj_count: passing pairs per probe row (+ build marks through a per-tile shared flag, probe marks per thread);
//   nlj_write: the pairs (build row, probe row) at their final place -- probe-row order, build-row order inside a
//              probe row -- skipping probe rows without pairs and ending a CTA's tile loop once its rows are done.
// Bytes: N_p * w_p + N_b * w_b * (probe tiles) + 16 * N_out.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "keyimg.cuh"

namespace b200 {

static const int NLJ_BLOCK = 256;  // probe rows per CTA == build rows per shared tile

// the value an operand is compared by: one signed 64-bit word (integers, UInt64 with its top bit flipped, doubles as
// their total-order key), a 128-bit decimal, or a string view {ptr, len}
__device__ __forceinline__ ulonglong2 nlj_load(const KeyCol& c, uint8_t vk, int64_t i) {
  ulonglong2 v;
  v.y = 0;
  switch (vk) {
    case NLJ_V_I128:
    case NLJ_V_STR: return ((const ulonglong2*)c.data)[i];
    case NLJ_V_F64: {
      const double d = c.phys == PH_F32 ? (double)((const float*)c.data)[i] : ((const double*)c.data)[i];
      long long x = __double_as_longlong(d);
      v.x = (unsigned long long)(x ^ (long long)((unsigned long long)(x >> 63) >> 1));
      return v;
    }
    case NLJ_V_U64: v.x = ((const unsigned long long*)c.data)[i] ^ (1ull << 63); return v;
    default: v.x = jkey_image(c, i); return v;
  }
}

// sign of (a - b)
__device__ __forceinline__ int nlj_cmp(uint8_t vk, ulonglong2 a, ulonglong2 b) {
  if (vk == NLJ_V_STR) {
    const uint8_t* s = (const uint8_t*)a.x;
    const uint8_t* t = (const uint8_t*)b.x;
    const uint32_t la = (uint32_t)a.y, lb = (uint32_t)b.y, n = la < lb ? la : lb;
    for (uint32_t k = 0; k < n; k++)
      if (s[k] != t[k]) return s[k] < t[k] ? -1 : 1;
    return la < lb ? -1 : (la > lb ? 1 : 0);
  }
  if (vk == NLJ_V_I128) {
    if (a.y != b.y) return (long long)a.y < (long long)b.y ? -1 : 1;
    return a.x < b.x ? -1 : (a.x > b.x ? 1 : 0);
  }
  return (long long)a.x < (long long)b.x ? -1 : ((long long)a.x > (long long)b.x ? 1 : 0);
}

__device__ __forceinline__ bool nlj_cmp_result(uint8_t op, int c) {
  switch (op) {
    case 0: return c == 0;
    case 1: return c != 0;
    case 2: return c < 0;
    case 3: return c <= 0;
    case 4: return c > 0;
    default: return c >= 0;
  }
}

// one side's Bool atom of row i: (T, F) bits at position k
__device__ __forceinline__ void nlj_bool_bits(const KeyCol& c, int64_t i, int k, uint32_t& t, uint32_t& f) {
  if (!jkey_valid(c, i)) return;
  if (((const uint8_t*)c.data)[i]) t |= 1u << k;
  else f |= 1u << k;
}

// MODE 0: nlj_count; MODE 1: nlj_write
template <int MODE>
__global__ void __launch_bounds__(NLJ_BLOCK) nlj_kernel(const __grid_constant__ NljSpec S, int64_t n_build, int64_t n_probe, uint32_t* __restrict__ counts,
                                                        uint8_t* __restrict__ build_mark, uint8_t* __restrict__ probe_mark,
                                                        const uint64_t* __restrict__ offsets, int64_t* __restrict__ out_b, int64_t* __restrict__ out_p) {
  __shared__ ulonglong2 s_val[NLJ_MAX_ATOMS][NLJ_BLOCK];  // build operands of the tile
  __shared__ uint32_t s_t[NLJ_BLOCK], s_f[NLJ_BLOCK];      // build Bool atoms (T / F bits)
  __shared__ uint32_t s_v[NLJ_BLOCK];                      // build operands that are not NULL (bit per atom)
  __shared__ uint8_t s_mark[NLJ_BLOCK];
  const int tid = threadIdx.x;
  const int64_t j = (int64_t)blockIdx.x * NLJ_BLOCK + tid;
  const bool live = j < n_probe;
  const int na = S.n_atoms;

  ulonglong2 pv[NLJ_MAX_ATOMS];
  uint32_t pt = 0, pf = 0, pvalid = 0;
#pragma unroll
  for (int k = 0; k < NLJ_MAX_ATOMS; k++) {
    pv[k].x = pv[k].y = 0;
    if (k < na && live) {
      const NljAtom& a = S.atoms[k];
      if (a.kind == NLJ_PROBE_BOOL) {
        nlj_bool_bits(a.probe, j, k, pt, pf);
      } else if (a.kind == NLJ_CMP && jkey_valid(a.probe, j)) {
        pv[k] = nlj_load(a.probe, a.vk, j);
        pvalid |= 1u << k;
      }
    }
  }
  uint32_t left = 0;  // nlj_write: pairs of this probe row still to write
  uint64_t pos = 0;
  if (MODE == 1 && live) {
    left = counts[j];
    pos = offsets[j];
  }
  uint32_t cnt = 0;

  for (int64_t t0 = 0; t0 < n_build; t0 += NLJ_BLOCK) {
    if (MODE == 1) {
      if (!__syncthreads_or(left != 0)) break;  // every probe row of the CTA has all its pairs
    } else {
      __syncthreads();  // the previous tile is consumed
    }
    const int tn = (int)(n_build - t0 < NLJ_BLOCK ? n_build - t0 : NLJ_BLOCK);
    if (tid < tn) {
      const int64_t i = t0 + tid;
      uint32_t bt = 0, bf = 0, bv = 0;
#pragma unroll
      for (int k = 0; k < NLJ_MAX_ATOMS; k++) {
        if (k < na) {
          const NljAtom& a = S.atoms[k];
          if (a.kind == NLJ_BUILD_BOOL) {
            nlj_bool_bits(a.build, i, k, bt, bf);
          } else if (a.kind == NLJ_CMP && jkey_valid(a.build, i)) {
            s_val[k][tid] = nlj_load(a.build, a.vk, i);
            bv |= 1u << k;
          }
        }
      }
      s_t[tid] = bt;
      s_f[tid] = bf;
      s_v[tid] = bv;
    }
    if (MODE == 0) s_mark[tid] = 0;
    __syncthreads();
    const bool work = MODE == 0 ? live : left != 0;
    if (work) {
      for (int r = 0; r < tn; r++) {
        bool pass = true;
        if (S.result >= 0) {
          uint32_t T = s_t[r] | pt, F = s_f[r] | pf;
          const uint32_t valid = s_v[r] & pvalid;
#pragma unroll
          for (int k = 0; k < NLJ_MAX_ATOMS; k++) {
            if (k < na && S.atoms[k].kind == NLJ_CMP && ((valid >> k) & 1u)) {
              const bool c = nlj_cmp_result(S.atoms[k].cmp, nlj_cmp(S.atoms[k].vk, s_val[k][r], pv[k]));
              if (c) T |= 1u << k;
              else F |= 1u << k;
            }
          }
          for (int s = 0; s < S.n_steps; s++) {
            const NljStep st = S.steps[s];
            const uint32_t ta = (T >> st.a) & 1u, fa = (F >> st.a) & 1u, tb = (T >> st.b) & 1u, fb = (F >> st.b) & 1u;
            uint32_t t, f;
            if (st.kind == NLJ_AND) {
              t = ta & tb;
              f = fa | fb;
            } else if (st.kind == NLJ_OR) {
              t = ta | tb;
              f = fa & fb;
            } else {
              t = fa;
              f = ta;
            }
            T |= t << st.dst;
            F |= f << st.dst;
          }
          pass = (T >> S.result) & 1u;
        }
        if (!pass) continue;
        if (MODE == 0) {
          cnt++;
          if (build_mark) s_mark[r] = 1;
        } else {
          out_b[pos] = t0 + r;
          out_p[pos] = j;
          pos++;
          if (--left == 0) break;
        }
      }
    }
    if (MODE == 0 && build_mark) {
      __syncthreads();
      if (tid < tn && s_mark[tid]) build_mark[t0 + tid] = 1;
    }
  }
  if (MODE == 0 && live) {
    counts[j] = cnt;
    if (probe_mark && cnt) probe_mark[j] = 1;
  }
}

void launch_nlj_count(const NljSpec& S, int64_t n_build, int64_t n_probe, uint32_t* counts, uint8_t* build_mark, uint8_t* probe_mark, cudaStream_t st) {
  if (n_probe <= 0) return;
  const int64_t g = (n_probe + NLJ_BLOCK - 1) / NLJ_BLOCK;
  launch_kernel(nlj_kernel<0>, (unsigned)g, NLJ_BLOCK, 0, st, S, n_build, n_probe, counts, build_mark, probe_mark, nullptr, nullptr, nullptr);
}

void launch_nlj_write(const NljSpec& S, int64_t n_build, int64_t n_probe, const uint32_t* counts, const uint64_t* offsets, int64_t* out_build_idx,
                      int64_t* out_probe_idx, cudaStream_t st) {
  if (n_probe <= 0 || n_build <= 0) return;
  const int64_t g = (n_probe + NLJ_BLOCK - 1) / NLJ_BLOCK;
  launch_kernel(nlj_kernel<1>, (unsigned)g, NLJ_BLOCK, 0, st, S, n_build, n_probe, const_cast<uint32_t*>(counts), nullptr, nullptr, offsets, out_build_idx, out_probe_idx);
}

}  // namespace b200
