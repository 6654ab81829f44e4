// Hash join kernels (sm_90a): HashJoinExec build + single-pass probe.
//
// Reference operator: HashJoinExec [EXT, DataFusion 53.1] (wire surface ballista/core/proto/datafusion.proto:1134-1144):
// the build side is collected into one batch + a chained hash map, probe batches are hashed, candidate pairs are
// verified by key equality and the output is gathered by (build index, probe index) pairs.  Same structure here:
//   build : one 16-byte node per build row {tag, next}; `heads[bucket]` is swung to the newest row with atomicExch.
//           tag = the key itself (sign-extended 64-bit image) when the join has ONE integer-like key -- every TPC-H
//           join key but q9's (suppkey, partkey) pair and the string keys -- so a probe step is ONE random 16-byte
//           access with no second look at the key columns; otherwise tag = the 64-bit row hash and candidates are
//           verified against the key columns.
//   probe : one pass.  Every warp stages its matches (build row, probe row) in shared memory and reserves output
//           space with one atomicAdd per ~100 pairs; semi / anti / outer joins get their "had a match" marks in the
//           same pass.  The host sizes the pair buffers optimistically (probe rows + build rows); the kernel keeps
//           counting past the capacity and the host re-runs with the exact size in that (rare: many-to-many) case.
// HBM bound (random access): algorithmic bytes N_b * w_b + N_p * w_p + N_out * w_out (SURVEY.md 8(d)).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../common/hash.hpp"
#include "kernels.h"
#include "keyimg.cuh"

namespace b200 {

static inline int join_grid(int64_t n, int block, int per_thread) {
  int64_t g = (n + (int64_t)block * per_thread - 1) / ((int64_t)block * per_thread);
  if (g < 1) g = 1;
  if (g > 132 * 16) g = 132 * 16;
  return (int)g;
}

template <bool EXACT>
__global__ void __launch_bounds__(256) join_build2_kernel(JoinKeys K, const uint64_t* __restrict__ build_hash, int64_t n, int32_t* __restrict__ heads,
                                                          uint64_t mask, JoinNode* __restrict__ nodes) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    JoinNode nd;
    nd._pad = 0;
    if (EXACT) {
      if (!jkey_valid(K.build[0], i)) {  // a NULL key never matches: the row stays out of the table
        nd.tag = 0;
        nd.next = -1;
        nodes[i] = nd;
        continue;
      }
      nd.tag = jkey_image(K.build[0], i);
    } else {
      nd.tag = build_hash[i];
    }
    nd.next = atomicExch(&heads[mix64(nd.tag) & mask], (int32_t)i);
    nodes[i] = nd;
  }
}

__device__ bool join_keys_equal(const JoinKeys& K, int64_t bi, int64_t pi);

static const int JP_BLOCK = 256;
static const int JP_STAGE = 128;  // staged pairs per warp

// MODE bit 0: emit pairs; bit 1: set probe_mark[j]; bit 2: set build_mark[i]
template <bool EXACT, int MODE>
__global__ void __launch_bounds__(JP_BLOCK) join_probe2_kernel(JoinKeys K, const JoinNode* __restrict__ nodes, const int32_t* __restrict__ heads, uint64_t mask,
                                                              const uint64_t* __restrict__ probe_hash, int64_t n_probe, unsigned long long* __restrict__ counter,
                                                              uint64_t cap, int64_t* __restrict__ out_b, int64_t* __restrict__ out_p,
                                                              uint8_t* __restrict__ probe_mark, uint8_t* __restrict__ build_mark) {
  __shared__ uint32_t st_b[JP_BLOCK / 32][JP_STAGE];
  __shared__ uint32_t st_p_lo[JP_BLOCK / 32][JP_STAGE];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  uint32_t staged = 0;  // warp-uniform
  int64_t stage_base_row = 0;
  auto flush = [&]() {
    if (staged == 0) return;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(counter, (unsigned long long)staged);
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    for (uint32_t k = lane; k < staged; k += 32) {
      const unsigned long long pos = base + k;
      if (pos < cap) {
        out_b[pos] = (int64_t)st_b[warp][k];
        out_p[pos] = stage_base_row + (int64_t)st_p_lo[warp][k];
      }
    }
    __syncwarp();
    staged = 0;
  };
  const int64_t stride = (int64_t)gridDim.x * JP_BLOCK;
  // warp-uniform trip count: every lane of a warp walks the loop together
  for (int64_t j0 = (int64_t)blockIdx.x * JP_BLOCK + warp * 32; j0 < n_probe; j0 += stride) {
    const int64_t j = j0 + lane;
    int32_t i = -1;
    uint64_t tag = 0;
    if (j < n_probe) {
      bool ok = true;
      if (EXACT) {
        ok = jkey_valid(K.probe[0], j);
        if (ok) tag = jkey_image(K.probe[0], j);
      } else {
        tag = probe_hash[j];
      }
      if (ok) i = heads[mix64(tag) & mask];
    }
    if (MODE & 1) {
      // staged probe rows are stored relative to the warp's first row of the current batch of staged pairs
      if (staged == 0) stage_base_row = j0;
    }
    bool any_hit = false;
    while (__any_sync(0xFFFFFFFFu, i >= 0)) {
      bool hit = false;
      int32_t cur = i;
      if (i >= 0) {
        const JoinNode nd = nodes[i];
        hit = nd.tag == tag && (EXACT || join_keys_equal(K, i, j));
        i = nd.next;
      }
      if (hit) {
        any_hit = true;
        if (MODE & 4) build_mark[cur] = 1;
      }
      if (MODE & 1) {
        const uint32_t hits = __ballot_sync(0xFFFFFFFFu, hit);
        if (hits) {
          if (staged + 32 > JP_STAGE || (uint64_t)(j0 + 31 - stage_base_row) > 0xFFFFFFFFull) {
            flush();
            stage_base_row = j0;
          }
          if (hit) {
            const uint32_t k = staged + __popc(hits & lt);
            st_b[warp][k] = (uint32_t)cur;
            st_p_lo[warp][k] = (uint32_t)(j - stage_base_row);
          }
          __syncwarp();
          staged += __popc(hits);
        }
      }
    }
    if ((MODE & 2) && j < n_probe && any_hit) probe_mark[j] = 1;
  }
  if (MODE & 1) flush();
}

template <bool EXACT>
static void launch_probe_mode(int mode, int grid, const JoinKeys& K, const JoinNode* nodes, const int32_t* heads, uint64_t mask, const uint64_t* probe_hash, int64_t n_probe,
                              unsigned long long* counter, uint64_t cap, int64_t* out_b, int64_t* out_p, uint8_t* probe_mark, uint8_t* build_mark, cudaStream_t st) {
#define JP_CASE(M)                                                                                                                                        \
  case M: launch_kernel(join_probe2_kernel<EXACT, M>, grid, JP_BLOCK, 0, st, K, nodes, heads, mask, probe_hash, n_probe, counter, cap, out_b, out_p, probe_mark, build_mark); break;
  switch (mode) {
    JP_CASE(1)
    JP_CASE(2)
    JP_CASE(3)
    JP_CASE(4)
    JP_CASE(5)
    JP_CASE(6)
    JP_CASE(7)
    default: break;
  }
#undef JP_CASE
}

void launch_join_build2(const JoinKeys& K, bool exact, const uint64_t* build_hash, int64_t n_build, int32_t* heads, uint64_t n_buckets, JoinNode* nodes, cudaStream_t st) {
  if (n_build <= 0) return;
  const int g = join_grid(n_build, 256, 4);
  if (exact) launch_kernel(join_build2_kernel<true>, g, 256, 0, st, K, build_hash, n_build, heads, n_buckets - 1, nodes);
  else launch_kernel(join_build2_kernel<false>, g, 256, 0, st, K, build_hash, n_build, heads, n_buckets - 1, nodes);
}

void launch_join_probe2(const JoinKeys& K, bool exact, int mode, const JoinNode* nodes, const int32_t* heads, uint64_t n_buckets, const uint64_t* probe_hash, int64_t n_probe,
                        unsigned long long* counter, uint64_t cap, int64_t* out_b, int64_t* out_p, uint8_t* probe_mark, uint8_t* build_mark, cudaStream_t st) {
  if (n_probe <= 0 || mode == 0) return;
  const int g = join_grid(n_probe, JP_BLOCK, 4);
  if (exact) launch_probe_mode<true>(mode, g, K, nodes, heads, n_buckets - 1, probe_hash, n_probe, counter, cap, out_b, out_p, probe_mark, build_mark, st);
  else launch_probe_mode<false>(mode, g, K, nodes, heads, n_buckets - 1, probe_hash, n_probe, counter, cap, out_b, out_p, probe_mark, build_mark, st);
}

// exact comparison of every key column of build row bi and probe row pi (hash-tagged tables).  Fixed-width keys compare
// their bytes: Float32 / Float64 keys are equal when their bit patterns are, as the engine's `=` has it (NaN = NaN with
// the same payload, -0.0 <> 0.0).  hash_f64 puts +-0.0 and every NaN in one bucket, which only costs a failed check.
__device__ bool join_keys_equal(const JoinKeys& K, int64_t bi, int64_t pi) {
  for (int k = 0; k < K.n_keys; k++) {
    const KeyCol& b = K.build[k];
    const KeyCol& p = K.probe[k];
    const bool bv = !b.valid || b.valid[bi], pv = !p.valid || p.valid[pi];
    if (!bv || !pv) {
      if (K.null_equals_null && !bv && !pv) continue;
      return false;
    }
    if (b.phys == PH_STRVIEW) {
      const unsigned long long* x = (const unsigned long long*)b.data + 2 * bi;
      const unsigned long long* y = (const unsigned long long*)p.data + 2 * pi;
      if (x[1] != y[1]) return false;
      const uint8_t *s = (const uint8_t*)x[0], *t = (const uint8_t*)y[0];
      for (uint32_t i = 0; i < (uint32_t)x[1]; i++)
        if (s[i] != t[i]) return false;
    } else {
      const uint8_t* x = (const uint8_t*)b.data + bi * b.width;
      const uint8_t* y = (const uint8_t*)p.data + pi * p.width;
      switch (b.width) {
        case 16:
          if (((const uint64_t*)x)[0] != ((const uint64_t*)y)[0] || ((const uint64_t*)x)[1] != ((const uint64_t*)y)[1]) return false;
          break;
        case 8:
          if (*(const uint64_t*)x != *(const uint64_t*)y) return false;
          break;
        case 4:
          if (*(const uint32_t*)x != *(const uint32_t*)y) return false;
          break;
        case 2:
          if (*(const uint16_t*)x != *(const uint16_t*)y) return false;
          break;
        default:
          if (*x != *y) return false;
      }
    }
  }
  return true;
}

}  // namespace b200
