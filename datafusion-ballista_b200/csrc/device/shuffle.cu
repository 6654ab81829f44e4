// Shuffle-side CUDA kernels (sm_90a): one-pass stable radix partition (ShuffleWriterExec /
// SortShuffleWriterExec), the exchange message packer, and the small-result export packer.
//
// Reference behaviour being reproduced:
//   * BatchPartitioner::partition / compute_partition_indices -- rows go to partition hash % P and keep
//     their input order inside a partition (ballista/core/src/execution_plans/sort_shuffle/writer.rs:729-749,
//     shuffle_writer.rs:291-343); here: per-tile histogram -> exclusive scan in partition-major order ->
//     per-tile stable ranks (warp match + per-warp running counters) -> every column scattered in the same
//     kernel.  HBM bound: 2 * N * w_row algorithmic bytes (+ 4 B/row of partition ids read twice).
//   * the per-partition IPC writers (shuffle_writer.rs:317-328): replaced by packing the column slices of
//     every (destination, partition) into one contiguous message (exchange_pack_kernel).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "../common/hash.hpp"
#include "kernels.h"
#include "keyimg.cuh"

namespace b200 {

static const int PT_BLOCK = 256;                      // 8 warps
static const int PT_WARPS = PT_BLOCK / 32;
static const int PT_ROUNDS = 8;                       // rows per thread
static const int PT_TILE = PT_BLOCK * PT_ROUNDS;      // 2048 rows per tile; warp w owns rows [w*256, (w+1)*256)

__device__ __forceinline__ uint32_t pid_of(const PidSrc& ps, int64_t i, uint32_t P) {
  if (ps.pid) return ps.pid[i];
  if (ps.n_keys == 0) return 0u;
  uint64_t h = jkey_valid(ps.keys[0], i) ? hash_i64((int64_t)jkey_image(ps.keys[0], i)) : 0ull;
  for (int k = 1; k < ps.n_keys; k++)
    if (jkey_valid(ps.keys[k], i)) h = combine_hashes(hash_i64((int64_t)jkey_image(ps.keys[k], i)), h);
  if (ps.salt) h = mix64(h ^ ((uint64_t)(uint32_t)ps.salt * 0xD1B54A32D192ED03ull));
  return (uint32_t)(h % (uint64_t)P);
}

__device__ __forceinline__ uint32_t str_len_of(const PartStrCol& c, int64_t i) {
  if (c.valid && !c.valid[i]) return 0u;
  if (c.is_view) return (uint32_t)((const unsigned long long*)c.data)[2 * i + 1];
  const int32_t* o = (const int32_t*)c.data;
  return (uint32_t)(o[i + 1] - o[i]);
}

// tile_hist[p * n_tiles + tile] = rows of partition p in the tile; counts[p] += the same;
// str_bytes[c * P + p] += string bytes of column c that go to partition p (ShuffleWritePartition.num_bytes)
__global__ void __launch_bounds__(PT_BLOCK) part_tile_hist_kernel(const PidSrc pid, int64_t n, uint32_t P, uint32_t n_tiles, uint32_t* __restrict__ tile_hist,
                                                                 unsigned long long* __restrict__ counts, PartStrCols sc, unsigned long long* __restrict__ str_bytes) {
  extern __shared__ unsigned int sh[];  // [P] counts, then [n_str][P] byte sums (as 2 x u32: lo/hi not needed: < 2^32 per tile)
  const int n_str = sc.n;
  for (uint32_t b = threadIdx.x; b < P * (1 + n_str); b += PT_BLOCK) sh[b] = 0;
  __syncthreads();
  const int64_t t0 = (int64_t)blockIdx.x * PT_TILE;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++) {
    const int64_t i = t0 + warp * (PT_TILE / PT_WARPS) + r * 32 + lane;
    if (i < n) {
      const uint32_t p = pid_of(pid, i, P);
      atomicAdd(&sh[p], 1u);
      for (int c = 0; c < n_str; c++) {
        const uint32_t len = str_len_of(sc.c[c], i);
        if (len) atomicAdd(&sh[P * (1 + c) + p], len);
      }
    }
  }
  __syncthreads();
  for (uint32_t p = threadIdx.x; p < P; p += PT_BLOCK) {
    const unsigned int v = sh[p];
    if (tile_hist) tile_hist[(size_t)p * n_tiles + blockIdx.x] = v;
    if (v) atomicAdd(&counts[p], (unsigned long long)v);
    for (int c = 0; c < n_str; c++) {
      const unsigned int bts = sh[P * (1 + c) + p];
      if (bts) atomicAdd(&str_bytes[(size_t)c * P + p], (unsigned long long)bts);
    }
  }
}

template <typename T>
__device__ __forceinline__ void scatter_rows(const GatherCol& c, const int64_t (&row)[PT_ROUNDS], const uint32_t (&dst)[PT_ROUNDS], const uint32_t (&p)[PT_ROUNDS],
                                             int64_t n) {
  const T* __restrict__ in = (const T*)c.in;
  T* __restrict__ out = (T*)c.out;
  T v[PT_ROUNDS];
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++)
    if (row[r] < n) v[r] = in[row[r]];
  if (c.part_base) {
    // per-partition destination bases (possibly peer memory): generic stores, NVLink carries the remote ones
#pragma unroll
    for (int r = 0; r < PT_ROUNDS; r++)
      if (row[r] < n) ((T*)c.part_base[p[r]])[dst[r]] = v[r];
    return;
  }
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++)
    if (row[r] < n) out[dst[r]] = v[r];
}

// offsets[p * n_tiles + tile] = first output row of (partition p, tile); the rank of a row inside its
// (p, tile) group is its stable position: rows of earlier warps, earlier rounds, lower lanes first.
__global__ void __launch_bounds__(PT_BLOCK) part_tile_scatter_kernel(const PidSrc pid, int64_t n, uint32_t P, uint32_t n_tiles,
                                                                    const uint64_t* __restrict__ offsets, GatherCols cols, uint32_t* __restrict__ dest_out) {
  extern __shared__ unsigned int sh[];  // [PT_WARPS][P] per-warp counts -> per-warp bases
  for (uint32_t b = threadIdx.x; b < P * PT_WARPS; b += PT_BLOCK) sh[b] = 0;
  __syncthreads();
  const int64_t t0 = (int64_t)blockIdx.x * PT_TILE;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned int* mine = sh + (size_t)warp * P;
  uint32_t p[PT_ROUNDS];
  int64_t row[PT_ROUNDS];
  uint32_t rank[PT_ROUNDS];
  const uint32_t lt = (1u << lane) - 1u;
  // pass 1: rank inside the warp's 256 rows (round-major, lane-minor == input order) and per-warp counts
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++) {
    row[r] = t0 + warp * (PT_TILE / PT_WARPS) + r * 32 + lane;
    const bool live = row[r] < n;
    p[r] = live ? pid_of(pid, row[r], P) : 0xFFFFFFFFu;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, p[r]);
    uint32_t base = 0;
    if (live) base = mine[p[r]];
    __syncwarp();
    rank[r] = base + __popc(peers & lt);
    if (live && (peers & lt) == 0) mine[p[r]] = base + __popc(peers);  // the lowest lane of each group advances the counter
    __syncwarp();
  }
  __syncthreads();
  // per partition: exclusive scan of the warp counts, seeded with the (partition, tile) output offset
  for (uint32_t q = threadIdx.x; q < P; q += PT_BLOCK) {
    uint64_t run = offsets[(size_t)q * n_tiles + blockIdx.x];
#pragma unroll
    for (int w = 0; w < PT_WARPS; w++) {
      const unsigned int c = sh[(size_t)w * P + q];
      sh[(size_t)w * P + q] = (unsigned int)run;  // < 2^32 rows per task (checked by the host)
      run += c;
    }
  }
  __syncthreads();
  uint32_t dst[PT_ROUNDS];
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++) dst[r] = row[r] < n ? mine[p[r]] + rank[r] : 0u;
  if (dest_out) {
#pragma unroll
    for (int r = 0; r < PT_ROUNDS; r++)
      if (row[r] < n) dest_out[row[r]] = dst[r];
  }
  for (int c = 0; c < cols.n; c++) {
    const GatherCol& gc = cols.c[c];
    switch (gc.width) {
      case 1: scatter_rows<uint8_t>(gc, row, dst, p, n); break;
      case 2: scatter_rows<uint16_t>(gc, row, dst, p, n); break;
      case 4: scatter_rows<uint32_t>(gc, row, dst, p, n); break;
      case 8: scatter_rows<uint64_t>(gc, row, dst, p, n); break;
      default: scatter_rows<ulonglong2>(gc, row, dst, p, n); break;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Staged variant (fan-out <= PT_STAGED_MAX_P): the tile's rows are first put in partition-major order in shared memory,
// then written out by consecutive threads -- every (tile, partition) group leaves the SM as one contiguous run (full
// 128-byte store instructions, whole sectors / maximum-size NVLink packets) instead of one 4..16-row fragment per
// warp round.  Used for the fused shuffle, whose remote stores pay per packet, not per byte.
// Shared memory: [PT_WARPS][P] warp bases | seed[P] (first output row of (p, tile) minus its first slot) | start[P + 1]
// (first slot of p) | part[PT_TILE] (uint16 partition of every slot) | val[PT_TILE] x 16 bytes.
// ------------------------------------------------------------------------------------------------
static const uint32_t PT_STAGED_MAX_P = 256;

template <typename T>
__device__ __forceinline__ void staged_column(const GatherCol& c, const int64_t (&row)[PT_ROUNDS], const uint32_t (&slot)[PT_ROUNDS], int64_t n, int tile_rows,
                                              const long long* seed, const unsigned short* part, T* val) {
  const T* __restrict__ in = (const T*)c.in;
  T v[PT_ROUNDS];
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++)
    if (row[r] < n) v[r] = in[row[r]];
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++)
    if (row[r] < n) val[slot[r]] = v[r];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < PT_ROUNDS; k++) {
    const int i = k * PT_BLOCK + (int)threadIdx.x;
    if (i < tile_rows) {
      const unsigned int q = part[i];
      const long long d = seed[q] + i;  // output row of slot i inside partition q's numbering
      T* o = c.part_base ? (T*)c.part_base[q] : (T*)c.out;
      o[d] = val[i];
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(PT_BLOCK) part_tile_scatter_staged_kernel(const PidSrc pid, int64_t n, uint32_t P, uint32_t n_tiles,
                                                                           const uint64_t* __restrict__ offsets, GatherCols cols) {
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned int* sh = (unsigned int*)smem;                            // [PT_WARPS][P]
  long long* seed = (long long*)(sh + (size_t)PT_WARPS * P + (((size_t)PT_WARPS * P) & 1));  // [P], 8-byte aligned
  unsigned int* start = (unsigned int*)(seed + P);                   // [P + 1]
  unsigned short* part = (unsigned short*)(start + P + 1 + ((P + 1) & 1));
  unsigned char* val = (unsigned char*)(((uintptr_t)(part + PT_TILE) + 15) & ~(uintptr_t)15);
  __shared__ unsigned int warp_tot[PT_WARPS];
  for (uint32_t b = threadIdx.x; b < P * PT_WARPS; b += PT_BLOCK) sh[b] = 0;
  __syncthreads();
  const int64_t t0 = (int64_t)blockIdx.x * PT_TILE;
  const int tile_rows = (int)min((int64_t)PT_TILE, n - t0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned int* mine = sh + (size_t)warp * P;
  uint32_t p[PT_ROUNDS];
  int64_t row[PT_ROUNDS];
  uint32_t rank[PT_ROUNDS];
  const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++) {
    row[r] = t0 + warp * (PT_TILE / PT_WARPS) + r * 32 + lane;
    const bool live = row[r] < n;
    p[r] = live ? pid_of(pid, row[r], P) : 0xFFFFFFFFu;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, p[r]);
    uint32_t base = 0;
    if (live) base = mine[p[r]];
    __syncwarp();
    rank[r] = base + __popc(peers & lt);
    if (live && (peers & lt) == 0) mine[p[r]] = base + __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  // per partition: rows of this tile, then an exclusive scan over the partitions (P <= 256: one value per thread)
  unsigned int cnt = 0;
  if (threadIdx.x < P) {
#pragma unroll
    for (int w = 0; w < PT_WARPS; w++) {
      const unsigned int c = sh[(size_t)w * P + threadIdx.x];
      sh[(size_t)w * P + threadIdx.x] = cnt;  // warp w's first slot inside the partition's group
      cnt += c;
    }
  }
  unsigned int incl = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned int o = __shfl_up_sync(0xFFFFFFFFu, incl, d);
    if (lane >= d) incl += o;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  unsigned int before = 0;
  for (int w = 0; w < warp; w++) before += warp_tot[w];
  if (threadIdx.x < P) {
    const unsigned int first = before + incl - cnt;  // first slot of this partition in the tile
    start[threadIdx.x] = first;
    seed[threadIdx.x] = (long long)offsets[(size_t)threadIdx.x * n_tiles + blockIdx.x] - (long long)first;
  }
  __syncthreads();
  uint32_t slot[PT_ROUNDS];
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++) {
    slot[r] = row[r] < n ? start[p[r]] + mine[p[r]] + rank[r] : 0u;
    if (row[r] < n) part[slot[r]] = (unsigned short)p[r];
  }
  __syncthreads();
  for (int c = 0; c < cols.n; c++) {
    const GatherCol& gc = cols.c[c];
    switch (gc.width) {
      case 1: staged_column<uint8_t>(gc, row, slot, n, tile_rows, seed, part, (uint8_t*)val); break;
      case 2: staged_column<uint16_t>(gc, row, slot, n, tile_rows, seed, part, (uint16_t*)val); break;
      case 4: staged_column<uint32_t>(gc, row, slot, n, tile_rows, seed, part, (uint32_t*)val); break;
      case 8: staged_column<uint64_t>(gc, row, slot, n, tile_rows, seed, part, (uint64_t*)val); break;
      default: staged_column<ulonglong2>(gc, row, slot, n, tile_rows, seed, part, (ulonglong2*)val); break;
    }
  }
}

// Warp-staged variant (fan-out <= 32): no CTA barrier in the column loop.  Every warp puts ITS 256 rows in partition-major
// order in a private 4 KB slice of shared memory and writes them out with consecutive lanes: runs of 256 / P rows per
// partition (P = 8: 32 rows = one full store instruction, 256..512 bytes) instead of 32 / P rows per warp round.
// Lane q keeps partition q's numbers (first slot of the group, first output row of the group) and hands them out by shuffle.
template <typename T>
__device__ __forceinline__ void wstaged_column(const GatherCol& c, const int64_t (&row)[PT_ROUNDS], const uint32_t (&slot)[PT_ROUNDS], int64_t n, int warp_rows,
                                               long long delta_mine, const unsigned char* part, T* val, int lane) {
  const T* __restrict__ in = (const T*)c.in;
  T v[PT_ROUNDS];
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++)
    if (row[r] < n) v[r] = in[row[r]];
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++)
    if (row[r] < n) val[slot[r]] = v[r];
  __syncwarp();
#pragma unroll
  for (int k = 0; k < PT_ROUNDS; k++) {
    const int i = k * 32 + lane;
    const unsigned int q = i < warp_rows ? part[i] : 0u;
    const long long d = __shfl_sync(0xFFFFFFFFu, delta_mine, (int)q) + i;  // output row of slot i
    if (i < warp_rows) {
      T* o = c.part_base ? (T*)c.part_base[q] : (T*)c.out;
      o[d] = val[i];
    }
  }
  __syncwarp();
}

__global__ void __launch_bounds__(PT_BLOCK) part_tile_scatter_wstaged_kernel(const PidSrc pid, int64_t n, uint32_t P, uint32_t n_tiles,
                                                                            const uint64_t* __restrict__ offsets, GatherCols cols) {
  __shared__ unsigned int sh[PT_WARPS][32];                                  // per-warp counts -> per-warp first output rows
  __shared__ unsigned long long gbase[PT_WARPS][32];
  __shared__ unsigned char part_s[PT_WARPS][PT_TILE / PT_WARPS];
  __shared__ __align__(16) unsigned char val_s[PT_WARPS][(PT_TILE / PT_WARPS) * 16];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  sh[warp][lane] = 0;
  __syncwarp();
  const int64_t t0 = (int64_t)blockIdx.x * PT_TILE;
  const int64_t w0 = t0 + warp * (PT_TILE / PT_WARPS);
  const int warp_rows = (int)max((int64_t)0, min((int64_t)(PT_TILE / PT_WARPS), n - w0));
  unsigned int* mine = sh[warp];
  uint32_t p[PT_ROUNDS];
  int64_t row[PT_ROUNDS];
  uint32_t rank[PT_ROUNDS];
  const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++) {
    row[r] = w0 + r * 32 + lane;
    const bool live = row[r] < n;
    p[r] = live ? pid_of(pid, row[r], P) : 0xFFFFFFFFu;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, p[r]);
    uint32_t base = 0;
    if (live) base = mine[p[r]];
    __syncwarp();
    rank[r] = base + __popc(peers & lt);
    if (live && (peers & lt) == 0) mine[p[r]] = base + __popc(peers);
    __syncwarp();
  }
  // lane q: this warp's rows of partition q, and the first slot of that group in the warp's partition-major order
  const unsigned int cnt = mine[lane];
  unsigned int incl = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned int o = __shfl_up_sync(0xFFFFFFFFu, incl, d);
    if (lane >= d) incl += o;
  }
  const unsigned int wstart = incl - cnt;
  __syncthreads();
  // first output row of (partition, tile, warp): the tile's offset plus the earlier warps' rows
  if (threadIdx.x < P) {
    unsigned long long run = offsets[(size_t)threadIdx.x * n_tiles + blockIdx.x];
#pragma unroll
    for (int w = 0; w < PT_WARPS; w++) {
      gbase[w][threadIdx.x] = run;
      run += sh[w][threadIdx.x];
    }
  }
  __syncthreads();
  const long long delta_mine = (uint32_t)lane < P ? (long long)gbase[warp][lane] - (long long)wstart : 0ll;
  uint32_t slot[PT_ROUNDS];
#pragma unroll
  for (int r = 0; r < PT_ROUNDS; r++) {
    const unsigned int ws = __shfl_sync(0xFFFFFFFFu, wstart, (int)(p[r] & 31u));
    slot[r] = row[r] < n ? ws + rank[r] : 0u;
    if (row[r] < n) part_s[warp][slot[r]] = (unsigned char)p[r];
  }
  __syncwarp();
  for (int c = 0; c < cols.n; c++) {
    const GatherCol& gc = cols.c[c];
    switch (gc.width) {
      case 1: wstaged_column<uint8_t>(gc, row, slot, n, warp_rows, delta_mine, part_s[warp], (uint8_t*)val_s[warp], lane); break;
      case 2: wstaged_column<uint16_t>(gc, row, slot, n, warp_rows, delta_mine, part_s[warp], (uint16_t*)val_s[warp], lane); break;
      case 4: wstaged_column<uint32_t>(gc, row, slot, n, warp_rows, delta_mine, part_s[warp], (uint32_t*)val_s[warp], lane); break;
      case 8: wstaged_column<uint64_t>(gc, row, slot, n, warp_rows, delta_mine, part_s[warp], (uint64_t*)val_s[warp], lane); break;
      default: wstaged_column<ulonglong2>(gc, row, slot, n, warp_rows, delta_mine, part_s[warp], (ulonglong2*)val_s[warp], lane); break;
    }
  }
}

static size_t partition_scatter_staged_smem(uint32_t P) {
  return ((size_t)PT_WARPS * P + 1) * 4 + (size_t)P * 8 + ((size_t)P + 2) * 4 + (size_t)PT_TILE * 2 + 16 + (size_t)PT_TILE * 16;
}

size_t partition_scatter_smem(uint32_t P) { return (size_t)P * PT_WARPS * sizeof(unsigned int); }
uint32_t partition_n_tiles(int64_t n) { return (uint32_t)((n + PT_TILE - 1) / PT_TILE); }

cudaError_t launch_partition_hist(const PidSrc& pid, int64_t n, uint32_t P, uint32_t* tile_hist, unsigned long long* counts, const PartStrCols& sc,
                                  unsigned long long* str_bytes, cudaStream_t st) {
  const uint32_t nt = partition_n_tiles(n);
  if (nt == 0) return cudaSuccess;
  const size_t sm = (size_t)P * (1 + sc.n) * sizeof(unsigned int);
  if (sm > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(part_tile_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    if (e != cudaSuccess) return e;
  }
  launch_kernel(part_tile_hist_kernel, nt, PT_BLOCK, sm, st, pid, n, P, nt, tile_hist, counts, sc, str_bytes);
  return cudaGetLastError();
}

cudaError_t launch_partition_scatter(const PidSrc& pid, int64_t n, uint32_t P, const uint64_t* offsets, const GatherCols& cols, uint32_t* dest_out,
                                     cudaStream_t st) {
  const uint32_t nt = partition_n_tiles(n);
  if (nt == 0) return cudaSuccess;
  bool peer = false;
  for (int c = 0; c < cols.n; c++) peer = peer || cols.c[c].part_base != nullptr;
  static const int force_staged = getenv("B200_SCATTER_STAGED") ? atoi(getenv("B200_SCATTER_STAGED")) : -1;  // measurement switch
  if (!dest_out && P <= 32 && (force_staged == 1 || (force_staged != 0 && peer))) {
    launch_kernel(part_tile_scatter_wstaged_kernel, nt, PT_BLOCK, 0, st, pid, n, P, nt, offsets, cols);
    return cudaGetLastError();
  }
  if (!dest_out && P <= PT_STAGED_MAX_P && (force_staged == 1 || (force_staged != 0 && peer))) {
    const size_t sm = partition_scatter_staged_smem(P);
    static bool attr_set = false;
    if (!attr_set) {
      cudaError_t e = cudaFuncSetAttribute(part_tile_scatter_staged_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)partition_scatter_staged_smem(PT_STAGED_MAX_P));
      if (e != cudaSuccess) return e;
      attr_set = true;
    }
    launch_kernel(part_tile_scatter_staged_kernel, nt, PT_BLOCK, sm, st, pid, n, P, nt, offsets, cols);
    return cudaGetLastError();
  }
  const size_t sm = partition_scatter_smem(P);
  if (sm > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(part_tile_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    if (e != cudaSuccess) return e;
  }
  launch_kernel(part_tile_scatter_kernel, nt, PT_BLOCK, sm, st, pid, n, P, nt, offsets, cols, dest_out);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Pack jobs: copy / convert column slices into a contiguous destination (exchange messages, small exports)
// ------------------------------------------------------------------------------------------------
// One CTA per job.  PK_COPY: plain bytes.  PK_BITMAP: validity bytes -> bitmap + null count.  PK_STR_VIEWS / PK_STR_UTF8: write `rows + 1` int32 offsets starting
// at 0 to dst and the character bytes to dst2 (block-wide running prefix sum over chunks of 256 rows).
__global__ void __launch_bounds__(256) pack_jobs_kernel(const PackJob* __restrict__ jobs, int n_jobs) {
  const int j = blockIdx.x;
  if (j >= n_jobs) return;
  const PackJob J = jobs[j];
  const int tid = threadIdx.x;
  if (J.kind == PK_COPY) {
    const uint8_t* s = (const uint8_t*)J.src;
    uint8_t* d = (uint8_t*)J.dst;
    if ((((uintptr_t)s | (uintptr_t)d) & 15) == 0) {
      const uint64_t n16 = J.bytes / 16;
      for (uint64_t k = tid; k < n16; k += 256) ((uint4*)d)[k] = ((const uint4*)s)[k];
      for (uint64_t k = n16 * 16 + tid; k < J.bytes; k += 256) d[k] = s[k];
    } else {
      for (uint64_t k = tid; k < J.bytes; k += 256) d[k] = s[k];
    }
    return;
  }
  if (J.kind == PK_UTF8_VIEWS) {
    // Arrow offsets + characters -> 16-byte views {pointer, length} (the layout intermediate batches carry)
    const int32_t* o = (const int32_t*)J.src;
    unsigned long long* v = (unsigned long long*)J.dst;
    for (int64_t i = tid; i < J.rows; i += 256) {
      const int32_t o0 = o[i], o1 = o[i + 1];
      v[2 * i] = (unsigned long long)(J.chars + o0);
      v[2 * i + 1] = (unsigned long long)(uint32_t)(o1 - o0);
    }
    return;
  }
  if (J.kind == PK_BITMAP) {
    // byte-per-value -> Arrow bitmap (+ number of zero values at dst2, if asked for)
    const uint8_t* s = (const uint8_t*)J.src;
    uint8_t* d = (uint8_t*)J.dst;
    const int64_t nbytes = (J.rows + 7) / 8;
    unsigned int zeros = 0;
    for (int64_t b = tid; b < nbytes; b += 256) {
      uint8_t v = 0;
      for (int k = 0; k < 8; k++) {
        const int64_t i = b * 8 + k;
        if (i < J.rows) {
          if (s[i]) v |= (uint8_t)(1u << k);
          else zeros++;
        }
      }
      d[b] = v;
    }
    if (J.dst2) {
      __shared__ unsigned int zsum;
      if (tid == 0) zsum = 0;
      __syncthreads();
      if (zeros) atomicAdd(&zsum, zeros);
      __syncthreads();
      if (tid == 0) *(unsigned long long*)J.dst2 = zsum;
    }
    return;
  }
  __shared__ uint32_t warp_sum[8];
  __shared__ uint32_t carry_sh;
  if (tid == 0) carry_sh = 0;
  __syncthreads();
  int32_t* off_out = (int32_t*)J.dst;
  uint8_t* ch_out = (uint8_t*)J.dst2;
  const int lane = tid & 31, warp = tid >> 5;
  for (int64_t r0 = 0; r0 < J.rows; r0 += 256) {
    const int64_t i = r0 + tid;
    uint32_t len = 0;
    const uint8_t* sp = nullptr;
    if (i < J.rows && !(J.valid && !J.valid[i])) {
      if (J.kind == PK_STR_VIEWS) {
        sp = (const uint8_t*)((const unsigned long long*)J.src)[2 * i];
        len = (uint32_t)((const unsigned long long*)J.src)[2 * i + 1];
      } else {
        const int32_t* o = (const int32_t*)J.src;
        sp = J.chars + o[i];
        len = (uint32_t)(o[i + 1] - o[i]);
      }
    }
    uint32_t inc = len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, inc, o);
      if (lane >= o) inc += v;
    }
    if (lane == 31) warp_sum[warp] = inc;
    __syncthreads();
    uint32_t base = carry_sh;
    for (int w = 0; w < warp; w++) base += warp_sum[w];
    const uint32_t excl = base + inc - len;
    if (i < J.rows) {
      off_out[i] = (int32_t)excl;
      if ((uint64_t)excl + len <= J.bytes)  // J.bytes = capacity of the character area (the host re-checks the total)
        for (uint32_t k = 0; k < len; k++) ch_out[excl + k] = sp[k];
    }
    __syncthreads();
    if (tid == 255) carry_sh = base + inc;
    __syncthreads();
  }
  if (tid == 0) off_out[J.rows] = (int32_t)carry_sh;
}

void launch_pack_jobs(const PackJob* jobs_dev, int n_jobs, cudaStream_t st) {
  if (n_jobs <= 0) return;
  launch_kernel(pack_jobs_kernel, n_jobs, 256, 0, st, jobs_dev, n_jobs);
}

}  // namespace b200
