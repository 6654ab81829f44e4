// Row hash used for (a) hash repartitioning in the shuffle writer and (b) group-by / join tables.
//
// Reference rule being restated (ballista/core/src/execution_plans/sort_shuffle/writer.rs:729-749,
// shuffle_writer.rs:284-291): per row, h = create_hashes(key columns, REPARTITION_RANDOM_STATE);
// partition = h % P.  `create_hashes` [EXT, datafusion-common 53.1 hash_utils.rs] sets the hash
// from the first key column and folds each further column with
//     combine_hashes(l, r) = (17*37 + l)*37 + r        (wrapping u64)
// leaving the running hash unchanged for NULL values.  The per-value hash there is ahash 0.8.12
// with fixed seeds, whose bit pattern depends on compile-time CPU features (AES vs fallback) and
// is asserted by no test in the reference (SURVEY.md §8(c) "not pinned" (ii)); results never
// depend on it, only on every writer of one shuffle agreeing.  We therefore define a
// GPU-friendly per-value hash (splitmix64 finaliser) and keep the *structure* (first column sets,
// later columns combine, NULL skips, `% P`).  The same header is compiled for host and device so
// the CPU oracle and the CUDA kernels agree bit for bit; tests/test_hash.py pins it with an
// independent numpy restatement and known answers.
#pragma once
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define B200_HD __host__ __device__ __forceinline__
#else
#define B200_HD inline
#endif

namespace b200 {

B200_HD uint64_t mix64(uint64_t x) {
  x ^= x >> 30;
  x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27;
  x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return x;
}

static const uint64_t kHashSeed = 0x9E3779B97F4A7C15ull;

B200_HD uint64_t hash_i64(int64_t v) { return mix64((uint64_t)v + kHashSeed); }

B200_HD uint64_t hash_f64(double d) {
  if (d == 0.0) d = 0.0;  // -0.0 == 0.0 must hash alike
  uint64_t bits;
#if defined(__CUDA_ARCH__)
  bits = (uint64_t)__double_as_longlong(d);
#else
  memcpy(&bits, &d, 8);
#endif
  if (d != d) bits = 0x7ff8000000000000ull;  // canonical NaN
  return mix64(bits + kHashSeed);
}

// Float32 <-> Float64 that keep every bit of a Float32, for group keys and MIN / MAX, which must give back the input's
// bits.  The hardware widening sets a signalling NaN's quiet bit (0x7F800001 and 0x7FC00001 would both become
// 0x7FF8000020000000), so a NaN is widened from its bits: sign, all-ones exponent, the 23 payload bits on top of the 52.
// The narrowing is its inverse; a NaN whose top 23 payload bits are zero (made by Float64 arithmetic, not by a widened
// Float32) narrows as the hardware does.  The widening keeps the IEEE total order of the Float32 bit patterns.
B200_HD uint64_t f32_bits_to_f64_bits(uint32_t b) {
  const uint32_t a = b & 0x7FFFFFFFu;
  if (a > 0x7F800000u) return ((uint64_t)(b >> 31) << 63) | 0x7FF0000000000000ull | ((uint64_t)(a & 0x7FFFFFu) << 29);
  float f;
  double d;
  uint64_t r;
  memcpy(&f, &b, 4);
  d = (double)f;
  memcpy(&r, &d, 8);
  return r;
}
B200_HD uint32_t f64_bits_to_f32_bits(uint64_t b) {
  const uint32_t pay = (uint32_t)(b >> 29) & 0x7FFFFFu;
  if ((b & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull && pay) return ((uint32_t)(b >> 63) << 31) | 0x7F800000u | pay;
  double d;
  float f;
  uint32_t r;
  memcpy(&d, &b, 8);
  f = (float)d;
  memcpy(&r, &f, 4);
  return r;
}

B200_HD uint64_t hash_i128(uint64_t lo, uint64_t hi) {
  // values that fit in 64 bits (sign-extended) hash like the same i64
  if ((int64_t)hi == ((int64_t)lo >> 63)) return hash_i64((int64_t)lo);
  return mix64(lo ^ mix64(hi + 0xD1B54A32D192ED03ull));
}

B200_HD uint64_t hash_bytes(const uint8_t* p, uint32_t len) {
  uint64_t h = kHashSeed ^ ((uint64_t)len * 0xFF51AFD7ED558CCDull);
  uint32_t i = 0;
  for (; i + 8 <= len; i += 8) {
    uint64_t w = 0;
    for (int k = 0; k < 8; k++) w |= (uint64_t)p[i + k] << (8 * k);
    h = mix64(h ^ w);
  }
  if (i < len) {
    uint64_t w = 0;
    for (int k = 0; i + k < len; k++) w |= (uint64_t)p[i + k] << (8 * k);
    h = mix64(h ^ w ^ 0x8000000000000000ull);
  }
  return mix64(h);
}

B200_HD uint64_t combine_hashes(uint64_t l, uint64_t r) { return (17ull * 37ull + l) * 37ull + r; }

}  // namespace b200
