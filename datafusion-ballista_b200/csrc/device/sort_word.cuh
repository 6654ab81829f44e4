// Order-preserving 64-bit words of one sort key: the device sort (sort_word_kernel, kernels.cu) and the first_value /
// last_value passes of the pipeline kernel (pipeline.cu) encode with these functions, so both follow one set of rules.
//  - the NULL-rank word (most significant, only for a nullable key) decides where NULLs go;
//  - value words: integers one word (sign bit flipped for signed ones), floats one word in the IEEE total order
//    (-0.0 before +0.0, NaN greatest), Decimal128 two (the signed high word, then the low one), strings 7 bytes per word
//    plus one byte that counts the bytes present (8 = continues), so that a proper prefix comes first.
//  A descending key inverts its value words; the NULL-rank word is not affected by the direction.
#pragma once
#include <stdint.h>

#include "program.h"  // SortWordKind

namespace b200 {

__device__ __forceinline__ uint64_t sort_null_word(bool valid, bool nulls_first) { return valid ? (nulls_first ? 1 : 0) : (nulls_first ? 0 : 1); }

// value word `word` of a non-NULL value
__device__ __forceinline__ uint64_t sort_value_word(int kind, uint64_t lo, uint64_t hi, int word, bool asc) {
  uint64_t w = 0;
  switch (kind) {
    case SWK_INT: w = lo ^ 0x8000000000000000ull; break;
    case SWK_UINT: w = lo; break;
    case SWK_F64: {
      // raw bits as an INTEGER: if the compiler sees a double here it turns `bits ^ signbit` into an FP negate, and
      // neg.f64 of a NaN does not return the sign-flipped bit pattern (NaN keys were ordered below -0.0); found by
      // tests/test_gpu_sort.py
      long long x = (long long)lo;
      asm volatile("" : "+l"(x));
      x ^= (long long)((unsigned long long)(x >> 63) >> 1);  // IEEE total order
      w = (uint64_t)x ^ 0x8000000000000000ull;
      break;
    }
    case SWK_DEC128: w = word == 0 ? (hi ^ 0x8000000000000000ull) : lo; break;  // word 0 = high (signed), word 1 = low
    case SWK_STR: {
      const uint8_t* s = (const uint8_t*)lo;
      const uint32_t len = (uint32_t)hi;
      const uint32_t base = (uint32_t)word * 7;  // 7 data bytes per word + 1 "has more/len" byte keeps prefixes ordered
      for (int b = 0; b < 7; b++) {
        const uint32_t p = base + b;
        w = (w << 8) | (p < len ? s[p] : 0);
      }
      const uint32_t rem = len > base ? len - base : 0;
      w = (w << 8) | (rem > 7 ? 8 : rem);  // bytes present in this word (8 = continues)
      break;
    }
    default: break;
  }
  return asc ? w : ~w;
}

}  // namespace b200
