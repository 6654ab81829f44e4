// Fused pipeline kernel for sm_90a:  scan -> [FilterExec | ProjectionExec]* -> sink
// (sink = materialise/compact | partial-or-final hash aggregate).
//
// Reference operators replaced (SURVEY.md 8(a) R9a-R9c): DataFusion FilterExec, ProjectionExec and
// AggregateExec pulled by the shuffle writers at ballista/core/src/execution_plans/
// shuffle_writer.rs:218 and sort_shuffle/writer.rs:214.  The CPU path evaluates each PhysicalExpr
// column-at-a-time over 8192-row batches and materialises every intermediate array; here one
// persistent CTA per SM streams column tiles HBM -> shared memory with 1-D TMA bulk copies
// (cp.async.bulk + mbarrier, multi-stage ring), evaluates the whole expression program on the
// resident tile (values never leave the SM) and folds rows straight into the sink.
//
// HBM traffic per row == the Arrow bytes of the referenced columns, once (SURVEY.md 8(d)
// "fused scan->filter->project->partial-agg": N*w_referenced + G*(w_keys+w_state)).
//
// Code-size discipline (the first version thrashed the instruction cache, profiles/r01_*):
//  * the pipeline program lives in __constant__ memory: descriptors are read through the constant
//    cache / uniform datapath, never through generic pointers;
//  * hot operations are register-blocked over the thread's VM_R rows with tiny bodies;
//  * everything else (division, casts, LIKE, string compares, generic group keys) runs in rolled
//    per-row __noinline__ paths that exist once in the binary.
#include <cuda_runtime.h>

#include <mutex>
#include <stdint.h>

#include "../common/hash.hpp"
#include "../common/regex_dfa.hpp"
#include "kernels.h"
#include "program.h"

namespace b200 {

typedef __int128 i128;
typedef unsigned __int128 u128;

__constant__ Program c_prog;  // the running pipeline (one at a time per device; set on the launch stream)
__constant__ FusedSpec c_fused;  // fused fast-path description (when the program matches the q1/q6 shape)
#define PROG c_prog

// ------------------------------------------------------------------------------------------------
// PTX wrappers: mbarrier + 1-D bulk async copy (TMA without a tensor map; SASS: UBLKCP / SYNCS)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ------------------------------------------------------------------------------------------------
// 128-bit helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ i128 make_i128(uint64_t lo, uint64_t hi) { return (i128)(((u128)hi << 64) | (u128)lo); }
__device__ __forceinline__ uint64_t lo64(i128 v) { return (uint64_t)v; }
__device__ __forceinline__ uint64_t hi64(i128 v) { return (uint64_t)((u128)v >> 64); }
__device__ __forceinline__ bool fits_i64(i128 v) { return (i128)(int64_t)v == v; }

// general checked multiply (out of line); returns true on overflow
__device__ __noinline__ bool mul_i128_slow(i128 a, i128 b, i128* out) {
  bool neg = (a < 0) != (b < 0);
  u128 ua = a < 0 ? (u128)0 - (u128)a : (u128)a;
  u128 ub = b < 0 ? (u128)0 - (u128)b : (u128)b;
  uint64_t al = (uint64_t)ua, ah = (uint64_t)(ua >> 64), bl = (uint64_t)ub, bh = (uint64_t)(ub >> 64);
  if (ah && bh) return true;
  uint64_t ch = ah ? ah : bh, cl = ah ? bl : al;  // cross term (at most one is non-zero)
  uint64_t cross_lo = ch * cl, cross_hi = __umul64hi(ch, cl);
  if (cross_hi) return true;
  uint64_t lo = al * bl, hi = __umul64hi(al, bl);
  uint64_t hi2 = hi + cross_lo;
  if (hi2 < hi) return true;
  u128 r = ((u128)hi2 << 64) | lo;
  if (neg) {
    if (r > ((u128)1 << 127)) return true;
    *out = (i128)((u128)0 - r);
  } else {
    if (r >> 127) return true;
    *out = (i128)r;
  }
  return false;
}
// hot-path multiply: 64x64 -> 128 inline (cannot overflow), everything else out of line
__device__ __forceinline__ bool mul_i128_fast(i128 a, i128 b, i128* out) {
  if (fits_i64(a) && fits_i64(b)) {
    int64_t x = (int64_t)a, y = (int64_t)b;
    *out = make_i128((uint64_t)x * (uint64_t)y, (uint64_t)__mul64hi(x, y));
    return false;
  }
  return mul_i128_slow(a, b, out);
}
__device__ __forceinline__ bool add_i128_checked(i128 a, i128 b, i128* out) {
  i128 r = (i128)((u128)a + (u128)b);
  *out = r;
  return ((a < 0) == (b < 0)) && ((r < 0) != (a < 0));
}
__device__ __forceinline__ bool sub_i128_checked(i128 a, i128 b, i128* out) {
  i128 r = (i128)((u128)a - (u128)b);
  *out = r;
  return ((a < 0) != (b < 0)) && ((r < 0) != (a < 0));
}
__device__ __noinline__ i128 pow10_dev(int n) {
  i128 r = 1;
  for (int i = 0; i < n; i++) r *= 10;
  return r;
}
// 10^n as the double nearest to it (exact for n <= 22): the scale factor of the decimal <-> float casts
__device__ __noinline__ double pow10_f64_dev(int n) {
  const double t[39] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11, 1e12, 1e13,
                        1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22, 1e23, 1e24, 1e25, 1e26, 1e27,
                        1e28, 1e29, 1e30, 1e31, 1e32, 1e33, 1e34, 1e35, 1e36, 1e37, 1e38};
  return t[n < 0 ? 0 : n > 38 ? 38 : n];
}
__device__ __noinline__ i128 div_i128_dev(i128 a, i128 b) { return a / b; }
__device__ __noinline__ i128 mod_i128_dev(i128 a, i128 b) { return a % b; }
__device__ __forceinline__ long long f64_order_key(double a) {
  long long x = __double_as_longlong(a);
  asm volatile("" : "+l"(x));  // integer from here on: no FP neg/abs folding of the bit tricks (NaN payloads)
  return x ^ (long long)((unsigned long long)(x >> 63) >> 1);
}

struct StrRef {
  const uint8_t* p;
  uint32_t len;
};

__device__ __noinline__ int str_cmp(StrRef a, StrRef b) {
  uint32_t n = a.len < b.len ? a.len : b.len;
  for (uint32_t i = 0; i < n; i++) {
    uint8_t x = a.p[i], y = b.p[i];
    if (x != y) return x < y ? -1 : 1;
  }
  return a.len < b.len ? -1 : (a.len > b.len ? 1 : 0);
}
// string MIN / MAX: does the view (xp, xl) order strictly before (MIN) / after (MAX) the view (cp, cl)?  A length of
// ACC_STR_NONE is "no value": it never wins and loses to every value
__device__ __noinline__ bool str_beats(bool is_min, uint64_t xp, uint64_t xl, uint64_t cp, uint64_t cl) {
  if (xl == ACC_STR_NONE) return false;
  if (cl == ACC_STR_NONE) return true;
  StrRef x, c;
  x.p = (const uint8_t*)xp;
  x.len = (uint32_t)xl;
  c.p = (const uint8_t*)cp;
  c.len = (uint32_t)cl;
  const int d = str_cmp(x, c);
  return is_min ? d < 0 : d > 0;
}
__device__ __noinline__ bool str_eq(StrRef a, StrRef b) {
  if (a.len != b.len) return false;
  for (uint32_t i = 0; i < a.len; i++)
    if (a.p[i] != b.p[i]) return false;
  return true;
}
__device__ __noinline__ bool like_match_dev(const uint8_t* s, uint32_t sn, const uint8_t* p, uint32_t pn) {
  uint32_t si = 0, pi = 0, star_p = 0xFFFFFFFFu, star_s = 0;
  while (si < sn) {
    if (pi < pn && p[pi] != '%' && (p[pi] == '_' || p[pi] == s[si])) {
      si++;
      pi++;
      continue;
    }
    if (pi < pn && p[pi] == '%') {
      star_p = pi++;
      star_s = si;
      continue;
    }
    if (star_p != 0xFFFFFFFFu) {
      pi = star_p + 1;
      si = ++star_s;
      continue;
    }
    return false;
  }
  while (pi < pn && p[pi] == '%') pi++;
  return pi == pn;
}
// proleptic Gregorian civil date of a day number (days since 1970-01-01), and back (H. Hinnant's algorithms)
__device__ __forceinline__ int64_t civil_from_days_dev(int64_t z, int64_t* month, int64_t* day) {
  z += 719468;
  int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  int64_t doe = z - era * 146097;
  int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  int64_t y = yoe + era * 400;
  int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  int64_t mp = (5 * doy + 2) / 153;
  int64_t m = mp < 10 ? mp + 3 : mp - 9;
  *month = m;
  *day = doy - (153 * mp + 2) / 5 + 1;
  return y + (m <= 2);
}
__device__ __forceinline__ int64_t jan1_days_dev(int64_t y) {  // day number of January 1st of year y
  y -= 1;
  const int64_t era = (y >= 0 ? y : y - 399) / 400;
  const int64_t yoe = y - era * 400;
  return era * 146097 + yoe * 365 + yoe / 4 - yoe / 100 + 306 - 719468;
}
__device__ __forceinline__ int64_t floor_mod7(int64_t v) { return ((v % 7) + 7) % 7; }
// date_part(part, Date32): week is the ISO 8601 week (that of the week's Thursday), dow 0 = Sunday, doy 1..366
__device__ __noinline__ int64_t date_part_dev(int64_t z, int part) {
  int64_t m, d;
  const int64_t y = civil_from_days_dev(z, &m, &d);
  switch (part) {
    case DP_YEAR: return y;
    case DP_QUARTER: return (m - 1) / 3 + 1;
    case DP_MONTH: return m;
    case DP_DAY: return d;
    case DP_DOY: return z - jan1_days_dev(y) + 1;
    case DP_DOW: return floor_mod7(z + 4);  // 1970-01-01 was a Thursday
    default: {
      const int64_t thu = z - floor_mod7(z + 3) + 3;  // floor_mod7(z + 3) = ISO weekday - 1 (Monday = 0)
      int64_t tm, td;
      const int64_t ty = civil_from_days_dev(thu, &tm, &td);
      return (thu - jan1_days_dev(ty)) / 7 + 1;
    }
  }
}
__device__ __noinline__ uint64_t hash_bytes_dev(const uint8_t* p, uint32_t len) { return hash_bytes(p, len); }

// len<<56 | up to 7 bytes (little endian); one or two aligned 8-byte loads (allocations carry slack)
__device__ __forceinline__ uint64_t pack8(const uint8_t* p, uint32_t len, int len_shift) {
  if (len == 0) return 0;
  const uint64_t* base = (const uint64_t*)((uintptr_t)p & ~(uintptr_t)7);
  const uint32_t sh = (uint32_t)((uintptr_t)p & 7) * 8;
  uint64_t v = base[0] >> sh;
  if (sh + len * 8 > 64) v |= base[1] << (64 - sh);
  v &= (len >= 8) ? ~0ull : ((1ull << (len * 8)) - 1);
  return v | ((uint64_t)len << len_shift);
}

// ------------------------------------------------------------------------------------------------
// Per-thread lane context: passed BY VALUE (registers), never through memory
// ------------------------------------------------------------------------------------------------
struct Lane {
  const uint8_t* stage;  // current stage buffer (source tile)
  uint8_t* regs;         // VM register file
  int tid;
  int B;  // blockDim.x
};

#define FOR_R for (int r = 0; r < VM_R; r++)

__device__ __forceinline__ uint32_t fetch_valid(const Lane L, const Operand o) {
  if (o.kind == OPD_COL) {
    const ColDesc& cd = PROG.cols[o.idx];
    if (!cd.valid) return 0xFFFFFFFFu;
    const uint8_t* v = L.stage + cd.valid_smem_off;
    uint32_t m = 0;
#pragma unroll
    FOR_R m |= (v[r * L.B + L.tid] ? 1u : 0u) << r;
    return m;
  }
  if (o.kind == OPD_REG) {
    const uint32_t vo = PROG.regs[o.idx].valid_off;
    if (vo == 0xFFFFFFFFu) return 0xFFFFFFFFu;
    return ((const uint32_t*)(L.regs + vo))[L.tid];
  }
  if (o.kind == OPD_IMM) return PROG.imms[o.idx].is_null ? 0u : 0xFFFFFFFFu;
  return 0xFFFFFFFFu;
}
__device__ __forceinline__ void store_valid(const Lane L, const Operand dst, uint32_t m) {
  const uint32_t vo = PROG.regs[dst.idx].valid_off;
  if (vo != 0xFFFFFFFFu) ((uint32_t*)(L.regs + vo))[L.tid] = m;
}

// ---- per-row accessors: generic over operand kind / encoding; compiled once ----------------------
__device__ __noinline__ int64_t ld1_i64(const Lane L, const Operand o, int r) {
  const int e = r * L.B + L.tid;
  if (o.kind == OPD_COL) {
    const ColDesc& cd = PROG.cols[o.idx];
    const uint8_t* base = L.stage + cd.smem_off;
    switch (cd.phys) {
      case PH_I32: return ((const int32_t*)base)[e];
      case PH_I64:
      case PH_U64: return ((const int64_t*)base)[e];
      case PH_U32: return ((const uint32_t*)base)[e];
      case PH_I16: return ((const int16_t*)base)[e];
      case PH_U16: return ((const uint16_t*)base)[e];
      case PH_I8: return ((const int8_t*)base)[e];
      case PH_DEC128: return (int64_t)((const ulonglong2*)base)[e].x;
      default: return ((const uint8_t*)base)[e];
    }
  }
  if (o.kind == OPD_REG) {
    const RegDesc& rd = PROG.regs[o.idx];
    if (rd.vk == VK_BOOL) return (((const uint32_t*)(L.regs + rd.smem_off))[L.tid] >> r) & 1;
    if (rd.vk == VK_I128) return (int64_t)((const ulonglong2*)(L.regs + rd.smem_off))[e].x;
    return ((const int64_t*)(L.regs + rd.smem_off))[e];
  }
  return (int64_t)PROG.imms[o.idx].lo;
}
__device__ __noinline__ double ld1_f64(const Lane L, const Operand o, int r) {
  const int e = r * L.B + L.tid;
  if (o.kind == OPD_COL) {
    const ColDesc& cd = PROG.cols[o.idx];
    const uint8_t* base = L.stage + cd.smem_off;
    if (cd.phys == PH_F32) return __longlong_as_double((long long)f32_bits_to_f64_bits(((const uint32_t*)base)[e]));
    return ((const double*)base)[e];
  }
  if (o.kind == OPD_REG) return ((const double*)(L.regs + PROG.regs[o.idx].smem_off))[e];
  return __longlong_as_double((long long)PROG.imms[o.idx].lo);
}
__device__ __noinline__ i128 ld1_i128(const Lane L, const Operand o, int r) {
  if (o.vk != VK_I128) return (i128)ld1_i64(L, o, r);
  const int e = r * L.B + L.tid;
  ulonglong2 x;
  if (o.kind == OPD_COL) x = ((const ulonglong2*)(L.stage + PROG.cols[o.idx].smem_off))[e];
  else if (o.kind == OPD_REG) x = ((const ulonglong2*)(L.regs + PROG.regs[o.idx].smem_off))[e];
  else x = make_ulonglong2(PROG.imms[o.idx].lo, PROG.imms[o.idx].hi);
  return make_i128(x.x, x.y);
}
__device__ __noinline__ StrRef ld1_str(const Lane L, const Operand o, int r) {
  const int e = r * L.B + L.tid;
  StrRef s;
  if (o.kind == OPD_COL) {
    const ColDesc& cd = PROG.cols[o.idx];
    if (cd.phys == PH_UTF8) {
      const int32_t* off = (const int32_t*)(L.stage + cd.smem_off);
      int32_t o0 = off[e], o1 = off[e + 1];
      s.p = cd.chars + o0;
      s.len = (uint32_t)(o1 - o0);
      return s;
    }
    ulonglong2 x = ((const ulonglong2*)(L.stage + cd.smem_off))[e];
    s.p = (const uint8_t*)x.x;
    s.len = (uint32_t)x.y;
    return s;
  }
  if (o.kind == OPD_REG) {
    ulonglong2 x = ((const ulonglong2*)(L.regs + PROG.regs[o.idx].smem_off))[e];
    s.p = (const uint8_t*)x.x;
    s.len = (uint32_t)x.y;
    return s;
  }
  s.p = (const uint8_t*)PROG.imms[o.idx].lo;
  s.len = (uint32_t)PROG.imms[o.idx].hi;
  return s;
}
__device__ __forceinline__ void st1_i64(const Lane L, const Operand dst, int r, int64_t v) {
  ((int64_t*)(L.regs + PROG.regs[dst.idx].smem_off))[r * L.B + L.tid] = v;
}
__device__ __forceinline__ void st1_f64(const Lane L, const Operand dst, int r, double v) {
  ((double*)(L.regs + PROG.regs[dst.idx].smem_off))[r * L.B + L.tid] = v;
}
__device__ __forceinline__ void st1_i128(const Lane L, const Operand dst, int r, i128 v) {
  ((ulonglong2*)(L.regs + PROG.regs[dst.idx].smem_off))[r * L.B + L.tid] = make_ulonglong2(lo64(v), hi64(v));
}
__device__ __forceinline__ void st1_str(const Lane L, const Operand dst, int r, StrRef v) {
  ((ulonglong2*)(L.regs + PROG.regs[dst.idx].smem_off))[r * L.B + L.tid] = make_ulonglong2((unsigned long long)v.p, (unsigned long long)v.len);
}

// ---- register-blocked accessors (hot ops) -------------------------------------------------------
// An operand is resolved ONCE into (base pointer, element width) -- tile column and VM register
// differ only in the base -- so each hot op carries a single small load sequence.
struct Src {
  const uint8_t* base;  // nullptr: immediate (value in imm_lo/imm_hi) or "slow" encoding
  uint32_t width;       // 4 (sign-extended int32), 8, 16; 0 = slow path through ld1_*
  uint64_t imm_lo, imm_hi;
};
__device__ __forceinline__ Src resolve_int(const Lane L, const Operand o) {
  Src s;
  s.base = nullptr;
  s.width = 0;
  s.imm_lo = s.imm_hi = 0;
  if (o.kind == OPD_COL) {
    const ColDesc& cd = PROG.cols[o.idx];
    if (cd.phys == PH_I32 || cd.phys == PH_I64 || cd.phys == PH_U64 || cd.phys == PH_DEC128) {
      s.base = L.stage + cd.smem_off;
      s.width = cd.width;
    }
  } else if (o.kind == OPD_REG) {
    const RegDesc& rd = PROG.regs[o.idx];
    if (rd.vk == VK_I64 || rd.vk == VK_I128) {
      s.base = L.regs + rd.smem_off;
      s.width = rd.vk == VK_I128 ? 16 : 8;
    }
  } else {
    s.imm_lo = PROG.imms[o.idx].lo;
    s.imm_hi = PROG.imms[o.idx].hi;
    s.width = 1;  // immediate
  }
  return s;
}
__device__ __forceinline__ void fetch_i64(const Lane L, const Operand o, int64_t v[VM_R]) {
  const Src s = resolve_int(L, o);
  if (s.width == 8) {
#pragma unroll
    FOR_R v[r] = ((const int64_t*)s.base)[r * L.B + L.tid];
  } else if (s.width == 16) {
#pragma unroll
    FOR_R v[r] = (int64_t)((const ulonglong2*)s.base)[r * L.B + L.tid].x;
  } else if (s.width == 4) {
#pragma unroll
    FOR_R v[r] = ((const int32_t*)s.base)[r * L.B + L.tid];
  } else if (s.width == 1) {
#pragma unroll
    FOR_R v[r] = (int64_t)s.imm_lo;
  } else {
#pragma unroll 1
    FOR_R v[r] = ld1_i64(L, o, r);
  }
}
__device__ __forceinline__ void fetch_f64(const Lane L, const Operand o, double v[VM_R]) {
  if (o.kind == OPD_COL && PROG.cols[o.idx].phys == PH_F64) {
    const double* p = (const double*)(L.stage + PROG.cols[o.idx].smem_off);
#pragma unroll
    FOR_R v[r] = p[r * L.B + L.tid];
  } else if (o.kind == OPD_REG) {
    const double* p = (const double*)(L.regs + PROG.regs[o.idx].smem_off);
#pragma unroll
    FOR_R v[r] = p[r * L.B + L.tid];
  } else if (o.kind == OPD_IMM) {
    const double x = __longlong_as_double((long long)PROG.imms[o.idx].lo);
#pragma unroll
    FOR_R v[r] = x;
  } else {
#pragma unroll 1
    FOR_R v[r] = ld1_f64(L, o, r);
  }
}
__device__ __forceinline__ void fetch_i128(const Lane L, const Operand o, i128 v[VM_R]) {
  const Src s = resolve_int(L, o);
  if (s.width == 16 && o.vk == VK_I128) {
#pragma unroll
    FOR_R {
      ulonglong2 x = ((const ulonglong2*)s.base)[r * L.B + L.tid];
      v[r] = make_i128(x.x, x.y);
    }
  } else if (s.width == 8 || s.width == 16) {  // 64-bit integer (or the low word of a narrow decimal view)
#pragma unroll
    FOR_R v[r] = (i128)(s.width == 8 ? ((const int64_t*)s.base)[r * L.B + L.tid] : (int64_t)((const ulonglong2*)s.base)[r * L.B + L.tid].x);
  } else if (s.width == 1) {
    const i128 x = o.vk == VK_I128 ? make_i128(s.imm_lo, s.imm_hi) : (i128)(int64_t)s.imm_lo;
#pragma unroll
    FOR_R v[r] = x;
  } else {
#pragma unroll 1
    FOR_R v[r] = ld1_i128(L, o, r);
  }
}
__device__ __forceinline__ uint32_t fetch_bool(const Lane L, const Operand o) {
  if (o.kind == OPD_REG && PROG.regs[o.idx].vk == VK_BOOL) return ((const uint32_t*)(L.regs + PROG.regs[o.idx].smem_off))[L.tid];
  uint32_t m = 0;
#pragma unroll 1
  FOR_R m |= (ld1_i64(L, o, r) != 0 ? 1u : 0u) << r;
  return m;
}
__device__ __forceinline__ void store_i64(const Lane L, const Operand dst, const int64_t v[VM_R]) {
  int64_t* p = (int64_t*)(L.regs + PROG.regs[dst.idx].smem_off);
#pragma unroll
  FOR_R p[r * L.B + L.tid] = v[r];
}
__device__ __forceinline__ void store_f64(const Lane L, const Operand dst, const double v[VM_R]) {
  double* p = (double*)(L.regs + PROG.regs[dst.idx].smem_off);
#pragma unroll
  FOR_R p[r * L.B + L.tid] = v[r];
}
__device__ __forceinline__ void store_i128(const Lane L, const Operand dst, const i128 v[VM_R]) {
  ulonglong2* p = (ulonglong2*)(L.regs + PROG.regs[dst.idx].smem_off);
#pragma unroll
  FOR_R p[r * L.B + L.tid] = make_ulonglong2(lo64(v[r]), hi64(v[r]));
}
__device__ __forceinline__ void store_bool(const Lane L, const Operand dst, uint32_t m) {
  ((uint32_t*)(L.regs + PROG.regs[dst.idx].smem_off))[L.tid] = m;
}

__device__ __forceinline__ void raise(unsigned int code) { atomicMax(&PROG.status->error, code); }

__device__ __forceinline__ bool cmp_result(int op, int c) {
  switch (op) {
    case OP_CMP_EQ: return c == 0;
    case OP_CMP_NE: return c != 0;
    case OP_CMP_LT: return c < 0;
    case OP_CMP_LE: return c <= 0;
    case OP_CMP_GT: return c > 0;
    default: return c >= 0;
  }
}
__device__ __forceinline__ uint32_t cmp_mask(int op, uint32_t lt, uint32_t gt) {
  const uint32_t eq = ~(lt | gt);
  switch (op) {
    case OP_CMP_EQ: return eq;
    case OP_CMP_NE: return ~eq;
    case OP_CMP_LT: return lt;
    case OP_CMP_LE: return lt | eq;
    case OP_CMP_GT: return gt;
    default: return gt | eq;
  }
}

// ------------------------------------------------------------------------------------------------
// Scalar functions (OP_ABS and up): rolled like the cold operations, in functions of their own so that
// cold_op and the interpreter do not grow.  String bytes are only read for live rows (a NULL or
// filtered row's view may point anywhere).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t utf8_seq_len(uint8_t c) { return c < 0x80 ? 1u : (c >> 5) == 6 ? 2u : (c >> 4) == 14 ? 3u : 4u; }
// is the code point p[0..n) one of the code points of the UTF-8 string set[0..sn)?
__device__ __noinline__ bool in_code_point_set(const uint8_t* p, uint32_t n, const uint8_t* set, uint32_t sn) {
  for (uint32_t i = 0; i < sn;) {
    const uint32_t k = utf8_seq_len(set[i]);
    bool eq = k == n && i + k <= sn;
    for (uint32_t j = 0; eq && j < n; j++) eq = set[i + j] == p[j];
    if (eq) return true;
    i += k;
  }
  return false;
}
__device__ __noinline__ StrRef trim_dev(StrRef s, int side, const uint8_t* set, uint32_t sn) {
  uint32_t b = 0, e = s.len;
  if (side != TRIM_TRAILING) {
    while (b < e) {
      const uint32_t k = utf8_seq_len(s.p[b]);
      if (b + k > e || !in_code_point_set(s.p + b, k, set, sn)) break;
      b += k;
    }
  }
  if (side != TRIM_LEADING) {
    while (e > b) {
      uint32_t q = e - 1;
      while (q > b && (s.p[q] & 0xC0) == 0x80) q--;
      if (!in_code_point_set(s.p + q, e - q, set, sn)) break;
      e = q;
    }
  }
  s.p += b;
  s.len = e - b;
  return s;
}
// abs / round / floor / ceil
__device__ __noinline__ void scalar_num_op(const Lane L, const uint32_t active, const int pc) {
  const VInstr ins = PROG.code[pc];
  const uint32_t va = fetch_valid(L, ins.a);
  const uint32_t live = active & va;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    const bool lv = (live >> r) & 1;
    if (ins.op == OP_ABS) {
      if (ins.t == VK_F64) {
        st1_f64(L, ins.dst, r, fabs(ld1_f64(L, ins.a, r)));
      } else if (ins.t == VK_I128) {
        const i128 a = ld1_i128(L, ins.a, r);
        if (a == make_i128(0, 0x8000000000000000ull) && lv) raise(1);
        st1_i128(L, ins.dst, r, a < 0 ? (i128)((u128)0 - (u128)a) : a);
      } else {
        const int64_t a = ld1_i64(L, ins.a, r);
        const int64_t mn = ins.aux == PH_I8 ? INT8_MIN : ins.aux == PH_I16 ? INT16_MIN : ins.aux == PH_I32 ? INT32_MIN : INT64_MIN;
        if (a == mn && lv) raise(1);  // DataFusion's abs is checked [EXT]
        st1_i64(L, ins.dst, r, a < 0 ? (int64_t)(0 - (uint64_t)a) : a);
      }
    } else if (ins.op == OP_ROUND) {  // round_half_away_from_zero(x * f) / f, each step rounded once (no contraction)
      const double x = ld1_f64(L, ins.a, r), f = __longlong_as_double((long long)PROG.imms[ins.imm].lo);
      double o = x;  // NaN: the input, bits included (the device would return its canonical NaN)
      if (x != x) {
      } else if (ins.aux == PH_F32) o = (double)__fdiv_rn(roundf(__fmul_rn((float)x, (float)f)), (float)f);
      else o = __ddiv_rn(round(__dmul_rn(x, f)), f);
      st1_f64(L, ins.dst, r, o);
    } else {
      const double x = ld1_f64(L, ins.a, r);
      st1_f64(L, ins.dst, r, ins.op == OP_FLOOR ? floor(x) : ceil(x));
    }
  }
  store_valid(L, ins.dst, va);
}
// nullif(a, b): a, NULL where b is not NULL and a = b by the engine's equality (floats: bitwise, i.e. total order)
__device__ __noinline__ void scalar_nullif_op(const Lane L, const uint32_t active, const int pc) {
  const VInstr ins = PROG.code[pc];
  const uint32_t va = fetch_valid(L, ins.a), vb = fetch_valid(L, ins.b);
  const uint32_t live = active & va & vb;
  uint32_t vout = va, bmask = 0;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    bool eq = false;
    if (ins.t == VK_STR) {
      const StrRef a = ld1_str(L, ins.a, r);
      if ((live >> r) & 1) eq = str_eq(a, ld1_str(L, ins.b, r));
      st1_str(L, ins.dst, r, a);
    } else if (ins.t == VK_I128) {
      const i128 a = ld1_i128(L, ins.a, r);
      eq = a == ld1_i128(L, ins.b, r);
      st1_i128(L, ins.dst, r, a);
    } else if (ins.t == VK_F64) {
      const double a = ld1_f64(L, ins.a, r);
      eq = __double_as_longlong(a) == __double_as_longlong(ld1_f64(L, ins.b, r));
      st1_f64(L, ins.dst, r, a);
    } else {
      const int64_t a = ld1_i64(L, ins.a, r);
      eq = a == ld1_i64(L, ins.b, r);
      if (ins.t == VK_BOOL) bmask |= (a ? 1u : 0u) << r;
      else st1_i64(L, ins.dst, r, a);
    }
    if (((vb >> r) & 1) && eq) vout &= ~(1u << r);
  }
  if (ins.t == VK_BOOL) store_bool(L, ins.dst, bmask);
  store_valid(L, ins.dst, vout);
}
// character / octet length, starts / ends_with, the trims
__device__ __noinline__ void scalar_str_op(const Lane L, const uint32_t active, const int pc) {
  const VInstr ins = PROG.code[pc];
  const uint32_t va = fetch_valid(L, ins.a);
  const uint32_t vb = ins.b.kind != OPD_NONE ? fetch_valid(L, ins.b) : 0xFFFFFFFFu;
  const uint32_t live = active & va & vb;
  uint32_t bmask = 0;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    const bool lv = (live >> r) & 1;
    StrRef a = ld1_str(L, ins.a, r);
    if (ins.op == OP_CHAR_LENGTH || ins.op == OP_OCTET_LENGTH) {
      int64_t n = a.len;
      if (ins.op == OP_CHAR_LENGTH) {
        n = 0;
        if (lv)
          for (uint32_t i = 0; i < a.len; i++) n += (a.p[i] & 0xC0) != 0x80;
      }
      st1_i64(L, ins.dst, r, n);
    } else if (ins.op == OP_TRIM) {
      if (lv) a = trim_dev(a, ins.aux, (const uint8_t*)PROG.imms[ins.imm].lo, (uint32_t)PROG.imms[ins.imm].hi);
      st1_str(L, ins.dst, r, a);
    } else {  // OP_STARTS_WITH / OP_ENDS_WITH
      bool hit = false;
      if (lv) {
        const StrRef b = ld1_str(L, ins.b, r);
        if (b.len <= a.len) {
          const uint8_t* p = a.p + (ins.op == OP_ENDS_WITH ? a.len - b.len : 0);
          hit = true;
          for (uint32_t i = 0; hit && i < b.len; i++) hit = p[i] == b.p[i];
        }
      }
      bmask |= (hit ? 1u : 0u) << r;
    }
  }
  if (ins.op == OP_STARTS_WITH || ins.op == OP_ENDS_WITH) store_bool(L, ins.dst, bmask);
  store_valid(L, ins.dst, va & vb);
}

// & | ^ << >> over integers of one type (aux = its Phys).  The values sit sign- or zero-extended in 64 bits, so & | ^ and
// an arithmetic (signed) or logical (unsigned) >> stay in range; the lowering narrows << to the width.  Shift counts are
// taken modulo the bit width, as Rust's wrapping_shl / wrapping_shr do in arrow-rs [EXT].
__device__ __noinline__ void scalar_bit_op(const Lane L, const uint32_t active, const int pc) {
  (void)active;
  const VInstr ins = PROG.code[pc];
  const uint32_t va = fetch_valid(L, ins.a), vb = fetch_valid(L, ins.b);
  const uint8_t ph = ins.aux;
  const uint64_t bits = (ph == PH_I8 || ph == PH_U8) ? 8 : (ph == PH_I16 || ph == PH_U16) ? 16 : (ph == PH_I32 || ph == PH_U32) ? 32 : 64;
  const bool is_unsigned = ph >= PH_U8 && ph <= PH_U64;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    const int64_t a = ld1_i64(L, ins.a, r), b = ld1_i64(L, ins.b, r);
    const uint32_t c = (uint32_t)((uint64_t)b & (bits - 1));
    int64_t o;
    switch (ins.op) {
      case OP_BIT_AND: o = a & b; break;
      case OP_BIT_OR: o = a | b; break;
      case OP_BIT_XOR: o = a ^ b; break;
      case OP_SHL: o = (int64_t)((uint64_t)a << c); break;
      default: o = is_unsigned ? (int64_t)((uint64_t)a >> c) : (a >> c); break;
    }
    st1_i64(L, ins.dst, r, o);
  }
  store_valid(L, ins.dst, va & vb);
}

// ILIKE, the regex operators and regexp_like: one thread walks one row's bytes through the DFA (regex_dfa.hpp, the same
// walk the host compiler's tests run), stopping at the matched or the dead state.  NULL in, NULL out.
__device__ __noinline__ void scalar_regex_op(const Lane L, const uint32_t active, const int pc) {
  const VInstr ins = PROG.code[pc];
  const uint32_t va = fetch_valid(L, ins.a);
  const uint32_t live = active & va;
  const uint8_t* dfa = (const uint8_t*)PROG.imms[ins.imm].lo;
  const uint64_t shape = PROG.imms[ins.imm].hi;
  uint32_t bmask = 0;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    bool hit = false;
    if ((live >> r) & 1) {
      const StrRef a = ld1_str(L, ins.a, r);
      hit = rx::dfa_is_match(dfa, shape, a.p, a.len);
    }
    bmask |= ((ins.aux ? !hit : hit) ? 1u : 0u) << r;
  }
  store_bool(L, ins.dst, bmask);
  store_valid(L, ins.dst, va);
}

// ------------------------------------------------------------------------------------------------
// String builders (OP_CONCAT and up): every result is written into the launch's character arena.
// Reservation: one 64-bit bump counter (RunStatus::arena_need), one atomic per warp per op and row slot.  A row whose
// bytes do not fit writes nothing but still counts, so the counter ends at the exact need and the host re-runs the launch
// with that capacity.  Such a row's view is "unwritten": {arena, need << 32}.  Every other reader takes the low 32 bits
// (length 0, nothing to read); the builders read the need, so a result built over it counts its true size too.
// ------------------------------------------------------------------------------------------------
struct BuildSrc {
  const uint8_t* p;
  uint32_t len;
  bool unwritten;
};
__device__ __noinline__ BuildSrc ld_build_src(const Lane L, const Operand o, int r) {
  BuildSrc b;
  if (o.kind == OPD_REG) {
    const ulonglong2 x = ((const ulonglong2*)(L.regs + PROG.regs[o.idx].smem_off))[r * L.B + L.tid];
    b.unwritten = (x.y >> 32) != 0;
    b.p = (const uint8_t*)x.x;
    b.len = b.unwritten ? (uint32_t)(x.y >> 32) : (uint32_t)x.y;
    return b;
  }
  const StrRef s = ld1_str(L, o, r);
  b.p = s.p;
  b.len = s.len;
  b.unwritten = false;
  return b;
}
// warp-aggregated reservation of len bytes (0 for rows that build nothing); every lane of the warp calls it
__device__ __forceinline__ unsigned long long arena_reserve(unsigned long long len) {
  const unsigned mask = __activemask();
  if (mask != 0xFFFFFFFFu) return atomicAdd(&PROG.status->arena_need, len);
  const int lane = threadIdx.x & 31;
  unsigned long long incl = len;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long t = __shfl_up_sync(mask, incl, d);
    if (lane >= d) incl += t;
  }
  unsigned long long base = 0;
  if (lane == 31 && incl) base = atomicAdd(&PROG.status->arena_need, incl);
  base = __shfl_sync(mask, base, 31);
  return base + incl - len;
}
// destination of a row's bytes, or nullptr when they do not fit (or an input was unwritten): store_built then records
// the need instead of a view
__device__ __forceinline__ uint8_t* arena_at(unsigned long long base, unsigned long long len, bool unwritten) {
  if (unwritten || base + len > PROG.arena_cap) return nullptr;
  return PROG.arena + base;
}
__device__ __forceinline__ void store_built(const Lane L, const Operand dst, int r, const uint8_t* out, unsigned long long len) {
  const ulonglong2 v = out ? make_ulonglong2((unsigned long long)out, len) : make_ulonglong2((unsigned long long)PROG.arena, len << 32);
  ((ulonglong2*)(L.regs + PROG.regs[dst.idx].smem_off))[r * L.B + L.tid] = v;
}
__device__ __forceinline__ void copy_bytes(uint8_t* d, const uint8_t* s, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) d[i] = s[i];
}
__device__ __forceinline__ uint32_t u128_digits(u128 v) {
  uint32_t n = 1;
  while (v >= 10) {
    v /= 10;
    n++;
  }
  return n;
}
// the digits of v, right-aligned ending at `end`
__device__ __forceinline__ void put_digits(uint8_t* end, u128 v, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) {
    *--end = (uint8_t)('0' + (uint32_t)(v % 10));
    v /= 10;
  }
}

// CAST(x AS Utf8): arrow's display of integers, Decimal128 (exactly `scale` fractional digits) and Bool, and chrono's
// %Y-%m-%d of a Date32 (4 digits within years 0..9999, else an explicit sign)
struct ToStr {
  uint32_t len;
  bool neg;
  u128 mag;     // integer / decimal magnitude; date: |year|
  uint32_t nd;  // digits of mag
  int64_t month, day;
};
__device__ __noinline__ ToStr to_str_shape(const Lane L, const VInstr& ins, int r) {
  ToStr t;
  t.neg = false;
  t.month = t.day = 0;
  if (ins.aux == TS_BOOL) {
    t.mag = ld1_i64(L, ins.a, r) != 0;
    t.len = t.mag ? 4 : 5;
    t.nd = 0;
    return t;
  }
  if (ins.aux == TS_DATE32) {
    const int64_t y = civil_from_days_dev(ld1_i64(L, ins.a, r), &t.month, &t.day);
    t.neg = y < 0;
    t.mag = (u128)(y < 0 ? -y : y);
    t.nd = u128_digits(t.mag);
    if (t.nd < 4) t.nd = 4;
    t.len = t.nd + 6 + ((y < 0 || y > 9999) ? 1 : 0);
    return t;
  }
  i128 v;
  if (ins.aux == TS_DEC128) v = ld1_i128(L, ins.a, r);
  else if (ins.aux == TS_UINT64) v = (i128)(uint64_t)ld1_i64(L, ins.a, r);
  else v = (i128)ld1_i64(L, ins.a, r);
  t.neg = v < 0;
  t.mag = t.neg ? (u128)0 - (u128)v : (u128)v;
  t.nd = u128_digits(t.mag);
  const uint32_t s = ins.aux == TS_DEC128 ? (uint32_t)ins.imm : 0;
  if (s > 0 && t.nd <= s) t.nd = s + 1;  // 0.0ddd
  t.len = t.nd + (t.neg ? 1 : 0) + (s > 0 ? 1 : 0);
  return t;
}
__device__ __noinline__ void to_str_write(uint8_t* out, const ToStr& t, const VInstr& ins) {
  if (ins.aux == TS_BOOL) {
    const char* w = t.mag ? "true" : "false";
    for (uint32_t i = 0; i < t.len; i++) out[i] = (uint8_t)w[i];
    return;
  }
  uint8_t* end = out + t.len;
  if (ins.aux == TS_DATE32) {
    put_digits(end, (u128)t.day, 2);
    end[-3] = '-';
    put_digits(end - 3, (u128)t.month, 2);
    end[-6] = '-';
    put_digits(end - 6, t.mag, t.nd);
    if (t.len > t.nd + 6) out[0] = t.neg ? '-' : '+';
    return;
  }
  const uint32_t s = ins.aux == TS_DEC128 ? (uint32_t)ins.imm : 0;
  if (s == 0) {
    put_digits(end, t.mag, t.nd);
  } else {
    u128 p = 1;
    for (uint32_t i = 0; i < s; i++) p *= 10;
    put_digits(end, t.mag % p, s);
    end[-(int)s - 1] = '.';
    put_digits(end - s - 1, t.mag / p, t.nd - s);
  }
  if (t.neg) out[0] = '-';
}

// OP_CONCAT's i-th argument: eight per immediate, from the instruction's first one on
__device__ __forceinline__ Operand build_arg(const int first, int i) {
  const ImmDesc& d = PROG.imms[first + (i >> 3)];
  const uint32_t w = (uint32_t)(((i & 7) < 4 ? d.lo : d.hi) >> (16 * (i & 3))) & 0xFFFFu;
  Operand o;
  o.kind = (uint8_t)(w >> 12);
  o.vk = VK_STR;
  o.idx = (uint16_t)(w & 0xFFFu);
  return o;
}

// concat / || / concat_ws, repeat, reverse and the casts to Utf8: for each row slot, the live rows' lengths, one warp
// reservation, then the bytes.  A thread that wrote bytes fences them before it goes on: a later instruction of the same
// program may publish a view of them to other threads (a group key of the global table, a string MIN / MAX cell).
__device__ __noinline__ void scalar_build_op(const Lane L, const uint32_t active, const int pc) {
  const VInstr ins = PROG.code[pc];
  uint32_t vout = 0xFFFFFFFFu;
  int n = 0;
  const int args = ins.imm;
  if (ins.op == OP_CONCAT) {
    n = (int)PROG.imms[args]._pad;
    for (int i = 0; i < n; i++) {
      if (ins.aux & BUILD_NULLS) vout &= fetch_valid(L, build_arg(args, i));
    }
    if (ins.aux & BUILD_WS) vout = fetch_valid(L, ins.a);
  } else {
    vout = fetch_valid(L, ins.a);
    if (ins.b.kind != OPD_NONE) vout &= fetch_valid(L, ins.b);
  }
  const uint32_t live = active & vout;
  bool wrote = false;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    const bool lv = (live >> r) & 1;
    unsigned long long len = 0;
    bool unwritten = false;
    BuildSrc a;
    a.len = 0;
    a.unwritten = false;
    int64_t times = 0;
    ToStr ts;
    if (lv) {
      if (ins.op == OP_CONCAT) {
        BuildSrc sep;
        sep.len = 0;
        sep.unwritten = false;
        if (ins.aux & BUILD_WS) sep = ld_build_src(L, ins.a, r);
        int present = 0;
        for (int i = 0; i < n; i++) {
          const Operand o = build_arg(args, i);
          if (!((fetch_valid(L, o) >> r) & 1)) continue;
          const BuildSrc x = ld_build_src(L, o, r);
          len += x.len + (present ? sep.len : 0);
          unwritten |= x.unwritten;
          present++;
        }
        if (present > 1) unwritten |= sep.unwritten;
        if (len > 0x7FFFFFFFull) raise(4);
      } else if (ins.op == OP_REPEAT) {
        a = ld_build_src(L, ins.a, r);
        times = ld1_i64(L, ins.b, r);
        if (times < 0) times = 0;
        if (a.len && (uint64_t)times > 0x7FFFFFFFull / a.len) raise(5);
        else len = (unsigned long long)a.len * (unsigned long long)times;
        unwritten = a.unwritten;
      } else if (ins.op == OP_REVERSE) {
        a = ld_build_src(L, ins.a, r);
        len = a.len;
        unwritten = a.unwritten;
      } else {
        ts = to_str_shape(L, ins, r);
        len = ts.len;
        if (ins.aux == TS_DATE32 && (ts.mag > (ts.neg ? 262144u : 262143u))) raise(6);
      }
      if (len > 0x7FFFFFFFull) len = 0;  // the launch fails (raised above)
    }
    const unsigned long long base = arena_reserve(len);
    uint8_t* out = lv ? arena_at(base, len, unwritten) : nullptr;
    if (out && len) {
      wrote = true;
      if (ins.op == OP_CONCAT) {
        BuildSrc sep;
        sep.len = 0;
        if (ins.aux & BUILD_WS) sep = ld_build_src(L, ins.a, r);
        uint8_t* w = out;
        bool first = true;
        for (int i = 0; i < n; i++) {
          const Operand o = build_arg(args, i);
          if (!((fetch_valid(L, o) >> r) & 1)) continue;
          if (!first) {
            copy_bytes(w, sep.p, sep.len);
            w += sep.len;
          }
          first = false;
          const BuildSrc x = ld_build_src(L, o, r);
          copy_bytes(w, x.p, x.len);
          w += x.len;
        }
      } else if (ins.op == OP_REPEAT) {
        for (int64_t k = 0; k < times; k++) copy_bytes(out + (uint64_t)k * a.len, a.p, a.len);
      } else if (ins.op == OP_REVERSE) {
        for (uint32_t i = 0; i < a.len;) {
          // a sequence cut short (invalid UTF-8: nothing upstream of every source checks it) keeps its bytes as they are
          const uint32_t k = min(utf8_seq_len(a.p[i]), a.len - i);
          copy_bytes(out + a.len - i - k, a.p + i, k);
          i += k;
        }
      } else {
        to_str_write(out, ts, ins);
      }
    }
    store_built(L, ins.dst, r, lv ? out : PROG.arena, lv ? len : 0);
  }
  if (wrote) __threadfence();
  store_valid(L, ins.dst, vout);
}

// the span DFAs of OP_REGEX_COUNT / OP_REGEX_REPLACE: two consecutive immediates from ins.imm on
__device__ __forceinline__ rx::RxSpans regex_spans(const VInstr& ins) {
  const ImmDesc& f = PROG.imms[ins.imm];
  const ImmDesc& b = PROG.imms[ins.imm + 1];
  rx::RxSpans d;
  d.fwd = (const uint8_t*)f.lo;
  d.fwd_shape = f.hi;
  d.rev = (const uint8_t*)b.lo;
  d.rev_shape = b.hi;
  return d;
}

// regexp_count: one thread per row slot counts 0 for an empty row, else skips start - 1 code points, then loops forward
// walk -> reverse walk -> iteration rule (regex_dfa.hpp regexp_count_row, the walk the host compiler's tests run).  A NULL
// row counts 0: the result is never NULL.
__device__ __noinline__ void scalar_regex_count_op(const Lane L, const uint32_t active, const int pc) {
  const VInstr ins = PROG.code[pc];
  const uint32_t live = active & fetch_valid(L, ins.a);
  const rx::RxSpans d = regex_spans(ins);
  const uint32_t skip = PROG.imms[ins.imm]._pad;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    int64_t c = 0;
    if ((live >> r) & 1) {
      const StrRef a = ld1_str(L, ins.a, r);
      c = rx::regexp_count_row(d, a.p, a.len, skip);
    }
    st1_i64(L, ins.dst, r, c);
  }
  store_valid(L, ins.dst, 0xFFFFFFFFu);
}

// regexp_replace: the string builders' protocol (scalar_build_op) -- a length pass over the row's matches, one warp
// reservation, then a write pass.  An input that is itself unwritten (an earlier builder's row that did not fit) counts
// the bound len + (len + 1) * |replacement| (g) or len + |replacement|, so the re-run's arena holds the row.
__device__ __noinline__ void scalar_regex_replace_op(const Lane L, const uint32_t active, const int pc) {
  const VInstr ins = PROG.code[pc];
  const uint32_t vout = fetch_valid(L, ins.a);
  const uint32_t live = active & vout;
  const rx::RxSpans d = regex_spans(ins);
  const bool global = ins.aux != 0;
  bool wrote = false;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    const bool lv = (live >> r) & 1;
    unsigned long long len = 0;
    BuildSrc a;
    a.p = nullptr;
    a.len = 0;
    a.unwritten = false;
    StrRef rep;
    rep.p = nullptr;
    rep.len = 0;
    if (lv) {
      a = ld_build_src(L, ins.a, r);
      rep = ld1_str(L, ins.b, r);
      if (a.unwritten) len = a.len + (global ? ((unsigned long long)a.len + 1) : 1ull) * rep.len;
      else len = rx::dfa_replace(d, a.p, a.len, rep.p, rep.len, global, nullptr);
      if (len > 0x7FFFFFFFull) {
        raise(7);
        len = 0;
      }
    }
    const unsigned long long base = arena_reserve(len);
    uint8_t* out = lv ? arena_at(base, len, a.unwritten) : nullptr;
    if (out && len) {
      wrote = true;
      rx::dfa_replace(d, a.p, a.len, rep.p, rep.len, global, out);
    }
    store_built(L, ins.dst, r, lv ? out : PROG.arena, lv ? len : 0);
  }
  if (wrote) __threadfence();
  store_valid(L, ins.dst, vout);
}

// ------------------------------------------------------------------------------------------------
// Cold operations: one rolled loop over the thread's rows; every body exists once in the binary.
// ------------------------------------------------------------------------------------------------
template <bool SFN>
__device__ __noinline__ void cold_op(const Lane L, const uint32_t active, const int pc) {
  if (SFN && PROG.code[pc].op >= OP_ABS) {  // the scalar functions (see run_generic)
    const uint8_t op = PROG.code[pc].op;
    if (op <= OP_CEIL) scalar_num_op(L, active, pc);
    else if (op == OP_NULLIF) scalar_nullif_op(L, active, pc);
    else if (op == OP_REGEX) scalar_regex_op(L, active, pc);
    else if (op == OP_REGEX_COUNT) scalar_regex_count_op(L, active, pc);
    else if (op == OP_REGEX_REPLACE) scalar_regex_replace_op(L, active, pc);
    else if (op > OP_REGEX) scalar_build_op(L, active, pc);
    else if (op >= OP_BIT_AND) scalar_bit_op(L, active, pc);
    else scalar_str_op(L, active, pc);
    return;
  }
  const VInstr ins = PROG.code[pc];
  uint32_t va = 0xFFFFFFFFu, vb = 0xFFFFFFFFu;
  if (ins.flags & IF_NULLCHK) {
    va = fetch_valid(L, ins.a);
    if (ins.b.kind != OPD_NONE) vb = fetch_valid(L, ins.b);
  }
  const uint32_t live = active & va & vb;
  uint32_t vout = va & vb;
  uint32_t bmask = 0;
  bool bool_result = false;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    const bool lv = (live >> r) & 1;
    switch (ins.op) {
      case OP_DIV:
      case OP_MOD: {
        if (ins.t == VK_I64) {  // aux = Phys of the result type
          int64_t a = ld1_i64(L, ins.a, r), b = ld1_i64(L, ins.b, r), o = 0;
          if (b == 0) {
            if (lv) raise(2);
          } else if (ins.aux == PH_U64) {
            o = (int64_t)(ins.op == OP_DIV ? (uint64_t)a / (uint64_t)b : (uint64_t)a % (uint64_t)b);
          } else if (b == -1) {  // the type's minimum / -1 overflows it; MIN % -1 is 0 [EXT]
            const int64_t mn = ins.aux == PH_I8 ? INT8_MIN : ins.aux == PH_I16 ? INT16_MIN : ins.aux == PH_I32 ? INT32_MIN : INT64_MIN;
            if (ins.op == OP_DIV) {
              if (a == mn && lv) raise(1);
              o = (int64_t)(0 - (uint64_t)a);
            }
          } else {
            o = ins.op == OP_DIV ? a / b : a % b;
          }
          st1_i64(L, ins.dst, r, o);
        } else if (ins.t == VK_F64) {
          double a = ld1_f64(L, ins.a, r), b = ld1_f64(L, ins.b, r);
          double o = ins.op == OP_DIV ? a / b : fmod(a, b);
          if (ins.aux == PH_F32) o = (double)(float)o;
          st1_f64(L, ins.dst, r, o);
        } else {
          // DIV: a * 10^imm / b (truncating); MOD: a % b (operands pre-scaled by the lowering)
          i128 a = ld1_i128(L, ins.a, r), b = ld1_i128(L, ins.b, r), o = 0;
          if (b == 0) {
            if (lv) raise(2);
          } else if (ins.op == OP_DIV) {
            i128 num;
            bool ovf = mul_i128_fast(a, pow10_dev(ins.imm), &num);
            if (ovf && lv) raise(1);
            o = ovf ? 0 : div_i128_dev(num, b);
          } else {
            o = mod_i128_dev(a, b);
          }
          st1_i128(L, ins.dst, r, o);
        }
        break;
      }
      case OP_NEG: {
        // floats: the sign bit flipped, a NaN's too (Rust's -x); nvcc's FP negation of a NaN does not flip it
        if (ins.t == VK_F64) st1_f64(L, ins.dst, r, __longlong_as_double(__double_as_longlong(ld1_f64(L, ins.a, r)) ^ (long long)0x8000000000000000ull));
        else if (ins.t == VK_I128) st1_i128(L, ins.dst, r, (i128)((u128)0 - (u128)ld1_i128(L, ins.a, r)));
        else st1_i64(L, ins.dst, r, (int64_t)(0 - (uint64_t)ld1_i64(L, ins.a, r)));
        break;
      }
      case OP_CMP_EQ:
      case OP_CMP_NE:
      case OP_CMP_LT:
      case OP_CMP_LE:
      case OP_CMP_GT:
      case OP_CMP_GE: {  // strings only (numeric compares are hot ops)
        bool_result = true;
        int cm = 0;
        if (lv) {
          StrRef a = ld1_str(L, ins.a, r), b = ld1_str(L, ins.b, r);
          cm = (ins.op == OP_CMP_EQ || ins.op == OP_CMP_NE) ? (str_eq(a, b) ? 0 : 1) : str_cmp(a, b);
        }
        bmask |= (cmp_result(ins.op, cm) ? 1u : 0u) << r;
        break;
      }
      case OP_CAST_I64_F64: {  // imm = 1: to Float32, rounded once from the integer
        int64_t a = ld1_i64(L, ins.a, r);
        double o;
        if (ins.imm == 1) o = ins.aux == PH_U64 ? (double)(float)(uint64_t)a : (double)(float)a;
        else o = ins.aux == PH_U64 ? (double)(uint64_t)a : (double)a;
        st1_f64(L, ins.dst, r, o);
        break;
      }
      case OP_CAST_I64_I128:  // aux = PH_U64: the operand's 64 bits are zero-extended
      case OP_CAST_I128_I128_UP: {
        i128 o;
        const i128 a = ins.aux == PH_U64 ? (i128)(uint64_t)ld1_i64(L, ins.a, r) : ld1_i128(L, ins.a, r);
        bool ovf = mul_i128_fast(a, pow10_dev(ins.imm), &o);
        if (ovf && lv) raise(1);
        st1_i128(L, ins.dst, r, o);
        break;
      }
      case OP_CAST_I128_I128_DOWN: {
        i128 a = ld1_i128(L, ins.a, r);
        i128 div = pow10_dev(ins.imm), half = div_i128_dev(div, 2);
        i128 q = div_i128_dev(a, div), rem = mod_i128_dev(a, div);
        if (a >= 0 && rem >= half) q += 1;
        else if (a < 0 && rem <= -half) q -= 1;
        st1_i128(L, ins.dst, r, q);
        break;
      }
      case OP_CHECK_PRECISION: {  // |v| >= 10^aux -> NULL (or error when checked)
        i128 a = ld1_i128(L, ins.a, r);
        i128 lim = pow10_dev(ins.aux);
        if (a >= lim || a <= -lim) {
          if (ins.flags & IF_CHECKED) {
            if (lv) raise(1);
          } else {
            vout &= ~(1u << r);
          }
        }
        st1_i128(L, ins.dst, r, a);
        break;
      }
      case OP_CAST_I128_F64: {
        i128 a = ld1_i128(L, ins.a, r);
        st1_f64(L, ins.dst, r, (double)a / pow10_f64_dev(ins.imm));
        break;
      }
      case OP_CAST_F64_I64: {  // aux = PH_U64: the target is UInt64, [0, 2^64)
        double t = trunc(ld1_f64(L, ins.a, r));
        int64_t o = 0;
        if (ins.aux == PH_U64) {
          if (!(t >= 0.0 && t < 1.8446744073709552e19)) vout &= ~(1u << r);
          else o = (int64_t)(uint64_t)t;
        } else if (!(t >= -9.2233720368547758e18 && t < 9.2233720368547758e18)) {
          vout &= ~(1u << r);
        } else {
          o = (int64_t)t;
        }
        st1_i64(L, ins.dst, r, o);
        break;
      }
      case OP_CAST_I128_I64: {  // aux = PH_U64: the target is UInt64
        i128 q = div_i128_dev(ld1_i128(L, ins.a, r), pow10_dev(ins.imm));
        if (ins.aux == PH_U64 ? (q < 0 || hi64(q) != 0) : !fits_i64(q)) vout &= ~(1u << r);
        st1_i64(L, ins.dst, r, (int64_t)q);
        break;
      }
      case OP_CAST_F64_I128: {
        double t = round(ld1_f64(L, ins.a, r) * pow10_f64_dev(ins.imm));
        i128 o = 0;
        if (!(fabs(t) < 1.7e38)) vout &= ~(1u << r);
        else o = (i128)t;
        st1_i128(L, ins.dst, r, o);
        break;
      }
      case OP_WRAP_I64:
      case OP_NARROW_I64: {  // OP_NARROW_I64 imm = 1: a negative 64-bit image is out of range too (UInt64 in or out)
        int64_t a = ld1_i64(L, ins.a, r), w;
        switch (ins.aux) {
          case PH_I8: w = (int8_t)a; break;
          case PH_I16: w = (int16_t)a; break;
          case PH_I32: w = (int32_t)a; break;
          case PH_U8: w = (uint8_t)a; break;
          case PH_U16: w = (uint16_t)a; break;
          case PH_U32: w = (uint32_t)a; break;
          default: w = a;
        }
        if (ins.op == OP_NARROW_I64 && (w != a || (ins.imm == 1 && a < 0))) vout &= ~(1u << r);
        st1_i64(L, ins.dst, r, w);
        break;
      }
      case OP_LIKE: {
        bool_result = true;
        bool hit = false;
        if (lv) {
          StrRef a = ld1_str(L, ins.a, r);
          hit = like_match_dev(a.p, a.len, (const uint8_t*)PROG.imms[ins.imm].lo, (uint32_t)PROG.imms[ins.imm].hi);
        }
        bmask |= ((ins.aux ? !hit : hit) ? 1u : 0u) << r;
        break;
      }
      case OP_DATE_PART: st1_i64(L, ins.dst, r, date_part_dev(ld1_i64(L, ins.a, r), ins.aux)); break;
      case OP_SUBSTR: {
        StrRef a = ld1_str(L, ins.a, r);
        int64_t st = ld1_i64(L, ins.b, r);
        const bool has_len = ins.imm >= 0;
        int64_t ln = has_len ? (int64_t)PROG.imms[ins.imm].lo : 0;
        int64_t s0 = st - 1, e0 = has_len ? s0 + ln : (int64_t)a.len;
        if (has_len && ln < 0 && lv) raise(3);
        if (s0 < 0) s0 = 0;
        if (e0 > (int64_t)a.len) e0 = a.len;
        if (e0 > s0) {
          a.p += s0;
          a.len = (uint32_t)(e0 - s0);
        } else {
          a.len = 0;
        }
        st1_str(L, ins.dst, r, a);
        break;
      }
      case OP_MOD_U64: st1_i64(L, ins.dst, r, (int64_t)((uint64_t)ld1_i64(L, ins.a, r) % PROG.imms[ins.imm].lo)); break;
      case OP_MADD_I64: st1_i64(L, ins.dst, r, (int64_t)((uint64_t)ld1_i64(L, ins.a, r) + (uint64_t)ld1_i64(L, ins.b, r) * PROG.imms[ins.imm].lo)); break;
      case OP_STR_PACK8: {  // generic operand encodings (the Utf8-column case is a hot op)
        uint64_t w = 0;
        if (lv) {
          StrRef a = ld1_str(L, ins.a, r);
          if (a.len > ins.aux) atomicExch(&PROG.status->pack_overflow, 1u);
          else w = pack8(a.p, a.len, ins.imm);
        }
        st1_i64(L, ins.dst, r, (int64_t)w);
        break;
      }
      default: break;
    }
  }
  if (bool_result) store_bool(L, ins.dst, bmask);
  store_valid(L, ins.dst, vout);
}

// OP_SELECT / OP_MOV: rolled, per row
__device__ __noinline__ void cold_move(const Lane L, const int pc) {
  const VInstr ins = PROG.code[pc];
  const bool sel = ins.op == OP_SELECT;
  const Operand src = sel ? ins.b : ins.a;
  const uint32_t cond = sel ? (fetch_bool(L, ins.a) & fetch_valid(L, ins.a)) : 0xFFFFFFFFu;
  const uint32_t vs = fetch_valid(L, src);
  const uint32_t vd = sel ? fetch_valid(L, ins.dst) : 0u;
  if (ins.t == VK_BOOL) {
    uint32_t b = fetch_bool(L, src), d = sel ? fetch_bool(L, ins.dst) : 0u;
    store_bool(L, ins.dst, (d & ~cond) | (b & cond));
  } else {
#pragma unroll 1
    for (int r = 0; r < VM_R; r++) {
      if (!((cond >> r) & 1)) continue;
      if (ins.t == VK_I128) st1_i128(L, ins.dst, r, ld1_i128(L, src, r));
      else if (ins.t == VK_F64) st1_f64(L, ins.dst, r, ld1_f64(L, src, r));
      else if (ins.t == VK_STR) st1_str(L, ins.dst, r, ld1_str(L, src, r));
      else st1_i64(L, ins.dst, r, ld1_i64(L, src, r));
    }
  }
  store_valid(L, ins.dst, (vd & ~cond) | (vs & cond));
}

__device__ __noinline__ void op_hash_generic(const Lane L, const uint32_t active, const int pc) {
  const VInstr ins = PROG.code[pc];
  const uint32_t v = fetch_valid(L, ins.a);
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    uint64_t h = 0;
    if ((v >> r) & 1) {
      if (ins.t == VK_F64) h = hash_f64(ld1_f64(L, ins.a, r));
      else if (ins.t == VK_I128) {
        i128 a = ld1_i128(L, ins.a, r);
        h = hash_i128(lo64(a), hi64(a));
      } else if (ins.t == VK_STR) {
        if ((active >> r) & 1) {
          StrRef a = ld1_str(L, ins.a, r);
          h = hash_bytes_dev(a.p, a.len);
        }
      } else {
        h = hash_i64(ld1_i64(L, ins.a, r));
      }
    }
    int64_t o;
    if (ins.op == OP_HASH) {
      o = (int64_t)h;
    } else {
      o = ld1_i64(L, ins.dst, r);
      if ((v >> r) & 1) o = (int64_t)combine_hashes(h, (uint64_t)o);
    }
    st1_i64(L, ins.dst, r, o);
  }
}

// ------------------------------------------------------------------------------------------------
// Pre-decoded micro-ops.  Chasing operand descriptors through constant memory costs ~100
// instructions per VM instruction; each CTA therefore decodes the program ONCE into this compact
// shared-memory form (resolved base selector / byte offset / element width / immediates) and the
// per-tile loop reads one or two broadcast LDS.128 per instruction instead.
// ------------------------------------------------------------------------------------------------
enum MicroFn : uint8_t { MF_GENERIC = 0, MF_CMP_I64, MF_ARITH_I64, MF_ARITH_I128, MF_DEC_MUL_LIT, MF_PACK8, MF_FILTER_BOOL, MF_LOGIC };
enum SrcSel : uint8_t { SEL_STAGE = 0, SEL_REGS = 1, SEL_IMM = 2 };

struct __align__(16) MicroOp {
  uint8_t fn, op, flags, aux;
  uint8_t a_sel, a_w, b_sel, b_w;  // widths: 4 (int32), 8, 16
  uint32_t a_off, b_off;
  uint32_t d_off, d_valid_off;
  int32_t imm;
  uint32_t _pad;
  uint64_t a_imm, b_imm;           // immediate values (low words)
  uint64_t lit_lo, lit_hi;         // third operand literal (fused decimal ops) / chars pointer (pack8)
};

struct __align__(16) AccOp {       // pre-resolved accumulator source (register sink)
  uint8_t kind, sel, w, nullable;
  uint32_t off;
  uint64_t imm;
};

__device__ __forceinline__ bool resolve_fast(const Operand o, uint8_t* sel, uint8_t* w, uint32_t* off, uint64_t* imm) {
  *imm = 0;
  *off = 0;
  if (o.kind == OPD_COL) {
    const ColDesc& cd = PROG.cols[o.idx];
    if (cd.valid) return false;
    if (!(cd.phys == PH_I32 || cd.phys == PH_I64 || cd.phys == PH_U64 || cd.phys == PH_DEC128)) return false;
    *sel = SEL_STAGE;
    *w = cd.width;
    *off = cd.smem_off;
    return true;
  }
  if (o.kind == OPD_REG) {
    const RegDesc& rd = PROG.regs[o.idx];
    if (rd.valid_off != 0xFFFFFFFFu) return false;
    if (!(rd.vk == VK_I64 || rd.vk == VK_I128)) return false;
    *sel = SEL_REGS;
    *w = rd.vk == VK_I128 ? 16 : 8;
    *off = rd.smem_off;
    return true;
  }
  if (o.kind == OPD_IMM) {
    if (PROG.imms[o.idx].is_null) return false;
    *sel = SEL_IMM;
    *w = 8;
    *imm = PROG.imms[o.idx].lo;
    return true;
  }
  return false;
}

__device__ __noinline__ void decode_micro(int pc, MicroOp* m) {
  const VInstr ins = PROG.code[pc];
  m->fn = MF_GENERIC;
  m->op = ins.op;
  m->flags = ins.flags;
  m->aux = ins.aux;
  m->imm = ins.imm;
  m->d_off = 0;
  m->d_valid_off = 0xFFFFFFFFu;
  m->lit_lo = m->lit_hi = 0;
  if (ins.flags & IF_NULLCHK) return;  // NULL-aware instructions keep the generic path
  if (ins.dst.kind == OPD_REG) {
    m->d_off = PROG.regs[ins.dst.idx].smem_off;
    m->d_valid_off = PROG.regs[ins.dst.idx].valid_off;
  }
  const bool a_ok = resolve_fast(ins.a, &m->a_sel, &m->a_w, &m->a_off, &m->a_imm);
  const bool b_ok = ins.b.kind != OPD_NONE && resolve_fast(ins.b, &m->b_sel, &m->b_w, &m->b_off, &m->b_imm);
  switch (ins.op) {
    case OP_CMP_EQ:
    case OP_CMP_NE:
    case OP_CMP_LT:
    case OP_CMP_LE:
    case OP_CMP_GT:
    case OP_CMP_GE:
      if ((ins.t == VK_I64) && a_ok && b_ok && ins.aux != PH_U64 && (ins.dst.kind == OPD_NONE || m->d_valid_off == 0xFFFFFFFFu)) m->fn = MF_CMP_I64;
      break;
    case OP_MADD_I64:
      if (a_ok && b_ok && m->d_valid_off == 0xFFFFFFFFu) {
        m->fn = MF_ARITH_I64;
        m->lit_lo = PROG.imms[ins.imm].lo;
      }
      break;
    case OP_ADD:
    case OP_SUB:
    case OP_MUL:
      if (a_ok && b_ok && m->d_valid_off == 0xFFFFFFFFu) {
        if (ins.t == VK_I64) m->fn = MF_ARITH_I64;
        else if (ins.t == VK_I128 && ((ins.a.vk == VK_I128) == (m->a_w == 16 || m->a_sel == SEL_IMM)) && ((ins.b.vk == VK_I128) == (m->b_w == 16 || m->b_sel == SEL_IMM))) {
          // immediates of I128 kind carry a high word: keep those generic unless they fit 64 bits
          bool imm_ok = true;
          if (m->a_sel == SEL_IMM && ins.a.vk == VK_I128) imm_ok &= (int64_t)PROG.imms[ins.a.idx].hi == ((int64_t)PROG.imms[ins.a.idx].lo >> 63);
          if (m->b_sel == SEL_IMM && ins.b.vk == VK_I128) imm_ok &= (int64_t)PROG.imms[ins.b.idx].hi == ((int64_t)PROG.imms[ins.b.idx].lo >> 63);
          if (imm_ok) m->fn = MF_ARITH_I128;
        }
      }
      break;
    case OP_DEC_MUL_LIT_MINUS:
    case OP_DEC_MUL_LIT_PLUS:
      if (a_ok && b_ok && m->a_sel != SEL_IMM && m->b_sel != SEL_IMM && m->d_valid_off == 0xFFFFFFFFu) {
        m->fn = MF_DEC_MUL_LIT;
        m->lit_lo = PROG.imms[ins.imm].lo;
        m->lit_hi = PROG.imms[ins.imm].hi;
      }
      break;
    case OP_STR_PACK8:
      if (ins.a.kind == OPD_COL && PROG.cols[ins.a.idx].phys == PH_UTF8 && !PROG.cols[ins.a.idx].valid && m->d_valid_off == 0xFFFFFFFFu) {
        m->fn = MF_PACK8;
        m->a_off = PROG.cols[ins.a.idx].smem_off;
        m->lit_lo = (uint64_t)PROG.cols[ins.a.idx].chars;
      }
      break;
    case OP_FILTER:
      if (ins.a.kind == OPD_REG && PROG.regs[ins.a.idx].vk == VK_BOOL && PROG.regs[ins.a.idx].valid_off == 0xFFFFFFFFu) {
        m->fn = MF_FILTER_BOOL;
        m->a_off = PROG.regs[ins.a.idx].smem_off;
      }
      break;
    case OP_AND:
    case OP_OR:
      if (ins.a.kind == OPD_REG && ins.b.kind == OPD_REG && PROG.regs[ins.a.idx].vk == VK_BOOL && PROG.regs[ins.b.idx].vk == VK_BOOL &&
          PROG.regs[ins.a.idx].valid_off == 0xFFFFFFFFu && PROG.regs[ins.b.idx].valid_off == 0xFFFFFFFFu && m->d_valid_off == 0xFFFFFFFFu) {
        m->fn = MF_LOGIC;
        m->a_off = PROG.regs[ins.a.idx].smem_off;
        m->b_off = PROG.regs[ins.b.idx].smem_off;
      }
      break;
    default: break;
  }
}

__device__ __noinline__ void decode_acc(int a, AccOp* o) {
  const AccDesc ad = PROG.acc[a];
  o->kind = ad.kind;
  o->nullable = ad.nullable;
  o->sel = 255;  // 255: slow (generic fetch)
  o->w = 0;
  o->off = 0;
  o->imm = 0;
  if (ad.kind == ACC_COUNT_STAR || (ad.kind == ACC_COUNT && !ad.nullable)) {
    o->sel = SEL_IMM;
    o->imm = 1;
    return;
  }
  if (ad.kind != ACC_SUM_I128 || ad.nullable) return;
  uint8_t sel, w;
  uint32_t off;
  uint64_t imm;
  if (!resolve_fast(ad.src, &sel, &w, &off, &imm)) return;
  if (sel == SEL_IMM && ad.src.vk == VK_I128) return;
  // a 16-byte source must really be a 128-bit value (not the narrow view of one)
  if ((w == 16) != (ad.src.vk == VK_I128) && sel != SEL_IMM) return;
  o->sel = sel;
  o->w = w;
  o->off = off;
  o->imm = imm;
}

// element e of a resolved integer operand, sign-extended to 64 bits
__device__ __forceinline__ int64_t ld_w(const uint8_t* base, uint32_t w, int e) {
  if (w == 8) return ((const int64_t*)base)[e];
  if (w == 16) return (int64_t)((const ulonglong2*)base)[e].x;
  return ((const int32_t*)base)[e];
}

// ------------------------------------------------------------------------------------------------
// Hot operations: one compact out-of-line function per (operation family, value kind) so that the
// instructions a given pipeline actually executes are few and contiguous (I-cache resident).
// ------------------------------------------------------------------------------------------------
#define OP_PROLOGUE                                           \
  const VInstr ins = PROG.code[pc];                           \
  uint32_t va = 0xFFFFFFFFu, vb = 0xFFFFFFFFu;                \
  if (ins.flags & IF_NULLCHK) {                               \
    va = fetch_valid(L, ins.a);                               \
    if (ins.b.kind != OPD_NONE) vb = fetch_valid(L, ins.b);   \
  }                                                           \
  const uint32_t live = active & va & vb;                     \
  (void)live;

__device__ __noinline__ void op_cmp_i64(const Lane L, const uint32_t active, const int pc) {
  OP_PROLOGUE
  int64_t a[VM_R], b[VM_R];
  fetch_i64(L, ins.a, a);
  fetch_i64(L, ins.b, b);
  uint32_t lt = 0, gt = 0;
  if (ins.aux == PH_U64) {
#pragma unroll
    FOR_R {
      lt |= ((uint64_t)a[r] < (uint64_t)b[r] ? 1u : 0u) << r;
      gt |= ((uint64_t)a[r] > (uint64_t)b[r] ? 1u : 0u) << r;
    }
  } else {
#pragma unroll
    FOR_R {
      lt |= (a[r] < b[r] ? 1u : 0u) << r;
      gt |= (a[r] > b[r] ? 1u : 0u) << r;
    }
  }
  store_bool(L, ins.dst, cmp_mask(ins.op, lt, gt));
  store_valid(L, ins.dst, va & vb);
}
__device__ __noinline__ void op_cmp_f64(const Lane L, const uint32_t active, const int pc) {
  OP_PROLOGUE
  double a[VM_R], b[VM_R];
  fetch_f64(L, ins.a, a);
  fetch_f64(L, ins.b, b);
  uint32_t lt = 0, gt = 0;
#pragma unroll
  FOR_R {
    long long x = f64_order_key(a[r]), y = f64_order_key(b[r]);
    lt |= (x < y ? 1u : 0u) << r;
    gt |= (x > y ? 1u : 0u) << r;
  }
  store_bool(L, ins.dst, cmp_mask(ins.op, lt, gt));
  store_valid(L, ins.dst, va & vb);
}
__device__ __noinline__ void op_cmp_i128(const Lane L, const uint32_t active, const int pc) {
  OP_PROLOGUE
  i128 a[VM_R], b[VM_R];
  fetch_i128(L, ins.a, a);
  fetch_i128(L, ins.b, b);
  uint32_t lt = 0, gt = 0;
#pragma unroll
  FOR_R {
    lt |= (a[r] < b[r] ? 1u : 0u) << r;
    gt |= (a[r] > b[r] ? 1u : 0u) << r;
  }
  store_bool(L, ins.dst, cmp_mask(ins.op, lt, gt));
  store_valid(L, ins.dst, va & vb);
}
__device__ __noinline__ void op_arith_i64(const Lane L, const uint32_t active, const int pc) {
  OP_PROLOGUE
  int64_t a[VM_R], b[VM_R];
  fetch_i64(L, ins.a, a);
  fetch_i64(L, ins.b, b);
  if (ins.op == OP_ADD) {
#pragma unroll
    FOR_R a[r] = (int64_t)((uint64_t)a[r] + (uint64_t)b[r]);
  } else if (ins.op == OP_SUB) {
#pragma unroll
    FOR_R a[r] = (int64_t)((uint64_t)a[r] - (uint64_t)b[r]);
  } else {
#pragma unroll
    FOR_R a[r] = (int64_t)((uint64_t)a[r] * (uint64_t)b[r]);
  }
  store_i64(L, ins.dst, a);
  store_valid(L, ins.dst, va & vb);
}
__device__ __noinline__ void op_arith_f64(const Lane L, const uint32_t active, const int pc) {
  OP_PROLOGUE
  double a[VM_R], b[VM_R];
  fetch_f64(L, ins.a, a);
  fetch_f64(L, ins.b, b);
  if (ins.op == OP_ADD) {
#pragma unroll
    FOR_R a[r] = a[r] + b[r];
  } else if (ins.op == OP_SUB) {
#pragma unroll
    FOR_R a[r] = a[r] - b[r];
  } else {
#pragma unroll
    FOR_R a[r] = a[r] * b[r];
  }
  if (ins.aux == PH_F32) {
#pragma unroll
    FOR_R a[r] = (double)(float)a[r];
  }
  store_f64(L, ins.dst, a);
  store_valid(L, ins.dst, va & vb);
}
__device__ __noinline__ void op_arith_i128(const Lane L, const uint32_t active, const int pc) {
  OP_PROLOGUE
  i128 a[VM_R], b[VM_R];
  fetch_i128(L, ins.a, a);
  fetch_i128(L, ins.b, b);
  uint32_t ovf = 0;
  if (ins.op == OP_ADD) {
#pragma unroll
    FOR_R ovf |= (add_i128_checked(a[r], b[r], &a[r]) ? 1u : 0u) << r;
  } else if (ins.op == OP_SUB) {
#pragma unroll
    FOR_R ovf |= (sub_i128_checked(a[r], b[r], &a[r]) ? 1u : 0u) << r;
  } else {
#pragma unroll
    FOR_R ovf |= (mul_i128_fast(a[r], b[r], &a[r]) ? 1u : 0u) << r;
  }
  if (ovf & live) raise(1);
  store_i128(L, ins.dst, a);
  store_valid(L, ins.dst, va & vb);
}
// dst = a * (imm +/- b): the TPC-H revenue shape l_extendedprice * (1 - l_discount)
__device__ __noinline__ void op_dec_mul_lit(const Lane L, const uint32_t active, const int pc) {
  OP_PROLOGUE
  i128 a[VM_R], b[VM_R];
  fetch_i128(L, ins.a, a);
  fetch_i128(L, ins.b, b);
  const i128 lit = make_i128(PROG.imms[ins.imm].lo, PROG.imms[ins.imm].hi);
  uint32_t ovf = 0;
  if (ins.op == OP_DEC_MUL_LIT_MINUS) {
#pragma unroll
    FOR_R ovf |= (sub_i128_checked(lit, b[r], &b[r]) ? 1u : 0u) << r;
  } else {
#pragma unroll
    FOR_R ovf |= (add_i128_checked(lit, b[r], &b[r]) ? 1u : 0u) << r;
  }
#pragma unroll
  FOR_R ovf |= (mul_i128_fast(a[r], b[r], &a[r]) ? 1u : 0u) << r;
  if (ovf & live) raise(1);
  store_i128(L, ins.dst, a);
  store_valid(L, ins.dst, va & vb);
}
__device__ __noinline__ void op_logic(const Lane L, const uint32_t active, const int pc) {
  OP_PROLOGUE
  if (ins.op == OP_NOT) {
    store_bool(L, ins.dst, ~fetch_bool(L, ins.a));
    store_valid(L, ins.dst, va);
    return;
  }
  if (ins.op == OP_IS_NULL || ins.op == OP_IS_NOT_NULL) {
    const uint32_t v = fetch_valid(L, ins.a);
    store_bool(L, ins.dst, ins.op == OP_IS_NULL ? ~v : v);
    store_valid(L, ins.dst, 0xFFFFFFFFu);
    return;
  }
  // Kleene AND / OR
  const uint32_t a = fetch_bool(L, ins.a), b = fetch_bool(L, ins.b);
  const uint32_t ta = a & va, tb = b & vb;    // definitely true
  const uint32_t fa = ~a & va, fb = ~b & vb;  // definitely false
  uint32_t val, vld;
  if (ins.op == OP_AND) {
    val = ta & tb;
    vld = (va & vb) | fa | fb;
  } else {
    val = ta | tb;
    vld = (va & vb) | ta | tb;
  }
  store_bool(L, ins.dst, val);
  store_valid(L, ins.dst, vld);
}
__device__ __noinline__ void op_pack8_utf8(const Lane L, const uint32_t active, const int pc) {
  OP_PROLOGUE
  const ColDesc& cd = PROG.cols[ins.a.idx];
  const int32_t* off = (const int32_t*)(L.stage + cd.smem_off);
  const uint8_t* chars = cd.chars;
  const uint32_t max_len = ins.aux;
  const int shift = ins.imm;
  int32_t o0[VM_R];
  uint32_t len[VM_R];
#pragma unroll
  FOR_R {
    const int e = r * L.B + L.tid;
    o0[r] = off[e];
    len[r] = (uint32_t)(off[e + 1] - o0[r]);
  }
  int64_t w[VM_R];
  uint32_t too_long = 0;
#pragma unroll
  FOR_R {
    const bool lv = (live >> r) & 1;
    too_long |= (lv && len[r] > max_len) ? 1u : 0u;
    w[r] = (lv && len[r] <= max_len) ? (int64_t)pack8(chars + o0[r], len[r], shift) : 0;
  }
  if (too_long) atomicExch(&PROG.status->pack_overflow, 1u);
  store_i64(L, ins.dst, w);
  store_valid(L, ins.dst, va);
}
__device__ __noinline__ void op_hash_i64(const Lane L, const uint32_t active, const int pc) {
  OP_PROLOGUE
  int64_t a[VM_R], o[VM_R];
  fetch_i64(L, ins.a, a);
  const uint32_t v = (ins.flags & IF_NULLCHK) ? va : fetch_valid(L, ins.a);
  if (ins.op == OP_HASH) {
#pragma unroll
    FOR_R o[r] = ((v >> r) & 1) ? (int64_t)hash_i64(a[r]) : 0;
  } else {
    fetch_i64(L, ins.dst, o);
#pragma unroll
    FOR_R if ((v >> r) & 1) o[r] = (int64_t)combine_hashes(hash_i64(a[r]), (uint64_t)o[r]);
  }
  store_i64(L, ins.dst, o);
}

// ---- micro-op fast paths (non-NULL operands, common encodings) -----------------------------------
#define SRC_BASE(sel, off) ((sel) == SEL_STAGE ? L.stage + (off) : (const uint8_t*)L.regs + (off))

__device__ __forceinline__ uint32_t mf_cmp_i64(const Lane L, uint32_t active, const MicroOp* mp) {
  const MicroOp& m = *mp;
  int64_t a[VM_R], b[VM_R];
  if (m.a_sel == SEL_IMM) {
#pragma unroll
    FOR_R a[r] = (int64_t)m.a_imm;
  } else {
    const uint8_t* pa = SRC_BASE(m.a_sel, m.a_off);
#pragma unroll
    FOR_R a[r] = ld_w(pa, m.a_w, r * L.B + L.tid);
  }
  if (m.b_sel == SEL_IMM) {
#pragma unroll
    FOR_R b[r] = (int64_t)m.b_imm;
  } else {
    const uint8_t* pb = SRC_BASE(m.b_sel, m.b_off);
#pragma unroll
    FOR_R b[r] = ld_w(pb, m.b_w, r * L.B + L.tid);
  }
  uint32_t lt = 0, gt = 0;
#pragma unroll
  FOR_R {
    lt |= (a[r] < b[r] ? 1u : 0u) << r;
    gt |= (a[r] > b[r] ? 1u : 0u) << r;
  }
  const uint32_t res = cmp_mask(m.op, lt, gt);
  if (m.flags & IF_FILTER) return active & res;
  ((uint32_t*)(L.regs + m.d_off))[L.tid] = res;
  return active;
}
__device__ __forceinline__ void mf_arith_i64(const Lane L, const MicroOp* mp) {
  const MicroOp& m = *mp;
  int64_t a[VM_R], b[VM_R];
  if (m.a_sel == SEL_IMM) {
#pragma unroll
    FOR_R a[r] = (int64_t)m.a_imm;
  } else {
    const uint8_t* pa = SRC_BASE(m.a_sel, m.a_off);
#pragma unroll
    FOR_R a[r] = ld_w(pa, m.a_w, r * L.B + L.tid);
  }
  if (m.b_sel == SEL_IMM) {
#pragma unroll
    FOR_R b[r] = (int64_t)m.b_imm;
  } else {
    const uint8_t* pb = SRC_BASE(m.b_sel, m.b_off);
#pragma unroll
    FOR_R b[r] = ld_w(pb, m.b_w, r * L.B + L.tid);
  }
  int64_t* d = (int64_t*)(L.regs + m.d_off);
  if (m.op == OP_MADD_I64) {
#pragma unroll
    FOR_R d[r * L.B + L.tid] = (int64_t)((uint64_t)a[r] + (uint64_t)b[r] * m.lit_lo);
  } else if (m.op == OP_ADD) {
#pragma unroll
    FOR_R d[r * L.B + L.tid] = (int64_t)((uint64_t)a[r] + (uint64_t)b[r]);
  } else if (m.op == OP_SUB) {
#pragma unroll
    FOR_R d[r * L.B + L.tid] = (int64_t)((uint64_t)a[r] - (uint64_t)b[r]);
  } else {
#pragma unroll
    FOR_R d[r * L.B + L.tid] = (int64_t)((uint64_t)a[r] * (uint64_t)b[r]);
  }
}
__device__ __forceinline__ i128 ld_w128(const uint8_t* base, uint32_t w, int e) {
  if (w == 16) {
    ulonglong2 x = ((const ulonglong2*)base)[e];
    return make_i128(x.x, x.y);
  }
  return (i128)ld_w(base, w, e);
}
__device__ __forceinline__ void mf_arith_i128(const Lane L, const uint32_t active, const MicroOp* mp) {
  const MicroOp& m = *mp;
  i128 a[VM_R], b[VM_R];
  if (m.a_sel == SEL_IMM) {
#pragma unroll
    FOR_R a[r] = (i128)(int64_t)m.a_imm;
  } else {
    const uint8_t* pa = SRC_BASE(m.a_sel, m.a_off);
#pragma unroll
    FOR_R a[r] = ld_w128(pa, m.a_w, r * L.B + L.tid);
  }
  if (m.b_sel == SEL_IMM) {
#pragma unroll
    FOR_R b[r] = (i128)(int64_t)m.b_imm;
  } else {
    const uint8_t* pb = SRC_BASE(m.b_sel, m.b_off);
#pragma unroll
    FOR_R b[r] = ld_w128(pb, m.b_w, r * L.B + L.tid);
  }
  uint32_t ovf = 0;
  if (m.op == OP_ADD) {
#pragma unroll
    FOR_R ovf |= (add_i128_checked(a[r], b[r], &a[r]) ? 1u : 0u) << r;
  } else if (m.op == OP_SUB) {
#pragma unroll
    FOR_R ovf |= (sub_i128_checked(a[r], b[r], &a[r]) ? 1u : 0u) << r;
  } else {
#pragma unroll
    FOR_R ovf |= (mul_i128_fast(a[r], b[r], &a[r]) ? 1u : 0u) << r;
  }
  if (ovf & active) raise(1);
  ulonglong2* d = (ulonglong2*)(L.regs + m.d_off);
#pragma unroll
  FOR_R d[r * L.B + L.tid] = make_ulonglong2(lo64(a[r]), hi64(a[r]));
}
__device__ __forceinline__ void mf_dec_mul_lit(const Lane L, const uint32_t active, const MicroOp* mp) {
  const MicroOp& m = *mp;
  const uint8_t* pa = SRC_BASE(m.a_sel, m.a_off);
  const uint8_t* pb = SRC_BASE(m.b_sel, m.b_off);
  const i128 lit = make_i128(m.lit_lo, m.lit_hi);
  i128 a[VM_R], b[VM_R];
#pragma unroll
  FOR_R {
    a[r] = ld_w128(pa, m.a_w, r * L.B + L.tid);
    b[r] = ld_w128(pb, m.b_w, r * L.B + L.tid);
  }
  uint32_t ovf = 0;
  if (m.op == OP_DEC_MUL_LIT_MINUS) {
#pragma unroll
    FOR_R ovf |= (sub_i128_checked(lit, b[r], &b[r]) ? 1u : 0u) << r;
  } else {
#pragma unroll
    FOR_R ovf |= (add_i128_checked(lit, b[r], &b[r]) ? 1u : 0u) << r;
  }
#pragma unroll
  FOR_R ovf |= (mul_i128_fast(a[r], b[r], &a[r]) ? 1u : 0u) << r;
  if (ovf & active) raise(1);
  ulonglong2* d = (ulonglong2*)(L.regs + m.d_off);
#pragma unroll
  FOR_R d[r * L.B + L.tid] = make_ulonglong2(lo64(a[r]), hi64(a[r]));
}
__device__ __forceinline__ void mf_pack8(const Lane L, const uint32_t active, const MicroOp* mp) {
  const MicroOp& m = *mp;
  const int32_t* off = (const int32_t*)(L.stage + m.a_off);
  const uint8_t* chars = (const uint8_t*)m.lit_lo;
  int32_t o0[VM_R];
  uint32_t len[VM_R];
#pragma unroll
  FOR_R {
    const int e = r * L.B + L.tid;
    o0[r] = off[e];
    len[r] = (uint32_t)(off[e + 1] - o0[r]);
  }
  int64_t* d = (int64_t*)(L.regs + m.d_off);
  uint32_t too_long = 0;
#pragma unroll
  FOR_R {
    const bool lv = (active >> r) & 1;
    too_long |= (lv && len[r] > m.aux) ? 1u : 0u;
    d[r * L.B + L.tid] = (lv && len[r] <= m.aux) ? (int64_t)pack8(chars + o0[r], len[r], m.imm) : 0;
  }
  if (too_long) atomicExch(&PROG.status->pack_overflow, 1u);
}

// ------------------------------------------------------------------------------------------------
// The interpreter: one pass over the expression program for the R rows this thread owns.
// All branches are warp-uniform (driven by the program, not by data).
// ------------------------------------------------------------------------------------------------
// SFN: the program holds scalar-function ops (OP_ABS and up).  Only the kernel variants compiled with it reach their
// functions, through a cold_op of their own, so every other variant's call graph -- and with it ptxas's register
// allocation, which spans a kernel's whole call graph -- stays as without them.
template <bool SFN>
__device__ __noinline__ uint32_t run_generic(const Lane L, uint32_t active, const int pc) {
  const uint32_t head = *(const uint32_t*)&PROG.code[pc];  // op | t<<8 | flags<<16 | aux<<24
  const uint32_t op = head & 0xFF, t = (head >> 8) & 0xFF;
  switch (op) {
    case OP_ADD:
    case OP_SUB:
    case OP_MUL:
      if (t == VK_I64) op_arith_i64(L, active, pc);
      else if (t == VK_F64) op_arith_f64(L, active, pc);
      else op_arith_i128(L, active, pc);
      break;
    case OP_DEC_MUL_LIT_MINUS:
    case OP_DEC_MUL_LIT_PLUS: op_dec_mul_lit(L, active, pc); break;
    case OP_CMP_EQ:
    case OP_CMP_NE:
    case OP_CMP_LT:
    case OP_CMP_LE:
    case OP_CMP_GT:
    case OP_CMP_GE: {
      if (t == VK_I64 || t == VK_BOOL) op_cmp_i64(L, active, pc);
      else if (t == VK_I128) op_cmp_i128(L, active, pc);
      else if (t == VK_F64) op_cmp_f64(L, active, pc);
      else cold_op<SFN>(L, active, pc);
      if ((head >> 16) & IF_FILTER) {  // fused FilterExec conjunct evaluated through a scratch bool register
        const Operand d = PROG.code[pc].dst;
        active &= fetch_bool(L, d) & fetch_valid(L, d);
      }
      break;
    }
    case OP_AND:
    case OP_OR:
    case OP_NOT:
    case OP_IS_NULL:
    case OP_IS_NOT_NULL: op_logic(L, active, pc); break;
    case OP_FILTER: {
      const Operand a = PROG.code[pc].a;
      active &= fetch_bool(L, a) & fetch_valid(L, a);
      break;
    }
    case OP_STR_PACK8: {
      const Operand a = PROG.code[pc].a;
      if (a.kind == OPD_COL && PROG.cols[a.idx].phys == PH_UTF8) op_pack8_utf8(L, active, pc);
      else cold_op<SFN>(L, active, pc);
      break;
    }
    case OP_HASH:
    case OP_HASH_COMBINE:
      if (t == VK_I64 || t == VK_BOOL) op_hash_i64(L, active, pc);
      else op_hash_generic(L, active, pc);
      break;
    case OP_SELECT:
    case OP_MOV: cold_move(L, pc); break;
    case OP_ACTIVE: {  // CASE: the rows the next instructions run for
      const VInstr& ins = PROG.code[pc];
      uint32_t m = ins.a.kind == OPD_NONE ? active : fetch_bool(L, ins.a);
      if (ins.b.kind != OPD_NONE) {
        const uint32_t c = fetch_bool(L, ins.b) & fetch_valid(L, ins.b);
        m &= ins.aux ? ~c : c;
      }
      if (ins.dst.kind == OPD_REG) store_bool(L, ins.dst, m);
      if (ins.a.kind != OPD_NONE) active = m;
      break;
    }
    case OP_NOP: break;
    default: cold_op<SFN>(L, active, pc); break;
  }
  return active;
}

template <bool SFN>
__device__ __forceinline__ uint32_t run_program(const Lane L, uint32_t active, const MicroOp* mops, int n_instr) {
  for (int pc = 0; pc < n_instr; pc++) {
    const MicroOp* m = &mops[pc];
    switch (m->fn) {
      case MF_CMP_I64: active = mf_cmp_i64(L, active, m); break;
      case MF_ARITH_I64: mf_arith_i64(L, m); break;
      case MF_ARITH_I128: mf_arith_i128(L, active, m); break;
      case MF_DEC_MUL_LIT: mf_dec_mul_lit(L, active, m); break;
      case MF_PACK8: mf_pack8(L, active, m); break;
      case MF_FILTER_BOOL: active &= ((const uint32_t*)(L.regs + m->a_off))[L.tid]; break;
      case MF_LOGIC: {
        const uint32_t x = ((const uint32_t*)(L.regs + m->a_off))[L.tid], y = ((const uint32_t*)(L.regs + m->b_off))[L.tid];
        ((uint32_t*)(L.regs + m->d_off))[L.tid] = m->op == OP_AND ? (x & y) : (x | y);
        break;
      }
      default: active = run_generic<SFN>(L, active, pc); break;
    }
  }
  return active;
}

// ------------------------------------------------------------------------------------------------
// Tile loading
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t col_tile_bytes(const ColDesc& cd, int tile_rows) {
  uint32_t b = (uint32_t)tile_rows * cd.width;
  if (cd.phys == PH_UTF8) b += 16;  // one extra offset (+ padding to a 16-byte multiple)
  return b;
}

// TMA path: one elected thread issues a bulk copy per staged column; completion is signalled on
// the stage's mbarrier through complete_tx.
__device__ __noinline__ void issue_tile_tma(uint8_t* stage, uint64_t* bar, int64_t row0, int tile_rows) {
  uint32_t total = 0;
  const int n_cols = PROG.n_cols;
  for (int i = 0; i < n_cols; i++) {
    const ColDesc& cd = PROG.cols[i];
    total += col_tile_bytes(cd, tile_rows);
    if (cd.valid) total += (uint32_t)tile_rows;
  }
  mbar_expect_tx(bar, total);
  for (int i = 0; i < n_cols; i++) {
    const ColDesc& cd = PROG.cols[i];
    bulk_g2s(stage + cd.smem_off, (const uint8_t*)cd.data + row0 * cd.width, col_tile_bytes(cd, tile_rows), bar);
    if (cd.valid) bulk_g2s(stage + cd.valid_smem_off, cd.valid + row0, (uint32_t)tile_rows, bar);
  }
}

// Fallback path (ragged last tile, unaligned slices): cooperative loads, zero fill past the end.
__device__ __noinline__ void load_tile_coop(uint8_t* stage, int64_t row0, int rows, int tile_rows, int tid, int B) {
  const int n_cols = PROG.n_cols;
  for (int i = 0; i < n_cols; i++) {
    const ColDesc& cd = PROG.cols[i];
    uint8_t* dst = stage + cd.smem_off;
    if (cd.phys == PH_UTF8) {
      const int32_t* src = (const int32_t*)cd.data + row0;
      int32_t* d = (int32_t*)dst;
      for (int k = tid; k <= tile_rows; k += B) d[k] = src[k <= rows ? k : rows];
    } else {
      const uint8_t* src = (const uint8_t*)cd.data + row0 * cd.width;
      uint32_t nb = (uint32_t)rows * cd.width, tb = (uint32_t)tile_rows * cd.width;
      if ((cd.width & 3) == 0 && (((uintptr_t)src) & 3) == 0) {
        const uint32_t* s4 = (const uint32_t*)src;
        uint32_t* d4 = (uint32_t*)dst;
        for (uint32_t k = tid; k < tb / 4; k += B) d4[k] = (k * 4 < nb) ? s4[k] : 0u;
      } else {
        for (uint32_t k = tid; k < tb; k += B) dst[k] = (k < nb) ? src[k] : 0;
      }
    }
    if (cd.valid) {
      uint8_t* dv = stage + cd.valid_smem_off;
      for (int k = tid; k < tile_rows; k += B) dv[k] = (k < rows) ? cd.valid[row0 + k] : 0;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Sink: materialise (FilterExec compaction + ProjectionExec outputs)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void store_out_i64(void* data, uint8_t phys, unsigned long long pos, int64_t v) {
  switch (phys) {
    case PH_I8:
    case PH_U8:
    case PH_BOOL8: ((int8_t*)data)[pos] = (int8_t)v; break;
    case PH_I16:
    case PH_U16: ((int16_t*)data)[pos] = (int16_t)v; break;
    case PH_I32:
    case PH_U32: ((int32_t*)data)[pos] = (int32_t)v; break;
    default: ((int64_t*)data)[pos] = v;
  }
}

// Output position of a tile = rows kept by all EARLIER tiles (decoupled look-back over one 64-bit word per tile:
// {flag:2, count:62}; flag 1 = this tile's own count, 2 = inclusive prefix), so FilterExec / ProjectionExec keep
// the input row order across tiles like their DataFusion counterparts (both are order-preserving operators).
// Tiles are dealt round-robin to co-resident CTAs that walk their tiles in increasing order, so a tile only ever
// waits for tiles that are already running.
__device__ __forceinline__ unsigned long long tile_ld_acquire(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void tile_st_release(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void sink_materialize(const Lane L, const uint32_t active, uint32_t* warp_tot /*[VM_R][32]*/, unsigned long long* tile_base_sh,
                                                 const int64_t t, const int64_t n_tiles) {
  const int lane = L.tid & 31, warp = L.tid >> 5, nwarps = L.B >> 5;
  uint32_t lane_pre[VM_R];
#pragma unroll
  FOR_R {
    uint32_t m = __ballot_sync(0xFFFFFFFFu, (active >> r) & 1);
    lane_pre[r] = __popc(m & ((1u << lane) - 1));
    if (lane == 0) warp_tot[r * 32 + warp] = __popc(m);
  }
  __syncthreads();
  // position of row (r, warp, lane) = number of live rows with smaller (r, warp) + lane_pre
  unsigned long long pos[VM_R];
  uint32_t run = 0;
#pragma unroll
  FOR_R {
    uint32_t mine = 0;
    for (int w = 0; w < nwarps; w++) {
      if (w == warp) mine = run;
      run += warp_tot[r * 32 + w];
    }
    pos[r] = mine + lane_pre[r];
  }
  if (warp == 0) {
    const unsigned long long F_AGG = 1ull << 62, F_PFX = 2ull << 62, CNT = (1ull << 62) - 1;
    unsigned long long* ts = PROG.tile_state;
    if (lane == 0 && t > 0) tile_st_release(&ts[t], F_AGG | (unsigned long long)run);
    unsigned long long excl = 0;
    for (int64_t p = t - 1; p >= 0; p -= 32) {
      const int64_t q = p - lane;
      unsigned long long v = F_PFX;  // before the first tile: an (empty) inclusive prefix
      if (q >= 0) {
        do {
          v = tile_ld_acquire(&ts[q]);
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
      tile_st_release(&ts[t], F_PFX | (excl + (unsigned long long)run));
      *tile_base_sh = excl;
      if (t == n_tiles - 1) PROG.status->out_rows = excl + (unsigned long long)run;
    }
  }
  __syncthreads();
  if (run == 0) return;
  const unsigned long long base = *tile_base_sh;
#pragma unroll
  FOR_R pos[r] += base;
  const int n_out = PROG.n_out;
  for (int j = 0; j < n_out; j++) {
    const OutCol oc = PROG.out[j];
    const uint32_t v = oc.valid ? fetch_valid(L, oc.src) : 0xFFFFFFFFu;
    if (oc.src.vk == VK_I128) {
      i128 a[VM_R];
      fetch_i128(L, oc.src, a);
#pragma unroll
      FOR_R if ((active >> r) & 1) ((ulonglong2*)oc.data)[pos[r]] = make_ulonglong2(lo64(a[r]), hi64(a[r]));
    } else if (oc.src.vk == VK_F64) {
      double a[VM_R];
      fetch_f64(L, oc.src, a);
      if (oc.phys == PH_F32) {
#pragma unroll
        FOR_R if ((active >> r) & 1) ((uint32_t*)oc.data)[pos[r]] = f64_bits_to_f32_bits((uint64_t)__double_as_longlong(a[r]));
      } else {
#pragma unroll
        FOR_R if ((active >> r) & 1) ((double*)oc.data)[pos[r]] = a[r];
      }
    } else if (oc.src.vk == VK_STR) {
#pragma unroll
      FOR_R {
        if ((active >> r) & 1) {
          const bool ok = (v >> r) & 1;
          StrRef a = ld1_str(L, oc.src, r);
          ((ulonglong2*)oc.data)[pos[r]] = make_ulonglong2(ok ? (unsigned long long)a.p : 0ull, ok ? (unsigned long long)a.len : 0ull);
        }
      }
    } else {
      int64_t a[VM_R];
      if (oc.src.vk == VK_BOOL) {
        const uint32_t m = fetch_bool(L, oc.src);
#pragma unroll
        FOR_R a[r] = (m >> r) & 1;
      } else {
        fetch_i64(L, oc.src, a);
      }
      if (oc.phys == PH_I64 || oc.phys == PH_U64) {
#pragma unroll
        FOR_R if ((active >> r) & 1) ((int64_t*)oc.data)[pos[r]] = a[r];
      } else if (oc.phys == PH_I32 || oc.phys == PH_U32) {
#pragma unroll
        FOR_R if ((active >> r) & 1) ((int32_t*)oc.data)[pos[r]] = (int32_t)a[r];
      } else {
#pragma unroll
        FOR_R if ((active >> r) & 1) store_out_i64(oc.data, oc.phys, pos[r], a[r]);
      }
    }
    if (oc.valid) {
#pragma unroll
      FOR_R if ((active >> r) & 1) oc.valid[pos[r]] = (v >> r) & 1;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Aggregate hash table (global memory, open addressing, linear probing)
// ------------------------------------------------------------------------------------------------
struct KeyVal {
  unsigned long long w0, w1;
  unsigned char valid;
  unsigned char vk;
};

__device__ __forceinline__ bool key_equal(const KeyVal& a, unsigned long long w0, unsigned long long w1, unsigned char valid) {
  if (a.valid != valid) return false;
  if (!valid) return true;
  if (a.vk == VK_STR) {
    StrRef x{(const uint8_t*)a.w0, (uint32_t)a.w1}, y{(const uint8_t*)w0, (uint32_t)w1};
    return str_eq(x, y);
  }
  if (a.vk == VK_I128) return a.w0 == w0 && a.w1 == w1;
  // every other key, floats included, by its 64-bit image: -0.0 and 0.0 are two groups, NaNs one per payload (DESIGN §6)
  return a.w0 == w0;
}

// find-or-insert; returns slot or ~0ull on overflow
__device__ __noinline__ unsigned long long table_upsert(int n_keys, unsigned long long h, const KeyVal* kv) {
  const AggTable& T = PROG.table;
  const unsigned long long mask = T.cap - 1;
  unsigned long long slot = mix64(h) & mask;
  for (unsigned long long probes = 0; probes < T.cap; probes++) {
    unsigned int st = *(volatile unsigned int*)&T.state[slot];
    if (st == 0) {
      unsigned int old = atomicCAS(&T.state[slot], 0u, 1u);
      if (old == 0) {
        T.hash[slot] = h;
        for (int k = 0; k < n_keys; k++) {
          T.keys[((unsigned long long)k * T.cap + slot) * 2 + 0] = kv[k].w0;
          T.keys[((unsigned long long)k * T.cap + slot) * 2 + 1] = kv[k].w1;
          T.key_valid[(unsigned long long)k * T.cap + slot] = kv[k].valid;
        }
        __threadfence();
        atomicExch(&T.state[slot], 2u);
        unsigned int ng = atomicAdd(T.n_groups, 1u);
        if ((unsigned long long)ng * 4 > T.cap * 3) return ~0ull;  // load factor > 0.75
        return slot;
      }
      st = old;
    }
    while (st == 1) st = *(volatile unsigned int*)&T.state[slot];
    __threadfence();
    if (*(volatile unsigned long long*)&T.hash[slot] == h) {
      bool eq = true;
      for (int k = 0; k < n_keys && eq; k++) {
        unsigned long long w0 = *(volatile unsigned long long*)&T.keys[((unsigned long long)k * T.cap + slot) * 2 + 0];
        unsigned long long w1 = *(volatile unsigned long long*)&T.keys[((unsigned long long)k * T.cap + slot) * 2 + 1];
        unsigned char vl = *(volatile unsigned char*)&T.key_valid[(unsigned long long)k * T.cap + slot];
        eq = key_equal(kv[k], w0, w1, vl);
      }
      if (eq) return slot;
    }
    slot = (slot + 1) & mask;
  }
  return ~0ull;
}

__device__ __forceinline__ void acc_add_i128_atomic(unsigned long long* cell, uint64_t lo, uint64_t hi) {
  unsigned long long old = atomicAdd(&cell[0], lo);
  unsigned long long carry = (old + lo) < old ? 1ull : 0ull;
  if (hi + carry) atomicAdd(&cell[1], hi + carry);
}
__device__ __forceinline__ void table_lock(unsigned long long slot) {
  while (atomicCAS(&PROG.table.lock[slot], 0u, 1u) != 0u) {
  }
  __threadfence();
}
__device__ __forceinline__ void table_unlock(unsigned long long slot) {
  __threadfence();
  atomicExch(&PROG.table.lock[slot], 0u);
}

struct Acc128 {
  uint64_t lo, hi;
};

// single-copy-atomic 16-byte load and compare-and-swap of a table cell (sm_90: LDG.E.128 / ATOMG.E.CAS.128)
__device__ __forceinline__ ulonglong2 ld_relaxed_b128(const unsigned long long* p) {
  ulonglong2 r;
  asm volatile(
      "{\n\t.reg .b128 t;\n\t"
      "ld.relaxed.gpu.global.b128 t, [%2];\n\t"
      "mov.b128 {%0, %1}, t;\n\t}"
      : "=l"(r.x), "=l"(r.y)
      : "l"(p)
      : "memory");
  return r;
}
__device__ __forceinline__ ulonglong2 atom_cas_b128(unsigned long long* p, ulonglong2 cmp, ulonglong2 val) {
  ulonglong2 r;
  asm volatile(
      "{\n\t.reg .b128 c, v, d;\n\t"
      "mov.b128 c, {%3, %4};\n\t"
      "mov.b128 v, {%5, %6};\n\t"
      "atom.relaxed.gpu.global.cas.b128 d, [%2], c, v;\n\t"
      "mov.b128 {%0, %1}, d;\n\t}"
      : "=l"(r.x), "=l"(r.y)
      : "l"(p), "l"(cmp.x), "l"(cmp.y), "l"(val.x), "l"(val.y)
      : "memory");
  return r;
}

// string MIN / MAX of a table cell: compare-and-swap of the whole 16-byte view, no lock.  The cell only ever moves
// towards the final answer, so a row that does not beat the value it last read can stop -- most rows issue no atomic.
// Input characters never change during a launch, so relaxed ordering suffices for them; a string builder's bytes
// (Program::arena) are written in the same launch by another thread, which fences them before it installs the view, so
// a program that builds strings reads the cell with acquire (a fence after the load or the failed CAS) before it
// compares bytes.  Kept apart from table_merge, which the fused kernel's and the add-only register sink's flushes call:
// they never see a string accumulator.
__device__ __noinline__ void table_merge_str(int kind, unsigned long long slot, int a, Acc128 x) {
  const AggTable& T = PROG.table;
  unsigned long long* cell = T.acc + ((unsigned long long)a * T.cap + slot) * 2;
  const bool is_min = kind == ACC_MIN_STR;
  const bool acquire = PROG.arena != nullptr;
  ulonglong2 cur = ld_relaxed_b128(cell);
  if (acquire) __threadfence();
  const ulonglong2 val = make_ulonglong2(x.lo, x.hi);
  while (str_beats(is_min, x.lo, x.hi, cur.x, cur.y)) {
    const ulonglong2 seen = atom_cas_b128(cell, cur, val);
    if (seen.x == cur.x && seen.y == cur.y) return;
    cur = seen;
    if (acquire) __threadfence();
  }
}

// merge one partial accumulator value into a table cell (atomics; 128-bit min/max under the lock)
__device__ __noinline__ void table_merge(int kind, unsigned long long slot, int a, Acc128 x) {
  const AggTable& T = PROG.table;
  unsigned long long* cell = T.acc + ((unsigned long long)a * T.cap + slot) * 2;
  switch (kind) {
    case ACC_COUNT_STAR:
    case ACC_COUNT: atomicAdd(&cell[0], (unsigned long long)x.lo); break;
    case ACC_SUM_I128: acc_add_i128_atomic(cell, x.lo, x.hi); break;
    case ACC_SUM_F64: atomicAdd((double*)&cell[0], __longlong_as_double((long long)x.lo)); break;
    case ACC_MIN_F64: atomicMin((long long*)&cell[0], (long long)x.lo); break;
    case ACC_MAX_F64: atomicMax((long long*)&cell[0], (long long)x.lo); break;
    default: {
      const i128 v = make_i128(x.lo, x.hi);
      table_lock(slot);
      i128 cur = make_i128(cell[0], cell[1]);
      bool take = kind == ACC_MIN_I128 ? v < cur : v > cur;
      if (take) {
        cell[0] = x.lo;
        cell[1] = x.hi;
      }
      table_unlock(slot);
    }
  }
}

__device__ __noinline__ void load_key(const Lane L, const Operand ko, int r, KeyVal* out) {
  const uint32_t v = fetch_valid(L, ko);
  out->vk = ko.vk;
  out->valid = (v >> r) & 1;
  out->w0 = out->w1 = 0;
  if (!out->valid) return;
  if (ko.vk == VK_STR) {
    StrRef s = ld1_str(L, ko, r);
    out->w0 = (unsigned long long)s.p;
    out->w1 = s.len;
  } else if (ko.vk == VK_I128) {
    i128 a = ld1_i128(L, ko, r);
    out->w0 = lo64(a);
    out->w1 = hi64(a);
  } else if (ko.vk == VK_F64) {
    double a = ld1_f64(L, ko, r);
    out->w0 = (unsigned long long)__double_as_longlong(a);
  } else {
    out->w0 = (unsigned long long)ld1_i64(L, ko, r);
  }
}

// per-row path (high cardinality): every live row upserts its group and updates with atomics
__device__ __noinline__ uint32_t sink_agg_global(const Lane L, uint32_t active) {
  if (*(volatile unsigned int*)&PROG.status->overflow) return active;
  const int n_keys = PROG.n_keys, n_acc = PROG.n_acc;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    if (!((active >> r) & 1)) continue;
    KeyVal kv[VM_MAX_KEYS];
    for (int k = 0; k < n_keys; k++) load_key(L, PROG.keys[k], r, &kv[k]);
    const unsigned long long h = n_keys ? (unsigned long long)ld1_i64(L, PROG.key_hash, r) : 0ull;
    const unsigned long long slot = table_upsert(n_keys, h, kv);
    if (slot == ~0ull) {
      atomicExch(&PROG.status->overflow, 1u);
      active &= ~(1u << r);
      continue;
    }
    for (int a = 0; a < n_acc; a++) {
      const AccDesc ad = PROG.acc[a];
      if (ad.kind != ACC_COUNT_STAR && ad.nullable && !((fetch_valid(L, ad.src) >> r) & 1)) continue;
      Acc128 x;
      x.lo = 1;
      x.hi = 0;
      if (ad.kind == ACC_SUM_I128 || ad.kind == ACC_MIN_I128 || ad.kind == ACC_MAX_I128) {
        i128 v = ld1_i128(L, ad.src, r);
        x.lo = lo64(v);
        x.hi = ad.zext ? 0ull : hi64(v);
      } else if (ad.kind == ACC_MIN_STR || ad.kind == ACC_MAX_STR) {
        const StrRef s = ld1_str(L, ad.src, r);
        x.lo = (uint64_t)s.p;
        x.hi = s.len;
      } else if (ad.kind == ACC_SUM_F64) {
        x.lo = (uint64_t)__double_as_longlong(ld1_f64(L, ad.src, r));
      } else if (ad.kind == ACC_MIN_F64 || ad.kind == ACC_MAX_F64) {
        x.lo = (uint64_t)f64_order_key(ld1_f64(L, ad.src, r));
      }
      if (ad.kind == ACC_MIN_STR || ad.kind == ACC_MAX_STR) table_merge_str(ad.kind, slot, a, x);
      else table_merge(ad.kind, slot, a, x);
    }
  }
  return active;
}

// 128-bit MIN / MAX of a table cell without the slot lock: a compare-and-swap of the whole 16-byte cell, as
// table_merge_str does for strings.  The coarse grouping sets (ROLLUP's () above all) send every row into a handful of
// cells, and most rows do not beat the value they read, so they issue no atomic.  Every write to such a cell in the
// grouping-set kernel is this 16-byte CAS (table_merge's locked path, which stores the two halves separately, is not
// used there), so the 16-byte load never sees a torn value.
__device__ __noinline__ void table_minmax_i128_cas(int kind, unsigned long long slot, int a, Acc128 x) {
  const AggTable& T = PROG.table;
  unsigned long long* cell = T.acc + ((unsigned long long)a * T.cap + slot) * 2;
  const i128 v = make_i128(x.lo, x.hi);
  const ulonglong2 val = make_ulonglong2(x.lo, x.hi);
  ulonglong2 cur = ld_relaxed_b128(cell);
  for (;;) {
    const i128 c = make_i128(cur.x, cur.y);
    if (kind == ACC_MIN_I128 ? !(v < c) : !(v > c)) return;
    const ulonglong2 seen = atom_cas_b128(cell, cur, val);
    if (seen.x == cur.x && seen.y == cur.y) return;
    cur = seen;
  }
}

// Grouping sets (ROLLUP / CUBE / GROUPING SETS): one pass over the input for all PROG.n_sets sets.  A live row loads its
// keys, key hashes and accumulator arguments once, then upserts once per set: the keys masked in the set are NULL, the
// set's __grouping_id is key n_keys, and the table hash combines the id with the hashes of the present keys (the mask is a
// function of the id, so equal groups hash equally).  Compiled only into the pipeline_kernel variant with GSETS = true.
__device__ __noinline__ uint32_t sink_agg_global_gsets(const Lane L, uint32_t active) {
  if (*(volatile unsigned int*)&PROG.status->overflow) return active;
  const int n_keys = PROG.n_keys, n_acc = PROG.n_acc, n_sets = PROG.n_sets;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    if (!((active >> r) & 1)) continue;
    KeyVal row[VM_MAX_KEYS], kv[VM_MAX_KEYS];
    unsigned long long kh[VM_MAX_KEYS];
    for (int k = 0; k < n_keys; k++) {
      load_key(L, PROG.keys[k], r, &row[k]);
      kh[k] = (unsigned long long)ld1_i64(L, PROG.key_hashes[k], r);
    }
    Acc128 x[VM_MAX_ACC];
    uint32_t present = 0;  // accumulators with a (non-NULL) contribution of this row
    for (int a = 0; a < n_acc; a++) {
      const AccDesc ad = PROG.acc[a];
      if (ad.kind != ACC_COUNT_STAR && ad.nullable && !((fetch_valid(L, ad.src) >> r) & 1)) continue;
      present |= 1u << a;
      x[a].lo = 1;
      x[a].hi = 0;
      if (ad.kind == ACC_SUM_I128 || ad.kind == ACC_MIN_I128 || ad.kind == ACC_MAX_I128) {
        i128 v = ld1_i128(L, ad.src, r);
        x[a].lo = lo64(v);
        x[a].hi = ad.zext ? 0ull : hi64(v);
      } else if (ad.kind == ACC_MIN_STR || ad.kind == ACC_MAX_STR) {
        const StrRef s = ld1_str(L, ad.src, r);
        x[a].lo = (uint64_t)s.p;
        x[a].hi = s.len;
      } else if (ad.kind == ACC_SUM_F64) {
        x[a].lo = (uint64_t)__double_as_longlong(ld1_f64(L, ad.src, r));
      } else if (ad.kind == ACC_MIN_F64 || ad.kind == ACC_MAX_F64) {
        x[a].lo = (uint64_t)f64_order_key(ld1_f64(L, ad.src, r));
      }
    }
    for (int s = 0; s < n_sets; s++) {
      const uint32_t mask = PROG.set_mask[s];
      const unsigned long long id = PROG.set_id[s];
      unsigned long long h = hash_i64((int64_t)id);
      for (int k = 0; k < n_keys; k++) {
        if ((mask >> k) & 1) {
          kv[k].w0 = kv[k].w1 = 0;
          kv[k].valid = 0;
          kv[k].vk = row[k].vk;
        } else {
          kv[k] = row[k];
          h = combine_hashes(kh[k], h);
        }
      }
      kv[n_keys].w0 = id;
      kv[n_keys].w1 = 0;
      kv[n_keys].valid = 1;
      kv[n_keys].vk = VK_I64;
      const unsigned long long slot = table_upsert(n_keys + 1, h, kv);
      if (slot == ~0ull) {
        atomicExch(&PROG.status->overflow, 1u);
        active &= ~(1u << r);
        break;
      }
      for (int a = 0; a < n_acc; a++) {
        if (!((present >> a) & 1)) continue;
        const uint8_t kind = PROG.acc[a].kind;
        if (kind == ACC_MIN_I128 || kind == ACC_MAX_I128) table_minmax_i128_cas(kind, slot, a, x[a]);
        else if (kind == ACC_MIN_STR || kind == ACC_MAX_STR) table_merge_str(kind, slot, a, x[a]);
        else table_merge(kind, slot, a, x[a]);
      }
    }
  }
  return active;
}

// ------------------------------------------------------------------------------------------------
// Register-resident aggregate sink: <= VM_REG_GROUPS groups, <= VM_REG_ACC accumulators.
// Every thread keeps the full (group x accumulator) matrix in registers: no atomics and no shared
// memory traffic in the per-row path.  Group ids are dense per CTA (tiny shared-memory key table);
// for a single integer-like key the published keys are cached in registers so that resolving a
// row's group is 4 register compares.
// ------------------------------------------------------------------------------------------------
struct RegGroupTable {  // shared memory
  unsigned long long hash[VM_REG_GROUPS];  // row hash (== the key itself for a single integer-like key)
  unsigned int state[VM_REG_GROUPS];
  unsigned long long key_w0[VM_REG_GROUPS][VM_MAX_KEYS];
  unsigned long long key_w1[VM_REG_GROUPS][VM_MAX_KEYS];
  unsigned char key_valid[VM_REG_GROUPS][VM_MAX_KEYS];
  unsigned int n_groups;
};

// Only the low 64-bit word of each 128-bit accumulator lives in a register; the high word sits in a
// per-thread global scratch slot that is touched only when a carry/borrow actually reaches it
// (never for the small positive addends TPC-H sums are made of), so a thread needs 2 registers per
// (group, accumulator) instead of 4 and 16 warps fit on an SM.
template <int G>
struct RegAggState {
  uint64_t lo[G][VM_REG_ACC];
  uint64_t hi_f64_or_minmax[G][1];  // unused placeholder (keeps the struct non-empty for G variants)
};

__device__ __noinline__ void acc_hi_bump(unsigned long long* cell, uint64_t delta) { *cell += delta; }

__device__ __forceinline__ void acc_lo_add(uint64_t& lo, unsigned long long* hi_cell, i128 v) {
  const uint64_t nl = lo + lo64(v);
  const uint64_t up = hi64(v) + (nl < lo ? 1ull : 0ull);
  lo = nl;
  if (up) acc_hi_bump(hi_cell, up);
}

__device__ __forceinline__ Acc128 acc_identity(int kind) {
  Acc128 x;
  x.lo = 0;
  x.hi = 0;
  switch (kind) {
    case ACC_MIN_I128: x.lo = ~0ull; x.hi = 0x7FFFFFFFFFFFFFFFull; break;
    case ACC_MAX_I128: x.lo = 0; x.hi = 0x8000000000000000ull; break;
    case ACC_MIN_F64: x.lo = 0x7FFFFFFFFFFFFFFFull; break;
    case ACC_MAX_F64: x.lo = 0x8000000000000000ull; break;
    default: break;
  }
  return x;
}

template <int G>
__device__ __forceinline__ void reg_agg_init(RegAggState<G>& S, unsigned long long* hi) {
#pragma unroll
  for (int a = 0; a < VM_REG_ACC; a++) {
    const Acc128 id = acc_identity(a < PROG.n_acc ? PROG.acc[a].kind : ACC_SUM_I128);
#pragma unroll
    for (int g = 0; g < G; g++) {
      S.lo[g][a] = id.lo;
      if (hi) hi[g * VM_REG_ACC + a] = id.hi;
    }
  }
}

// find-or-insert in the CTA's tiny group table; returns the dense group id or -1 when a (G+1)-th
// group shows up
__device__ __noinline__ int reg_group_lookup(RegGroupTable* gt, int G, int n_keys, unsigned long long hh, const KeyVal* kv) {
  for (int g = 0; g < G; g++) {
    unsigned int st = *(volatile unsigned int*)&gt->state[g];
    if (st == 0) {
      unsigned int old = atomicCAS(&gt->state[g], 0u, 1u);
      if (old == 0) {
        gt->hash[g] = hh;
        for (int k = 0; k < n_keys; k++) {
          gt->key_w0[g][k] = kv[k].w0;
          gt->key_w1[g][k] = kv[k].w1;
          gt->key_valid[g][k] = kv[k].valid;
        }
        __threadfence_block();
        atomicExch(&gt->state[g], 2u);
        atomicAdd(&gt->n_groups, 1u);
        return g;
      }
      st = old;
    }
    while (st == 1) st = *(volatile unsigned int*)&gt->state[g];
    if (*(volatile unsigned long long*)&gt->hash[g] != hh) continue;
    __threadfence_block();
    bool eq = true;
    for (int k = 0; k < n_keys && eq; k++)
      eq = key_equal(kv[k], *(volatile unsigned long long*)&gt->key_w0[g][k], *(volatile unsigned long long*)&gt->key_w1[g][k],
                     *(volatile unsigned char*)&gt->key_valid[g][k]);
    if (eq) return g;
  }
  return -1;
}

// slow path of group resolution for row r (generic keys, or a key not yet in the register cache)
__device__ __noinline__ int reg_resolve_row(const Lane L, RegGroupTable* gt, int G, int r) {
  const int n_keys = PROG.n_keys;
  KeyVal kv[VM_MAX_KEYS];
  for (int k = 0; k < n_keys; k++) load_key(L, PROG.keys[k], r, &kv[k]);
  return reg_group_lookup(gt, G, n_keys, (unsigned long long)ld1_i64(L, PROG.key_hash, r), kv);
}

// rare path of the ADD_ONLY register sink: merge one large addend of group g directly into the
// global table (same key -> same slot as the end-of-kernel flush)
__device__ __noinline__ void reg_merge_big(RegGroupTable* gt, int G, int g, int a, i128 v) {
  const int n_keys = PROG.n_keys;
  KeyVal kv[VM_MAX_KEYS];
  unsigned long long h = 0;
  if (G > 1) {
    h = gt->hash[g];
    for (int k = 0; k < n_keys; k++) {
      kv[k].w0 = gt->key_w0[g][k];
      kv[k].w1 = gt->key_w1[g][k];
      kv[k].valid = gt->key_valid[g][k];
      kv[k].vk = PROG.keys[k].vk;
    }
  }
  const unsigned long long slot = table_upsert(n_keys, h, kv);
  if (slot == ~0ull) {
    atomicExch(&PROG.status->overflow, 1u);
    return;
  }
  Acc128 x;
  x.lo = lo64(v);
  x.hi = hi64(v);
  table_merge(ACC_SUM_I128, slot, a, x);
}

// ---- side accumulators of the general register sink: string MIN / MAX and UInt64 MIN / MAX ----------------------------
// Their per-thread state lives in memory, not in the register matrix: the 64-bit value (string: the view's pointer) in
// the acc_side scratch, a string's length in the acc_hi scratch (ACC_STR_NONE: no value yet).  They are folded in by one
// rolled call per tile and merged by their own flush, all of it only in the pipeline_kernel variants instantiated with
// SIDE = true (launched when the program has such an accumulator): every other variant, the fused kernel included,
// compiles exactly as it does without them.
__device__ __forceinline__ bool acc_is_side(const AccDesc& ad) { return ad.kind == ACC_MIN_STR || ad.kind == ACC_MAX_STR || ad.zext; }

__device__ __noinline__ void reg_side_init(unsigned long long* hi, unsigned long long* side) {
  for (int a = 0; a < PROG.n_acc && a < VM_REG_ACC; a++) {
    const AccDesc ad = PROG.acc[a];
    if (!acc_is_side(ad)) continue;
    for (int g = 0; g < VM_REG_GROUPS; g++) {
      const int w = g * VM_REG_ACC + a;
      if (ad.zext) {
        side[w] = ad.kind == ACC_MIN_I128 ? ~0ull : 0ull;  // UInt64 identities: no value orders below / above them
      } else {
        side[w] = 0;
        hi[w] = ACC_STR_NONE;
      }
    }
  }
}

// fold the tile's rows of this thread into its side accumulators; gp: group of row r in byte r
__device__ __noinline__ void reg_side_rows(const Lane L, uint32_t active, uint32_t gp, unsigned long long* hi, unsigned long long* side) {
  for (int a = 0; a < PROG.n_acc && a < VM_REG_ACC; a++) {
    const AccDesc ad = PROG.acc[a];
    if (!acc_is_side(ad)) continue;
    const uint32_t v = ad.nullable ? (active & fetch_valid(L, ad.src)) : active;
    for (int r = 0; r < VM_R; r++) {
      if (!((v >> r) & 1)) continue;
      const int w = (int)((gp >> (8 * r)) & 0xFFu) * VM_REG_ACC + a;
      if (ad.zext) {
        const uint64_t u = (uint64_t)ld1_i64(L, ad.src, r);
        if (ad.kind == ACC_MIN_I128 ? u < side[w] : u > side[w]) side[w] = u;
      } else {
        const StrRef s = ld1_str(L, ad.src, r);
        if (str_beats(ad.kind == ACC_MIN_STR, (uint64_t)s.p, s.len, side[w], hi[w])) {
          side[w] = (uint64_t)s.p;
          hi[w] = s.len;
        }
      }
    }
  }
}

template <int G, bool ADD_ONLY, bool SIDE>
__device__ __forceinline__ uint32_t sink_agg_reg(const Lane L, uint32_t active, RegAggState<G>& S, unsigned long long* hi, unsigned long long* side,
                                                 RegGroupTable* gt, unsigned long long (&dir)[G], uint32_t& dir_n, const AccOp* accops) {
  uint32_t gid[VM_R];
#pragma unroll
  FOR_R gid[r] = 0;
  if (G > 1) {
    int64_t h[VM_R];
    fetch_i64(L, PROG.key_hash, h);
    // `fast`: the hash register holds an injective 64-bit image of the whole key (host guarantees),
    // so equal hash <=> equal key and the register cache can answer without touching memory
    const bool fast = PROG.keys_all_i64 != 0;
#pragma unroll
    FOR_R {
      if ((active >> r) & 1) {
        int g = -1;
        if (fast) {
#pragma unroll
          for (int q = 0; q < G; q++)
            if (q < (int)dir_n && dir[q] == (unsigned long long)h[r]) g = q;
        }
        if (g < 0) {
          g = reg_resolve_row(L, gt, G, r);
          if (fast) {  // refresh the register cache with the published prefix of the table
            uint32_t pub = 0;
#pragma unroll
            for (int q = 0; q < G; q++) {
              const bool ok = (q == (int)pub) && (*(volatile unsigned int*)&gt->state[q] == 2u);
              if (ok) {
                dir[q] = *(volatile unsigned long long*)&gt->hash[q];
                pub++;
              }
            }
            dir_n = pub;
          }
        }
        if (g < 0) {
          atomicExch(&PROG.status->overflow, 1u);  // the host re-runs the pipeline with the global-table sink
          active &= ~(1u << r);
        } else {
          gid[r] = (uint32_t)g;
        }
      }
    }
  }
  // accumulate: static register indexing only
  const int n_acc = PROG.n_acc;
  if (ADD_ONLY) {
    // Every accumulator is a COUNT or an integer/decimal SUM.  Per-thread partial sums are kept as
    // plain int64: a thread sees < 2^16 rows (host-checked) and every addend is range-checked to
    // |v| < 2^46, so the partial cannot overflow and is exact; the rare larger addend bypasses the
    // registers and is merged into the global table directly.
#pragma unroll
    for (int a = 0; a < VM_REG_ACC; a++) {
      if (a >= n_acc) break;
      const AccOp& ao = accops[a];
      int64_t vl[VM_R];
      uint32_t v = active;
      if (ao.sel == SEL_IMM) {
#pragma unroll
        FOR_R vl[r] = (int64_t)ao.imm;
      } else {
        i128 vi[VM_R];
        if (ao.sel == 255) {
          const AccDesc ad = PROG.acc[a];
          if (ad.kind != ACC_COUNT_STAR && ad.nullable) v &= fetch_valid(L, ad.src);
          if (ad.kind == ACC_SUM_I128) {
            fetch_i128(L, ad.src, vi);
          } else {
#pragma unroll
            FOR_R vi[r] = 1;
          }
        } else {
          const uint8_t* p = SRC_BASE(ao.sel, ao.off);
#pragma unroll
          FOR_R vi[r] = ld_w128(p, ao.w, r * L.B + L.tid);
        }
        uint32_t big = 0;
#pragma unroll
        FOR_R {
          vl[r] = (int64_t)lo64(vi[r]);
          const bool small = fits_i64(vi[r]) && vl[r] < (1ll << 46) && vl[r] > -(1ll << 46);
          big |= (small ? 0u : 1u) << r;
        }
        big &= v;
        if (big) {  // rare: exact 128-bit merge straight into the global table
#pragma unroll 1
          for (int r = 0; r < VM_R; r++)
            if ((big >> r) & 1) reg_merge_big(gt, G, (int)gid[r], a, vi[r]);
          v &= ~big;
        }
      }
#pragma unroll
      FOR_R {
#pragma unroll
        for (int g = 0; g < G; g++)
          if (((v >> r) & 1) && (G == 1 || gid[r] == (uint32_t)g)) S.lo[g][a] += (uint64_t)vl[r];
      }
    }
    return active;
  }
#pragma unroll
  for (int a = 0; a < VM_REG_ACC; a++) {
    if (a >= n_acc) break;
    const AccDesc ad = PROG.acc[a];
    uint32_t v = (ad.kind == ACC_COUNT_STAR) ? 0xFFFFFFFFu : (ad.nullable ? fetch_valid(L, ad.src) : 0xFFFFFFFFu);
    v &= active;
    if (ad.kind == ACC_COUNT || ad.kind == ACC_COUNT_STAR || ad.kind == ACC_SUM_I128) {
      i128 vi[VM_R];
      if (ad.kind == ACC_SUM_I128) {
        fetch_i128(L, ad.src, vi);
      } else {
#pragma unroll
        FOR_R vi[r] = 1;
      }
#pragma unroll
      FOR_R {
#pragma unroll
        for (int g = 0; g < G; g++)
          if (((v >> r) & 1) && (G == 1 || gid[r] == (uint32_t)g)) acc_lo_add(S.lo[g][a], &hi[g * VM_REG_ACC + a], vi[r]);
      }
    } else if (ad.kind == ACC_SUM_F64) {
      double vf[VM_R];
      fetch_f64(L, ad.src, vf);
#pragma unroll
      FOR_R {
#pragma unroll
        for (int g = 0; g < G; g++)
          if (((v >> r) & 1) && (G == 1 || gid[r] == (uint32_t)g))
            S.lo[g][a] = (uint64_t)__double_as_longlong(__longlong_as_double((long long)S.lo[g][a]) + vf[r]);
      }
    } else if (ad.kind == ACC_MIN_F64 || ad.kind == ACC_MAX_F64) {
      double vf[VM_R];
      fetch_f64(L, ad.src, vf);
      const bool is_min = ad.kind == ACC_MIN_F64;
#pragma unroll
      FOR_R {
        const long long k = f64_order_key(vf[r]);
#pragma unroll
        for (int g = 0; g < G; g++)
          if (((v >> r) & 1) && (G == 1 || gid[r] == (uint32_t)g)) {
            const long long cur = (long long)S.lo[g][a];
            if (is_min ? k < cur : k > cur) S.lo[g][a] = (uint64_t)k;
          }
      }
    } else if (!SIDE || !acc_is_side(ad)) {
      i128 vi[VM_R];
      fetch_i128(L, ad.src, vi);
      const bool is_min = ad.kind == ACC_MIN_I128;
#pragma unroll
      FOR_R {
#pragma unroll
        for (int g = 0; g < G; g++)
          if (((v >> r) & 1) && (G == 1 || gid[r] == (uint32_t)g)) {
            const i128 cur = make_i128(S.lo[g][a], hi[g * VM_REG_ACC + a]);
            if (is_min ? vi[r] < cur : vi[r] > cur) {
              S.lo[g][a] = lo64(vi[r]);
              hi[g * VM_REG_ACC + a] = hi64(vi[r]);
            }
          }
      }
    }
  }
  if (SIDE) {
    uint32_t gp = 0;
#pragma unroll
    FOR_R gp |= gid[r] << (8 * r);
    reg_side_rows(L, active, gp, hi, side);
  }
  return active;
}

__device__ __noinline__ Acc128 acc_combine(int kind, Acc128 x, Acc128 y) {
  switch (kind) {
    case ACC_COUNT_STAR:
    case ACC_COUNT: x.lo += y.lo; return x;
    case ACC_SUM_I128: {
      uint64_t lo = x.lo + y.lo;
      x.hi += y.hi + (lo < x.lo ? 1 : 0);
      x.lo = lo;
      return x;
    }
    case ACC_SUM_F64: x.lo = (uint64_t)__double_as_longlong(__longlong_as_double((long long)x.lo) + __longlong_as_double((long long)y.lo)); return x;
    case ACC_MIN_F64: return (long long)y.lo < (long long)x.lo ? y : x;
    case ACC_MAX_F64: return (long long)y.lo > (long long)x.lo ? y : x;
    case ACC_MIN_I128: return make_i128(y.lo, y.hi) < make_i128(x.lo, x.hi) ? y : x;
    default: return make_i128(y.lo, y.hi) > make_i128(x.lo, x.hi) ? y : x;
  }
}

// acc_combine plus the side accumulators (a zero-extended UInt64 compares correctly as a 128-bit integer)
__device__ __noinline__ Acc128 acc_combine_side(int kind, Acc128 x, Acc128 y) {
  if (kind == ACC_MIN_STR || kind == ACC_MAX_STR) return str_beats(kind == ACC_MIN_STR, y.lo, y.hi, x.lo, x.hi) ? y : x;
  return acc_combine(kind, x, y);
}

// rolled CTA reduction of scratch[a][thread] -> scratch[a][0], then merge into the global table.  SIDE (general register
// sink only): the side accumulators' values are taken from their scratch first, and strings merge by compare-and-swap.
template <bool SIDE>
__device__ __noinline__ void reg_flush_group(RegGroupTable* gt, Acc128* scratch, int g, int G, int tid, int B) {
  const int n_acc = PROG.n_acc, n_keys = PROG.n_keys;
  if (SIDE) {
    const size_t t = ((size_t)blockIdx.x * B + tid) * (VM_REG_GROUPS * VM_REG_ACC) + (size_t)g * VM_REG_ACC;
    for (int a = 0; a < n_acc; a++)
      if (acc_is_side(PROG.acc[a])) {
        scratch[a * B + tid].lo = PROG.acc_side[t + a];
        scratch[a * B + tid].hi = PROG.acc[a].zext ? 0ull : PROG.acc_hi[t + a];
      }
  }
  __syncthreads();
  for (int n = B; n > 1;) {  // B need not be a power of two
    const int half = (n + 1) >> 1;
    for (int a = 0; a < n_acc; a++)
      if (tid < n - half)
        scratch[a * B + tid] = SIDE ? acc_combine_side(PROG.acc[a].kind, scratch[a * B + tid], scratch[a * B + tid + half])
                                    : acc_combine(PROG.acc[a].kind, scratch[a * B + tid], scratch[a * B + tid + half]);
    __syncthreads();
    n = half;
  }
  if (tid == 0) {
    KeyVal kv[VM_MAX_KEYS];
    unsigned long long h = 0;
    if (G > 1) {
      h = gt->hash[g];
      for (int k = 0; k < n_keys; k++) {
        kv[k].w0 = gt->key_w0[g][k];
        kv[k].w1 = gt->key_w1[g][k];
        kv[k].valid = gt->key_valid[g][k];
        kv[k].vk = PROG.keys[k].vk;
      }
    }
    const unsigned long long slot = table_upsert(n_keys, h, kv);
    if (slot == ~0ull) {
      atomicExch(&PROG.status->overflow, 1u);
    } else {
      for (int a = 0; a < n_acc; a++) {
        const int kind = PROG.acc[a].kind;
        if (SIDE && (kind == ACC_MIN_STR || kind == ACC_MAX_STR)) table_merge_str(kind, slot, a, scratch[a * B]);
        else table_merge(kind, slot, a, scratch[a * B]);
      }
    }
  }
  __syncthreads();
}

// End of kernel: reduce the per-thread matrices over the CTA (through shared memory, one group at a
// time) and merge them into the global table with atomics.
template <int G, bool ADD_ONLY, bool SIDE = false>
__device__ __forceinline__ void reg_agg_flush(RegAggState<G>& S, const unsigned long long* hi, RegGroupTable* gt, Acc128* scratch /*[VM_REG_ACC][B]*/, int tid,
                                              int B) {
  const unsigned int ng = (G == 1) ? 1u : gt->n_groups;
#pragma unroll
  for (int g = 0; g < G; g++) {
    if (g >= (int)ng) break;
#pragma unroll
    for (int a = 0; a < VM_REG_ACC; a++) {
      Acc128 x;
      x.lo = S.lo[g][a];
      x.hi = ADD_ONLY ? (uint64_t)((int64_t)S.lo[g][a] >> 63) : hi[g * VM_REG_ACC + a];
      scratch[a * B + tid] = x;
    }
    reg_flush_group<SIDE>(gt, scratch, g, G, tid, B);
  }
}

__device__ __noinline__ int fused_resolve_slow(RegGroupTable* gt, int G, int n_keys, unsigned long long ck, unsigned long long k0, unsigned long long k1) {
  KeyVal kv[2];
  kv[0].w0 = k0;
  kv[0].w1 = 0;
  kv[0].valid = 1;
  kv[0].vk = VK_I64;
  kv[1].w0 = k1;
  kv[1].w1 = 0;
  kv[1].valid = 1;
  kv[1].vk = VK_I64;
  return reg_group_lookup(gt, G, n_keys, ck, kv);
}

// raw (lo, hi) of a tile operand of width 4 / 8 / 16
__device__ __forceinline__ void ld_raw128(const uint8_t* base, uint32_t w, int e, uint64_t& lo, uint64_t& hi) {
  if (w == 16) {
    const ulonglong2 x = ((const ulonglong2*)base)[e];
    lo = x.x;
    hi = x.y;
  } else {
    const int64_t v = (w == 8) ? ((const int64_t*)base)[e] : (int64_t)((const int32_t*)base)[e];
    lo = (uint64_t)v;
    hi = (uint64_t)(v >> 63);
  }
}
__device__ __forceinline__ uint32_t addsub128(bool minus, uint64_t llo, uint64_t lhi, uint64_t& blo, uint64_t& bhi) {
  // b := lit -/+ b with signed-overflow detection
  const uint64_t xlo = blo, xhi = bhi;
  uint64_t rlo, rhi;
  if (minus) {
    rlo = llo - xlo;
    rhi = lhi - xhi - (llo < xlo ? 1ull : 0ull);
    blo = rlo;
    bhi = rhi;
    return (((int64_t)lhi < 0) != ((int64_t)xhi < 0)) && (((int64_t)rhi < 0) != ((int64_t)lhi < 0)) ? 1u : 0u;
  }
  rlo = llo + xlo;
  rhi = lhi + xhi + (rlo < llo ? 1ull : 0ull);
  blo = rlo;
  bhi = rhi;
  return (((int64_t)lhi < 0) == ((int64_t)xhi < 0)) && (((int64_t)rhi < 0) != ((int64_t)lhi < 0)) ? 1u : 0u;
}

// ------------------------------------------------------------------------------------------------
// Pass 2 of the statistical aggregates (VAR / STDDEV / COVAR / CORR): centred co-moments
// The same lowered program runs twice over the same rows.  Pass 1 (the sinks above) fills each group's count and f64
// sums; pass 2 adds w * (x - mx) * (y - my) + b per row into the co-moment columns (MomDesc), centred on the pass-1 mean
// of the row's group.  Two passes keep the accuracy of a two-pass variance (no cancellation of power sums) without a
// per-slot lock.  This code is compiled only into the pipeline_kernel variants with MOM = true, launched for pass 2.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t mom_valid(const Lane L, const MomDesc& md) {
  return fetch_valid(L, md.x) & fetch_valid(L, md.y) & fetch_valid(L, md.w) & fetch_valid(L, md.b);
}

// one row's terms {w (x - mx) (y - my) + b, w (x - mx), w (y - my)}; a zero weight (an empty partial state) contributes its
// b alone, so that an undefined centre never leaks
struct MomTerm {
  double co, dx, dy;
};
__device__ __noinline__ MomTerm mom_term(const Lane L, int m, int r, double mx, double my) {
  const MomDesc md = PROG.mom[m];
  const double b = md.b.kind == OPD_NONE ? 0.0 : ld1_f64(L, md.b, r);
  const double w = md.w.kind == OPD_NONE ? 1.0 : ld1_f64(L, md.w, r);
  if (w == 0.0) return MomTerm{b, 0.0, 0.0};
  const double dx = w * (ld1_f64(L, md.x, r) - mx), ey = ld1_f64(L, md.y, r) - my;
  return MomTerm{dx * ey + b, dx, w * ey};
}

// the pass-1 centres of co-moment m in table slot `slot`
__device__ __forceinline__ void mom_centre(int m, unsigned long long slot, double& mx, double& my) {
  const AggTable& T = PROG.table;
  const MomDesc md = PROG.mom[m];
  const double n = (double)T.acc[((unsigned long long)md.cnt * T.cap + slot) * 2];
  mx = __longlong_as_double((long long)T.acc[((unsigned long long)md.sx * T.cap + slot) * 2]) / n;
  my = __longlong_as_double((long long)T.acc[((unsigned long long)md.sy * T.cap + slot) * 2]) / n;
}

__device__ __noinline__ uint32_t sink_mom_global(const Lane L, uint32_t active) {
  if (*(volatile unsigned int*)&PROG.status->overflow) return active;
  const int n_keys = PROG.n_keys, n_mom = PROG.n_mom;
  const AggTable& T = PROG.table;
  uint32_t ok[VM_MAX_MOM];
  for (int m = 0; m < n_mom; m++) ok[m] = mom_valid(L, PROG.mom[m]);
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    if (!((active >> r) & 1)) continue;
    KeyVal kv[VM_MAX_KEYS];
    for (int k = 0; k < n_keys; k++) load_key(L, PROG.keys[k], r, &kv[k]);
    const unsigned long long h = n_keys ? (unsigned long long)ld1_i64(L, PROG.key_hash, r) : 0ull;
    const unsigned long long slot = table_upsert(n_keys, h, kv);  // pass 1 published every group: a lookup
    if (slot == ~0ull) {
      atomicExch(&PROG.status->overflow, 1u);
      active &= ~(1u << r);
      continue;
    }
    for (int m = 0; m < n_mom; m++) {
      if (!((ok[m] >> r) & 1)) continue;
      double mx, my;
      mom_centre(m, slot, mx, my);
      const MomTerm t = mom_term(L, m, r, mx, my);
      const unsigned long long c0 = PROG.mom[m].col;
      atomicAdd((double*)&T.acc[(c0 * T.cap + slot) * 2], t.co);
      atomicAdd((double*)&T.acc[((c0 + 1) * T.cap + slot) * 2], t.dx);
      atomicAdd((double*)&T.acc[((c0 + 2) * T.cap + slot) * 2], t.dy);
    }
  }
  return active;
}

// register sink: each CTA looks a group up in the global table once, the first time one of its threads meets the group,
// and keeps the slot and the centres here
struct MomCentres {  // shared memory
  unsigned int state[VM_REG_GROUPS];  // 0: not loaded, 1: loading, 2: ready
  unsigned long long slot[VM_REG_GROUPS];
  double mx[VM_REG_GROUPS][VM_MAX_MOM], my[VM_REG_GROUPS][VM_MAX_MOM];
};
__device__ __forceinline__ MomCentres* mom_centres() {
  __shared__ MomCentres mc;
  return &mc;
}

__device__ __noinline__ void mom_load_centres(RegGroupTable* gt, MomCentres* mc, int G, int g) {
  unsigned int st = *(volatile unsigned int*)&mc->state[g];
  if (st == 0 && atomicCAS(&mc->state[g], 0u, 1u) == 0u) {
    const int n_keys = PROG.n_keys;
    KeyVal kv[VM_MAX_KEYS];
    unsigned long long h = 0;
    if (G > 1) {
      h = gt->hash[g];
      for (int k = 0; k < n_keys; k++) {
        kv[k].w0 = gt->key_w0[g][k];
        kv[k].w1 = gt->key_w1[g][k];
        kv[k].valid = gt->key_valid[g][k];
        kv[k].vk = PROG.keys[k].vk;
      }
    }
    const unsigned long long slot = table_upsert(n_keys, h, kv);
    mc->slot[g] = slot;
    if (slot == ~0ull) atomicExch(&PROG.status->overflow, 1u);
    for (int m = 0; m < PROG.n_mom; m++) {
      double mx = 0.0, my = 0.0;
      if (slot != ~0ull) mom_centre(m, slot, mx, my);
      mc->mx[g][m] = mx;
      mc->my[g][m] = my;
    }
    __threadfence_block();
    atomicExch(&mc->state[g], 2u);
    return;
  }
  while (*(volatile unsigned int*)&mc->state[g] != 2u) {
  }
  __threadfence_block();
}

template <int G>
__device__ __forceinline__ uint32_t sink_mom_reg(const Lane L, uint32_t active, double (&acc)[G][VM_MAX_MOM][3], RegGroupTable* gt, MomCentres* mc) {
  uint32_t gid[VM_R];
#pragma unroll
  FOR_R gid[r] = 0;
#pragma unroll 1
  for (int r = 0; r < VM_R; r++) {
    if (!((active >> r) & 1)) continue;
    const int g = G > 1 ? reg_resolve_row(L, gt, G, r) : 0;
    if (g < 0) {
      atomicExch(&PROG.status->overflow, 1u);
      active &= ~(1u << r);
      continue;
    }
    gid[r] = (uint32_t)g;
    if (*(volatile unsigned int*)&mc->state[g] != 2u) mom_load_centres(gt, mc, G, g);
  }
  __threadfence_block();  // acquire: the centres read below were published before their state became 2
  const int n_mom = PROG.n_mom;
#pragma unroll
  for (int m = 0; m < VM_MAX_MOM; m++) {
    if (m >= n_mom) break;
    const uint32_t v = active & mom_valid(L, PROG.mom[m]);
#pragma unroll
    FOR_R {
      if ((v >> r) & 1) {
        const MomTerm t = mom_term(L, m, r, mc->mx[gid[r]][m], mc->my[gid[r]][m]);
#pragma unroll
        for (int g = 0; g < G; g++)
          if (gid[r] == (uint32_t)g) {
            acc[g][m][0] += t.co;
            acc[g][m][1] += t.dx;
            acc[g][m][2] += t.dy;
          }
      }
    }
  }
  return active;
}

// end of pass 2 in the register sink: a warp reduction per (group, co-moment), then one f64 atomic per warp
template <int G>
__device__ __forceinline__ void mom_reg_flush(double (&acc)[G][VM_MAX_MOM][3], MomCentres* mc, int tid) {
  const int n_mom = PROG.n_mom;
  const AggTable& T = PROG.table;
#pragma unroll
  for (int g = 0; g < G; g++) {
    const bool used = mc->state[g] == 2u && mc->slot[g] != ~0ull;
#pragma unroll
    for (int m = 0; m < VM_MAX_MOM; m++) {
      if (m >= n_mom) break;
#pragma unroll
      for (int j = 0; j < 3; j++) {
        double x = acc[g][m][j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xFFFFFFFFu, x, o);
        if (used && (tid & 31) == 0) atomicAdd((double*)&T.acc[((unsigned long long)(PROG.mom[m].col + j) * T.cap + mc->slot[g]) * 2], x);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// The kernel
// ------------------------------------------------------------------------------------------------
template <int SINK, int G, bool ADD_ONLY, bool SIDE, bool MOM = false, bool SFN = false, bool GSETS = false>
__global__ void __launch_bounds__(512, 1) pipeline_kernel() {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t full_bar[VM_MAX_STAGES];
  __shared__ uint32_t warp_tot[VM_R * 32];
  __shared__ unsigned long long tile_base_sh;
  __shared__ RegGroupTable gtable;
  __shared__ MicroOp mops[VM_MAX_INSTR];
  __shared__ AccOp accops[VM_MAX_ACC];

  const int tid = threadIdx.x, B = blockDim.x;
  const int TILE = B * VM_R;
  const int64_t n_rows = PROG.n_rows;
  const int64_t n_tiles = (n_rows + TILE - 1) / TILE;
  const int S = (int)PROG.n_stages;
  const uint32_t stage_bytes = PROG.stage_bytes;
  const bool use_tma = PROG.use_tma != 0;
  uint8_t* stage0 = smem;
  uint8_t* regs = smem + (size_t)S * stage_bytes;

  if (tid == 0) {
    for (int s = 0; s < S; s++) mbar_init(&full_bar[s], 1);
    mbar_fence_init();
  }
  const int n_instr = PROG.n_instr;
  for (int pc = tid; pc < n_instr; pc += B) decode_micro(pc, &mops[pc]);
  if (SINK == SINK_AGG_REG && !MOM && tid >= 64 && tid < 64 + PROG.n_acc) decode_acc(tid - 64, &accops[tid - 64]);
  if (SINK == SINK_AGG_REG && tid < VM_REG_GROUPS) {
    gtable.state[tid] = 0;
    gtable.hash[tid] = 0;
    if (tid == 0) gtable.n_groups = 0;
    if (MOM) mom_centres()->state[tid] = 0;
  }
  __syncthreads();

  RegAggState<G> S_reg;
  unsigned long long dir[G];
  uint32_t dir_n = 0;
  unsigned long long* acc_hi = nullptr;
  unsigned long long* acc_side = nullptr;
  double macc[MOM ? G : 1][VM_MAX_MOM][3];
  if (MOM) {
#pragma unroll
    for (int g = 0; g < (MOM ? G : 1); g++)
#pragma unroll
      for (int m = 0; m < VM_MAX_MOM; m++) macc[g][m][0] = macc[g][m][1] = macc[g][m][2] = 0.0;
  }
  if (SINK == SINK_AGG_REG && !MOM) {
    if (!ADD_ONLY) acc_hi = PROG.acc_hi + ((size_t)blockIdx.x * B + tid) * (VM_REG_GROUPS * VM_REG_ACC);
    reg_agg_init<G>(S_reg, acc_hi);
    if (SIDE) {
      acc_side = PROG.acc_side + ((size_t)blockIdx.x * B + tid) * (VM_REG_GROUPS * VM_REG_ACC);
      reg_side_init(acc_hi, acc_side);
    }
#pragma unroll
    for (int q = 0; q < G; q++) dir[q] = 0xFFFFFFFFFFFFFFFFull;
  }
  uint32_t live_rows = 0;

  Lane L;
  L.regs = regs;
  L.tid = tid;
  L.B = B;

  // tiles are dealt round-robin: tile(k) = blockIdx.x + k * gridDim.x
  auto tile_of = [&](int64_t k) { return (int64_t)blockIdx.x + k * (int64_t)gridDim.x; };
  auto tile_is_tma = [&](int64_t t) { return use_tma && (t + 1) * (int64_t)TILE <= n_rows; };

  if (tid == 0) {
    for (int k = 0; k < S - 1; k++) {
      int64_t t = tile_of(k);
      if (t < n_tiles && tile_is_tma(t)) issue_tile_tma(stage0 + (size_t)(k % S) * stage_bytes, &full_bar[k % S], t * TILE, TILE);
    }
  }
  uint32_t phase_bits = 0;
  int s = 0;  // k % S, maintained incrementally
  for (int64_t k = 0;; k++, s = (s + 1 == S) ? 0 : s + 1) {
    const int64_t t = tile_of(k);
    if (t >= n_tiles) break;
    uint8_t* stage = stage0 + (size_t)s * stage_bytes;
    // prefetch tile k+S-1 into the buffer released at the end of iteration k-1
    if (tid == 0) {
      const int64_t kn = k + S - 1, tn = tile_of(kn);
      const int sn = (s == 0) ? S - 1 : s - 1;  // (k + S - 1) % S
      if (tn < n_tiles && tile_is_tma(tn)) issue_tile_tma(stage0 + (size_t)sn * stage_bytes, &full_bar[sn], tn * TILE, TILE);
    }
    const int64_t row0 = t * TILE;
    const int rows = (int)((n_rows - row0) < TILE ? (n_rows - row0) : TILE);
    if (tile_is_tma(t)) {
      mbar_wait(&full_bar[s], (phase_bits >> s) & 1);
      phase_bits ^= 1u << s;
    } else {
      load_tile_coop(stage, row0, rows, TILE, tid, B);
      __syncthreads();
    }
    L.stage = stage;
    // the sink-overflow flag is sampled by one thread before the tile's arithmetic (its latency hides
    // behind the compute) and published CTA-uniformly by the end-of-tile barrier
    const unsigned int stop_early = (SINK != SINK_MATERIALIZE && tid == 0) ? *(volatile unsigned int*)&PROG.status->overflow : 0u;
    uint32_t active = 0;
#pragma unroll
    FOR_R if (r * B + tid < rows) active |= 1u << r;
    {
      active = run_program<SFN>(L, active, mops, n_instr);
    }
    if (MOM) {
      if (SINK == SINK_AGG_GLOBAL) active = sink_mom_global(L, active);
      else active = sink_mom_reg<(MOM ? G : 1)>(L, active, macc, &gtable, mom_centres());
      live_rows += __popc(active);
    } else if (SINK == SINK_MATERIALIZE) {
      sink_materialize(L, active, warp_tot, &tile_base_sh, t, n_tiles);
    } else if (SINK == SINK_AGG_GLOBAL) {
      active = GSETS ? sink_agg_global_gsets(L, active) : sink_agg_global(L, active);
      live_rows += __popc(active);
    } else {
      active = sink_agg_reg<G, ADD_ONLY, SIDE>(L, active, S_reg, acc_hi, acc_side, &gtable, dir, dir_n, accops);
      live_rows += __popc(active);
    }
    // everyone is done with this stage buffer (and the VM registers); the sink-overflow flag is
    // sampled CTA-uniformly so that all threads leave the loop together
    if (__syncthreads_or(stop_early != 0)) {
      // drain bulk copies that are still in flight before the CTA may exit
      for (int64_t kk = k + 1; kk < k + S; kk++) {
        const int64_t tt = tile_of(kk);
        if (tt < n_tiles && tile_is_tma(tt)) {
          mbar_wait(&full_bar[kk % S], (phase_bits >> (kk % S)) & 1);
          phase_bits ^= 1u << (kk % S);
        }
      }
      break;
    }
  }
  if (SINK != SINK_MATERIALIZE) {
    live_rows = __reduce_add_sync(0xFFFFFFFFu, live_rows);
    if ((tid & 31) == 0 && live_rows) atomicAdd(&PROG.status->in_active, (unsigned long long)live_rows);
  }
  if (SINK == SINK_AGG_GLOBAL && PROG.n_keys == 0 && blockIdx.x == 0 && tid == 0) {
    // a scalar aggregate owns exactly one output group even if no row survived
    KeyVal none[1];
    if (table_upsert(0, 0ull, none) == ~0ull) atomicExch(&PROG.status->overflow, 1u);
  }
  if (MOM && SINK == SINK_AGG_REG) {
    __syncthreads();
    mom_reg_flush<(MOM ? G : 1)>(macc, mom_centres(), tid);
  } else if (SINK == SINK_AGG_REG) {
    __syncthreads();
    // scalar aggregates emit their single group even when no CTA saw a row: CTA 0 always flushes
    const bool has_rows = tile_of(0) < n_tiles;
    if (has_rows || (G == 1 && blockIdx.x == 0)) reg_agg_flush<G, ADD_ONLY, SIDE>(S_reg, acc_hi, &gtable, (Acc128*)smem, tid, B);
  }
}

}  // namespace b200
#include "fused.cuh"
namespace b200 {

// ------------------------------------------------------------------------------------------------
// Host launcher
// ------------------------------------------------------------------------------------------------
// The running program lives in __constant__ memory, one copy per device.  Up to `concurrent_tasks` host threads
// (and possibly several streams) drive one engine (cpu_bound_executor.rs:94-131), so {upload, launch} is one
// critical section per device, and the upload additionally waits (on the device) for the previous pipeline
// kernel of ANY stream: a pipeline kernel occupies every SM anyway, so nothing is lost by running them one
// after the other, while all the small kernels around them still overlap freely.
struct ProgramGate {
  std::mutex mu;
  cudaEvent_t last = nullptr;
};
static ProgramGate g_gate[64];

struct GateLock {
  ProgramGate& g;
  cudaStream_t st;
  cudaError_t err = cudaSuccess;
  GateLock(cudaStream_t s) : g(g_gate[current_device() & 63]), st(s) {
    g.mu.lock();
    if (!g.last) err = cudaEventCreateWithFlags(&g.last, cudaEventDisableTiming);
    else err = cudaStreamWaitEvent(st, g.last, 0);
  }
  ~GateLock() {
    if (g.last) cudaEventRecord(g.last, st);
    g.mu.unlock();
  }
  static int current_device() {
    int d = 0;
    cudaGetDevice(&d);
    return d;
  }
};

template <bool SFN, int SINK, int G, bool ADD_ONLY, bool SIDE = false, bool MOM = false, bool GSETS = false>
static cudaError_t launch_one(int grid, int block, size_t smem, cudaStream_t st) {
  // the opt-in to large dynamic shared memory is per (function, device) and sticky: raise it only when needed
  static size_t granted[64] = {0};
  const int dev = GateLock::current_device() & 63;
  if (smem > granted[dev]) {
    cudaError_t e = cudaFuncSetAttribute(pipeline_kernel<SINK, G, ADD_ONLY, SIDE, MOM, SFN, GSETS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    granted[dev] = smem;
  }
  launch_kernel(pipeline_kernel<SINK, G, ADD_ONLY, SIDE, MOM, SFN, GSETS>, grid, block, smem, st);
  return cudaGetLastError();
}

bool pipeline_add_only(const Program& P, int grid, int block) {
  bool add_only = true;
  for (int a = 0; a < P.n_acc; a++)
    add_only &= (P.acc[a].kind == ACC_SUM_I128 || P.acc[a].kind == ACC_COUNT || P.acc[a].kind == ACC_COUNT_STAR);
  // exactness bound of the int64 register partials: fewer than 2^16 rows per thread (see sink_agg_reg)
  add_only &= (P.n_rows / ((int64_t)grid * block) + 2 * VM_R) < 60000;
  return add_only;
}

template <bool SFN>
static cudaError_t launch_variant(const Program& P, int reg_groups, int grid, int block, size_t smem, cudaStream_t st) {
  const bool add_only = pipeline_add_only(P, grid, block);
  if (P.mom_pass) {  // pass 2 of VAR / STDDEV / COVAR / CORR
    if (P.sink == SINK_AGG_GLOBAL) return launch_one<SFN, SINK_AGG_GLOBAL, 1, true, false, true>(grid, block, smem, st);
    return reg_groups <= 1 ? launch_one<SFN, SINK_AGG_REG, 1, false, false, true>(grid, block, smem, st)
                           : launch_one<SFN, SINK_AGG_REG, VM_REG_GROUPS, false, false, true>(grid, block, smem, st);
  }
  // grouping sets: the global sink's variant that upserts every row once per set (run_aggregate never gives them another sink)
  if (P.n_sets) return launch_one<SFN, SINK_AGG_GLOBAL, 1, true, false, false, true>(grid, block, smem, st);
  switch (P.sink) {
    case SINK_MATERIALIZE: return launch_one<SFN, SINK_MATERIALIZE, 1, true>(grid, block, smem, st);
    case SINK_AGG_GLOBAL: return launch_one<SFN, SINK_AGG_GLOBAL, 1, true>(grid, block, smem, st);
    default:
      // string / UInt64 MIN / MAX are never add-only
      if (P.has_side_acc) return reg_groups <= 1 ? launch_one<SFN, SINK_AGG_REG, 1, false, true>(grid, block, smem, st) : launch_one<SFN, SINK_AGG_REG, VM_REG_GROUPS, false, true>(grid, block, smem, st);
      if (reg_groups <= 1) return add_only ? launch_one<SFN, SINK_AGG_REG, 1, true>(grid, block, smem, st) : launch_one<SFN, SINK_AGG_REG, 1, false>(grid, block, smem, st);
      return add_only ? launch_one<SFN, SINK_AGG_REG, VM_REG_GROUPS, true>(grid, block, smem, st) : launch_one<SFN, SINK_AGG_REG, VM_REG_GROUPS, false>(grid, block, smem, st);
  }
}

cudaError_t launch_pipeline(const Program& P, int reg_groups, int grid, int block, size_t smem, cudaStream_t st) {
  GateLock gate(st);
  if (gate.err != cudaSuccess) return gate.err;
  // stream-ordered upload of the program into constant memory
  cudaError_t e = cudaMemcpyToSymbolAsync(c_prog, &P, sizeof(Program), 0, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  bool sfn = false;
  for (int i = 0; i < P.n_instr; i++) sfn = sfn || P.code[i].op >= OP_ABS;
  return sfn ? launch_variant<true>(P, reg_groups, grid, block, smem, st) : launch_variant<false>(P, reg_groups, grid, block, smem, st);
}

// exactness bound of the fused kernel's int64 partials: |addend| < 2^40 and (tiles are claimed
// dynamically, so in the worst case one warp handles every tile of its CTA) < 2^22 rows per thread
bool fused_rows_ok(const Program& P, int grid, int block, int rows_per_thread) {
  (void)block;
  return (P.n_rows / ((int64_t)grid * 32) + 2 * rows_per_thread) < (1ll << 22) && P.n_rows < (1ll << 36);
}

cudaError_t launch_fused_pipeline(const Program& P, const FusedSpec& F, FusedShape shape, int reg_groups, int grid, int block, size_t smem, cudaStream_t st,
                                  int* is_static) {
  GateLock gate(st);
  if (gate.err != cudaSuccess) return gate.err;
  cudaError_t e = cudaMemcpyToSymbolAsync(c_prog, &P, sizeof(Program), 0, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  e = cudaMemcpyToSymbolAsync(c_fused, &F, sizeof(FusedSpec), 0, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  return launch_fused(F, shape, reg_groups, grid, block, smem, st, is_static);
}

}  // namespace b200
