// Value converters shared by the CSV scan (csv.cu) and the newline-delimited JSON scan (json.cu): one thread per row
// and column turns a 16-byte view {pointer, length} into the engine's HBM column layout.  Both scans instantiate
// text_convert<FAM, JSON>; with JSON = false the body is the CSV rule (an empty field is NULL), with JSON = true a NULL
// is a null pointer and the view's high length word carries the JSON kind (JsonKind), which must suit the column.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace b200 {

static __device__ __forceinline__ void csv_error(unsigned long long* err, int64_t row, int reason, uint32_t detail) {
  const unsigned long long w = ((unsigned long long)row << 24) | ((unsigned long long)reason << 16) | (detail & 0xFFFFu);
  if (w < *(volatile unsigned long long*)err) atomicMin(err, w);
}

// ---- conversion --------------------------------------------------------------------------------------------------------
static __device__ __forceinline__ bool csv_digit(uint8_t b) { return b >= '0' && b <= '9'; }
static __device__ __forceinline__ uint8_t csv_lower(uint8_t b) { return (b >= 'A' && b <= 'Z') ? (uint8_t)(b + 32) : b; }
static __device__ __forceinline__ bool csv_ieq(const uint8_t* p, uint32_t n, const char* lit) {
  uint32_t k = 0;
  for (; lit[k]; k++)
    if (k >= n || csv_lower(p[k]) != (uint8_t)lit[k]) return false;
  return k == n;
}

// integers: [+-]?digits, '-' only for signed types; range [lo, hi] as i128
static __device__ int csv_parse_int(const uint8_t* p, uint32_t n, bool is_signed, __int128 lo, __int128 hi, __int128* out) {
  uint32_t k = 0;
  bool neg = false;
  if (k < n && (p[k] == '+' || (is_signed && p[k] == '-'))) neg = p[k++] == '-';
  if (k >= n) return CSV_E_INT;
  unsigned __int128 v = 0;
  for (; k < n; k++) {
    if (!csv_digit(p[k])) return CSV_E_INT;
    v = v * 10 + (p[k] - '0');
    if (v > ((unsigned __int128)1 << 65)) return CSV_E_INT_RANGE;
  }
  const __int128 s = neg ? -(__int128)v : (__int128)v;
  if (s < lo || s > hi) return CSV_E_INT_RANGE;
  *out = s;
  return 0;
}

static __device__ int csv_parse_decimal(const uint8_t* p, uint32_t n, int precision, int scale, __int128* out) {
  uint32_t k = 0;
  bool neg = false;
  if (k < n && (p[k] == '+' || p[k] == '-')) neg = p[k++] == '-';
  unsigned __int128 v = 0;
  int int_digits = 0, frac_digits = 0, sig = 0;
  for (; k < n && csv_digit(p[k]); k++) {
    int_digits++;
    if (sig || p[k] != '0') sig++;
    if (sig > 38) return CSV_E_DEC_RANGE;
    v = v * 10 + (p[k] - '0');
  }
  if (k < n && p[k] == '.') {
    k++;
    for (; k < n && csv_digit(p[k]); k++) {
      frac_digits++;
      if (frac_digits > scale) return CSV_E_DEC_SCALE;
      if (sig || p[k] != '0') sig++;
      if (sig > 38) return CSV_E_DEC_RANGE;
      v = v * 10 + (p[k] - '0');
    }
    if (frac_digits == 0) return CSV_E_DEC;
  }
  if (k < n && (p[k] == 'e' || p[k] == 'E')) return CSV_E_DEC_EXP;
  if (k != n || int_digits + frac_digits == 0) return CSV_E_DEC;
  // the value has sig + (scale - frac_digits) digits once scaled: it fits the precision when that is at most p
  if (v != 0 && sig + (scale - frac_digits) > precision) return CSV_E_DEC_RANGE;
  for (int f = frac_digits; f < scale; f++) v *= 10;
  *out = neg ? -(__int128)v : (__int128)v;
  return 0;
}

// exact Date32: YYYY-MM-DD, proleptic Gregorian, days since 1970-01-01
static __device__ int csv_parse_date(const uint8_t* p, uint32_t n, int32_t* out) {
  if (n != 10 || p[4] != '-' || p[7] != '-') return CSV_E_DATE;
  int v[3] = {0, 0, 0};
  const int at[3] = {0, 5, 8}, len[3] = {4, 2, 2};
  for (int f = 0; f < 3; f++)
    for (int k = 0; k < len[f]; k++) {
      const uint8_t b = p[at[f] + k];
      if (!csv_digit(b)) return CSV_E_DATE;
      v[f] = v[f] * 10 + (b - '0');
    }
  const int y = v[0], m = v[1], dd = v[2];
  if (m < 1 || m > 12 || dd < 1) return CSV_E_DATE;
  const bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
  const int mdays[12] = {31, leap ? 29 : 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
  if (dd > mdays[m - 1]) return CSV_E_DATE;
  const int yy = y - (m <= 2);
  const int era = (yy >= 0 ? yy : yy - 399) / 400;
  const int yoe = yy - era * 400;
  const int doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + dd - 1;
  const int doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  *out = era * 146097 + doe - 719468;
  return 0;
}

static __device__ bool csv_valid_utf8(const uint8_t* p, uint32_t n) {
  uint32_t k = 0;
  while (k < n) {
    const uint8_t b = p[k];
    if (b < 0x80) {
      k++;
      continue;
    }
    int len;
    uint32_t cp;
    if (b >= 0xC2 && b <= 0xDF) {
      len = 2;
      cp = b & 0x1F;
    } else if (b >= 0xE0 && b <= 0xEF) {
      len = 3;
      cp = b & 0x0F;
    } else if (b >= 0xF0 && b <= 0xF4) {
      len = 4;
      cp = b & 0x07;
    } else {
      return false;
    }
    if (k + len > n) return false;
    for (int j = 1; j < len; j++) {
      const uint8_t c = p[k + j];
      if ((c & 0xC0) != 0x80) return false;
      cp = (cp << 6) | (c & 0x3F);
    }
    if ((len == 3 && (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF))) || (len == 4 && (cp < 0x10000 || cp > 0x10FFFF))) return false;
    k += len;
  }
  return true;
}

// ---- floats: exact decimal -> binary ------------------------------------------------------------------------------------
// Big unsigned integers for the exact comparison; CSV_BIG_WORDS x 32 bits holds 5^1100 times a 55-bit mantissa.
static const int CSV_BIG_WORDS = 88;
static const int CSV_MAX_DIGITS = 800;  // significant digits kept; any further non-zero digit is a sticky bit
struct CsvBig {
  uint32_t w[CSV_BIG_WORDS];
  int n;
};
static __device__ __forceinline__ void big_set(CsvBig& a, uint64_t v) {
  a.w[0] = (uint32_t)v;
  a.w[1] = (uint32_t)(v >> 32);
  a.n = a.w[1] ? 2 : a.w[0] ? 1 : 0;
}
static __device__ void big_muladd(CsvBig& a, uint32_t m, uint32_t add) {
  uint64_t carry = add;
  for (int i = 0; i < a.n; i++) {
    const uint64_t t = (uint64_t)a.w[i] * m + carry;
    a.w[i] = (uint32_t)t;
    carry = t >> 32;
  }
  if (carry && a.n < CSV_BIG_WORDS) a.w[a.n++] = (uint32_t)carry;
}
static __device__ void big_mul_pow5(CsvBig& a, int e) {
  while (e >= 13) {
    big_muladd(a, 1220703125u, 0);  // 5^13
    e -= 13;
  }
  uint32_t m = 1;
  for (int k = 0; k < e; k++) m *= 5;
  if (m > 1) big_muladd(a, m, 0);
}
// r = a * v (v < 2^64)
static __device__ void big_mul_u64(const CsvBig& a, uint64_t v, CsvBig& r) {
  const uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
  for (int i = 0; i < CSV_BIG_WORDS; i++) r.w[i] = 0;
  r.n = 0;
  for (int pass = 0; pass < 2; pass++) {
    const uint32_t m = pass ? hi : lo;
    if (!m) continue;
    uint64_t carry = 0;
    int i = 0;
    for (; i < a.n; i++) {
      const int j = i + pass;
      if (j >= CSV_BIG_WORDS) break;
      const uint64_t t = (uint64_t)a.w[i] * m + r.w[j] + carry;
      r.w[j] = (uint32_t)t;
      carry = t >> 32;
    }
    for (int j = i + pass; carry && j < CSV_BIG_WORDS; j++) {
      const uint64_t t = (uint64_t)r.w[j] + carry;
      r.w[j] = (uint32_t)t;
      carry = t >> 32;
    }
  }
  r.n = CSV_BIG_WORDS;
  while (r.n > 0 && r.w[r.n - 1] == 0) r.n--;
}
// word i of (a << s)
static __device__ __forceinline__ uint32_t big_word_shl(const CsvBig& a, int s, int i) {
  const int ws = s >> 5, bs = s & 31;
  const int j = i - ws;
  const uint32_t hi = (j >= 0 && j < a.n) ? a.w[j] : 0u;
  if (!bs) return hi;
  const uint32_t lo = (j - 1 >= 0 && j - 1 < a.n) ? a.w[j - 1] : 0u;
  return (hi << bs) | (lo >> (32 - bs));
}
// sign of (a << sa) - (b << sb)
static __device__ int big_cmp_shl(const CsvBig& a, int sa, const CsvBig& b, int sb) {
  const int na = a.n + (sa >> 5) + 1, nb = b.n + (sb >> 5) + 1;
  for (int i = (na > nb ? na : nb) - 1; i >= 0; i--) {
    const uint32_t x = big_word_shl(a, sa, i), y = big_word_shl(b, sb, i);
    if (x != y) return x < y ? -1 : 1;
  }
  return 0;
}

struct CsvDec {
  bool neg, special_inf, special_nan, sticky;
  int nd;        // significant digits kept
  int e10;       // value = D * 10^e10, D = the kept digits as an integer
  uint64_t w;    // the first (up to) 19 kept digits
  int nw;        // how many digits w holds
};

static __device__ int csv_scan_float(const uint8_t* p, uint32_t n, CsvDec& o) {
  o.neg = o.special_inf = o.special_nan = o.sticky = false;
  o.nd = o.e10 = o.nw = 0;
  o.w = 0;
  uint32_t k = 0;
  if (k < n && (p[k] == '+' || p[k] == '-')) o.neg = p[k++] == '-';
  if (k < n && !csv_digit(p[k]) && p[k] != '.') {
    if (csv_ieq(p + k, n - k, "inf") || csv_ieq(p + k, n - k, "infinity")) {
      o.special_inf = true;
      return 0;
    }
    if (csv_ieq(p + k, n - k, "nan")) {
      o.special_nan = true;
      return 0;
    }
    return CSV_E_FLOAT;
  }
  int digits = 0;
  bool frac = false;
  for (; k < n; k++) {
    const uint8_t b = p[k];
    if (b == '.') {
      if (frac) return CSV_E_FLOAT;
      frac = true;
      continue;
    }
    if (!csv_digit(b)) break;
    digits++;
    const int dv = b - '0';
    if (o.nd == 0 && dv == 0) {
      if (frac) o.e10--;
      continue;
    }
    if (o.nd < CSV_MAX_DIGITS) {
      o.nd++;
      if (frac) o.e10--;
      if (o.nw < 19) {
        o.w = o.w * 10 + (uint64_t)dv;
        o.nw++;
      }
    } else {
      if (dv) o.sticky = true;
      if (!frac) o.e10++;
    }
  }
  if (digits == 0) return CSV_E_FLOAT;
  if (k < n && (p[k] == 'e' || p[k] == 'E')) {
    k++;
    bool eneg = false;
    if (k < n && (p[k] == '+' || p[k] == '-')) eneg = p[k++] == '-';
    if (k >= n) return CSV_E_FLOAT;
    int ev = 0;
    for (; k < n; k++) {
      if (!csv_digit(p[k])) return CSV_E_FLOAT;
      if (ev < 100000) ev = ev * 10 + (p[k] - '0');
    }
    o.e10 += eneg ? -ev : ev;
  }
  if (k != n) return CSV_E_FLOAT;
  return 0;
}

// the kept significant digits of the field as a big integer
static __device__ void csv_digits_big(const uint8_t* p, uint32_t n, int nd, CsvBig& D) {
  big_set(D, 0);
  int got = 0;
  uint32_t chunk = 0, mul = 1;
  for (uint32_t k = 0; k < n && got < nd; k++) {
    const uint8_t b = p[k];
    if (b == 'e' || b == 'E') break;
    if (!csv_digit(b)) continue;
    if (got == 0 && b == '0') continue;
    chunk = chunk * 10 + (b - '0');
    mul *= 10;
    got++;
    if (mul == 1000000000u) {
      big_muladd(D, mul, chunk);
      chunk = 0;
      mul = 1;
    }
  }
  if (mul > 1) big_muladd(D, mul, chunk);
}

// correctly rounded (nearest, ties to even) value of the decimal with P mantissa bits (53 / 24); returns the IEEE bits
// of the magnitude
template <int P>
static __device__ uint64_t csv_exact_float(const uint8_t* p, uint32_t n, const CsvDec& dd) {
  const int kmin = P == 53 ? -1074 : -149;
  const int kmax = P == 53 ? 971 : 104;
  const uint64_t top = 1ull << (P - 1);
  const uint64_t inf_bits = P == 53 ? 0x7FF0000000000000ull : 0x7F800000ull;
  const int mag = dd.nd + dd.e10;
  if (mag > (P == 53 ? 310 : 40)) return inf_bits;
  if (mag < (P == 53 ? -324 : -46)) return 0;
  // starting point: w * 10^(e10 + nd - nw) with a double kept normalised by frexp (a few ulps off at most)
  int K = 0;
  double a = frexp((double)dd.w, &K);
  int e = dd.e10 + dd.nd - dd.nw;
  while (e != 0) {
    const int step = e > 0 ? (e > 22 ? 22 : e) : (e < -22 ? -22 : e);
    double pw = 1.0;
    for (int q = 0; q < (step > 0 ? step : -step); q++) pw *= 10.0;
    a = step > 0 ? a * pw : a / pw;
    int ex = 0;
    a = frexp(a, &ex);
    K += ex;
    e -= step;
  }
  // a in [0.5, 1): value ~ a * 2^K = m * 2^k with m in [2^(P-1), 2^P)
  uint64_t m = (uint64_t)ldexp(a, P);
  int k = K - P;
  if (m >= (1ull << P)) {
    m >>= 1;
    k++;
  }
  if (k < kmin) {
    const int sh = kmin - k;
    m = sh >= 64 ? 0 : m >> sh;
    k = kmin;
  }
  if (k > kmax) {
    m = top;
    k = kmax + 1;
  }
  CsvBig L, P5, R;
  csv_digits_big(p, n, dd.nd, L);
  int lexp = 0;
  if (dd.e10 >= 0) {
    big_mul_pow5(L, dd.e10);
    lexp = dd.e10;
  } else {
    lexp = dd.e10;
    big_set(P5, 1);
    big_mul_pow5(P5, -dd.e10);
  }
  // sign of value - H * 2^h
  auto cmp = [&](uint64_t H, int h) -> int {
    int c;
    if (dd.e10 >= 0) {
      big_set(R, H);
      const int d = lexp - h;
      c = d >= 0 ? big_cmp_shl(L, d, R, 0) : big_cmp_shl(L, 0, R, -d);
    } else {
      big_mul_u64(P5, H, R);
      const int d = lexp - h;
      c = d >= 0 ? big_cmp_shl(L, d, R, 0) : big_cmp_shl(L, 0, R, -d);
    }
    if (c == 0 && dd.sticky) c = 1;
    return c;
  };
  for (int it = 0; it < 4096; it++) {
    const bool is_inf = k > kmax;
    if (!is_inf) {
      const int c = cmp(2 * m + 1, k - 1);
      if (c > 0 || (c == 0 && (m & 1))) {
        m++;
        if (m == (1ull << P)) {
          m = top;
          k++;
        }
        continue;
      }
    }
    if (m > 0) {
      const bool edge = m == top && k > kmin;
      const int c = edge ? cmp(4 * m - 1, k - 2) : cmp(2 * m - 1, k - 1);
      if (c < 0 || (c == 0 && (m & 1))) {
        if (edge) {
          m = (1ull << P) - 1;
          k--;
        } else {
          m--;
        }
        continue;
      }
    }
    break;
  }
  if (k > kmax) return inf_bits;
  if (m < top) return m;  // subnormal (k == kmin) or zero
  return ((uint64_t)(k - kmin + 1) << (P - 1)) | (m - top);
}

template <int P>
static __device__ int csv_parse_float(const uint8_t* p, uint32_t n, uint64_t* bits) {
  CsvDec dd;
  const int rc = csv_scan_float(p, n, dd);
  if (rc) return rc;
  const uint64_t sign = dd.neg ? (P == 53 ? 0x8000000000000000ull : 0x80000000ull) : 0;
  if (dd.special_nan) {
    *bits = P == 53 ? 0x7FF8000000000000ull : 0x7FC00000ull;
    return 0;
  }
  if (dd.special_inf) {
    *bits = sign | (P == 53 ? 0x7FF0000000000000ull : 0x7F800000ull);
    return 0;
  }
  if (dd.nd == 0) {
    *bits = sign;
    return 0;
  }
  // Clinger: an exact mantissa and an exact power of ten, one correctly rounded IEEE operation
  if (P == 53 && !dd.sticky && dd.nd <= 15 && dd.e10 >= -22 && dd.e10 <= 22) {
    double pw = 1.0;
    for (int q = 0; q < (dd.e10 >= 0 ? dd.e10 : -dd.e10); q++) pw *= 10.0;
    const double v = dd.e10 >= 0 ? (double)dd.w * pw : (double)dd.w / pw;
    *bits = sign | (uint64_t)__double_as_longlong(v);
    return 0;
  }
  if (P == 24 && !dd.sticky && dd.nd <= 7 && dd.e10 >= -10 && dd.e10 <= 10) {
    float pw = 1.0f;
    for (int q = 0; q < (dd.e10 >= 0 ? dd.e10 : -dd.e10); q++) pw *= 10.0f;
    const float v = dd.e10 >= 0 ? __fmul_rn((float)dd.w, pw) : __fdiv_rn((float)dd.w, pw);
    *bits = sign | (uint64_t)__float_as_uint(v);
    return 0;
  }
  *bits = sign | csv_exact_float<P>(p, n, dd);
  return 0;
}

template <int FAM, bool JSON>
__device__ __forceinline__ void text_convert(const CsvConvertArgs& A) {
  unsigned long long nulls = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < A.n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t* p = (const uint8_t*)A.views[2 * i];
    const uint32_t len = (uint32_t)A.views[2 * i + 1];
    if (JSON ? p == nullptr : len == 0) {
      // CSV: empty or "" is NULL for every type; JSON: null or a missing key ("" is an empty string)
      A.valid[i] = 0;
      nulls++;
      if (!A.nullable) csv_error(A.err, i, CSV_E_NULL, 0);
      if (FAM == CSV_FAM_UTF8) {
        unsigned long long* o = (unsigned long long*)A.out + 2 * i;
        o[0] = (unsigned long long)p;
        o[1] = 0;
      } else {
        uint8_t* o = (uint8_t*)A.out + (size_t)i * A.width;
        for (int b = 0; b < A.width; b++) o[b] = 0;
      }
      continue;
    }
    A.valid[i] = 1;
    int rc = 0;
    const int kind = JSON ? (int)((A.views[2 * i + 1] >> 32) & 0xFF) : 0;
    if (JSON && (FAM == CSV_FAM_BOOL ? kind != JK_TRUE && kind != JK_FALSE
                                     : kind != (FAM == CSV_FAM_DATE || FAM == CSV_FAM_UTF8 ? JK_STRING : JK_NUMBER))) {
      // a value of another JSON kind: refused, the output kept defined
      if (FAM == CSV_FAM_UTF8) {
        unsigned long long* o = (unsigned long long*)A.out + 2 * i;
        o[0] = (unsigned long long)p;
        o[1] = len;
      } else {
        uint8_t* o = (uint8_t*)A.out + (size_t)i * A.width;
        for (int b = 0; b < A.width; b++) o[b] = 0;
      }
      csv_error(A.err, i, JSON_E_KIND, (uint32_t)kind);
      continue;
    }
    if (FAM == CSV_FAM_INT) {
      __int128 v = 0;
      rc = csv_parse_int(p, len, A.is_signed, A.lo, A.hi, &v);
      const uint64_t u = (uint64_t)v;
      uint8_t* o = (uint8_t*)A.out + (size_t)i * A.width;
      if (A.width == 1) *o = (uint8_t)u;
      else if (A.width == 2) *(uint16_t*)o = (uint16_t)u;
      else if (A.width == 4) *(uint32_t*)o = (uint32_t)u;
      else *(uint64_t*)o = u;
    } else if (FAM == CSV_FAM_DEC) {
      __int128 v = 0;
      rc = csv_parse_decimal(p, len, A.precision, A.scale, &v);
      ((__int128*)A.out)[i] = v;
    } else if (FAM == CSV_FAM_F64) {
      uint64_t b = 0;
      rc = csv_parse_float<53>(p, len, &b);
      ((uint64_t*)A.out)[i] = b;
    } else if (FAM == CSV_FAM_F32) {
      uint64_t b = 0;
      rc = csv_parse_float<24>(p, len, &b);
      ((uint32_t*)A.out)[i] = (uint32_t)b;
    } else if (FAM == CSV_FAM_DATE) {
      int32_t v = 0;
      rc = csv_parse_date(p, len, &v);
      ((int32_t*)A.out)[i] = v;
    } else if (FAM == CSV_FAM_BOOL) {
      uint8_t v = 0;
      if (JSON) v = kind == JK_TRUE;
      else if (csv_ieq(p, len, "true")) v = 1;
      else if (!csv_ieq(p, len, "false")) rc = CSV_E_BOOL;
      ((uint8_t*)A.out)[i] = v;
    } else {
      if (!JSON && !csv_valid_utf8(p, len)) rc = CSV_E_UTF8;  // JSON strings are validated while they are tokenized
      unsigned long long* o = (unsigned long long*)A.out + 2 * i;
      o[0] = (unsigned long long)p;
      o[1] = len;
    }
    if (rc) csv_error(A.err, i, rc, 0);
  }
  if (nulls) atomicAdd(A.null_count, nulls);
}

}  // namespace b200
