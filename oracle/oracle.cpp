// ORACLE -- TEST INFRASTRUCTURE ONLY.  Nothing under datafusion-ballista_b200/ links, imports or
// executes this file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference legs may load liboracle.so (as the checker / the timed CPU arm).
//
// What it is: a plain, single-threaded-per-task, column-at-a-time CPU restatement of the
// reference hot path -- a Ballista executor task (ballista/executor/src/execution_engine.rs:235-254)
// pulling a DataFusion operator tree (FilterExec / ProjectionExec / AggregateExec / HashJoinExec /
// SortExec) and hash-repartitioning its output (ballista/core/src/execution_plans/
// shuffle_writer.rs:270-394, sort_shuffle/writer.rs:199-373, partition rule :729-749), plus the
// ShuffleReaderExec side (shuffle_reader.rs:248-318: concatenate all map outputs of a partition).
//
// PARITY STATUS: the operator arithmetic lives in un-vendored crates (datafusion 53.1.0,
// arrow 58.1.0; Cargo.lock:192,2053) and the reference cannot be built here (no rustc/cargo).
// The oracle is pinned against (a) every golden table the reference's own tests hold for this path
// (tests/golden/reference_tests.json, lifted from ballista/client/tests/{context_checks,
// sort_shuffle,context_basic}.rs and shuffle writer unit tests) and (b) two independent engines
// available offline (pyarrow compute/Acero and sqlite3) in tests/test_oracle_*.py.  Rules that no
// reference test asserts (decimal promotion, AVG truncation) are marked [EXT] and restated from
// arrow-rs / DataFusion documented behaviour.  Absolute partition hash values are "parity
// unpinned" by construction (see csrc/common/hash.hpp).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <deque>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../datafusion-ballista_b200/csrc/common/arrow_host.hpp"
#include "../datafusion-ballista_b200/csrc/common/hash.hpp"
#include "../datafusion-ballista_b200/csrc/common/plan.hpp"
#include "../datafusion-ballista_b200/csrc/common/tpch_gen.hpp"
#include "../include/b200exec.h"

using namespace b200;

namespace {

struct ExecError : std::runtime_error {
  int code;
  ExecError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
[[noreturn]] void exec_fail(const std::string& m) { throw ExecError(B200_ERR_EXECUTION, m); }
[[noreturn]] void unsupported(const std::string& m) { throw ExecError(B200_ERR_UNSUPPORTED, m); }

// ------------------------------------------------------------------------------------------------
// Columns
// ------------------------------------------------------------------------------------------------
struct OCol {
  std::string name;
  DataType type;
  bool nullable = true;
  size_t n = 0;
  std::vector<uint8_t> valid;  // empty => all valid
  std::vector<int64_t> i;      // Bool/ints/date/ts
  std::vector<double> f;
  std::vector<i128> d;
  std::vector<std::string> s;

  bool is_valid(size_t r) const { return valid.empty() || valid[r]; }
  void resize(size_t m) {
    n = m;
    switch (type.pk()) {
      case PK::Bool:
      case PK::I64: i.resize(m); break;
      case PK::F64: f.resize(m); break;
      case PK::I128: d.resize(m); break;
      case PK::Str: s.resize(m); break;
    }
    if (!valid.empty()) valid.resize(m, 1);
  }
  void set_null(size_t r) {
    if (valid.empty()) valid.assign(n, 1);
    valid[r] = 0;
  }
  void copy_row_from(const OCol& src, size_t sr, size_t dr) {
    switch (type.pk()) {
      case PK::Bool:
      case PK::I64: i[dr] = src.i[sr]; break;
      case PK::F64: f[dr] = src.f[sr]; break;
      case PK::I128: d[dr] = src.d[sr]; break;
      case PK::Str: s[dr] = src.s[sr]; break;
    }
    if (!src.is_valid(sr)) set_null(dr);
  }
};

OCol make_col(const DataType& t, size_t n, const std::string& name = "") {
  OCol c;
  c.type = t;
  c.name = name;
  c.resize(n);
  return c;
}

struct OBatch {
  std::vector<OCol> cols;
  size_t n = 0;
};

OBatch empty_batch(const Schema& s) {
  OBatch b;
  for (auto& f : s) {
    OCol c = make_col(f.type, 0, f.name);
    c.nullable = f.nullable;
    b.cols.push_back(c);
  }
  return b;
}

OCol take(const OCol& c, const std::vector<int64_t>& idx) {  // idx < 0 => null
  OCol o = make_col(c.type, idx.size(), c.name);
  o.nullable = c.nullable;
  for (size_t k = 0; k < idx.size(); k++) {
    if (idx[k] < 0) {
      o.set_null(k);
      o.nullable = true;
    } else {
      o.copy_row_from(c, (size_t)idx[k], k);
    }
  }
  return o;
}
OBatch take(const OBatch& b, const std::vector<int64_t>& idx) {
  OBatch o;
  o.n = idx.size();
  for (auto& c : b.cols) o.cols.push_back(take(c, idx));
  return o;
}
void append(OBatch& dst, const OBatch& src) {
  if (dst.cols.empty()) {
    dst = src;
    return;
  }
  if (dst.cols.size() != src.cols.size()) exec_fail("concat: column count mismatch");
  for (size_t c = 0; c < dst.cols.size(); c++) {
    OCol& d = dst.cols[c];
    const OCol& s = src.cols[c];
    if (d.type != s.type) exec_fail("concat: type mismatch in column " + d.name + ": " + d.type.str() + " vs " + s.type.str());
    size_t base = d.n;
    if (!s.valid.empty() && d.valid.empty()) d.valid.assign(d.n, 1);
    d.resize(d.n + s.n);
    for (size_t r = 0; r < s.n; r++) d.copy_row_from(s, r, base + r);
  }
  dst.n += src.n;
}

// ------------------------------------------------------------------------------------------------
// Arrow import / export
// ------------------------------------------------------------------------------------------------
OBatch import_batch(ArrowArray* arr, ArrowSchema* sch) {
  int64_t n = 0;
  std::vector<ImportedCol> ics = import_record_batch(arr, sch, &n);
  OBatch b;
  b.n = (size_t)n;
  for (auto& ic : ics) {
    OCol c = make_col(ic.type, (size_t)n, ic.name);
    c.nullable = ic.nullable;
    for (int64_t r = 0; r < n; r++) {
      int64_t p = r + ic.offset;
      bool v = ic.type.id != TypeId::Null && (!ic.validity || ((ic.validity[p >> 3] >> (p & 7)) & 1));
      if (!v) {
        c.set_null((size_t)r);
        continue;
      }
      switch (ic.type.id) {
        case TypeId::Bool: c.i[r] = (ic.data[p >> 3] >> (p & 7)) & 1; break;
        case TypeId::Int8: c.i[r] = ((const int8_t*)ic.data)[p]; break;
        case TypeId::UInt8: c.i[r] = ((const uint8_t*)ic.data)[p]; break;
        case TypeId::Int16: c.i[r] = ((const int16_t*)ic.data)[p]; break;
        case TypeId::UInt16: c.i[r] = ((const uint16_t*)ic.data)[p]; break;
        case TypeId::Int32:
        case TypeId::Date32: c.i[r] = ((const int32_t*)ic.data)[p]; break;
        case TypeId::UInt32: c.i[r] = ((const uint32_t*)ic.data)[p]; break;
        case TypeId::Int64:
        case TypeId::Timestamp: c.i[r] = ((const int64_t*)ic.data)[p]; break;
        case TypeId::UInt64: c.i[r] = (int64_t)((const uint64_t*)ic.data)[p]; break;
        case TypeId::Float32: {
          const uint64_t w = f32_bits_to_f64_bits(((const uint32_t*)ic.data)[p]);
          memcpy(&c.f[r], &w, 8);
          break;
        }
        case TypeId::Float64: c.f[r] = ((const double*)ic.data)[p]; break;
        case TypeId::Decimal128: memcpy(&c.d[r], ic.data + 16 * p, 16); break;
        case TypeId::Utf8: {
          int64_t o0, o1;
          if (ic.large_offsets) {
            o0 = ((const int64_t*)ic.data)[p];
            o1 = ((const int64_t*)ic.data)[p + 1];
          } else {
            o0 = ((const int32_t*)ic.data)[p];
            o1 = ((const int32_t*)ic.data)[p + 1];
          }
          c.s[r].assign((const char*)ic.extra + o0, (size_t)(o1 - o0));
          break;
        }
        default: break;
      }
    }
    b.cols.push_back(std::move(c));
  }
  if (arr->release) arr->release(arr);
  if (sch->release) sch->release(sch);
  return b;
}

void export_batch(const OBatch& b, const Schema* names, ArrowArray* out, ArrowSchema* out_schema) {
  std::vector<HostCol> hcs;
  for (size_t ci = 0; ci < b.cols.size(); ci++) {
    const OCol& c = b.cols[ci];
    HostCol h;
    h.name = names ? (*names)[ci].name : c.name;
    h.type = c.type;
    h.n = (int64_t)c.n;
    h.nullable = true;
    size_t n = c.n;
    if (!c.valid.empty()) {
      h.validity.assign((n + 7) / 8, 0);
      for (size_t r = 0; r < n; r++) {
        if (c.valid[r]) h.validity[r >> 3] |= (uint8_t)(1u << (r & 7));
        else h.null_count++;
      }
      if (h.null_count == 0) h.validity.clear();
    }
    int w = c.type.width();
    switch (c.type.id) {
      case TypeId::Null: h.null_count = (int64_t)n; break;
      case TypeId::Bool:
        h.data.assign((n + 7) / 8, 0);
        for (size_t r = 0; r < n; r++)
          if (c.i[r]) h.data[r >> 3] |= (uint8_t)(1u << (r & 7));
        break;
      case TypeId::Utf8: {
        h.data.resize((n + 1) * 4);
        int32_t off = 0;
        for (size_t r = 0; r < n; r++) {
          memcpy(&h.data[r * 4], &off, 4);
          if (c.is_valid(r)) {
            h.extra.insert(h.extra.end(), c.s[r].begin(), c.s[r].end());
            off += (int32_t)c.s[r].size();
          }
        }
        memcpy(&h.data[n * 4], &off, 4);
        break;
      }
      case TypeId::Float32:
        h.data.resize(n * 4);
        for (size_t r = 0; r < n; r++) {
          uint64_t w;
          memcpy(&w, &c.f[r], 8);
          const uint32_t v = f64_bits_to_f32_bits(w);
          memcpy(&h.data[r * 4], &v, 4);
        }
        break;
      case TypeId::Float64:
        h.data.resize(n * 8);
        if (n) memcpy(h.data.data(), c.f.data(), n * 8);
        break;
      case TypeId::Decimal128:
        h.data.resize(n * 16);
        if (n) memcpy(h.data.data(), c.d.data(), n * 16);
        break;
      default:
        h.data.resize(n * (size_t)w);
        for (size_t r = 0; r < n; r++) memcpy(&h.data[r * (size_t)w], &c.i[r], (size_t)w);  // little endian truncation
    }
    hcs.push_back(std::move(h));
  }
  export_record_batch(std::move(hcs), (int64_t)b.n, out, out_schema);
}

// ------------------------------------------------------------------------------------------------
// Scalar helpers
// ------------------------------------------------------------------------------------------------
i128 checked_mul(i128 a, i128 b) {
  i128 r;
  if (__builtin_mul_overflow(a, b, &r)) exec_fail("Arithmetic overflow: decimal multiply");
  return r;
}
i128 checked_add(i128 a, i128 b) {
  i128 r;
  if (__builtin_add_overflow(a, b, &r)) exec_fail("Arithmetic overflow: decimal add");
  return r;
}
i128 checked_sub(i128 a, i128 b) {
  i128 r;
  if (__builtin_sub_overflow(a, b, &r)) exec_fail("Arithmetic overflow: decimal subtract");
  return r;
}
i128 rescale_up(i128 v, int by) {
  if (by <= 0) return v;
  if (by > 38) exec_fail("Arithmetic overflow: decimal rescale");
  return checked_mul(v, pow10_i128(by));
}
int64_t wrap_int(int64_t v, TypeId t) {
  switch (t) {
    case TypeId::Int8: return (int8_t)v;
    case TypeId::Int16: return (int16_t)v;
    case TypeId::Int32:
    case TypeId::Date32: return (int32_t)v;
    case TypeId::UInt8: return (uint8_t)v;
    case TypeId::UInt16: return (uint16_t)v;
    case TypeId::UInt32: return (uint32_t)v;
    default: return v;
  }
}
// IEEE total order (arrow-ord compares floats with total_cmp [EXT])
int total_cmp(double a, double b) {
  int64_t x, y;
  memcpy(&x, &a, 8);
  memcpy(&y, &b, 8);
  x ^= (int64_t)((uint64_t)(x >> 63) >> 1);
  y ^= (int64_t)((uint64_t)(y >> 63) >> 1);
  return x < y ? -1 : x > y ? 1 : 0;
}
double dec_to_f64(i128 v, int scale) { return (double)v / pow10_f64(scale); }  // arrow: x as f64 / 10_f64.powi(scale)

bool like_match(const char* s, size_t sn, const char* p, size_t pn) {
  // SQL LIKE with % and _ (no escape), bytewise
  size_t si = 0, pi = 0, star_p = (size_t)-1, star_s = 0;
  while (si < sn) {
    if (pi < pn && (p[pi] == '_' || p[pi] == s[si])) {
      if (p[pi] == '%') {
      } else {
        si++;
        pi++;
        continue;
      }
    }
    if (pi < pn && p[pi] == '%') {
      star_p = pi++;
      star_s = si;
      continue;
    }
    if (star_p != (size_t)-1) {
      pi = star_p + 1;
      si = ++star_s;
      continue;
    }
    return false;
  }
  while (pi < pn && p[pi] == '%') pi++;
  return pi == pn;
}

int32_t year_of_days(int64_t z) {  // civil-from-days (proleptic Gregorian)
  z += 719468;
  int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  int64_t doe = z - era * 146097;
  int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  int64_t y = yoe + era * 400;
  int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  int64_t mp = (5 * doy + 2) / 153;
  int64_t m = mp < 10 ? mp + 3 : mp - 9;
  return (int32_t)(y + (m <= 2));
}

// ------------------------------------------------------------------------------------------------
// Expression evaluation (column-at-a-time, like PhysicalExpr::evaluate)
// ------------------------------------------------------------------------------------------------
OCol eval(const Expr& e, const OBatch& b);

// numeric view of a column as decimal(scale) / double
i128 as_dec(const OCol& c, size_t r) {
  if (c.type.is_decimal()) return c.d[r];
  return c.type.id == TypeId::UInt64 ? (i128)(uint64_t)c.i[r] : (i128)c.i[r];
}
int dec_scale(const OCol& c) { return c.type.is_decimal() ? c.type.scale : 0; }
double as_f64(const OCol& c, size_t r) {
  switch (c.type.pk()) {
    case PK::F64: return c.f[r];
    case PK::I128: return dec_to_f64(c.d[r], c.type.scale);
    default: return c.type.id == TypeId::UInt64 ? (double)(uint64_t)c.i[r] : (double)c.i[r];
  }
}

int compare_values(const OCol& a, size_t ra, const OCol& b, size_t rb) {
  PK pa = a.type.pk(), pb = b.type.pk();
  if (pa == PK::Str && pb == PK::Str) {
    int c = a.s[ra].compare(b.s[rb]);
    return c < 0 ? -1 : c > 0 ? 1 : 0;
  }
  if (pa == PK::F64 || pb == PK::F64) return total_cmp(as_f64(a, ra), as_f64(b, rb));
  if (pa == PK::I128 || pb == PK::I128) {
    int sa = dec_scale(a), sb = dec_scale(b), s = std::max(sa, sb);
    i128 x = rescale_up(as_dec(a, ra), s - sa), y = rescale_up(as_dec(b, rb), s - sb);
    return x < y ? -1 : x > y ? 1 : 0;
  }
  if (a.type.id == TypeId::UInt64 && b.type.id == TypeId::UInt64) {
    uint64_t x = (uint64_t)a.i[ra], y = (uint64_t)b.i[rb];
    return x < y ? -1 : x > y ? 1 : 0;
  }
  int64_t x = a.i[ra], y = b.i[rb];
  return x < y ? -1 : x > y ? 1 : 0;
}

OCol eval_arith(const Expr& e, const OCol& l, const OCol& r) {
  size_t n = l.n;
  const DataType& rt = e.type;
  OCol o = make_col(rt, n);
  for (size_t k = 0; k < n; k++) {
    if (!l.is_valid(k) || !r.is_valid(k)) {
      o.set_null(k);
      continue;
    }
    if (rt.is_float()) {
      double x = as_f64(l, k), y = as_f64(r, k), z = 0;
      switch (e.op) {
        case BinOp::Add: z = x + y; break;
        case BinOp::Sub: z = x - y; break;
        case BinOp::Mul: z = x * y; break;
        case BinOp::Div: z = x / y; break;
        case BinOp::Mod: z = std::fmod(x, y); break;
        default: break;
      }
      o.f[k] = rt.id == TypeId::Float32 ? (double)(float)z : z;
    } else if (rt.is_decimal()) {
      DataType lt = l.type.is_decimal() ? l.type : int_as_decimal(l.type);
      DataType rtt = r.type.is_decimal() ? r.type : int_as_decimal(r.type);
      i128 x = as_dec(l, k), y = as_dec(r, k);
      int s1 = lt.scale, s2 = rtt.scale;
      switch (e.op) {
        case BinOp::Add: o.d[k] = checked_add(rescale_up(x, rt.scale - s1), rescale_up(y, rt.scale - s2)); break;
        case BinOp::Sub: o.d[k] = checked_sub(rescale_up(x, rt.scale - s1), rescale_up(y, rt.scale - s2)); break;
        case BinOp::Mul: o.d[k] = checked_mul(x, y); break;
        case BinOp::Div: {
          if (y == 0) exec_fail("Divide by zero");
          int mul_pow = rt.scale - s1 + s2;
          o.d[k] = rescale_up(x, mul_pow) / y;  // truncates toward zero (i128::div_checked) [EXT]
          break;
        }
        case BinOp::Mod: {
          if (y == 0) exec_fail("Divide by zero");
          int s = std::max(s1, s2);
          o.d[k] = rescale_up(x, s - s1) % rescale_up(y, s - s2);
          break;
        }
        default: break;
      }
    } else {
      int64_t x = l.i[k], y = r.i[k], z = 0;
      switch (e.op) {  // DataFusion uses the wrapping kernels for + - * on integers [EXT]
        case BinOp::Add: z = (int64_t)((uint64_t)x + (uint64_t)y); break;
        case BinOp::Sub: z = (int64_t)((uint64_t)x - (uint64_t)y); break;
        case BinOp::Mul: z = (int64_t)((uint64_t)x * (uint64_t)y); break;
        case BinOp::Div:  // arrow's div_checked: a quotient outside the type (its minimum / -1) is an error
          if (y == 0) exec_fail("Divide by zero");
          if (rt.id == TypeId::UInt64) {
            z = (int64_t)((uint64_t)x / (uint64_t)y);
            break;
          }
          if (x == INT64_MIN && y == -1) exec_fail("Arithmetic overflow: integer divide");
          z = x / y;
          if (wrap_int(z, rt.id) != z) exec_fail("Arithmetic overflow: integer divide");
          break;
        case BinOp::Mod:  // the dividend's sign; MIN % -1 is 0 [EXT]
          if (y == 0) exec_fail("Divide by zero");
          if (rt.id == TypeId::UInt64) z = (int64_t)((uint64_t)x % (uint64_t)y);
          else z = (y == -1) ? 0 : x % y;
          break;
        default: break;
      }
      o.i[k] = wrap_int(z, rt.id);
    }
  }
  return o;
}

OCol eval_cast(const OCol& c, const DataType& to) {
  if (c.type == to) return c;
  size_t n = c.n;
  OCol o = make_col(to, n, c.name);
  PK from = c.type.pk(), dst = to.pk();
  for (size_t k = 0; k < n; k++) {
    if (!c.is_valid(k)) {
      o.set_null(k);
      continue;
    }
    if (dst == PK::I64 && from == PK::I64) {
      int64_t v = c.i[k];
      // arrow "safe" cast: overflow -> NULL [EXT]; a negative 64-bit image is a negative value going to UInt64 or a
      // UInt64 at or above 2^63 going to another type
      const bool sign_bad = v < 0 && c.type.is_integer() && to.is_integer() && ((c.type.id == TypeId::UInt64) != (to.id == TypeId::UInt64));
      if (sign_bad || wrap_int(v, to.id) != v) o.set_null(k);
      else o.i[k] = v;
    } else if (dst == PK::I64 && from == PK::Bool) {
      o.i[k] = c.i[k];
    } else if (dst == PK::Bool && from == PK::I64) {
      o.i[k] = c.i[k] != 0;
    } else if (dst == PK::F64 && from == PK::I64 && to.id == TypeId::Float32) {  // rounded once, as Rust's `as f32`
      o.f[k] = c.type.id == TypeId::UInt64 ? (double)(float)(uint64_t)c.i[k] : (double)(float)c.i[k];
    } else if (dst == PK::F64 && (from == PK::I64 || from == PK::F64 || from == PK::I128)) {
      double v = as_f64(c, k);
      o.f[k] = to.id == TypeId::Float32 ? (double)(float)v : v;
    } else if (dst == PK::I64 && from == PK::F64) {
      double v = std::trunc(c.f[k]);
      if (to.id == TypeId::UInt64) {
        if (!(v >= 0.0 && v < 1.8446744073709552e19)) o.set_null(k);
        else o.i[k] = (int64_t)(uint64_t)v;
      } else if (!(v >= -9.2233720368547758e18 && v < 9.2233720368547758e18) || wrap_int((int64_t)v, to.id) != (int64_t)v) {
        o.set_null(k);
      } else {
        o.i[k] = (int64_t)v;
      }
    } else if (dst == PK::I128 && from == PK::I64) {
      i128 v = rescale_up(as_dec(c, k), to.scale);
      if (v >= pow10_i128(to.precision) || v <= -pow10_i128(to.precision)) exec_fail("cast: value does not fit " + to.str());
      o.d[k] = v;
    } else if (dst == PK::I128 && from == PK::I128) {
      int ds = to.scale - c.type.scale;
      i128 v = c.d[k];
      if (ds >= 0) {
        v = rescale_up(v, ds);
      } else {  // round half away from zero (arrow-cast convert_to_smaller_scale_decimal) [EXT]
        i128 div = pow10_i128(-ds), half = div / 2;
        i128 q = v / div, rem = v % div;
        if (v >= 0 && rem >= half) q += 1;
        else if (v < 0 && rem <= -half) q -= 1;
        v = q;
      }
      if (v >= pow10_i128(to.precision) || v <= -pow10_i128(to.precision)) o.set_null(k);
      else o.d[k] = v;
    } else if (dst == PK::I128 && from == PK::F64) {
      double v = std::round(c.f[k] * pow10_f64(to.scale));  // half away from zero; beyond the precision: NULL
      if (!(std::fabs(v) < 1.7e38) || (i128)v >= pow10_i128(to.precision) || (i128)v <= -pow10_i128(to.precision)) o.set_null(k);
      else o.d[k] = (i128)v;
    } else if (dst == PK::I64 && from == PK::I128) {
      i128 v = c.d[k] / pow10_i128(c.type.scale);  // truncation toward zero [EXT]
      if (to.id == TypeId::UInt64) {
        if (v < 0 || v > (i128)UINT64_MAX) o.set_null(k);
        else o.i[k] = (int64_t)(uint64_t)v;
      } else if (v > INT64_MAX || v < INT64_MIN || wrap_int((int64_t)v, to.id) != (int64_t)v) {
        o.set_null(k);
      } else {
        o.i[k] = (int64_t)v;
      }
    } else if (dst == PK::Str && from == PK::Str) {
      o.s[k] = c.s[k];
    } else if (dst == PK::Str && from == PK::I64) {
      o.s[k] = std::to_string(c.i[k]);
    } else {
      unsupported("cast " + c.type.str() + " -> " + to.str());
    }
  }
  return o;
}

OCol eval(const Expr& e, const OBatch& b) {
  size_t n = b.n;
  switch (e.kind) {
    case Expr::Col: return b.cols[(size_t)e.col];
    case Expr::Lit: {
      OCol o = make_col(e.type, n);
      for (size_t k = 0; k < n; k++) {
        if (e.lit.is_null) {
          o.set_null(k);
          continue;
        }
        switch (e.type.pk()) {
          case PK::Bool:
          case PK::I64: o.i[k] = e.lit.i; break;
          case PK::F64: o.f[k] = e.lit.f; break;
          case PK::I128: o.d[k] = e.lit.d; break;
          case PK::Str: o.s[k] = e.lit.s; break;
        }
      }
      if (e.lit.is_null && n == 0) o.valid.clear();
      return o;
    }
    case Expr::Bin: {
      OCol l = eval(*e.args[0], b), r = eval(*e.args[1], b);
      if (is_arith(e.op)) return eval_arith(e, l, r);
      OCol o = make_col(DataType(TypeId::Bool), n);
      if (is_logic(e.op)) {  // Kleene logic
        for (size_t k = 0; k < n; k++) {
          bool lv = l.is_valid(k), rv = r.is_valid(k);
          bool x = lv && l.i[k], y = rv && r.i[k];
          if (e.op == BinOp::And) {
            if ((lv && !x) || (rv && !y)) o.i[k] = 0;
            else if (lv && rv) o.i[k] = 1;
            else o.set_null(k);
          } else {
            if (x || y) o.i[k] = 1;
            else if (lv && rv) o.i[k] = 0;
            else o.set_null(k);
          }
        }
        return o;
      }
      for (size_t k = 0; k < n; k++) {
        if (!l.is_valid(k) || !r.is_valid(k)) {
          o.set_null(k);
          continue;
        }
        int c = compare_values(l, k, r, k);
        bool v = false;
        switch (e.op) {
          case BinOp::Eq: v = c == 0; break;
          case BinOp::Ne: v = c != 0; break;
          case BinOp::Lt: v = c < 0; break;
          case BinOp::Le: v = c <= 0; break;
          case BinOp::Gt: v = c > 0; break;
          case BinOp::Ge: v = c >= 0; break;
          default: break;
        }
        o.i[k] = v;
      }
      return o;
    }
    case Expr::Not: {
      OCol x = eval(*e.args[0], b);
      OCol o = make_col(DataType(TypeId::Bool), n);
      for (size_t k = 0; k < n; k++) {
        if (!x.is_valid(k)) o.set_null(k);
        else o.i[k] = !x.i[k];
      }
      return o;
    }
    case Expr::Neg: {
      OCol x = eval(*e.args[0], b);
      for (size_t k = 0; k < n; k++) {
        switch (x.type.pk()) {
          case PK::F64: x.f[k] = -x.f[k]; break;
          case PK::I128: x.d[k] = (i128)(0 - (u128)x.d[k]); break;
          default: x.i[k] = wrap_int((int64_t)(0 - (uint64_t)x.i[k]), x.type.id);
        }
      }
      return x;
    }
    case Expr::IsNull:
    case Expr::IsNotNull: {
      OCol x = eval(*e.args[0], b);
      OCol o = make_col(DataType(TypeId::Bool), n);
      for (size_t k = 0; k < n; k++) o.i[k] = (e.kind == Expr::IsNull) ? !x.is_valid(k) : x.is_valid(k);
      return o;
    }
    case Expr::Cast: return eval_cast(eval(*e.args[0], b), e.type);
    case Expr::Case: {  // DataFusion's CaseExpr: each WHEN on the rows left, each THEN / the ELSE on the rows it takes
      OCol o = make_col(e.type, n);
      for (size_t k = 0; k < n; k++) o.set_null(k);
      std::vector<int64_t> rem(n);
      for (size_t k = 0; k < n; k++) rem[k] = (int64_t)k;
      auto on_rows = [&](const Expr& x, const std::vector<int64_t>& rows) {  // x over those rows (its columns only)
        std::vector<uint8_t> used(b.cols.size(), 0);
        std::function<void(const Expr&)> mark = [&](const Expr& y) {
          if (y.kind == Expr::Col && (size_t)y.col < used.size()) used[(size_t)y.col] = 1;
          for (auto& a : y.args) mark(*a);
        };
        mark(x);
        OBatch sub;
        sub.n = rows.size();
        for (size_t i = 0; i < b.cols.size(); i++) sub.cols.push_back(used[i] ? take(b.cols[i], rows) : make_col(b.cols[i].type, 0));
        return eval(x, sub);
      };
      auto put = [&](const OCol& v, size_t j, size_t k) {
        o.copy_row_from(v, j, k);
        if (v.is_valid(j)) o.valid[k] = 1;
      };
      size_t npairs = (e.args.size() - (e.has_else ? 1 : 0)) / 2;
      for (size_t w = 0; w < npairs && !rem.empty(); w++) {
        OCol c = on_rows(*e.args[2 * w], rem);
        std::vector<int64_t> hit, left;
        for (size_t j = 0; j < rem.size(); j++) (c.is_valid(j) && c.i[j] ? hit : left).push_back(rem[j]);
        if (!hit.empty()) {
          OCol v = eval_cast(on_rows(*e.args[2 * w + 1], hit), e.type);
          for (size_t j = 0; j < hit.size(); j++) put(v, j, (size_t)hit[j]);
        }
        rem.swap(left);
      }
      if (e.has_else && !rem.empty()) {
        OCol v = eval_cast(on_rows(*e.args.back(), rem), e.type);
        for (size_t j = 0; j < rem.size(); j++) put(v, j, (size_t)rem[j]);
      }
      return o;
    }
    case Expr::InList: {
      OCol x = eval(*e.args[0], b);
      std::vector<OCol> items;
      for (size_t a = 1; a < e.args.size(); a++) items.push_back(eval(*e.args[a], b));
      OCol o = make_col(DataType(TypeId::Bool), n);
      for (size_t k = 0; k < n; k++) {
        if (!x.is_valid(k)) {
          o.set_null(k);
          continue;
        }
        bool found = false, saw_null = false;
        for (auto& it : items) {
          if (!it.is_valid(k)) saw_null = true;
          else if (compare_values(x, k, it, k) == 0) found = true;
        }
        if (found) o.i[k] = !e.negated;
        else if (saw_null) o.set_null(k);
        else o.i[k] = e.negated;
      }
      return o;
    }
    case Expr::Like: {
      OCol x = eval(*e.args[0], b);
      OCol o = make_col(DataType(TypeId::Bool), n);
      for (size_t k = 0; k < n; k++) {
        if (!x.is_valid(k)) {
          o.set_null(k);
          continue;
        }
        bool m = like_match(x.s[k].data(), x.s[k].size(), e.pattern.data(), e.pattern.size());
        o.i[k] = e.negated ? !m : m;
      }
      return o;
    }
    case Expr::Fn: {
      if (e.fn == "date_part_year") {
        OCol x = eval(*e.args[0], b);
        OCol o = make_col(e.type, n);
        for (size_t k = 0; k < n; k++) {
          if (!x.is_valid(k)) o.set_null(k);
          else o.i[k] = year_of_days(x.i[k]);
        }
        return o;
      }
      if (e.fn == "substr") {  // substr(s, start[, len]); 1-based; bytewise (ASCII data)
        OCol x = eval(*e.args[0], b), st = eval(*e.args[1], b);
        OCol ln;
        bool has_len = e.args.size() > 2;
        if (has_len) ln = eval(*e.args[2], b);
        OCol o = make_col(e.type, n);
        for (size_t k = 0; k < n; k++) {
          if (!x.is_valid(k) || !st.is_valid(k) || (has_len && !ln.is_valid(k))) {
            o.set_null(k);
            continue;
          }
          int64_t start = st.i[k], len = has_len ? ln.i[k] : (int64_t)x.s[k].size() + 1;
          if (has_len && len < 0) exec_fail("negative substring length not allowed");
          int64_t s0 = start - 1, e0 = has_len ? s0 + len : (int64_t)x.s[k].size();
          s0 = std::max<int64_t>(0, s0);
          e0 = std::min<int64_t>((int64_t)x.s[k].size(), e0);
          o.s[k] = e0 > s0 ? x.s[k].substr((size_t)s0, (size_t)(e0 - s0)) : std::string();
        }
        return o;
      }
      unsupported("scalar function " + e.fn);
    }
  }
  unsupported("expression kind");
}

// ------------------------------------------------------------------------------------------------
// Row key encoding (group-by / join keys)
// ------------------------------------------------------------------------------------------------
// floats are encoded by their bit pattern, for group and join keys alike: equal when `=` says so, -0.0 <> 0.0, NaN = NaN
// only with the same payload
static inline bool encode_key_col(const OCol& c, size_t r, std::string& out) {
  if (!c.is_valid(r)) {
    out.push_back('\0');
    return false;
  }
  out.push_back('\1');
  switch (c.type.pk()) {
    case PK::Bool:
    case PK::I64: out.append((const char*)&c.i[r], 8); break;
    case PK::F64: out.append((const char*)&c.f[r], 8); break;
    case PK::I128: out.append((const char*)&c.d[r], 16); break;
    case PK::Str: {
      uint32_t len = (uint32_t)c.s[r].size();
      out.append((const char*)&len, 4);
      out.append(c.s[r]);
      break;
    }
  }
  return true;
}
bool encode_key(const std::vector<OCol>& keys, size_t r, std::string& out) {  // returns false if any key is NULL
  out.clear();
  bool all_valid = true;
  for (auto& c : keys) all_valid &= encode_key_col(c, r, out);
  return all_valid;
}
bool encode_key(const std::vector<const OCol*>& keys, size_t r, std::string& out) {  // same, over borrowed columns
  out.clear();
  bool all_valid = true;
  for (auto* c : keys) all_valid &= encode_key_col(*c, r, out);
  return all_valid;
}

uint64_t row_hash(const std::vector<OCol>& keys, size_t r) {  // structure of create_hashes [EXT]; see hash.hpp
  uint64_t h = 0;
  bool first = true;
  for (auto& c : keys) {
    if (c.is_valid(r)) {
      uint64_t v;
      switch (c.type.pk()) {
        case PK::F64: v = hash_f64(c.f[r]); break;
        case PK::I128: v = hash_i128((uint64_t)c.d[r], (uint64_t)((u128)c.d[r] >> 64)); break;
        case PK::Str: v = hash_bytes((const uint8_t*)c.s[r].data(), (uint32_t)c.s[r].size()); break;
        default: v = hash_i64(c.i[r]);
      }
      h = first ? v : combine_hashes(v, h);
    }
    first = false;
  }
  return h;
}

// ------------------------------------------------------------------------------------------------
// Aggregation
// ------------------------------------------------------------------------------------------------
struct Acc {
  bool has = false;
  int64_t cnt = 0;
  int64_t si = 0;
  i128 sd = 0;
  double sf = 0, comp = 0;  // Neumaier compensated sum
  int64_t mi = 0;
  double mf = 0;
  i128 md = 0;
  std::string ms;
  void add_f64(double v) {
    double t = sf + v;
    if (std::fabs(sf) >= std::fabs(v)) comp += (sf - t) + v;
    else comp += (v - t) + sf;
    sf = t;
  }
  double f64_sum() const { return sf + comp; }
};

void acc_minmax(Acc& a, const OCol& c, size_t r, bool is_min) {
  if (!a.has) {
    a.has = true;
    switch (c.type.pk()) {
      case PK::F64: a.mf = c.f[r]; break;
      case PK::I128: a.md = c.d[r]; break;
      case PK::Str: a.ms = c.s[r]; break;
      default: a.mi = c.i[r];
    }
    return;
  }
  switch (c.type.pk()) {
    case PK::F64: {
      int cm = total_cmp(c.f[r], a.mf);
      if (is_min ? cm < 0 : cm > 0) a.mf = c.f[r];
      break;
    }
    case PK::I128:
      if (is_min ? c.d[r] < a.md : c.d[r] > a.md) a.md = c.d[r];
      break;
    case PK::Str:
      if (is_min ? c.s[r] < a.ms : c.s[r] > a.ms) a.ms = c.s[r];
      break;
    default:
      if (c.type.id == TypeId::UInt64) {
        if (is_min ? (uint64_t)c.i[r] < (uint64_t)a.mi : (uint64_t)c.i[r] > (uint64_t)a.mi) a.mi = c.i[r];
      } else if (is_min ? c.i[r] < a.mi : c.i[r] > a.mi) {
        a.mi = c.i[r];
      }
  }
}

OBatch do_aggregate(const PlanNode& node, const OBatch& in) {
  bool from_states = agg_mode_consumes_states(node.agg_mode);
  bool emit_states = agg_mode_emits_states(node.agg_mode);
  size_t ng = node.group_by.size(), na = node.aggs.size();
  // plain column references (keys, aggregate arguments, state columns) are borrowed from `in`; only
  // computed expressions are materialised (into `store`, a deque so that the addresses stay put)
  std::deque<OCol> store;
  auto borrow = [&](const Expr& e) -> const OCol* {
    if (e.kind == Expr::Col && e.col >= 0 && (size_t)e.col < in.cols.size()) return &in.cols[(size_t)e.col];
    store.push_back(eval(e, in));
    return &store.back();
  };
  std::vector<const OCol*> keys;
  for (auto& g : node.group_by) keys.push_back(borrow(*g.expr));
  // inputs per aggregate: raw: [arg]; from states: the state columns
  std::vector<std::vector<const OCol*>> ainp(na);
  size_t sc = ng;
  for (size_t a = 0; a < na; a++) {
    const AggExpr& ae = node.aggs[a];
    if (from_states) {
      for (int k = 0; k < ae.n_state_cols(); k++) ainp[a].push_back(&in.cols.at(sc++));
    } else if (ae.arg) {
      const OCol* c = borrow(*ae.arg);
      if (ae.fn == AggFn::Avg && !c->type.is_decimal()) {
        store.push_back(eval_cast(*c, DataType(TypeId::Float64)));
        c = &store.back();
      }
      ainp[a].push_back(c);
    }
  }
  struct AinRow {  // keeps the body below reading `ain[a][k]` as a column
    const std::vector<const OCol*>* v;
    const OCol& operator[](size_t k) const { return *(*v)[k]; }
  };
  struct AinAll {
    const std::vector<std::vector<const OCol*>>* v;
    AinRow operator[](size_t a) const { return AinRow{&(*v)[a]}; }
  } ain{&ainp};
  std::unordered_map<std::string, size_t> index;
  std::vector<size_t> first_row;
  std::vector<std::vector<Acc>> accs;  // [group][agg]
  std::string k;
  if (ng == 0) {  // scalar aggregate: always exactly one group, even on empty input
    first_row.push_back(0);
    accs.emplace_back(na);
  }
  for (size_t r = 0; r < in.n; r++) {
    size_t g = 0;
    if (ng) {
      encode_key(keys, r, k);
      auto it = index.find(k);
      if (it == index.end()) {
        g = accs.size();
        index.emplace(k, g);
        first_row.push_back(r);
        accs.emplace_back(na);
      } else {
        g = it->second;
      }
    }
    for (size_t a = 0; a < na; a++) {
      const AggExpr& ae = node.aggs[a];
      Acc& ac = accs[g][a];
      if (from_states) {
        const OCol& s0 = ain[a][0];
        switch (ae.fn) {
          case AggFn::Count:
            if (s0.is_valid(r)) ac.cnt += s0.i[r];
            break;
          case AggFn::Sum:
            if (s0.is_valid(r)) {
              ac.has = true;
              if (s0.type.pk() == PK::F64) ac.add_f64(s0.f[r]);
              else if (s0.type.pk() == PK::I128) ac.sd = (i128)((u128)ac.sd + (u128)s0.d[r]);
              else ac.si = (int64_t)((uint64_t)ac.si + (uint64_t)s0.i[r]);
            }
            break;
          case AggFn::Min:
          case AggFn::Max:
            if (s0.is_valid(r)) acc_minmax(ac, s0, r, ae.fn == AggFn::Min);
            break;
          case AggFn::Avg: {
            const OCol& s1 = ain[a][1];
            if (s0.is_valid(r)) ac.cnt += s0.i[r];
            if (s1.is_valid(r)) {
              ac.has = true;
              if (s1.type.pk() == PK::F64) ac.add_f64(s1.f[r]);
              else ac.sd = (i128)((u128)ac.sd + (u128)s1.d[r]);
            }
            break;
          }
        }
      } else {
        if (ae.fn == AggFn::Count && !ae.arg) {
          ac.cnt++;
          continue;
        }
        const OCol& c = ain[a][0];
        if (!c.is_valid(r)) continue;
        switch (ae.fn) {
          case AggFn::Count: ac.cnt++; break;
          case AggFn::Sum:
          case AggFn::Avg:
            ac.has = true;
            ac.cnt++;
            if (c.type.pk() == PK::F64) ac.add_f64(c.f[r]);
            else if (c.type.pk() == PK::I128) ac.sd = (i128)((u128)ac.sd + (u128)c.d[r]);  // wrapping [EXT]
            else ac.si = (int64_t)((uint64_t)ac.si + (uint64_t)c.i[r]);
            break;
          case AggFn::Min:
          case AggFn::Max: acc_minmax(ac, c, r, ae.fn == AggFn::Min); break;
        }
      }
    }
  }
  size_t G = accs.size();
  OBatch out;
  out.n = G;
  std::vector<int64_t> fr(first_row.begin(), first_row.end());
  for (size_t g = 0; g < ng; g++) {
    OCol kc = take(*keys[g], fr);
    kc.name = node.group_by[g].name;
    out.cols.push_back(std::move(kc));
  }
  for (size_t a = 0; a < na; a++) {
    const AggExpr& ae = node.aggs[a];
    auto sum_col = [&](const DataType& t) {
      OCol c = make_col(t, G);
      for (size_t g = 0; g < G; g++) {
        const Acc& ac = accs[g][a];
        if (!ac.has) {
          c.set_null(g);
          continue;
        }
        if (t.pk() == PK::F64) c.f[g] = ac.f64_sum();
        else if (t.pk() == PK::I128) c.d[g] = ac.sd;
        else c.i[g] = ac.si;
      }
      return c;
    };
    auto minmax_col = [&](const DataType& t) {
      OCol c = make_col(t, G);
      for (size_t g = 0; g < G; g++) {
        const Acc& ac = accs[g][a];
        if (!ac.has) {
          c.set_null(g);
          continue;
        }
        switch (t.pk()) {
          case PK::F64: c.f[g] = ac.mf; break;
          case PK::I128: c.d[g] = ac.md; break;
          case PK::Str: c.s[g] = ac.ms; break;
          default: c.i[g] = ac.mi;
        }
      }
      return c;
    };
    auto count_col = [&](const DataType& t) {
      OCol c = make_col(t, G);
      for (size_t g = 0; g < G; g++) c.i[g] = accs[g][a].cnt;
      return c;
    };
    if (emit_states) {
      switch (ae.fn) {
        case AggFn::Count: out.cols.push_back(count_col(DataType(TypeId::Int64))); break;
        case AggFn::Sum: out.cols.push_back(sum_col(ae.sum_type)); break;
        case AggFn::Min:
        case AggFn::Max: out.cols.push_back(minmax_col(ae.sum_type)); break;
        case AggFn::Avg:
          out.cols.push_back(count_col(DataType(TypeId::UInt64)));
          out.cols.push_back(sum_col(ae.sum_type));
          break;
      }
    } else {
      switch (ae.fn) {
        case AggFn::Count: out.cols.push_back(count_col(DataType(TypeId::Int64))); break;
        case AggFn::Sum: out.cols.push_back(sum_col(ae.result_type)); break;
        case AggFn::Min:
        case AggFn::Max: out.cols.push_back(minmax_col(ae.result_type)); break;
        case AggFn::Avg: {
          OCol c = make_col(ae.result_type, G);
          for (size_t g = 0; g < G; g++) {
            const Acc& ac = accs[g][a];
            if (ac.cnt == 0 || !ac.has) {
              c.set_null(g);
              continue;
            }
            if (ae.result_type.is_decimal()) {
              // DecimalAverager::avg [EXT]: sum * 10^(target_scale - sum_scale) / count, truncating; an overflow of the
              // product or a quotient beyond the result precision is an error
              i128 v = checked_mul(ac.sd, pow10_i128(ae.result_type.scale - ae.sum_type.scale)) / (i128)ac.cnt;
              if (v >= pow10_i128(ae.result_type.precision) || v <= -pow10_i128(ae.result_type.precision))
                exec_fail("Arithmetic overflow: decimal average");
              c.d[g] = v;
            } else {
              c.f[g] = ac.f64_sum() / (double)ac.cnt;
            }
          }
          out.cols.push_back(std::move(c));
          break;
        }
      }
    }
  }
  for (size_t c = 0; c < out.cols.size(); c++) out.cols[c].name = node.schema[c].name;
  return out;
}

// ------------------------------------------------------------------------------------------------
// Join / sort
// ------------------------------------------------------------------------------------------------
OBatch do_hash_join(const PlanNode& node, const OBatch& L, const OBatch& R) {
  std::vector<OCol> lk, rk;
  for (auto& on : node.on) {
    lk.push_back(eval(*on.first, L));
    rk.push_back(eval(*on.second, R));
  }
  std::unordered_map<std::string, std::vector<int64_t>> table;
  std::string k;
  for (size_t r = 0; r < L.n; r++) {
    bool allv = encode_key(lk, r, k);
    if (!allv && !node.null_equals_null) continue;
    table[k].push_back((int64_t)r);
  }
  std::vector<int64_t> li, ri;
  for (size_t r = 0; r < R.n; r++) {
    bool allv = encode_key(rk, r, k);
    if (!allv && !node.null_equals_null) continue;
    auto it = table.find(k);
    if (it == table.end()) continue;
    for (int64_t l : it->second) {
      li.push_back(l);
      ri.push_back((int64_t)r);
    }
  }
  if (node.join_filter) {
    OBatch cat = take(L, li);
    OBatch rr = take(R, ri);
    for (auto& c : rr.cols) cat.cols.push_back(std::move(c));
    cat.n = li.size();
    OCol m = eval(*node.join_filter, cat);
    std::vector<int64_t> l2, r2;
    for (size_t p = 0; p < li.size(); p++)
      if (m.is_valid(p) && m.i[p]) {
        l2.push_back(li[p]);
        r2.push_back(ri[p]);
      }
    li.swap(l2);
    ri.swap(r2);
  }
  std::vector<uint8_t> lm(L.n, 0), rm(R.n, 0);
  for (size_t p = 0; p < li.size(); p++) {
    lm[(size_t)li[p]] = 1;
    rm[(size_t)ri[p]] = 1;
  }
  OBatch out;
  auto semi = [&](const OBatch& side, const std::vector<uint8_t>& mark, bool want) {
    std::vector<int64_t> idx;
    for (size_t r = 0; r < side.n; r++)
      if ((mark[r] != 0) == want) idx.push_back((int64_t)r);
    return take(side, idx);
  };
  switch (node.join_type) {
    case JoinType::LeftSemi: out = semi(L, lm, true); break;
    case JoinType::LeftAnti: out = semi(L, lm, false); break;
    case JoinType::RightSemi: out = semi(R, rm, true); break;
    case JoinType::RightAnti: out = semi(R, rm, false); break;
    default: {
      if (node.join_type == JoinType::Left || node.join_type == JoinType::Full)
        for (size_t r = 0; r < L.n; r++)
          if (!lm[r]) {
            li.push_back((int64_t)r);
            ri.push_back(-1);
          }
      if (node.join_type == JoinType::Right || node.join_type == JoinType::Full)
        for (size_t r = 0; r < R.n; r++)
          if (!rm[r]) {
            li.push_back(-1);
            ri.push_back((int64_t)r);
          }
      out = take(L, li);
      OBatch rr = take(R, ri);
      for (auto& c : rr.cols) out.cols.push_back(std::move(c));
      out.n = li.size();
    }
  }
  if (node.has_projection) {
    OBatch p;
    p.n = out.n;
    for (int idx : node.projection) p.cols.push_back(out.cols[(size_t)idx]);
    out = std::move(p);
  }
  for (size_t c = 0; c < out.cols.size(); c++) out.cols[c].name = node.schema[c].name;
  return out;
}

OBatch do_sort(const std::vector<SortKey>& keys, int64_t fetch, const OBatch& in) {
  std::vector<OCol> kc;
  for (auto& k : keys) kc.push_back(eval(*k.expr, in));
  std::vector<int64_t> idx(in.n);
  for (size_t r = 0; r < in.n; r++) idx[r] = (int64_t)r;
  std::stable_sort(idx.begin(), idx.end(), [&](int64_t a, int64_t b) {
    for (size_t k = 0; k < keys.size(); k++) {
      bool va = kc[k].is_valid((size_t)a), vb = kc[k].is_valid((size_t)b);
      if (!va || !vb) {
        if (va == vb) continue;
        bool a_first = !va ? keys[k].nulls_first : !keys[k].nulls_first;
        return a_first;
      }
      int c = compare_values(kc[k], (size_t)a, kc[k], (size_t)b);
      if (c == 0) continue;
      return keys[k].asc ? c < 0 : c > 0;
    }
    return false;
  });
  if (fetch >= 0 && (size_t)fetch < idx.size()) idx.resize((size_t)fetch);
  return take(in, idx);
}

// ------------------------------------------------------------------------------------------------
// Engine
// ------------------------------------------------------------------------------------------------
struct Piece {
  int64_t file_id;
  OBatch batch;
};
struct ShuffleKey {
  std::string job;
  int64_t stage;
  int64_t part;
  bool operator<(const ShuffleKey& o) const {
    if (job != o.job) return job < o.job;
    if (stage != o.stage) return stage < o.stage;
    return part < o.part;
  }
};

uint64_t batch_bytes(const OBatch& b) {
  uint64_t t = 0;
  for (auto& c : b.cols) {
    if (c.type.id == TypeId::Bool) t += (c.n + 7) / 8;
    else if (c.type.id == TypeId::Utf8) {
      t += 4 * (c.n + 1);
      for (size_t r = 0; r < c.n; r++)
        if (c.is_valid(r)) t += c.s[r].size();
    } else t += (uint64_t)c.type.width() * c.n;
  }  // validity bitmaps are not counted: num_bytes = data buffers (values / offsets / chars)
  return t;
}

struct Oracle {
  std::mutex mu;
  std::map<std::string, std::map<int, std::shared_ptr<OBatch>>> tables;
  std::map<ShuffleKey, std::vector<Piece>> shuffle;
  int64_t batch_size = 8192;
  std::string err;

  int n_partitions(const PlanNode& n, const std::string& job) {
    switch (n.op) {
      case PlanNode::Scan: {
        std::lock_guard<std::mutex> g(mu);
        auto it = tables.find(n.table);
        if (it == tables.end()) exec_fail("table not registered: " + n.table);
        return it->second.empty() ? 0 : it->second.rbegin()->first + 1;
      }
      case PlanNode::ShuffleReader: {
        std::lock_guard<std::mutex> g(mu);
        int mx = 0;
        for (auto& kv : shuffle)
          if (kv.first.job == job && kv.first.stage == n.reader_stage_id) mx = std::max(mx, (int)kv.first.part + 1);
        return mx;
      }
      case PlanNode::SortPreservingMerge: return 1;
      case PlanNode::Passthrough:
        if (n.op_name == "CoalescePartitionsExec") return 1;
        return n_partitions(*n.children[0], job);
      case PlanNode::HashJoin: return n_partitions(*n.children[1], job);
      default: return n_partitions(*n.children[0], job);
    }
  }

  OBatch exec_all(const PlanNode& n, const std::string& job) {
    int np = n_partitions(n, job);
    OBatch out = empty_batch(n.schema);
    for (int p = 0; p < np; p++) append(out, exec(n, p, job));
    return out;
  }

  OBatch exec(const PlanNode& n, int part, const std::string& job) {
    switch (n.op) {
      case PlanNode::Scan: {
        std::shared_ptr<OBatch> src;
        {
          std::lock_guard<std::mutex> g(mu);
          auto it = tables.find(n.table);
          if (it == tables.end()) exec_fail("table not registered: " + n.table);
          auto pit = it->second.find(part);
          if (pit != it->second.end()) src = pit->second;
        }
        OBatch out;
        if (!src) return empty_batch(n.schema);
        out.n = src->n;
        for (int idx : n.scan_projection) {
          if ((size_t)idx >= src->cols.size()) exec_fail("scan projection out of range for " + n.table);
          out.cols.push_back(src->cols[(size_t)idx]);
        }
        for (size_t c = 0; c < out.cols.size(); c++)
          if (out.cols[c].type != n.schema[c].type)
            exec_fail("scan: column " + n.schema[c].name + " has type " + out.cols[c].type.str() + ", plan says " + n.schema[c].type.str());
        return out;
      }
      case PlanNode::ShuffleReader: {
        std::lock_guard<std::mutex> g(mu);
        OBatch out = empty_batch(n.schema);
        auto it = shuffle.find(ShuffleKey{job, n.reader_stage_id, n.broadcast ? 0 : part});
        if (it != shuffle.end())
          for (auto& p : it->second) append(out, p.batch);
        return out;
      }
      case PlanNode::Filter: {
        // A filter directly over a table scan whose projection is the identity reads the registered
        // batch in place (no private copy of every column first); only the surviving rows of the
        // columns the filter's own projection keeps are materialised.  Same values, fewer copies.
        std::shared_ptr<OBatch> direct;
        OBatch owned;
        const PlanNode& ch = *n.children[0];
        if (ch.op == PlanNode::Scan) {
          std::lock_guard<std::mutex> g(mu);
          auto it = tables.find(ch.table);
          if (it != tables.end()) {
            auto pit = it->second.find(part);
            if (pit != it->second.end()) {
              bool identity = ch.scan_projection.size() == pit->second->cols.size();
              for (size_t k = 0; identity && k < ch.scan_projection.size(); k++)
                identity = ch.scan_projection[k] == (int)k && pit->second->cols[k].type == ch.schema[k].type;
              if (identity) direct = pit->second;
            }
          }
        }
        if (!direct) owned = exec(ch, part, job);
        const OBatch& in = direct ? *direct : owned;
        OCol m = eval(*n.predicate, in);
        std::vector<int64_t> idx;
        for (size_t r = 0; r < in.n; r++)
          if (m.is_valid(r) && m.i[r]) idx.push_back((int64_t)r);
        if (n.fetch >= 0 && (size_t)n.fetch < idx.size()) idx.resize((size_t)n.fetch);
        OBatch out;
        out.n = idx.size();
        if (n.has_projection) {
          for (int i : n.projection) out.cols.push_back(take(in.cols.at((size_t)i), idx));
        } else {
          for (auto& c : in.cols) out.cols.push_back(take(c, idx));
        }
        return out;
      }
      case PlanNode::Projection: {
        OBatch in = exec(*n.children[0], part, job);
        OBatch out;
        out.n = in.n;
        // computed expressions first (they read `in`); then the plain column references, moved out of the
        // input batch when this is their last use instead of copied
        out.cols.resize(n.exprs.size());
        for (size_t k = 0; k < n.exprs.size(); k++)
          if (n.exprs[k].expr->kind != Expr::Col) out.cols[k] = eval(*n.exprs[k].expr, in);
        for (size_t k = 0; k < n.exprs.size(); k++) {
          const Expr& e = *n.exprs[k].expr;
          if (e.kind != Expr::Col) continue;
          if ((size_t)e.col >= in.cols.size()) exec_fail("projection column out of range");
          // every computed expression has already been evaluated; other plain references still need the column
          bool last = true;
          for (size_t k2 = k + 1; k2 < n.exprs.size() && last; k2++)
            last = !(n.exprs[k2].expr->kind == Expr::Col && n.exprs[k2].expr->col == e.col);
          if (last) out.cols[k] = std::move(in.cols[(size_t)e.col]);
          else out.cols[k] = in.cols[(size_t)e.col];
        }
        for (size_t k = 0; k < n.exprs.size(); k++) out.cols[k].name = n.exprs[k].name;
        return out;
      }
      case PlanNode::Aggregate: {
        // Final (non-partitioned) and Single see all input partitions of their child
        bool all = (n.agg_mode == AggMode::Final || n.agg_mode == AggMode::Single) && part == 0 &&
                   n_partitions(*n.children[0], job) > 1;
        OBatch in = all ? exec_all(*n.children[0], job) : exec(*n.children[0], part, job);
        return do_aggregate(n, in);
      }
      case PlanNode::HashJoin: {
        OBatch L = n.partition_mode == "CollectLeft" ? exec_all(*n.children[0], job) : exec(*n.children[0], part, job);
        OBatch R = exec(*n.children[1], part, job);
        OBatch J = do_hash_join(n, L, R);
        if (!n.sort_keys.empty()) return do_sort(n.sort_keys, -1, J);  // SortMergeJoinExec output order (plan.hpp)
        return J;
      }
      case PlanNode::Sort: {
        OBatch in = exec(*n.children[0], part, job);
        return do_sort(n.sort_keys, n.fetch, in);
      }
      case PlanNode::SortPreservingMerge: {
        OBatch in = exec_all(*n.children[0], job);
        return do_sort(n.sort_keys, n.fetch, in);
      }
      case PlanNode::Passthrough:
        if (n.op_name == "CoalescePartitionsExec") return exec_all(*n.children[0], job);
        return exec(*n.children[0], part, job);
      case PlanNode::Limit: {
        OBatch in = (n.op_name == "GlobalLimitExec") ? exec_all(*n.children[0], job) : exec(*n.children[0], part, job);
        std::vector<int64_t> idx;
        for (size_t r = (size_t)std::max<int64_t>(0, n.skip); r < in.n; r++) {
          if (n.fetch >= 0 && (int64_t)idx.size() >= n.fetch) break;
          idx.push_back((int64_t)r);
        }
        return take(in, idx);
      }
      case PlanNode::ShuffleWriter: exec_fail("nested ShuffleWriterExec");
    }
    exec_fail("unknown operator");
  }

  // ShuffleWriterExec::execute_shuffle_write / SortShuffleWriterExec::execute_shuffle_write
  std::vector<b200_shuffle_write_partition> execute_stage(const PlanNode& root, const std::string& job_id,
                                                          int64_t stage_id, int input_partition) {
    if (root.op != PlanNode::ShuffleWriter) exec_fail("stage plan root must be a ShuffleWriterExec");
    OBatch in = exec(*root.children[0], input_partition, job_id);
    for (size_t c = 0; c < in.cols.size(); c++) in.cols[c].name = root.schema[c].name;
    std::vector<b200_shuffle_write_partition> res;
    auto nbatches = [&](uint64_t rows) { return (rows + (uint64_t)batch_size - 1) / (uint64_t)batch_size; };
    if (root.n_out_partitions == 0) {
      // None branch (shuffle_writer.rs:221-268): one file, partition_id = input partition, file_id None
      b200_shuffle_write_partition w{};
      w.partition_id = (uint64_t)input_partition;
      w.num_rows = in.n;
      w.num_batches = nbatches(in.n);
      w.num_bytes = batch_bytes(in);
      w.file_id = -1;
      w.is_sort_shuffle = 0;
      std::lock_guard<std::mutex> g(mu);
      auto& v = shuffle[ShuffleKey{job_id, stage_id, input_partition}];
      v.clear();
      v.push_back(Piece{-1, std::move(in)});
      res.push_back(w);
      return res;
    }
    // Hash branch: p = hash(keys) % P (sort_shuffle/writer.rs:744-747); rows keep input order inside a partition
    std::vector<OCol> keys;
    for (auto& e : root.part_exprs) keys.push_back(eval(*e, in));
    size_t P = (size_t)root.n_out_partitions;
    std::vector<std::vector<int64_t>> buckets(P);
    for (size_t r = 0; r < in.n; r++) buckets[row_hash(keys, r) % P].push_back((int64_t)r);
    for (size_t p = 0; p < P; p++) {
      // a re-run of the same map task replaces its previous output (retry semantics)
      {
        std::lock_guard<std::mutex> g(mu);
        auto it = shuffle.find(ShuffleKey{job_id, stage_id, (int64_t)p});
        if (it != shuffle.end()) {
          auto& v = it->second;
          v.erase(std::remove_if(v.begin(), v.end(), [&](const Piece& pc) { return pc.file_id == input_partition; }), v.end());
        }
      }
      if (buckets[p].empty()) continue;  // only partitions with rows are reported (sort_shuffle/writer.rs:357-369)
      OBatch sub = take(in, buckets[p]);
      b200_shuffle_write_partition w{};
      w.partition_id = p;
      w.num_rows = sub.n;
      w.num_batches = nbatches(sub.n);
      w.num_bytes = batch_bytes(sub);
      w.file_id = input_partition;
      w.is_sort_shuffle = root.sort_shuffle ? 1 : 0;
      std::lock_guard<std::mutex> g(mu);
      shuffle[ShuffleKey{job_id, stage_id, (int64_t)p}].push_back(Piece{input_partition, std::move(sub)});
      res.push_back(w);
    }
    return res;
  }
};

OBatch tpch_generate(int table, int64_t msf, int64_t r0, int64_t r1, const std::vector<int>& cols) {
  using namespace tpch;
  OBatch b;
  b.n = (size_t)(r1 - r0);
  for (int c : cols) {
    const ColDef& cd = kCols[table][c];
    DataType t;
    switch (cd.kind) {
      case K_I64: t = DataType(TypeId::Int64); break;
      case K_I32: t = DataType(TypeId::Int32); break;
      case K_DEC: t = DataType::decimal(15, 2); break;
      case K_DATE: t = DataType(TypeId::Date32); break;
      case K_STR: t = DataType(TypeId::Utf8); break;
    }
    OCol col = make_col(t, b.n, cd.name);
    col.nullable = false;
    char buf[kMaxStrLen];
    for (int64_t r = r0; r < r1; r++) {
      size_t k = (size_t)(r - r0);
      if (cd.kind == K_STR) {
        uint32_t n = gen_str(table, c, r, msf, buf);
        col.s[k].assign(buf, n);
      } else if (cd.kind == K_DEC) {
        col.d[k] = (i128)gen_i64(table, c, r, msf);
      } else {
        col.i[k] = gen_i64(table, c, r, msf);
      }
    }
    b.cols.push_back(std::move(col));
  }
  return b;
}

thread_local std::string g_err;

template <class F>
int guard(Oracle* o, F&& f) {
  try {
    f();
    return 0;
  } catch (const ExecError& e) {
    g_err = e.what();
    return e.code;
  } catch (const std::exception& e) {
    g_err = e.what();
    return B200_ERR_INVALID;
  }
}

}  // namespace

extern "C" {

void* oracle_create() { return new Oracle(); }
void oracle_destroy(void* o) { delete (Oracle*)o; }
const char* oracle_last_error() { return g_err.c_str(); }

int oracle_set_config(void* o_, const char* key, const char* value) {
  Oracle* o = (Oracle*)o_;
  if (std::string(key) == "datafusion.execution.batch_size") o->batch_size = std::max<int64_t>(1, atoll(value));
  return 0;
}

int oracle_register_batch(void* o_, const char* table, int partition, ArrowArray* arr, ArrowSchema* sch) {
  Oracle* o = (Oracle*)o_;
  return guard(o, [&] {
    OBatch b = import_batch(arr, sch);
    std::lock_guard<std::mutex> g(o->mu);
    auto& slot = o->tables[table][partition];
    if (!slot || slot->cols.empty()) {
      slot = std::make_shared<OBatch>(std::move(b));
    } else {
      auto merged = std::make_shared<OBatch>(*slot);
      append(*merged, b);
      slot = merged;
    }
  });
}

int oracle_drop_table(void* o_, const char* table) {
  Oracle* o = (Oracle*)o_;
  std::lock_guard<std::mutex> g(o->mu);
  o->tables.erase(table);
  return 0;
}

static int table_id(const std::string& name) {
  static const char* names[] = {"lineitem", "orders", "customer", "supplier", "part", "partsupp", "nation", "region"};
  for (int i = 0; i < 8; i++)
    if (name == names[i]) return i;
  return -1;
}

int64_t oracle_tpch_table_rows(const char* table, int64_t msf) {
  int t = table_id(table);
  return t < 0 ? -1 : tpch::table_rows(t, msf);
}

int oracle_tpch_generate(void* o_, const char* table, int64_t msf, int partition, int64_t row_begin, int64_t row_end,
                         const char* columns_csv) {
  Oracle* o = (Oracle*)o_;
  return guard(o, [&] {
    int t = table_id(table);
    if (t < 0) throw std::runtime_error(std::string("unknown TPC-H table ") + table);
    std::vector<int> cols;
    if (columns_csv && *columns_csv) {
      std::string s(columns_csv);
      size_t p = 0;
      while (p <= s.size()) {
        size_t q = s.find(',', p);
        if (q == std::string::npos) q = s.size();
        std::string nm = s.substr(p, q - p);
        int found = -1;
        for (int c = 0; c < tpch::kNumCols[t]; c++)
          if (nm == tpch::kCols[t][c].name) found = c;
        if (found < 0) throw std::runtime_error("unknown column " + nm);
        cols.push_back(found);
        p = q + 1;
      }
    } else {
      for (int c = 0; c < tpch::kNumCols[t]; c++) cols.push_back(c);
    }
    OBatch b = tpch_generate(t, msf, row_begin, row_end, cols);
    std::lock_guard<std::mutex> g(o->mu);
    o->tables[table][partition] = std::make_shared<OBatch>(std::move(b));
  });
}

int oracle_export_table(void* o_, const char* table, int partition, ArrowArray* out, ArrowSchema* out_schema) {
  Oracle* o = (Oracle*)o_;
  return guard(o, [&] {
    std::lock_guard<std::mutex> g(o->mu);
    auto it = o->tables.find(table);
    if (it == o->tables.end() || !it->second.count(partition)) throw ExecError(B200_ERR_NOT_FOUND, "no such table partition");
    export_batch(*it->second[partition], nullptr, out, out_schema);
  });
}

int oracle_execute_stage(void* o_, const char* job_id, int64_t stage_id, const char* plan_json, int input_partition,
                         b200_shuffle_write_partition* out, int cap, int* n_out) {
  Oracle* o = (Oracle*)o_;
  return guard(o, [&] {
    Json j = parse_json(plan_json, strlen(plan_json));
    PlanPtr plan = parse_plan(j);
    auto res = o->execute_stage(*plan, job_id, stage_id, input_partition);
    if ((int)res.size() > cap) throw std::runtime_error("output array too small");
    for (size_t i = 0; i < res.size(); i++) out[i] = res[i];
    *n_out = (int)res.size();
  });
}

int oracle_partition_export(void* o_, const char* job_id, int64_t stage_id, int out_partition, const char* schema_json,
                            ArrowArray* out, ArrowSchema* out_schema) {
  Oracle* o = (Oracle*)o_;
  return guard(o, [&] {
    std::lock_guard<std::mutex> g(o->mu);
    auto it = o->shuffle.find(ShuffleKey{job_id, stage_id, out_partition});
    if (it == o->shuffle.end()) throw ExecError(B200_ERR_NOT_FOUND, "no such shuffle partition");
    OBatch all;
    for (auto& p : it->second) append(all, p.batch);
    (void)schema_json;
    export_batch(all, nullptr, out, out_schema);
  });
}

int64_t oracle_partition_rows(void* o_, const char* job_id, int64_t stage_id, int out_partition) {
  Oracle* o = (Oracle*)o_;
  std::lock_guard<std::mutex> g(o->mu);
  auto it = o->shuffle.find(ShuffleKey{job_id, stage_id, out_partition});
  if (it == o->shuffle.end()) return -1;
  int64_t n = 0;
  for (auto& p : it->second) n += (int64_t)p.batch.n;
  return n;
}

int oracle_remove_job_data(void* o_, const char* job_id) {
  Oracle* o = (Oracle*)o_;
  std::lock_guard<std::mutex> g(o->mu);
  for (auto it = o->shuffle.begin(); it != o->shuffle.end();) {
    if (it->first.job == job_id) it = o->shuffle.erase(it);
    else ++it;
  }
  return 0;
}

// Partition id of every row of a batch under the shuffle hash -- lets tests check the kernel's
// per-row assignment, not just per-partition counts (drift-test idea, sort_shuffle/writer.rs:1140-1198).
int oracle_hash_partition_ids(void* o_, ArrowArray* arr, ArrowSchema* sch, const char* key_cols_csv, int64_t P,
                              uint64_t* out_hash, int32_t* out_pid) {
  Oracle* o = (Oracle*)o_;
  return guard(o, [&] {
    OBatch b = import_batch(arr, sch);
    std::vector<OCol> keys;
    std::string s(key_cols_csv);
    size_t p = 0;
    while (p < s.size()) {
      size_t q = s.find(',', p);
      if (q == std::string::npos) q = s.size();
      keys.push_back(b.cols.at((size_t)atoi(s.substr(p, q - p).c_str())));
      p = q + 1;
    }
    for (size_t r = 0; r < b.n; r++) {
      uint64_t h = row_hash(keys, r);
      if (out_hash) out_hash[r] = h;
      if (out_pid) out_pid[r] = (int32_t)(h % (uint64_t)P);
    }
  });
}

}  // extern "C"
