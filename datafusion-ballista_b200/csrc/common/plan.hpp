// Stage-plan IR: the physical operator tree a Ballista task hands to an ExecutionEngine
// (ballista/executor/src/execution_engine.rs:50-58), restated as a small typed tree parsed from
// JSON.  Node and field names follow the vendored DataFusion plan protobuf that pins the shape of
// every operator the executor can receive: ballista/core/proto/datafusion.proto
//   FilterExecNode :1027-1034, ProjectionExecNode :1211-1215, AggregateExecNode :1257-1271
//   (modes :1217-1224), HashJoinExecNode :1134-1144 (PartitionMode :1128-1132), SortExecNode
//   :1286-1292, SortPreservingMergeExecNode :1294-1298, PhysicalExprNode :851-901,
//   PhysicalBinaryExprNode :957-961; ShuffleWriterExecNode / ShuffleReaderExecNode are Ballista's
//   own (ballista/core/proto/ballista.proto:47-99).
//
// Type rules marked [EXT] restate arrow-rs 58.1 / DataFusion 53.1 behaviour (crates not vendored
// under /root/reference, Cargo.lock:192,2053) and are documented in DESIGN.md §"Semantics".
//
// This header is shared by the product (csrc/host) and by the CPU oracle (oracle/): it contains
// parsing and *typing* only -- no arithmetic on data.
#pragma once
#include <climits>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "json.hpp"
#include "regex_dfa.hpp"

namespace b200 {

typedef __int128 i128;
typedef unsigned __int128 u128;

enum class TypeId : uint8_t {
  Null = 0, Bool, Int8, Int16, Int32, Int64, UInt8, UInt16, UInt32, UInt64,
  Float32, Float64, Date32, Timestamp, Decimal128, Utf8
};

// Physical (compute) kind a logical type maps onto inside both engines.
enum class PK : uint8_t { Bool = 0, I64 = 1, F64 = 2, I128 = 3, Str = 4 };

struct DataType {
  TypeId id = TypeId::Null;
  uint8_t precision = 0;
  int8_t scale = 0;
  DataType() {}
  DataType(TypeId i) : id(i) {}
  static DataType decimal(int p, int s) {
    DataType t(TypeId::Decimal128);
    t.precision = (uint8_t)p;
    t.scale = (int8_t)s;
    return t;
  }
  bool operator==(const DataType& o) const {
    return id == o.id && (id != TypeId::Decimal128 || (precision == o.precision && scale == o.scale));
  }
  bool operator!=(const DataType& o) const { return !(*this == o); }
  bool is_decimal() const { return id == TypeId::Decimal128; }
  bool is_float() const { return id == TypeId::Float32 || id == TypeId::Float64; }
  bool is_signed_int() const { return id >= TypeId::Int8 && id <= TypeId::Int64; }
  bool is_unsigned_int() const { return id >= TypeId::UInt8 && id <= TypeId::UInt64; }
  bool is_integer() const { return is_signed_int() || is_unsigned_int(); }
  bool is_numeric() const { return is_integer() || is_float() || is_decimal(); }
  bool is_string() const { return id == TypeId::Utf8; }
  PK pk() const {
    switch (id) {
      case TypeId::Bool: return PK::Bool;
      case TypeId::Float32:
      case TypeId::Float64: return PK::F64;
      case TypeId::Decimal128: return PK::I128;
      case TypeId::Utf8: return PK::Str;
      default: return PK::I64;
    }
  }
  // Arrow in-memory width of one value in the values buffer (Utf8: the int32 offset).
  int width() const {
    switch (id) {
      case TypeId::Null: return 0;
      case TypeId::Bool: return 0;  // bit-packed
      case TypeId::Int8:
      case TypeId::UInt8: return 1;
      case TypeId::Int16:
      case TypeId::UInt16: return 2;
      case TypeId::Int32:
      case TypeId::UInt32:
      case TypeId::Float32:
      case TypeId::Date32: return 4;
      case TypeId::Decimal128: return 16;
      case TypeId::Utf8: return 4;
      default: return 8;
    }
  }
  std::string str() const {
    switch (id) {
      case TypeId::Null: return "null";
      case TypeId::Bool: return "bool";
      case TypeId::Int8: return "i8";
      case TypeId::Int16: return "i16";
      case TypeId::Int32: return "i32";
      case TypeId::Int64: return "i64";
      case TypeId::UInt8: return "u8";
      case TypeId::UInt16: return "u16";
      case TypeId::UInt32: return "u32";
      case TypeId::UInt64: return "u64";
      case TypeId::Float32: return "f32";
      case TypeId::Float64: return "f64";
      case TypeId::Date32: return "date32";
      case TypeId::Timestamp: return "ts";
      case TypeId::Utf8: return "utf8";
      case TypeId::Decimal128:
        return "dec(" + std::to_string((int)precision) + "," + std::to_string((int)scale) + ")";
    }
    return "?";
  }
};

inline DataType parse_type(const Json& j) {
  if (j.is_obj()) {
    const Json& d = j.at("dec");
    return DataType::decimal((int)d.at(0).as_int(), (int)d.at(1).as_int());
  }
  const std::string& s = j.str();
  static const std::pair<const char*, TypeId> tab[] = {
      {"null", TypeId::Null},     {"bool", TypeId::Bool},     {"i8", TypeId::Int8},
      {"i16", TypeId::Int16},     {"i32", TypeId::Int32},     {"i64", TypeId::Int64},
      {"u8", TypeId::UInt8},      {"u16", TypeId::UInt16},    {"u32", TypeId::UInt32},
      {"u64", TypeId::UInt64},    {"f32", TypeId::Float32},   {"f64", TypeId::Float64},
      {"date32", TypeId::Date32}, {"ts", TypeId::Timestamp},  {"utf8", TypeId::Utf8}};
  for (auto& kv : tab)
    if (s == kv.first) return DataType(kv.second);
  throw std::runtime_error("plan IR: unknown type '" + s + "'");
}

inline std::string type_json(const DataType& t) {
  if (t.is_decimal())
    return "{\"dec\":[" + std::to_string((int)t.precision) + "," + std::to_string((int)t.scale) + "]}";
  return "\"" + t.str() + "\"";
}

struct Field {
  std::string name;
  DataType type;
  bool nullable = true;
};
typedef std::vector<Field> Schema;

inline Schema parse_schema(const Json& j) {
  Schema s;
  for (size_t i = 0; i < j.size(); i++) {
    const Json& f = j.at(i);
    Field fd;
    fd.name = f.at("name").str();
    fd.type = parse_type(f.at("type"));
    fd.nullable = f.get_bool("nullable", true);
    s.push_back(fd);
  }
  return s;
}

// ----------------------------------------------------------------------------------------------
// Decimal helpers (typing only)
// ----------------------------------------------------------------------------------------------
static const int kMaxDecimalPrecision = 38;
static const int kMaxDecimalScale = 38;

inline i128 pow10_i128(int n) {
  i128 r = 1;
  for (int i = 0; i < n; i++) r *= 10;
  return r;
}

// 10^n as the double nearest to it (exact for 0 <= n <= 22): the scale factor of the decimal <-> float casts, the same
// table the device uses (pipeline.cu pow10_f64_dev)
inline double pow10_f64(int n) {
  static const double t[39] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11, 1e12, 1e13,
                               1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22, 1e23, 1e24, 1e25, 1e26, 1e27,
                               1e28, 1e29, 1e30, 1e31, 1e32, 1e33, 1e34, 1e35, 1e36, 1e37, 1e38};
  return t[n < 0 ? 0 : n > 38 ? 38 : n];
}

inline i128 parse_i128(const std::string& s) {
  size_t k = 0;
  bool neg = false;
  if (k < s.size() && (s[k] == '-' || s[k] == '+')) neg = s[k++] == '-';
  u128 v = 0;
  if (k >= s.size()) throw std::runtime_error("plan IR: bad integer literal '" + s + "'");
  for (; k < s.size(); k++) {
    if (s[k] < '0' || s[k] > '9') throw std::runtime_error("plan IR: bad integer literal '" + s + "'");
    v = v * 10 + (unsigned)(s[k] - '0');
  }
  return neg ? -(i128)v : (i128)v;
}

inline std::string i128_to_string(i128 v) {
  if (v == 0) return "0";
  bool neg = v < 0;
  u128 u = neg ? (u128)(-(v + 1)) + 1 : (u128)v;
  std::string s;
  while (u) {
    s += (char)('0' + (int)(u % 10));
    u /= 10;
  }
  if (neg) s += '-';
  return std::string(s.rbegin(), s.rend());
}

// Integer -> decimal coercion precision used by DataFusion when an integer meets a decimal
// (datafusion-expr type_coercion/binary.rs `coerce_numeric_type_to_decimal`) [EXT].
inline DataType int_as_decimal(const DataType& t) {
  switch (t.id) {
    case TypeId::Int8: return DataType::decimal(3, 0);
    case TypeId::Int16: return DataType::decimal(5, 0);
    case TypeId::Int32: return DataType::decimal(10, 0);
    case TypeId::Int64: return DataType::decimal(20, 0);
    case TypeId::UInt8: return DataType::decimal(3, 0);
    case TypeId::UInt16: return DataType::decimal(5, 0);
    case TypeId::UInt32: return DataType::decimal(10, 0);
    case TypeId::UInt64: return DataType::decimal(20, 0);
    default: return t;
  }
}

enum class BinOp : uint8_t {
  Add, Sub, Mul, Div, Mod, Eq, Ne, Lt, Le, Gt, Ge, And, Or, BitAnd, BitOr, BitXor, Shl, Shr,
  RegexMatch, RegexIMatch, RegexNotMatch, RegexNotIMatch,  // ~  ~*  !~  !~*
  StringConcat                                             // ||
};

inline BinOp parse_binop(const std::string& s) {
  static const std::pair<const char*, BinOp> tab[] = {
      {"+", BinOp::Add},  {"-", BinOp::Sub},  {"*", BinOp::Mul},  {"/", BinOp::Div},
      {"%", BinOp::Mod},  {"=", BinOp::Eq},   {"==", BinOp::Eq},  {"!=", BinOp::Ne},
      {"<>", BinOp::Ne},  {"<", BinOp::Lt},   {"<=", BinOp::Le},  {">", BinOp::Gt},
      {">=", BinOp::Ge},  {"and", BinOp::And}, {"or", BinOp::Or},  {"AND", BinOp::And},
      {"OR", BinOp::Or},  {"&", BinOp::BitAnd}, {"|", BinOp::BitOr}, {"^", BinOp::BitXor},
      {"<<", BinOp::Shl}, {">>", BinOp::Shr}, {"~", BinOp::RegexMatch}, {"~*", BinOp::RegexIMatch},
      {"!~", BinOp::RegexNotMatch}, {"!~*", BinOp::RegexNotIMatch}, {"||", BinOp::StringConcat}};
  for (auto& kv : tab)
    if (s == kv.first) return kv.second;
  throw std::runtime_error("plan IR: unknown binary operator '" + s + "'");
}
inline bool is_arith(BinOp o) { return o <= BinOp::Mod; }
inline bool is_compare(BinOp o) { return o >= BinOp::Eq && o <= BinOp::Ge; }
inline bool is_logic(BinOp o) { return o == BinOp::And || o == BinOp::Or; }
inline bool is_bitwise(BinOp o) { return o >= BinOp::BitAnd && o <= BinOp::Shr; }
inline bool is_regex(BinOp o) { return o >= BinOp::RegexMatch && o <= BinOp::RegexNotIMatch; }

// Grouping sets (ROLLUP / CUBE / GROUPING SETS) and the bitwise operators DataFusion rewrites GROUPING() into are typed
// here for every consumer of the plan IR, but only a consumer built with B200_PLAN_GROUPING_SETS=1 computes them (the
// device engine: Makefile NVFLAGS).  Any other consumer -- the CPU oracle -- refuses such a plan instead of mis-evaluating it.
#ifndef B200_PLAN_GROUPING_SETS
#define B200_PLAN_GROUPING_SETS 0
#endif
// the grouping-set id occupies one more group key of the device table (VM_MAX_KEYS = 8, csrc/device/program.h)
static const size_t kMaxGroupingSetKeys = 7;
static const size_t kMaxGroupingSets = 32;
// [EXT] DataFusion 53 PhysicalGroupBy: the keys are folded from first to last, id = id << 1 | is_null, so the first key is
// the most significant bit; `mask` has bit k set when key k is replaced by NULL in the set
inline uint64_t grouping_id(uint32_t mask, size_t n_keys) {
  uint64_t id = 0;
  for (size_t k = 0; k < n_keys; k++) id = id << 1 | ((mask >> k) & 1u);
  return id;
}
// [EXT] the type of __grouping_id: the narrowest unsigned integer with a bit per key
inline DataType grouping_id_type(size_t n_keys) {
  return DataType(n_keys <= 8 ? TypeId::UInt8 : n_keys <= 16 ? TypeId::UInt16 : n_keys <= 32 ? TypeId::UInt32 : TypeId::UInt64);
}

// Result type of decimal (op) decimal, following arrow-arith 58 `decimal_op` [EXT]:
//   add/sub: scale = max(s1,s2); precision = min(38, max(p1-s1,p2-s2) + scale + 1)
//   mul:     scale = s1+s2;      precision = min(38, p1+p2+1)
//   div:     scale = min(38, s1+4); precision = min(38, p1 + (scale - s1 + s2))
//   mod:     scale = max(s1,s2); precision = min(38, min(p1-s1,p2-s2) + scale)
inline DataType decimal_result_type(BinOp op, const DataType& a, const DataType& b) {
  int p1 = a.precision, s1 = a.scale, p2 = b.precision, s2 = b.scale;
  int p, s;
  switch (op) {
    case BinOp::Add:
    case BinOp::Sub:
      s = std::max(s1, s2);
      p = std::min(kMaxDecimalPrecision, std::max(p1 - s1, p2 - s2) + s + 1);
      break;
    case BinOp::Mul:
      s = s1 + s2;
      if (s > kMaxDecimalScale) throw std::runtime_error("decimal multiply: result scale exceeds 38");
      p = std::min(kMaxDecimalPrecision, p1 + p2 + 1);
      break;
    case BinOp::Div: {
      s = std::min(kMaxDecimalScale, s1 + 4);
      int mul_pow = s - s1 + s2;
      p = std::min(kMaxDecimalPrecision, p1 + mul_pow);
      break;
    }
    case BinOp::Mod:
      s = std::max(s1, s2);
      p = std::min(kMaxDecimalPrecision, std::min(p1 - s1, p2 - s2) + s);
      break;
    default: throw std::runtime_error("decimal_result_type: not arithmetic");
  }
  return DataType::decimal(p, s);
}

// ----------------------------------------------------------------------------------------------
// Expressions
// ----------------------------------------------------------------------------------------------
struct LitValue {
  bool is_null = false;
  int64_t i = 0;   // Bool / ints / Date32 / Timestamp
  double f = 0;    // floats
  i128 d = 0;      // Decimal128 unscaled
  std::string s;   // Utf8
};

struct Expr;
typedef std::shared_ptr<Expr> ExprPtr;

struct Expr {
  enum Kind { Col, Lit, Bin, Not, Neg, IsNull, IsNotNull, Cast, Case, InList, Like, Fn } kind = Lit;
  DataType type;          // resolved output type
  bool nullable = true;
  int col = -1;           // Col
  LitValue lit;           // Lit
  BinOp op = BinOp::Add;  // Bin
  std::string fn;         // Fn: "date_part_<part>", "substr", "abs", "round", ... (type_scalar_fn)
  std::vector<ExprPtr> args;  // Bin: l,r; unary: x; Case: [w0,t0,w1,t1,...,(else)]; InList: x, items...; Fn args
  bool has_else = false;  // Case
  bool negated = false;   // InList / Like
  std::string pattern;    // Like
  bool case_insensitive = false;  // Like: ILIKE
  // ILIKE, the regex operators and regexp_like: the pattern compiled at typing (null when the pattern or the flags are a
  // NULL literal: the result is NULL), and the key the engine caches its device copy under
  std::shared_ptr<const rx::Dfa> regex;
  std::string regex_key;
  // regexp_count / regexp_replace: `regex` is the forward span DFA and regex_rev the reverse one (regex_dfa.hpp); the
  // count's start (1-based code points) and the replacement's g flag
  std::shared_ptr<const rx::Dfa> regex_rev;
  int64_t regex_start = 1;
  bool regex_global = false;
  std::string name;       // display only
};

inline ExprPtr make_col(int idx, const Schema& in) {
  if (idx < 0 || (size_t)idx >= in.size()) throw std::runtime_error("plan IR: column index out of range");
  auto e = std::make_shared<Expr>();
  e->kind = Expr::Col;
  e->col = idx;
  e->type = in[idx].type;
  e->nullable = in[idx].nullable;
  e->name = in[idx].name;
  return e;
}

// rewrite every column reference k -> target[k] (in place)
inline void remap_columns(const ExprPtr& e, const std::vector<int>& target) {
  if (!e) return;
  if (e->kind == Expr::Col) {
    if (e->col < 0 || (size_t)e->col >= target.size()) throw std::runtime_error("plan IR: column index out of range in remap");
    e->col = target[(size_t)e->col];
  }
  for (auto& a : e->args) remap_columns(a, target);
}

inline LitValue parse_lit_value(const DataType& t, const Json& v) {
  LitValue l;
  if (v.is_null()) {
    l.is_null = true;
    return l;
  }
  switch (t.pk()) {
    case PK::Bool: l.i = v.as_bool(); break;
    case PK::I64: l.i = v.is_str() ? (int64_t)parse_i128(v.str()) : v.as_int(); break;
    case PK::F64: l.f = v.is_str() ? strtod(v.str().c_str(), nullptr) : v.as_double(); break;
    case PK::I128: l.d = v.is_str() ? parse_i128(v.str()) : (v.is_int ? (i128)v.i : parse_i128(v.s)); break;
    case PK::Str: l.s = v.str(); break;
  }
  return l;
}

inline DataType arith_result_type(BinOp op, DataType a, DataType b) {
  if (a.id == TypeId::Null) return b;
  if (b.id == TypeId::Null) return a;
  if (a.is_float() || b.is_float()) {
    if (a.id == TypeId::Float32 && b.id == TypeId::Float32) return DataType(TypeId::Float32);
    return DataType(TypeId::Float64);
  }
  if (a.is_decimal() || b.is_decimal()) {
    if (!a.is_decimal()) a = int_as_decimal(a);
    if (!b.is_decimal()) b = int_as_decimal(b);
    if (!a.is_decimal() || !b.is_decimal())
      throw std::runtime_error("arithmetic between " + a.str() + " and " + b.str() + " is not supported");
    return decimal_result_type(op, a, b);
  }
  if (a.is_integer() && b.is_integer()) {
    if (a == b) return a;
    return DataType(TypeId::Int64);
  }
  if (a.id == TypeId::Date32 && b.is_integer() && (op == BinOp::Add || op == BinOp::Sub)) return a;
  if (a.id == TypeId::Date32 && b.id == TypeId::Date32 && op == BinOp::Sub) return DataType(TypeId::Int64);
  throw std::runtime_error("arithmetic between " + a.str() + " and " + b.str() + " is not supported");
}

ExprPtr parse_expr(const Json& j, const Schema& in);

// A plan the engine understands but does not run (e.g. statistical states laid out in an unknown way): B200_ERR_UNSUPPORTED
struct PlanUnsupported : std::runtime_error {
  explicit PlanUnsupported(const std::string& m) : std::runtime_error(m) {}
};

// The date_part family: IR "date_part_<part>", parts in the order of DatePart (csrc/device/program.h); -1 for another name
inline int date_part_index(const std::string& fn) {
  static const char* const parts[] = {"year", "quarter", "month", "week", "day", "doy", "dow"};
  if (fn.compare(0, 10, "date_part_") != 0) return -1;
  for (int i = 0; i < 7; i++)
    if (fn.compare(10, std::string::npos, parts[i]) == 0) return i;
  return -1;
}

// ILIKE, `~` / `~*` / `!~` / `!~*` and regexp_like are typed here for every consumer of the plan IR, but only a consumer
// built with B200_PLAN_REGEX=1 computes them (the device engine: Makefile NVFLAGS).  Semantics: DESIGN.md §6 (x),
// csrc/common/regex_dfa.hpp.  The pattern (and regexp_like's flags) must be Utf8 literals; it is compiled here, so that an
// invalid or unsupported pattern fails when the stage is prepared.
#ifndef B200_PLAN_REGEX
#define B200_PLAN_REGEX 0
#endif
inline void type_regex(Expr& e, const std::string& what, const ExprPtr& pattern, const ExprPtr& flags, bool ci) {
  if (!B200_PLAN_REGEX) throw PlanUnsupported(what + " is not computed by this consumer of the plan IR");
  const DataType& t = e.args[0]->type;
  if (!t.is_string() && t.id != TypeId::Null) throw PlanUnsupported(what + " does not support an operand of type " + t.str());
  e.type = DataType(TypeId::Bool);
  e.nullable = true;
  bool null_arg = false;
  auto literal = [&](const ExprPtr& a, const char* role) -> const std::string& {
    if (a->kind != Expr::Lit) throw PlanUnsupported(what + ": the " + role + " must be a literal");
    if (!a->type.is_string() && a->type.id != TypeId::Null) throw PlanUnsupported(what + ": the " + role + " must be utf8, not " + a->type.str());
    null_arg = null_arg || a->lit.is_null;
    return a->lit.s;
  };
  auto fail = [&](int rc, const std::string& msg) {
    if (rc == rx::RX_UNSUPPORTED) throw PlanUnsupported(msg);
    throw std::runtime_error(msg);
  };
  auto d = std::make_shared<rx::Dfa>();
  std::string err;
  int rc;
  if (!pattern) {  // ILIKE: arrow's LIKE-to-regex translation under the flags i and s
    rc = rx::compile_ilike(e.pattern, *d, err);
    e.regex_key = "like:" + e.pattern;
  } else {
    const std::string& p = literal(pattern, "pattern");
    bool fi = false, fs = false;
    if (flags) {
      const std::string& f = literal(flags, "flags argument");
      if (!null_arg && (rc = rx::parse_regex_flags(f, fi, fs, err)) != rx::RX_OK) fail(rc, err);
    }
    if (null_arg) return;
    fi = fi || ci;
    rc = rx::compile_regex(p, fi, fs, *d, err);
    e.regex_key = std::string(fi ? "i" : "") + (fs ? "s" : "") + ":" + p;
  }
  if (rc != rx::RX_OK) fail(rc, err);
  e.regex = d;
}

// regexp_count(str, pattern [, start [, flags]]) -> Int64 and regexp_replace(str, pattern, replacement [, flags]) -> Utf8,
// gated like type_regex.  Rules [EXT, DESIGN.md §6 (xiii)], restated from DataFusion 53 and unpinned:
//   regexp_count: a NULL or empty str counts 0, and a NULL or empty pattern 0 for every row (no row is NULL, though the
//     result is typed nullable as a scalar UDF's is); start is a non-NULL Int64 literal >= 1 counted in code points (the
//     haystack loses its first start - 1 of them); the flags must be a non-NULL literal without g.
//   regexp_replace: NULL when any argument is; a NULL literal makes every row NULL; the flag g replaces every match, else
//     only the first; the replacement is a literal inserted verbatim, refused when it holds '\' or '$' (DataFusion rewrites
//     \N into ${N} and Rust expands $name / ${N} / $$: group references a DFA cannot give).
// Both DFAs are compiled here, so that a bad pattern fails when the stage is prepared; their cache keys ("fwd:" / "rev:"
// + regex_key) never equal an is_match key.
inline void type_regex_fn(Expr& e) {
  const std::string& f = e.fn;
  const bool count = f == "regexp_count";
  const size_t n = e.args.size();
  if (!B200_PLAN_REGEX) throw PlanUnsupported(f + " is not computed by this consumer of the plan IR");
  const DataType& t = e.args[0]->type;
  if (!t.is_string() && t.id != TypeId::Null) throw PlanUnsupported(f + " does not support an operand of type " + t.str());
  e.type = DataType(count ? TypeId::Int64 : TypeId::Utf8);
  e.nullable = true;
  bool null_arg = false;
  auto literal = [&](const ExprPtr& a, const char* role) -> const std::string& {
    if (a->kind != Expr::Lit) throw PlanUnsupported(f + ": the " + role + " must be a literal");
    if (!a->type.is_string() && a->type.id != TypeId::Null) throw PlanUnsupported(f + ": the " + role + " must be utf8, not " + a->type.str());
    null_arg = null_arg || a->lit.is_null;
    return a->lit.s;
  };
  auto fail = [&](int rc, const std::string& msg) {
    if (rc == rx::RX_UNSUPPORTED) throw PlanUnsupported(msg);
    throw std::runtime_error(msg);
  };
  const std::string& p = literal(e.args[1], "pattern");
  const bool null_pattern = null_arg;
  if (count && n >= 3) {
    const Expr& s = *e.args[2];
    if (s.kind != Expr::Lit || s.type.id != TypeId::Int64 || s.lit.is_null)
      throw PlanUnsupported("regexp_count: the start must be a non-NULL Int64 literal");
    if (s.lit.i < 1) throw std::runtime_error("regexp_count: the start must be at least 1, not " + std::to_string(s.lit.i));
    e.regex_start = s.lit.i;
  }
  if (!count) {
    const std::string& r = literal(e.args[2], "replacement");
    if (r.find_first_of("\\$") != std::string::npos)
      throw PlanUnsupported("regexp_replace: the replacement '" + r + "' holds '\\' or '$' (a group reference), which is not supported by the device engine");
  }
  bool fi = false, fs = false;
  std::string err;
  if (n == 4) {
    // the flags literal is checked on its own, whatever the other arguments are (a NULL pattern included)
    const std::string& fl = literal(e.args[3], "flags argument");
    const bool null_flags = e.args[3]->lit.is_null;
    if (count && null_flags) throw PlanUnsupported("regexp_count: the flags argument must not be NULL");
    int rc;
    if (!null_flags && (rc = rx::parse_regex_flags(fl, fi, fs, err, f.c_str(), count ? nullptr : &e.regex_global)) != rx::RX_OK) fail(rc, err);
  }
  if (null_arg || (count && (null_pattern || p.empty()))) return;  // every row NULL (replace) or 0 (count)
  auto fwd = std::make_shared<rx::Dfa>();
  auto rev = std::make_shared<rx::Dfa>();
  const int rc = rx::compile_regex_spans(p, fi, fs, *fwd, *rev, err);
  if (rc != rx::RX_OK) fail(rc, err);
  e.regex = fwd;
  e.regex_rev = rev;
  e.regex_key = std::string(fi ? "i" : "") + (fs ? "s" : "") + ":" + p;
}

// concat, `||`, concat_ws, repeat and reverse are typed here for every consumer of the plan IR, but only a consumer built
// with B200_PLAN_STRINGS=1 computes them (the device engine: Makefile NVFLAGS).  Semantics: DESIGN.md §6 (xi).  Their
// arguments are the ones DataFusion's planner leaves after its casts (Utf8; repeat's count Int64).
#ifndef B200_PLAN_STRINGS
#define B200_PLAN_STRINGS 0
#endif
inline bool is_string_builder(const std::string& f) { return f == "concat" || f == "concat_ws" || f == "repeat" || f == "reverse"; }
// string functions whose reference semantics this engine does not restate: refused by name
inline bool is_refused_string_fn(const std::string& f) {
  static const char* const names[] = {"lpad", "rpad", "to_hex", "to_char", "left", "right", "split_part", "translate", "initcap"};
  for (const char* n : names)
    if (f == n) return true;
  return false;
}

// The one-argument float math functions (DESIGN.md §6 (xviii)) in the order of MathFn1 (csrc/device/program.h); -1 for
// another name.  isnan and iszero give Bool, the others their argument's type.
inline int math_fn1_index(const std::string& f) {
  static const char* const names[] = {"sqrt",  "cbrt",  "exp",   "ln",    "log2",  "log10", "sin",     "cos",
                                      "tan",   "asin",  "acos",  "atan",  "sinh",  "cosh",  "tanh",    "asinh",
                                      "acosh", "atanh", "cot",   "degrees", "radians", "signum", "isnan", "iszero"};
  for (int i = 0; i < (int)(sizeof(names) / sizeof(names[0])); i++)
    if (f == names[i]) return i;
  return -1;
}
enum { MATH_ISNAN = 22, MATH_ISZERO = 23 };
inline bool is_math_fn(const std::string& f) {
  return math_fn1_index(f) >= 0 || f == "log" || f == "atan2" || f == "nanvl" || f == "power" || f == "trunc" || f == "gcd" ||
         f == "lcm" || f == "factorial" || f == "pi";
}

// Result type and nullability of a scalar function call (DESIGN.md §3, rules [EXT] in §6).  A known function over an
// argument type it does not take is refused with PlanUnsupported naming the type; an unknown name or a wrong argument
// count is a malformed plan.
inline void type_scalar_fn(Expr& e) {
  const std::string& f = e.fn;
  const size_t n = e.args.size();
  auto arity = [&](size_t lo, size_t hi) {
    if (n < lo || n > hi) throw std::runtime_error("plan IR: " + f + " takes " + std::to_string(lo) + (hi > lo ? ".." + std::to_string(hi) : "") + " argument(s)");
  };
  auto arg_t = [&](size_t i) -> const DataType& { return e.args[i]->type; };
  auto refuse = [&](size_t i) -> void { throw PlanUnsupported(f + " does not support an argument of type " + arg_t(i).str()); };
  auto any_nullable = [&]() {
    bool r = false;
    for (auto& a : e.args) r = r || a->nullable;
    return r;
  };
  auto need_utf8 = [&](size_t i) {
    if (!arg_t(i).is_string() && arg_t(i).id != TypeId::Null) refuse(i);
  };
  if (date_part_index(f) >= 0) {
    arity(1, 1);
    // DataFusion: date_part(part, Date32) -> Int32 [EXT]
    if (arg_t(0).id != TypeId::Date32 && arg_t(0).id != TypeId::Null) refuse(0);
    e.type = DataType(TypeId::Int32);
    e.nullable = e.args[0]->nullable;
  } else if (f == "substr") {
    e.type = DataType(TypeId::Utf8);
    e.nullable = n ? e.args[0]->nullable : false;
  } else if (f == "abs") {
    arity(1, 1);
    if (!arg_t(0).is_numeric()) refuse(0);
    e.type = arg_t(0);
    e.nullable = e.args[0]->nullable;
  } else if (f == "round" || f == "floor" || f == "ceil") {
    arity(1, f == "round" ? 2 : 1);
    if (!arg_t(0).is_float()) refuse(0);
    if (n == 2) {
      if (!arg_t(1).is_integer()) refuse(1);
      const Expr& d = *e.args[1];
      // f = 10^|n| must be exact in binary64 for the result to be the one the formula defines
      if (d.kind == Expr::Lit && !d.lit.is_null && (d.lit.i > 22 || d.lit.i < -22))
        throw PlanUnsupported("round to " + std::to_string(d.lit.i) + " digits is not supported (|digits| <= 22)");
    }
    e.type = arg_t(0);
    e.nullable = any_nullable();
  } else if (is_math_fn(f)) {
    // DESIGN.md §6 (xviii): floats keep their type (Float32 computes in f32); power takes (Float64, Float64) or
    // (Int64, Int64); gcd / lcm / factorial take Int64; every other type is refused, naming it
    const int m1 = math_fn1_index(f);
    const bool two = f == "atan2" || f == "nanvl" || f == "power" || f == "gcd" || f == "lcm";
    if (f == "pi") arity(0, 0);
    else if (f == "log" || f == "trunc") arity(1, 2);
    else arity(two ? 2 : 1, two ? 2 : 1);
    auto need = [&](size_t i, bool ok) {
      if (!ok) refuse(i);
    };
    if (f == "gcd" || f == "lcm" || f == "factorial") {
      for (size_t i = 0; i < n; i++) need(i, arg_t(i).id == TypeId::Int64);
    } else if (f == "power") {
      need(0, arg_t(0).id == TypeId::Int64 || arg_t(0).id == TypeId::Float64);
      need(1, arg_t(1) == arg_t(0));
    } else if (f == "trunc") {
      need(0, arg_t(0).is_float());
      if (n == 2) {
        need(1, arg_t(1).is_integer());
        const Expr& d = *e.args[1];
        // round's factor and limit (the lowering refuses a non-literal digit count)
        if (d.kind == Expr::Lit && !d.lit.is_null && (d.lit.i > 22 || d.lit.i < -22))
          throw PlanUnsupported("trunc to " + std::to_string(d.lit.i) + " digits is not supported (|digits| <= 22)");
      }
    } else {
      for (size_t i = 0; i < n; i++) need(i, arg_t(i).is_float() && arg_t(i) == arg_t(0));
    }
    e.type = f == "pi" ? DataType(TypeId::Float64) : (m1 == MATH_ISNAN || m1 == MATH_ISZERO) ? DataType(TypeId::Bool) : arg_t(0);
    e.nullable = any_nullable();
  } else if (f == "nullif") {
    arity(2, 2);
    if (arg_t(0) != arg_t(1) && arg_t(1).id != TypeId::Null)
      throw PlanUnsupported("nullif of " + arg_t(0).str() + " and " + arg_t(1).str() + " (the arguments must have one type)");
    e.type = arg_t(0);
    e.nullable = true;
  } else if (f == "coalesce") {
    if (n == 0) throw std::runtime_error("plan IR: coalesce takes at least one argument");
    DataType t;
    bool all_nullable = true;
    for (size_t i = 0; i < n; i++) {
      if (arg_t(i).id != TypeId::Null) {
        if (t.id != TypeId::Null && arg_t(i) != t)
          throw PlanUnsupported("coalesce of " + t.str() + " and " + arg_t(i).str() + " (the arguments must have one type)");
        t = arg_t(i);
      }
      all_nullable = all_nullable && e.args[i]->nullable;
    }
    e.type = t;
    e.nullable = all_nullable;
  } else if (f == "character_length" || f == "octet_length") {
    arity(1, 1);
    need_utf8(0);
    e.type = DataType(TypeId::Int32);
    e.nullable = e.args[0]->nullable;
  } else if (f == "starts_with" || f == "ends_with") {
    arity(2, 2);
    need_utf8(0);
    need_utf8(1);
    e.type = DataType(TypeId::Bool);
    e.nullable = any_nullable();
  } else if (f == "regexp_like") {
    arity(2, 3);
    type_regex(e, "regexp_like", e.args[1], n == 3 ? e.args[2] : nullptr, false);
  } else if (f == "regexp_count" || f == "regexp_replace") {
    arity(f == "regexp_count" ? 2 : 3, 4);
    type_regex_fn(e);
  } else if (f == "btrim" || f == "ltrim" || f == "rtrim") {
    arity(1, 2);
    need_utf8(0);
    if (n == 2) need_utf8(1);
    e.type = DataType(TypeId::Utf8);
    e.nullable = any_nullable();
  } else if (is_string_builder(f)) {
    if (!B200_PLAN_STRINGS) throw PlanUnsupported(f + " is not computed by this consumer of the plan IR");
    if (f == "concat") {
      if (n == 0) throw std::runtime_error("plan IR: concat takes at least one argument");
    } else if (f == "concat_ws") {
      if (n < 2) throw std::runtime_error("plan IR: concat_ws takes at least two arguments");
    } else {
      arity(f == "repeat" ? 2 : 1, f == "repeat" ? 2 : 1);
    }
    for (size_t i = 0; i < n; i++) {
      if (f == "repeat" && i == 1) {
        if (arg_t(1).id != TypeId::Int64 && arg_t(1).id != TypeId::Null) refuse(1);
      } else {
        need_utf8(i);
      }
    }
    e.type = DataType(TypeId::Utf8);
    // concat skips NULL arguments (never NULL); concat_ws is NULL iff its separator is
    e.nullable = f == "concat" ? false : f == "concat_ws" ? e.args[0]->nullable : any_nullable();
  } else if (is_refused_string_fn(f)) {
    throw PlanUnsupported("scalar function " + f + " is not supported by the device engine");
  } else {
    throw std::runtime_error("plan IR: unknown scalar function '" + f + "'");
  }
}

inline ExprPtr parse_expr(const Json& j, const Schema& in) {
  auto e = std::make_shared<Expr>();
  if (j.has("col") || j.find("col")) {
    const Json& c = j.at("col");
    if (c.is_str()) {
      for (size_t i = 0; i < in.size(); i++)
        if (in[i].name == c.str()) return make_col((int)i, in);
      throw std::runtime_error("plan IR: unknown column '" + c.str() + "'");
    }
    return make_col((int)c.as_int(), in);
  }
  if (j.find("lit")) {
    const Json& l = j.at("lit");
    e->kind = Expr::Lit;
    e->type = parse_type(l.at("t"));
    const Json* v = l.find("v");
    Json nullj;
    e->lit = parse_lit_value(e->type, v ? *v : nullj);
    e->nullable = e->lit.is_null;
    return e;
  }
  if (j.find("bin")) {
    e->kind = Expr::Bin;
    e->op = parse_binop(j.at("bin").str());
    e->args.push_back(parse_expr(j.at("l"), in));
    e->args.push_back(parse_expr(j.at("r"), in));
    const DataType& a = e->args[0]->type;
    const DataType& b = e->args[1]->type;
    if (is_regex(e->op)) {
      static const char* const names[] = {"~", "~*", "!~", "!~*"};
      const int k = (int)e->op - (int)BinOp::RegexMatch;
      e->negated = e->op == BinOp::RegexNotMatch || e->op == BinOp::RegexNotIMatch;
      type_regex(*e, std::string("the operator ") + names[k], e->args[1], nullptr, e->op == BinOp::RegexIMatch || e->op == BinOp::RegexNotIMatch);
      return e;
    }
    if (e->op == BinOp::StringConcat) {
      if (!B200_PLAN_STRINGS) throw PlanUnsupported("the operator || is not computed by this consumer of the plan IR");
      for (const DataType* t : {&a, &b})
        if (!t->is_string() && t->id != TypeId::Null) throw PlanUnsupported("the operator || does not support an operand of type " + t->str());
      e->type = DataType(TypeId::Utf8);
      e->nullable = e->args[0]->nullable || e->args[1]->nullable;
      return e;
    }
    if (is_bitwise(e->op)) {
      // [EXT] arrow-rs bitwise kernels: integer operands of one type, the result has that type (DESIGN.md §6)
      if (!B200_PLAN_GROUPING_SETS) throw PlanUnsupported("bitwise operators are not computed by this consumer of the plan IR");
      if (!a.is_integer() || a != b) throw PlanUnsupported("bitwise operator between " + a.str() + " and " + b.str() + " (integer operands of one type only)");
      e->type = a;
      e->nullable = e->args[0]->nullable || e->args[1]->nullable;
      return e;
    }
    if (is_arith(e->op)) e->type = arith_result_type(e->op, a, b);
    else e->type = DataType(TypeId::Bool);
    if (is_logic(e->op) && (a.id != TypeId::Bool || b.id != TypeId::Bool) && a.id != TypeId::Null && b.id != TypeId::Null)
      throw std::runtime_error("AND/OR need boolean operands");
    if (is_compare(e->op)) {
      bool ok = (a.pk() == b.pk()) || (a.is_numeric() && b.is_numeric()) || a.id == TypeId::Null || b.id == TypeId::Null;
      if (!ok) throw std::runtime_error("cannot compare " + a.str() + " with " + b.str());
    }
    e->nullable = e->args[0]->nullable || e->args[1]->nullable || e->op == BinOp::Div || e->op == BinOp::Mod;
    return e;
  }
  if (j.find("not")) {
    e->kind = Expr::Not;
    e->args.push_back(parse_expr(j.at("not"), in));
    e->type = DataType(TypeId::Bool);
    e->nullable = e->args[0]->nullable;
    return e;
  }
  if (j.find("neg")) {
    e->kind = Expr::Neg;
    e->args.push_back(parse_expr(j.at("neg"), in));
    e->type = e->args[0]->type;
    e->nullable = e->args[0]->nullable;
    return e;
  }
  if (j.find("is_null") || j.find("is_not_null")) {
    bool isn = j.find("is_null") != nullptr;
    e->kind = isn ? Expr::IsNull : Expr::IsNotNull;
    e->args.push_back(parse_expr(j.at(isn ? "is_null" : "is_not_null"), in));
    e->type = DataType(TypeId::Bool);
    e->nullable = false;
    return e;
  }
  if (j.find("cast")) {
    e->kind = Expr::Cast;
    e->args.push_back(parse_expr(j.at("cast"), in));
    e->type = parse_type(j.at("to"));
    e->nullable = e->args[0]->nullable;
    return e;
  }
  if (j.find("case")) {
    e->kind = Expr::Case;
    const Json& c = j.at("case");
    const Json& whens = c.at("when");
    DataType rt;
    for (size_t i = 0; i < whens.size(); i++) {
      e->args.push_back(parse_expr(whens.at(i).at(0), in));
      e->args.push_back(parse_expr(whens.at(i).at(1), in));
      if (rt.id == TypeId::Null) rt = e->args.back()->type;
    }
    if (c.has("else")) {
      e->args.push_back(parse_expr(c.at("else"), in));
      e->has_else = true;
      if (rt.id == TypeId::Null) rt = e->args.back()->type;
    }
    e->type = rt;
    e->nullable = true;
    return e;
  }
  if (j.find("in")) {
    e->kind = Expr::InList;
    e->args.push_back(parse_expr(j.at("in"), in));
    const Json& lst = j.at("list");
    for (size_t i = 0; i < lst.size(); i++) e->args.push_back(parse_expr(lst.at(i), in));
    e->negated = j.get_bool("negated", false);
    e->type = DataType(TypeId::Bool);
    e->nullable = e->args[0]->nullable;
    return e;
  }
  if (j.find("like")) {
    e->kind = Expr::Like;
    e->args.push_back(parse_expr(j.at("like"), in));
    e->pattern = j.at("pattern").str();
    e->negated = j.get_bool("negated", false);
    e->case_insensitive = j.get_bool("case_insensitive", false);
    e->type = DataType(TypeId::Bool);
    e->nullable = e->args[0]->nullable;
    if (!e->args[0]->type.is_string()) throw std::runtime_error("LIKE needs a utf8 operand");
    if (e->case_insensitive) type_regex(*e, "ILIKE", nullptr, nullptr, true);
    return e;
  }
  if (j.find("fn")) {
    e->kind = Expr::Fn;
    e->fn = j.at("fn").str();
    const Json& as = j.at("args");
    for (size_t i = 0; i < as.size(); i++) e->args.push_back(parse_expr(as.at(i), in));
    type_scalar_fn(*e);
    return e;
  }
  throw std::runtime_error("plan IR: unrecognised expression node");
}

// ----------------------------------------------------------------------------------------------
// Aggregates
// ----------------------------------------------------------------------------------------------
enum class AggFn : uint8_t { Sum, Min, Max, Count, Avg, VarSamp, VarPop, StddevSamp, StddevPop, CovarSamp, CovarPop, Corr,
                              RegrSlope, RegrIntercept, RegrCount, RegrR2, RegrAvgx, RegrAvgy, RegrSxx, RegrSyy, RegrSxy,
                              BoolAnd, BoolOr, BitAnd, BitOr, BitXor, FirstValue, LastValue };
enum class AggMode : uint8_t { Partial, Final, FinalPartitioned, Single, SinglePartitioned };

inline bool agg_mode_consumes_states(AggMode m) { return m == AggMode::Final || m == AggMode::FinalPartitioned; }
inline bool agg_mode_emits_states(AggMode m) { return m == AggMode::Partial; }

// The statistical aggregates: variance / standard deviation (one argument), covariance / correlation and the linear
// regression aggregates (two arguments).  All of them need the two-pass co-moment machinery.
inline bool agg_is_regr(AggFn f) { return f >= AggFn::RegrSlope && f <= AggFn::RegrSxy; }
inline bool agg_is_stat(AggFn f) { return f >= AggFn::VarSamp && f <= AggFn::RegrSxy; }
inline bool agg_is_bivariate(AggFn f) { return f == AggFn::CovarSamp || f == AggFn::CovarPop || f == AggFn::Corr || agg_is_regr(f); }
// bool_and / bool_or / bit_and / bit_or / bit_xor: one-pass folds of a 64-bit word, one state column of the argument's type
inline bool agg_is_bitwise(AggFn f) { return f >= AggFn::BoolAnd && f <= AggFn::BitXor; }
// first_value / last_value: the value of the first / last candidate row under an ordering (DESIGN.md §6 (xvii))
inline bool agg_is_first_last(AggFn f) { return f == AggFn::FirstValue || f == AggFn::LastValue; }
// ordering keys of one first_value / last_value (a stated limit: more are refused, never run partly)
static const size_t kMaxFirstLastKeys = 4;
// [EXT] partial state columns, read by position and checked by suffix in Final modes:
//  var / stddev:  [count] UInt64, [mean] Float64, [m2] Float64  (datafusion-functions-aggregate variance.rs)
//  covar:         [count], [mean1], [mean2], [algo_const]        (covariance.rs)
//  corr:          [count], [mean1], [m2_1], [mean2], [m2_2], [algo_const]  -- unpinned: no reference test fixes it
//  regr_*:        [count], [mean_x], [mean_y], [m2_x], [m2_y], [algo_const]  -- unpinned (regr.rs; DESIGN.md §6 (xvi))
inline std::vector<std::string> stat_state_suffixes(AggFn f) {
  if (agg_is_regr(f)) return {"count", "mean_x", "mean_y", "m2_x", "m2_y", "algo_const"};
  if (f == AggFn::Corr) return {"count", "mean1", "m2_1", "mean2", "m2_2", "algo_const"};
  if (agg_is_bivariate(f)) return {"count", "mean1", "mean2", "algo_const"};
  return {"count", "mean", "m2"};
}

struct SortKey {
  ExprPtr expr;
  bool asc = true;
  bool nulls_first = false;
};

struct AggExpr {
  AggFn fn = AggFn::Sum;
  ExprPtr arg;           // null for COUNT(*) and in Final modes
  ExprPtr arg2;          // COVAR / CORR: the second argument (raw modes only)
  // Final regr_* whose node carries the original arguments and "input_schema" (the protobuf form): y and x typed against
  // that schema.  Every regr_* over one pair has the same partial state, so the engine merges it once per pair.
  ExprPtr state_y, state_x;
  DataType input_type;   // type of arg (after AVG's integer->f64 coercion); for Final: taken from IR
  DataType sum_type;     // accumulator type for Sum/Avg
  DataType result_type;  // final value type
  bool distinct = false;
  std::string name;
  // first_value / last_value: the ordering (raw modes: expressions over the input; Final modes: the state's ordering
  // columns, under the directions the node carries) and IGNORE NULLS
  std::vector<SortKey> order_by;
  bool ignore_nulls = false;
  int n_state_cols() const {
    if (agg_is_first_last(fn)) return 2 + (int)order_by.size();
    return agg_is_stat(fn) ? (int)stat_state_suffixes(fn).size() : fn == AggFn::Avg ? 2 : 1;
  }
};

// [EXT] datafusion-functions-aggregate 53: SUM(Decimal128(p,s)) -> Decimal128(min(38,p+10), s);
// SUM(int) -> Int64, SUM(uint) -> UInt64, SUM(float) -> Float64.
inline DataType sum_result_type(const DataType& t) {
  if (t.is_decimal()) return DataType::decimal(std::min(kMaxDecimalPrecision, t.precision + 10), t.scale);
  if (t.is_signed_int()) return DataType(TypeId::Int64);
  if (t.is_unsigned_int()) return DataType(TypeId::UInt64);
  if (t.is_float()) return DataType(TypeId::Float64);
  throw std::runtime_error("SUM does not support " + t.str());
}
// [EXT] AVG(Decimal128(p,s)) -> Decimal128(min(38,p+4), min(38,s+4)); AVG(other numeric) -> Float64
inline DataType avg_result_type(const DataType& t) {
  if (t.is_decimal())
    return DataType::decimal(std::min(kMaxDecimalPrecision, t.precision + 4), std::min(kMaxDecimalScale, t.scale + 4));
  if (t.is_numeric()) return DataType(TypeId::Float64);
  throw std::runtime_error("AVG does not support " + t.str());
}

// [EXT] VAR / STDDEV / COVAR / CORR take any integer, unsigned, float or Decimal128 argument, coerced to Float64, and return
// a nullable Float64
inline void check_stat_arg(const std::string& fn, const DataType& t) {
  if (!(t.is_integer() || t.is_float() || t.is_decimal())) throw PlanUnsupported(fn + " does not support an argument of type " + t.str());
}
// [EXT] bool_and / bool_or take Bool; bit_and / bit_or / bit_xor take Int8-Int64 and UInt8-UInt64.  The result (and the
// partial state) has the argument's type.
inline void check_bitwise_arg(AggFn f, const std::string& fn, const DataType& t) {
  const bool ok = (f == AggFn::BoolAnd || f == AggFn::BoolOr) ? t.id == TypeId::Bool : t.is_integer();
  if (!ok) throw PlanUnsupported(fn + " does not support an argument of type " + t.str());
}
// [EXT] first_value / last_value take and return any type the engine holds; their ordering keys likewise
inline void check_first_last_type(const std::string& what, const DataType& t) {
  const bool ok = t.id == TypeId::Bool || t.is_integer() || t.is_float() || t.is_decimal() || t.id == TypeId::Date32 || t.id == TypeId::Timestamp ||
                  t.id == TypeId::Utf8;
  if (!ok) throw PlanUnsupported(what + " of type " + t.str() + " is not supported");
}
inline const char* first_last_state_suffix(AggFn f) { return f == AggFn::FirstValue ? "first_value" : "last_value"; }
inline const char* bitwise_state_suffix(AggFn f) {
  switch (f) {
    case AggFn::BoolAnd: return "bool_and";
    case AggFn::BoolOr: return "bool_or";
    case AggFn::BitAnd: return "bit_and";
    case AggFn::BitOr: return "bit_or";
    default: return "bit_xor";
  }
}

// The statistical, regression, bool and bit aggregates are typed here for every consumer of the plan IR, but only a
// consumer built with B200_PLAN_STAT_AGGREGATES=1 computes them (the device engine: Makefile NVFLAGS, for every
// translation unit of the library alike).  Any other consumer -- the CPU oracle -- refuses such a plan instead of
// mis-evaluating it.
#ifndef B200_PLAN_STAT_AGGREGATES
#define B200_PLAN_STAT_AGGREGATES 0
#endif
// the gated names; AggFn::Sum: not one of them
inline AggFn parse_stat_aggfn(const std::string& s) {
  // the lower-cased names and aliases the function registry resolves (datafusion-functions-aggregate)
  if (s == "var" || s == "var_samp" || s == "var_sample") return AggFn::VarSamp;
  if (s == "var_pop" || s == "var_population") return AggFn::VarPop;
  if (s == "stddev" || s == "stddev_samp") return AggFn::StddevSamp;
  if (s == "stddev_pop") return AggFn::StddevPop;
  if (s == "covar" || s == "covar_samp") return AggFn::CovarSamp;
  if (s == "covar_pop") return AggFn::CovarPop;
  if (s == "corr") return AggFn::Corr;
  if (s == "regr_slope") return AggFn::RegrSlope;
  if (s == "regr_intercept") return AggFn::RegrIntercept;
  if (s == "regr_count") return AggFn::RegrCount;
  if (s == "regr_r2") return AggFn::RegrR2;
  if (s == "regr_avgx") return AggFn::RegrAvgx;
  if (s == "regr_avgy") return AggFn::RegrAvgy;
  if (s == "regr_sxx") return AggFn::RegrSxx;
  if (s == "regr_syy") return AggFn::RegrSyy;
  if (s == "regr_sxy") return AggFn::RegrSxy;
  if (s == "bool_and") return AggFn::BoolAnd;
  if (s == "bool_or") return AggFn::BoolOr;
  if (s == "bit_and") return AggFn::BitAnd;
  if (s == "bit_or") return AggFn::BitOr;
  if (s == "bit_xor") return AggFn::BitXor;
  if (s == "first_value") return AggFn::FirstValue;
  if (s == "last_value") return AggFn::LastValue;
  return AggFn::Sum;
}
inline AggFn parse_aggfn(const std::string& s) {
  const AggFn st = parse_stat_aggfn(s);
  if (st != AggFn::Sum) {
    if (!B200_PLAN_STAT_AGGREGATES) throw PlanUnsupported("aggregate '" + s + "' is not computed by this consumer of the plan IR");
    return st;
  }
  if (s == "sum") return AggFn::Sum;
  if (s == "min") return AggFn::Min;
  if (s == "max") return AggFn::Max;
  if (s == "count") return AggFn::Count;
  if (s == "avg") return AggFn::Avg;
  throw std::runtime_error("plan IR: unknown aggregate '" + s + "'");
}
inline AggMode parse_aggmode(const std::string& s) {
  if (s == "Partial") return AggMode::Partial;
  if (s == "Final") return AggMode::Final;
  if (s == "FinalPartitioned") return AggMode::FinalPartitioned;
  if (s == "Single") return AggMode::Single;
  if (s == "SinglePartitioned") return AggMode::SinglePartitioned;
  throw std::runtime_error("plan IR: unknown aggregate mode '" + s + "'");
}

// ----------------------------------------------------------------------------------------------
// Plan nodes
// ----------------------------------------------------------------------------------------------
enum class JoinType : uint8_t { Inner, Left, Right, Full, LeftSemi, RightSemi, LeftAnti, RightAnti };
inline JoinType parse_join_type(const std::string& s) {
  static const std::pair<const char*, JoinType> tab[] = {
      {"Inner", JoinType::Inner},         {"Left", JoinType::Left},           {"Right", JoinType::Right},
      {"Full", JoinType::Full},           {"LeftSemi", JoinType::LeftSemi},   {"RightSemi", JoinType::RightSemi},
      {"LeftAnti", JoinType::LeftAnti},   {"RightAnti", JoinType::RightAnti}};
  for (auto& kv : tab)
    if (s == kv.first) return kv.second;
  throw std::runtime_error("plan IR: unknown join type '" + s + "'");
}

struct NamedExpr {
  ExprPtr expr;
  std::string name;
};

// ----------------------------------------------------------------------------------------------
// Window functions (WindowAggExec / BoundedWindowAggExec): typed here for every consumer of the plan IR, computed only
// by a consumer built with B200_PLAN_WINDOW=1 (the device engine: Makefile NVFLAGS).  Semantics: DESIGN.md §6 (viii).
// ----------------------------------------------------------------------------------------------
#ifndef B200_PLAN_WINDOW
#define B200_PLAN_WINDOW 0
#endif
enum class WinFn : uint8_t {
  RowNumber, Rank, DenseRank, PercentRank, CumeDist, Ntile, Lag, Lead, FirstValue, LastValue, NthValue, Count, Sum, Avg, Min, Max
};
inline bool win_fn_is_agg(WinFn f) { return f >= WinFn::Count; }
inline bool win_fn_uses_frame(WinFn f) { return f >= WinFn::FirstValue; }
// one frame bound; kind follows csrc/device/kernels.h WinBound: 0 UNBOUNDED PRECEDING, 1 n PRECEDING, 2 CURRENT ROW,
// 3 n FOLLOWING, 4 UNBOUNDED FOLLOWING
struct WindowBound {
  uint8_t kind = 0;
  uint64_t n = 0;
};
struct WindowFrame {
  bool range = true;  // RANGE (the default with and without ORDER BY) or ROWS
  WindowBound start, end;
};
struct WindowExpr {
  WinFn fn = WinFn::RowNumber;
  std::string fn_name;      // as written in the plan (aliases kept for the dump)
  std::string name;         // output column
  std::vector<ExprPtr> args;
  int64_t n = 0;            // ntile / nth_value: n; lag / lead: the offset (lead +k, lag -k after the sign of k)
  ExprPtr default_value;    // lag / lead: a literal of the argument's type, or null
  WindowFrame frame;
  DataType result_type;
  bool nullable = true;
};

// Offsets and positions beyond any partition (the operator takes < 2^32 rows) are clamped to this, which keeps every row
// index the kernels form from them far inside int64
static const int64_t kWindowMaxOffset = (int64_t)1 << 40;

// The LAG / LEAD default `d` (a non-NULL literal) as a literal of type `to`, or null when `to` cannot hold it exactly.
// Integers, Date32 and Timestamp take integers in range; Float64 / Float32 take numbers; Decimal128 takes integers and
// decimals of a scale not above its own, within its precision.
inline ExprPtr window_default_as(const ExprPtr& d, const DataType& to) {
  if (d->type == to) return d;
  auto out = std::make_shared<Expr>(*d);
  out->type = to;
  out->nullable = false;
  const DataType& from = d->type;
  const bool from_int = from.is_integer();
  if (to.is_integer() || to.id == TypeId::Date32 || to.id == TypeId::Timestamp) {
    if (!from_int) return nullptr;
    const int64_t v = d->lit.i;
    if (from.id == TypeId::UInt64 && v < 0) return nullptr;  // above INT64_MAX
    static const std::pair<TypeId, std::pair<int64_t, int64_t>> range[] = {
        {TypeId::Int8, {-128, 127}}, {TypeId::Int16, {-32768, 32767}}, {TypeId::Int32, {INT32_MIN, INT32_MAX}},
        {TypeId::UInt8, {0, 255}},   {TypeId::UInt16, {0, 65535}},     {TypeId::UInt32, {0, (int64_t)UINT32_MAX}},
        {TypeId::UInt64, {0, INT64_MAX}}, {TypeId::Date32, {INT32_MIN, INT32_MAX}}};
    for (auto& r : range)
      if (to.id == r.first && (v < r.second.first || v > r.second.second)) return nullptr;
    return out;
  }
  if (to.is_float()) {
    if (from.is_float()) out->lit.f = d->lit.f;
    else if (from_int) out->lit.f = from.id == TypeId::UInt64 ? (double)(uint64_t)d->lit.i : (double)d->lit.i;
    else return nullptr;
    return out;
  }
  if (to.is_decimal()) {
    i128 v;
    if (from_int) {
      if (from.id == TypeId::UInt64 && d->lit.i < 0) return nullptr;
      v = (i128)d->lit.i * pow10_i128(to.scale);
    } else if (from.is_decimal() && from.scale <= to.scale) {
      v = d->lit.d * pow10_i128(to.scale - from.scale);
    } else {
      return nullptr;
    }
    const i128 lim = pow10_i128(to.precision);
    if (v >= lim || v <= -lim) return nullptr;
    out->lit.d = v;
    return out;
  }
  return nullptr;  // Utf8 / Bool arguments take a default of their own type only
}

// structural equality of two typed expressions (window PARTITION BY / ORDER BY against the node's and the sort's keys)
inline bool expr_equal(const ExprPtr& a, const ExprPtr& b) {
  if (!a || !b) return a == b;
  if (a->kind != b->kind || a->type != b->type || a->col != b->col || a->op != b->op || a->fn != b->fn || a->negated != b->negated || a->case_insensitive != b->case_insensitive ||
      a->has_else != b->has_else || a->pattern != b->pattern || a->args.size() != b->args.size())
    return false;
  if (a->kind == Expr::Lit && (a->lit.is_null != b->lit.is_null || a->lit.i != b->lit.i || a->lit.d != b->lit.d || a->lit.s != b->lit.s ||
                               !(a->lit.f == b->lit.f || (a->lit.f != a->lit.f && b->lit.f != b->lit.f))))
    return false;
  for (size_t k = 0; k < a->args.size(); k++)
    if (!expr_equal(a->args[k], b->args[k])) return false;
  return true;
}

struct PlanNode;
typedef std::unique_ptr<PlanNode> PlanPtr;

struct PlanNode {
  enum Op {
    Scan, ShuffleReader, Filter, Projection, Aggregate, HashJoin, Sort, SortPreservingMerge,
    Passthrough /* CoalesceBatches, CoalescePartitions, round-robin Repartition */, Limit, ShuffleWriter, Window
  } op = Scan;
  std::string op_name;
  std::vector<PlanPtr> children;
  Schema schema;  // output schema

  // Scan
  std::string table;
  std::vector<int> scan_projection;  // indices into the registered table's schema
  // ShuffleReader
  int64_t reader_stage_id = 0;
  bool broadcast = false;
  // Filter
  ExprPtr predicate;
  std::vector<int> projection;  // Filter / HashJoin optional output projection
  bool has_projection = false;
  // Projection
  std::vector<NamedExpr> exprs;
  // Aggregate
  AggMode agg_mode = AggMode::Single;
  std::vector<NamedExpr> group_by;
  std::vector<AggExpr> aggs;
  std::vector<uint32_t> grouping_sets;  // empty: a plain GROUP BY; else one mask per set, bit k = key k replaced by NULL
  // HashJoin
  JoinType join_type = JoinType::Inner;
  std::string partition_mode;  // CollectLeft | Partitioned
  std::vector<std::pair<ExprPtr, ExprPtr>> on;
  bool null_equals_null = false;
  ExprPtr join_filter;  // over concat(left schema, right schema)
  bool nested_loop = false;  // NestedLoopJoinExec: no keys, every (build, probe) pair is tested against the filter
  // Sort / SPM / Limit
  std::vector<SortKey> sort_keys;
  int64_t fetch = -1;
  int64_t skip = 0;
  bool preserve_partitioning = false;
  // ShuffleWriter
  std::string job_id;
  int64_t stage_id = 0;
  std::vector<ExprPtr> part_exprs;
  int64_t n_out_partitions = 0;  // 0 => no repartitioning ("None" branch, shuffle_writer.rs:221-268)
  bool sort_shuffle = true;
  // Window: the input's columns, then one column per expression.  All expressions share the partition keys and ORDER BY.
  bool window_sorted = false;        // BoundedWindowAggExec (input_order_mode sorted); false: WindowAggExec
  std::vector<ExprPtr> window_partition;
  std::vector<SortKey> window_order;
  std::vector<WindowExpr> window_exprs;
};

// deep copy of an expression with every column reference moved by `delta` positions
inline ExprPtr shift_cols(const ExprPtr& e, int delta) {
  if (!e || delta == 0) return e;
  auto c = std::make_shared<Expr>(*e);
  if (c->kind == Expr::Col) c->col += delta;
  for (auto& a : c->args) a = shift_cols(a, delta);
  return c;
}

inline std::vector<SortKey> parse_sort_keys(const Json& j, const Schema& in) {
  std::vector<SortKey> ks;
  for (size_t i = 0; i < j.size(); i++) {
    SortKey k;
    k.expr = parse_expr(j.at(i).at("expr"), in);
    k.asc = j.at(i).get_bool("asc", true);
    k.nulls_first = j.at(i).get_bool("nulls_first", !k.asc);  // SQL default: NULLS LAST for ASC, FIRST for DESC
    ks.push_back(k);
  }
  return ks;
}

PlanPtr parse_plan(const Json& j);

inline PlanPtr parse_plan(const Json& j) {
  auto n = PlanPtr(new PlanNode());
  const std::string& op = j.at("op").str();
  n->op_name = op;
  auto parse_child = [&](const char* key) {
    n->children.push_back(parse_plan(j.at(key)));
    return n->children.back().get();
  };
  if (op == "DataSourceExec" || op == "MemoryScan" || op == "Scan") {
    n->op = PlanNode::Scan;
    n->table = j.at("table").str();
    Schema full = parse_schema(j.at("schema"));
    if (j.has("projection")) {
      const Json& p = j.at("projection");
      for (size_t i = 0; i < p.size(); i++) {
        int idx = (int)p.at(i).as_int();
        if (idx < 0 || (size_t)idx >= full.size()) throw std::runtime_error("scan projection out of range");
        n->scan_projection.push_back(idx);
        n->schema.push_back(full[idx]);
      }
    } else {
      for (size_t i = 0; i < full.size(); i++) n->scan_projection.push_back((int)i);
      n->schema = full;
    }
  } else if (op == "ShuffleReaderExec" || op == "UnresolvedShuffleExec") {
    n->op = PlanNode::ShuffleReader;
    n->reader_stage_id = j.at("stage_id").as_int();
    n->schema = parse_schema(j.at("schema"));
    n->broadcast = j.get_bool("broadcast", false);
  } else if (op == "FilterExec") {
    n->op = PlanNode::Filter;
    PlanNode* c = parse_child("input");
    n->predicate = parse_expr(j.at("predicate"), c->schema);
    if (n->predicate->type.id != TypeId::Bool) throw std::runtime_error("FilterExec predicate must be boolean");
    if (j.has("projection")) {
      n->has_projection = true;
      const Json& p = j.at("projection");
      for (size_t i = 0; i < p.size(); i++) {
        int idx = (int)p.at(i).as_int();
        if (idx < 0 || (size_t)idx >= c->schema.size()) throw std::runtime_error("filter projection out of range");
        n->projection.push_back(idx);
        n->schema.push_back(c->schema[idx]);
      }
    } else {
      n->schema = c->schema;
    }
    n->fetch = j.get_int("fetch", -1);
  } else if (op == "ProjectionExec") {
    n->op = PlanNode::Projection;
    PlanNode* c = parse_child("input");
    const Json& es = j.at("exprs");
    for (size_t i = 0; i < es.size(); i++) {
      NamedExpr ne;
      ne.expr = parse_expr(es.at(i).at("expr"), c->schema);
      ne.name = es.at(i).get_str("name", ne.expr->name.empty() ? ("c" + std::to_string(i)) : ne.expr->name);
      n->exprs.push_back(ne);
      Field f;
      f.name = ne.name;
      f.type = ne.expr->type;
      f.nullable = ne.expr->nullable;
      n->schema.push_back(f);
    }
  } else if (op == "AggregateExec") {
    n->op = PlanNode::Aggregate;
    PlanNode* c = parse_child("input");
    n->agg_mode = parse_aggmode(j.at("mode").str());
    bool from_states = agg_mode_consumes_states(n->agg_mode);
    const Json& gs = j.at("group_by");
    for (size_t i = 0; i < gs.size(); i++) {
      NamedExpr ne;
      if (from_states) ne.expr = make_col((int)i, c->schema);  // group keys are the leading columns of the partial output
      else ne.expr = parse_expr(gs.at(i).at("expr"), c->schema);
      ne.name = gs.at(i).get_str("name", ne.expr->name.empty() ? ("g" + std::to_string(i)) : ne.expr->name);
      n->group_by.push_back(ne);
      Field f;
      f.name = ne.name;
      f.type = ne.expr->type;
      f.nullable = ne.expr->nullable;
      n->schema.push_back(f);
    }
    if (j.has("grouping_sets")) {
      // every row is aggregated once per set; the output holds the keys (all nullable), then __grouping_id (DESIGN.md §6)
      if (!B200_PLAN_GROUPING_SETS) throw PlanUnsupported("grouping sets are not computed by this consumer of the plan IR");
      if (from_states) throw std::runtime_error("AggregateExec: a Final-mode aggregate carries no grouping sets");
      const Json& sets = j.at("grouping_sets");
      const size_t nk = gs.size();
      if (sets.size() == 0) throw std::runtime_error("AggregateExec: empty grouping_sets");
      for (size_t s = 0; s < sets.size(); s++) {
        const Json& set = sets.at(s);
        if (set.size() != nk) throw std::runtime_error("AggregateExec: grouping set " + std::to_string(s) + " has " + std::to_string(set.size()) + " entries for " + std::to_string(nk) + " keys");
        uint32_t mask = 0;
        for (size_t k = 0; k < nk && k < 32; k++) mask |= (set.at(k).as_bool() ? 1u : 0u) << k;
        n->grouping_sets.push_back(mask);
      }
      if (nk == 0) throw PlanUnsupported("grouping sets without a group key are not supported");
      if (nk > kMaxGroupingSetKeys)
        throw PlanUnsupported("grouping sets over " + std::to_string(nk) + " keys are not supported (at most " + std::to_string(kMaxGroupingSetKeys) + ")");
      if (sets.size() > kMaxGroupingSets)
        throw PlanUnsupported(std::to_string(sets.size()) + " grouping sets are not supported (at most " + std::to_string(kMaxGroupingSets) + ")");
      for (size_t s = 0; s < n->grouping_sets.size(); s++)
        for (size_t t = 0; t < s; t++)
          if (n->grouping_sets[s] == n->grouping_sets[t])
            throw PlanUnsupported("duplicate grouping set " + std::to_string(s) + " (same as set " + std::to_string(t) + ", __grouping_id " +
                                  std::to_string(grouping_id(n->grouping_sets[s], nk)) + ")");
      for (auto& f : n->schema) f.nullable = true;
      n->schema.push_back(Field{"__grouping_id", grouping_id_type(nk), false});
    }
    const Json& as = j.at("aggr");
    size_t state_col = gs.size();
    for (size_t i = 0; i < as.size(); i++) {
      const Json& a = as.at(i);
      AggExpr ae;
      ae.fn = parse_aggfn(a.at("fn").str());
      ae.distinct = a.get_bool("distinct", false);
      if (ae.distinct) throw std::runtime_error("DISTINCT aggregates must be lowered to two-level aggregation by the planner");
      ae.name = a.get_str("name", a.at("fn").str() + "_" + std::to_string(i));
      if (agg_is_first_last(ae.fn)) {
        const std::string fnn = a.at("fn").str();
        ae.ignore_nulls = a.get_bool("ignore_nulls", false);
        Json no_keys;
        const Json& ob = a.has("order_by") ? a.at("order_by") : no_keys;
        if (ob.size() > kMaxFirstLastKeys)
          throw PlanUnsupported(fnn + " (" + ae.name + ") with " + std::to_string(ob.size()) + " ordering keys is not supported (at most " +
                                std::to_string(kMaxFirstLastKeys) + ")");
        if (from_states) {
          // [<name>[first_value|last_value]] (x), one column per ordering key, [is_set] Bool: read positionally and refused
          // when the layout differs.  The ordering comes from those columns, under the directions this node carries.
          const size_t nk = ob.size();
          if (state_col + 1 + nk >= c->schema.size()) throw std::runtime_error("Final aggregate: missing state columns of " + ae.name);
          auto ends_with = [](const std::string& a, const std::string& b) { return a.size() >= b.size() && a.compare(a.size() - b.size(), b.size(), b) == 0; };
          const Field& fv = c->schema[state_col];
          const std::string want = std::string("[") + first_last_state_suffix(ae.fn) + "]";
          if (!ends_with(fv.name, want)) throw PlanUnsupported("Final " + fnn + ": state column '" + fv.name + "' is not the expected '" + want + "'");
          const Field& fs = c->schema[state_col + 1 + nk];
          if (!ends_with(fs.name, "is_set") || fs.type.id != TypeId::Bool)
            throw PlanUnsupported("Final " + fnn + ": state column '" + fs.name + "' (" + fs.type.str() + ") is not the expected 'is_set' (bool) after " +
                                  std::to_string(nk) + " ordering column(s)");
          check_first_last_type("Final " + fnn + " state column '" + fv.name + "'", fv.type);
          for (size_t k = 0; k < nk; k++) {
            SortKey sk;
            sk.expr = make_col((int)(state_col + 1 + k), c->schema);
            sk.asc = ob.at(k).get_bool("asc", true);
            sk.nulls_first = ob.at(k).get_bool("nulls_first", !sk.asc);
            check_first_last_type("Final " + fnn + " ordering state column '" + c->schema[state_col + 1 + k].name + "'", sk.expr->type);
            ae.order_by.push_back(sk);
          }
          ae.input_type = fv.type;
          state_col += ae.n_state_cols();
        } else {
          if (!a.has("args") || a.at("args").size() != 1) throw std::runtime_error(fnn + " takes 1 argument(s)");
          ae.arg = parse_expr(a.at("args").at(0), c->schema);
          check_first_last_type(fnn + " argument", ae.arg->type);
          ae.order_by = parse_sort_keys(ob, c->schema);
          for (auto& k : ae.order_by) check_first_last_type(fnn + " ordering key", k.expr->type);
          ae.input_type = ae.arg->type;
        }
        ae.sum_type = ae.input_type;
        ae.result_type = ae.input_type;
      } else if (from_states && agg_is_stat(ae.fn)) {
        // states are read positionally; a column whose name does not end in the expected suffix means a layout this
        // engine does not know, which is refused rather than misread
        const std::vector<std::string> sfx = stat_state_suffixes(ae.fn);
        for (size_t k = 0; k < sfx.size(); k++) {
          if (state_col + k >= c->schema.size()) throw std::runtime_error("Final aggregate: missing state columns of " + ae.name);
          const Field& f = c->schema[state_col + k];
          const std::string want = "[" + sfx[k] + "]";
          const bool name_ok = f.name.size() >= want.size() && f.name.compare(f.name.size() - want.size(), want.size(), want) == 0;
          const bool type_ok = k == 0 ? f.type.is_integer() : f.type.id == TypeId::Float64;
          if (!name_ok || !type_ok)
            throw PlanUnsupported("Final " + a.at("fn").str() + ": state column '" + f.name + "' (" + f.type.str() + ") is not the expected '" + want + "'");
        }
        if (agg_is_regr(ae.fn) && j.has("input_schema") && a.has("args") && a.at("args").size() == 2) {
          const auto is = parse_schema(j.at("input_schema"));
          ae.state_y = parse_expr(a.at("args").at(0), is);
          ae.state_x = parse_expr(a.at("args").at(1), is);
          check_stat_arg(a.at("fn").str(), ae.state_y->type);
          check_stat_arg(a.at("fn").str(), ae.state_x->type);
        }
        ae.input_type = DataType(TypeId::Float64);
        ae.sum_type = ae.input_type;
        ae.result_type = ae.fn == AggFn::RegrCount ? DataType(TypeId::UInt64) : ae.input_type;
        state_col += ae.n_state_cols();
      } else if (from_states && agg_is_bitwise(ae.fn)) {
        // one state column of the argument's type, merged with the same operation
        if (state_col >= c->schema.size()) throw std::runtime_error("Final aggregate: missing state column of " + ae.name);
        check_bitwise_arg(ae.fn, "Final " + a.at("fn").str() + " state column '" + c->schema[state_col].name + "':", c->schema[state_col].type);
        ae.input_type = c->schema[state_col].type;
        ae.sum_type = ae.input_type;
        ae.result_type = ae.input_type;
        state_col += ae.n_state_cols();
      } else if (from_states) {
        // states are read positionally: AVG -> (count:UInt64, sum), others -> one column
        if (ae.fn == AggFn::Avg) {
          if (state_col + 1 >= c->schema.size()) throw std::runtime_error("Final aggregate: missing AVG state columns");
          ae.sum_type = c->schema[state_col + 1].type;
          if (a.has("input_type")) {
            ae.input_type = parse_type(a.at("input_type"));
          } else if (j.has("input_schema") && a.has("args") && a.at("args").size() > 0) {
            // the protobuf form (AggregateExecNode.input_schema = 7 + the original argument expression): typed here
            ae.input_type = parse_expr(a.at("args").at(0), parse_schema(j.at("input_schema")))->type;
          } else {
            throw std::runtime_error("Final AVG needs \"input_type\" (or the original argument and \"input_schema\")");
          }
          ae.result_type = avg_result_type(ae.input_type);
        } else {
          if (state_col >= c->schema.size()) throw std::runtime_error("Final aggregate: missing state column");
          ae.input_type = c->schema[state_col].type;
          ae.sum_type = ae.input_type;
          ae.result_type = ae.input_type;
        }
        state_col += ae.n_state_cols();
      } else {
        if (a.has("args") && a.at("args").size() > 0) {
          ae.arg = parse_expr(a.at("args").at(0), c->schema);
          // COUNT(<non-null literal>) is COUNT(*)
          if (ae.fn == AggFn::Count && ae.arg->kind == Expr::Lit && !ae.arg->lit.is_null) ae.arg = nullptr;
        }
        if (!ae.arg && ae.fn != AggFn::Count) throw std::runtime_error("aggregate needs an argument");
        DataType it = ae.arg ? ae.arg->type : DataType(TypeId::Int64);
        if (agg_is_stat(ae.fn)) {
          const size_t want = agg_is_bivariate(ae.fn) ? 2 : 1;
          if (a.at("args").size() != want) throw std::runtime_error(a.at("fn").str() + " takes " + std::to_string(want) + " argument(s)");
          check_stat_arg(a.at("fn").str(), it);
          if (want == 2) {
            ae.arg2 = parse_expr(a.at("args").at(1), c->schema);
            check_stat_arg(a.at("fn").str(), ae.arg2->type);
          }
          it = DataType(TypeId::Float64);
        } else if (agg_is_bitwise(ae.fn)) {
          if (a.at("args").size() != 1) throw std::runtime_error(a.at("fn").str() + " takes 1 argument(s)");
          check_bitwise_arg(ae.fn, a.at("fn").str(), it);
        }
        switch (ae.fn) {
          case AggFn::Sum:
            ae.input_type = it;
            ae.sum_type = sum_result_type(it);
            ae.result_type = ae.sum_type;
            break;
          case AggFn::Avg:
            ae.input_type = it;
            // [EXT] AVG over non-decimal numerics is computed in Float64 (input cast to f64 first)
            ae.sum_type = it.is_decimal() ? sum_result_type(it) : DataType(TypeId::Float64);
            ae.result_type = avg_result_type(it);
            break;
          case AggFn::Count:
            ae.input_type = it;
            ae.sum_type = DataType(TypeId::Int64);
            ae.result_type = DataType(TypeId::Int64);
            break;
          case AggFn::RegrCount:
            ae.input_type = it;
            ae.sum_type = it;
            ae.result_type = DataType(TypeId::UInt64);
            break;
          default:
            ae.input_type = it;
            ae.sum_type = it;
            ae.result_type = it;
        }
      }
      n->aggs.push_back(ae);
      if (agg_mode_emits_states(n->agg_mode)) {
        if (agg_is_stat(ae.fn)) {
          const std::vector<std::string> sfx = stat_state_suffixes(ae.fn);
          for (size_t k = 0; k < sfx.size(); k++)
            n->schema.push_back(Field{ae.name + "[" + sfx[k] + "]", DataType(k == 0 ? TypeId::UInt64 : TypeId::Float64), true});
        } else if (ae.fn == AggFn::Avg) {
          n->schema.push_back(Field{ae.name + "[count]", DataType(TypeId::UInt64), true});
          n->schema.push_back(Field{ae.name + "[sum]", ae.sum_type, true});
        } else if (ae.fn == AggFn::Count) {
          n->schema.push_back(Field{ae.name + "[count]", DataType(TypeId::Int64), false});
        } else if (ae.fn == AggFn::Sum) {
          n->schema.push_back(Field{ae.name + "[sum]", ae.sum_type, true});
        } else if (agg_is_bitwise(ae.fn)) {
          n->schema.push_back(Field{ae.name + "[" + bitwise_state_suffix(ae.fn) + "]", ae.sum_type, true});
        } else if (agg_is_first_last(ae.fn)) {
          // [EXT-unverified] the ordering columns are named by the sort expression's display string ("ts@2" for a column)
          n->schema.push_back(Field{ae.name + "[" + first_last_state_suffix(ae.fn) + "]", ae.result_type, true});
          for (size_t k = 0; k < ae.order_by.size(); k++) {
            const Expr& e = *ae.order_by[k].expr;
            const std::string nm = e.kind == Expr::Col ? c->schema[(size_t)e.col].name + "@" + std::to_string(e.col) : ae.name + "[order_" + std::to_string(k) + "]";
            n->schema.push_back(Field{nm, e.type, true});
          }
          n->schema.push_back(Field{"is_set", DataType(TypeId::Bool), true});
        } else {
          n->schema.push_back(Field{ae.name + (ae.fn == AggFn::Min ? "[min]" : "[max]"), ae.sum_type, true});
        }
      } else {
        // [EXT] COUNT and regr_count are never NULL (0 for an empty group)
        n->schema.push_back(Field{ae.name, ae.result_type, ae.fn != AggFn::Count && ae.fn != AggFn::RegrCount});
      }
      if (!n->grouping_sets.empty() && (agg_is_stat(ae.fn) || agg_is_first_last(ae.fn)))
        throw PlanUnsupported(a.at("fn").str() + " (" + ae.name + ") alongside grouping sets is not supported");
    }
  } else if (op == "HashJoinExec" || op == "SortMergeJoinExec" || op == "NestedLoopJoinExec") {
    // SortMergeJoinExec (datafusion.proto:1433, Ballista's default join, extension.rs:683): same matching
    // semantics as the hash join over co-partitioned inputs; its contract adds an output ordered by the
    // join keys (sort_options), which both engines establish by sorting the join result.
    // NestedLoopJoinExec (datafusion.proto:1301-1307): a join without equality keys.  DataFusion requires a single
    // partition on its left input, so the left side is the build side and every task reads it whole (CollectLeft).
    const bool smj = op == "SortMergeJoinExec";
    const bool nlj = op == "NestedLoopJoinExec";
    n->op = PlanNode::HashJoin;
    n->nested_loop = nlj;
    PlanNode* l = parse_child("left");
    PlanNode* r = parse_child("right");
    n->join_type = parse_join_type(j.get_str("join_type", "Inner"));
    n->partition_mode = smj ? std::string("Partitioned") : nlj ? std::string("CollectLeft") : j.get_str("mode", "Partitioned");
    n->null_equals_null = j.get_bool("null_equals_null", false);
    Json no_keys;
    const Json& on = nlj ? (j.has("on") ? j.at("on") : no_keys) : j.at("on");
    if (nlj && on.size() > 0) throw std::runtime_error("NestedLoopJoinExec has no equality keys");
    for (size_t i = 0; i < on.size(); i++) {
      ExprPtr le = parse_expr(on.at(i).at(0), l->schema);
      ExprPtr re = parse_expr(on.at(i).at(1), r->schema);
      if (le->type.pk() != re->type.pk()) throw std::runtime_error("join key types differ: " + le->type.str() + " vs " + re->type.str());
      n->on.emplace_back(le, re);
    }
    Schema both;
    bool lnull = n->join_type == JoinType::Right || n->join_type == JoinType::Full;
    bool rnull = n->join_type == JoinType::Left || n->join_type == JoinType::Full;
    Schema cat = l->schema;
    cat.insert(cat.end(), r->schema.begin(), r->schema.end());
    if (j.has("filter") && j.has("filter_columns")) {
      // the protobuf form (JoinFilter, datafusion.proto:1343-1352): the expression indexes an intermediate schema whose k-th
      // column is (side, index) of an input; rewritten here onto the left ++ right schema the engines evaluate it on
      const Json& fc = j.at("filter_columns");
      Schema inter;
      std::vector<int> target;
      for (size_t k = 0; k < fc.size(); k++) {
        const int side = (int)fc.at(k).at(0).as_int(), idx = (int)fc.at(k).at(1).as_int();
        const Schema& src = side == 0 ? l->schema : r->schema;
        if (side < 0 || side > 1 || idx < 0 || (size_t)idx >= src.size()) throw std::runtime_error("join filter column out of range");
        inter.push_back(src[idx]);
        target.push_back(side == 0 ? idx : (int)l->schema.size() + idx);
      }
      n->join_filter = parse_expr(j.at("filter"), inter);
      remap_columns(n->join_filter, target);
    } else if (j.has("filter")) {
      n->join_filter = parse_expr(j.at("filter"), cat);
    }
    switch (n->join_type) {
      case JoinType::LeftSemi:
      case JoinType::LeftAnti: both = l->schema; break;
      case JoinType::RightSemi:
      case JoinType::RightAnti: both = r->schema; break;
      default:
        for (auto f : l->schema) {
          f.nullable = f.nullable || lnull;
          both.push_back(f);
        }
        for (auto f : r->schema) {
          f.nullable = f.nullable || rnull;
          both.push_back(f);
        }
    }
    if (j.has("projection")) {
      n->has_projection = true;
      const Json& p = j.at("projection");
      for (size_t i = 0; i < p.size(); i++) {
        int idx = (int)p.at(i).as_int();
        if (idx < 0 || (size_t)idx >= both.size()) throw std::runtime_error("join projection out of range");
        n->projection.push_back(idx);
        n->schema.push_back(both[idx]);
      }
    } else {
      n->schema = both;
    }
    if (smj) {
      if (n->has_projection) throw std::runtime_error("SortMergeJoinExec has no projection");
      const bool right_side = n->join_type == JoinType::Right || n->join_type == JoinType::RightSemi || n->join_type == JoinType::RightAnti;
      const int shift = n->join_type == JoinType::Right ? (int)l->schema.size() : 0;
      for (size_t i = 0; i < n->on.size(); i++) {
        SortKey k;
        k.expr = right_side ? shift_cols(n->on[i].second, shift) : n->on[i].first;
        if (j.has("sort_options") && i < j.at("sort_options").size()) {
          const Json& so = j.at("sort_options").at(i);
          k.asc = so.get_bool("asc", true);
          k.nulls_first = so.get_bool("nulls_first", !k.asc);
        }
        n->sort_keys.push_back(k);
      }
    }
  } else if (op == "SortExec" || op == "SortPreservingMergeExec") {
    n->op = op == "SortExec" ? PlanNode::Sort : PlanNode::SortPreservingMerge;
    PlanNode* c = parse_child("input");
    n->schema = c->schema;
    n->sort_keys = parse_sort_keys(j.at("expr"), c->schema);
    n->fetch = j.get_int("fetch", -1);
    n->preserve_partitioning = j.get_bool("preserve_partitioning", false);
  } else if (op == "CoalesceBatchesExec" || op == "CoalescePartitionsExec" || op == "RepartitionExec") {
    n->op = PlanNode::Passthrough;
    PlanNode* c = parse_child("input");
    n->schema = c->schema;
  } else if (op == "WindowAggExec" || op == "BoundedWindowAggExec") {
    n->op = PlanNode::Window;
    PlanNode* c = parse_child("input");
    if (!B200_PLAN_WINDOW) throw PlanUnsupported("window functions are not computed by this consumer of the plan IR");
    if (j.has("mode") && !j.at("mode").is_null()) {
      const std::string m = j.at("mode").str();
      if (m == "linear" || m == "partially_sorted") throw PlanUnsupported("window input order mode " + m + " is not supported");
      if (m != "sorted") throw std::runtime_error("WindowAggExec: unknown input order mode '" + m + "'");
      n->window_sorted = true;
    }
    if (op == "BoundedWindowAggExec") n->window_sorted = true;
    if (j.has("partition_keys"))
      for (size_t i = 0; i < j.at("partition_keys").size(); i++) n->window_partition.push_back(parse_expr(j.at("partition_keys").at(i), c->schema));
    n->schema = c->schema;
    const Json& ws = j.at("window_expr");
    if (ws.size() == 0) throw std::runtime_error("WindowAggExec without window expressions");
    for (size_t i = 0; i < ws.size(); i++) {
      const Json& w = ws.at(i);
      WindowExpr we;
      we.fn_name = w.at("fn").str();
      we.name = w.get_str("name", we.fn_name + "_" + std::to_string(i));
      const std::string& f = we.fn_name;
      const std::string who = f + " (" + we.name + ")";
      if (w.get_bool("ignore_nulls", false)) throw PlanUnsupported("IGNORE NULLS in window function " + who + " is not supported");
      if (w.get_bool("distinct", false)) throw PlanUnsupported("DISTINCT window function " + who + " is not supported");
      static const std::pair<const char*, WinFn> fns[] = {
          {"row_number", WinFn::RowNumber}, {"rank", WinFn::Rank},         {"dense_rank", WinFn::DenseRank}, {"percent_rank", WinFn::PercentRank},
          {"cume_dist", WinFn::CumeDist},   {"ntile", WinFn::Ntile},       {"lag", WinFn::Lag},              {"lead", WinFn::Lead},
          {"first_value", WinFn::FirstValue}, {"last_value", WinFn::LastValue}, {"nth_value", WinFn::NthValue}, {"count", WinFn::Count},
          {"sum", WinFn::Sum},              {"avg", WinFn::Avg},           {"mean", WinFn::Avg},             {"min", WinFn::Min},
          {"max", WinFn::Max}};
      bool known = false;
      for (auto& kv : fns)
        if (f == kv.first) {
          we.fn = kv.second;
          known = true;
        }
      if (!known) throw PlanUnsupported("window function " + who + " is not supported");
      std::vector<ExprPtr> part;
      if (w.has("partition_by"))
        for (size_t k = 0; k < w.at("partition_by").size(); k++) part.push_back(parse_expr(w.at("partition_by").at(k), c->schema));
      bool same_part = part.size() == n->window_partition.size();
      for (size_t k = 0; k < part.size() && same_part; k++) {
        bool found = false;
        for (auto& pk : n->window_partition) found = found || expr_equal(part[k], pk);
        same_part = found;
      }
      if (!same_part) throw PlanUnsupported("window function " + who + ": its PARTITION BY differs from the node's partition keys");
      std::vector<SortKey> order = w.has("order_by") ? parse_sort_keys(w.at("order_by"), c->schema) : std::vector<SortKey>();
      if (i == 0) {
        n->window_order = order;
      } else {
        bool same = order.size() == n->window_order.size();
        for (size_t k = 0; k < order.size() && same; k++)
          same = expr_equal(order[k].expr, n->window_order[k].expr) && order[k].asc == n->window_order[k].asc && order[k].nulls_first == n->window_order[k].nulls_first;
        if (!same) throw PlanUnsupported("window function " + who + ": its ORDER BY differs from that of the node's other expressions");
      }
      if (w.has("frame") && !w.at("frame").is_null()) {
        const Json& fr = w.at("frame");
        const std::string units = fr.get_str("units", "range");
        if (units == "groups") throw PlanUnsupported("GROUPS window frame of " + who + " is not supported");
        if (units != "rows" && units != "range") throw std::runtime_error("window frame units '" + units + "'");
        we.frame.range = units == "range";
        auto bound = [&](const Json& b, const char* side) {
          static const char* kinds[] = {"unbounded_preceding", "preceding", "current_row", "following", "unbounded_following"};
          WindowBound wb;
          const std::string k = b.at("kind").str();
          bool ok = false;
          for (uint8_t t = 0; t < 5; t++)
            if (k == kinds[t]) {
              wb.kind = t;
              ok = true;
            }
          if (!ok) throw std::runtime_error("window frame bound '" + k + "'");
          if (wb.kind == 1 || wb.kind == 3) {
            if (we.frame.range) throw PlanUnsupported("RANGE window frame with an offset bound (" + std::string(side) + " of " + who + ") is not supported");
            const Json& v = b.at("n");
            if (!v.is_int || v.i < 0) throw PlanUnsupported("ROWS frame offset of " + who + " must be a non-negative integer literal");
            wb.n = (uint64_t)v.i;
          }
          return wb;
        };
        we.frame.start = bound(fr.at("start"), "start");
        we.frame.end = bound(fr.at("end"), "end");
        if (we.frame.start.kind == 4) throw std::runtime_error("window frame of " + who + " starts at UNBOUNDED FOLLOWING");
        if (we.frame.end.kind == 0) throw std::runtime_error("window frame of " + who + " ends at UNBOUNDED PRECEDING");
      } else {
        we.frame.range = true;
        we.frame.start.kind = 0;
        we.frame.end.kind = 2;
      }
      const Json no_args;
      const Json& as = w.has("args") ? w.at("args") : no_args;
      for (size_t k = 0; k < as.size(); k++) we.args.push_back(parse_expr(as.at(k), c->schema));
      auto int_literal = [&](size_t k, const char* what) -> int64_t {
        const ExprPtr& e = we.args[k];
        if (e->kind != Expr::Lit || e->lit.is_null || !(e->type.is_integer()))
          throw PlanUnsupported(std::string(what) + " of " + who + " must be an integer literal");
        return e->lit.i;
      };
      auto want_args = [&](size_t lo, size_t hi) {
        if (we.args.size() < lo || we.args.size() > hi) throw std::runtime_error(who + " takes " + std::to_string(lo) + ".." + std::to_string(hi) + " arguments");
      };
      switch (we.fn) {
        case WinFn::RowNumber:
        case WinFn::Rank:
        case WinFn::DenseRank:
          want_args(0, 0);
          we.result_type = DataType(TypeId::UInt64);
          we.nullable = false;
          break;
        case WinFn::PercentRank:
        case WinFn::CumeDist:
          want_args(0, 0);
          we.result_type = DataType(TypeId::Float64);
          we.nullable = false;
          break;
        case WinFn::Ntile:
          want_args(1, 1);
          we.n = int_literal(0, "the bucket count");
          if (we.n < 1) throw std::runtime_error("ntile of " + who + " needs n >= 1, got " + std::to_string(we.n));
          we.args.clear();
          we.result_type = DataType(TypeId::UInt64);
          break;
        case WinFn::Lag:
        case WinFn::Lead: {
          want_args(1, 3);
          int64_t k = we.args.size() > 1 ? int_literal(1, "the offset") : 1;
          k = std::max<int64_t>(-kWindowMaxOffset, std::min<int64_t>(k, kWindowMaxOffset));  // past any partition: the default
          we.n = we.fn == WinFn::Lead ? k : -k;
          if (we.args.size() > 2) {
            const ExprPtr& d = we.args[2];
            if (d->kind != Expr::Lit) throw PlanUnsupported("the default of " + who + " must be a literal");
            if (!d->lit.is_null) {
              // [EXT] DataFusion casts the default to the argument's type; a value the type cannot hold exactly is refused
              we.default_value = window_default_as(d, we.args[0]->type);
              if (!we.default_value)
                throw PlanUnsupported("the default of " + who + " has type " + d->type.str() + " and does not cast exactly to the argument's " + we.args[0]->type.str());
            }
          }
          we.args.resize(1);
          we.result_type = we.args[0]->type;
          break;
        }
        case WinFn::FirstValue:
        case WinFn::LastValue:
          want_args(1, 1);
          we.result_type = we.args[0]->type;
          break;
        case WinFn::NthValue:
          want_args(2, 2);
          we.n = int_literal(1, "the position");
          if (we.n < 1) throw std::runtime_error("nth_value of " + who + " needs n >= 1, got " + std::to_string(we.n));
          we.n = std::min<int64_t>(we.n, kWindowMaxOffset);  // past any frame (< 2^32 rows): NULL, and no overflow in fs + n
          we.args.resize(1);
          we.result_type = we.args[0]->type;
          break;
        case WinFn::Count:
          want_args(0, 1);
          if (!we.args.empty() && we.args[0]->kind == Expr::Lit && !we.args[0]->lit.is_null) we.args.clear();  // COUNT(<literal>) is COUNT(*)
          we.result_type = DataType(TypeId::Int64);
          we.nullable = false;
          break;
        default: {  // Sum, Avg, Min, Max
          want_args(1, 1);
          const DataType& t = we.args[0]->type;
          const bool ok = we.fn == WinFn::Sum || we.fn == WinFn::Avg
                              ? t.is_numeric()
                              : (t.is_numeric() || t.id == TypeId::Date32 || t.id == TypeId::Timestamp || t.id == TypeId::Bool);
          if (!ok) throw PlanUnsupported("window function " + who + " does not support an argument of type " + t.str());
          we.result_type = we.fn == WinFn::Sum ? sum_result_type(t) : we.fn == WinFn::Avg ? avg_result_type(t) : t;
        }
      }
      n->schema.push_back(Field{we.name, we.result_type, we.nullable});
      n->window_exprs.push_back(we);
    }
  } else if (op == "GlobalLimitExec" || op == "LocalLimitExec") {
    n->op = PlanNode::Limit;
    PlanNode* c = parse_child("input");
    n->schema = c->schema;
    n->fetch = j.get_int("fetch", -1);
    n->skip = j.get_int("skip", 0);
  } else if (op == "ShuffleWriterExec" || op == "SortShuffleWriterExec") {
    n->op = PlanNode::ShuffleWriter;
    PlanNode* c = parse_child("input");
    n->schema = c->schema;
    n->job_id = j.get_str("job_id", "job");
    n->stage_id = j.get_int("stage_id", 0);
    n->sort_shuffle = (op == "SortShuffleWriterExec") || j.get_bool("sort_shuffle", false);
    if (j.has("partitioning")) {
      const Json& p = j.at("partitioning");
      const Json& hs = p.at("hash");
      for (size_t i = 0; i < hs.size(); i++) n->part_exprs.push_back(parse_expr(hs.at(i), c->schema));
      n->n_out_partitions = p.at("n").as_int();
      if (n->n_out_partitions <= 0) throw std::runtime_error("shuffle writer: partition count must be positive");
    }
  } else {
    throw std::runtime_error("plan IR: unknown operator '" + op + "'");
  }
  return n;
}

}  // namespace b200
