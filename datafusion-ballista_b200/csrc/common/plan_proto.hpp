// Decoder for the plan bytes a Ballista task carries: `TaskDefinition.plan` / `MultiTaskDefinition.plan`
// (ballista/core/proto/ballista.proto:518-529,551-560) = a protobuf-encoded datafusion.PhysicalPlanNode
// (ballista/core/proto/datafusion.proto:716-757) whose Ballista-specific nodes travel as PhysicalExtensionNode
// { node = BallistaPhysicalPlanNode bytes, inputs = [child] } (ballista/core/src/serde/mod.rs:481-640, `input: None`).
//
// Output: the stage-plan IR of plan.hpp as JSON text, i.e. exactly what b200_stage_prepare consumes -- so an executor can
// hand the scheduler's bytes to the engine as they arrive (b200_stage_prepare_proto) and the Rust side does not walk the
// plan at all.  Hand-written wire-format reader (varint / 64-bit / length-delimited / 32-bit; unknown fields skipped), no
// protobuf library: the library has no dependencies beyond CUDA.  Field numbers are the reference's, cited per message.
//
// Two constructs carry information the IR used to leave to the shim and are now resolved by plan.hpp itself:
//   * Final / FinalPartitioned aggregates: the proto gives the ORIGINAL argument expressions plus `input_schema` (the partial
//     stage's input, AggregateExecNode.input_schema = 7); the IR's "input_type" is typed from them ("input_schema" key);
//   * join filters: JoinFilter.expression indexes an intermediate schema described by column_indices (side, index); the IR's
//     filter indexes left ++ right, so the decoder emits "filter_columns" and plan.hpp remaps.
// Scans: ParquetScanExecNode -> DataSourceExec on the table named after the files' directory (or file stem); the file
// groups are passed through ("file_groups") for the host side to register (b200_engine_register_parquet).
// CsvScanExecNode -> the same, plus "format": "csv", the reader options ("csv") and, when any file carries a byte range,
// "file_ranges" shaped like "file_groups" ([start, end] or null), for b200_engine_register_csv.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

namespace b200 {
namespace pbp {

struct Slice {
  const uint8_t* p = nullptr;
  size_t n = 0;
};

struct Entry {
  uint32_t field;
  uint32_t wire;   // 0 varint, 1 fixed64, 2 bytes, 5 fixed32
  uint64_t v;      // varint / fixed value
  Slice b;         // wire 2
};

// protobuf `string` fields are UTF-8 by contract; bytes off the network are checked before they end up in JSON text
inline void require_utf8(const uint8_t* p, size_t n) {
  size_t i = 0;
  while (i < n) {
    const uint8_t c = p[i];
    size_t len = c < 0x80 ? 1 : (c >> 5) == 0x6 ? 2 : (c >> 4) == 0xe ? 3 : (c >> 3) == 0x1e ? 4 : 0;
    if (len == 0 || i + len > n) throw std::runtime_error("plan proto: string field is not valid UTF-8");
    for (size_t k = 1; k < len; k++)
      if ((p[i + k] & 0xc0) != 0x80) throw std::runtime_error("plan proto: string field is not valid UTF-8");
    if (len == 2 && c < 0xc2) throw std::runtime_error("plan proto: string field is not valid UTF-8");                       // overlong
    if (len == 3 && c == 0xe0 && p[i + 1] < 0xa0) throw std::runtime_error("plan proto: string field is not valid UTF-8");   // overlong
    if (len == 3 && c == 0xed && p[i + 1] >= 0xa0) throw std::runtime_error("plan proto: string field is not valid UTF-8");  // surrogates
    if (len == 4 && (c > 0xf4 || (c == 0xf0 && p[i + 1] < 0x90) || (c == 0xf4 && p[i + 1] >= 0x90)))
      throw std::runtime_error("plan proto: string field is not valid UTF-8");
    i += len;
  }
}

struct Msg {
  std::vector<Entry> e;
  Msg() {}
  explicit Msg(Slice s) { parse(s); }
  static uint64_t varint(const uint8_t*& p, const uint8_t* end) {
    uint64_t v = 0;
    int shift = 0;
    while (true) {
      if (p >= end) throw std::runtime_error("plan proto: truncated varint");
      const uint8_t c = *p++;
      if (shift < 64) v |= (uint64_t)(c & 0x7f) << shift;
      if (!(c & 0x80)) break;
      shift += 7;
      if (shift > 70) throw std::runtime_error("plan proto: varint too long");
    }
    return v;
  }
  void parse(Slice s) {
    const uint8_t* p = s.p;
    const uint8_t* end = s.p + s.n;
    while (p < end) {
      const uint64_t key = varint(p, end);
      Entry en;
      en.field = (uint32_t)(key >> 3);
      en.wire = (uint32_t)(key & 7);
      en.v = 0;
      if (en.field == 0) throw std::runtime_error("plan proto: field number 0");
      switch (en.wire) {
        case 0: en.v = varint(p, end); break;
        case 1:
          if (end - p < 8) throw std::runtime_error("plan proto: truncated fixed64");
          memcpy(&en.v, p, 8);
          p += 8;
          break;
        case 2: {
          const uint64_t len = varint(p, end);
          if (len > (uint64_t)(end - p)) throw std::runtime_error("plan proto: truncated length-delimited field");
          en.b.p = p;
          en.b.n = (size_t)len;
          p += len;
          break;
        }
        case 5: {
          if (end - p < 4) throw std::runtime_error("plan proto: truncated fixed32");
          uint32_t t;
          memcpy(&t, p, 4);
          en.v = t;
          p += 4;
          break;
        }
        default: throw std::runtime_error("plan proto: unsupported wire type " + std::to_string(en.wire));
      }
      e.push_back(en);
    }
  }
  const Entry* last(uint32_t f) const {  // protobuf: the last occurrence of a singular field wins
    const Entry* r = nullptr;
    for (auto& x : e)
      if (x.field == f) r = &x;
    return r;
  }
  bool has(uint32_t f) const { return last(f) != nullptr; }
  uint64_t u64(uint32_t f, uint64_t dflt = 0) const {
    const Entry* x = last(f);
    return x ? x->v : dflt;
  }
  int64_t i64(uint32_t f, int64_t dflt = 0) const { return (int64_t)u64(f, (uint64_t)dflt); }
  bool boolean(uint32_t f) const { return u64(f) != 0; }
  std::string str(uint32_t f) const {
    const Entry* x = last(f);
    if (!x) return std::string();
    require_utf8(x->b.p, x->b.n);
    return std::string((const char*)x->b.p, x->b.n);
  }
  Slice bytes(uint32_t f) const {
    const Entry* x = last(f);
    return x ? x->b : Slice();
  }
  Msg sub(uint32_t f) const { return Msg(bytes(f)); }
  std::vector<Msg> subs(uint32_t f) const {
    std::vector<Msg> r;
    for (auto& x : e)
      if (x.field == f && x.wire == 2) r.push_back(Msg(x.b));
    return r;
  }
  std::vector<std::string> strs(uint32_t f) const {
    std::vector<std::string> r;
    for (auto& x : e)
      if (x.field == f && x.wire == 2) {
        require_utf8(x.b.p, x.b.n);
        r.push_back(std::string((const char*)x.b.p, x.b.n));
      }
    return r;
  }
  // repeated scalar: packed (wire 2) or one entry per element
  std::vector<uint64_t> varints(uint32_t f) const {
    std::vector<uint64_t> r;
    for (auto& x : e) {
      if (x.field != f) continue;
      if (x.wire == 0) r.push_back(x.v);
      else if (x.wire == 2) {
        const uint8_t* p = x.b.p;
        const uint8_t* end = p + x.b.n;
        while (p < end) r.push_back(varint(p, end));
      }
    }
    return r;
  }
  // the one populated member of a oneof: the LAST entry whose field number is in [lo, hi] \ {skip}
  const Entry* oneof(std::initializer_list<uint32_t> members) const {
    const Entry* r = nullptr;
    for (auto& x : e)
      for (uint32_t m : members)
        if (x.field == m) r = &x;
    return r;
  }
};

inline std::string jstr(const std::string& s) {
  std::string o = "\"";
  for (unsigned char c : s) {
    switch (c) {
      case '"': o += "\\\""; break;
      case '\\': o += "\\\\"; break;
      case '\n': o += "\\n"; break;
      case '\r': o += "\\r"; break;
      case '\t': o += "\\t"; break;
      default:
        if (c < 0x20) {
          char b[8];
          snprintf(b, sizeof b, "\\u%04x", c);
          o += b;
        } else {
          o += (char)c;
        }
    }
  }
  return o + "\"";
}

inline std::string i128_to_string(__int128 v) {
  if (v == 0) return "0";
  const bool neg = v < 0;
  unsigned __int128 u = neg ? (unsigned __int128)(-(v + 1)) + 1 : (unsigned __int128)v;
  std::string s;
  while (u) {
    s.insert(s.begin(), (char)('0' + (int)(u % 10)));
    u /= 10;
  }
  return neg ? "-" + s : s;
}

struct Unsupported : std::runtime_error {
  explicit Unsupported(const std::string& m) : std::runtime_error(m) {}
};

// plan bytes come off the network: bound the recursion (a legitimate plan nests a few dozen levels)
struct DepthGuard {
  static int& depth() {
    static thread_local int d = 0;
    return d;
  }
  DepthGuard() {
    if (++depth() > 512) {
      --depth();
      throw std::runtime_error("plan proto: nesting deeper than 512 levels");
    }
  }
  ~DepthGuard() { --depth(); }
};

// ---- datafusion_common.ArrowType (datafusion_common.proto:365-410) ---------------------------------------------------------
inline std::string type_json(const Msg& t) {
  const Entry* x = t.oneof({1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 36, 40, 41, 42});
  if (!x) throw std::runtime_error("plan proto: ArrowType without a variant");
  switch (x->field) {
    case 1: return "\"null\"";
    case 2: return "\"bool\"";
    case 3: return "\"u8\"";
    case 4: return "\"i8\"";
    case 5: return "\"u16\"";
    case 6: return "\"i16\"";
    case 7: return "\"u32\"";
    case 8: return "\"i32\"";
    case 9: return "\"u64\"";
    case 10: return "\"i64\"";
    case 12: return "\"f32\"";
    case 13: return "\"f64\"";
    case 14:   // UTF8
    case 35:   // UTF8_VIEW: Ballista runs with Utf8 (extension.rs:655-661); a view column carries the same values
      return "\"utf8\"";
    case 17: return "\"date32\"";
    case 20: return "\"ts\"";
    case 24: {  // Decimal128Type { precision = 3, scale = 4 } (datafusion_common.proto:151-155)
      const Msg d(x->b);
      return "{\"dec\":[" + std::to_string(d.u64(3)) + "," + std::to_string((int32_t)d.u64(4)) + "]}";
    }
    default: throw Unsupported("Arrow type variant " + std::to_string(x->field) + " is not supported by the device engine");
  }
}

// datafusion_common.Schema { columns = 1 } / Field { name = 1, arrow_type = 2, nullable = 3 } (datafusion_common.proto:106-119)
inline std::string schema_json(const Msg& s) {
  std::string o = "[";
  bool first = true;
  for (auto& f : s.subs(1)) {
    if (!first) o += ",";
    first = false;
    o += "{\"name\":" + jstr(f.str(1)) + ",\"type\":" + type_json(f.sub(2)) + ",\"nullable\":" + (f.boolean(3) ? "true" : "false") + "}";
  }
  return o + "]";
}

// ---- datafusion_common.ScalarValue (datafusion_common.proto:280-338) -------------------------------------------------------
inline std::string literal_json(const Msg& v) {
  const Entry* x = v.oneof({33, 1, 2, 3, 23, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 20, 21, 26});
  if (!x) throw Unsupported("literal: scalar value variant not supported");
  auto lit = [](const std::string& t, const std::string& val) { return "{\"lit\":{\"t\":" + t + ",\"v\":" + val + "}}"; };
  switch (x->field) {
    case 33: return lit(type_json(Msg(x->b)), "null");
    case 1: return lit("\"bool\"", x->v ? "true" : "false");
    case 2:
    case 23:
      require_utf8(x->b.p, x->b.n);
      return lit("\"utf8\"", jstr(std::string((const char*)x->b.p, x->b.n)));
    case 4: return lit("\"i8\"", std::to_string((int32_t)x->v));
    case 5: return lit("\"i16\"", std::to_string((int32_t)x->v));
    case 6: return lit("\"i32\"", std::to_string((int32_t)x->v));
    case 7: return lit("\"i64\"", std::to_string((int64_t)x->v));
    case 8: return lit("\"u8\"", std::to_string((uint32_t)x->v));
    case 9: return lit("\"u16\"", std::to_string((uint32_t)x->v));
    case 10: return lit("\"u32\"", std::to_string((uint32_t)x->v));
    case 11: return lit("\"u64\"", std::to_string((uint64_t)x->v));
    case 12: {
      float f;
      const uint32_t b = (uint32_t)x->v;
      memcpy(&f, &b, 4);
      char buf[64];
      snprintf(buf, sizeof buf, "%.9g", (double)f);
      return lit("\"f32\"", buf);
    }
    case 13: {
      double d;
      memcpy(&d, &x->v, 8);
      char buf[64];
      snprintf(buf, sizeof buf, "%.17g", d);
      return lit("\"f64\"", buf);
    }
    case 14: return lit("\"date32\"", std::to_string((int32_t)x->v));
    case 20: {  // Decimal128 { value = 1 (i128, big-endian two's complement), p = 2, s = 3 } (datafusion_common.proto:352-356)
      const Msg d(x->b);
      const Slice b = d.bytes(1);
      const std::string dt = "{\"dec\":[" + std::to_string(d.i64(2)) + "," + std::to_string(d.i64(3)) + "]}";
      if (b.n == 0) return lit(dt, "null");  // no value bytes: a NULL of that decimal type
      if (b.n > 16) throw std::runtime_error("plan proto: Decimal128 literal with more than 16 value bytes");
      __int128 val = (b.p[0] & 0x80) ? -1 : 0;
      for (size_t i = 0; i < b.n; i++) val = (__int128)(((unsigned __int128)val << 8) | b.p[i]);
      return lit(dt, "\"" + i128_to_string(val) + "\"");
    }
    default: throw Unsupported("literal: scalar value variant " + std::to_string(x->field) + " not supported");
  }
}

// ---- datafusion.PhysicalExprNode (datafusion.proto:851-901) -----------------------------------------------------------------
inline std::string binop_symbol(const std::string& op) {
  // BinaryExpr.op is the Debug name of datafusion_expr::Operator [EXT, datafusion-proto to_proto]
  static const std::pair<const char*, const char*> tab[] = {
      {"Eq", "="},     {"NotEq", "!="},   {"Lt", "<"},       {"LtEq", "<="},  {"Gt", ">"},   {"GtEq", ">="}, {"Plus", "+"},
      {"Minus", "-"},  {"Multiply", "*"}, {"Divide", "/"},   {"Modulo", "%"}, {"And", "and"}, {"Or", "or"},
      {"BitwiseAnd", "&"}, {"BitwiseOr", "|"}, {"BitwiseXor", "^"}, {"BitwiseShiftLeft", "<<"}, {"BitwiseShiftRight", ">>"},
      {"RegexMatch", "~"}, {"RegexIMatch", "~*"}, {"RegexNotMatch", "!~"}, {"RegexNotIMatch", "!~*"},
      {"StringConcat", "||"}};
  for (auto& kv : tab)
    if (op == kv.first) return kv.second;
  throw Unsupported("binary operator " + op + " is not supported by the device engine");
}

inline std::string expr_json(const Msg& e);

inline std::string exprs_json(const std::vector<Msg>& v) {
  std::string o = "[";
  for (size_t i = 0; i < v.size(); i++) o += (i ? "," : "") + expr_json(v[i]);
  return o + "]";
}

inline bool literal_utf8(const Msg& e, std::string& out) {
  const Entry* x = e.oneof({1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 14, 15, 16, 18, 19, 20, 21});
  if (!x || x->field != 2) return false;
  const Msg v(x->b);
  const Entry* s = v.oneof({2, 3, 23});
  if (!s) return false;
  require_utf8(s->b.p, s->b.n);
  out.assign((const char*)s->b.p, s->b.n);
  return true;
}

inline std::string expr_json(const Msg& e) {
  DepthGuard dg;
  const Entry* x = e.oneof({1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 14, 15, 16, 18, 19, 20, 21});
  if (!x) throw std::runtime_error("plan proto: PhysicalExprNode without ExprType");
  const Msg m(x->b);
  switch (x->field) {
    case 1: return "{\"col\":" + std::to_string(m.u64(2)) + "}";  // PhysicalColumn { name = 1, index = 2 } (:1189-1192)
    case 2: return literal_json(m);
    case 3:  // PhysicalBinaryExprNode { l = 1, r = 2, op = 3 } (:957-961)
      return "{\"bin\":" + jstr(binop_symbol(m.str(3))) + ",\"l\":" + expr_json(m.sub(1)) + ",\"r\":" + expr_json(m.sub(2)) + "}";
    case 5: return "{\"is_null\":" + expr_json(m.sub(1)) + "}";
    case 6: return "{\"is_not_null\":" + expr_json(m.sub(1)) + "}";
    case 7: return "{\"not\":" + expr_json(m.sub(1)) + "}";
    case 8: {  // PhysicalCaseNode { expr = 1, when_then_expr = 2 { when = 1, then = 2 }, else_expr = 3 } (:982-997)
      const bool simple = m.has(1);  // CASE x WHEN v ...  ==  CASE WHEN x = v ...
      std::string o = "{\"case\":{\"when\":[";
      bool first = true;
      for (auto& wt : m.subs(2)) {
        if (!first) o += ",";
        first = false;
        std::string w = expr_json(wt.sub(1));
        if (simple) w = "{\"bin\":\"=\",\"l\":" + expr_json(m.sub(1)) + ",\"r\":" + w + "}";
        o += "[" + w + "," + expr_json(wt.sub(2)) + "]";
      }
      o += "]";
      if (m.has(3)) o += ",\"else\":" + expr_json(m.sub(3));
      return o + "}}";
    }
    case 9:    // PhysicalCastNode { expr = 1, arrow_type = 2 } (:1004-1007)
    case 14:   // PhysicalTryCastNode (:999-1002)
      return "{\"cast\":" + expr_json(m.sub(1)) + ",\"to\":" + type_json(m.sub(2)) + "}";
    case 11: return "{\"neg\":" + expr_json(m.sub(1)) + "}";
    case 12:  // PhysicalInListNode { expr = 1, list = 2, negated = 3 } (:987-991)
      return "{\"in\":" + expr_json(m.sub(1)) + ",\"list\":" + exprs_json(m.subs(2)) + ",\"negated\":" + (m.boolean(3) ? "true" : "false") + "}";
    case 16: {  // PhysicalScalarUdfNode { name = 1, args = 2, return_type = 4 } (:903-910)
      std::string name = m.str(1);
      std::vector<Msg> args = m.subs(2);
      for (auto& ch : name) ch = (char)tolower((unsigned char)ch);
      if (name == "date_part" || name == "datepart") {
        std::string part;
        if (args.size() != 2 || !literal_utf8(args[0], part)) throw Unsupported("date_part with a non-literal part");
        for (auto& ch : part) ch = (char)tolower((unsigned char)ch);
        static const char* const parts[] = {"year", "quarter", "month", "week", "day", "doy", "dow"};
        bool known = false;
        for (const char* p : parts) known = known || part == p;
        if (!known) throw Unsupported("date_part('" + part + "', ..) is not supported by the device engine");
        return "{\"fn\":\"date_part_" + part + "\",\"args\":[" + expr_json(args[1]) + "]}";
      }
      if (name == "substr" || name == "substring") return "{\"fn\":\"substr\",\"args\":" + exprs_json(args) + "}";
      // the scalar functions of DESIGN §3, under the names the function registry resolves
      static const std::pair<const char*, const char*> fns[] = {
          {"abs", "abs"},         {"round", "round"},       {"floor", "floor"},
          {"ceil", "ceil"},       {"nullif", "nullif"},     {"coalesce", "coalesce"},
          {"character_length", "character_length"},         {"char_length", "character_length"},
          {"length", "character_length"},                   {"octet_length", "octet_length"},
          {"starts_with", "starts_with"},                   {"ends_with", "ends_with"},
          {"btrim", "btrim"},     {"trim", "btrim"},        {"ltrim", "ltrim"},
          {"rtrim", "rtrim"},     {"regexp_like", "regexp_like"},
          {"concat", "concat"},   {"concat_ws", "concat_ws"}, {"repeat", "repeat"},
          {"reverse", "reverse"}};
      for (auto& kv : fns)
        if (name == kv.first) return "{\"fn\":\"" + std::string(kv.second) + "\",\"args\":" + exprs_json(args) + "}";
      throw Unsupported("scalar function " + name + " is not supported by the device engine");
    }
    case 18: {  // PhysicalLikeExprNode { negated = 1, case_insensitive = 2, expr = 3, pattern = 4 } (:969-974)
      std::string pat;
      if (!literal_utf8(m.sub(4), pat)) throw Unsupported(std::string(m.boolean(2) ? "ILIKE" : "LIKE") + " with a non-literal pattern");
      return "{\"like\":" + expr_json(m.sub(3)) + ",\"pattern\":" + jstr(pat) + ",\"negated\":" + (m.boolean(1) ? "true" : "false") +
             (m.boolean(2) ? ",\"case_insensitive\":true" : "") + "}";
    }
    default: throw Unsupported("physical expression variant " + std::to_string(x->field) + " is not supported by the device engine");
  }
}

// PhysicalSortExprNode { expr = 1, asc = 2, nulls_first = 3 } (:976-980)
inline std::string sort_expr_json(const Msg& s) {
  return "{\"expr\":" + expr_json(s.sub(1)) + ",\"asc\":" + (s.boolean(2) ? "true" : "false") + ",\"nulls_first\":" + (s.boolean(3) ? "true" : "false") + "}";
}
// ... wrapped in PhysicalExprNode.sort = 10 (SortExec, SortPreservingMergeExec)
inline std::string sort_exprs_json(const std::vector<Msg>& v) {
  std::string o = "[";
  for (size_t i = 0; i < v.size(); i++) {
    const Entry* x = v[i].last(10);
    if (!x) throw std::runtime_error("plan proto: sort expression expected");
    o += std::string(i ? "," : "") + sort_expr_json(Msg(x->b));
  }
  return o + "]";
}

// WindowFrameBound { window_frame_bound_type = 1 (CURRENT_ROW 0, PRECEDING 1, FOLLOWING 2), bound_value = 2 } (:627-635).
// [EXT] datafusion-proto writes UNBOUNDED as a NULL bound value (ScalarValue.null_value = 33); an absent value means the same.
// An integer value becomes "n"; any other value (an interval, a float) becomes "n": null, which the typing refuses.
inline std::string window_bound_json(const Msg& b) {
  const uint64_t t = b.u64(1);
  if (t == 0) return "{\"kind\":\"current_row\"}";
  if (t > 2) throw std::runtime_error("plan proto: window frame bound type " + std::to_string(t));
  const char* side = t == 1 ? "preceding" : "following";
  const Msg v = b.sub(2);
  const Entry* x = v.e.empty() ? nullptr : &v.e.back();
  if (!x || x->field == 33) return std::string("{\"kind\":\"unbounded_") + side + "\"}";
  std::string n = "null";
  if (x->field >= 4 && x->field <= 7) n = std::to_string((int64_t)x->v);        // int8 .. int64 values
  else if (x->field >= 8 && x->field <= 11) n = std::to_string((uint64_t)x->v);  // uint8 .. uint64 values
  return std::string("{\"kind\":\"") + side + "\",\"n\":" + n + "}";
}
// WindowFrame { window_frame_units = 1 (ROWS 0, RANGE 1, GROUPS 2), start_bound = 2, bound = 3 (the end) } (:610-625)
inline std::string window_frame_json(const Msg& f) {
  static const char* units[] = {"rows", "range", "groups"};
  const uint64_t u = f.u64(1);
  if (u > 2) throw std::runtime_error("plan proto: window frame units " + std::to_string(u));
  return std::string("{\"units\":\"") + units[u] + "\",\"start\":" + window_bound_json(f.sub(2)) + ",\"end\":" + window_bound_json(f.sub(3)) + "}";
}

inline std::string u32_list_json(const std::vector<uint64_t>& v) {
  std::string o = "[";
  for (size_t i = 0; i < v.size(); i++) o += (i ? "," : "") + std::to_string(v[i]);
  return o + "]";
}

inline const char* join_type_name(uint64_t v) {  // datafusion_common.JoinType (datafusion_common.proto:80-91)
  switch (v) {
    case 0: return "Inner";
    case 1: return "Left";
    case 2: return "Right";
    case 3: return "Full";
    case 4: return "LeftSemi";
    case 5: return "LeftAnti";
    case 6: return "RightSemi";
    case 7: return "RightAnti";
    default: throw Unsupported("mark joins are not supported by the device engine");
  }
}

inline std::string table_of_path(const std::string& path) {
  // ".../lineitem/part-0.parquet" -> lineitem ; ".../lineitem.parquet" -> lineitem
  auto base = [](const std::string& p) {
    size_t e = p.size();
    while (e > 0 && p[e - 1] == '/') e--;
    size_t b = p.rfind('/', e ? e - 1 : 0);
    b = (b == std::string::npos) ? 0 : b + 1;
    return p.substr(b, e - b);
  };
  auto stem = [](std::string s) {
    size_t d = s.find('.');
    if (d != std::string::npos && d > 0) s = s.substr(0, d);
    return s;
  };
  const std::string file = base(path);
  const size_t slash = path.rfind('/');
  if ((file.rfind("part-", 0) == 0 || file.rfind("part.", 0) == 0 || file.rfind("partition", 0) == 0) && slash != std::string::npos && slash > 0)
    return stem(base(path.substr(0, slash)));
  return stem(file);
}

inline std::string plan_json(const Msg& n, const std::string& override_job = std::string());

// JoinOn { left = 1, right = 2 } (:1198-1201); JoinFilter { expression = 1, column_indices = 2 { index = 1, side = 2 }, schema = 3 } (:1343-1352)
// f_on = 0: the node has no equality keys (NestedLoopJoinExecNode) and no "on" key is written
inline std::string join_common_json(const Msg& m, uint32_t f_on, uint32_t f_type, uint32_t f_filter) {
  std::string o;
  if (f_on) {
    o = ",\"on\":[";
    bool first = true;
    for (auto& on : m.subs(f_on)) {
      if (!first) o += ",";
      first = false;
      o += "[" + expr_json(on.sub(1)) + "," + expr_json(on.sub(2)) + "]";
    }
    o += "]";
  }
  o += std::string(",\"join_type\":\"") + join_type_name(m.u64(f_type)) + "\"";
  if (m.has(f_filter)) {
    const Msg f = m.sub(f_filter);
    if (f.has(1)) {
      o += ",\"filter\":" + expr_json(f.sub(1)) + ",\"filter_columns\":[";
      bool ff = true;
      for (auto& ci : f.subs(2)) {
        if (!ff) o += ",";
        ff = false;
        const uint64_t side = ci.u64(2);  // JoinSide: LEFT_SIDE = 0, RIGHT_SIDE = 1 (datafusion_common.proto:608-612)
        if (side > 1) throw Unsupported("join filter column without a side");
        o += "[" + std::to_string(side) + "," + std::to_string(ci.u64(1)) + "]";
      }
      o += "]";
    }
  }
  return o;
}

// NullEquality { NULL_EQUALS_NOTHING = 0, NULL_EQUALS_NULL = 1 } (datafusion_common.proto:98-101): with NULL_EQUALS_NULL a
// NULL join key matches a NULL key (INTERSECT / EXCEPT, IS NOT DISTINCT FROM keys)
inline std::string null_equality_json(const Msg& m, uint32_t f) {
  const uint64_t v = m.u64(f);
  if (v > 1) throw Unsupported("join null equality " + std::to_string(v));
  return v == 1 ? ",\"null_equals_null\":true" : "";
}

inline std::string plan_json(const Msg& n, const std::string& override_job) {
  DepthGuard dg;
  const Entry* x = n.oneof({1, 2, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 36, 37, 38});
  if (!x) throw std::runtime_error("plan proto: PhysicalPlanNode without PhysicalPlanType");
  const Msg m(x->b);
  auto in = [&](uint32_t f) { return plan_json(m.sub(f)); };
  switch (x->field) {
    case 1:    // ParquetScanExecNode { base_conf = 1 } (:1058-1077)
    case 2: {  // CsvScanExecNode { base_conf = 1, has_header = 2, delimiter = 3, quote = 4, escape = 5, comment = 6,
               //                   newlines_in_values = 7, truncate_rows = 8 } (:1088-1101)
      // FileScanExecConf { file_groups = 1, schema = 2, projection = 4 } (:1058-1086)
      const bool csv = x->field == 2;
      if (csv && m.has(6)) throw Unsupported("CsvScanExecNode option 'comment' is not supported by the device engine");
      if (csv && m.u64(8)) throw Unsupported("CsvScanExecNode option 'truncate_rows' is not supported by the device engine");
      const Msg conf = m.sub(1);
      std::string table, groups = "[", ranges = "[";
      bool fg = true, any_range = false;
      for (auto& g : conf.subs(1)) {
        if (!fg) {
          groups += ",";
          ranges += ",";
        }
        fg = false;
        groups += "[";
        ranges += "[";
        bool ff = true;
        for (auto& f : g.subs(1)) {  // PartitionedFile { path = 1, range = 5 } (:1354-1361)
          const std::string path = f.str(1);
          if (table.empty()) table = table_of_path(path);
          groups += std::string(ff ? "" : ",") + jstr(path);
          ranges += ff ? "" : ",";
          ff = false;
          if (f.has(5)) {  // FileRange { start = 1, end = 2 } (:1363-1366)
            const Msg r = f.sub(5);
            const int64_t a = r.i64(1), b = r.i64(2);
            if (a < 0 || b < a) throw std::runtime_error("plan proto: file range with end before start");
            ranges += "[" + std::to_string(a) + "," + std::to_string(b) + "]";
            any_range = true;
          } else {
            ranges += "null";
          }
        }
        groups += "]";
        ranges += "]";
      }
      groups += "]";
      ranges += "]";
      if (table.empty()) throw std::runtime_error(csv ? "plan proto: csv scan without files" : "plan proto: parquet scan without files");
      std::string o = "{\"op\":\"DataSourceExec\",\"table\":" + jstr(table) + ",\"schema\":" + schema_json(conf.sub(2));
      std::vector<uint64_t> proj = conf.varints(4);
      if (proj.empty() && conf.has(13)) {
        // newer encoders: projection_exprs = 13 { projections = 1 { alias = 1, expr = 2 } } (:1049-1056,1075): plain column
        // selections are a projection; computed expressions would be a ProjectionExec the planner has not split off
        for (auto& pe : conf.sub(13).subs(1)) {
          const Entry* cx = pe.sub(2).last(1);
          if (!cx) throw Unsupported("scan projection with computed expressions is not supported by the device engine");
          proj.push_back(Msg(cx->b).u64(2));
        }
      }
      if (!proj.empty()) o += ",\"projection\":" + u32_list_json(proj);
      o += ",\"file_groups\":" + groups;
      if (!csv) return o + "}";
      // reader options as b200_engine_register_csv takes them: one ASCII byte each (escape may be absent)
      auto opt = [&](uint32_t f, const char* name) {
        const std::string v = m.str(f);
        if (v.size() != 1 || (unsigned char)v[0] >= 0x80)
          throw std::runtime_error(std::string("plan proto: CsvScanExecNode option '") + name + "' must be one ASCII byte");
        return jstr(v);
      };
      o += ",\"format\":\"csv\",\"csv\":{\"has_header\":" + std::string(m.u64(2) ? "true" : "false") + ",\"delimiter\":" + opt(3, "delimiter") +
           ",\"quote\":" + opt(4, "quote") + ",\"escape\":" + (m.has(5) ? opt(5, "escape") : std::string("null")) +
           ",\"newlines_in_values\":" + (m.u64(7) ? "true" : "false") + "}";
      if (any_range) o += ",\"file_ranges\":" + ranges;
      return o + "}";
    }
    case 4: {  // ProjectionExecNode { input = 1, expr = 2, expr_name = 3 } (:1211-1215)
      const std::vector<Msg> es = m.subs(2);
      const std::vector<std::string> names = m.strs(3);
      if (names.size() != es.size()) throw std::runtime_error("plan proto: projection names do not match its expressions");
      std::string o = "{\"op\":\"ProjectionExec\",\"exprs\":[";
      for (size_t i = 0; i < es.size(); i++) o += std::string(i ? "," : "") + "{\"expr\":" + expr_json(es[i]) + ",\"name\":" + jstr(names[i]) + "}";
      return o + "],\"input\":" + in(1) + "}";
    }
    case 6: {  // GlobalLimitExecNode { input = 1, skip = 2, fetch = 3 (negative: none) } (:1273-1279)
      std::string o = "{\"op\":\"GlobalLimitExec\",\"input\":" + in(1) + ",\"skip\":" + std::to_string(m.u64(2));
      if (m.i64(3, -1) >= 0) o += ",\"fetch\":" + std::to_string(m.i64(3));
      return o + "}";
    }
    case 7:  // LocalLimitExecNode { input = 1, fetch = 2 } (:1281-1284)
      return "{\"op\":\"LocalLimitExec\",\"input\":" + in(1) + ",\"skip\":0,\"fetch\":" + std::to_string(m.u64(2)) + "}";
    case 8: {  // AggregateExecNode (:1257-1271)
      static const char* modes[] = {"Partial", "Final", "FinalPartitioned", "Single", "SinglePartitioned"};
      const uint64_t mode = m.u64(3);
      if (mode > 4) throw Unsupported("aggregate mode PartialReduce is not supported by the device engine");
      for (auto& f : m.subs(10))
        if (f.has(1)) throw Unsupported("aggregate FILTER clauses are not supported by the device engine");
      const std::vector<Msg> gs = m.subs(1), as = m.subs(2);
      const std::vector<std::string> gn = m.strs(5), an = m.strs(6);
      if (gn.size() != gs.size() || an.size() != as.size()) throw std::runtime_error("plan proto: aggregate names do not match its expressions");
      std::string o = std::string("{\"op\":\"AggregateExec\",\"mode\":\"") + modes[mode] + "\",\"group_by\":[";
      for (size_t i = 0; i < gs.size(); i++) o += std::string(i ? "," : "") + "{\"expr\":" + expr_json(gs[i]) + ",\"name\":" + jstr(gn[i]) + "}";
      // grouping sets: groups = 9 (S x n bools, row-major; true = the key is NULL in that set), null_expr = 8 (n NULL
      // literals), has_grouping_set = 12.  A node is a grouping-set node iff has_grouping_set is set or some entry of
      // groups is true [EXT]: a plain GROUP BY carries one all-false set and decodes as before, whatever null_expr holds.
      const std::vector<uint64_t> groups = m.varints(9);
      bool gsets = m.boolean(12);
      for (uint64_t g : groups) gsets = gsets || g != 0;
      if (gsets) {
        const size_t nk = gs.size();
        if (groups.empty() || nk == 0 || groups.size() % nk != 0)
          throw std::runtime_error("plan proto: " + std::to_string(groups.size()) + " grouping-set entries for " + std::to_string(nk) + " group keys");
        const std::vector<Msg> nulls = m.subs(8);
        if (nulls.size() != nk) throw std::runtime_error("plan proto: " + std::to_string(nulls.size()) + " null_expr for " + std::to_string(nk) + " group keys");
        static const std::string lit_head = "{\"lit\":", null_tail = ",\"v\":null}}";
        for (auto& ne : nulls) {
          const std::string lj = expr_json(ne);
          if (lj.compare(0, lit_head.size(), lit_head) != 0 || lj.size() < null_tail.size() ||
              lj.compare(lj.size() - null_tail.size(), null_tail.size(), null_tail) != 0)
            throw std::runtime_error("plan proto: a grouping-set null_expr is not a NULL literal");
        }
        o += "],\"grouping_sets\":[";
        for (size_t s = 0; s < groups.size() / nk; s++) {
          o += s ? ",[" : "[";
          for (size_t k = 0; k < nk; k++) o += std::string(k ? "," : "") + (groups[s * nk + k] ? "true" : "false");
          o += "]";
        }
      }
      o += "],\"aggr\":[";
      for (size_t i = 0; i < as.size(); i++) {
        const Entry* ax = as[i].last(4);  // PhysicalExprNode.aggregate_expr
        if (!ax) throw std::runtime_error("plan proto: aggregate expression expected");
        const Msg a(ax->b);  // PhysicalAggregateExprNode { user_defined_aggr_function = 4, expr = 2, distinct = 3 } (:912-922)
        std::string fn = a.str(4);
        for (auto& ch : fn) ch = (char)tolower((unsigned char)ch);
        if (fn == "mean") fn = "avg";
        if (!a.subs(5).empty()) throw Unsupported("ordered aggregates are not supported by the device engine");
        o += std::string(i ? "," : "") + "{\"fn\":" + jstr(fn) + ",\"name\":" + jstr(an[i]) + ",\"args\":" + exprs_json(a.subs(2));
        if (a.boolean(3)) o += ",\"distinct\":true";
        o += "}";
      }
      o += "]";
      if (m.has(7)) o += ",\"input_schema\":" + schema_json(m.sub(7));
      return o + ",\"input\":" + in(4) + "}";
    }
    case 9: {  // HashJoinExecNode { left = 1, right = 2, on = 3, join_type = 4, partition_mode = 6, null_equality = 7, filter = 8, projection = 9,
               // null_aware = 10 } (:1134-1145)
      const uint64_t pm = m.u64(6);
      if (pm > 1) throw Unsupported("hash join partition mode Auto must be resolved by the planner");
      // a null-aware anti join (NOT IN) returns nothing once the subquery side holds a NULL key anywhere; tasks here are
      // independent, so no task can know that of a side spread over partitions
      if (m.boolean(10)) throw Unsupported("null-aware hash join (NOT IN)");
      std::string o = "{\"op\":\"HashJoinExec\",\"left\":" + in(1) + ",\"right\":" + in(2) + join_common_json(m, 3, 4, 8) + null_equality_json(m, 7) +
                      ",\"mode\":\"" + (pm == 0 ? "CollectLeft" : "Partitioned") + "\"";
      const std::vector<uint64_t> proj = m.varints(9);
      if (!proj.empty()) o += ",\"projection\":" + u32_list_json(proj);
      return o + "}";
    }
    case 10: {  // SortExecNode { input = 1, expr = 2, fetch = 3 (negative: none), preserve_partitioning = 4 } (:1286-1292)
      std::string o = "{\"op\":\"SortExec\",\"expr\":" + sort_exprs_json(m.subs(2)) + ",\"input\":" + in(1) + ",\"preserve_partitioning\":" +
                      (m.boolean(4) ? "true" : "false");
      if (m.i64(3, -1) >= 0) o += ",\"fetch\":" + std::to_string(m.i64(3));
      return o + "}";
    }
    case 11: return "{\"op\":\"CoalesceBatchesExec\",\"input\":" + in(1) + "}";     // CoalesceBatchesExecNode { input = 1 } (:1309-1313)
    case 12: {  // FilterExecNode { input = 1, expr = 2, projection = 9, fetch = 11 } (:1027-1034)
      std::string o = "{\"op\":\"FilterExec\",\"predicate\":" + expr_json(m.sub(2)) + ",\"input\":" + in(1);
      const std::vector<uint64_t> proj = m.varints(9);
      if (!proj.empty()) o += ",\"projection\":" + u32_list_json(proj);
      if (m.has(11)) o += ",\"fetch\":" + std::to_string(m.u64(11));
      return o + "}";
    }
    case 13: return "{\"op\":\"CoalescePartitionsExec\",\"input\":" + in(1) + "}";  // CoalescePartitionsExecNode { input = 1 } (:1315-1318)
    case 14: {  // RepartitionExecNode { input = 1, partitioning = 5 } (:1325-1333): inside a stage only the row-preserving kinds
      const Msg part = m.sub(5);  // Partitioning { round_robin = 1, hash = 2, unknown = 3 } (:1335-1341)
      if (part.has(2)) throw Unsupported("hash RepartitionExec inside a stage (the distributed planner cuts stages there)");
      return "{\"op\":\"RepartitionExec\",\"input\":" + in(1) + "}";
    }
    case 22: {  // NestedLoopJoinExecNode { left = 1, right = 2, join_type = 3, filter = 4, projection = 5 } (:1301-1307)
      std::string o = "{\"op\":\"NestedLoopJoinExec\",\"left\":" + in(1) + ",\"right\":" + in(2) + join_common_json(m, 0, 3, 4);
      const std::vector<uint64_t> proj = m.varints(5);
      if (!proj.empty()) o += ",\"projection\":" + u32_list_json(proj);
      return o + "}";
    }
    case 32: return in(1);                                                             // CooperativeExecNode: a scheduling wrapper (:1125-1127)
    case 18: {  // PhysicalExtensionNode { node = 1, inputs = 2 } (:845-848) -> BallistaPhysicalPlanNode (ballista.proto:47-54)
      const Msg b(m.bytes(1));
      const Entry* bx = b.oneof({1, 2, 3, 4});
      if (!bx) throw Unsupported("extension node that is not a Ballista plan node");
      const Msg w(bx->b);
      const std::vector<Msg> inputs = m.subs(2);
      switch (bx->field) {
        case 1:    // ShuffleWriterExecNode { job_id = 1, stage_id = 2, output_partitioning = 4 } (ballista.proto:56-63)
        case 4: {  // SortShuffleWriterExecNode (+ batch_size = 8) (ballista.proto:66-73)
          if (inputs.size() != 1) throw std::runtime_error("plan proto: shuffle writer needs exactly one input");
          std::string o = std::string("{\"op\":\"") + (bx->field == 1 ? "ShuffleWriterExec" : "SortShuffleWriterExec") + "\",\"job_id\":" +
                          jstr(override_job.empty() ? w.str(1) : override_job) + ",\"stage_id\":" + std::to_string(w.u64(2)) + ",\"input\":" + plan_json(inputs[0]);
          if (w.has(4)) {  // PhysicalHashRepartition { hash_expr = 1, partition_count = 2 } (datafusion.proto:1320-1323)
            const Msg hp = w.sub(4);
            o += ",\"partitioning\":{\"hash\":" + exprs_json(hp.subs(1)) + ",\"n\":" + std::to_string(hp.u64(2)) + "}";
          }
          return o + "}";
        }
        case 2: {  // ShuffleReaderExecNode { partition = 1, schema = 2, stage_id = 3, broadcast = 5 } (ballista.proto:83-92)
          // "locations": per output partition, where its map outputs live -- PartitionLocation { map_partition_id = 1,
          // partition_id = 2 { job_id = 1, stage_id = 2, partition_id = 4 }, executor_meta = 3 { id = 1, host = 2, port = 3 },
          // partition_stats = 4 { num_rows = 1, num_batches = 2, num_bytes = 3 }, file_id = 6, is_sort_shuffle = 7 }
          // (ballista.proto:244-264,272-277,339-346).  The engine reads what sits in its shuffle store; the host side uses
          // this list to fetch the pieces that live elsewhere (b200_shuffle_read_file / the exchange).
          std::string loc = "[";
          bool fp = true;
          for (auto& part : w.subs(1)) {
            loc += std::string(fp ? "" : ",") + "[";
            fp = false;
            bool fl = true;
            for (auto& l : part.subs(1)) {
              const Msg pid = l.sub(2), ex = l.sub(3), st = l.sub(4);
              loc += std::string(fl ? "" : ",") + "{\"map_partition_id\":" + std::to_string(l.u64(1)) + ",\"job_id\":" + jstr(pid.str(1)) + ",\"stage_id\":" +
                     std::to_string(pid.u64(2)) + ",\"partition_id\":" + std::to_string(pid.u64(4)) + ",\"executor_id\":" + jstr(ex.str(1)) + ",\"host\":" +
                     jstr(ex.str(2)) + ",\"port\":" + std::to_string(ex.u64(3)) + ",\"num_rows\":" + std::to_string(st.i64(1)) + ",\"num_bytes\":" +
                     std::to_string(st.i64(3)) + ",\"is_sort_shuffle\":" + (l.boolean(7) ? "true" : "false");
              if (l.has(6)) loc += ",\"file_id\":" + std::to_string(l.u64(6));
              loc += "}";
              fl = false;
            }
            loc += "]";
          }
          loc += "]";
          return "{\"op\":\"ShuffleReaderExec\",\"stage_id\":" + std::to_string(w.u64(3)) + ",\"schema\":" + schema_json(w.sub(2)) + ",\"broadcast\":" +
                 (w.boolean(5) ? "true" : "false") + ",\"locations\":" + loc + "}";
        }
        default:  // UnresolvedShuffleExecNode { stage_id = 1, schema = 2, broadcast = 6 } (ballista.proto:75-81)
          return "{\"op\":\"UnresolvedShuffleExec\",\"stage_id\":" + std::to_string(w.u64(1)) + ",\"schema\":" + schema_json(w.sub(2)) + ",\"broadcast\":" +
                 (w.boolean(6) ? "true" : "false") + "}";
      }
    }
    case 21: {  // SortPreservingMergeExecNode { input = 1, expr = 2, fetch = 3 } (:1294-1299)
      std::string o = "{\"op\":\"SortPreservingMergeExec\",\"expr\":" + sort_exprs_json(m.subs(2)) + ",\"input\":" + in(1);
      if (m.i64(3, -1) >= 0) o += ",\"fetch\":" + std::to_string(m.i64(3));
      return o + "}";
    }
    case 34: {  // SortMergeJoinExecNode { left = 1, right = 2, on = 3, join_type = 4, filter = 5, sort_options = 6 { asc = 2, nulls_first = 3 },
                // null_equality = 7 } (:1433-1441)
      std::string o = "{\"op\":\"SortMergeJoinExec\",\"left\":" + in(1) + ",\"right\":" + in(2) + join_common_json(m, 3, 4, 5) + null_equality_json(m, 7) +
                      ",\"sort_options\":[";
      bool first = true;
      for (auto& so : m.subs(6)) {
        o += std::string(first ? "" : ",") + "{\"asc\":" + (so.boolean(2) ? "true" : "false") + ",\"nulls_first\":" + (so.boolean(3) ? "true" : "false") + "}";
        first = false;
      }
      return o + "]}";
    }
    case 15: {  // WindowAggExecNode { input = 1, window_expr = 2, partition_keys = 5, linear = 7 | partially_sorted = 8 | sorted = 9 } (:1230-1240)
      // no input order mode: WindowAggExec; sorted: BoundedWindowAggExec; the other two modes are refused by the typing
      const char* mode = m.has(9) ? "\"sorted\"" : m.has(8) ? "\"partially_sorted\"" : m.has(7) ? "\"linear\"" : "null";
      std::string o = std::string("{\"op\":\"WindowAggExec\",\"mode\":") + mode + ",\"partition_keys\":" + exprs_json(m.subs(5)) + ",\"window_expr\":[";
      const std::vector<Msg> ws = m.subs(2);
      for (size_t i = 0; i < ws.size(); i++) {
        // PhysicalWindowExprNode { user_defined_aggr_function = 3 | user_defined_window_function = 10, args = 4, partition_by = 5,
        // order_by = 6, window_frame = 7, name = 8, ignore_nulls = 11, distinct = 12 } (:924-938); fun_definition = 9 is
        // ignored, as the aggregate decoder ignores UDAF payloads
        const Msg& w = ws[i];
        std::string fn = w.has(10) ? w.str(10) : w.str(3);
        if (fn.empty()) throw std::runtime_error("plan proto: window expression without a function name");
        for (auto& ch : fn) ch = (char)tolower((unsigned char)ch);
        o += std::string(i ? "," : "") + "{\"fn\":" + jstr(fn) + ",\"name\":" + jstr(w.str(8)) + ",\"args\":" + exprs_json(w.subs(4)) +
             ",\"partition_by\":" + exprs_json(w.subs(5)) + ",\"order_by\":[";
        const std::vector<Msg> ob = w.subs(6);
        for (size_t k = 0; k < ob.size(); k++) o += std::string(k ? "," : "") + sort_expr_json(ob[k]);
        o += "]";
        if (w.has(7)) o += ",\"frame\":" + window_frame_json(w.sub(7));
        if (w.boolean(11)) o += ",\"ignore_nulls\":true";
        if (w.boolean(12)) o += ",\"distinct\":true";
        o += "}";
      }
      return o + "],\"input\":" + in(1) + "}";
    }
    default: throw Unsupported("physical plan node variant " + std::to_string(x->field) + " is not supported by the device engine");
  }
}

// Entry point: bytes of a datafusion.PhysicalPlanNode -> stage-plan IR (JSON text).  `override_job` replaces the job id
// stored in the shuffle writer node when non-empty (the task definition carries the authoritative one).
inline std::string plan_proto_to_json(const void* bytes, size_t n, const std::string& override_job = std::string()) {
  Slice s;
  s.p = (const uint8_t*)bytes;
  s.n = n;
  return plan_json(Msg(s), override_job);
}

// ---- ballista.protobuf.TaskDefinition / MultiTaskDefinition (ballista.proto:518-542) ------------------------------------------
// What an executor receives for a task (LaunchTask / LaunchMultiTask / PollWork): identity, session properties and the plan
// bytes.  Decoded to {"job_id","stage_id","stage_attempt_num","session_id","launch_time","tasks":[{"task_id",
// "task_attempt_num","partition_id"}],"props":{..}}; *plan receives the embedded PhysicalPlanNode bytes.
struct TaskInfo {
  std::string job_id, session_id;
  uint64_t stage_id = 0, stage_attempt = 0, launch_time = 0;
  struct Task {
    uint64_t task_id, attempt, partition;
  };
  std::vector<Task> tasks;
  std::vector<std::pair<std::string, std::string>> props;  // KeyValuePair { key = 1, optional value = 2 } (:203-206)
  Slice plan;
};

inline TaskInfo decode_task_definition(const void* bytes, size_t n, bool multi) {
  Slice s;
  s.p = (const uint8_t*)bytes;
  s.n = n;
  const Msg m(s);
  TaskInfo t;
  std::vector<Msg> props;
  if (multi) {  // MultiTaskDefinition { task_ids = 1, job_id = 2, stage_id = 3, stage_attempt_num = 4, plan = 5, session_id = 7, launch_time = 8, props = 9 }
    for (auto& id : m.subs(1)) t.tasks.push_back(TaskInfo::Task{id.u64(1), id.u64(2), id.u64(3)});  // TaskId (:266-270)
    t.job_id = m.str(2);
    t.stage_id = m.u64(3);
    t.stage_attempt = m.u64(4);
    t.plan = m.bytes(5);
    t.session_id = m.str(7);
    t.launch_time = m.u64(8);
    props = m.subs(9);
  } else {  // TaskDefinition { task_id = 1, task_attempt_num = 2, job_id = 3, stage_id = 4, stage_attempt_num = 5, partition_id = 6, plan = 7, session_id = 9, launch_time = 10, props = 11 }
    t.tasks.push_back(TaskInfo::Task{m.u64(1), m.u64(2), m.u64(6)});
    t.job_id = m.str(3);
    t.stage_id = m.u64(4);
    t.stage_attempt = m.u64(5);
    t.plan = m.bytes(7);
    t.session_id = m.str(9);
    t.launch_time = m.u64(10);
    props = m.subs(11);
  }
  for (auto& kv : props) t.props.push_back({kv.str(1), kv.str(2)});
  if (t.plan.n == 0) throw std::runtime_error("task definition without plan bytes");
  return t;
}

inline std::string task_info_json(const TaskInfo& t) {
  std::string o = "{\"job_id\":" + jstr(t.job_id) + ",\"stage_id\":" + std::to_string(t.stage_id) + ",\"stage_attempt_num\":" + std::to_string(t.stage_attempt) +
                  ",\"session_id\":" + jstr(t.session_id) + ",\"launch_time\":" + std::to_string(t.launch_time) + ",\"tasks\":[";
  for (size_t i = 0; i < t.tasks.size(); i++)
    o += std::string(i ? "," : "") + "{\"task_id\":" + std::to_string(t.tasks[i].task_id) + ",\"task_attempt_num\":" + std::to_string(t.tasks[i].attempt) +
         ",\"partition_id\":" + std::to_string(t.tasks[i].partition) + "}";
  o += "],\"props\":{";
  for (size_t i = 0; i < t.props.size(); i++) o += std::string(i ? "," : "") + jstr(t.props[i].first) + ":" + jstr(t.props[i].second);
  return o + "}}";
}

// ---- protobuf writer (for the way back: TaskStatus) ------------------------------------------------------------------------
struct Writer {
  std::string out;
  void varint(uint64_t v) {
    while (v >= 0x80) {
      out.push_back((char)(v | 0x80));
      v >>= 7;
    }
    out.push_back((char)v);
  }
  void key(uint32_t field, uint32_t wire) { varint(((uint64_t)field << 3) | wire); }
  // proto3: scalar fields at their default value are not written
  void u64(uint32_t field, uint64_t v) {
    if (!v) return;
    key(field, 0);
    varint(v);
  }
  void u64_always(uint32_t field, uint64_t v) {  // members of a oneof / optional fields are written even when zero
    key(field, 0);
    varint(v);
  }
  void boolean(uint32_t field, bool v) { u64(field, v ? 1 : 0); }
  void str(uint32_t field, const std::string& v) {
    if (v.empty()) return;
    key(field, 2);
    varint(v.size());
    out += v;
  }
  void msg(uint32_t field, const Writer& m) {  // sub-messages are written even when empty (presence)
    key(field, 2);
    varint(m.out.size());
    out += m.out;
  }
};

}  // namespace pbp
}  // namespace b200
