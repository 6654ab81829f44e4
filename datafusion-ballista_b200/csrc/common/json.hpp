// Minimal JSON value + recursive-descent parser + writer (header-only).
// Used for the stage-plan IR that crosses the C-ABI (`b200_stage_prepare`), which is the
// wire form a Rust shim would produce from the DataFusion physical plan whose node shapes are
// pinned by ballista/core/proto/datafusion.proto:716-757 (plan nodes) and :851-901 (expr nodes).
#pragma once
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

namespace b200 {

struct Json {
  enum Kind { Null, Bool, Num, Str, Arr, Obj } kind = Null;
  bool b = false;
  double num = 0;
  bool is_int = false;
  int64_t i = 0;
  std::string s;  // string value; for Num also the raw token text (big decimals)
  std::vector<Json> a;
  std::vector<std::pair<std::string, Json>> o;

  bool is_null() const { return kind == Null; }
  bool is_obj() const { return kind == Obj; }
  bool is_arr() const { return kind == Arr; }
  bool is_str() const { return kind == Str; }
  bool is_num() const { return kind == Num; }
  bool is_bool() const { return kind == Bool; }

  const Json* find(const std::string& k) const {
    if (kind != Obj) return nullptr;
    for (auto& kv : o)
      if (kv.first == k) return &kv.second;
    return nullptr;
  }
  bool has(const std::string& k) const {
    const Json* j = find(k);
    return j && !j->is_null();
  }
  const Json& at(const std::string& k) const {
    const Json* j = find(k);
    if (!j) throw std::runtime_error("plan IR: missing key '" + k + "'");
    return *j;
  }
  const Json& at(size_t idx) const {
    if (kind != Arr || idx >= a.size()) throw std::runtime_error("plan IR: array index out of range");
    return a[idx];
  }
  size_t size() const { return kind == Arr ? a.size() : kind == Obj ? o.size() : 0; }
  const std::string& str() const {
    if (kind != Str) throw std::runtime_error("plan IR: expected string");
    return s;
  }
  int64_t as_int() const {
    if (kind == Num) return is_int ? i : (int64_t)num;
    if (kind == Bool) return b;
    throw std::runtime_error("plan IR: expected integer");
  }
  double as_double() const {
    if (kind != Num) throw std::runtime_error("plan IR: expected number");
    return is_int ? (double)i : num;
  }
  bool as_bool() const {
    if (kind == Bool) return b;
    if (kind == Num) return as_int() != 0;
    throw std::runtime_error("plan IR: expected bool");
  }
  std::string get_str(const std::string& k, const std::string& dflt) const {
    const Json* j = find(k);
    return (j && j->kind == Str) ? j->s : dflt;
  }
  int64_t get_int(const std::string& k, int64_t dflt) const {
    const Json* j = find(k);
    return (j && (j->kind == Num || j->kind == Bool)) ? j->as_int() : dflt;
  }
  bool get_bool(const std::string& k, bool dflt) const {
    const Json* j = find(k);
    return (j && (j->kind == Bool || j->kind == Num)) ? j->as_bool() : dflt;
  }
};

class JsonParser {
 public:
  explicit JsonParser(const char* p, size_t n) : p_(p), e_(p + n) {}
  Json parse() {
    Json v = value();
    ws();
    if (p_ != e_) fail("trailing characters");
    return v;
  }

 private:
  const char* p_;
  const char* e_;
  [[noreturn]] void fail(const char* m) { throw std::runtime_error(std::string("JSON parse error: ") + m); }
  void ws() {
    while (p_ < e_ && (*p_ == ' ' || *p_ == '\n' || *p_ == '\t' || *p_ == '\r')) ++p_;
  }
  Json value() {
    ws();
    if (p_ >= e_) fail("unexpected end");
    char c = *p_;
    if (c == '{') return object();
    if (c == '[') return array();
    if (c == '"') {
      Json j;
      j.kind = Json::Str;
      j.s = string();
      return j;
    }
    if (c == 't' && e_ - p_ >= 4 && !memcmp(p_, "true", 4)) {
      p_ += 4;
      Json j;
      j.kind = Json::Bool;
      j.b = true;
      return j;
    }
    if (c == 'f' && e_ - p_ >= 5 && !memcmp(p_, "false", 5)) {
      p_ += 5;
      Json j;
      j.kind = Json::Bool;
      j.b = false;
      return j;
    }
    if (c == 'n' && e_ - p_ >= 4 && !memcmp(p_, "null", 4)) {
      p_ += 4;
      return Json();
    }
    return number();
  }
  Json number() {
    const char* s = p_;
    bool isint = true;
    if (p_ < e_ && (*p_ == '-' || *p_ == '+')) ++p_;
    while (p_ < e_ && ((*p_ >= '0' && *p_ <= '9') || *p_ == '.' || *p_ == 'e' || *p_ == 'E' || *p_ == '-' || *p_ == '+')) {
      if (*p_ == '.' || *p_ == 'e' || *p_ == 'E') isint = false;
      ++p_;
    }
    if (p_ == s) fail("bad token");
    Json j;
    j.kind = Json::Num;
    j.s.assign(s, p_ - s);
    j.is_int = isint;
    if (isint) {
      errno = 0;
      j.i = strtoll(j.s.c_str(), nullptr, 10);
      j.num = (double)j.i;
    } else {
      j.num = strtod(j.s.c_str(), nullptr);
      j.i = (int64_t)j.num;
    }
    return j;
  }
  std::string string() {
    ++p_;  // opening quote
    std::string out;
    while (p_ < e_ && *p_ != '"') {
      if (*p_ == '\\') {
        ++p_;
        if (p_ >= e_) fail("bad escape");
        switch (*p_) {
          case 'n': out += '\n'; break;
          case 't': out += '\t'; break;
          case 'r': out += '\r'; break;
          case 'b': out += '\b'; break;
          case 'f': out += '\f'; break;
          case 'u': {
            if (e_ - p_ < 5) fail("bad \\u escape");
            unsigned cp = (unsigned)strtoul(std::string(p_ + 1, 4).c_str(), nullptr, 16);
            p_ += 4;
            // a surrogate pair (what JSON writers emit for a code point above U+FFFF) is one 4-byte UTF-8 sequence
            if (cp >= 0xD800 && cp <= 0xDBFF && e_ - p_ >= 7 && p_[1] == '\\' && p_[2] == 'u') {
              const unsigned lo = (unsigned)strtoul(std::string(p_ + 3, 4).c_str(), nullptr, 16);
              if (lo >= 0xDC00 && lo <= 0xDFFF) {
                cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
                p_ += 6;
                out += (char)(0xF0 | (cp >> 18));
                out += (char)(0x80 | ((cp >> 12) & 0x3F));
                out += (char)(0x80 | ((cp >> 6) & 0x3F));
                out += (char)(0x80 | (cp & 0x3F));
                break;
              }
            }
            if (cp < 0x80) out += (char)cp;
            else if (cp < 0x800) {
              out += (char)(0xC0 | (cp >> 6));
              out += (char)(0x80 | (cp & 0x3F));
            } else {
              out += (char)(0xE0 | (cp >> 12));
              out += (char)(0x80 | ((cp >> 6) & 0x3F));
              out += (char)(0x80 | (cp & 0x3F));
            }
            break;
          }
          default: out += *p_;
        }
        ++p_;
      } else {
        out += *p_++;
      }
    }
    if (p_ >= e_) fail("unterminated string");
    ++p_;
    return out;
  }
  Json array() {
    ++p_;
    Json j;
    j.kind = Json::Arr;
    ws();
    if (p_ < e_ && *p_ == ']') {
      ++p_;
      return j;
    }
    for (;;) {
      j.a.push_back(value());
      ws();
      if (p_ >= e_) fail("unterminated array");
      if (*p_ == ',') {
        ++p_;
        continue;
      }
      if (*p_ == ']') {
        ++p_;
        return j;
      }
      fail("expected , or ]");
    }
  }
  Json object() {
    ++p_;
    Json j;
    j.kind = Json::Obj;
    ws();
    if (p_ < e_ && *p_ == '}') {
      ++p_;
      return j;
    }
    for (;;) {
      ws();
      if (p_ >= e_ || *p_ != '"') fail("expected key");
      std::string k = string();
      ws();
      if (p_ >= e_ || *p_ != ':') fail("expected :");
      ++p_;
      j.o.emplace_back(std::move(k), value());
      ws();
      if (p_ >= e_) fail("unterminated object");
      if (*p_ == ',') {
        ++p_;
        continue;
      }
      if (*p_ == '}') {
        ++p_;
        return j;
      }
      fail("expected , or }");
    }
  }
};

inline Json parse_json(const char* p, size_t n) { return JsonParser(p, n).parse(); }
inline Json parse_json(const std::string& s) { return JsonParser(s.data(), s.size()).parse(); }

inline void json_escape(const std::string& s, std::string& out) {
  out += '"';
  for (unsigned char c : s) {
    switch (c) {
      case '"': out += "\\\""; break;
      case '\\': out += "\\\\"; break;
      case '\n': out += "\\n"; break;
      case '\t': out += "\\t"; break;
      case '\r': out += "\\r"; break;
      default:
        if (c < 0x20) {
          char buf[8];
          snprintf(buf, sizeof buf, "\\u%04x", c);
          out += buf;
        } else {
          out += (char)c;
        }
    }
  }
  out += '"';
}

}  // namespace b200
