// Regular expressions as byte DFAs: the compiler (host, pure C++) and the walk (host and device, one function).
//
// Semantics follow the Rust `regex` crate, through which DataFusion evaluates `~` / `~*` / `!~` / `!~*`, regexp_like and
// ILIKE (arrow-rs `regexp_is_match`, and `like` with case_insensitive = true) [EXT, DESIGN.md §6 (x)]:
//   * a match is unanchored (Regex::is_match);
//   * `.` is any Unicode scalar value except `\n` (any value under the flag s); `^` / `\A` is the start of the text,
//     `$` / `\z` its end (not before a trailing `\n`: no multi-line mode);
//   * `\d` is general category Nd and `\s` White_Space (Unicode mode, csrc/common/unicode_tables.hpp);
//   * under the flag i, an ASCII letter matches its other case, k / K also match U+212A KELVIN SIGN and s / S also
//     U+017F LATIN SMALL LETTER LONG S (Rust's simple case folding restricted to ASCII); a negated class is folded before
//     it is negated.
// Anything outside the accepted subset is refused, never approximated: `\w \W \b \B \< \> \p \P`, the flags m x U u R,
// class set operations, non-ASCII literals under i and patterns whose DFA exceeds kMaxStates / kMaxTransBytes are
// unsupported (RX_UNSUPPORTED); what Rust itself rejects is invalid (RX_INVALID, with the byte offset).
//
// Pipeline: parser -> NFA over UTF-8 bytes (code point sets become UTF-8 byte-sequence automata; column strings are
// validated UTF-8, so no invalid sequence needs a path) -> byte equivalence classes -> subset construction for an
// unanchored search (start of text resolved in the start state) -> one blob the walk reads:
//   [256] byte -> class   [n_states, padded to 8] accepts-at-end flag   [n_states][n_cls] uint16 next state
// State 0 is dead (the walk stops: no match), state 1 has matched (the walk stops: match).
// regexp_count and regexp_replace need match spans, so the same parser and NFA also give two span DFAs (SpanDfaBuilder,
// DESIGN.md §6 (xiii)): a forward leftmost-first one and a reverse anchored one, in the same blob layout with per-state
// flags instead of an absorbing matched state.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B200_RX_HD __host__ __device__
#else
#define B200_RX_HD
#endif

namespace b200 {
namespace rx {

static const uint32_t kDead = 0, kMatched = 1;
static const uint32_t kMaxStates = 65535;
static const uint64_t kMaxTransBytes = (uint64_t)1 << 20;

B200_RX_HD inline uint32_t dfa_trans_offset(uint32_t n_states) { return 256u + ((n_states + 7u) & ~7u); }
// the shape travels with the device pointer in one 64-bit word (ImmDesc::hi of OP_REGEX)
B200_RX_HD inline uint64_t dfa_shape_pack(uint32_t n_states, uint32_t n_cls, uint32_t start) {
  return (uint64_t)n_states << 32 | (uint64_t)n_cls << 16 | start;
}

B200_RX_HD inline uint32_t rx_ld8(const uint8_t* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(p);
#else
  return *p;
#endif
}
B200_RX_HD inline uint32_t rx_ld16(const uint16_t* p) {
#if defined(__CUDA_ARCH__)
  return __ldg(p);
#else
  return *p;
#endif
}

// Does the DFA `blob` (shape packed by dfa_shape_pack) match somewhere in s[0..n)?  Reads the tables through the read-only
// path; stops at the first byte that reaches the matched or the dead state.
B200_RX_HD inline bool dfa_is_match(const uint8_t* blob, uint64_t shape, const uint8_t* s, uint32_t n) {
  const uint32_t n_states = (uint32_t)(shape >> 32), n_cls = (uint32_t)(shape >> 16) & 0xFFFFu;
  const uint16_t* tr = (const uint16_t*)(blob + dfa_trans_offset(n_states));
  uint32_t st = (uint32_t)shape & 0xFFFFu;
  for (uint32_t i = 0; i < n && st > kMatched; i++) st = rx_ld16(tr + st * n_cls + rx_ld8(blob + s[i]));
  return rx_ld8(blob + 256 + st) != 0;
}

// ---- match spans: regexp_count and regexp_replace [EXT, DESIGN.md §6 (xiii)] ------------------------------------------------
// Two more DFAs per pattern (SpanDfaBuilder below): a forward one that finds where the leftmost-first match beginning at or
// after a search start ends (Regex::find), and a reverse one that runs back from that end to find where it begins.  A
// state's flags byte says whether a match ends (forward) or begins (reverse) at the current offset.
static const uint32_t kSpanHere = 1, kSpanAtEdge = 2;                // flags: here; only at the text's end / offset 0
static const uint32_t kSpanStartEdge = 1, kSpanStartInside = 2;      // start states: at the text's edge or not

// bytes of the UTF-8 sequence led by c (1 for a stray continuation byte), at most `left`
B200_RX_HD inline uint32_t rx_cp_len(uint32_t c, uint32_t left) {
  const uint32_t k = c >= 0xF0 ? 4 : c >= 0xE0 ? 3 : c >= 0xC0 ? 2 : 1;
  return k < left ? k : left;
}
// byte offset of s[0..n) after its first k code points (n when it has fewer)
B200_RX_HD inline uint32_t rx_skip_cps(const uint8_t* s, uint32_t n, int64_t k) {
  uint32_t i = 0;
  for (; k > 0 && i < n; k--) i += rx_cp_len(s[i], n - i);
  return i;
}

// End of the leftmost-first match of s[0..n) that begins at or after pos, or -1: the forward walk runs until the dead
// state or the end of the text and keeps the last offset where a match ended.
B200_RX_HD inline int64_t dfa_find_end(const uint8_t* blob, uint64_t shape, const uint8_t* s, uint32_t n, uint32_t pos) {
  const uint32_t n_states = (uint32_t)(shape >> 32), n_cls = (uint32_t)(shape >> 16) & 0xFFFFu;
  const uint16_t* tr = (const uint16_t*)(blob + dfa_trans_offset(n_states));
  uint32_t st = pos == 0 ? kSpanStartEdge : kSpanStartInside;
  int64_t end = -1;
  for (uint32_t i = pos;; i++) {
    if (rx_ld8(blob + 256 + st) & (i == n ? kSpanAtEdge : kSpanHere)) end = i;
    if (i == n) break;
    st = rx_ld16(tr + st * n_cls + rx_ld8(blob + s[i]));
    if (st == kDead) break;
  }
  return end;
}
// Start of the match that ends at `end`: the reverse walk runs from end back to pos (never further) and keeps the smallest
// offset where the reversed pattern accepts.  end is an offset where a match found from pos ends, so one exists.
B200_RX_HD inline uint32_t dfa_find_start(const uint8_t* blob, uint64_t shape, const uint8_t* s, uint32_t n, uint32_t pos, uint32_t end) {
  const uint32_t n_states = (uint32_t)(shape >> 32), n_cls = (uint32_t)(shape >> 16) & 0xFFFFu;
  const uint16_t* tr = (const uint16_t*)(blob + dfa_trans_offset(n_states));
  uint32_t st = end == n ? kSpanStartEdge : kSpanStartInside;
  uint32_t start = end;
  for (uint32_t j = end;; j--) {
    if (rx_ld8(blob + 256 + st) & (j == 0 ? kSpanAtEdge : kSpanHere)) start = j;
    if (j == pos) break;
    st = rx_ld16(tr + st * n_cls + rx_ld8(blob + s[j - 1]));
    if (st == kDead) break;
  }
  return start;
}

// The span DFAs of one pattern and the state of one find_iter over s[0..n) (the Rust regex crate's iteration):
//   1. search from pos;
//   2. an empty match ending where the last reported match ended is not reported: the search restarts one code point on;
//   3. after any other empty match the next search starts one code point past it;
//   4. after a non-empty match it starts at the match's end.
struct RxSpans {
  const uint8_t* fwd;
  uint64_t fwd_shape;
  const uint8_t* rev;
  uint64_t rev_shape;
};
struct RxIter {
  uint32_t pos;
  int64_t last;  // end of the last reported match, -1 before the first
};
// The next reported match of the iteration: its span in [*ms, *me), false when there is none
B200_RX_HD inline bool dfa_next_match(const RxSpans& d, const uint8_t* s, uint32_t n, RxIter& it, uint32_t* ms, uint32_t* me) {
  while (it.pos <= n) {
    const int64_t e = dfa_find_end(d.fwd, d.fwd_shape, s, n, it.pos);
    if (e < 0) return false;
    const uint32_t b = dfa_find_start(d.rev, d.rev_shape, s, n, it.pos, (uint32_t)e);
    const uint32_t step = (uint32_t)e < n ? rx_cp_len(s[e], n - (uint32_t)e) : 1;
    if (b == (uint32_t)e && e == it.last) {  // rule 2
      it.pos = (uint32_t)e + step;
      continue;
    }
    *ms = b;
    *me = (uint32_t)e;
    it.last = e;
    it.pos = b == (uint32_t)e ? (uint32_t)e + step : (uint32_t)e;  // rules 3 and 4
    return true;
  }
  return false;
}
// regexp_count: the number of reported matches in s[0..n)
B200_RX_HD inline uint32_t dfa_count(const RxSpans& d, const uint8_t* s, uint32_t n) {
  RxIter it = {0, -1};
  uint32_t ms, me, c = 0;
  while (dfa_next_match(d, s, n, it, &ms, &me)) c++;
  return c;
}
// regexp_count of one non-NULL row: an empty str counts 0 before `start` applies (DataFusion returns 0 for it at once);
// otherwise the haystack loses its first `skip` (start - 1) code points -- past the end it is '', where a pattern that
// matches empty still counts 1 -- and its matches are counted
B200_RX_HD inline uint32_t regexp_count_row(const RxSpans& d, const uint8_t* s, uint32_t n, int64_t skip) {
  if (n == 0) return 0;
  const uint32_t off = rx_skip_cps(s, n, skip);
  return dfa_count(d, s + off, n - off);
}
// regexp_replace: s[0..n) with the first match (every match when `global`) replaced by rep[0..rep_len).  Returns the
// result's length; writes the result to out unless it is null (the length pass).
B200_RX_HD inline uint64_t dfa_replace(const RxSpans& d, const uint8_t* s, uint32_t n, const uint8_t* rep, uint32_t rep_len, bool global,
                                       uint8_t* out) {
  RxIter it = {0, -1};
  uint32_t ms, me, done = 0;
  uint64_t len = 0;
  while (dfa_next_match(d, s, n, it, &ms, &me)) {
    if (out) {
      for (uint32_t i = done; i < ms; i++) out[len + i - done] = s[i];
      for (uint32_t i = 0; i < rep_len; i++) out[len + ms - done + i] = rep[i];
    }
    len += (ms - done) + rep_len;
    done = me;
    if (!global) break;
  }
  if (out)
    for (uint32_t i = done; i < n; i++) out[len + i - done] = s[i];
  return len + (n - done);
}

}  // namespace rx
}  // namespace b200

// ---- the compiler (host) ----------------------------------------------------------------------------------------------------
#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <utility>
#include <vector>

#include "unicode_tables.hpp"

namespace b200 {
namespace rx {

enum { RX_OK = 0, RX_INVALID = -1, RX_UNSUPPORTED = -2 };

struct Dfa {
  uint32_t n_states = 0, n_cls = 0, start = 0;
  std::vector<uint8_t> blob;
  uint64_t shape() const { return dfa_shape_pack(n_states, n_cls, start); }
  bool is_match(const std::string& s) const { return dfa_is_match(blob.data(), shape(), (const uint8_t*)s.data(), (uint32_t)s.size()); }
};

struct Error {
  int code;
  std::string msg;
};

typedef std::vector<std::pair<uint32_t, uint32_t>> CpSet;  // sorted, disjoint, non-adjacent code point ranges

inline CpSet cp_normalize(CpSet s) {
  std::sort(s.begin(), s.end());
  CpSet o;
  for (auto& r : s) {
    if (!o.empty() && r.first <= o.back().second + 1) o.back().second = std::max(o.back().second, r.second);
    else o.push_back(r);
  }
  return o;
}
inline CpSet cp_negate(const CpSet& s) {
  CpSet o;
  uint32_t next = 0;
  for (auto& r : s) {
    if (r.first > next) o.push_back({next, r.first - 1});
    next = r.second + 1;
  }
  if (next <= 0x10FFFF) o.push_back({next, 0x10FFFF});
  return o;
}
inline bool cp_has(const CpSet& s, uint32_t c) {
  for (auto& r : s)
    if (c >= r.first && c <= r.second) return true;
  return false;
}
// Rust's simple case folding restricted to ASCII letters and the two non-ASCII code points that fold onto them
inline CpSet cp_fold(const CpSet& s) {
  CpSet o = s;
  for (auto& r : s) {
    const uint32_t lo = std::max<uint32_t>(r.first, 'A'), hi = std::min<uint32_t>(r.second, 'Z');
    if (lo <= hi) o.push_back({lo + 32, hi + 32});
    const uint32_t lo2 = std::max<uint32_t>(r.first, 'a'), hi2 = std::min<uint32_t>(r.second, 'z');
    if (lo2 <= hi2) o.push_back({lo2 - 32, hi2 - 32});
  }
  const bool k = cp_has(s, 'k') || cp_has(s, 'K') || cp_has(s, 0x212A), ls = cp_has(s, 's') || cp_has(s, 'S') || cp_has(s, 0x17F);
  if (k) o.insert(o.end(), {{'k', 'k'}, {'K', 'K'}, {0x212A, 0x212A}});
  if (ls) o.insert(o.end(), {{'s', 's'}, {'S', 'S'}, {0x17F, 0x17F}});
  return cp_normalize(o);
}
inline CpSet cp_table(const uint32_t (*t)[2], int n) {
  CpSet o;
  for (int i = 0; i < n; i++) o.push_back({t[i][0], t[i][1]});
  return o;
}

// UTF-8 byte-range sequences of the code points [lo, hi] (surrogates excluded): the classic range splitting
inline int utf8_len(uint32_t c) { return c < 0x80 ? 1 : c < 0x800 ? 2 : c < 0x10000 ? 3 : 4; }
inline int utf8_encode(uint32_t c, uint8_t* b) {
  if (c < 0x80) { b[0] = (uint8_t)c; return 1; }
  if (c < 0x800) { b[0] = (uint8_t)(0xC0 | c >> 6); b[1] = (uint8_t)(0x80 | (c & 0x3F)); return 2; }
  if (c < 0x10000) { b[0] = (uint8_t)(0xE0 | c >> 12); b[1] = (uint8_t)(0x80 | ((c >> 6) & 0x3F)); b[2] = (uint8_t)(0x80 | (c & 0x3F)); return 3; }
  b[0] = (uint8_t)(0xF0 | c >> 18); b[1] = (uint8_t)(0x80 | ((c >> 12) & 0x3F)); b[2] = (uint8_t)(0x80 | ((c >> 6) & 0x3F)); b[3] = (uint8_t)(0x80 | (c & 0x3F));
  return 4;
}
typedef std::vector<std::pair<uint8_t, uint8_t>> ByteSeq;
inline void utf8_sequences(uint32_t lo, uint32_t hi, std::vector<ByteSeq>& out) {
  if (lo > hi) return;
  if (lo <= 0xDFFF && hi >= 0xD800) {  // no surrogate is a scalar value
    if (lo < 0xD800) utf8_sequences(lo, 0xD7FF, out);
    if (hi > 0xDFFF) utf8_sequences(0xE000, hi, out);
    return;
  }
  static const uint32_t max_of_len[] = {0x7F, 0x7FF, 0xFFFF, 0x10FFFF};
  for (int k = 0; k < 3; k++)
    if (lo <= max_of_len[k] && hi > max_of_len[k]) {
      utf8_sequences(lo, max_of_len[k], out);
      utf8_sequences(max_of_len[k] + 1, hi, out);
      return;
    }
  const int n = utf8_len(lo);
  for (int i = 1; i < n; i++) {
    const uint32_t m = (1u << (6 * i)) - 1;
    if ((lo & ~m) != (hi & ~m)) {
      if ((lo & m) != 0) {
        utf8_sequences(lo, lo | m, out);
        utf8_sequences((lo | m) + 1, hi, out);
        return;
      }
      if ((hi & m) != m) {
        utf8_sequences(lo, (hi & ~m) - 1, out);
        utf8_sequences(hi & ~m, hi, out);
        return;
      }
    }
  }
  uint8_t a[4], b[4];
  utf8_encode(lo, a);
  utf8_encode(hi, b);
  ByteSeq s;
  for (int i = 0; i < n; i++) s.push_back({a[i], b[i]});
  out.push_back(s);
}

struct Node {
  enum Kind { Empty, Set, Cat, Alt, Rep, Start, End } k = Empty;
  CpSet set;
  std::vector<Node> kids;
  int mn = 0, mx = -1;  // Rep: mx = -1 is unbounded
  bool greedy = true;   // Rep: false after a trailing '?' (only the leftmost-first span DFA tells the two apart)
};

class Parser {
 public:
  Parser(const std::string& p, const std::string& shown) : p_(p), shown_(shown) {}

  Node parse(bool ci, bool dotall) {
    Flags f{ci, dotall};
    Node n = parse_alt(f, 0);
    if (pos_ < p_.size()) invalid("unopened group: ')' without a matching '('", pos_);
    return n;
  }

  [[noreturn]] void invalid(const std::string& what, size_t at) const {
    throw Error{RX_INVALID, "regex parse error in '" + shown_ + "' at byte offset " + std::to_string(at) + ": " + what};
  }
  [[noreturn]] void unsupported(const std::string& what) const {
    throw Error{RX_UNSUPPORTED, "regex '" + shown_ + "': " + what + " is not supported by the device engine"};
  }

 private:
  struct Flags {
    bool i, s;
  };
  const std::string& p_;
  const std::string& shown_;
  size_t pos_ = 0;
  std::set<std::string> names_;

  bool eof() const { return pos_ >= p_.size(); }
  char peek(size_t k = 0) const { return pos_ + k < p_.size() ? p_[pos_ + k] : '\0'; }

  uint32_t next_cp() {
    const size_t at = pos_;
    const uint8_t c = (uint8_t)p_[pos_];
    const int n = c < 0x80 ? 1 : (c >> 5) == 6 ? 2 : (c >> 4) == 14 ? 3 : (c >> 3) == 30 ? 4 : 0;
    if (!n || pos_ + n > p_.size()) invalid("the pattern is not valid UTF-8", at);
    uint32_t v = n == 1 ? c : n == 2 ? (c & 0x1F) : n == 3 ? (c & 0x0F) : (c & 0x07);
    for (int i = 1; i < n; i++) {
      const uint8_t d = (uint8_t)p_[pos_ + i];
      if ((d & 0xC0) != 0x80) invalid("the pattern is not valid UTF-8", at);
      v = v << 6 | (d & 0x3F);
    }
    static const uint32_t min_of_len[] = {0, 0, 0x80, 0x800, 0x10000};
    if (v < min_of_len[n] || v > 0x10FFFF || (v >= 0xD800 && v <= 0xDFFF)) invalid("the pattern is not valid UTF-8", at);
    pos_ += n;
    return v;
  }

  static std::string cp_name(uint32_t c) {
    char b[16];
    snprintf(b, sizeof b, "U+%04X", c);
    uint8_t u[4];
    const int n = utf8_encode(c, u);
    return "'" + std::string((const char*)u, (size_t)n) + "' (" + b + ")";
  }

  // a literal code point as a set, folded under i (ASCII only)
  Node literal(uint32_t c, const Flags& f) {
    Node n;
    n.k = Node::Set;
    if (f.i && c >= 0x80) unsupported("case-insensitive matching of the non-ASCII character " + cp_name(c));
    n.set = {{c, c}};
    if (f.i) n.set = cp_fold(n.set);
    return n;
  }
  static Node set_node(const CpSet& s) {
    Node n;
    n.k = Node::Set;
    n.set = cp_normalize(s);
    return n;
  }

  // groups and bracket classes share one nesting limit, as in Rust's parser (nest_limit 250); it also bounds the recursion
  static const int kMaxNest = 250;
  void check_nest(int depth) const {
    if (depth > kMaxNest) unsupported("nesting of groups and classes deeper than " + std::to_string(kMaxNest));
  }

  Node parse_alt(Flags& f, int depth) {
    check_nest(depth);
    std::vector<Node> alts;
    Node cat;
    cat.k = Node::Cat;
    enum { NONE, ATOM, REP, FLAGS } last = NONE;
    while (!eof()) {
      const char c = peek();
      if (c == ')') break;
      if (c == '|') {
        pos_++;
        alts.push_back(cat);
        cat.kids.clear();
        last = NONE;
        continue;
      }
      if (c == '*' || c == '+' || c == '?' || c == '{') {
        const size_t at = pos_;
        if (last == NONE || last == FLAGS) invalid("repetition operator missing expression", at);
        if (last == REP) unsupported("a repetition of a repetition ('" + p_.substr(at, 1) + "' after a repetition operator)");
        Node r;
        r.k = Node::Rep;
        parse_repetition(r);
        r.kids.push_back(cat.kids.back());
        cat.kids.back() = r;
        last = REP;
        continue;
      }
      bool is_flags = false;
      Node a = parse_atom(f, depth, is_flags);
      if (is_flags) {
        last = FLAGS;
        continue;
      }
      cat.kids.push_back(a);
      last = ATOM;
    }
    alts.push_back(cat);
    if (alts.size() == 1) return alts[0];
    Node n;
    n.k = Node::Alt;
    n.kids = alts;
    return n;
  }

  uint32_t parse_count(size_t at) {
    if (!(peek() >= '0' && peek() <= '9')) invalid("invalid repetition count", at);
    uint64_t v = 0;
    while (peek() >= '0' && peek() <= '9') {
      v = v * 10 + (uint64_t)(peek() - '0');
      if (v > 0xFFFFFFFFu) invalid("repetition count overflows", at);
      pos_++;
    }
    return (uint32_t)v;
  }
  void parse_repetition(Node& r) {
    const size_t at = pos_;
    const char c = p_[pos_++];
    if (c == '*') r.mn = 0, r.mx = -1;
    else if (c == '+') r.mn = 1, r.mx = -1;
    else if (c == '?') r.mn = 0, r.mx = 1;
    else {
      if (peek() == ',') unsupported("the repetition {,m}");
      const uint32_t lo = parse_count(at);
      uint32_t hi = lo;
      bool unbounded = false;
      if (peek() == ',') {
        pos_++;
        if (peek() == '}') unbounded = true;
        else hi = parse_count(at);
      }
      if (peek() != '}') invalid("unclosed counted repetition", at);
      pos_++;
      if (!unbounded && lo > hi) invalid("invalid repetition range {" + std::to_string(lo) + "," + std::to_string(hi) + "}", at);
      if (lo > 1000 || (!unbounded && hi > 1000)) unsupported("a repetition count above 1000");
      r.mn = (int)lo;
      r.mx = unbounded ? -1 : (int)hi;
    }
    if (peek() == '?') {  // lazy: the same is_match, another leftmost-first span
      pos_++;
      r.greedy = false;
    }
  }

  Node parse_atom(Flags& f, int depth, bool& is_flags) {
    const size_t at = pos_;
    const char c = peek();
    if (c == '(') return parse_group(f, depth, is_flags);
    if (c == '[') {
      pos_++;
      return set_node(parse_class(f, at, depth + 1));
    }
    if (c == '.') {
      pos_++;
      return set_node(f.s ? CpSet{{0, 0x10FFFF}} : CpSet{{0, 9}, {11, 0x10FFFF}});
    }
    if (c == '^' || c == '$') {
      pos_++;
      Node n;
      n.k = c == '^' ? Node::Start : Node::End;
      return n;
    }
    if (c == '\\') {
      pos_++;
      Node n;
      CpSet s;
      uint32_t cp = 0;
      const int kind = parse_escape(at, false, s, cp, &n);
      if (kind == 2) return n;
      if (kind == 1) return set_node(s);
      return literal(cp, f);
    }
    return literal(next_cp(), f);
  }

  Node parse_group(Flags& f, int depth, bool& is_flags) {
    const size_t at = pos_;
    pos_++;
    Flags inner = f;
    if (peek() == '?') {
      pos_++;
      if (peek() == 'P' || peek() == '<') {
        if (peek() == 'P') pos_++;
        if (peek() == '=' || peek() == '!') invalid("look-around is not supported", at);
        if (peek() != '<') invalid("unrecognized group syntax", at);
        pos_++;
        const size_t nb = pos_;
        while (!eof() && peek() != '>') pos_++;
        if (eof()) invalid("unclosed capture group name", at);
        const std::string name = p_.substr(nb, pos_ - nb);
        pos_++;
        bool ok = !name.empty() && (isalpha((unsigned char)name[0]) || name[0] == '_');
        for (char ch : name) ok = ok && (isalnum((unsigned char)ch) || ch == '_' || ch == '.' || ch == '[' || ch == ']');
        if (!ok) invalid("invalid capture group name '" + name + "'", nb);
        if (!names_.insert(name).second) invalid("duplicate capture group name '" + name + "'", nb);
      } else if (peek() == '=' || peek() == '!') {
        invalid("look-around is not supported", at);
      } else {
        // flags: (?flags) for the rest of the enclosing group, (?flags:...) for this group only
        bool neg = false, any = false, dangling = false;
        std::string seen;
        while (!eof() && peek() != ':' && peek() != ')') {
          const char ch = p_[pos_];
          if (ch == '-') {
            if (neg) invalid("repeated negation in flags", pos_);
            neg = true;
            dangling = true;
            pos_++;
            continue;
          }
          if (seen.find(ch) != std::string::npos) invalid(std::string("duplicate flag '") + ch + "'", pos_);
          seen += ch;
          if (ch == 'i') inner.i = !neg;
          else if (ch == 's') inner.s = !neg;
          else if (ch == 'm' || ch == 'x' || ch == 'U' || ch == 'u' || ch == 'R') unsupported(std::string("the flag '") + ch + "'");
          else invalid(std::string("unrecognized flag '") + ch + "'", pos_);
          any = true;
          dangling = false;
          pos_++;
        }
        if (eof()) invalid("unclosed group", at);
        if (dangling || (!any && peek() == ')')) invalid("expected a flag", pos_);  // (?:...) is a plain non-capturing group
        if (peek() == ')') {
          pos_++;
          f = inner;
          is_flags = true;
          return Node();
        }
        pos_++;  // ':'
      }
    }
    Node n = parse_alt(inner, depth + 1);
    if (eof()) invalid("unclosed group", at);
    pos_++;  // ')'
    return n;
  }

  // After a backslash.  Returns 0 with a literal code point in cp, 1 with a set in s, 2 with an assertion node in *assert_node
  int parse_escape(size_t at, bool in_class, CpSet& s, uint32_t& cp, Node* assert_node) {
    if (eof()) invalid("incomplete escape sequence", at);
    const char c = p_[pos_];
    switch (c) {
      case 'd': case 'D': case 's': case 'S': {
        pos_++;
        const bool digit = c == 'd' || c == 'D';
        s = digit ? cp_table(kUnicodeNd, kUnicodeNd_N) : cp_table(kUnicodeWhiteSpace, kUnicodeWhiteSpace_N);
        if (c == 'D' || c == 'S') s = cp_negate(s);
        return 1;
      }
      case 'w': case 'W': unsupported(std::string("\\") + c + " (Unicode word characters)");
      case 'b': case 'B': unsupported(std::string("\\") + c + " (word boundary assertion)");
      case '<': case '>': unsupported(std::string("\\") + c + " (word boundary assertion)");
      case 'p': case 'P': unsupported(std::string("\\") + c + "{...} (Unicode property class)");
      case 'A': case 'z': {
        if (in_class) invalid(std::string("\\") + c + " is not allowed in a character class", at);
        pos_++;
        assert_node->k = c == 'A' ? Node::Start : Node::End;
        return 2;
      }
      case 'n': pos_++; cp = '\n'; return 0;
      case 't': pos_++; cp = '\t'; return 0;
      case 'r': pos_++; cp = '\r'; return 0;
      case 'f': pos_++; cp = '\f'; return 0;
      case 'v': pos_++; cp = '\v'; return 0;
      case 'a': pos_++; cp = 7; return 0;
      case 'x': case 'u': case 'U': {
        pos_++;
        const int fixed = c == 'x' ? 2 : c == 'u' ? 4 : 8;
        uint64_t v = 0;
        auto hexv = [](char h) { return h >= '0' && h <= '9' ? h - '0' : h >= 'a' && h <= 'f' ? h - 'a' + 10 : h >= 'A' && h <= 'F' ? h - 'A' + 10 : -1; };
        if (peek() == '{') {
          pos_++;
          int n = 0;
          while (!eof() && peek() != '}') {
            const int d = hexv(peek());
            if (d < 0) invalid("invalid hexadecimal escape", at);
            v = std::min<uint64_t>(v * 16 + (uint64_t)d, 0x110000);  // any number of digits; the value is checked below
            n++;
            pos_++;
          }
          if (eof() || n == 0) invalid("invalid hexadecimal escape", at);
          pos_++;
        } else {
          for (int i = 0; i < fixed; i++) {
            const int d = hexv(peek());
            if (d < 0) invalid("invalid hexadecimal escape", at);
            v = v * 16 + (uint64_t)d;
            pos_++;
          }
        }
        if (v > 0x10FFFF || (v >= 0xD800 && v <= 0xDFFF)) invalid("escape is not a Unicode scalar value", at);
        cp = (uint32_t)v;
        return 0;
      }
      default: break;
    }
    const unsigned char uc = (unsigned char)c;
    if (uc < 0x80 && !isalnum(uc)) {  // any ASCII punctuation, symbol, space or control escapes to itself
      pos_++;
      cp = uc;
      return 0;
    }
    if (c >= '0' && c <= '9') invalid("backreferences and octal escapes are not supported", at);
    invalid("unrecognized escape sequence", at);
  }

  // after '[': a bracket class, folded under i before it is negated
  CpSet parse_class(const Flags& f, size_t at, int depth) {
    check_nest(depth);
    bool neg = false;
    if (peek() == '^') {
      neg = true;
      pos_++;
    }
    CpSet set;
    bool first = true;
    for (;;) {
      if (eof()) invalid("unclosed character class", at);
      const char c = peek();
      if (c == ']' && !first) {
        pos_++;
        break;
      }
      first = false;
      if ((c == '&' && peek(1) == '&') || (c == '-' && peek(1) == '-') || (c == '~' && peek(1) == '~'))
        unsupported(std::string("the class set operation '") + c + c + "'");
      if (c == '[') {
        if (peek(1) == ':') {
          const size_t close = p_.find(":]", pos_ + 2);
          if (close != std::string::npos) {
            std::string name = p_.substr(pos_ + 2, close - pos_ - 2);
            bool pneg = false;
            if (!name.empty() && name[0] == '^') {
              pneg = true;
              name = name.substr(1);
            }
            CpSet ps;
            if (posix_class(name, ps)) {
              pos_ = close + 2;
              // like every class item: folded under i before it is negated ([[:^lower:]] under i excludes 'A' too)
              ps = cp_normalize(ps);
              if (f.i) ps = cp_fold(ps);
              if (pneg) ps = cp_negate(ps);
              set.insert(set.end(), ps.begin(), ps.end());
              continue;
            }
          }
        }
        const size_t nat = pos_;
        pos_++;
        CpSet inner = parse_class(f, nat, depth + 1);
        set.insert(set.end(), inner.begin(), inner.end());
        continue;
      }
      CpSet item;
      uint32_t lo = 0;
      const size_t iat = pos_;
      if (class_item(item, lo)) {
        // a class such as \d cannot start a range (Rust: a range endpoint must be a single literal)
        if (peek() == '-' && peek(1) != ']' && pos_ + 1 < p_.size() && peek(1) != '-') invalid("invalid range start in a character class", iat);
        set.insert(set.end(), item.begin(), item.end());
        continue;
      }
      uint32_t hi = lo;
      if (peek() == '-' && peek(1) != ']' && pos_ + 1 < p_.size()) {
        if (peek(1) == '-') unsupported("the class set operation '--'");
        pos_++;
        const size_t hat = pos_;
        if (peek() == '[') invalid("invalid range end in a character class", hat);
        CpSet hs;
        if (class_item(hs, hi)) invalid("invalid range end in a character class", hat);
        if (hi < lo) invalid("invalid character class range (start above end)", iat);
      }
      if (f.i && (lo >= 0x80 || hi >= 0x80)) unsupported("case-insensitive matching of the non-ASCII character " + cp_name(lo >= 0x80 ? lo : hi));
      set.push_back({lo, hi});
    }
    set = cp_normalize(set);
    if (f.i) set = cp_fold(set);
    if (neg) set = cp_negate(set);
    return set;
  }
  // one class member: true with a set (\d, \s, ...), false with a code point
  bool class_item(CpSet& s, uint32_t& cp) {
    if (peek() == '\\') {
      const size_t at = pos_;
      pos_++;
      Node dummy;
      return parse_escape(at, true, s, cp, &dummy) == 1;
    }
    cp = next_cp();
    return false;
  }
  static bool posix_class(const std::string& n, CpSet& s) {
    if (n == "alnum") s = {{'0', '9'}, {'A', 'Z'}, {'a', 'z'}};
    else if (n == "alpha") s = {{'A', 'Z'}, {'a', 'z'}};
    else if (n == "ascii") s = {{0, 0x7F}};
    else if (n == "blank") s = {{'\t', '\t'}, {' ', ' '}};
    else if (n == "cntrl") s = {{0, 0x1F}, {0x7F, 0x7F}};
    else if (n == "digit") s = {{'0', '9'}};
    else if (n == "graph") s = {{'!', '~'}};
    else if (n == "lower") s = {{'a', 'z'}};
    else if (n == "print") s = {{' ', '~'}};
    else if (n == "punct") s = {{'!', '/'}, {':', '@'}, {'[', '`'}, {'{', '~'}};
    else if (n == "space") s = {{'\t', '\r'}, {' ', ' '}};
    else if (n == "upper") s = {{'A', 'Z'}};
    else if (n == "word") s = {{'0', '9'}, {'A', 'Z'}, {'_', '_'}, {'a', 'z'}};
    else if (n == "xdigit") s = {{'0', '9'}, {'A', 'F'}, {'a', 'f'}};
    else return false;
    return true;
  }
};

// ---- NFA over bytes ------------------------------------------------------------------------------------------------------
struct NState {
  enum Kind : uint8_t { Byte, Split, Eps, Start, End, Match } k;
  uint8_t lo = 0, hi = 0;
  int a = -1, b = -1;
};

// kMatch: the is_match NFA (split order is irrelevant there).  kForward: the same language with every split in priority
// order, lazy repetitions preferring to stop, and the Rust `regex` crate's shapes for repetitions (below).  kReverse: the
// reversed language (concatenations and UTF-8 sequences backwards, ^ and $ swapped), read from a match end backwards.
enum NfaMode { kNfaMatch, kNfaForward, kNfaReverse };

class NfaBuilder {
 public:
  std::vector<NState> st;
  explicit NfaBuilder(const Parser& p, NfaMode mode = kNfaMatch) : p_(p), mode_(mode) {}

  int add(NState::Kind k, int a = -1, int b = -1, uint8_t lo = 0, uint8_t hi = 0) {
    if (st.size() >= kMaxNfa) p_.unsupported("a pattern this large (its automaton exceeds " + std::to_string(kMaxNfa) + " NFA states)");
    NState s;
    s.k = k;
    s.a = a;
    s.b = b;
    s.lo = lo;
    s.hi = hi;
    st.push_back(s);
    return (int)st.size() - 1;
  }
  static bool compiles_to_nothing(const Node& n) {
    if (n.k == Node::Empty) return true;
    if (n.k == Node::Cat) {
      for (auto& k : n.kids)
        if (!compiles_to_nothing(k)) return false;
      return true;
    }
    if (n.k == Node::Rep) return n.mx == 0 || compiles_to_nothing(n.kids[0]);
    return false;
  }
  // Rust's minimum_len() == 0: a repetition of such a body is compiled as (x+)? in priority order
  static bool possibly_empty(const Node& n) {
    switch (n.k) {
      case Node::Set: return false;
      case Node::Cat:
        for (auto& k : n.kids)
          if (!possibly_empty(k)) return false;
        return true;
      case Node::Alt:
        for (auto& k : n.kids)
          if (possibly_empty(k)) return true;
        return false;
      case Node::Rep: return n.mn == 0 || possibly_empty(n.kids[0]);
      default: return true;
    }
  }
  // a split preferring `first` (greedy) or `second` (lazy)
  int prio_split(bool greedy, int first, int second) { return greedy ? add(NState::Split, first, second) : add(NState::Split, second, first); }
  // x+ in priority order: x, then a split between x again (its start) and `next`
  int compile_plus(const Node& r, int next) {
    const int loop = prio_split(r.greedy, -1, next);
    const int body = compile(r.kids[0], loop);
    (r.greedy ? st[(size_t)loop].a : st[(size_t)loop].b) = body;
    return body;
  }
  // repetitions in priority order, shaped like the Rust regex crate's Thompson compiler: x{n,m} is n copies of x, then m - n
  // nested optional copies; x{n,} with n >= 1 is n - 1 copies, then x+; x* is a loop, or (x+)? when x can match empty
  int compile_rep_ordered(const Node& n, int next) {
    const Node& x = n.kids[0];
    int cont = next;
    if (n.mx < 0) {
      if (n.mn == 0) {
        if (possibly_empty(x)) return prio_split(n.greedy, compile_plus(n, next), next);
        const int loop = prio_split(n.greedy, -1, next);
        const int body = compile(x, loop);
        (n.greedy ? st[(size_t)loop].a : st[(size_t)loop].b) = body;
        return loop;
      }
      cont = compile_plus(n, next);
      for (int k = 1; k < n.mn; k++) cont = compile(x, cont);
      return cont;
    }
    for (int k = 0; k < n.mx - n.mn; k++) cont = prio_split(n.greedy, compile(x, cont), next);
    for (int k = 0; k < n.mn; k++) cont = compile(x, cont);
    return cont;
  }
  int compile(const Node& n, int next) {
    const bool rev = mode_ == kNfaReverse;
    switch (n.k) {
      case Node::Empty: return next;
      case Node::Start: return add(rev ? NState::End : NState::Start, next);
      case Node::End: return add(rev ? NState::Start : NState::End, next);
      case Node::Cat:
        if (rev) {
          for (size_t i = 0; i < n.kids.size(); i++) next = compile(n.kids[i], next);
        } else {
          for (size_t i = n.kids.size(); i-- > 0;) next = compile(n.kids[i], next);
        }
        return next;
      case Node::Alt: {
        int entry = compile(n.kids.back(), next);
        for (size_t i = n.kids.size() - 1; i-- > 0;) entry = add(NState::Split, compile(n.kids[i], next), entry);
        return entry;
      }
      case Node::Rep: {
        const Node& x = n.kids[0];
        // a body that compiles to no state repeats to nothing: without this, nested counts ((?:){1000}){1000}... would
        // loop without adding a state, so the state cap would never stop them
        if (n.mx == 0 || compiles_to_nothing(x)) return next;
        if (mode_ == kNfaForward) return compile_rep_ordered(n, next);
        int cont = next;
        if (n.mx < 0) {
          const int loop = add(NState::Split, -1, next);
          const int body = compile(x, loop);
          st[(size_t)loop].a = body;
          cont = loop;
        } else {
          for (int k = 0; k < n.mx - n.mn; k++) cont = add(NState::Split, compile(x, cont), next);
        }
        for (int k = 0; k < n.mn; k++) cont = compile(x, cont);
        return cont;
      }
      case Node::Set: {
        std::vector<ByteSeq> seqs;
        for (auto& r : n.set) utf8_sequences(r.first, r.second, seqs);
        if (seqs.empty()) return add(NState::Eps, -1);  // matches nothing
        int entry = -1;
        for (size_t i = seqs.size(); i-- > 0;) {
          int s = next;
          const size_t len = seqs[i].size();
          for (size_t k = 0; k < len; k++) {
            const size_t j = rev ? k : len - 1 - k;
            s = add(NState::Byte, s, -1, seqs[i][j].first, seqs[i][j].second);
          }
          entry = entry < 0 ? s : add(NState::Split, s, entry);
        }
        return entry;
      }
    }
    return next;
  }

 private:
  static const size_t kMaxNfa = 1 << 18;
  const Parser& p_;
  NfaMode mode_;
};

// ---- subset construction ---------------------------------------------------------------------------------------------------
// byte equivalence classes: bytes no Byte state tells apart.  Writes the 256-entry byte -> class map as the blob's head and
// one representative byte per class; returns the number of classes.
inline uint32_t byte_classes(const std::vector<NState>& nfa, std::vector<uint8_t>& blob, std::vector<uint8_t>& rep) {
  bool brk[257] = {false};
  for (auto& s : nfa)
    if (s.k == NState::Byte) brk[s.lo] = brk[(int)s.hi + 1] = true;
  blob.assign(256, 0);
  uint32_t cls = 0;
  for (int b = 0; b < 256; b++) {
    if (b > 0 && brk[b]) cls++;
    blob[(size_t)b] = (uint8_t)cls;
    if (rep.size() == cls) rep.push_back((uint8_t)b);
  }
  return cls + 1;
}

class DfaBuilder {
 public:
  DfaBuilder(const std::vector<NState>& nfa, int start, const Parser& p) : nfa_(nfa), start_(start), p_(p), mark_(nfa.size(), 0) {}

  Dfa build() {
    Dfa d;
    std::vector<uint8_t> rep;
    d.n_cls = byte_classes(nfa_, d.blob, rep);
    n_cls_ = d.n_cls;
    keys_.clear();
    states_.clear();
    states_.push_back({{}, false});  // dead
    states_.push_back({{}, false});  // matched
    std::vector<int> fr;
    bool matched = closure({start_}, true, false, fr);
    d.start = matched ? kMatched : intern(fr, true);
    std::vector<uint16_t> trans;
    for (size_t i = 0; i < states_.size(); i++) {
      if (i <= kMatched) {
        for (uint32_t c = 0; c < d.n_cls; c++) trans.push_back((uint16_t)i);
        continue;
      }
      for (uint32_t c = 0; c < d.n_cls; c++) {
        std::vector<int> seed;
        for (int s : states_[i].fr)
          if (nfa_[(size_t)s].k == NState::Byte && rep[c] >= nfa_[(size_t)s].lo && rep[c] <= nfa_[(size_t)s].hi) seed.push_back(nfa_[(size_t)s].a);
        seed.push_back(start_);  // unanchored: a match may begin at every byte
        std::vector<int> nf;
        const bool m = closure(seed, false, false, nf);
        trans.push_back((uint16_t)(m ? kMatched : intern(nf, false)));
      }
    }
    d.n_states = (uint32_t)states_.size();
    d.blob.resize(dfa_trans_offset(d.n_states), 0);
    d.blob[256 + kMatched] = 1;
    for (size_t i = 2; i < states_.size(); i++) {
      std::vector<int> ignored;
      d.blob[256 + i] = closure(states_[i].fr, states_[i].at_start, true, ignored) ? 1 : 0;
    }
    const size_t off = d.blob.size();
    d.blob.resize(off + trans.size() * 2);
    memcpy(d.blob.data() + off, trans.data(), trans.size() * 2);
    return d;
  }

 private:
  struct DState {
    std::vector<int> fr;  // sorted Byte and (unpassed) End states
    bool at_start;
  };
  const std::vector<NState>& nfa_;
  int start_;
  const Parser& p_;
  std::vector<uint32_t> mark_;
  uint32_t gen_ = 0;
  uint32_t n_cls_ = 1;
  uint64_t work_ = 0;  // closure steps: bounds the construction's time, not only the table's size
  static const uint64_t kMaxWork = (uint64_t)1 << 25;
  std::map<std::pair<bool, std::vector<int>>, uint32_t> keys_;
  std::vector<DState> states_;

  uint32_t intern(const std::vector<int>& fr, bool at_start) {
    if (fr.empty()) return kDead;
    auto key = std::make_pair(at_start, fr);
    auto it = keys_.find(key);
    if (it != keys_.end()) return it->second;
    const uint32_t id = (uint32_t)states_.size();
    if (id >= kMaxStates) p_.unsupported("a pattern whose DFA exceeds " + std::to_string(kMaxStates) + " states");
    if ((uint64_t)(id + 1) * n_cls_ * 2 > kMaxTransBytes)
      p_.unsupported("a pattern whose DFA table exceeds 1 MiB (over " + std::to_string(id) + " states x " + std::to_string(n_cls_) + " byte classes)");
    states_.push_back({fr, at_start});
    keys_[key] = id;
    return id;
  }
  // epsilon closure of `seed`; fills the frontier (Byte states, and End states unless at_end) and says whether Match is reached
  bool closure(const std::vector<int>& seed, bool at_start, bool at_end, std::vector<int>& fr) {
    gen_++;
    fr.clear();
    bool matched = false;
    std::vector<int> stack(seed.rbegin(), seed.rend());
    while (!stack.empty()) {
      const int s = stack.back();
      stack.pop_back();
      if (++work_ > kMaxWork) p_.unsupported("a pattern this expensive to compile (its DFA construction exceeds " + std::to_string(kMaxWork) + " steps)");
      if (s < 0 || mark_[(size_t)s] == gen_) continue;
      mark_[(size_t)s] = gen_;
      const NState& n = nfa_[(size_t)s];
      switch (n.k) {
        case NState::Byte: fr.push_back(s); break;
        case NState::Match: matched = true; break;
        case NState::Eps: stack.push_back(n.a); break;
        case NState::Split:
          stack.push_back(n.b);
          stack.push_back(n.a);
          break;
        case NState::Start:
          if (at_start) stack.push_back(n.a);
          break;
        case NState::End:
          if (at_end) stack.push_back(n.a);
          else fr.push_back(s);
          break;
      }
    }
    std::sort(fr.begin(), fr.end());
    return matched;
  }
};

// ---- span DFAs (regexp_count, regexp_replace) ---------------------------------------------------------------------------
// The same blob layout as the is_match DFA, but no state is absorbing: a flags byte per state (kSpanHere, kSpanAtEdge),
// state 0 dead, states 1 and 2 the two start states (kSpanStartEdge, kSpanStartInside).
//   forward (kNfaForward NFA, unanchored): the state after reading s[pos..i) is the ordered thread list of a Pike VM
//     running leftmost-first.  The closure follows splits in priority order and stops at the first Match: every thread of
//     lower priority, the restart of the unanchored search included, is dropped.  The restart (a new match beginning at
//     the next byte) is a flag of the state, the last item of the list; once any match was seen it is gone for good.
//     kSpanHere: a match ends at i; kSpanAtEdge: a match ends at i if i is the end of the text.  Start states: at
//     offset 0 (^ holds) or not.
//   reverse (kNfaReverse NFA, anchored at the match end, every thread kept): the state after reading s[j..end) backwards.
//     kSpanHere: s[j..end) matches; kSpanAtEdge: it matches if j is offset 0 (the original ^ holds).  Start states: the
//     walk begins at the end of the text (the original $ holds) or not.
class SpanDfaBuilder {
 public:
  SpanDfaBuilder(const std::vector<NState>& nfa, int start, const Parser& p, bool forward)
      : nfa_(nfa), start_(start), p_(p), forward_(forward), mark_(nfa.size(), 0) {}

  Dfa build() {
    Dfa d;
    std::vector<uint8_t> rep;
    d.n_cls = byte_classes(nfa_, d.blob, rep);
    n_cls_ = d.n_cls;
    states_.push_back(SState());  // dead
    std::vector<int> fr;
    // a restart that reaches nothing (every match needs ^) is left out, so such a search stops at its first dead end
    const bool restart_useful = forward_ && (closure({start_}, false, false, fr) || !fr.empty());
    for (int k = 0; k < 2; k++) {  // kSpanStartEdge, kSpanStartInside: always their own slots
      const bool edge = k == 0;
      const bool m = closure({start_}, edge, false, fr);
      add_state(fr, edge, m, restart_useful && !m);
    }
    std::vector<uint16_t> trans;
    for (size_t i = 0; i < states_.size(); i++) {
      for (uint32_t c = 0; c < d.n_cls; c++) {
        if (i == kDead) {
          trans.push_back((uint16_t)kDead);
          continue;
        }
        std::vector<int> seed;
        for (int s : states_[i].fr)
          if (nfa_[(size_t)s].k == NState::Byte && rep[c] >= nfa_[(size_t)s].lo && rep[c] <= nfa_[(size_t)s].hi) seed.push_back(nfa_[(size_t)s].a);
        const bool restart = states_[i].restart;
        if (restart) seed.push_back(start_);  // lowest priority: a match beginning at the next byte
        std::vector<int> nf;
        const bool m = closure(seed, false, false, nf);
        trans.push_back((uint16_t)intern(nf, false, m, restart && !m));
      }
    }
    d.n_states = (uint32_t)states_.size();
    d.start = kSpanStartEdge;
    d.blob.resize(dfa_trans_offset(d.n_states), 0);
    for (size_t i = 1; i < states_.size(); i++) d.blob[256 + i] = states_[i].flags;
    const size_t off = d.blob.size();
    d.blob.resize(off + trans.size() * 2);
    memcpy(d.blob.data() + off, trans.data(), trans.size() * 2);
    return d;
  }

 private:
  struct SState {
    std::vector<int> fr;  // Byte and (unpassed) End states: in priority order (forward) or sorted (reverse)
    bool at_start = false, matched = false, restart = false;
    uint8_t flags = 0;
  };
  typedef std::pair<std::vector<int>, int> Key;
  const std::vector<NState>& nfa_;
  int start_;
  const Parser& p_;
  bool forward_;
  std::vector<uint32_t> mark_;
  uint32_t gen_ = 0;
  uint32_t n_cls_ = 1;
  uint64_t work_ = 0;
  static const uint64_t kMaxWork = (uint64_t)1 << 25;
  std::map<Key, uint32_t> keys_;
  std::vector<SState> states_;

  uint32_t add_state(const std::vector<int>& fr, bool at_start, bool matched, bool restart) {
    const uint32_t id = (uint32_t)states_.size();
    if (id >= kMaxStates) p_.unsupported("a pattern whose DFA exceeds " + std::to_string(kMaxStates) + " states");
    if ((uint64_t)(id + 1) * n_cls_ * 2 > kMaxTransBytes)
      p_.unsupported("a pattern whose DFA table exceeds 1 MiB (over " + std::to_string(id) + " states x " + std::to_string(n_cls_) + " byte classes)");
    SState s;
    s.fr = fr;
    s.at_start = at_start;
    s.matched = matched;
    s.restart = restart;
    std::vector<int> ignored;
    s.flags = (uint8_t)((matched ? kSpanHere : 0) | ((matched || closure(fr, at_start, true, ignored)) ? kSpanAtEdge : 0));
    states_.push_back(s);
    keys_.emplace(Key(fr, (at_start ? 1 : 0) | (matched ? 2 : 0) | (restart ? 4 : 0)), id);
    return id;
  }
  uint32_t intern(const std::vector<int>& fr, bool at_start, bool matched, bool restart) {
    if (fr.empty() && !matched && !restart) return kDead;
    auto it = keys_.find(Key(fr, (at_start ? 1 : 0) | (matched ? 2 : 0) | (restart ? 4 : 0)));
    if (it != keys_.end()) return it->second;
    return add_state(fr, at_start, matched, restart);
  }
  // epsilon closure of `seed`, each seed in turn and depth first along the splits' priority.  Forward: stops at the first
  // Match (the threads after it lose to it).  Reverse: explores everything and sorts the frontier.  Says whether Match
  // was reached.
  bool closure(const std::vector<int>& seed, bool at_start, bool at_end, std::vector<int>& fr) {
    gen_++;
    fr.clear();
    bool matched = false;
    std::vector<int> stack;
    for (int sd : seed) {
      stack.assign(1, sd);
      while (!stack.empty()) {
        const int s = stack.back();
        stack.pop_back();
        if (++work_ > kMaxWork) p_.unsupported("a pattern this expensive to compile (its DFA construction exceeds " + std::to_string(kMaxWork) + " steps)");
        if (s < 0 || mark_[(size_t)s] == gen_) continue;
        mark_[(size_t)s] = gen_;
        const NState& n = nfa_[(size_t)s];
        switch (n.k) {
          case NState::Byte: fr.push_back(s); break;
          case NState::Match:
            matched = true;
            if (forward_) return true;
            break;
          case NState::Eps: stack.push_back(n.a); break;
          case NState::Split:
            stack.push_back(n.b);
            stack.push_back(n.a);
            break;
          case NState::Start:
            if (at_start) stack.push_back(n.a);
            break;
          case NState::End:
            if (at_end) stack.push_back(n.a);
            else fr.push_back(s);
            break;
        }
      }
    }
    if (!forward_) std::sort(fr.begin(), fr.end());
    return matched;
  }
};

inline Dfa compile_node(const Parser& p, const Node& root) {
  NfaBuilder nb(p);
  const int match = nb.add(NState::Match);
  const int start = nb.compile(root, match);
  DfaBuilder db(nb.st, start, p);
  return db.build();
}

// Compiles `pattern` under the flags i (ci) and s (dotall).  Returns RX_OK, RX_INVALID or RX_UNSUPPORTED; err names the
// pattern and the construct or byte offset.
inline int compile_regex(const std::string& pattern, bool ci, bool dotall, Dfa& out, std::string& err) {
  try {
    Parser p(pattern, pattern);
    Node root = p.parse(ci, dotall);
    out = compile_node(p, root);
    return RX_OK;
  } catch (const Error& e) {
    err = e.msg;
    return e.code;
  }
}

// The forward (leftmost-first, unanchored) and reverse (anchored at a match end) span DFAs of `pattern` under the flags i
// and s: what regexp_count and regexp_replace walk (dfa_next_match).  Same return codes and messages as compile_regex.
inline int compile_regex_spans(const std::string& pattern, bool ci, bool dotall, Dfa& fwd, Dfa& rev, std::string& err) {
  try {
    Parser p(pattern, pattern);
    Node root = p.parse(ci, dotall);
    for (int k = 0; k < 2; k++) {
      NfaBuilder nb(p, k == 0 ? kNfaForward : kNfaReverse);
      const int match = nb.add(NState::Match);
      const int start = nb.compile(root, match);
      SpanDfaBuilder db(nb.st, start, p, k == 0);
      (k == 0 ? fwd : rev) = db.build();
    }
    return RX_OK;
  } catch (const Error& e) {
    err = e.msg;
    return e.code;
  }
}

// The flags argument of regexp_like, regexp_count and regexp_replace (`fn` names the function): only i and s [EXT], and g
// where `global` is given (regexp_replace); the other functions refuse g as DataFusion does.
inline int parse_regex_flags(const std::string& flags, bool& ci, bool& dotall, std::string& err, const char* fn = "regexp_like",
                             bool* global = nullptr) {
  ci = dotall = false;
  if (global) *global = false;
  for (char c : flags) {
    if (c == 'i') ci = true;
    else if (c == 's') dotall = true;
    else if (c == 'g' && global) *global = true;
    else if (c == 'g') {
      err = std::string(fn) + " does not support the \"global\" option (flag 'g')";
      return RX_INVALID;
    } else if (c == 'm' || c == 'x' || c == 'U' || c == 'u' || c == 'R') {
      err = std::string(fn) + ": the flag '" + c + "' is not supported by the device engine";
      return RX_UNSUPPORTED;
    } else {
      err = std::string(fn) + ": unrecognized flag '" + c + "' in '" + flags + "'";
      return RX_INVALID;
    }
  }
  return RX_OK;
}

inline bool is_meta(char c) { return c && strchr("\\.+*?()|[]{}^$#&-~", c) != nullptr; }

// arrow-rs's translation of a LIKE pattern into a regex, matched with the flags i and s: anchored, % -> .*, _ -> ., a
// backslash escapes the next character, everything else is literal.  A trailing backslash is refused as malformed.
inline int like_to_regex(const std::string& like, std::string& out, std::string& err) {
  out = "^";
  for (size_t i = 0; i < like.size(); i++) {
    char c = like[i];
    if (c == '\\') {
      if (i + 1 == like.size()) {
        err = "ILIKE pattern '" + like + "': trailing escape character at byte offset " + std::to_string(i);
        return RX_INVALID;
      }
      c = like[++i];
      if (is_meta(c)) out += '\\';
      out += c;
      continue;
    }
    if (c == '%') out += ".*";
    else if (c == '_') out += '.';
    else {
      if (is_meta(c)) out += '\\';
      out += c;
    }
  }
  out += '$';
  return RX_OK;
}

inline int compile_ilike(const std::string& like, Dfa& out, std::string& err) {
  std::string re;
  const int rc = like_to_regex(like, re, err);
  if (rc != RX_OK) return rc;
  try {
    Parser p(re, like);
    Node root = p.parse(true, true);
    out = compile_node(p, root);
    return RX_OK;
  } catch (const Error& e) {
    err = e.code == RX_UNSUPPORTED ? "ILIKE pattern " + e.msg.substr(6) : e.msg;  // "regex '<like>': ..." -> "ILIKE pattern '<like>': ..."
    return e.code;
  }
}

}  // namespace rx
}  // namespace b200
