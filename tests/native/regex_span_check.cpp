// Drives the span DFAs of csrc/common/regex_dfa.hpp on the host: the forward / reverse walks and the find_iter step that the
// regexp_count and regexp_replace device operations run.  Input (argv[1]) as for regex_check.cpp, every text hex-encoded:
//   <n>                    number of subject strings
//   <hex string>           n lines
//   r <flags> <hex>        one line per pattern (flags: letters or "-")
// argv[2] is the mode:
//   span <hex replacement>  one line per pattern: "0" then, per subject, "fs,fe,c1,c2,cp,crcg,lg,crc1,l1": the first
//                           match's byte span (-1,-1 when none), regexp_count from start 1, 2 and past the end (0 for an
//                           empty subject), and the CRC-32 and length of the string with every match / the first match
//                           replaced
//   blob                    one line per pattern: "0 <hex blob> <shape>" of the is_match DFA
// A refused pattern gives "<status> <hex message>" (status -1 invalid, -2 unsupported).
#include <cstdio>
#include <fstream>
#include <iostream>
#include <string>

#include "../../datafusion-ballista_b200/csrc/common/regex_dfa.hpp"

static std::string unhex(const std::string& h) {
  std::string o;
  for (size_t i = 0; i + 1 < h.size(); i += 2) o += (char)std::stoi(h.substr(i, 2), nullptr, 16);
  return o;
}
static std::string hex(const std::string& s) {
  static const char* d = "0123456789abcdef";
  std::string o;
  for (unsigned char c : s) {
    o += d[c >> 4];
    o += d[c & 15];
  }
  return o;
}
static uint32_t crc32(const uint8_t* p, size_t n) {
  uint32_t c = 0xFFFFFFFFu;
  for (size_t i = 0; i < n; i++) {
    c ^= p[i];
    for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
  }
  return ~c;
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  const std::string mode = argv[2];
  const std::string repl = argc > 3 && std::string(argv[3]) != "-" ? unhex(argv[3]) : std::string();
  std::ifstream in(argv[1]);
  size_t n = 0;
  in >> n;
  std::vector<std::string> subjects(n);
  for (size_t i = 0; i < n; i++) {
    std::string h;
    in >> h;
    subjects[i] = h == "-" ? std::string() : unhex(h);
  }
  std::string kind, flags, hp;
  std::string out;
  while (in >> kind >> flags >> hp) {
    const std::string pat = hp == "-" ? std::string() : unhex(hp);
    bool ci = false, dotall = false;
    std::string err;
    int rc = b200::rx::parse_regex_flags(flags == "-" ? "" : flags, ci, dotall, err, "regexp_count");
    if (mode == "blob") {
      b200::rx::Dfa d;
      if (rc == 0) rc = b200::rx::compile_regex(pat, ci, dotall, d, err);
      if (rc != 0) {
        out += std::to_string(rc) + " " + hex(err) + "\n";
        continue;
      }
      out += "0 " + hex(std::string(d.blob.begin(), d.blob.end())) + " " + std::to_string(d.shape()) + "\n";
      continue;
    }
    b200::rx::Dfa fwd, rev;
    if (rc == 0) rc = b200::rx::compile_regex_spans(pat, ci, dotall, fwd, rev, err);
    if (rc != 0) {
      out += std::to_string(rc) + " " + hex(err) + "\n";
      continue;
    }
    const b200::rx::RxSpans sp = {fwd.blob.data(), fwd.shape(), rev.blob.data(), rev.shape()};
    out += "0";
    std::vector<uint8_t> buf;
    for (const std::string& str : subjects) {
      const uint8_t* s = (const uint8_t*)str.data();
      const uint32_t len = (uint32_t)str.size();
      b200::rx::RxIter it = {0, -1};
      uint32_t ms = 0, me = 0;
      const bool any = b200::rx::dfa_next_match(sp, s, len, it, &ms, &me);
      uint32_t counts[3];
      const int64_t starts[3] = {1, 2, 1 << 30};
      for (int k = 0; k < 3; k++) counts[k] = b200::rx::regexp_count_row(sp, s, len, starts[k] - 1);
      std::string reps;
      for (int g = 1; g >= 0; g--) {
        const uint8_t* r = (const uint8_t*)repl.data();
        const uint64_t need = b200::rx::dfa_replace(sp, s, len, r, (uint32_t)repl.size(), g != 0, nullptr);
        buf.assign(need + 1, 0);
        const uint64_t wrote = b200::rx::dfa_replace(sp, s, len, r, (uint32_t)repl.size(), g != 0, buf.data());
        if (wrote != need) return 3;
        reps += "," + std::to_string(crc32(buf.data(), need)) + "," + std::to_string(need);
      }
      out += " " + (any ? std::to_string(ms) + "," + std::to_string(me) : std::string("-1,-1")) + "," + std::to_string(counts[0]) + "," +
             std::to_string(counts[1]) + "," + std::to_string(counts[2]) + reps;
    }
    out += "\n";
  }
  fwrite(out.data(), 1, out.size(), stdout);
  return 0;
}
