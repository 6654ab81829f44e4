// Drives the regex compiler and the DFA walk of csrc/common/regex_dfa.hpp on the host: the same walk the OP_REGEX device
// operation runs.  Input (argv[1]), every text hex-encoded so that any byte can travel:
//   <n>                    number of subject strings
//   <hex string>           n lines
//   <kind> <flags> <hex>   one line per pattern; kind r = regex (flags: letters or "-"), l = ILIKE pattern
// Output, one line per pattern: "<status> <states> <bits>" with one '0' / '1' per subject string, or
// "<status> <hex message>" when the compiler refused the pattern (status -1 invalid, -2 unsupported).
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

int main(int argc, char** argv) {
  if (argc < 2) return 2;
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
    b200::rx::Dfa d;
    std::string err;
    int rc;
    if (kind == "l") {
      rc = b200::rx::compile_ilike(pat, d, err);
    } else {
      bool ci = false, dotall = false;
      rc = b200::rx::parse_regex_flags(flags == "-" ? "" : flags, ci, dotall, err);
      if (rc == 0) rc = b200::rx::compile_regex(pat, ci, dotall, d, err);
    }
    if (rc != 0) {
      out += std::to_string(rc) + " " + hex(err) + "\n";
      continue;
    }
    std::string bits(n, '0');
    for (size_t i = 0; i < n; i++)
      if (d.is_match(subjects[i])) bits[i] = '1';
    out += "0 " + std::to_string(d.n_states) + " " + (n ? bits : std::string("-")) + "\n";
  }
  fwrite(out.data(), 1, out.size(), stdout);
  return 0;
}
