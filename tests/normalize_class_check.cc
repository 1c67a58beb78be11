// The C++ class's Normalize overloads on a batch (test_gpu_normalize.py builds and runs this).
// usage: normalize_class_check MODEL INPUT -- INPUT holds one sentence per line in hex; prints, per sentence, the hex of
// the batch overload's normalized text and its norm_to_orig ("-" when empty), after checking that the three
// single-sentence overloads and NormalizePacked give the same.
#include <cstdio>
#include <fstream>
#include <string>
#include <vector>

#include "host/sentencepiece_processor.h"

static std::string unhex(const std::string &h) {
  std::string s;
  for (size_t i = 0; i + 1 < h.size(); i += 2) s.push_back(static_cast<char>(std::stoi(h.substr(i, 2), nullptr, 16)));
  return s;
}

static std::string hex(const std::string &s) {
  static const char *d = "0123456789abcdef";
  std::string h;
  for (unsigned char c : s) { h.push_back(d[c >> 4]); h.push_back(d[c & 15]); }
  return h;
}

#define CHECK(c)                                                        \
  do {                                                                  \
    if (!(c)) { fprintf(stderr, "check failed: %s\n", #c); return 1; } \
  } while (0)

int main(int argc, char **argv) {
  if (argc != 3) return 2;
  sentencepiece::SentencePieceProcessor sp;
  CHECK(sp.Load(argv[1]).ok());
  std::ifstream in(argv[2]);
  std::vector<std::string> lines;
  for (std::string l; std::getline(in, l);) lines.push_back(unhex(l));
  std::vector<std::string_view> views(lines.begin(), lines.end());
  std::vector<std::string> norm, norm2;
  std::vector<std::vector<size_t>> maps;
  CHECK(sp.Normalize(views, &norm, &maps).ok());
  CHECK(sp.Normalize(views, &norm2).ok());
  CHECK(norm == norm2 && norm.size() == lines.size() && maps.size() == lines.size());
  std::string packed;
  std::vector<uint64_t> offs(1, 0);
  for (const auto &l : lines) { packed += l; offs.push_back(packed.size()); }
  const char *text;
  const uint64_t *no;
  const uint32_t *n2o;
  CHECK(sp.NormalizePacked(packed.data(), offs.data(), lines.size(), false, &text, &no, &n2o).ok() && n2o == nullptr);
  for (size_t i = 0; i < lines.size(); ++i) CHECK(std::string(text + no[i], text + no[i + 1]) == norm[i]);
  for (size_t i = 0; i < lines.size(); ++i) {
    std::string a, b;
    std::vector<size_t> m;
    CHECK(sp.Normalize(lines[i], &a, &m).ok() && a == norm[i] && m == maps[i]);
    CHECK(sp.Normalize(lines[i], &b).ok() && b == norm[i]);
    CHECK(sp.Normalize(lines[i]) == norm[i]);
    printf("%s", hex(norm[i]).c_str());
    if (maps[i].empty()) printf(" -");
    for (size_t v : maps[i]) printf(" %zu", v);
    printf("\n");
  }
  return 0;
}
