// The C++ class's EncodeWithOffsets overloads on a batch (test_gpu_offsets.py builds and runs this).
// usage: offsets_class_check MODEL INPUT OPTIONS -- INPUT holds one sentence per line in hex, OPTIONS is the
// SetEncodeExtraOptions string ("-" for none).  Prints, per sentence, its tokens as "piece:id:surface:begin:end"
// (piece and surface in hex) separated by spaces, then the same for the last sentence through the single-sentence
// overload, after checking that EncodeOffsetsPacked gives the same ids and offsets.
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

using Spans = std::vector<sentencepiece::SentencePieceProcessor::PieceSpan>;

static void print(const Spans &v) {
  std::string row;
  for (const auto &s : v) {
    if (!row.empty()) row += ' ';
    row += hex(s.piece) + ":" + std::to_string(s.id) + ":" + hex(s.surface) + ":" + std::to_string(s.begin) + ":" +
           std::to_string(s.end);
  }
  printf("%s\n", row.c_str());
}

int main(int argc, char **argv) {
  if (argc != 4) return 2;
  sentencepiece::SentencePieceProcessor sp;
  CHECK(sp.Load(argv[1]).ok());
  if (std::string(argv[3]) != "-") CHECK(sp.SetEncodeExtraOptions(argv[3]).ok());
  std::ifstream in(argv[2]);
  std::vector<std::string> lines;
  for (std::string l; std::getline(in, l);) lines.push_back(unhex(l));
  CHECK(!lines.empty());
  std::vector<std::string_view> views(lines.begin(), lines.end());
  std::vector<Spans> all;
  CHECK(sp.EncodeWithOffsets(views, &all).ok());
  CHECK(all.size() == lines.size());
  // the packed form: the same tokens
  std::string bytes;
  std::vector<uint64_t> offs{0};
  for (const auto &l : lines) { bytes += l; offs.push_back(bytes.size()); }
  const int32_t *ids;
  const uint64_t *ido, *to;
  const uint32_t *b, *e, *pe;
  const char *text;
  CHECK(sp.EncodeOffsetsPacked(bytes.data(), offs.data(), lines.size(), &ids, &ido, &b, &e, &text, &to, &pe).ok());
  for (size_t i = 0; i < lines.size(); ++i) {
    CHECK(ido[i + 1] - ido[i] == all[i].size());
    for (uint64_t k = ido[i]; k < ido[i + 1]; ++k) {
      const auto &s = all[i][k - ido[i]];
      CHECK(s.id == ids[k] && s.begin == b[k] && s.end == e[k]);
    }
  }
  for (const auto &v : all) print(v);
  Spans one;
  CHECK(sp.EncodeWithOffsets(views.back(), &one).ok());
  print(one);
  return 0;
}
