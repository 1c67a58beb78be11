// The C++ class's DecodeWithOffsets overloads on a batch (test_gpu_decode_offsets.py builds and runs this).
// usage: decode_offsets_class_check MODEL INPUT -- INPUT holds one id list per line, ids separated by spaces.  Prints,
// per list, the decoded text in hex and its tokens as "id:piece:surface:begin:end" (piece and surface in hex), all
// separated by spaces; then the same for the last list through the single-list overload, after checking that
// DecodeOffsetsPacked gives the same text and ends; then the error of a list holding the id GetPieceSize().
#include <cstdio>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "host/sentencepiece_processor.h"

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

static void print(const std::string &text, const Spans &v) {
  std::string row = hex(text);
  for (const auto &s : v)
    row += ' ' + std::to_string(s.id) + ":" + hex(s.piece) + ":" + hex(s.surface) + ":" + std::to_string(s.begin) + ":" +
           std::to_string(s.end);
  printf("%s\n", row.c_str());
}

int main(int argc, char **argv) {
  if (argc != 3) return 2;
  sentencepiece::SentencePieceProcessor sp;
  CHECK(sp.Load(argv[1]).ok());
  std::ifstream in(argv[2]);
  std::vector<std::vector<int>> lists;
  for (std::string l; std::getline(in, l);) {
    std::istringstream is(l);
    lists.emplace_back();
    for (int id; is >> id;) lists.back().push_back(id);
  }
  CHECK(!lists.empty());
  std::vector<std::string> texts;
  std::vector<Spans> all;
  CHECK(sp.DecodeWithOffsets(lists, &texts, &all).ok());
  CHECK(texts.size() == lists.size() && all.size() == lists.size());
  // the packed form: the same text and ends
  std::vector<int32_t> ids;
  std::vector<uint64_t> offs{0};
  for (const auto &l : lists) { ids.insert(ids.end(), l.begin(), l.end()); offs.push_back(ids.size()); }
  const char *text;
  const uint64_t *to;
  const uint32_t *te;
  CHECK(sp.DecodeOffsetsPacked(ids.data(), offs.data(), lists.size(), &text, &to, &te).ok());
  for (size_t i = 0; i < lists.size(); ++i) {
    CHECK(std::string(text + to[i], text + to[i + 1]) == texts[i]);
    CHECK(all[i].size() == lists[i].size());
    for (uint64_t k = offs[i]; k < offs[i + 1]; ++k) {
      const auto &s = all[i][k - offs[i]];
      CHECK(s.id == ids[k] && s.end == te[k] && s.piece == sp.IdToPiece(s.id));
    }
  }
  for (size_t i = 0; i < lists.size(); ++i) print(texts[i], all[i]);
  std::string one;
  Spans spans;
  CHECK(sp.DecodeWithOffsets(lists.back(), &one, &spans).ok());
  print(one, spans);
  const auto st = sp.DecodeWithOffsets(std::vector<int>{0, sp.GetPieceSize()}, &one, &spans);
  CHECK(!st.ok());
  std::string msg = st.ToString();
  const size_t at = msg.find("Invalid id:");
  printf("error: %s\n", at == std::string::npos ? msg.c_str() : msg.substr(at).c_str());
  return 0;
}
