// decode_offsets_reference.cc -- what the unmodified reference's SentencePieceProcessor::Decode(const std::vector<int>&,
// SentencePieceText*) returns for each id list (src/sentencepiece_processor.cc:766-925), the source of
// tests/golden/reference_digests_decode_offsets.json.  tools/record_decode_offsets_reference.py builds it against the
// reference library that oracle/Makefile compiles into oracle/_ref and runs it; it is never part of the product or of
// a test run.
// usage: decode_offsets_reference MODEL INPUT -- INPUT holds one id list per line, ids separated by spaces.  Prints, per
// list, the decoded text in hex and then its pieces as "id:piece:surface:begin:end" (piece and surface in hex), all
// separated by spaces.  Fails when a piece's id is not the input id, its surface is not text[begin, end), or it does
// not begin where the piece before it ends (0 for the first).
#include <cstdio>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "sentencepiece.pb.h"
#include "sentencepiece_processor.h"

static std::string hex(const std::string &s) {
  static const char *d = "0123456789abcdef";
  std::string h;
  for (unsigned char c : s) { h.push_back(d[c >> 4]); h.push_back(d[c & 15]); }
  return h;
}

int main(int argc, char **argv) {
  if (argc != 3) return 2;
  sentencepiece::SentencePieceProcessor sp;
  if (!sp.Load(argv[1]).ok()) { fprintf(stderr, "cannot load %s\n", argv[1]); return 1; }
  std::ifstream in(argv[2]);
  size_t line = 0;
  for (std::string l; std::getline(in, l); ++line) {
    std::vector<int> ids;
    std::istringstream is(l);
    for (int id; is >> id;) ids.push_back(id);
    sentencepiece::SentencePieceText spt;
    if (!sp.Decode(ids, &spt).ok()) { fprintf(stderr, "decode failed on line %zu\n", line); return 1; }
    const std::string &text = spt.text();
    if (static_cast<size_t>(spt.pieces_size()) != ids.size()) { fprintf(stderr, "line %zu: piece count\n", line); return 1; }
    std::string row = hex(text);
    uint32_t prev = 0;
    for (int k = 0; k < spt.pieces_size(); ++k) {
      const auto &p = spt.pieces(k);
      if (p.id() != ids[k] || p.begin() != prev || p.end() < p.begin() || p.end() > text.size() ||
          p.surface() != text.substr(p.begin(), p.end() - p.begin())) {
        fprintf(stderr, "line %zu, piece %d: id, tiling or surface check failed\n", line, k);
        return 1;
      }
      prev = p.end();
      row += ' ' + std::to_string(p.id()) + ":" + hex(p.piece()) + ":" + hex(p.surface()) + ":" +
             std::to_string(p.begin()) + ":" + std::to_string(p.end());
    }
    printf("%s\n", row.c_str());
  }
  return 0;
}
