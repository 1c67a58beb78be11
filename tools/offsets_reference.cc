// offsets_reference.cc -- what the unmodified reference's SentencePieceProcessor::Encode(absl::string_view,
// SentencePieceText*) returns for each input (src/sentencepiece_processor.cc:547-636 and ApplyExtraOptions,
// :1019-1064), the source of tests/golden/reference_digests_offsets.json.  tools/record_offsets_reference.py builds it
// against the reference library that oracle/Makefile compiles into oracle/_ref and runs it; it is never part of the
// product or of a test run.
// usage: offsets_reference MODEL OPTIONS INPUT -- OPTIONS is the SetEncodeExtraOptions string ("-" for none), INPUT
// holds one sentence per line in hex.  Prints, per sentence, its pieces as "id:piece:surface:begin:end" (piece and
// surface in hex) separated by spaces.  Fails when a piece's surface is not input[begin, end).
#include <cstdio>
#include <fstream>
#include <string>

#include "sentencepiece.pb.h"
#include "sentencepiece_processor.h"

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

int main(int argc, char **argv) {
  if (argc != 4) return 2;
  sentencepiece::SentencePieceProcessor sp;
  if (!sp.Load(argv[1]).ok()) { fprintf(stderr, "cannot load %s\n", argv[1]); return 1; }
  if (std::string(argv[2]) != "-" && !sp.SetEncodeExtraOptions(argv[2]).ok()) {
    fprintf(stderr, "bad options %s\n", argv[2]);
    return 1;
  }
  std::ifstream in(argv[3]);
  size_t line = 0;
  for (std::string l; std::getline(in, l); ++line) {
    const std::string s = unhex(l);
    sentencepiece::SentencePieceText spt;
    if (!sp.Encode(absl::string_view(s), &spt).ok()) { fprintf(stderr, "encode failed on line %zu\n", line); return 1; }
    std::string row;
    for (const auto &p : spt.pieces()) {
      if (p.begin() > p.end() || p.end() > s.size() || p.surface() != s.substr(p.begin(), p.end() - p.begin())) {
        fprintf(stderr, "line %zu: surface is not input[begin, end)\n", line);
        return 1;
      }
      if (!row.empty()) row += ' ';
      row += std::to_string(p.id()) + ":" + hex(p.piece()) + ":" + hex(p.surface()) + ":" + std::to_string(p.begin()) +
             ":" + std::to_string(p.end());
    }
    printf("%s\n", row.c_str());
  }
  return 0;
}
