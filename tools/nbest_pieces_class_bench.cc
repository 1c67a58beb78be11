// tools/nbest_pieces_class_bench.cc -- times SentencePieceProcessor::NBestEncode(inputs, nbest_size, pieces) of the
// C++ host class, the vector-of-strings form a C++ caller uses.  Built by tools/nbest_pieces_bench.py against a given
// build of the class, so that two builds can be timed in one session.
// Usage: driver MODEL BYTES_FILE OFFSETS_FILE NBEST REPS -> prints "best_ms hash [packed_ms]" (hash: FNV-1a over all
// pieces; packed_ms: the engine call alone, NBestEncodePiecesPacked, for a build that has it: -DHAS_PACKED).
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <fstream>
#include <iterator>
#include <string>
#include <string_view>
#include <vector>

#include "host/sentencepiece_processor.h"

int main(int argc, char **argv) {
  if (argc != 6) return 2;
  std::ifstream fb(argv[2], std::ios::binary), fo(argv[3], std::ios::binary);
  const std::string bytes((std::istreambuf_iterator<char>(fb)), std::istreambuf_iterator<char>());
  const std::string ob((std::istreambuf_iterator<char>(fo)), std::istreambuf_iterator<char>());
  std::vector<uint64_t> offs(ob.size() / 8);
  for (size_t i = 0; i < offs.size(); ++i) offs[i] = reinterpret_cast<const uint64_t *>(ob.data())[i];
  const size_t n = offs.size() - 1;
  std::vector<std::string_view> views(n);
  for (size_t i = 0; i < n; ++i) views[i] = std::string_view(bytes.data() + offs[i], offs[i + 1] - offs[i]);
  sentencepiece::SentencePieceProcessor sp;
  if (!sp.Load(argv[1]).ok()) return 1;
  const int nbest = std::stoi(argv[4]), reps = std::stoi(argv[5]);
  std::vector<std::vector<std::vector<std::string>>> pieces;
  double best = 1e300;
  for (int r = 0; r <= reps; ++r) {  // the first call is a warm-up
    const auto t0 = std::chrono::steady_clock::now();
    if (!sp.NBestEncode(views, nbest, &pieces).ok()) return 3;
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (r && ms < best) best = ms;
  }
  uint64_t h = 1469598103934665603ull;
  auto mix = [&](unsigned char c) { h = (h ^ c) * 1099511628211ull; };
  for (const auto &s : pieces) {
    for (const auto &c : s) {
      for (const auto &p : c) { for (const char ch : p) mix(static_cast<unsigned char>(ch)); mix(0xFF); }
      mix(0xFE);
    }
    mix(0xFD);
  }
  printf("%.3f %016llx", best, static_cast<unsigned long long>(h));
#ifdef HAS_PACKED
  double packed = 1e300;
  for (int r = 0; r <= reps; ++r) {
    const char *text;
    const uint64_t *to, *co;
    const uint32_t *ends, *nc;
    const auto t0 = std::chrono::steady_clock::now();
    if (!sp.NBestEncodePiecesPacked(bytes.data(), offs.data(), n, nbest, -1, &text, &to, &ends, &co, &nc).ok()) return 4;
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (r && ms < packed) packed = ms;
  }
  printf(" %.3f", packed);
#endif
  printf("\n");
  return 0;
}
