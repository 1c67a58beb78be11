// host/spm_encode_main.cc -- the `spm_encode` caller re-looped for batches.
//
// The reference CLI (src/spm_encode_main.cc:102-165) encodes one line per call in a
// single-threaded getline loop.  This drop-in keeps its flags (--model, --input, --output,
// --output_format=piece|id|sample_piece|sample_id|nbest_piece|nbest_id, --extra_options,
// --nbest_size, --alpha, --random_seed, --vocabulary, --vocabulary_threshold,
// --generate_vocabulary) but reads --batch_lines lines at a time into one packed buffer,
// makes ONE batch call into the engine, and writes the lines back in order.  The *_proto
// formats print nothing in the reference either; they are accepted and run the same calls.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <map>
#include <string>
#include <vector>

#include "host/sentencepiece_processor.h"

namespace {
bool Flag(const char *arg, const char *name, std::string *val) {
  const size_t l = strlen(name);
  if (strncmp(arg, name, l) == 0 && arg[l] == '=') { *val = arg + l + 1; return true; }
  return false;
}
}  // namespace

int main(int argc, char **argv) {
  std::string model, input, output, format = "piece", extra, batch = "1000000", device = "0";
  std::string nbest_s = "10", alpha_s = "0.5", seed_s, vocabulary, vocab_thr = "0", genvocab_s;
  bool verbose = false, generate_vocabulary = false;
  for (int i = 1; i < argc; ++i) {
    std::string v;
    if (Flag(argv[i], "--model", &model) || Flag(argv[i], "--input", &input) || Flag(argv[i], "--output", &output) ||
        Flag(argv[i], "--output_format", &format) || Flag(argv[i], "--extra_options", &extra) ||
        Flag(argv[i], "--batch_lines", &batch) || Flag(argv[i], "--device", &device) ||
        Flag(argv[i], "--nbest_size", &nbest_s) || Flag(argv[i], "--alpha", &alpha_s) ||
        Flag(argv[i], "--random_seed", &seed_s) || Flag(argv[i], "--vocabulary", &vocabulary) ||
        Flag(argv[i], "--vocabulary_threshold", &vocab_thr))
      continue;
    if (Flag(argv[i], "--generate_vocabulary", &genvocab_s)) { generate_vocabulary = genvocab_s != "false" && genvocab_s != "0"; continue; }
    if (!strcmp(argv[i], "--generate_vocabulary")) { generate_vocabulary = true; continue; }
    if (!strcmp(argv[i], "--verbose")) { verbose = true; continue; }
    if (argv[i][0] != '-') { input = argv[i]; continue; }
    std::cerr << "unknown flag " << argv[i] << "\n";
    return 2;
  }
  if (model.empty()) { std::cerr << "--model is required\n"; return 2; }
  static const char *kFormats[] = {"piece", "id", "proto", "sample_piece", "sample_id", "sample_proto",
                                   "nbest_piece", "nbest_id", "nbest_proto"};
  if (std::find_if(std::begin(kFormats), std::end(kFormats), [&](const char *f) { return format == f; }) == std::end(kFormats)) {
    std::cerr << "Unknown output format: " << format << "\n";  // spm_encode_main.cc:154-157
    return 2;
  }
  const int nbest_size = std::stoi(nbest_s);
  const float alpha = static_cast<float>(std::stod(alpha_s));
  if (!seed_s.empty() && static_cast<uint32_t>(std::stoull(seed_s)) != static_cast<uint32_t>(-1))
    sentencepiece::SetRandomGeneratorSeed(static_cast<uint32_t>(std::stoull(seed_s)));  // spm_encode_main.cc:65-67
  sentencepiece::SentencePieceProcessor sp;
  sp.SetDevice(std::stoi(device));
  auto st = sp.Load(model);
  if (!st.ok()) { std::cerr << st.ToString() << "\n"; return 1; }
  st = sp.SetEncodeExtraOptions(extra);
  if (!st.ok()) { std::cerr << st.ToString() << "\n"; return 1; }
  if (!vocabulary.empty()) {  // spm_encode_main.cc:83-92
    st = sp.LoadVocabulary(vocabulary, std::stoi(vocab_thr));
    if (!st.ok()) { std::cerr << st.ToString() << "\n"; return 1; }
  }

  std::ifstream fin;
  if (!input.empty()) { fin.open(input, std::ios::binary); if (!fin) { std::cerr << "cannot open " << input << "\n"; return 1; } }
  std::istream &in = input.empty() ? std::cin : fin;
  std::ofstream fout;
  if (!output.empty()) { fout.open(output, std::ios::binary); if (!fout) { std::cerr << "cannot open " << output << "\n"; return 1; } }
  std::ostream &out = output.empty() ? std::cout : fout;

  const size_t batch_lines = std::max<size_t>(1, std::stoull(batch));
  std::vector<std::string> lines;
  std::vector<std::string_view> views;
  std::string line, buf;
  double enc_s = 0;
  size_t total = 0;
  std::map<std::string, int> vocab;
  bool eof = false;
  while (!eof) {
    lines.clear();
    while (lines.size() < batch_lines) {
      if (!std::getline(in, line)) { eof = true; break; }
      lines.push_back(line);
    }
    if (lines.empty()) break;
    views.assign(lines.begin(), lines.end());
    const auto t0 = std::chrono::steady_clock::now();
    buf.clear();
    auto join_ids = [&](const std::vector<int> &v) {
      for (size_t k = 0; k < v.size(); ++k) { if (k) buf += ' '; buf += std::to_string(v[k]); }
      buf += '\n';
    };
    if (generate_vocabulary) {  // spm_encode_main.cc:102-110: counts of the pieces that are neither unknown nor control
      std::vector<std::vector<int>> ids;
      st = sp.Encode(views, &ids);
      if (!st.ok()) { std::cerr << st.ToString() << "\n"; return 1; }
      for (const auto &v : ids)
        for (const int id : v)
          if (!sp.IsUnknown(id) && !sp.IsControl(id)) vocab[sp.IdToPiece(id)]++;
    } else if (format == "id") {
      std::vector<std::vector<int>> ids;
      st = sp.Encode(views, &ids);
      if (!st.ok()) { std::cerr << st.ToString() << "\n"; return 1; }
      for (const auto &v : ids) join_ids(v);
    } else if (format == "piece" || format == "sample_piece" || format == "nbest_piece") {
      // the engine writes each line's (candidate's) pieces joined by ' '
      std::string packed;
      std::vector<uint64_t> offs(lines.size() + 1, 0);
      for (size_t i = 0; i < lines.size(); ++i) { packed += lines[i]; offs[i + 1] = packed.size(); }
      const char *text;
      const uint64_t *to, *ido;
      const uint32_t *ends;
      const uint32_t *nc = nullptr;
      size_t K = 1;
      if (format == "piece") {
        st = sp.EncodePiecesPacked(packed.data(), offs.data(), lines.size(), ' ', &text, &to, &ends, &ido);
      } else if (format == "sample_piece") {
        st = sp.SampleEncodePiecesPacked(packed.data(), offs.data(), lines.size(), nbest_size, alpha, ' ', &text, &to,
                                         &ends, &ido);
      } else {
        st = sp.NBestEncodePiecesPacked(packed.data(), offs.data(), lines.size(), nbest_size, ' ', &text, &to, &ends, &ido,
                                        &nc);
        K = static_cast<size_t>(std::max(1, std::min(nbest_size, 1024)));
      }
      if (!st.ok()) { std::cerr << st.ToString() << "\n"; return 1; }
      buf.reserve(to[lines.size() * K] + lines.size() * K);
      for (size_t i = 0; i < lines.size(); ++i)
        for (size_t c = 0; c < (nc ? nc[i] : 1u); ++c) {
          const size_t j = i * K + c;
          buf.append(text + to[j], to[j + 1] - to[j]);
          buf += '\n';
        }
    } else if (format == "proto") {
      std::vector<std::vector<std::string>> pcs;
      st = sp.Encode(views, &pcs);
      if (!st.ok()) { std::cerr << st.ToString() << "\n"; return 1; }
    } else if (format == "sample_id" || format == "sample_proto") {
      std::vector<std::vector<int>> ids;
      st = sp.SampleEncode(views, nbest_size, alpha, &ids);
      if (!st.ok()) { std::cerr << st.ToString() << "\n"; return 1; }
      if (format == "sample_id") for (const auto &v : ids) join_ids(v);
    } else if (format == "nbest_id" || format == "nbest_proto") {
      std::vector<std::vector<std::vector<int>>> ids;
      st = sp.NBestEncode(views, nbest_size, &ids);
      if (!st.ok()) { std::cerr << st.ToString() << "\n"; return 1; }
      if (format == "nbest_id") for (const auto &c : ids) for (const auto &v : c) join_ids(v);
    }
    enc_s += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    out.write(buf.data(), buf.size());
    total += lines.size();
  }
  if (generate_vocabulary) {  // Sorted(vocab): by count descending, then by key (trainer_interface.h:35-50)
    std::vector<std::pair<std::string, int>> v(vocab.begin(), vocab.end());
    std::sort(v.begin(), v.end(), [](const auto &a, const auto &b) { return a.second != b.second ? a.second > b.second : a.first < b.first; });
    for (const auto &it : v) out << it.first << "\t" << it.second << "\n";
  }
  if (verbose) fprintf(stderr, "encoded %zu lines, %.3f s in Encode+format\n", total, enc_s);
  return 0;
}
