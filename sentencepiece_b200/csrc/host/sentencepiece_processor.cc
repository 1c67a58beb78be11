// host/sentencepiece_processor.cc -- see the header.  All heavy lifting is behind the C ABI.
#include "host/sentencepiece_processor.h"

#include <algorithm>
#include <atomic>
#include <cstring>
#include <fstream>
#include <functional>
#include <set>
#include <sstream>
#include <thread>
#include <unordered_map>

#include "model_reader.h"
#include "spm_b200.h"

namespace sentencepiece {

struct SentencePieceProcessor::Impl {
  spm_b200::ModelData model;
  std::vector<std::string> pieces;
  std::unordered_map<std::string, int> piece_to_id;
  std::vector<uint8_t> loaded_types;
};

namespace {
std::atomic<unsigned int> g_seed{0};
std::atomic<bool> g_seed_set{false};
util::Status Internal(const std::string &m) { return util::Status(util::StatusCode::kInternal, m); }
util::Status FromEngine(const spm_engine *e, int rc) {
  if (rc == 0) return util::OkStatus();
  return Internal(std::string("spm_b200(") + std::to_string(rc) + "): " + spm_last_error(e));
}
}  // namespace

void SetRandomGeneratorSeed(unsigned int seed) {
  g_seed = seed;
  g_seed_set = true;
}

SentencePieceProcessor::SentencePieceProcessor() : impl_(new Impl) {}
SentencePieceProcessor::~SentencePieceProcessor() {
  if (engine_) spm_engine_destroy(engine_);
}

util::Status SentencePieceProcessor::status() const {
  if (!engine_) return Internal("Model is not initialized.");  // sentencepiece_processor.cc:293-299
  return util::OkStatus();
}

util::Status SentencePieceProcessor::Load(std::string_view filename) {
  std::ifstream f(std::string(filename), std::ios::binary);
  if (!f) return util::Status(util::StatusCode::kNotFound, "\"" + std::string(filename) + "\": No such file or directory");
  std::stringstream ss;
  ss << f.rdbuf();
  return LoadFromSerializedProto(ss.str());
}

util::Status SentencePieceProcessor::LoadFromSerializedProto(std::string_view serialized) {
  std::string err;
  if (!spm_b200::ParseModelProto(serialized.data(), serialized.size(), &impl_->model, &err)) return Internal(err);
  if (engine_) { spm_engine_destroy(engine_); engine_ = nullptr; }
  const int rc = spm_engine_create_from_serialized(serialized.data(), serialized.size(), device_, &engine_);
  if (rc) { engine_ = nullptr; return FromEngine(nullptr, rc); }
  const auto &m = impl_->model;
  impl_->pieces.clear();
  impl_->piece_to_id.clear();
  unk_id_ = -1;
  for (int i = 0; i < m.vocab_size(); ++i) {
    impl_->pieces.emplace_back(m.piece(i), m.piece_len(i));
    impl_->piece_to_id.emplace(impl_->pieces.back(), i);  // first definition wins, like InsertIfNotPresent
    if (m.types[i] == SPM_UNKNOWN) unk_id_ = i;
  }
  impl_->loaded_types = m.types;
  extra_.clear();
  frame_p_.clear();
  frame_s_.clear();
  frame_rev_ = false;
  seeded_ = false;
  return util::OkStatus();
}

bool SentencePieceProcessor::IsControl(int id) const {
  return id >= 0 && id < GetPieceSize() && impl_->model.types[id] == SPM_CONTROL;
}

// the reference's generator is thread_local and takes the global seed when it is first used (util.cc:202-204)
void SentencePieceProcessor::SeedOnce() const {
  if (seeded_) return;
  seeded_ = true;
  if (g_seed_set) spm_set_random_seed(engine_, g_seed);
}

util::Status SentencePieceProcessor::LoadVocabulary(std::string_view filename, int threshold) {
  if (!engine_) return status();
  std::ifstream f(std::string(filename), std::ios::binary);
  if (!f) return util::Status(util::StatusCode::kNotFound, "\"" + std::string(filename) + "\": No such file or directory");
  std::vector<std::string> vocab;
  std::string line;
  while (std::getline(f, line)) {
    const size_t tab = line.find('\t');
    const std::string piece = line.substr(0, tab);
    if (piece.empty()) return Internal("empty piece in the vocabulary file");
    long freq = 1;
    if (tab != std::string::npos) {
      const std::string fs = line.substr(tab + 1, line.find('\t', tab + 1) - tab - 1);
      char *end = nullptr;
      freq = strtol(fs.c_str(), &end, 10);
      if (fs.empty() || *end) return Internal("Could not parse the frequency");
    }
    if (freq >= threshold) vocab.push_back(piece);
  }
  std::vector<std::string_view> views(vocab.begin(), vocab.end());
  return SetVocabulary(views);
}

int SentencePieceProcessor::GetPieceSize() const { return static_cast<int>(impl_->pieces.size()); }
int SentencePieceProcessor::PieceToId(std::string_view piece) const {
  const auto it = impl_->piece_to_id.find(std::string(piece));
  return it == impl_->piece_to_id.end() ? unk_id_ : it->second;  // model_interface.cc:51-61
}
const std::string &SentencePieceProcessor::IdToPiece(int id) const {
  static const std::string kEmpty;
  return id >= 0 && id < GetPieceSize() ? impl_->pieces[id] : kEmpty;
}
int SentencePieceProcessor::bos_id() const {
  const int id = PieceToId(impl_->model.bos_piece);
  return id == unk_id_ ? -1 : id;
}
int SentencePieceProcessor::eos_id() const {
  const int id = PieceToId(impl_->model.eos_piece);
  return id == unk_id_ ? -1 : id;
}

// ParseExtraOptions, sentencepiece_processor.cc:1067-1101; the engine then writes the options' id effect into every id
// result (spm_engine_set_encode_frame), whatever the outcome of the parse left in extra_
util::Status SentencePieceProcessor::SetEncodeExtraOptions(std::string_view extra_option) {
  const util::Status st = ParseExtraOptions(extra_option);
  if (!engine_) return st;
  // the canonical form P ++ (r or reversed r) ++ S of the options applied in order
  frame_p_.clear();
  frame_s_.clear();
  frame_rev_ = false;
  for (const auto o : extra_) {
    if (o == REVERSE) {
      std::swap(frame_p_, frame_s_);
      std::reverse(frame_p_.begin(), frame_p_.end());
      std::reverse(frame_s_.begin(), frame_s_.end());
      frame_rev_ = !frame_rev_;
    } else if (o == BOS) {
      frame_p_.insert(frame_p_.begin(), PieceToId(impl_->model.bos_piece));
    } else if (o == EOS) {
      frame_s_.push_back(PieceToId(impl_->model.eos_piece));
    }
  }
  const int rc = spm_engine_set_encode_frame(engine_, frame_p_.data(), static_cast<uint32_t>(frame_p_.size()), frame_rev_,
                                             frame_s_.data(), static_cast<uint32_t>(frame_s_.size()));
  if (rc) {
    const util::Status err = FromEngine(engine_, rc);
    extra_.clear();
    frame_p_.clear();
    frame_s_.clear();
    frame_rev_ = false;
    spm_engine_set_encode_frame(engine_, nullptr, 0, 0, nullptr, 0);
    return err;
  }
  return st;
}

util::Status SentencePieceProcessor::ParseExtraOptions(std::string_view extra_option) {
  extra_.clear();
  if (extra_option.empty()) return util::OkStatus();
  if (!engine_) return status();
  size_t pos = 0;
  while (pos <= extra_option.size()) {
    size_t nxt = extra_option.find(':', pos);
    if (nxt == std::string_view::npos) nxt = extra_option.size();
    const std::string s(extra_option.substr(pos, nxt - pos));
    if (s == "bos") {
      if (IsUnknown(PieceToId(impl_->model.bos_piece))) return Internal("id for `" + impl_->model.bos_piece + "` is not defined.");
      extra_.push_back(BOS);
    } else if (s == "eos") {
      if (IsUnknown(PieceToId(impl_->model.eos_piece))) return Internal("id for `" + impl_->model.eos_piece + "` is not defined.");
      extra_.push_back(EOS);
    } else if (s == "reverse") {
      extra_.push_back(REVERSE);
    } else if (s == "unk" || s == "unk_piece") {
      extra_.push_back(UNK_PIECE);
    } else {
      extra_.clear();
      return Internal("option \"" + s + "\" is not available.");
    }
    pos = nxt + 1;
  }
  return util::OkStatus();
}

// sentencepiece_processor.cc:301-330: pieces of one character are always kept
util::Status SentencePieceProcessor::SetVocabulary(const std::vector<std::string_view> &valid_vocab) {
  if (!engine_) return status();
  auto &m = impl_->model;
  const std::set<std::string_view> vocab(valid_vocab.begin(), valid_vocab.end());
  static const unsigned char kLen[16] = {1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 3, 4};
  for (int i = 0; i < m.vocab_size(); ++i) {
    uint8_t &t = m.types[i];
    if (t == SPM_CONTROL || t == SPM_UNKNOWN || t == SPM_USER_DEFINED) continue;
    const std::string &p = impl_->pieces[i];
    const bool one_char = kLen[static_cast<unsigned char>(p[0]) >> 4] == p.size();
    if (t == SPM_BYTE) continue;  // byte pieces never enter pieces_; their class is fixed
    t = (vocab.count(p) || one_char) ? SPM_NORMAL : SPM_UNUSED;
  }
  return FromEngine(engine_, spm_engine_set_types(engine_, m.types.data()));
}

util::Status SentencePieceProcessor::ResetVocabulary() {
  if (!engine_) return status();
  for (auto &t : impl_->model.types)
    if (t == SPM_UNUSED) t = SPM_NORMAL;
  return FromEngine(engine_, spm_engine_set_types(engine_, impl_->model.types.data()));
}

util::Status SentencePieceProcessor::EncodePacked(const char *bytes, const uint64_t *offsets, size_t n,
                                                  const int32_t **ids, const uint64_t **id_offsets) const {
  if (!engine_) return status();
  return FromEngine(engine_, spm_encode_ids(engine_, bytes, offsets, n, ids, id_offsets));
}

util::Status SentencePieceProcessor::Decode(const std::vector<std::vector<int>> &ids,
                                            std::vector<std::string> *detokenized) const {
  if (!engine_) return status();
  if (!detokenized) return Internal("output container is null");  // CHECK_OR_RETURN_STATUS_STL
  detokenized->clear();
  std::vector<int32_t> packed;
  std::vector<uint64_t> offs(1, 0);
  for (const auto &l : ids) {
    packed.insert(packed.end(), l.begin(), l.end());
    offs.push_back(packed.size());
  }
  const char *text = nullptr;
  const uint64_t *to = nullptr;
  const int rc = spm_decode_ids(engine_, packed.data(), offs.data(), ids.size(), &text, &to);
  if (rc) return FromEngine(engine_, rc);
  detokenized->reserve(ids.size());
  for (size_t i = 0; i < ids.size(); ++i) detokenized->emplace_back(text + to[i], text + to[i + 1]);
  return util::OkStatus();
}

util::Status SentencePieceProcessor::Decode(const std::vector<int> &ids, std::string *detokenized) const {
  if (!engine_) return status();
  if (!detokenized) return Internal("output container is null");
  std::vector<std::string> out;
  const util::Status st = Decode(std::vector<std::vector<int>>{ids}, &out);
  if (!st.ok()) return st;
  *detokenized = std::move(out[0]);
  return util::OkStatus();
}

std::string SentencePieceProcessor::DecodeIds(const std::vector<int> &ids) const {
  std::string out;
  Decode(ids, &out);
  return out;
}

util::Status SentencePieceProcessor::DecodeOffsetsPacked(const int32_t *ids, const uint64_t *id_offsets, size_t n,
                                                         const char **text, const uint64_t **text_offsets,
                                                         const uint32_t **tok_end) const {
  if (!engine_) return status();
  return FromEngine(engine_, spm_decode_offsets(engine_, ids, id_offsets, n, text, text_offsets, tok_end));
}

namespace {
// runs fn(lo, hi) over [0, n) on a few host threads (the container conversions around a batch call are the only
// per-sentence host work left; the reference's Python layer uses a thread pool for the same reason,
// python/src/sentencepiece/sentencepiece.i:235-267)
template <typename F>
void ParallelFor(size_t n, F fn) {
  const size_t T = n < 16384 ? 1 : std::max<size_t>(1, std::min<size_t>(std::thread::hardware_concurrency(), 16));
  if (T == 1) { fn(size_t{0}, n); return; }
  std::vector<std::thread> th;
  const size_t per = (n + T - 1) / T;
  for (size_t t = 1; t < T; ++t) th.emplace_back(fn, std::min(n, t * per), std::min(n, (t + 1) * per));
  fn(size_t{0}, std::min(n, per));
  for (auto &t : th) t.join();
}

void Pack(const std::vector<std::string_view> &in, std::string *bytes, std::vector<uint64_t> *offs) {
  offs->resize(in.size() + 1);
  uint64_t total = 0;
  for (size_t i = 0; i < in.size(); ++i) { (*offs)[i] = total; total += in[i].size(); }
  (*offs)[in.size()] = total;
  bytes->resize(total);
  char *dst = bytes->data();
  const uint64_t *o = offs->data();
  ParallelFor(in.size(), [&](size_t lo, size_t hi) {
    for (size_t i = lo; i < hi; ++i)
      if (!in[i].empty()) memcpy(dst + o[i], in[i].data(), in[i].size());
  });
}
}  // namespace

util::Status SentencePieceProcessor::Encode(const std::vector<std::string_view> &inputs,
                                            std::vector<std::vector<int>> *ids) const {
  if (!engine_) return status();
  if (!ids) return Internal("output container is null");  // CHECK_OR_RETURN_STATUS_STL
  ids->clear();
  std::string bytes;
  std::vector<uint64_t> offs;
  Pack(inputs, &bytes, &offs);
  const int32_t *out;
  const uint64_t *oo;
  const auto st = EncodePacked(bytes.data(), offs.data(), inputs.size(), &out, &oo);
  if (!st.ok()) return st;
  ids->resize(inputs.size());
  ParallelFor(inputs.size(), [&](size_t lo, size_t hi) {
    for (size_t i = lo; i < hi; ++i) {
      auto &v = (*ids)[i];
      v.assign(out + oo[i], out + oo[i + 1]);
    }
  });
  return util::OkStatus();
}

util::Status SentencePieceProcessor::NormalizePacked(const char *bytes, const uint64_t *offsets, size_t n,
                                                     bool with_offsets, const char **normalized,
                                                     const uint64_t **norm_offsets, const uint32_t **n2o) const {
  if (!engine_) return status();
  return FromEngine(engine_, spm_normalize(engine_, bytes, offsets, n, with_offsets ? 1 : 0, normalized, norm_offsets, n2o));
}

util::Status SentencePieceProcessor::Normalize(const std::vector<std::string_view> &inputs,
                                               std::vector<std::string> *normalized,
                                               std::vector<std::vector<size_t>> *norm_to_orig) const {
  if (!engine_) return status();
  if (!normalized) return Internal("output container is null");
  normalized->clear();
  if (norm_to_orig) norm_to_orig->clear();
  std::string bytes;
  std::vector<uint64_t> offs;
  Pack(inputs, &bytes, &offs);
  const char *text = nullptr;
  const uint64_t *no = nullptr;
  const uint32_t *n2o = nullptr;
  const auto st = NormalizePacked(bytes.data(), offs.data(), inputs.size(), norm_to_orig != nullptr, &text, &no, &n2o);
  if (!st.ok()) return st;
  normalized->resize(inputs.size());
  if (norm_to_orig) norm_to_orig->resize(inputs.size());
  ParallelFor(inputs.size(), [&](size_t lo, size_t hi) {
    for (size_t i = lo; i < hi; ++i) {
      (*normalized)[i].assign(text + no[i], text + no[i + 1]);
      if (!norm_to_orig) continue;
      const uint32_t *m = n2o + no[i] + i;
      if (m[0] != SPM_NORM_TO_ORIG_EMPTY) (*norm_to_orig)[i].assign(m, m + (no[i + 1] - no[i]) + 1);
    }
  });
  return util::OkStatus();
}

util::Status SentencePieceProcessor::Normalize(std::string_view input, std::string *normalized,
                                               std::vector<size_t> *norm_to_orig) const {
  if (!engine_) return status();
  if (!normalized || !norm_to_orig) return Internal("output container is null");
  std::vector<std::string> t;
  std::vector<std::vector<size_t>> m;
  const auto st = Normalize(std::vector<std::string_view>{input}, &t, &m);
  if (!st.ok()) return st;
  *normalized = std::move(t[0]);
  *norm_to_orig = std::move(m[0]);
  return util::OkStatus();
}

util::Status SentencePieceProcessor::Normalize(std::string_view input, std::string *normalized) const {
  if (!engine_) return status();
  if (!normalized) return Internal("output container is null");
  std::vector<std::string> t;
  const auto st = Normalize(std::vector<std::string_view>{input}, &t);
  if (!st.ok()) return st;
  *normalized = std::move(t[0]);
  return util::OkStatus();
}

std::string SentencePieceProcessor::Normalize(std::string_view input) const {
  std::string normalized;
  Normalize(input, &normalized).IgnoreError();
  return normalized;
}

// The engine writes the pieces with the options applied: bos / eos / reverse are the frame SetEncodeExtraOptions set,
// UNK_PIECE is passed as trainer_spec.unk_piece.
const std::string *SentencePieceProcessor::UnkPiece() const {
  const bool unk = std::find(extra_.begin(), extra_.end(), UNK_PIECE) != extra_.end();
  return unk ? &impl_->model.unk_piece : nullptr;
}

util::Status SentencePieceProcessor::EncodePiecesPacked(const char *bytes, const uint64_t *offsets, size_t n, int sep,
                                                        const char **text, const uint64_t **text_offsets,
                                                        const uint32_t **piece_end, const uint64_t **id_offsets) const {
  if (!engine_) return status();
  const std::string *up = UnkPiece();
  const int32_t *ids;
  return FromEngine(engine_, spm_encode_pieces(engine_, bytes, offsets, n, up ? up->data() : nullptr, up ? up->size() : 0,
                                               sep, text, text_offsets, piece_end, &ids, id_offsets));
}

util::Status SentencePieceProcessor::NBestEncodePiecesPacked(const char *bytes, const uint64_t *offsets, size_t n,
                                                             int nbest_size, int sep, const char **text,
                                                             const uint64_t **text_offsets, const uint32_t **piece_end,
                                                             const uint64_t **cand_offsets, const uint32_t **n_cands) const {
  if (!engine_) return status();
  const std::string *up = UnkPiece();
  const int32_t *ids;
  const float *scores;
  return FromEngine(engine_, spm_nbest_encode_pieces(engine_, bytes, offsets, n, nbest_size, up ? up->data() : nullptr,
                                                     up ? up->size() : 0, sep, text, text_offsets, piece_end, &ids,
                                                     cand_offsets, &scores, n_cands));
}

util::Status SentencePieceProcessor::SampleEncodePiecesPacked(const char *bytes, const uint64_t *offsets, size_t n,
                                                              int nbest_size, float alpha, int sep, const char **text,
                                                              const uint64_t **text_offsets, const uint32_t **piece_end,
                                                              const uint64_t **id_offsets) const {
  if (!engine_) return status();
  SeedOnce();
  const std::string *up = UnkPiece();
  const int32_t *ids;
  return FromEngine(engine_, spm_sample_encode_pieces(engine_, bytes, offsets, n, nbest_size, alpha,
                                                      up ? up->data() : nullptr, up ? up->size() : 0, sep, text,
                                                      text_offsets, piece_end, &ids, id_offsets));
}

util::Status SentencePieceProcessor::EncodeOffsetsPacked(const char *bytes, const uint64_t *offsets, size_t n,
                                                         const int32_t **ids, const uint64_t **id_offsets,
                                                         const uint32_t **begin, const uint32_t **end, const char **text,
                                                         const uint64_t **text_offsets,
                                                         const uint32_t **piece_end) const {
  if (!engine_) return status();
  const std::string *up = UnkPiece();
  return FromEngine(engine_, spm_encode_offsets(engine_, bytes, offsets, n, eos_id(), up ? up->data() : nullptr,
                                                up ? up->size() : 0, -1, ids, id_offsets, begin, end, text,
                                                text_offsets, piece_end));
}

util::Status SentencePieceProcessor::EncodeWithOffsets(const std::vector<std::string_view> &inputs,
                                                       std::vector<std::vector<PieceSpan>> *pieces) const {
  if (!engine_) return status();
  if (!pieces) return Internal("output container is null");
  pieces->clear();
  std::string bytes;
  std::vector<uint64_t> offs;
  Pack(inputs, &bytes, &offs);
  const int32_t *ids;
  const uint64_t *ido, *to;
  const uint32_t *b, *e, *pe;
  const char *text;
  const auto st = EncodeOffsetsPacked(bytes.data(), offs.data(), inputs.size(), &ids, &ido, &b, &e, &text, &to, &pe);
  if (!st.ok()) return st;
  pieces->resize(inputs.size());
  ParallelFor(inputs.size(), [&](size_t lo, size_t hi) {
    for (size_t i = lo; i < hi; ++i) {
      auto &v = (*pieces)[i];
      v.resize(ido[i + 1] - ido[i]);
      const char *t = text + to[i];
      for (uint64_t k = ido[i]; k < ido[i + 1]; ++k) {
        PieceSpan &s = v[k - ido[i]];
        const uint32_t p0 = k > ido[i] ? pe[k - 1] : 0u;
        s.piece.assign(t + p0, t + pe[k]);
        s.id = ids[k];
        s.surface.assign(inputs[i].data() + b[k], e[k] - b[k]);
        s.begin = b[k];
        s.end = e[k];
      }
    }
  });
  return util::OkStatus();
}

util::Status SentencePieceProcessor::EncodeWithOffsets(std::string_view input, std::vector<PieceSpan> *pieces) const {
  if (!engine_) return status();
  if (!pieces) return Internal("output container is null");
  std::vector<std::vector<PieceSpan>> v;
  const auto st = EncodeWithOffsets(std::vector<std::string_view>{input}, &v);
  if (!st.ok()) return st;
  *pieces = std::move(v[0]);
  return util::OkStatus();
}

util::Status SentencePieceProcessor::DecodeWithOffsets(const std::vector<std::vector<int>> &ids,
                                                       std::vector<std::string> *text,
                                                       std::vector<std::vector<PieceSpan>> *pieces) const {
  if (!engine_) return status();
  if (!text || !pieces) return Internal("output container is null");
  text->clear();
  pieces->clear();
  std::vector<int32_t> packed;
  std::vector<uint64_t> offs(1, 0);
  for (const auto &l : ids) {
    packed.insert(packed.end(), l.begin(), l.end());
    offs.push_back(packed.size());
  }
  const char *t;
  const uint64_t *to;
  const uint32_t *te;
  const auto st = DecodeOffsetsPacked(packed.data(), offs.data(), ids.size(), &t, &to, &te);
  if (!st.ok()) return st;
  text->resize(ids.size());
  pieces->resize(ids.size());
  ParallelFor(ids.size(), [&](size_t lo, size_t hi) {
    for (size_t i = lo; i < hi; ++i) {
      std::string &s = (*text)[i];
      s.assign(t + to[i], t + to[i + 1]);
      auto &v = (*pieces)[i];
      v.resize(offs[i + 1] - offs[i]);
      uint32_t begin = 0;
      for (uint64_t k = offs[i]; k < offs[i + 1]; ++k) {
        PieceSpan &p = v[k - offs[i]];
        p.id = packed[k];
        p.piece = IdToPiece(p.id);
        p.begin = begin;
        p.end = te[k];
        p.surface.assign(s, p.begin, p.end - p.begin);
        begin = p.end;
      }
    }
  });
  return util::OkStatus();
}

util::Status SentencePieceProcessor::DecodeWithOffsets(const std::vector<int> &ids, std::string *text,
                                                       std::vector<PieceSpan> *pieces) const {
  if (!engine_) return status();
  if (!text || !pieces) return Internal("output container is null");
  std::vector<std::string> t;
  std::vector<std::vector<PieceSpan>> v;
  const auto st = DecodeWithOffsets(std::vector<std::vector<int>>{ids}, &t, &v);
  if (!st.ok()) return st;
  *text = std::move(t[0]);
  *pieces = std::move(v[0]);
  return util::OkStatus();
}

namespace {
// list j of a packed pieces result (sep = -1) as strings
std::vector<std::string> PieceList(const char *text, const uint64_t *to, const uint32_t *ends, const uint64_t *ido,
                                   size_t j) {
  std::vector<std::string> v;
  v.reserve(ido[j + 1] - ido[j]);
  uint32_t begin = 0;
  for (uint64_t k = ido[j]; k < ido[j + 1]; ++k) {
    v.emplace_back(text + to[j] + begin, ends[k] - begin);
    begin = ends[k];
  }
  return v;
}
}  // namespace

util::Status SentencePieceProcessor::Encode(const std::vector<std::string_view> &inputs,
                                            std::vector<std::vector<std::string>> *pieces) const {
  if (!engine_) return status();
  if (!pieces) return Internal("output container is null");
  pieces->clear();
  std::string bytes;
  std::vector<uint64_t> offs;
  Pack(inputs, &bytes, &offs);
  const char *text;
  const uint64_t *to, *ido;
  const uint32_t *ends;
  const auto st = EncodePiecesPacked(bytes.data(), offs.data(), inputs.size(), -1, &text, &to, &ends, &ido);
  if (!st.ok()) return st;
  pieces->resize(inputs.size());
  ParallelFor(inputs.size(), [&](size_t lo, size_t hi) {
    for (size_t i = lo; i < hi; ++i) (*pieces)[i] = PieceList(text, to, ends, ido, i);
  });
  return util::OkStatus();
}

// ---- n-best and sampling: the engine writes the pieces of every candidate, the options applied ----
util::Status SentencePieceProcessor::NBestEncode(const std::vector<std::string_view> &inputs, int nbest_size,
                                                 std::vector<std::vector<std::vector<int>>> *ids) const {
  if (!engine_) return status();
  if (!ids) return Internal("output container is null");
  ids->clear();
  std::string bytes;
  std::vector<uint64_t> offs;
  Pack(inputs, &bytes, &offs);
  const int32_t *out;
  const uint64_t *co;
  const float *sc;
  const uint32_t *nc;
  const int rc = spm_nbest_encode(engine_, bytes.data(), offs.data(), inputs.size(), nbest_size, &out, &co, &sc, &nc);
  if (rc) return FromEngine(engine_, rc);
  const size_t K = static_cast<size_t>(std::max(1, std::min(nbest_size, 1024)));
  ids->resize(inputs.size());
  for (size_t i = 0; i < inputs.size(); ++i) {
    auto &cands = (*ids)[i];
    cands.resize(nc[i]);
    for (uint32_t c = 0; c < nc[i]; ++c) {
      cands[c].assign(out + co[i * K + c], out + co[i * K + c + 1]);
    }
  }
  return util::OkStatus();
}

util::Status SentencePieceProcessor::NBestEncode(const std::vector<std::string_view> &inputs, int nbest_size,
                                                 std::vector<std::vector<std::vector<std::string>>> *pieces) const {
  if (!engine_) return status();
  if (!pieces) return Internal("output container is null");
  pieces->clear();
  std::string bytes;
  std::vector<uint64_t> offs;
  Pack(inputs, &bytes, &offs);
  const char *text;
  const uint64_t *to, *co;
  const uint32_t *ends, *nc;
  const auto st = NBestEncodePiecesPacked(bytes.data(), offs.data(), inputs.size(), nbest_size, -1, &text, &to, &ends, &co, &nc);
  if (!st.ok()) return st;
  const size_t K = static_cast<size_t>(std::max(1, std::min(nbest_size, 1024)));
  // One thread: with many host threads, materialising tens of millions of strings (uni32k at nbest_size 64) took
  // four times as long as on one, on the H100 host measured in DESIGN §5.
  pieces->resize(inputs.size());
  for (size_t i = 0; i < inputs.size(); ++i) {
    auto &cands = (*pieces)[i];
    cands.resize(nc[i]);
    for (uint32_t c = 0; c < nc[i]; ++c) cands[c] = PieceList(text, to, ends, co, i * K + c);
  }
  return util::OkStatus();
}

util::Status SentencePieceProcessor::SampleEncode(const std::vector<std::string_view> &inputs, int nbest_size, float alpha,
                                                  std::vector<std::vector<int>> *ids) const {
  if (!engine_) return status();
  if (!ids) return Internal("output container is null");
  ids->clear();
  SeedOnce();
  std::string bytes;
  std::vector<uint64_t> offs;
  Pack(inputs, &bytes, &offs);
  const int32_t *out;
  const uint64_t *oo;
  const int rc = spm_sample_encode_ids(engine_, bytes.data(), offs.data(), inputs.size(), nbest_size, alpha, &out, &oo);
  if (rc) return FromEngine(engine_, rc);
  ids->resize(inputs.size());
  for (size_t i = 0; i < inputs.size(); ++i) {
    (*ids)[i].assign(out + oo[i], out + oo[i + 1]);
  }
  return util::OkStatus();
}

util::Status SentencePieceProcessor::SampleEncode(const std::vector<std::string_view> &inputs, int nbest_size, float alpha,
                                                  std::vector<std::vector<std::string>> *pieces) const {
  if (!engine_) return status();
  if (!pieces) return Internal("output container is null");
  pieces->clear();
  std::string bytes;
  std::vector<uint64_t> offs;
  Pack(inputs, &bytes, &offs);
  const char *text;
  const uint64_t *to, *ido;
  const uint32_t *ends;
  const auto st = SampleEncodePiecesPacked(bytes.data(), offs.data(), inputs.size(), nbest_size, alpha, -1, &text, &to,
                                           &ends, &ido);
  if (!st.ok()) return st;
  pieces->resize(inputs.size());
  ParallelFor(inputs.size(), [&](size_t lo, size_t hi) {
    for (size_t i = lo; i < hi; ++i) (*pieces)[i] = PieceList(text, to, ends, ido, i);
  });
  return util::OkStatus();
}

util::Status SentencePieceProcessor::CalculateEntropy(const std::vector<std::string_view> &inputs, float alpha,
                                                      std::vector<float> *entropy) const {
  if (!engine_) return status();
  if (!entropy) return Internal("output container is null");
  entropy->clear();
  std::string bytes;
  std::vector<uint64_t> offs;
  Pack(inputs, &bytes, &offs);
  const float *ent = nullptr;
  const int rc = spm_calculate_entropy(engine_, bytes.data(), offs.data(), inputs.size(), alpha, &ent);
  if (rc) return FromEngine(engine_, rc);
  entropy->assign(ent, ent + inputs.size());
  return util::OkStatus();
}
util::Status SentencePieceProcessor::CalculateEntropy(std::string_view input, float alpha, float *entropy) const {
  if (!engine_) return status();
  if (!entropy) return Internal("output container is null");
  std::vector<float> out;
  const auto st = CalculateEntropy(std::vector<std::string_view>{input}, alpha, &out);
  if (!st.ok()) return st;
  *entropy = out[0];
  return util::OkStatus();
}
float SentencePieceProcessor::CalculateEntropy(std::string_view input, float alpha) const {
  float e = 0.f;
  CalculateEntropy(input, alpha, &e).IgnoreError();
  return e;
}

std::vector<std::pair<std::vector<int>, float>> SentencePieceProcessor::SampleEncodeAndScoreAsIds(
    std::string_view input, int num_samples, float alpha, bool wor, bool include_best) const {
  std::vector<std::pair<std::vector<int>, float>> out;
  if (!engine_) return out;
  SeedOnce();
  const uint64_t offs[2] = {0, input.size()};
  const int32_t *ids;
  const uint64_t *co;
  const float *sc;
  if (spm_sample_encode_and_score(engine_, input.data(), offs, 1, num_samples, alpha, wor, include_best, &ids, &co, &sc)) return out;
  for (int c = 0; c < num_samples; ++c) {
    out.emplace_back(std::vector<int>(ids + co[c], ids + co[c + 1]), sc[c]);
  }
  return out;
}
std::vector<std::pair<std::vector<std::string>, float>> SentencePieceProcessor::SampleEncodeAndScoreAsPieces(
    std::string_view input, int num_samples, float alpha, bool wor, bool include_best) const {
  std::vector<std::pair<std::vector<std::string>, float>> out;
  if (!engine_) return out;
  SeedOnce();
  const uint64_t offs[2] = {0, input.size()};
  const std::string *up = UnkPiece();
  const char *text;
  const uint64_t *to, *co;
  const uint32_t *ends;
  const int32_t *ids;
  const float *sc;
  if (spm_sample_encode_and_score_pieces(engine_, input.data(), offs, 1, num_samples, alpha, wor, include_best,
                                         up ? up->data() : nullptr, up ? up->size() : 0, -1, &text, &to, &ends, &ids,
                                         &co, &sc))
    return out;
  for (int c = 0; c < num_samples; ++c) out.emplace_back(PieceList(text, to, ends, co, c), sc[c]);
  return out;
}

util::Status SentencePieceProcessor::NBestEncode(std::string_view input, int nbest_size,
                                                 std::vector<std::vector<int>> *ids) const {
  if (!engine_) return status();
  if (!ids) return Internal("output container is null");
  std::vector<std::vector<std::vector<int>>> out;
  const auto st = NBestEncode(std::vector<std::string_view>{input}, nbest_size, &out);
  if (!st.ok()) return st;
  *ids = std::move(out[0]);
  return util::OkStatus();
}
util::Status SentencePieceProcessor::NBestEncode(std::string_view input, int nbest_size,
                                                 std::vector<std::vector<std::string>> *pieces) const {
  if (!engine_) return status();
  if (!pieces) return Internal("output container is null");
  std::vector<std::vector<std::vector<std::string>>> out;
  const auto st = NBestEncode(std::vector<std::string_view>{input}, nbest_size, &out);
  if (!st.ok()) return st;
  *pieces = std::move(out[0]);
  return util::OkStatus();
}
util::Status SentencePieceProcessor::SampleEncode(std::string_view input, int nbest_size, float alpha,
                                                  std::vector<int> *ids) const {
  if (!engine_) return status();
  if (!ids) return Internal("output container is null");
  std::vector<std::vector<int>> out;
  const auto st = SampleEncode(std::vector<std::string_view>{input}, nbest_size, alpha, &out);
  if (!st.ok()) return st;
  *ids = std::move(out[0]);
  return util::OkStatus();
}
util::Status SentencePieceProcessor::SampleEncode(std::string_view input, int nbest_size, float alpha,
                                                  std::vector<std::string> *pieces) const {
  if (!engine_) return status();
  if (!pieces) return Internal("output container is null");
  std::vector<std::vector<std::string>> out;
  const auto st = SampleEncode(std::vector<std::string_view>{input}, nbest_size, alpha, &out);
  if (!st.ok()) return st;
  *pieces = std::move(out[0]);
  return util::OkStatus();
}
std::vector<std::vector<std::string>> SentencePieceProcessor::NBestEncodeAsPieces(std::string_view input, int nbest_size) const {
  std::vector<std::vector<std::string>> out;
  NBestEncode(input, nbest_size, &out).IgnoreError();
  return out;
}
std::vector<std::vector<int>> SentencePieceProcessor::NBestEncodeAsIds(std::string_view input, int nbest_size) const {
  std::vector<std::vector<int>> out;
  NBestEncode(input, nbest_size, &out).IgnoreError();
  return out;
}
std::vector<std::string> SentencePieceProcessor::SampleEncodeAsPieces(std::string_view input, int nbest_size, float alpha) const {
  std::vector<std::string> out;
  SampleEncode(input, nbest_size, alpha, &out).IgnoreError();
  return out;
}
std::vector<int> SentencePieceProcessor::SampleEncodeAsIds(std::string_view input, int nbest_size, float alpha) const {
  std::vector<int> out;
  SampleEncode(input, nbest_size, alpha, &out).IgnoreError();
  return out;
}

util::Status SentencePieceProcessor::Encode(std::string_view input, std::vector<int> *ids) const {
  if (!engine_) return status();
  if (!ids) return Internal("output container is null");
  std::vector<std::vector<int>> out;
  const auto st = Encode(std::vector<std::string_view>{input}, &out);
  if (!st.ok()) return st;
  *ids = std::move(out[0]);
  return util::OkStatus();
}

util::Status SentencePieceProcessor::Encode(std::string_view input, std::vector<std::string> *pieces) const {
  if (!engine_) return status();
  if (!pieces) return Internal("output container is null");
  std::vector<std::vector<std::string>> out;
  const auto st = Encode(std::vector<std::string_view>{input}, &out);
  if (!st.ok()) return st;
  *pieces = std::move(out[0]);
  return util::OkStatus();
}

// the value-returning forms swallow errors (macro at sentencepiece_processor.h:432-436)
std::vector<std::string> SentencePieceProcessor::EncodeAsPieces(std::string_view input) const {
  std::vector<std::string> out;
  Encode(input, &out).IgnoreError();
  return out;
}
std::vector<int> SentencePieceProcessor::EncodeAsIds(std::string_view input) const {
  std::vector<int> out;
  Encode(input, &out).IgnoreError();
  return out;
}

}  // namespace sentencepiece
