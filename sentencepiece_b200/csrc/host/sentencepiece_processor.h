// host/sentencepiece_processor.h -- C++ host layer over the C ABI (include/spm_b200.h).
//
// Keeps the reference's public encode surface for this path -- class name, namespace,
// method names, argument meaning and error behaviour of
// /root/reference/src/sentencepiece_processor.h:238-460 (Load :245,
// LoadFromSerializedProto :261, SetEncodeExtraOptions :267, SetVocabulary :276,
// Encode(pieces) :295, Encode(ids) :299, EncodeAsPieces :453, EncodeAsIds :458) --
// so a caller such as spm_encode compiles against it unchanged, and adds the batch
// overloads that a GPU needs.  Single-sentence calls are batches of one.
// N-best and sampling (NBestEncode :318-324, SampleEncode :345-351, the value-returning forms :465-481,
// SetRandomGeneratorSeed :731) ride on the engine's n-best / sampling kernels; training stays the reference's.
#ifndef SPM_B200_HOST_SENTENCEPIECE_PROCESSOR_H_
#define SPM_B200_HOST_SENTENCEPIECE_PROCESSOR_H_

#include <cstdint>
#include <memory>
#include <string>
#include <string_view>
#include <vector>

struct spm_engine;

namespace sentencepiece {
namespace util {

enum class StatusCode : int { kOk = 0, kNotFound = 5, kInternal = 13 };

// Value-type status, ok() <=> no error (reference: sentencepiece_processor.h:54-76).
class Status {
 public:
  Status() = default;
  Status(StatusCode code, std::string msg) : code_(code), msg_(std::move(msg)) {}
  bool ok() const { return code_ == StatusCode::kOk; }
  StatusCode code() const { return code_; }
  const std::string &message() const { return msg_; }
  std::string ToString() const { return ok() ? "OK" : msg_; }
  void IgnoreError() const {}

 private:
  StatusCode code_ = StatusCode::kOk;
  std::string msg_;
};
inline Status OkStatus() { return Status(); }

}  // namespace util

class SentencePieceProcessor {
 public:
  SentencePieceProcessor();
  ~SentencePieceProcessor();
  SentencePieceProcessor(const SentencePieceProcessor &) = delete;
  SentencePieceProcessor &operator=(const SentencePieceProcessor &) = delete;

  // `device`: CUDA ordinal (one engine per GPU).  Set before Load.
  void SetDevice(int device) { device_ = device; }

  util::Status Load(std::string_view filename);
  util::Status LoadFromSerializedProto(std::string_view serialized);
  util::Status status() const;

  // "bos", "eos", "reverse", "unk"/"unk_piece", colon separated (sentencepiece_processor.cc:1067-1101)
  util::Status SetEncodeExtraOptions(std::string_view extra_option);
  util::Status SetVocabulary(const std::vector<std::string_view> &valid_vocab);
  util::Status ResetVocabulary();
  // "<piece>\t<freq>" lines; pieces with freq < threshold become UNUSED (sentencepiece_processor.cc:342-365)
  util::Status LoadVocabulary(std::string_view filename, int threshold);

  // ---- single sentence (reference signatures) ----
  util::Status Encode(std::string_view input, std::vector<std::string> *pieces) const;
  util::Status Encode(std::string_view input, std::vector<int> *ids) const;
  std::vector<std::string> EncodeAsPieces(std::string_view input) const;
  std::vector<int> EncodeAsIds(std::string_view input) const;

  // ---- n-best and sampling, single sentence (reference signatures, sentencepiece_processor.h:318-351,465-481).
  //      Errors like the reference: n-best is not available for BPE models (sentencepiece_processor.cc:662-663),
  //      nbest_size > 512 fails SampleEncode (:683). ----
  util::Status NBestEncode(std::string_view input, int nbest_size, std::vector<std::vector<std::string>> *pieces) const;
  util::Status NBestEncode(std::string_view input, int nbest_size, std::vector<std::vector<int>> *ids) const;
  util::Status SampleEncode(std::string_view input, int nbest_size, float alpha, std::vector<std::string> *pieces) const;
  util::Status SampleEncode(std::string_view input, int nbest_size, float alpha, std::vector<int> *ids) const;
  std::vector<std::vector<std::string>> NBestEncodeAsPieces(std::string_view input, int nbest_size) const;
  std::vector<std::vector<int>> NBestEncodeAsIds(std::string_view input, int nbest_size) const;
  std::vector<std::string> SampleEncodeAsPieces(std::string_view input, int nbest_size, float alpha) const;
  std::vector<int> SampleEncodeAsIds(std::string_view input, int nbest_size, float alpha) const;
  // ---- full-lattice operations of unigram models (sentencepiece_processor.h:364-379,401-410,483-500,521-526):
  //      num_samples lattice samples with their scores (wor / include_best are not on the accelerated path), and the
  //      entropy of the segmentation lattice ----
  std::vector<std::pair<std::vector<int>, float>> SampleEncodeAndScoreAsIds(std::string_view input, int num_samples,
                                                                            float alpha, bool wor, bool include_best) const;
  std::vector<std::pair<std::vector<std::string>, float>> SampleEncodeAndScoreAsPieces(std::string_view input, int num_samples,
                                                                                       float alpha, bool wor,
                                                                                       bool include_best) const;
  util::Status CalculateEntropy(std::string_view input, float alpha, float *entropy) const;
  float CalculateEntropy(std::string_view input, float alpha) const;
  util::Status CalculateEntropy(const std::vector<std::string_view> &inputs, float alpha, std::vector<float> *entropy) const;

  // ---- batch (what the reference's Python layer does with a thread pool,
  //      python/src/sentencepiece/sentencepiece.i:245-267) ----
  util::Status Encode(const std::vector<std::string_view> &inputs, std::vector<std::vector<int>> *ids) const;
  util::Status Encode(const std::vector<std::string_view> &inputs, std::vector<std::vector<std::string>> *pieces) const;
  // one device call for all sentences; the draws of SampleEncode are taken in input order on one generator, which is
  // what a single-threaded loop over the reference's SampleEncode does
  util::Status NBestEncode(const std::vector<std::string_view> &inputs, int nbest_size,
                           std::vector<std::vector<std::vector<int>>> *ids) const;
  util::Status NBestEncode(const std::vector<std::string_view> &inputs, int nbest_size,
                           std::vector<std::vector<std::vector<std::string>>> *pieces) const;
  util::Status SampleEncode(const std::vector<std::string_view> &inputs, int nbest_size, float alpha,
                            std::vector<std::vector<int>> *ids) const;
  util::Status SampleEncode(const std::vector<std::string_view> &inputs, int nbest_size, float alpha,
                            std::vector<std::vector<std::string>> *pieces) const;
  // zero-copy form: packed input, packed output owned by the engine until the next call
  util::Status EncodePacked(const char *bytes, const uint64_t *offsets, size_t n, const int32_t **ids,
                            const uint64_t **id_offsets) const;
  // the same for pieces with the extra options applied: sentence i is text[text_offsets[i] .. text_offsets[i+1]), its
  // pieces separated by the byte `sep` (-1: none); piece_end / id_offsets as spm_encode_pieces returns them
  util::Status EncodePiecesPacked(const char *bytes, const uint64_t *offsets, size_t n, int sep, const char **text,
                                  const uint64_t **text_offsets, const uint32_t **piece_end,
                                  const uint64_t **id_offsets) const;
  // NBestEncode / SampleEncode to pieces in the same layout, one list per candidate: candidate c of sentence i is list
  // i * K + c (K = nbest_size clamped to [1, 1024]), n_cands[i] of the K are real (spm_nbest_encode_pieces)
  util::Status NBestEncodePiecesPacked(const char *bytes, const uint64_t *offsets, size_t n, int nbest_size, int sep,
                                       const char **text, const uint64_t **text_offsets, const uint32_t **piece_end,
                                       const uint64_t **cand_offsets, const uint32_t **n_cands) const;
  util::Status SampleEncodePiecesPacked(const char *bytes, const uint64_t *offsets, size_t n, int nbest_size, float alpha,
                                        int sep, const char **text, const uint64_t **text_offsets,
                                        const uint32_t **piece_end, const uint64_t **id_offsets) const;

  // ---- Encode with offsets: what SentencePieceText (EncodeAsImmutableProto) holds per token, without protobuf.
  //      begin / end are byte offsets into the input (the reference's, before any ConvertToUnicodeSpans), surface is
  //      input[begin, end); the extra options apply as for EncodeAsPieces: bos / eos entries get (0, 0) and
  //      (size, size), reverse reverses the offsets with the pieces, unk replaces the piece string only. ----
  struct PieceSpan {
    std::string piece;
    int id = 0;
    std::string surface;
    uint32_t begin = 0, end = 0;
  };
  util::Status EncodeWithOffsets(std::string_view input, std::vector<PieceSpan> *pieces) const;
  // one device call for all sentences
  util::Status EncodeWithOffsets(const std::vector<std::string_view> &inputs,
                                 std::vector<std::vector<PieceSpan>> *pieces) const;
  // zero-copy form, the layout of spm_encode_offsets with the pieces (sep = -1): token k of sentence i is ids[k] with
  // begin[k] / end[k] relative to offsets[i], for k in [id_offsets[i], id_offsets[i+1]); owned by the engine until the
  // next call
  util::Status EncodeOffsetsPacked(const char *bytes, const uint64_t *offsets, size_t n, const int32_t **ids,
                                   const uint64_t **id_offsets, const uint32_t **begin, const uint32_t **end,
                                   const char **text, const uint64_t **text_offsets, const uint32_t **piece_end) const;

  // ---- Normalize (sentencepiece_processor.h:621-631): the model's normalizer, on the device (spm_normalize).
  //      norm_to_orig as the reference returns it: empty for empty input and for input that is all heading
  //      whitespace, else one entry per normalized byte and one for the end. ----
  util::Status Normalize(std::string_view input, std::string *normalized) const;
  util::Status Normalize(std::string_view input, std::string *normalized, std::vector<size_t> *norm_to_orig) const;
  std::string Normalize(std::string_view input) const;
  // one device call for all sentences; norm_to_orig may be null
  util::Status Normalize(const std::vector<std::string_view> &inputs, std::vector<std::string> *normalized,
                         std::vector<std::vector<size_t>> *norm_to_orig = nullptr) const;
  // zero-copy form, the layout of spm_normalize: sentence i is normalized[norm_offsets[i] .. norm_offsets[i+1]), its
  // norm_to_orig at n2o[norm_offsets[i] + i ...] (n2o null unless with_offsets), owned by the engine until the next call
  util::Status NormalizePacked(const char *bytes, const uint64_t *offsets, size_t n, bool with_offsets,
                               const char **normalized, const uint64_t **norm_offsets, const uint32_t **n2o) const;

  // ---- Decode(ids) (src/sentencepiece_processor.h Decode(const std::vector<int>&, std::string*)); the batch form is
  //      one device call for all lists.  An id outside [0, GetPieceSize()) fails the call like the reference's
  //      kOutOfRange (sentencepiece_processor.cc:915-918); decode_extra_options are not applied. ----
  util::Status Decode(const std::vector<int> &ids, std::string *detokenized) const;
  util::Status Decode(const std::vector<std::vector<int>> &ids, std::vector<std::string> *detokenized) const;
  std::string DecodeIds(const std::vector<int> &ids) const;

  // ---- Decode with offsets: what SentencePieceText (DecodeIdsAsImmutableProto) holds per token, without protobuf.
  //      piece is IdToPiece(id), surface is text[begin, end) (byte offsets into the decoded text, before any
  //      ConvertToUnicodeSpans); the surfaces tile the text in token order.  Errors as Decode. ----
  util::Status DecodeWithOffsets(const std::vector<int> &ids, std::string *text, std::vector<PieceSpan> *pieces) const;
  // one device call for all lists
  util::Status DecodeWithOffsets(const std::vector<std::vector<int>> &ids, std::vector<std::string> *text,
                                 std::vector<std::vector<PieceSpan>> *pieces) const;
  // zero-copy form, the layout of spm_decode_offsets: list i is text[text_offsets[i] .. text_offsets[i+1]), token k of it
  // ends at tok_end[k - id_offsets[0]] relative to text_offsets[i] and begins where token k-1 ends (0 for the first
  // token of a list); owned by the engine until the next call
  util::Status DecodeOffsetsPacked(const int32_t *ids, const uint64_t *id_offsets, size_t n, const char **text,
                                   const uint64_t **text_offsets, const uint32_t **tok_end) const;

  // ---- vocabulary accessors used by callers of the encode path ----
  int GetPieceSize() const;
  int PieceToId(std::string_view piece) const;
  const std::string &IdToPiece(int id) const;
  bool IsUnknown(int id) const { return id == unk_id_; }
  bool IsControl(int id) const;
  int unk_id() const { return unk_id_; }
  int bos_id() const;
  int eos_id() const;

 private:
  struct Impl;
  enum ExtraOption { REVERSE, BOS, EOS, UNK_PIECE };
  std::unique_ptr<Impl> impl_;
  spm_engine *engine_ = nullptr;
  int device_ = 0;
  int unk_id_ = -1;
  std::vector<ExtraOption> extra_;
  mutable bool seeded_ = false;  // the engine's generator took the global seed (first sampling call)
  void SeedOnce() const;
  // the id effect of extra_ as the engine writes it: frame_p_ ++ (r or reversed r) ++ frame_s_
  std::vector<int> frame_p_, frame_s_;
  bool frame_rev_ = false;
  util::Status ParseExtraOptions(std::string_view extra_option);
  // the unk_piece argument of the pieces calls: trainer_spec.unk_piece under UNK_PIECE, else null
  const std::string *UnkPiece() const;
};

// sentencepiece_processor.h:731 / util.cc:23-31: the seed every generator created afterwards starts from; this
// layer's generators live in the engines and take it at their first sampling call
void SetRandomGeneratorSeed(unsigned int seed);

}  // namespace sentencepiece
#endif
