/* spm_b200.h -- C ABI of the H100 batched subword-encode engine.
 *
 * This is the drop-in boundary for ONE path of google/sentencepiece: the batched
 *   normalize -> (unigram Viterbi | BPE merge) -> PopulateSentencePieceText(id path)
 * pipeline that SentencePieceProcessor::Encode runs per sentence
 * (reference: src/sentencepiece_processor.cc:638-651).  Everything else in the
 * reference (training, decoding, protobuf, CLI) stays the reference's.
 *
 * Conventions
 *   - plain C, no C++/torch types; every function returns 0 on success and a
 *     non-zero code on failure, with text available from spm_last_error();
 *     the C++ host layer wraps a failure into util::Status(kInternal, text)
 *     exactly as the reference's CHECK_OR_RETURN does (src/util.h:394-399).
 *   - there is NO CPU fallback: if no CUDA device is usable, create fails.
 *   - a batch is a packed byte buffer + n+1 offsets (sentence i =
 *     bytes[offsets[i], offsets[i+1]) ), any bytes allowed (NUL, malformed UTF-8).
 *   - results are bit-identical to the reference's ids for the same model/input.
 *
 * Each entry point cites the reference interface it replaces.
 */
#ifndef SPM_B200_H_
#define SPM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct spm_engine spm_engine; /* opaque */

/* ModelProto::SentencePiece::Type (src/sentencepiece_model.proto:296-304) */
enum spm_piece_type {
  SPM_NORMAL = 1, SPM_UNKNOWN = 2, SPM_CONTROL = 3, SPM_USER_DEFINED = 4, SPM_UNUSED = 5, SPM_BYTE = 6
};
/* TrainerSpec::ModelType (src/sentencepiece_model.proto:48-53) */
enum spm_model_type { SPM_UNIGRAM = 1, SPM_BPE = 2 };

/* The model as the reference holds it after Load(): what
 * ModelInterface::InitializePieces (src/model_interface.cc:63-151),
 * unigram::Model::Model (src/unigram_model.cc:652-670) and
 * normalizer::Normalizer::Init (src/normalizer.cc:47-69) consume.  A maintainer
 * wiring the engine into SentencePieceProcessor::Load fills this from
 * model_proto_ (see INTEGRATION.md); all pointers are host memory, read only
 * during spm_engine_create. */
typedef struct {
  int32_t model_type;            /* trainer_spec.model_type: SPM_UNIGRAM | SPM_BPE */
  int32_t vocab_size;            /* pieces_size() */
  const char *piece_bytes;       /* pieces(i).piece(), concatenated */
  const uint32_t *piece_off;     /* [vocab_size+1] byte offsets into piece_bytes */
  const float *scores;           /* pieces(i).score() */
  const uint8_t *types;          /* pieces(i).type()  */
  uint8_t byte_fallback;                 /* trainer_spec.byte_fallback */
  uint8_t treat_whitespace_as_suffix;    /* trainer_spec.treat_whitespace_as_suffix */
  uint8_t add_dummy_prefix;              /* normalizer_spec.add_dummy_prefix */
  uint8_t remove_extra_whitespaces;      /* normalizer_spec.remove_extra_whitespaces */
  uint8_t escape_whitespaces;            /* normalizer_spec.escape_whitespaces */
  uint8_t reserved_[3];
  const void *charsmap;          /* normalizer_spec.precompiled_charsmap verbatim; may be NULL */
  size_t charsmap_bytes;
} spm_model_desc;

/* Replaces the table-building half of SentencePieceProcessor::Load
 * (src/sentencepiece_processor.cc:242-281): ModelFactory::Create +
 * Normalizer ctor.  `device` is the CUDA ordinal this engine lives on
 * (one engine per GPU; one process per GPU in multi-GPU runs). */
int spm_engine_create(const spm_model_desc *desc, int device, spm_engine **out);

/* Same, from a serialized ModelProto (the bytes of a .model file):
 * SentencePieceProcessor::LoadFromSerializedProto (src/sentencepiece_processor.h:261).
 * Uses the engine's own wire-format reader (no protobuf dependency). */
int spm_engine_create_from_serialized(const void *model_proto, size_t len, int device, spm_engine **out);

void spm_engine_destroy(spm_engine *e);

/* Live piece types: SetVocabulary / ResetVocabulary mutate pieces(i).type in
 * place and the CPU models read them on every call
 * (src/sentencepiece_processor.cc:301-340, src/model_interface.h:217-225).
 * Call with the full types array after either. */
int spm_engine_set_types(spm_engine *e, const uint8_t *types);

/* Empties the engine's internal memo tables (today: the BPE word cache, which
 * remembers the ids of words that were merged before; results never depend on
 * it).  No counterpart in the reference -- bpe::Model has no state across
 * calls (src/bpe_model.cc:38-203).  For measurements that must not profit
 * from earlier batches; spm_engine_set_types empties the tables as well. */
int spm_engine_cache_reset(spm_engine *e);

/* Text of the last failure on this engine (or of the last failed create when
 * e == NULL).  Never NULL. */
const char *spm_last_error(const spm_engine *e);

/* ------------------------------------------------------------------------
 * Batch encode, HOST buffers (the end-to-end path).
 * Replaces the per-sentence loop over
 *   SentencePieceProcessor::Encode(absl::string_view, std::vector<int>*)
 * (src/sentencepiece_processor.cc:392-403; spm_encode's loop
 * src/spm_encode_main.cc:159-165; the Python batch entry
 * python/src/sentencepiece/sentencepiece.i:245-267).
 *
 * in : bytes / offsets[n+1] caller-owned host memory (pinned memory from
 *      spm_host_alloc gives full PCIe speed; pageable memory also works).
 * out: *ids, *id_offsets[n+1] engine-owned pinned host buffers, valid until the
 *      next call on this engine.  Sentence i's ids are
 *      ids[id_offsets[i] .. id_offsets[i+1]).
 * One call may be in flight per engine (calls are serialized internally). */
int spm_encode_ids(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n,
                   const int32_t **ids, const uint64_t **id_offsets);

/* As spm_encode_ids plus what EncodeAsPieces / the SentencePieceText overload
 * need (src/sentencepiece_processor.cc:379-390,547-636): for every output token
 * its exclusive end offset in the sentence's normalized text, the normalized
 * text itself and the normalized->original byte alignment (norm_to_orig,
 * src/normalizer.cc:181-183; norm_offsets[i+1]-norm_offsets[i]+1 entries per
 * sentence, stored at n2o[norm_offsets[i] + i ...]). */
int spm_encode_spans(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n,
                     const int32_t **ids, const uint32_t **tok_end, const uint64_t **id_offsets,
                     const char **normalized, const uint64_t **norm_offsets, const uint32_t **n2o);

/* ------------------------------------------------------------------------
 * Batch encode, DEVICE buffers (inputs already resident in HBM; used when the
 * caller keeps corpora on the GPU, and by bench.py for the kernel-only number).
 * d_bytes / d_offsets[n+1] are device pointers on the engine's device;
 * d_ids (capacity ids_capacity int32) and d_id_offsets[n+1] are caller-provided
 * device buffers.  *total_ids receives the number of ids produced.  Returns
 * SPM_ERR_CAPACITY (and the required size in *total_ids) if d_ids is too small.
 * `stream` is a cudaStream_t (NULL = the engine's own stream); the call returns
 * after the work has completed on that stream. */
int spm_encode_ids_device(spm_engine *e, const char *d_bytes, const uint64_t *d_offsets, size_t n,
                          uint64_t total_bytes, int32_t *d_ids, uint64_t ids_capacity,
                          uint64_t *d_id_offsets, uint64_t *total_ids, void *stream);

/* ------------------------------------------------------------------------
 * N-best and sampling (unigram models; BASELINE.json config 5).
 *
 * spm_nbest_encode replaces SentencePieceProcessor::NBestEncode(input, nbest_size, ids)
 * (src/sentencepiece_processor.cc:653-676 -> unigram::Model::NBestEncode,
 * src/unigram_model.cc:695-721): for every sentence up to nbest_size candidate id sequences in
 * the reference's order (libstdc++ heap order among ties included) with their float scores.
 * nbest_size is clamped to [1, 1024] like the reference; nbest_size <= 1 gives the Viterbi
 * segmentation with score 0.  Candidate c of sentence i is
 * ids[cand_offsets[i*K + c] .. cand_offsets[i*K + c + 1]) with K = the clamped nbest_size;
 * n_cands[i] tells how many of the K slots are real.
 * Sentences of any length the encode path takes: sentences the per-lane kernel cannot hold (over
 * 512 normalized bytes, a lattice over 2112 nodes, a full hypothesis pool or agenda) are computed by
 * one warp each with 32-bit positions and a pool that grows on demand (counted in
 * spm_engine_info.last_deferred); device memory is then the only limit. */
int spm_nbest_encode(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int nbest_size,
                     const int32_t **ids, const uint64_t **cand_offsets, const float **scores,
                     const uint32_t **n_cands);

/* sentencepiece::SetRandomGeneratorSeed (src/sentencepiece_processor.h:731) for this engine's
 * std::mt19937; the engine draws for the sentences of a batch in order on one generator, which is
 * what the reference does on one thread. */
int spm_set_random_seed(spm_engine *e, uint32_t seed);

/* Replaces SentencePieceProcessor::SampleEncode(input, nbest_size, alpha, ids)
 * (src/sentencepiece_processor.cc:678-722), nbest_size <= 512 like the reference:
 *   nbest_size of 0 or 1: the plain Encode (:695-698);
 *   nbest_size > 1: the n-best list is computed on the GPU and one candidate is drawn with probability
 *     proportional to exp(alpha * score) exactly as the reference does (log-sum-exp in double,
 *     std::discrete_distribution on std::mt19937);
 *   nbest_size < 0: forward-filtering / backward-sampling over the whole lattice (:689-693 ->
 *     unigram::Model::SampleEncode, src/unigram_model.cc:511-542,722-739): the lattice and the forward
 *     scores come from the GPU, the backward draw runs on the host in sentence order on the engine's
 *     generator -- a seeded batch reproduces the reference's single-threaded stream bit for bit.
 * BPE models: alpha <= 0 is the plain Encode; BPE-dropout (alpha > 0, src/bpe_model.cc:132-139) is
 * not on the accelerated path (SPM_ERR_UNSUPPORTED). */
int spm_sample_encode_ids(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int nbest_size,
                          float alpha, const int32_t **ids, const uint64_t **id_offsets);

/* Replaces SentencePieceProcessor::CalculateEntropy(input, alpha, &entropy)
 * (src/sentencepiece_processor.cc:747-760 -> src/unigram_model.cc:266-291,857-864) for n sentences:
 * entropy[i] of the segmentation lattice of sentence i at inverse temperature alpha (unigram models).
 * Float results agree with the reference to rounding (the device's expf is not glibc's).
 * This and the lattice sampling of spm_sample_encode_ids / spm_sample_encode_and_score take
 * sentences of any length the encode path takes: those over 512 normalized bytes are computed by one
 * warp each with 32-bit positions (counted in spm_engine_info.last_deferred). */
int spm_calculate_entropy(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, float alpha,
                          const float **entropy);

/* Replaces SentencePieceProcessor::SampleEncodeAndScore(input, num_samples, alpha, wor, include_best, ...)
 * (src/sentencepiece_processor.cc:722-745 -> src/unigram_model.cc:741-855) with wor == 0 and
 * include_best == 0: num_samples independent lattice samples per sentence (one generator, sentence
 * order, sample order), each with score = sum(alpha * piece score) - log Z.  Sample c of sentence i is
 * ids[cand_offsets[i*num_samples + c] .. cand_offsets[i*num_samples + c + 1]), score scores[i*num_samples + c].
 * Sampling without replacement (wor) / include_best are not on the accelerated path. */
int spm_sample_encode_and_score(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int num_samples,
                                float alpha, int wor, int include_best, const int32_t **ids,
                                const uint64_t **cand_offsets, const float **scores);

/* Replaces SentencePieceProcessor::Decode(const std::vector<int>& ids, std::string* detokenized)
 * (src/sentencepiece_processor.cc:911-925 -> :765-909), one call for n id lists: `ids` is the packed
 * concatenation, id_offsets[n+1] delimits the lists (exactly what spm_encode_ids returns).  Outputs
 * (engine-owned pinned memory, valid until the next call on this engine): the concatenated UTF-8
 * text and text_offsets[n+1].  CONTROL pieces are invisible, UNKNOWN pieces become the model's
 * unk_surface, the leading U+2581 rule of add_dummy_prefix / remove_extra_whitespaces and the
 * UTF-8 reassembly of BYTE pieces (U+FFFD per invalid byte) follow the reference bit for bit.
 * Errors like the reference: an id outside [0, vocab) fails the call (SPM_ERR_ARG, "Invalid id: N").
 * Not on the device path: models with a denormalizer_spec charsmap (SPM_ERR_UNSUPPORTED) and
 * decode_extra_options (a host-side reordering the caller applies to the id lists). */
int spm_decode_ids(spm_engine *e, const int32_t *ids, const uint64_t *id_offsets, size_t n, const char **text,
                   const uint64_t **text_offsets);

/* TrainerSpec.unk_surface (src/sentencepiece_model.proto:228, read at sentencepiece_processor.cc:771-773) for
 * engines created from an spm_model_desc; engines created from a serialized ModelProto take it from the proto. */
int spm_engine_set_unk_surface(spm_engine *e, const char *surface, size_t bytes);

/* Pinned host memory helpers for callers that want zero staging copies. */
void *spm_host_alloc(size_t bytes);
void spm_host_free(void *p);

/* Introspection for benchmarks / tests. */
typedef struct {
  int32_t device;
  int32_t sm_count;
  int32_t model_type;
  int32_t vocab_size;
  int32_t unk_id;
  float min_score, max_score;       /* unigram_model.cc:657-664 (FLT_MIN quirk kept) */
  uint32_t trie_units;              /* units of the device piece trie */
  uint32_t trie_hot_units;          /* units staged into shared memory per CTA */
  uint32_t charsmap_units;
  uint64_t last_kernel_launches;    /* kernels launched by the last encode call */
  float last_kernel_ms;             /* device time of the last encode call's kernels (CUDA events) */
  float last_main_kernel_ms;        /* device time of the dominant (encode) kernel alone */
  uint64_t last_h2d_bytes, last_d2h_bytes;
  uint64_t last_deferred;           /* sentences that took the long-sentence path */
} spm_engine_info;
int spm_engine_get_info(const spm_engine *e, spm_engine_info *info);

/* Tuning knobs (benchmark use).  lanes_per_sentence selects the encode kernels: 1 = the lane
 * kernels, one sentence per lane (default), 32 = the general kernels, one sentence per warp, for
 * every batch; any other value is rejected.  smem_norm_cap = per-sentence shared-memory capacity
 * of the general kernels in normalized bytes; ctas_per_sm >= 32 is read as threads per CTA.
 * 0 keeps the current value. */
int spm_engine_set_tuning(spm_engine *e, int lanes_per_sentence, int smem_norm_cap, int ctas_per_sm);

enum spm_error {
  SPM_OK = 0, SPM_ERR_ARG = 1, SPM_ERR_MODEL = 2, SPM_ERR_CUDA = 3, SPM_ERR_CAPACITY = 4,
  SPM_ERR_ENCODE = 5, /* the reference would return a non-OK Status for some sentence */
  SPM_ERR_UNSUPPORTED = 6
};

#ifdef __cplusplus
}
#endif
#endif /* SPM_B200_H_ */
