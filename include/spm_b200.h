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

/* The id effect of the encode extra options: SentencePieceProcessor::ApplyExtraOptions
 * (src/sentencepiece_processor.cc:1019-1064) after SetEncodeExtraOptions, and the Python binding's
 * encode(add_bos=, add_eos=, reverse=) (python/src/sentencepiece/sentencepiece.i:138-145).  Any list of
 * REVERSE / BOS / EOS options applied in order turns a sentence's ids r into
 *   prefix ++ (reverse ? reversed(r) : r) ++ suffix
 * with constant id lists: BOS prepends to the prefix, EOS appends to the suffix, REVERSE swaps the two, reverses
 * both and flips `reverse`.  UNK_PIECE changes piece strings only.  Parsing option strings and looking up the
 * bos / eos pieces stay with the caller.
 * The frame is engine state, like the live types: every later call that returns encode ids writes it, until it is
 * set again; all zeros / NULL restores the plain output.  It applies to spm_encode_ids, spm_encode_ids_device
 * (total_ids and the SPM_ERR_CAPACITY answer include it), every candidate of spm_nbest_encode, spm_sample_encode_ids
 * and every sample of spm_sample_encode_and_score.  Empty sentences are framed too, as the reference frames the empty
 * encode; the exception is spm_sample_encode_and_score, where the reference returns no sample for an empty sentence
 * and its slots stay empty.  spm_encode_spans keeps returning the raw segmentation, on which tok_end is defined.
 * Every id must lie in [0, vocab) and n_prefix, n_suffix <= 64, else SPM_ERR_ARG. */
int spm_engine_set_encode_frame(spm_engine *e, const int32_t *prefix, uint32_t n_prefix, int reverse,
                                const int32_t *suffix, uint32_t n_suffix);

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
 * sentence, stored at n2o[norm_offsets[i] + i ...]).  The ids are the raw segmentation, on which tok_end is defined:
 * the encode frame (spm_engine_set_encode_frame) is not applied here. */
int spm_encode_spans(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n,
                     const int32_t **ids, const uint32_t **tok_end, const uint64_t **id_offsets,
                     const char **normalized, const uint64_t **norm_offsets, const uint32_t **n2o);

/* The n2o entry of a sentence whose reference norm_to_orig is empty: its input is empty (src/normalizer.cc:77-79), or
 * remove_extra_whitespaces drops all of it as heading whitespace (:97-100).  A sentence that normalizes to nothing
 * otherwise gets {consumed}, as the reference does. */
#define SPM_NORM_TO_ORIG_EMPTY 0xFFFFFFFFu

/* Replaces SentencePieceProcessor::Normalize (src/sentencepiece_processor.cc:933-950, all three overloads) and
 * Normalizer::Normalize (src/normalizer.cc:71-186) for n sentences: the model's own normalizer, with the prefix matcher
 * of its USER_DEFINED pieces (those stay verbatim, normalizer.cc:201-205), for unigram and BPE models alike.  The
 * encode frame does not apply.  Inputs as spm_encode_ids.
 * out (engine-owned pinned memory, valid until the next call): normalized[norm_offsets[i] .. norm_offsets[i+1]) is
 *   sentence i's text, U+2581 as its three bytes; with_offsets != 0: n2o holds its norm_to_orig,
 *   norm_offsets[i+1]-norm_offsets[i]+1 entries stored at n2o[norm_offsets[i] + i ...] (the spm_encode_spans layout),
 *   the one entry SPM_NORM_TO_ORIG_EMPTY where the reference's norm_to_orig is empty; with_offsets == 0: *n2o = NULL
 *   (n2o itself may then be NULL).
 * Argument errors and "sentence too long" as spm_encode_ids; n == 0 succeeds with norm_offsets = {0}. */
int spm_normalize(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int with_offsets,
                  const char **normalized, const uint64_t **norm_offsets, const uint32_t **n2o);

/* Replaces the per-sentence loop over SentencePieceProcessor::Encode(absl::string_view, std::vector<std::string>*)
 * (src/sentencepiece_processor.cc:379-390 -> :547-636) for n sentences, with the encode frame
 * (spm_engine_set_encode_frame) applied to pieces and ids alike.  The piece of a token is IdToPiece(id), except for
 * the unknown id: its surface in the normalized text (a run of unknown characters is one token).
 * unk_piece: NULL keeps the normalized surface of unknown tokens; otherwise it is the string that UNK_PIECE
 *   writes (trainer_spec.unk_piece; the caller owns option parsing, as for the frame).
 * sep: -1 = pieces abut; 0..255 = that byte between consecutive pieces of a sentence (spm_encode uses ' ').
 * out (engine-owned pinned memory, valid until the next call): text[text_offsets[i] .. text_offsets[i+1]) is sentence
 *   i's pieces; piece_end[id_offsets[i] + k] is the exclusive end of its k-th piece relative to text_offsets[i]
 *   (the tok_end convention of spm_encode_spans); ids / id_offsets are the framed ids of those pieces, identical to
 *   what spm_encode_ids returns.
 * The ids come from the kernels of spm_encode_ids; only sentences that hold the unknown id (and only when unk_piece is
 * NULL) are encoded a second time, by the path of spm_encode_spans, for their normalized text
 * (spm_engine_info.last_unk_detour counts them).  Argument errors as spm_encode_ids. */
int spm_encode_pieces(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n,
                      const char *unk_piece, size_t unk_piece_len, int sep,
                      const char **text, const uint64_t **text_offsets, const uint32_t **piece_end,
                      const int32_t **ids, const uint64_t **id_offsets);

/* Replaces the per-sentence loop over SentencePieceProcessor::Encode(absl::string_view, SentencePieceText*) /
 * EncodeAsImmutableProto (src/sentencepiece_processor.cc:547-636 and ApplyExtraOptions, :1019-1064) for n sentences:
 * the ids of every token and where it came from in the input.
 * out (engine-owned pinned memory, valid until the next call):
 *   ids / id_offsets: exactly what spm_encode_ids returns under the current encode frame;
 *   begin[k] / end[k]: the byte range of ids[k] in its sentence's input (relative to offsets[i]), as the reference's
 *     SentencePieceText.pieces(k).begin() / end().  A normal or user-defined piece covers the input that normalized to
 *     it; an unknown token (a whole run of unknown characters) the run's input; with byte fallback, the byte tokens of
 *     an unknown character all begin at the character, the last ends after it and the others end where they begin.
 *     Frame entries equal to eos_id get (len, len), every other frame entry (0, 0); the frame reverses the body
 *     together with its offsets.  The surface of a token is input[begin, end).
 *   text != NULL: text / text_offsets / piece_end are exactly spm_encode_pieces with the same unk_piece and sep.
 *     text == NULL: no pieces are written (text_offsets and piece_end may be NULL too); unk_piece and sep are only
 *     checked.
 * Sentences that hold the unknown id are encoded a second time by the spans path for the extents of their unknown
 * tokens, with or without unk_piece (spm_engine_info.last_unk_detour counts them).  Argument errors as
 * spm_encode_pieces, and "sentence too long" as spm_normalize; n == 0 succeeds with id_offsets = {0}. */
int spm_encode_offsets(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int32_t eos_id,
                       const char *unk_piece, size_t unk_piece_len, int sep,
                       const int32_t **ids, const uint64_t **id_offsets,
                       const uint32_t **begin, const uint32_t **end,
                       const char **text, const uint64_t **text_offsets, const uint32_t **piece_end);

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

/* The same batch as rows of one width, the layout a model consumes: an int32 [n, w] id tensor in row-major order.
 * Row i holds F_i, sentence i's framed ids exactly as spm_encode_ids_device returns them, and pad_id (any int32,
 * -1 included) in every other cell.  d_lengths[i] receives the number of real cells of row i.
 *   width: 0 = the longest |F_i| of the batch; otherwise the fixed width w.
 *   SPM_PAD_TRUNCATE: a row longer than a fixed width keeps its frame, prefix ++ body[:width - np - ns] ++ suffix,
 *     where body is the framed list's middle part (already reversed under a reversing frame) and np / ns the frame's
 *     prefix and suffix sizes; width < np + ns is SPM_ERR_ARG.  Without it, a row longer than a fixed width fails the
 *     call with SPM_ERR_CAPACITY and the longest row length in *width_out.
 *   SPM_PAD_LEFT: the real ids sit at the end of their row (left padding, as batched generation prompts want).
 * Rows are written at stride w into d_out (capacity out_capacity int32); if n * w > out_capacity the call returns
 * SPM_ERR_CAPACITY with *width_out = w.  In both capacity errors nothing is written to d_out or d_lengths; the batch
 * has been encoded, and a retry with room enough encodes it again.  On success *width_out = w.
 * Device pointers, stream, synchronisation and argument rules as spm_encode_ids_device; n == 0 writes nothing and sets
 * *width_out = 0.  There is no offsets scan: one synchronisation reads the longest row back. */
enum { SPM_PAD_TRUNCATE = 1, SPM_PAD_LEFT = 2 };
int spm_encode_ids_device_padded(spm_engine *e, const char *d_bytes, const uint64_t *d_offsets, size_t n,
                                 uint64_t total_bytes, int32_t *d_out, uint64_t out_capacity, uint32_t width,
                                 int32_t pad_id, uint32_t flags, int32_t *d_lengths, uint32_t *width_out,
                                 void *stream);

/* The padded rows of spm_encode_ids_device_padded together with every token's begin / end in its input, aligned cell
 * for cell (what other fast tokenizers call an offsets mapping): the ids and offsets a token-classification, span or
 * question-answering model consumes, for a batch already in device memory.
 *   d_ids (int32 [n, w], capacity out_capacity cells), d_lengths and *width_out: exactly what
 *     spm_encode_ids_device_padded writes for the same batch, encode frame, width, pad_id and SPM_PAD_TRUNCATE /
 *     SPM_PAD_LEFT flags, including both SPM_ERR_CAPACITY cases (nothing written; *width_out the longest row or the
 *     width used).
 *   d_spans (int32 [n, w, 2], room for 2 * out_capacity int32, 8-byte aligned): cell (i, j) holds (begin, end) of the token in
 *     d_ids[i, j]: for a real cell what spm_encode_offsets returns for that token with the same eos_id; frame entries
 *     equal to eos_id get (len, len) and other frame entries (0, 0); a reversing frame reverses the offsets with the
 *     body; truncation keeps exactly the cells the id row keeps; pad cells get (0, 0).
 *   Units: byte offsets in the sentence's input (relative to d_offsets[i]); with SPM_OFFSETS_CHARS every offset p
 *     becomes the index of the character that holds byte min(p, len) (len: the number of characters), the table of
 *     the reference's ConvertToUnicodeSpans, characters being stepped by their lead byte's length as the reference
 *     does, malformed input included.  The rows then hold exactly EncodeAsImmutableProto's begin / end.
 * Argument rules, stream, "returns after the work is done on `stream`" and n == 0 as spm_encode_ids_device_padded;
 * flags other than these three bits are SPM_ERR_ARG.  Sentences whose offsets do not add up to their normalized
 * length ("all normalized characters are not consumed") give SPM_ERR_ENCODE, and a sentence too long for the offsets
 * path SPM_ERR_UNSUPPORTED, as in spm_encode_offsets.  Sentences that hold the unknown id are encoded a second time by
 * the spans path (spm_engine_info.last_unk_detour).  No per-sentence data crosses PCIe: the host reads back a fixed
 * number of status words (the detour count, the longest row, the chunk plan). */
enum { SPM_OFFSETS_CHARS = 4 };
int spm_encode_offsets_device_padded(spm_engine *e, const char *d_bytes, const uint64_t *d_offsets, size_t n,
                                     uint64_t total_bytes, int32_t eos_id,
                                     int32_t *d_ids, int32_t *d_spans, uint64_t out_capacity, uint32_t width,
                                     int32_t pad_id, uint32_t flags, int32_t *d_lengths, uint32_t *width_out,
                                     void *stream);

/* A device batch as overlapping windows of one width (what other fast tokenizers call overflowing tokens with a
 * stride): long inputs for extractive QA, long-document classification, token classification or retrieval chunks,
 * with every token kept.
 * For sentence i: F_i = prefix ++ body_i ++ suffix is the framed list spm_encode_ids_device returns (body_i already
 * reversed when the frame reverses), np / ns the prefix and suffix sizes, L_i = |body_i|.  For width w and an overlap
 * `stride`: B = w - np - ns, which must satisfy B >= 1 and 0 <= stride < B (else SPM_ERR_ARG); step = B - stride.
 *   Sentence i gets m_i = 1 row if L_i <= B, else 1 + ceil((L_i - B) / step) rows.  Window j holds
 *   prefix ++ body_i[j*step : min(j*step + B, L_i)] ++ suffix: every window carries the whole frame, every window after
 *   the first starts step tokens later and holds at least one token the one before it does not, and an empty sentence
 *   gets one row that holds the frame only.
 *   Rows are ordered by sentence, then window; R = sum m_i.  Row r is written at d_ids + r * w with pad_id in the other
 *   cells (SPM_PAD_LEFT: the real cells at the end of the row); d_lengths[r] = its real cells; d_row_sentence[r] = i
 *   (the overflow-to-sample mapping); d_row_first[r] = j*step, the index in body_i of the window's first body token.
 *   d_spans (optional, int32 [R, w, 2], 8-byte aligned; NULL = no offsets): cell (r, c) holds the (begin, end)
 *   spm_encode_offsets_device_padded gives the same token with the same eos_id; frame entries equal to eos_id get
 *   (len, len), other frame entries and pad cells (0, 0); SPM_OFFSETS_CHARS gives characters as there.  Without
 *   d_spans, no normalizer walk runs: the ids cost what spm_encode_ids_device_padded's cost.
 * When every L_i <= B the result is exactly spm_encode_ids_device_padded / spm_encode_offsets_device_padded with width
 * w: the same rows, lengths and spans, R = n, row_sentence = 0..n-1, row_first = 0.
 * R is known only after the encode and comes back with the call's status words: if R > rows_capacity the call returns
 * SPM_ERR_CAPACITY with *rows_out = R and writes nothing to any output (a retry with room encodes the batch again);
 * on success *rows_out = R.  SPM_ERR_ARG: width == 0, SPM_PAD_TRUNCATE (windows never drop tokens), SPM_OFFSETS_CHARS
 * without d_spans, other flags, null pointers, a misaligned d_spans.  SPM_ERR_UNSUPPORTED: a body longer than
 * 2^31 - 1 ids, or R over 2^31 - 1.  With d_spans: a sentence too long for the offsets path, SPM_ERR_ENCODE on
 * unconsumed characters and the unknown-id detour (spm_engine_info.last_unk_detour) as in
 * spm_encode_offsets_device_padded.  Stream, "returns after the work is done on `stream`" and n == 0 (*rows_out = 0)
 * as the padded calls.  No per-token data crosses PCIe: the host reads back a fixed number of status words. */
int spm_encode_windows_device(spm_engine *e, const char *d_bytes, const uint64_t *d_offsets, size_t n,
                              uint64_t total_bytes, uint32_t width, uint32_t stride, int32_t pad_id, uint32_t flags,
                              int32_t eos_id, int32_t *d_ids, int32_t *d_spans, uint64_t rows_capacity,
                              int32_t *d_lengths, int32_t *d_row_sentence, int32_t *d_row_first,
                              uint64_t *rows_out, void *stream);

/* Sentence pairs: two inputs per padded row, for cross-encoders and rerankers (query, passage), NLI and paraphrase
 * classifiers (premise, hypothesis) and extractive QA (question, context).
 * The device batch holds 2n sentences (d_offsets: 2n + 1 entries): pair i is A_i = sentence i and B_i = sentence n + i,
 * each as the raw ids spm_encode_ids_device gives it with no frame.  The engine's encode frame does not apply to this
 * call (it stays set for later calls); the call's own template does: prefix, middle and suffix (host arrays of at most
 * 64 ids each in [0, vocab); T = n_prefix + n_middle + n_suffix).  The row of pair i before truncation is
 *   prefix ++ A_i ++ middle ++ B_i ++ suffix
 * which covers T5's "A </s> B </s>", "<s> A </s></s> B </s>" and "[CLS] A [SEP] B [SEP]".
 * Truncation (`truncation`), with a = |A_i|, b = |B_i| and the body room Bt = width - T (width > T required):
 *   SPM_PAIR_TRUNC_NONE: nothing is cut.  width == 0 takes the longest row of the batch as w; a fixed width that some
 *     row exceeds gives SPM_ERR_CAPACITY with the longest row in *width_out.
 *   SPM_PAIR_TRUNC_LONGEST_FIRST: while a + b > Bt, the last id of the longer body is dropped (B's on ties); that is
 *     a' = min(a, max(Bt - b, ceil(Bt / 2))), b' = min(b, Bt - a').
 *   SPM_PAIR_TRUNC_ONLY_FIRST / _ONLY_SECOND: only that member is cut, from its end, to the room r = Bt - |other|.
 *   Only right truncation is offered.  These rules are this project's definitions, not a claim of parity with any other
 *   library's truncation.
 * SPM_PAIR_OVERFLOW (flag; with ONLY_FIRST / ONLY_SECOND only): the cut member is not dropped but split into windows as
 *   spm_encode_windows_device splits a body, with room r_i = Bt - |other_i| and step s_i = r_i - stride per pair.  Pair
 *   i gets 1 row if the member fits, else 1 + ceil((L - r_i) / s_i) rows (L: the member's length); window j holds
 *   the member's ids [j*s_i, min(j*s_i + r_i, L)), and every row repeats the template and the whole other member.
 *   Without the flag, stride must be 0.
 * A pair under ONLY_* that needs cutting but has r_i < 1 (or r_i <= stride under overflow) cannot be laid out: the call
 * returns SPM_ERR_CAPACITY with *rows_out = 0 and in *width_out the least width at which every pair would pass.
 * Outputs, for R rows (R = n without the overflow flag; rows ordered by pair, then window) of width w (*width_out):
 *   d_ids int32 [R, w]: the row, then pad_id (SPM_PAD_LEFT: the real cells at the end of the row).
 *   d_type_ids int32 [R, w] (required): 0 on the prefix, A's cells and the middle; 1 on B's cells and the suffix; 0 on
 *     pad cells.
 *   d_lengths, d_row_pair, d_row_first int32 [R]: the real cells; the pair of the row; the index of the window's first
 *     id within the windowed member's ids (0 without the overflow flag).
 *   d_spans (optional, int32 [R, w, 2], 8-byte aligned; NULL = no offsets): an A cell holds its token's (begin, end) in
 *     A's input, a B cell its token's (begin, end) in B's input, as spm_encode_offsets gives them; template and pad
 *     cells (0, 0).  SPM_OFFSETS_CHARS counts characters as spm_encode_offsets_device_padded does.  A sentence too long
 *     for the offsets path, SPM_ERR_ENCODE on unconsumed characters and the unknown-id detour are as there.
 * Capacities: d_lengths, d_row_pair and d_row_first hold rows_capacity entries, d_ids and d_type_ids cells_capacity
 * cells and d_spans 2 * cells_capacity.  R > rows_capacity or R * w > cells_capacity gives SPM_ERR_CAPACITY with R in
 * *rows_out and w in *width_out; like the width failure above, it writes nothing to any output (a retry encodes the
 * batch again).  On success *rows_out = R, *width_out = w.
 * SPM_ERR_ARG: null pointers, unknown flags or strategy, SPM_PAD_TRUNCATE, a template list over 64 ids or an id
 * outside [0, vocab), width 0 or width <= T with any strategy but NONE, the overflow flag with NONE or LONGEST_FIRST,
 * stride != 0 without it, SPM_OFFSETS_CHARS without d_spans, a misaligned d_spans, 2n over the sentence limit.
 * SPM_ERR_UNSUPPORTED: a row of 2^32 - 1 ids or more, R over 2^31 - 1.  n == 0 succeeds with *rows_out = 0.  Stream
 * and "returns after the work is done on `stream`" as the padded calls.  No per-token data crosses PCIe: the template
 * goes up and a fixed number of status words come back. */
enum {
  SPM_PAIR_TRUNC_NONE = 0, SPM_PAIR_TRUNC_LONGEST_FIRST = 1, SPM_PAIR_TRUNC_ONLY_FIRST = 2,
  SPM_PAIR_TRUNC_ONLY_SECOND = 3
};
enum { SPM_PAIR_OVERFLOW = 8 };
int spm_encode_pairs_device(spm_engine *e, const char *d_bytes, const uint64_t *d_offsets, size_t n,
                            uint64_t total_bytes, const int32_t *prefix, uint32_t n_prefix, const int32_t *middle,
                            uint32_t n_middle, const int32_t *suffix, uint32_t n_suffix, uint32_t width,
                            uint32_t truncation, uint32_t stride, int32_t pad_id, uint32_t flags, int32_t *d_ids,
                            int32_t *d_type_ids, int32_t *d_spans, uint64_t rows_capacity, uint64_t cells_capacity,
                            int32_t *d_lengths, int32_t *d_row_pair, int32_t *d_row_first, uint64_t *rows_out,
                            uint32_t *width_out, void *stream);

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

/* The same three calls with pieces, as spm_encode_pieces writes them: NBestEncodeAsPieces, SampleEncodeAsPieces and
 * SampleEncodeAndScoreAsPieces over a batch.  unk_piece, sep and the packed layout are those of spm_encode_pieces with
 * one list per candidate (per sample): text[text_offsets[j] .. text_offsets[j+1]) is list j's pieces,
 * piece_end[cand_offsets[j] + k] the end of its k-th piece relative to text_offsets[j], ids the framed ids.  Every
 * id, cand_offset, score and n_cands equals what the ids call returns, and each call consumes the engine's generator
 * exactly as its ids call does.  Argument checks and errors are those of the ids calls and of spm_encode_pieces.
 *   spm_nbest_encode_pieces: candidate-major as spm_nbest_encode; empty slots stay empty and unframed.
 *     nbest_size <= 1 gives spm_encode_pieces' result with score 0.  The unknown tokens' surfaces come from the n-best
 *     kernels themselves (token ends and the normalized text of sentences whose lattice holds an unknown character).
 *   spm_sample_encode_pieces: as spm_sample_encode_ids; nbest_size > 1 writes the pieces of the drawn candidates on
 *     the device, nbest_size < 0 writes them on the host next to the ids of the lattice draw.
 *   spm_sample_encode_and_score_pieces: as spm_sample_encode_and_score (num_samples slots per sentence; an empty
 *     sentence leaves its slots empty).
 * Outputs are engine-owned memory, valid until the next call on this engine. */
int spm_nbest_encode_pieces(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int nbest_size,
                            const char *unk_piece, size_t unk_piece_len, int sep, const char **text,
                            const uint64_t **text_offsets, const uint32_t **piece_end, const int32_t **ids,
                            const uint64_t **cand_offsets, const float **scores, const uint32_t **n_cands);
int spm_sample_encode_pieces(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int nbest_size,
                             float alpha, const char *unk_piece, size_t unk_piece_len, int sep, const char **text,
                             const uint64_t **text_offsets, const uint32_t **piece_end, const int32_t **ids,
                             const uint64_t **id_offsets);
int spm_sample_encode_and_score_pieces(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n,
                                       int num_samples, float alpha, int wor, int include_best, const char *unk_piece,
                                       size_t unk_piece_len, int sep, const char **text, const uint64_t **text_offsets,
                                       const uint32_t **piece_end, const int32_t **ids, const uint64_t **cand_offsets,
                                       const float **scores);

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

/* Replaces SentencePieceProcessor::Decode(const std::vector<int>& ids, SentencePieceText*) /
 * DecodeIdsAsImmutableProto (src/sentencepiece_processor.cc:766-925) for n id lists: the text and where every token's
 * surface lies in it.  text / text_offsets are byte for byte what spm_decode_ids returns for the same lists;
 * tok_end[k - id_offsets[0]] is the end of token k's surface, relative to text_offsets[i] of its list.  The surfaces
 * tile the text in token order (SetSurface, :822-828), so token k begins where token k-1 ends and the first token of a
 * list at 0: a CONTROL token's surface is empty, an UNKNOWN token's is unk_surface, and in a run of BYTE pieces the
 * first c-1 tokens of a valid c-byte character get an empty surface and the last one the whole character, while an
 * invalid byte's token gets U+FFFD.  Outputs are engine-owned pinned memory, valid until the next call.  Arguments,
 * errors and refusals are those of spm_decode_ids; n == 0 succeeds. */
int spm_decode_offsets(spm_engine *e, const int32_t *ids, const uint64_t *id_offsets, size_t n, const char **text,
                       const uint64_t **text_offsets, const uint32_t **tok_end);

/* Decode of device-resident id rows, e.g. a generation output tensor [n, >= row_len] still on the GPU: row i starts at
 * element i * row_stride of d_ids (int32 when id_bytes == 4, int64 when 8 -- a cast of int64 ids to int32 would wrap
 * large values silently) and holds min(row_len, d_lengths[i]) ids (row_len when d_lengths is NULL; a negative length is
 * 0), cut further just before its first stop_id when stop_id >= 0.  Cells after a row's end are never read or
 * validated.  The text of a row is exactly spm_decode_ids of its id list, with the same errors ("Invalid id: N", where
 * int64 ids outside the int32 range are invalid too) and the same outputs: engine-owned pinned text and
 * text_offsets[n+1], valid until the next call on this engine.  Models with a denormalizer_spec charsmap:
 * SPM_ERR_UNSUPPORTED.  `stream` as in spm_encode_ids_device; the call returns after the text has arrived. */
int spm_decode_ids_device(spm_engine *e, const void *d_ids, uint32_t id_bytes, uint64_t row_stride, size_t n,
                          uint32_t row_len, const int32_t *d_lengths, int64_t stop_id, const char **text,
                          const uint64_t **text_offsets, void *stream);

/* The state of one streamed row of spm_decode_stream_device, in device memory.  16 bytes; all zeros is a fresh row. */
typedef struct {
  uint64_t text_bytes; /* bytes of text returned for this row so far */
  uint32_t ids;        /* ids consumed so far, held ones included */
  uint8_t flags;       /* bit 0: done; bits 1-2: held byte ids (0..3); bit 3: the leading-U+2581 rule no longer applies
                          (the reference's is_bos_ws would be false at the next token: bos_ws_seen, or text non-empty) */
  uint8_t held[3];     /* the byte values of the held BYTE ids, in order */
} spm_decode_stream_state;

/* Streaming Decode of device-resident generation output: each call takes the next ids of n sequences and returns, per
 * row, the text those ids settle.  Row i's new ids are read as spm_decode_ids_device reads a row (int32 / int64 at
 * d_ids + i * row_stride elements, min(row_len, d_lengths[i]) of them, cut before the first stop_id when stop_id >= 0),
 * so a [n, 1] column slice of one step's sampled ids or a [n, k] block of accepted speculative ids is passed as it is.
 * d_state[i] (16-byte aligned device memory) carries row i from call to call.
 * Let S be every id row i has consumed, this call's included.  The held tail of S is empty unless S ends in a run of
 * BYTE pieces in which a UTF-8 decision is pending: from the first position p of that run whose lead byte b0 needs more
 * bytes than the run has left (2 for 110xxxxx, 3 for 1110xxxx, 4 for 11110xxx; every other byte needs 1), the rest of
 * the run is held, at most 3 ids.  Row i's text is Decode(S) from d_state[i].text_bytes up to the end of the last token
 * before the held tail (that token's end as spm_decode_offsets gives it).  So the texts of all a row's calls, through
 * the one that finishes it, concatenate to spm_decode_ids of all its ids, and each text is whole UTF-8 characters.
 * A row finishes in the call where its new ids stop at stop_id, or where d_final[i] != 0 (d_final: nullable int32 [n]):
 * its held bytes are then decoded as the reference decodes a run at the end of a list (U+FFFD per invalid byte), and
 * it is marked done.  A done row returns empty text, and its ids are neither read nor validated until the caller zeroes
 * its state, which starts a new sequence in that slot.
 * Outputs: engine-owned pinned text and text_offsets[n+1], valid until the next call on this engine.  Errors: an id
 * outside [0, vocab) gives SPM_ERR_ARG "Invalid id: N" (the whole int64 value), a BYTE piece not of the form <0xXX>
 * SPM_ERR_ENCODE, a row's id count above 2^32 - 1 SPM_ERR_UNSUPPORTED, as do models with a denormalizer_spec charsmap.
 * On any error no state changes and no text is returned: the new states are written to engine scratch and copied over
 * d_state on `stream` only after the call's status words read back clean.  n == 0 succeeds.  No per-row data goes to
 * the device; the text, its offsets and the status words come back.  `stream` as in spm_encode_ids_device; the call
 * returns after the text and the new states have arrived.  decode_extra_options are not applied. */
int spm_decode_stream_device(spm_engine *e, const void *d_ids, uint32_t id_bytes, uint64_t row_stride, size_t n,
                             uint32_t row_len, const int32_t *d_lengths, int64_t stop_id, const int32_t *d_final,
                             spm_decode_stream_state *d_state, const char **text, const uint64_t **text_offsets,
                             void *stream);

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
  uint64_t last_unk_detour;         /* spm_encode_pieces: sentences encoded again for the surfaces of unknown tokens */
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
