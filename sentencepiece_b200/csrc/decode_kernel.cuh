// decode_kernel.cuh -- K7: batched Decode(ids) -> text (SURVEY.md 8f item 2, the step after the path).
//
// Reference: SentencePieceProcessor::Decode(const std::vector<int>&, SentencePieceText*)
// (src/sentencepiece_processor.cc:765-925), text only:
//   * every id must be in range (:915-918);
//   * CONTROL pieces are invisible, UNKNOWN pieces become TrainerSpec.unk_surface (:779-790);
//   * while the text is still empty and no leading U+2581 has been consumed yet (`is_bos_ws`,
//     :879-887), a piece that starts with U+2581 loses it when add_dummy_prefix or
//     remove_extra_whitespaces is set; with remove_extra_whitespaces the state is not closed by
//     that, so every leading U+2581 goes until the text is non-empty (:792-807);
//   * U+2581 -> ' ' everywhere else (:809);
//   * a run of BYTE pieces is reassembled one Unicode character at a time, every structurally
//     invalid byte becoming U+FFFD (:817-876).
// The engine precomputes, per id, the decoded bytes (U+2581 already replaced) and an info word, so
// the kernel is a gather: one WARP per id list, one token per lane; the bos rule is evaluated with a
// ballot ("the first token that would end the bos state"), output positions with a warp scan.
// Lists that contain BYTE pieces take a sequential path on lane 0 (the UTF-8 reassembly is a
// character-by-character loop in the reference too).  Text is appended to a temporary buffer in
// completion order; the scan / gather kernels of the encode path put it into list order.
#ifndef SPM_B200_DECODE_KERNEL_CUH_
#define SPM_B200_DECODE_KERNEL_CUH_

#include <cstdint>
#include <type_traits>

namespace spm_b200 {

// dec_info word
constexpr uint32_t kDecKindMask = 3u;     // 0 normal, 1 control, 2 unknown, 3 byte
constexpr uint32_t kDecKindNormal = 0u, kDecKindControl = 1u, kDecKindUnknown = 2u, kDecKindByte = 3u;
constexpr uint32_t kDecLeadWs = 1u << 2;  // normal piece that starts with U+2581
constexpr uint32_t kDecBadByte = 1u << 3; // BYTE piece that is not "<0xXX>" (PieceToByte fails, model_interface.cc:214-230)
constexpr uint32_t kDecByteShift = 8;

// spm_decode_stream_state as the kernel sees it (16 bytes): word = flags | held[0] << 8 | held[1] << 16 | held[2] << 24
struct alignas(16) DecStreamState {
  unsigned long long text_bytes;
  uint32_t ids;
  uint32_t word;
};
constexpr uint32_t kStDone = 1u;          // the row has finished
constexpr uint32_t kStHeldShift = 1;      // bits 1-2: held byte ids (0..3)
constexpr uint32_t kStHeldMask = 3u << kStHeldShift;
constexpr uint32_t kStBosOver = 1u << 3;  // the next non-byte token is decoded with is_bos_ws false

struct KDecode {
  const int32_t *ids;
  const unsigned long long *id_offsets;  // [n+1]
  uint32_t n;
  int32_t vocab;
  const uint32_t *dec_off;   // [vocab+1] into dec_bytes
  const uint8_t *dec_bytes;
  const uint32_t *dec_info;  // [vocab]
  uint32_t strip;            // add_dummy_prefix || remove_extra_whitespaces
  uint32_t rm;               // remove_extra_whitespaces
  uint8_t *tmp;              // text in completion order
  unsigned long long tmp_cap;
  unsigned long long *cursor;
  unsigned long long *sent_start;  // [n]
  uint32_t *sent_count;            // [n]
  uint32_t *status;                // [1] error: 2 = id out of range, 1 = malformed byte piece; [2] overflow; [3] the offending id
  // ROWS mode (decode_warp_kernel<IdT, true>): list i is ids[i * row_stride ..] of row_len[i] ids, and an id out of
  // range is also stored whole, sign-extended, at cursor[1]
  unsigned long long row_stride;
  const uint32_t *row_len;  // [n]
  // ENDS mode (decode_warp_kernel<int32_t, false, true>): tok_end[k] = the end of id k's surface in its list's text, for
  // every k in [id_offsets[0], id_offsets[n]) (indexed like ids).  The surfaces tile the text in token order
  // (SetSurface, :822-828), so the end of token k-1 is the begin of token k.
  uint32_t *tok_end;
};

// STREAM mode's own arguments (decode_warp_kernel<IdT, true, false, true>, spm_decode_stream_device), a second kernel
// parameter so that KDecode, and with it the code of the other modes, stays as it is.  Rows are read as in ROWS mode,
// but row i's length comes from decode_row_end (row_cap, lengths, stop_id) and KDecode::row_len is not used; row i
// continues the stream described by state_in[i] and leaves its new state in state_out[i].  fin (nullable): rows to
// finish.
struct KDecodeStream {
  const DecStreamState *state_in;
  DecStreamState *state_out;
  const int32_t *lengths;
  const int32_t *fin;
  long long stop_id;
  uint32_t row_cap;
};
struct KNoStream {};
template <bool STREAM>
using KStreamArg = typename std::conditional<STREAM, KDecodeStream, KNoStream>::type;

// IsValidDecodeUTF8 (src/util.h:173-176 over DecodeUTF8, src/util.cc:51-84): bytes consumed by one valid character
// at b[0..avail), 0 if the byte is structurally invalid (the caller then consumes one byte).
__device__ __forceinline__ uint32_t dec_utf8_valid(const uint32_t *b, uint32_t avail) {
  const uint32_t b0 = b[0];
  auto trail = [](uint32_t x) { return (x & 0xC0u) == 0x80u; };
  if (b0 < 0x80u) return 1;
  if (avail >= 2 && (b0 & 0xE0u) == 0xC0u) {
    const uint32_t cp = ((b0 & 0x1Fu) << 6) | (b[1] & 0x3Fu);
    return (trail(b[1]) && cp >= 0x80u) ? 2u : 0u;
  }
  if (avail >= 3 && (b0 & 0xF0u) == 0xE0u) {
    const uint32_t cp = ((b0 & 0x0Fu) << 12) | ((b[1] & 0x3Fu) << 6) | (b[2] & 0x3Fu);
    return (trail(b[1]) && trail(b[2]) && cp >= 0x800u && (cp < 0xD800u || cp >= 0xE000u)) ? 3u : 0u;
  }
  if (avail >= 4 && (b0 & 0xF8u) == 0xF0u) {
    const uint32_t cp = ((b0 & 0x07u) << 18) | ((b[1] & 0x3Fu) << 12) | ((b[2] & 0x3Fu) << 6) | (b[3] & 0x3Fu);
    return (trail(b[1]) && trail(b[2]) && trail(b[3]) && cp >= 0x10000u && cp <= 0x10FFFFu) ? 4u : 0u;
  }
  return 0;
}

// The bytes dec_utf8_valid reads to decide at lead byte b0: with that many available (or the run ended) its result is
// final.  1 for ASCII and for bytes that cannot lead a character, else the length the lead byte announces.
__device__ __forceinline__ uint32_t dec_utf8_need(uint32_t b0) {
  return (b0 & 0xE0u) == 0xC0u ? 2u : (b0 & 0xF0u) == 0xE0u ? 3u : (b0 & 0xF8u) == 0xF0u ? 4u : 1u;
}

// Sequential restatement for one list (lists with BYTE pieces); WRITE = false only counts.  IdT: the ids' type (every
// id has been checked to lie in [0, vocab) before).  ENDS (with WRITE): also the end of every token's surface, as
// ProcessBytePieces sets them: the first c-1 byte tokens of a valid c-byte character end where they begin and the last
// one after the character, an invalid byte's token after its U+FFFD.
// STREAM: the list continues a stream whose state word (DecStreamState::word) is *sw: its held byte values come first,
// the leading-U+2581 rule starts from its kStBosOver bit, and unless kStDone is set a trailing byte run whose next
// decision lacks bytes (fewer than dec_utf8_need of them) is held instead of decoded.  *sw is updated to the new state.
template <bool WRITE, typename IdT = int32_t, bool ENDS = false, bool STREAM = false>
__device__ __forceinline__ uint32_t decode_list_sequential(const KDecode &D, unsigned long long a, uint32_t L, uint8_t *out,
                                                           uint32_t *sw = nullptr) {
  const IdT *ids = reinterpret_cast<const IdT *>(D.ids);
  uint32_t n = 0;  // bytes of text so far
  bool is_bos_ws = true, bos_ws_seen = false;
  uint32_t i = 0;
  uint32_t h = 0, held = 0;  // STREAM: held bytes before the ids, and after them
  if constexpr (STREAM) {
    h = (*sw & kStHeldMask) >> kStHeldShift;
    L += h;
    is_bos_ws = !(*sw & kStBosOver);
  }
  // STREAM: the info word of element k of the list, the held bytes first, then the ids
  auto info_at = [&](uint32_t k) -> uint32_t {
    if (k < h) return kDecKindByte | (((*sw >> (8 + 8 * k)) & 0xFFu) << kDecByteShift);
    return __ldg(D.dec_info + static_cast<int32_t>(ids[a + (k - h)]));
  };
  while (i < L) {
    int32_t id;
    uint32_t info;
    if constexpr (STREAM) {
      id = i < h ? 0 : static_cast<int32_t>(ids[a + (i - h)]);
      info = info_at(i);
    } else {
      id = static_cast<int32_t>(ids[a + i]);
      info = __ldg(D.dec_info + id);
    }
    const uint32_t kind = info & kDecKindMask;
    if (kind == kDecKindByte) {
      // one Unicode character from the run of byte pieces that starts here
      uint32_t b[4] = {info >> kDecByteShift, 0, 0, 0};
      uint32_t avail = 1;
      while (avail < 4 && i + avail < L) {
        uint32_t inf2;
        if constexpr (STREAM) inf2 = info_at(i + avail);
        else inf2 = __ldg(D.dec_info + static_cast<int32_t>(ids[a + i + avail]));
        if ((inf2 & kDecKindMask) != kDecKindByte) break;
        b[avail] = inf2 >> kDecByteShift;
        ++avail;
      }
      if constexpr (STREAM) {
        if (!(*sw & kStDone) && i + avail == L && avail < dec_utf8_need(b[0])) {
          held = avail;  // <= 3: the decision at i waits for more bytes
          for (uint32_t k = 0; k < avail; ++k) held |= b[k] << (8 + 8 * k);
          break;
        }
      }
      const uint32_t c = dec_utf8_valid(b, avail);
      if (c == 0) {
        if (WRITE) { out[n] = 0xEF; out[n + 1] = 0xBF; out[n + 2] = 0xBD; }
        n += 3;
        if constexpr (ENDS) D.tok_end[a + i] = n;
        i += 1;
      } else {
        if (WRITE) for (uint32_t k = 0; k < c; ++k) out[n + k] = static_cast<uint8_t>(b[k]);
        if constexpr (ENDS) for (uint32_t k = 0; k < c; ++k) D.tok_end[a + i + k] = k + 1 == c ? n + c : n;
        n += c;
        i += c;
      }
      continue;
    }
    if (bos_ws_seen || n != 0) is_bos_ws = false;
    const uint32_t off = __ldg(D.dec_off + id);
    uint32_t len = __ldg(D.dec_off + id + 1) - off;
    uint32_t skip = 0;
    bool has_bos_ws = false;
    if (kind == kDecKindNormal && is_bos_ws && D.strip && (info & kDecLeadWs)) {
      skip = 1;  // the ' ' that stands for the leading U+2581
      has_bos_ws = !D.rm;
    }
    len -= skip;
    if (WRITE) for (uint32_t k = 0; k < len; ++k) out[n + k] = __ldg(D.dec_bytes + off + skip + k);
    n += len;
    if constexpr (ENDS) D.tok_end[a + i] = n;
    bos_ws_seen = has_bos_ws;
    ++i;
  }
  if constexpr (STREAM) {
    // the held bytes are decoded before any later token, so they too close the rule
    const bool over = !is_bos_ws || bos_ws_seen || n != 0 || held != 0;
    *sw = (*sw & kStDone) | ((held & 3u) << kStHeldShift) | (held & ~0xFFu) | (over ? kStBosOver : 0u);
  }
  return n;
}

// The end of row `row` of a padded id tensor, for the whole warp: min(row_len, lengths[row]) ids (row_len when lengths
// is null; a negative length is 0), cut before the first stop_id in them when stop_id >= 0.
template <typename IdT>
__device__ __forceinline__ uint32_t decode_row_end(const IdT *ids, unsigned long long row_stride, uint32_t row,
                                                   uint32_t row_len, const int32_t *lengths, long long stop_id,
                                                   uint32_t lane) {
  uint32_t L = row_len;
  if (lengths) L = min(L, static_cast<uint32_t>(max(lengths[row], 0)));
  if (stop_id >= 0) {
    const IdT *r = ids + static_cast<unsigned long long>(row) * row_stride;
    for (uint32_t base = 0; base < L; base += 32) {
      const uint32_t t = base + lane;
      const uint32_t hit = __ballot_sync(0xFFFFFFFFu, t < L && static_cast<long long>(r[t]) == stop_id);
      if (hit) {
        L = base + __ffs(hit) - 1u;
        break;
      }
    }
  }
  return L;
}

// STREAM: row i's new state after `bytes` more text, `ids` more ids and with state word w.  text_bytes and ids are read
// again rather than kept in registers through the row.
__device__ __forceinline__ void dec_put_state(const KDecodeStream &S, uint32_t i, uint32_t bytes, uint32_t ids, uint32_t w) {
  const DecStreamState o = S.state_in[i];
  S.state_out[i] = DecStreamState{o.text_bytes + bytes, o.ids + ids, w};
}

// IdT, ROWS: the ids are int32 or int64, and list i is either [id_offsets[i], id_offsets[i+1]) (packed) or row_len[i]
// ids from i * row_stride (rows of a padded [n, row_stride] tensor).  ENDS: also write D.tok_end (packed lists only).
// Template flags, so that the packed int32 instantiation keeps its code.
// STREAM (with ROWS): each row is the next ids of a stream, described by S (KDecodeStream).  A done row writes no text and
// keeps its state; its ids are not read.  Otherwise the row's text is the part of its stream's text that this call
// settles, and the new state goes to state_out (copied over state_in by the host only when the call succeeds).
template <typename IdT = int32_t, bool ROWS = false, bool ENDS = false, bool STREAM = false>
__global__ void __launch_bounds__(256) decode_warp_kernel(const KDecode D, const KStreamArg<STREAM> S) {
  static_assert(ROWS || sizeof(IdT) == 4, "packed lists are int32");
  static_assert(!(ROWS && ENDS), "token ends are written for packed lists only");
  static_assert(ROWS || !STREAM, "streams are rows");
  const IdT *ids = reinterpret_cast<const IdT *>(D.ids);
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t sent = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; sent < D.n; sent += warps) {
    unsigned long long a, len64;
    // STREAM: the row's state word, with kStDone when this call finishes the row; ovf: its id count would overflow
    uint32_t word = 0;
    bool ovf = false;
    if constexpr (STREAM) {
      const DecStreamState ss = S.state_in[sent];
      word = ss.word;
      if (word & kStDone) {
        if (lane == 0) { D.sent_start[sent] = 0; D.sent_count[sent] = 0; S.state_out[sent] = ss; }
        continue;
      }
      a = static_cast<unsigned long long>(sent) * D.row_stride;
      len64 = decode_row_end(ids, D.row_stride, sent, S.row_cap, S.lengths, S.stop_id, lane);
      // the row stops at stop_id when the cut above shortened it
      const uint32_t lim = S.lengths ? min(S.row_cap, static_cast<uint32_t>(max(S.lengths[sent], 0))) : S.row_cap;
      if (len64 < lim || (S.fin && S.fin[sent] != 0)) word |= kStDone;
      ovf = ss.ids + len64 > 0xFFFFFFFFull;
    } else if constexpr (ROWS) {
      a = static_cast<unsigned long long>(sent) * D.row_stride;
      len64 = D.row_len[sent];
    } else {
      a = D.id_offsets[sent];
      len64 = D.id_offsets[sent + 1] - a;
    }
    const uint32_t L = static_cast<uint32_t>(len64);
    // ---- pass 0: ids in range, any BYTE piece ----
    uint32_t err = len64 > 0x7FFFFFFFull ? 2u : 0u;  // 2 = id out of range (checked first by the reference), 1 = malformed byte piece
    if constexpr (STREAM) if (ovf) err = 3;  // 3 = the stream's id count overflows
    int32_t err_id = 0;
    bool has_byte = false, stop = err != 0;
    for (uint32_t base = 0; base < L && !stop; base += 32) {
      const uint32_t t = base + lane;
      if (t < L) {
        const IdT id = ids[a + t];
        if (id < 0 || id >= D.vocab) {
          err = 2;
          err_id = static_cast<int32_t>(id);
          if constexpr (ROWS) atomicExch(D.cursor + 1, static_cast<unsigned long long>(static_cast<long long>(id)));
        } else {
          const uint32_t info = __ldg(D.dec_info + id);
          has_byte |= (info & kDecKindMask) == kDecKindByte;
          if ((info & kDecBadByte) && !err) { err = 1; err_id = id; }
        }
      }
      stop = __any_sync(0xFFFFFFFFu, err != 0);
    }
    if (stop) {
      if (err) {
        atomicMax(D.status + 1, err);
        atomicExch(D.status + 3, static_cast<uint32_t>(err_id));
      }
      if (lane == 0) { D.sent_start[sent] = 0; D.sent_count[sent] = 0; }
      continue;
    }
    if constexpr (STREAM) has_byte |= (word & kStHeldMask) != 0;
    has_byte = __any_sync(0xFFFFFFFFu, has_byte);
    uint32_t total = 0;
    unsigned long long pos = 0;
    if (has_byte) {
      // ---- sequential path on lane 0 ----
      if (lane == 0) {
        uint32_t sw = word;
        total = decode_list_sequential<false, IdT, false, STREAM>(D, a, L, nullptr, &sw);
        pos = atomicAdd(D.cursor, static_cast<unsigned long long>(total));
        if (pos + total > D.tmp_cap) { atomicOr(D.status + 2, 1u); total = 0; }
        else decode_list_sequential<true, IdT, ENDS, STREAM>(D, a, L, D.tmp + pos, &word);
        D.sent_start[sent] = pos;
        D.sent_count[sent] = total;
        if constexpr (STREAM) dec_put_state(S, sent, total, L, word);
      }
      __syncwarp();
      continue;
    }
    // ---- parallel path: one token per lane, two passes (count, write) ----
    for (int pass = 0; pass < 2; ++pass) {
      bool bos_over = !D.strip;
      if constexpr (STREAM) bos_over = bos_over || (word & kStBosOver);
      uint32_t run = 0;
      for (uint32_t base = 0; base < L; base += 32) {
        const uint32_t t = base + lane;
        const bool valid = t < L;
        uint32_t info = kDecKindControl, off = 0, n0 = 0;
        if (valid) {
          const int32_t id = static_cast<int32_t>(ids[a + t]);
          info = __ldg(D.dec_info + id);
          off = __ldg(D.dec_off + id);
          n0 = __ldg(D.dec_off + id + 1) - off;
        }
        const uint32_t kind = info & kDecKindMask;
        const bool lead = kind == kDecKindNormal && (info & kDecLeadWs);
        // would this token end the bos state if it were processed in it?
        const bool ends = valid && (kind == kDecKindUnknown ? n0 > 0
                                    : kind == kDecKindNormal ? (lead ? (!D.rm || n0 > 1) : n0 > 0)
                                                             : false);
        const uint32_t mask = __ballot_sync(0xFFFFFFFFu, ends);
        const bool in_bos = !bos_over && (mask & ((1u << lane) - 1u)) == 0u;
        const uint32_t skip = (in_bos && lead) ? 1u : 0u;
        const uint32_t len = n0 - skip;
        bos_over = bos_over || mask != 0u;
        uint32_t incl = len;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, d);
          if (lane >= static_cast<uint32_t>(d)) incl += v;
        }
        if (pass == 1) {
          if constexpr (ENDS) if (valid) D.tok_end[a + t] = run + incl;
          uint8_t *dst = D.tmp + pos + run + (incl - len);
          const uint8_t *src = D.dec_bytes + off + skip;
          const uint32_t mx = __reduce_max_sync(0xFFFFFFFFu, len);
          for (uint32_t k = 0; k < mx; ++k)
            if (k < len) dst[k] = __ldg(src + k);
        }
        run += __shfl_sync(0xFFFFFFFFu, incl, 31);
      }
      if (pass == 0) {
        total = run;
        if (lane == 0) {
          pos = atomicAdd(D.cursor, static_cast<unsigned long long>(total));
          if (pos + total > D.tmp_cap) atomicOr(D.status + 2, 1u);
          D.sent_start[sent] = pos;
          D.sent_count[sent] = pos + total > D.tmp_cap ? 0u : total;
        }
        pos = __shfl_sync(0xFFFFFFFFu, pos, 0);
        if (pos + total > D.tmp_cap) break;
      }
      if constexpr (STREAM)
        if (pass == 1 && lane == 0)
          dec_put_state(S, sent, total, L, word | (bos_over ? kStBosOver : 0u));
    }
  }
}

// Row ends of a padded id tensor for decode_warp_kernel<IdT, true>, one warp per row: row i holds
// min(row_len, lengths[i]) ids (row_len when lengths is null; a negative length is 0), cut before its first stop_id
// when stop_id >= 0.  Ids past a row's end are never read.
template <typename IdT>
__global__ void __launch_bounds__(256) decode_row_len_kernel(const IdT *ids, unsigned long long row_stride, uint32_t n,
                                                             uint32_t row_len, const int32_t *lengths, long long stop_id,
                                                             uint32_t *len_out) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < n; row += warps) {
    const uint32_t L = decode_row_end(ids, row_stride, row, row_len, lengths, stop_id, lane);
    if (lane == 0) len_out[row] = L;
  }
}

}  // namespace spm_b200
#endif
