// offsets_kernel.cuh -- K11, spm_encode_offsets: the begin / end of every token of an encode in the input, as
// SentencePieceProcessor::PopulateSentencePieceText (src/sentencepiece_processor.cc:547-636) and ApplyExtraOptions
// (:1019-1064) set them in SentencePieceText.
//
// Let c be the normalized bytes consumed before a token and n2o the sentence's norm_to_orig:
//   - a normal or user-defined piece of L bytes (U+2581 as three): begin = n2o[c], end = n2o[c + L];
//   - the unknown id (a run of unknown characters, merged into one token by the encode): the same, with L the extent
//     of the run, which the spans path gives (tok_end) for the sentences that hold it;
//   - byte fallback: an unknown character of k bytes is k byte tokens of one byte each.  All of them begin at
//     n2o[c_char], where c_char is the character's first byte; the first k - 1 end there too, the last at
//     n2o[c_char + k].  The normalized text is valid UTF-8, so a byte token whose byte is a continuation byte
//     (10xxxxxx) belongs to the character of the token before it;
//   - the frame: an entry equal to eos_id gets (len, len), every other entry (0, 0) (BOS prepends (0, 0), EOS
//     appends (text.size(), text.size())); REVERSE reverses the body together with its offsets.
//
// One warp per sentence: normalize_tile (kernels.cuh) writes the sentence's n2o into its own slab, as K10 does
// (normalize_kernel.cuh, the same slab layout and bound); then the body is walked 32 tokens per trip, each lane takes
// its token's normalized length, a warp scan turns the lengths into c, and begin / end go straight to the token's
// place in the framed, packed output.  Sentence i's output starts at id_offsets[i] + i * (np + ns): the body has as
// many ids as the raw segmentation.  The lengths must add up to the normalized length ("all normalized characters
// are not consumed", which the reference reports as an error): status bit 0 otherwise.  Status bit 1: a sentence
// normalized to more bytes than its slab holds (the bound of normalize_kernel.cuh says it cannot).
//
// The byte-fallback grouping assumes the normalized text is valid UTF-8, so that every unknown piece is exactly one
// character.  The normalizer guarantees that for every input (a malformed byte becomes U+FFFD) as long as the
// model's charsmap targets are valid UTF-8; the engine refuses models whose targets are not.
#ifndef SPM_B200_OFFSETS_KERNEL_CUH_
#define SPM_B200_OFFSETS_KERNEL_CUH_

#include <cstdint>

#include "device_model.h"
#include "kernels.cuh"
#include "normalize_kernel.cuh"
#include "pieces_kernel.cuh"

namespace spm_b200 {

constexpr uint8_t kTypeByte = 6;  // SPM_BYTE

struct KOffsets {
  // raw segmentation, unknown-surface subset, piece table and frame, as K9 reads them (pieces_src)
  KPieces P;
  // this launch's sentences: first .. first + n - 1 of the batch; their input at bytes + offsets[i] - offsets[first]
  const uint8_t *bytes;
  const uint64_t *offsets;  // [batch + 1]
  uint32_t first, n;
  uint32_t expand;  // as KNormalize
  uint8_t *slab_text;
  uint32_t *slab_n2o;
  int32_t eos_id;
  // out, framed and packed
  uint32_t *begin;
  uint32_t *end;
  int32_t *out_ids;                    // null: the ids are written by K9
  unsigned long long *out_id_offsets;  // with out_ids
  uint32_t *status;  // bit 0: lengths do not add up; bit 1: slab overflow
};

__global__ void __launch_bounds__(256, 1) offsets_kernel(const KModel M, const KOffsets A) {
  const Tile T;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  const KPieces &P = A.P;
  const uint32_t fr = P.F.np + P.F.ns;
  const uint64_t base = A.offsets[A.first];
  for (uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < A.n; s += warps) {
    const uint32_t sent = A.first + s;
    const uint64_t lo = A.offsets[sent] - base, hi = A.offsets[sent + 1] - base;
    const uint32_t len = static_cast<uint32_t>(hi - lo);
    const unsigned long long start = norm_slab_start(lo, s, A.expand);
    TileMem tm{};
    tm.text = A.slab_text + start;
    tm.n2o = A.slab_n2o + start;
    tm.ncap = static_cast<uint32_t>(norm_slab_start(hi, s + 1, A.expand) - start - 1);
    const NormResult r = normalize_tile<true>(M, T, A.bytes + lo, len, tm);
    const PiecesSrc src = pieces_src(P, sent);
    const unsigned long long raw = P.id_offsets[sent];
    const uint32_t L = src.L;
    const unsigned long long out = raw + static_cast<unsigned long long>(sent) * fr;
    const bool overflow = r.n > tm.ncap;
    bool bad = overflow || L != P.id_offsets[sent + 1] - raw;
    if (A.out_ids && T.lane == 0) {
      if (sent == 0) A.out_id_offsets[0] = 0;
      A.out_id_offsets[sent + 1] = P.id_offsets[sent + 1] + static_cast<unsigned long long>(sent + 1) * fr;
    }
    // the frame
    for (uint32_t t = T.lane; t < fr; t += 32) {
      const int32_t id = P.F.ids[t];
      const uint32_t o = id == A.eos_id ? len : 0u;
      const unsigned long long k = out + (t < P.F.np ? t : L + t);
      A.begin[k] = o;
      A.end[k] = o;
      if (A.out_ids) A.out_ids[k] = id;
    }
    // the body
    uint32_t c0 = 0;      // normalized bytes before this trip
    uint32_t cchar = 0;   // c of the character the last byte token of the previous trip belongs to
    for (uint32_t tb = 0; tb < L && !bad; tb += 32) {
      const uint32_t q = tb + T.lane;
      const bool act = q < L;
      int32_t id = 0;
      uint32_t w = 0;
      bool byte = false;
      if (act) {
        id = src.ids[q];
        byte = __ldg(M.types + id) == kTypeByte;
        if (src.tok_end) w = src.tok_end[q] - (q ? src.tok_end[q - 1] : 0u);
        else if (byte) w = 1;
        else w = __ldg(P.pc_off + id + 1) - __ldg(P.pc_off + id);
      }
      const uint32_t c1 = c0 + T.incl_scan(w);  // end of this token in the normalized text
      const uint32_t c = c1 - w;
      // byte tokens: a continuation byte continues the character of the token before it (the normalized text is
      // valid UTF-8, see the top of this file)
      const bool cont = byte && c < r.n && (tm.text[c] & 0xC0u) == 0x80u;
      uint32_t head = act && !cont ? c : 0u;
      if (T.lane == 0 && cont) head = cchar;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = T.shfl(head, T.lane >= d ? T.lane - d : T.lane);
        head = head > v ? head : v;
      }
      bool next_cont = T.shfl(cont, T.lane < 31 ? T.lane + 1 : 31) && T.lane < 31;
      if (T.lane == 31 && q + 1 < L) {
        const int32_t nid = src.ids[q + 1];
        next_cont = __ldg(M.types + nid) == kTypeByte && c1 < r.n && (tm.text[c1] & 0xC0u) == 0x80u;
      }
      if (act) {
        if (c1 > r.n) {
          bad = true;
        } else {
          const uint32_t b = tm.n2o[byte ? head : c];
          const uint32_t e = byte && next_cont ? b : tm.n2o[c1];
          const unsigned long long k = out + P.F.np + (P.F.reverse ? L - 1u - q : q);
          A.begin[k] = b;
          A.end[k] = e;
          if (A.out_ids) A.out_ids[k] = id;
        }
      }
      bad = T.ballot(bad) != 0u;
      c0 = T.shfl(c1, 31);
      cchar = T.shfl(head, 31);
    }
    if (!bad && c0 != r.n) bad = true;
    if (bad && T.lane == 0) atomicOr(A.status, overflow ? 2u : 1u);
  }
}

}  // namespace spm_b200
#endif
