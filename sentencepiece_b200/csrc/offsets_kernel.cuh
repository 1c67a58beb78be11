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
// Padded mode (offsets_padded_kernel, spm_encode_offsets_device_padded): the same walk, but the warp owns row `sent` of
// an [n, w] id tensor and its [n, w, 2] begin / end tensor and writes every cell of it, as write_padded_kernel
// (padded_kernel.cuh) lays the row out: the frame's prefix, body positions k < B (k = L - 1 - q under a reversing frame,
// else q; B = L, or min(L, w - np - ns) when truncating), the suffix, all shifted by w - real when padding on the left,
// and pad_id / (0, 0) in the other cells.  Tokens past B are walked (the lengths still have to add up) but not stored.
//
// Windows (spm_encode_windows_device) run K11 in packed mode, once per sentence, and write_window_spans_kernel gathers
// each window row from the packed lists: a token that lies in several windows is walked once.
// Sentence pairs (spm_encode_pairs_device) do the same over their 2n sentences with no frame, and
// write_pair_spans_kernel gathers each pair row.
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
#include "padded_kernel.cuh"
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
  // padded mode: rows of width w at pad_ids + sent * w and (begin, end) pairs at spans + sent * w; lengths[sent] =
  // the row's real cells
  int32_t *pad_ids;
  int2 *spans;
  int32_t *lengths;
  uint32_t w;
  int32_t pad_id;
  uint32_t truncate, left;
};

template <bool PADDED>
__device__ __forceinline__ void offsets_walk(const KModel &M, const KOffsets &A) {
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
    // padded mode: the row's kept body B, its real cells and the pad cells before them
    [[maybe_unused]] uint32_t B = L, lead = 0;
    [[maybe_unused]] int32_t *row_ids = nullptr;
    [[maybe_unused]] int2 *row_sp = nullptr;
    if constexpr (PADDED) {
      B = A.truncate ? min(L, A.w - fr) : L;
      const uint32_t real = B + fr;
      lead = A.left ? A.w - real : 0u;
      row_ids = A.pad_ids + static_cast<unsigned long long>(sent) * A.w;
      row_sp = A.spans + static_cast<unsigned long long>(sent) * A.w;
      for (uint32_t t = T.lane; t < A.w; t += 32)
        if (t - lead >= real) {  // (wraps for the leading pad cells)
          __stcs(row_ids + t, A.pad_id);
          __stcs(row_sp + t, make_int2(0, 0));
        }
      if (T.lane == 0) A.lengths[sent] = static_cast<int32_t>(real);
    } else if (A.out_ids && T.lane == 0) {
      if (sent == 0) A.out_id_offsets[0] = 0;
      A.out_id_offsets[sent + 1] = P.id_offsets[sent + 1] + static_cast<unsigned long long>(sent + 1) * fr;
    }
    // the frame
    for (uint32_t t = T.lane; t < fr; t += 32) {
      const int32_t id = P.F.ids[t];
      const uint32_t o = id == A.eos_id ? len : 0u;
      if constexpr (PADDED) {
        const uint32_t c = lead + (t < P.F.np ? t : B + t);
        __stcs(row_ids + c, id);
        __stcs(row_sp + c, make_int2(static_cast<int32_t>(o), static_cast<int32_t>(o)));
      } else {
        const unsigned long long k = out + (t < P.F.np ? t : L + t);
        A.begin[k] = o;
        A.end[k] = o;
        if (A.out_ids) A.out_ids[k] = id;
      }
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
          if constexpr (PADDED) {
            const uint32_t k = P.F.reverse ? L - 1u - q : q;
            if (k < B) {
              __stcs(row_ids + lead + P.F.np + k, id);
              __stcs(row_sp + lead + P.F.np + k, make_int2(static_cast<int32_t>(b), static_cast<int32_t>(e)));
            }
          } else {
            const unsigned long long k = out + P.F.np + (P.F.reverse ? L - 1u - q : q);
            A.begin[k] = b;
            A.end[k] = e;
            if (A.out_ids) A.out_ids[k] = id;
          }
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

__global__ void __launch_bounds__(256, 1) offsets_kernel(const KModel M, const KOffsets A) { offsets_walk<false>(M, A); }

__global__ void __launch_bounds__(256, 1) offsets_padded_kernel(const KModel M, const KOffsets A) {
  offsets_walk<true>(M, A);
}

// The offset rows of spm_encode_windows_device: one warp per window row, gathered from K11's framed, packed output
// (ids, begin, end; sentence i's list at id_offsets[i], np + L + ns entries).  Window f of sentence i takes the list's
// entries [0, np), [np + f, np + f + b) and [np + L, np + L + ns), b = min(L - f, w - np - ns), laid out as
// write_windows_kernel (padded_kernel.cuh) lays out its id rows, and pad_id / (0, 0) in the other cells.
__global__ void __launch_bounds__(256) write_window_spans_kernel(const int32_t *ids, const uint32_t *begin,
                                                                 const uint32_t *end,
                                                                 const unsigned long long *id_offsets, uint32_t rows,
                                                                 const int32_t *row_sentence, const int32_t *row_first,
                                                                 uint32_t np, uint32_t fr, uint32_t w, int32_t pad_id,
                                                                 uint32_t left, int32_t *out, int2 *spans,
                                                                 int32_t *lengths) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
    const uint32_t i = static_cast<uint32_t>(row_sentence[row]), f = static_cast<uint32_t>(row_first[row]);
    const unsigned long long o = id_offsets[i];
    const uint32_t L = static_cast<uint32_t>(id_offsets[i + 1] - o) - fr;
    const uint32_t body = min(L - f, w - fr);
    const uint32_t real = body + fr;
    const uint32_t lead = left ? w - real : 0u;
    int32_t *ro = out + static_cast<unsigned long long>(row) * w;
    int2 *rs = spans + static_cast<unsigned long long>(row) * w;
    for (uint32_t t = lane; t < w; t += 32) {
      const uint32_t k = t - lead;  // wraps past `real` for the leading pad cells
      if (k < real) {
        const unsigned long long q = o + (k < np ? k : k < np + body ? k + f : k + L - body);
        __stcs(ro + t, ids[q]);
        __stcs(rs + t, make_int2(static_cast<int32_t>(begin[q]), static_cast<int32_t>(end[q])));
      } else {
        __stcs(ro + t, pad_id);
        __stcs(rs + t, make_int2(0, 0));
      }
    }
    if (lane == 0) lengths[row] = static_cast<int32_t>(real);
  }
}

// The rows of spm_encode_pairs_device with offsets: one warp per pair row, gathered from K11's packed output over the
// 2n sentences with no frame (sentence i's list at id_offsets[i]), laid out as write_pair_rows_kernel
// (padded_kernel.cuh) lays out its id rows; template and pad cells get (0, 0).
__global__ void __launch_bounds__(256) write_pair_spans_kernel(const int32_t *ids, const uint32_t *begin,
                                                               const uint32_t *end,
                                                               const unsigned long long *id_offsets, uint32_t n,
                                                               uint32_t rows, KPairs T, const uint2 *keep,
                                                               const int32_t *row_pair, const int32_t *row_first,
                                                               uint32_t w, int32_t pad_id, uint32_t left, int32_t *out,
                                                               int32_t *type_ids, int2 *spans, int32_t *lengths) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
    const uint32_t i = static_cast<uint32_t>(row_pair[row]);
    const unsigned long long oa = id_offsets[i], ob = id_offsets[n + i];
    const PairRow p = pair_row(T, static_cast<uint32_t>(row_first[row]), keep[i],
                               static_cast<uint32_t>(id_offsets[i + 1] - oa),
                               static_cast<uint32_t>(id_offsets[n + i + 1] - ob));
    const uint32_t lead = left ? w - p.real : 0u;
    const uint32_t second = T.np + p.ca + T.nm;
    const unsigned long long at = static_cast<unsigned long long>(row) * w;
    for (uint32_t t = lane; t < w; t += 32) {
      const uint32_t k = t - lead;  // wraps past `real` for the leading pad cells
      int32_t id = pad_id, type = 0;
      int2 sp = make_int2(0, 0);
      if (k < p.real) {
        uint32_t q;
        const uint32_t c = pair_cell(T, p, k, q);
        if (c == 0) {
          id = T.tmpl[q];
        } else {
          const unsigned long long g = (c == 1 ? oa : ob) + q;
          id = ids[g];
          sp = make_int2(static_cast<int32_t>(begin[g]), static_cast<int32_t>(end[g]));
        }
        type = k >= second ? 1 : 0;
      }
      __stcs(out + at + t, id);
      __stcs(type_ids + at + t, type);
      __stcs(spans + at + t, sp);
    }
    if (lane == 0) lengths[row] = static_cast<int32_t>(p.real);
  }
}

// The chunk plan of a device batch (spm_encode_offsets_device_padded): the cuts spm_encode_offsets makes on the host
// -- chunk c is the longest run of sentences from its first whose slabs (norm_slab_start) stay within chunk_slab, at
// least one sentence -- found by warp 0 of block 0 with a 32-way search per cut (the slab of a run grows with its end).
// plan[0] = the chunks, plan[1] = the largest chunk slab, plan[2] = the longest sentence in bytes (every block);
// plan[4 + 2c] / plan[5 + 2c] = chunk c's first sentence and its byte offset, for c < max_cuts.  plan[0..3) are zeroed
// by the caller.  n > 0.
__global__ void __launch_bounds__(256) offsets_plan_kernel(const uint64_t *offs, uint32_t n, uint32_t expand,
                                                           unsigned long long chunk_slab, uint32_t max_cuts,
                                                           unsigned long long *plan) {
  unsigned long long longest = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    longest = max(longest, static_cast<unsigned long long>(offs[i + 1] - offs[i]));
  longest = __reduce_max_sync(0xFFFFFFFFu, static_cast<unsigned>(min(longest, 0xFFFFFFFFull)));
  if ((threadIdx.x & 31) == 0) atomicMax(plan + 2, longest);
  if (blockIdx.x != 0 || threadIdx.x >= 32) return;
  const uint32_t lane = threadIdx.x;
  uint32_t chunks = 0;
  unsigned long long slab_max = 0;
  for (uint32_t lo = 0; lo < n;) {
    const uint64_t base = offs[lo];
    // the largest hi in [lo + 1, n] whose run [lo, hi) fits, or lo + 1.  It lies in [a, b]; lane j probes
    // h_j = a + ceil((b - a)(j + 1) / 32), which rises with j to h_31 = b, and `fits` falls as h rises
    uint32_t a = lo + 1, b = n;
    while (a < b) {
      const unsigned long long span = b - a;
      const uint32_t h = a + static_cast<uint32_t>((span * (lane + 1) + 31u) / 32u);
      const uint32_t m = __ballot_sync(0xFFFFFFFFu, norm_slab_start(offs[h] - base, h - lo, expand) <= chunk_slab);
      const uint32_t h0 = a + static_cast<uint32_t>((span + 31u) / 32u);
      if (!m) {
        b = h0 - 1u;
      } else {
        const uint32_t last = 31u - __clz(m);
        const uint32_t ha = __shfl_sync(0xFFFFFFFFu, h, last);
        const uint32_t hb = __shfl_sync(0xFFFFFFFFu, h, last < 31u ? last + 1u : 31u);
        a = ha;
        b = last < 31u ? hb - 1u : b;
      }
    }
    const uint32_t hi = a;
    if (lane == 0 && chunks < max_cuts) {
      plan[4 + 2 * chunks] = lo;
      plan[5 + 2 * chunks] = base;
    }
    slab_max = max(slab_max, norm_slab_start(offs[hi] - base, hi - lo, expand));
    ++chunks;
    lo = hi;
  }
  if (lane == 0) {
    plan[0] = chunks;
    plan[1] = slab_max;
  }
}

}  // namespace spm_b200
#endif
