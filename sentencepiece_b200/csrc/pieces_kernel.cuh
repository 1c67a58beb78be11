// pieces_kernel.cuh -- K9: batched EncodeAsPieces -> packed piece strings (spm_encode_pieces).
//
// Reference: SentencePieceProcessor::PopulateSentencePieceText (src/sentencepiece_processor.cc:547-636) followed by
// ApplyExtraOptions (:1019-1064).  The piece of token k of the raw segmentation is IdToPiece(id) for every id but the
// unknown one; an unknown token (a whole run of unknown characters, merged by K4) is its surface in the normalized
// text.  The options then reverse the list, put bos / eos pieces around it (the encode frame, KFrame) and, with
// UNK_PIECE, replace the piece of every unknown token by trainer_spec.unk_piece.
//
// The model has exactly one UNKNOWN piece (ModelInterface::InitializePieces, model_interface.cc:101-110), so "unknown"
// is id == unk_id.  Every other piece comes from a per-id table of the raw piece bytes (U+2581 kept).  Unknown
// surfaces come from the spans path, which only the sentences that hold an unknown id take (the flag pass below).
//
// One WARP per list, one token per lane, output positions by a warp scan -- the shape of K7
// (decode_kernel.cuh).  A size pass writes each list's byte and token counts; the scan kernels of the encode path
// turn them into offsets; the write pass writes the bytes, the piece ends and the framed ids in place.
//
// A list is one sentence's segmentation (EncodeAsPieces) or one candidate of the n-best / sampling paths
// (spm_nbest_encode_pieces, spm_sample_encode_pieces): list j then reads its ids from the candidate buffer at
// list_start[j], the ends of its tokens from the parallel tok_end, and the normalized text of sentence j / per, which
// K5 exported only for sentences whose lattice holds an UNK node.
#ifndef SPM_B200_PIECES_KERNEL_CUH_
#define SPM_B200_PIECES_KERNEL_CUH_

#include <cstdint>

#include "device_model.h"

namespace spm_b200 {

constexpr uint32_t kNoSub = 0xFFFFFFFFu;  // sub_of[i]: sentence i did not take the unknown-surface path
constexpr uint32_t kPieceWarpCopy = 32;   // pieces longer than this are copied by the whole warp

struct KPieces {
  uint32_t n;  // lists
  // raw segmentation (no frame): list j is ids[id_offsets[j], id_offsets[j + 1]) or, when list_start is given,
  // ids[list_start[j], + list_count[j])
  const int32_t *ids;
  const unsigned long long *id_offsets;
  const unsigned long long *list_start;
  const uint32_t *list_count;
  // token ends parallel to ids (null: none); list j's normalized text at sent_norm + sent_norm_start[j / per] (kNoNorm:
  // the sentence has no unknown surface)
  const uint32_t *tok_end;
  const uint8_t *sent_norm;
  const unsigned long long *sent_norm_start;
  uint32_t per;
  // the unknown-surface subset: sentence i is sentence sub_of[i] of a spans run (null: no subset)
  const uint32_t *sub_of;
  const int32_t *sub_ids;
  const uint32_t *sub_tok_end;
  const unsigned long long *sub_id_offsets;
  const uint8_t *norm;
  const unsigned long long *norm_offsets;
  // piece table
  const uint32_t *pc_off;  // [vocab+1]
  const uint8_t *pc_bytes;
  int32_t unk_id;
  const uint8_t *unk_piece;  // null: unknown tokens keep their surface
  uint32_t unk_len;
  int32_t sep;  // -1: pieces abut; else this byte between consecutive pieces of a sentence
  KFrame F;
  // size pass
  uint32_t *text_len;  // [n]
  uint32_t *n_tok;     // [n]
  // write pass
  const unsigned long long *text_offsets;  // [n+1]
  const unsigned long long *out_id_offsets;
  uint8_t *text;
  uint32_t *piece_end;
  int32_t *out_ids;
};

// The raw segmentation of one sentence: its ids and, when it took the spans path, the ends of its tokens in its
// normalized text.
struct PiecesSrc {
  const int32_t *ids;
  const uint32_t *tok_end;  // null: no unknown surfaces
  const uint8_t *norm;
  uint32_t L;
};

__device__ __forceinline__ PiecesSrc pieces_src(const KPieces &P, uint32_t sent) {
  PiecesSrc s{};
  const uint32_t j = P.sub_of ? P.sub_of[sent] : kNoSub;
  if (j == kNoSub) {
    unsigned long long a;
    if (P.list_start) {
      a = P.list_start[sent];
      s.L = P.list_count[sent];
    } else {
      a = P.id_offsets[sent];
      s.L = static_cast<uint32_t>(P.id_offsets[sent + 1] - a);
    }
    s.ids = P.ids + a;
    if (P.tok_end) {
      const unsigned long long b = P.sent_norm_start[sent / P.per];
      if (b != kNoNorm) {
        s.tok_end = P.tok_end + a;
        s.norm = P.sent_norm + b;
      }
    }
  } else {
    const unsigned long long a = P.sub_id_offsets[j];
    s.ids = P.sub_ids + a;
    s.tok_end = P.sub_tok_end + a;
    s.norm = P.norm + P.norm_offsets[j];
    s.L = static_cast<uint32_t>(P.sub_id_offsets[j + 1] - a);
  }
  return s;
}

// Token t (< np + L + ns) of the framed list: its id and the bytes of its piece.  np = 0 for a list without a frame.
__device__ __forceinline__ int32_t piece_at(const KPieces &P, const PiecesSrc &s, uint32_t np, uint32_t t,
                                            const uint8_t **src, uint32_t *len) {
  int32_t id;
  uint32_t q = 0xFFFFFFFFu;  // index in the raw segmentation, for body tokens
  if (t < np) {
    id = P.F.ids[t];
  } else if (t - np < s.L) {
    q = P.F.reverse ? s.L - 1u - (t - np) : t - np;
    id = s.ids[q];
  } else {
    id = P.F.ids[np + (t - np - s.L)];
  }
  if (id == P.unk_id && P.unk_piece) {
    *src = P.unk_piece;
    *len = P.unk_len;
  } else if (id == P.unk_id && q != 0xFFFFFFFFu && s.tok_end) {
    const uint32_t b = q ? s.tok_end[q - 1] : 0u;
    *src = s.norm + b;
    *len = s.tok_end[q] - b;
  } else {
    const uint32_t o = __ldg(P.pc_off + id);
    *src = P.pc_bytes + o;
    *len = __ldg(P.pc_off + id + 1) - o;
  }
  return id;
}

// Flag pass: sub_len[i] = 1 when the raw segmentation of sentence i holds the unknown id.
__global__ void __launch_bounds__(256) pieces_unk_flag_kernel(const int32_t *ids, const unsigned long long *id_offsets,
                                                              uint32_t n, int32_t unk_id, uint32_t *flag) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t sent = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; sent < n; sent += warps) {
    const unsigned long long a = id_offsets[sent];
    const uint32_t L = static_cast<uint32_t>(id_offsets[sent + 1] - a);
    bool hit = false;
    for (uint32_t base = 0; base < L && !hit; base += 32)
      hit = __any_sync(0xFFFFFFFFu, base + lane < L && ids[a + base + lane] == unk_id);
    if (lane == 0) flag[sent] = hit ? 1u : 0u;
  }
}

// The flagged sentences as a list: sub_of[i] = their rank (pos = exclusive scan of the flags), and the source range of
// each flagged sentence's bytes for the gather that packs them.
__global__ void __launch_bounds__(256) pieces_sub_list_kernel(const uint32_t *flag, const unsigned long long *pos,
                                                              const uint64_t *offsets, uint32_t n, uint32_t *sub_of,
                                                              unsigned long long *sub_start, uint32_t *sub_len) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!flag[i]) { sub_of[i] = kNoSub; continue; }
    const uint32_t j = static_cast<uint32_t>(pos[i]);
    sub_of[i] = j;
    sub_start[j] = offsets[i];
    sub_len[j] = static_cast<uint32_t>(offsets[i + 1] - offsets[i]);
  }
}

// WRITE = false: the size pass (text_len, n_tok); WRITE = true: the write pass at text_offsets / out_id_offsets.
template <bool WRITE>
__global__ void __launch_bounds__(256) pieces_warp_kernel(const KPieces P) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t sep_w = P.sep >= 0 ? 1u : 0u;
  for (uint32_t sent = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; sent < P.n; sent += warps) {
    const PiecesSrc s = pieces_src(P, sent);
    const uint32_t added = P.F.added(sent);  // 0: an empty n-best slot, which stays empty
    const uint32_t np = added ? P.F.np : 0u;
    const uint32_t T = s.L + added;
    uint8_t *out = nullptr;
    uint32_t *ends = nullptr;
    int32_t *oids = nullptr;
    if (WRITE) {
      out = P.text + P.text_offsets[sent];
      ends = P.piece_end + P.out_id_offsets[sent];
      oids = P.out_ids + P.out_id_offsets[sent];
    }
    uint32_t run = 0;  // bytes of the sentence written by earlier trips
    for (uint32_t base = 0; base < T; base += 32) {
      const uint32_t t = base + lane;
      const uint8_t *src = nullptr;
      uint32_t len = 0, w = 0;
      int32_t id = 0;
      if (t < T) {
        id = piece_at(P, s, np, t, &src, &len);
        w = len + (t + 1 < T ? sep_w : 0u);
      }
      uint32_t incl = w;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if (lane >= static_cast<uint32_t>(d)) incl += v;
      }
      if (WRITE) {
        const uint32_t start = run + incl - w;
        uint8_t *dst = out + start;
        if (t < T) {
          ends[t] = start + len;
          oids[t] = id;
          if (w > len) dst[len] = static_cast<uint8_t>(P.sep);
        }
        // short pieces: every lane copies its own; long ones (unknown runs): the whole warp, one piece at a time
        const bool own = len <= kPieceWarpCopy;
        const uint32_t mx = __reduce_max_sync(0xFFFFFFFFu, own ? len : 0u);
        for (uint32_t k = 0; k < mx; ++k)
          if (own && k < len) dst[k] = src[k];
        for (uint32_t m = __ballot_sync(0xFFFFFFFFu, !own); m; m &= m - 1u) {
          const int j = __ffs(m) - 1;
          const uint8_t *js = reinterpret_cast<const uint8_t *>(__shfl_sync(0xFFFFFFFFu, reinterpret_cast<unsigned long long>(src), j));
          uint8_t *jd = reinterpret_cast<uint8_t *>(__shfl_sync(0xFFFFFFFFu, reinterpret_cast<unsigned long long>(dst), j));
          const uint32_t jl = __shfl_sync(0xFFFFFFFFu, len, j);
          for (uint32_t k = lane; k < jl; k += 32) jd[k] = js[k];
        }
      }
      run += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
    if (!WRITE && lane == 0) {
      P.text_len[sent] = run;
      P.n_tok[sent] = T;
    }
  }
}

}  // namespace spm_b200
#endif
