// kernels.cuh -- sm_90a kernels of the batched subword-encode engine: the general path.
//
// One sentence is owned by one warp (a TILE of 32 lanes).  The 32 lanes split the
// parallel parts of the reference algorithm -- normalizing from every byte position,
// walking the piece trie from every character start -- and take the inherently serial
// parts -- the Viterbi relaxation order and the back-trace -- in the reference's
// order.  All cross-lane traffic is warp shuffles / ballots / redux.
//
// Per sentence, entirely inside shared memory:
//   K1 normalize   Normalizer::Normalize + NormalizePrefix   normalizer.cc:71-253
//                  (+ Darts commonPrefixSearch over the charsmap, darts.h:469-513)
//   K2 viterbi     unigram::Model::EncodeOptimized           unigram_model.cc:889-1020
//   K4 finish      PopulateSentencePieceText id path         sentencepiece_processor.cc:547-636
// (K3, the BPE merge loop, lives in bpe_kernel.cuh.)
//
// HBM traffic per sentence is the input bytes + offsets in, ids + offsets out;
// the model tables (~1 MB) are L2 resident and their hot prefix is staged into
// shared memory once per CTA with a bulk (TMA) copy.
#ifndef SPM_B200_KERNELS_CUH_
#define SPM_B200_KERNELS_CUH_

#include <cuda_runtime.h>
#include <stdint.h>

#include "device_model.h"
#include "trie_builder.h"

namespace spm_b200 {

// ---------------------------------------------------------------- tile ----

struct Tile {
  int lane;  // lane inside the warp
  __device__ __forceinline__ Tile() : lane(threadIdx.x & 31) {}
  __device__ __forceinline__ uint32_t ballot(bool p) const { return __ballot_sync(0xFFFFFFFFu, p); }
  template <typename T>
  __device__ __forceinline__ T shfl(T v, int src) const { return __shfl_sync(0xFFFFFFFFu, v, src, 32); }
  __device__ __forceinline__ uint32_t red_or(uint32_t v) const { return __reduce_or_sync(0xFFFFFFFFu, v); }
  __device__ __forceinline__ uint32_t red_add(uint32_t v) const { return __reduce_add_sync(0xFFFFFFFFu, v); }
  __device__ __forceinline__ void sync() const { __syncwarp(0xFFFFFFFFu); }
  // inclusive scan over the tile
  __device__ __forceinline__ uint32_t incl_scan(uint32_t v) const {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, v, d, 32);
      if (lane >= d) v += t;
    }
    return v;
  }
  __device__ __forceinline__ uint32_t below() const { return (1u << lane) - 1u; }
};

// Scratch of one tile (generic pointers: shared memory on the fast path, a global
// slab on the long-sentence path).
struct TileMem {
  uint8_t *text;    // [ncap + 16]  normalized text
  float *score;     // [ncap + 4]   best_path_score per byte position
  uint32_t *bidx;   // [ncap + 4]   trie unit of the winning piece (kIdxUnk for UNK)
  uint16_t *blen;   // [ncap + 4]   byte length of the winning piece; 0 = unset (starts_at == -1)
  uint32_t *mval;   // [32 * K]     match buffer: score bits / marker
  uint32_t *midx;   // [32 * K]     match buffer: trie unit
  uint16_t *mlen;   // [32 * K]     match buffer: piece byte length
  uint32_t *n2o;    // [ncap + 4]   (spans) norm_to_orig
  uint8_t *stage;   // input staging (aliases score/bidx)
  uint32_t ncap;
  uint32_t stage_cap;
};

__host__ __device__ inline uint32_t tile_bytes_for(uint32_t ncap, uint32_t K, bool spans) {
  uint32_t b = (ncap + 16);                 // text
  b += 4 * (ncap + 4) * 2;                  // score, bidx
  b += 2 * (ncap + 4);                      // blen
  b += 32 * K * (4 + 4 + 2);                // match buffer
  if (spans) b += 4 * (ncap + 4);
  return (b + 15u) & ~15u;
}

__device__ __forceinline__ TileMem carve_tile(uint8_t *base, uint32_t ncap, uint32_t K, bool spans) {
  TileMem m;
  uint8_t *p = base;
  m.score = reinterpret_cast<float *>(p); p += 4 * (ncap + 4);
  m.bidx = reinterpret_cast<uint32_t *>(p); p += 4 * (ncap + 4);
  m.stage = reinterpret_cast<uint8_t *>(m.score);
  m.stage_cap = 8 * (ncap + 4);
  m.mval = reinterpret_cast<uint32_t *>(p); p += 4 * 32 * K;
  m.midx = reinterpret_cast<uint32_t *>(p); p += 4 * 32 * K;
  m.n2o = reinterpret_cast<uint32_t *>(p); if (spans) p += 4 * (ncap + 4);
  m.blen = reinterpret_cast<uint16_t *>(p); p += 2 * (ncap + 4);
  m.mlen = reinterpret_cast<uint16_t *>(p); p += 2 * 32 * K;
  m.text = p;
  m.ncap = ncap;
  return m;
}

// Hot prefix of the piece trie in shared memory.
struct HotTrie {
  const uint32_t *s_link;
  const uint32_t *s_val;
  const uint32_t *g_link;
  const uint32_t *g_val;
  uint32_t hot_link, hot_val;
  __device__ __forceinline__ uint32_t link(uint32_t u) const { return u < hot_link ? s_link[u] : __ldg(g_link + u); }
  __device__ __forceinline__ uint32_t val(uint32_t u) const { return u < hot_val ? s_val[u] : __ldg(g_val + u); }
};

// ---------------------------------------------------------------- utf-8 ---

// string_util::OneCharLen, src/util.h:151-153
__device__ __forceinline__ uint32_t one_char_len(uint32_t lead) {
  // "\1\1\1\1\1\1\1\1\1\1\1\1\2\2\3\4"[lead >> 4], packed 2 bits per entry (len - 1)
  return ((0xE5000000u >> ((lead >> 4) * 2)) & 3u) + 1u;
}
__device__ __forceinline__ bool is_trail(uint32_t c) { return (c & 0xC0u) == 0x80u; }

// DecodeUTF8 + IsValidDecodeUTF8, src/util.cc:51-84, src/util.h:173-176.
// Returns the byte length of a valid character at p (1..4) or 0 if malformed.
__device__ __forceinline__ uint32_t valid_utf8_len(const uint8_t *p, uint32_t len) {
  const uint32_t b0 = p[0];
  if (b0 < 0x80u) return 1;
  if (len >= 2 && (b0 & 0xE0u) == 0xC0u) {
    const uint32_t b1 = p[1];
    const uint32_t cp = ((b0 & 0x1Fu) << 6) | (b1 & 0x3Fu);
    if (is_trail(b1) && cp >= 0x80u) return 2;
  } else if (len >= 3 && (b0 & 0xF0u) == 0xE0u) {
    const uint32_t b1 = p[1], b2 = p[2];
    const uint32_t cp = ((b0 & 0x0Fu) << 12) | ((b1 & 0x3Fu) << 6) | (b2 & 0x3Fu);
    if (is_trail(b1) && is_trail(b2) && cp >= 0x800u && (cp < 0xD800u || cp >= 0xE000u)) return 3;
  } else if (len >= 4 && (b0 & 0xF8u) == 0xF0u) {
    const uint32_t b1 = p[1], b2 = p[2], b3 = p[3];
    const uint32_t cp = ((b0 & 0x07u) << 18) | ((b1 & 0x3Fu) << 12) | ((b2 & 0x3Fu) << 6) | (b3 & 0x3Fu);
    if (is_trail(b1) && is_trail(b2) && is_trail(b3) && cp >= 0x10000u && cp <= 0x10FFFFu) return 4;
  }
  return 0;
}

// ------------------------------------------------------------ charsmap ----

// Darts::DoubleArrayUnit, third_party/darts_clone/darts.h:50-80
__device__ __forceinline__ uint32_t da_offset(uint32_t u) { return (u >> 10) << ((u & (1u << 9)) >> 6); }
__device__ __forceinline__ uint32_t da_label(uint32_t u) { return u & ((1u << 31) | 0xFFu); }

// Longest key of the charsmap that is a prefix of p[0..len) -- the loop of
// commonPrefixSearch (darts.h:469-513) keeping only the last (= longest) result,
// as NormalizePrefix does (normalizer.cc:215-228).
__device__ __forceinline__ uint32_t charsmap_longest(const KModel &M, const uint8_t *p, uint32_t len, uint32_t *value) {
  uint32_t longest = 0;
  uint32_t node = 0;
  uint32_t unit = __ldg(M.cm_units);
  node ^= da_offset(unit);
  for (uint32_t i = 0; i < len; ++i) {
    const uint32_t c = p[i];
    node ^= c;
    if (node >= M.cm_nunits) break;
    unit = __ldg(M.cm_units + node);
    if (da_label(unit) != c) break;
    node ^= da_offset(unit);
    if ((unit >> 8) & 1u) {
      longest = i + 1;
      *value = __ldg(M.cm_units + node) & 0x7FFFFFFFu;
    }
  }
  return longest;
}

// The same walk with the first `have` bytes taken from a register window (the lane kernels' ByteStream holds the next
// 5..8 input bytes): no global byte load in front of every trie step for the usual 2..4-byte keys.
__device__ __forceinline__ uint32_t charsmap_longest_win(const KModel &M, unsigned long long win, uint32_t have,
                                                         const uint8_t *p, uint32_t len, uint32_t *value) {
  uint32_t longest = 0;
  uint32_t node = 0;
  uint32_t unit = __ldg(M.cm_units);
  node ^= da_offset(unit);
  for (uint32_t i = 0; i < len; ++i) {
    const uint32_t c = i < have ? static_cast<uint32_t>(win >> (8u * i)) & 0xFFu : static_cast<uint32_t>(p[i]);
    node ^= c;
    if (node >= M.cm_nunits) break;
    unit = __ldg(M.cm_units + node);
    if (da_label(unit) != c) break;
    node ^= da_offset(unit);
    if ((unit >> 8) & 1u) {
      longest = i + 1;
      *value = __ldg(M.cm_units + node) & 0x7FFFFFFFu;
    }
  }
  return longest;
}

// PrefixMatcher::PrefixMatch over the user-defined-symbol trie (normalizer.cc:324-346):
// longest user symbol that is a prefix of p, 0 if none.
__device__ __forceinline__ uint32_t user_longest(const KModel &M, const uint8_t *p, uint32_t len) {
  uint32_t longest = 0;
  uint32_t l = __ldg(M.user_link);
  for (uint32_t i = 0; i < len; ++i) {
    const uint32_t c = p[i];
    const uint32_t v = (l >> kLinkBaseShift) ^ c;
    l = __ldg(M.user_link + v);
    if ((l & kLinkLabelMask) != c) break;
    if ((l >> kLinkKindShift) & 3u) longest = i + 1;
  }
  return longest;
}

// --------------------------------------------------------- K1 normalize ---

// Result of normalizing one sentence.
struct NormResult {
  uint32_t n;          // normalized length (may exceed ncap: then nothing past ncap was stored)
  uint32_t consumed;   // final `consumed` (norm_to_orig[n]), spans only
};

// chunk kinds
enum : uint32_t { kChunkChar = 0, kChunkTarget = 1, kChunkFffd = 2, kChunkVerbatim = 3 };

template <bool SPANS>
__device__ __forceinline__ NormResult normalize_tile(const KModel &M, const Tile &T, const uint8_t *in,
                                                     uint32_t len, const TileMem &tm) {
  const bool rm = M.flags & kFlagRemoveExtraWs;
  const bool esc = M.flags & kFlagEscapeWs;
  const bool suffix = M.flags & kFlagWsSuffix;
  const bool addp = M.flags & kFlagAddDummyPrefix;
  const uint32_t w = esc ? 3u : 1u;
  const uint32_t ncap = tm.ncap;
  uint8_t *text = tm.text;
  NormResult r;
  r.n = 0;
  r.consumed = 0;
  if (len == 0) return r;  // normalizer.cc:77-79

  uint32_t out = 0;
  // dummy prefix (normalizer.cc:128); its norm_to_orig entries are patched below once the
  // number of heading-space bytes is known.
  if (addp && !suffix) {
    if (T.lane == 0) {
      if (esc) { text[0] = 0xE2; text[1] = 0x96; text[2] = 0x81; } else { text[0] = ' '; }
    }
    out = w;
  }
  bool prev_space = rm;  // is_prev_space, normalizer.cc:130
  bool seen = !rm;       // a chunk other than " " was seen: heading-space loop (:86-95) is over
  uint32_t first_q = 0;  // bytes consumed by the heading-space loop
  uint32_t carry = 0;    // bytes at the start of the window owned by a chunk of the previous one

  for (uint32_t pos = 0; pos < len; pos += 32) {
    const uint32_t q = pos + T.lane;
    const bool act = q < len;
    const uint32_t b = act ? in[q] : 0u;
    uint32_t clen = 1, kind = kChunkChar, tgt = 0;
    // ---- NormalizePrefix at every byte position of the window (speculative) ----
    if (act) {
      bool done = false;
      if (M.flags & kFlagHasUserSymbols) {  // normalizer.cc:201-205
        const uint32_t ul = user_longest(M, in + q, len - q);
        if (ul) { clen = ul; kind = kChunkVerbatim; done = true; }
      }
      if (!done) {
        uint32_t longest = 0, value = 0;
        if (M.flags & kFlagHasCharsmap) {
          const bool lead = (__ldg(M.cm_lead + (b >> 5)) >> (b & 31u)) & 1u;
          if (lead) {
            if (b < 0x80u) {
              // ASCII fast path: if root->b has no child on the next byte, the only
              // possible rule is the one-byte key b itself.
              bool cont = false;
              if (q + 1 < len) {
                const uint32_t c = in[q + 1];
                cont = (__ldg(M.cm_pair + ((b * 256u + c) >> 5)) >> (c & 31u)) & 1u;
              }
              if (cont) {
                longest = charsmap_longest(M, in + q, len - q, &value);
              } else {
                const int32_t so = __ldg(M.cm_solo + b);
                if (so >= 0) { longest = 1; value = static_cast<uint32_t>(so); }
              }
            } else {
              longest = charsmap_longest(M, in + q, len - q, &value);
            }
          }
        }
        if (longest) {
          clen = longest; kind = kChunkTarget; tgt = value;
        } else {  // normalizer.cc:231-244
          const uint32_t l = valid_utf8_len(in + q, len - q);
          if (l) { clen = l; kind = kChunkChar; } else { clen = 1; kind = kChunkFffd; }
        }
      }
    }
    // ---- which positions are real chunk starts: follow q -> q + clen from `carry` ----
    const uint32_t actmask = T.ballot(act);
    uint32_t startmask;
    if (T.ballot(act && clen != 1) == 0) {
      startmask = carry < 32u ? (actmask & ~((1u << carry) - 1u)) : 0u;
    } else {
      startmask = carry < 32u ? (1u << carry) : 0u;
      uint32_t nxt = T.lane + clen;
      if (nxt > 32u) nxt = 32;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {  // pointer doubling: reach 2^k - 1 hops after k rounds
        const uint32_t contrib = (((startmask >> T.lane) & 1u) && nxt < 32u) ? (1u << nxt) : 0u;
        startmask |= T.red_or(contrib);
        const uint32_t n2 = T.shfl(nxt, nxt < 32u ? static_cast<int>(nxt) : 0);
        nxt = nxt < 32u ? n2 : 32u;
      }
      startmask &= actmask;
    }
    const bool st = (startmask >> T.lane) & 1u;
    if (startmask) {
      const int last = 31 - __clz(startmask);
      const uint32_t jl = T.shfl(static_cast<uint32_t>(T.lane) + clen, last);
      carry = jl > 32u ? jl - 32 : 0u;
    } else {
      carry -= 32;
    }
    // ---- the chunk's replacement string: length, spaces, leading spaces, last byte ----
    uint32_t L = 0, nsp = 0, lead_sp = 0;
    bool ends_sp = false;
    const uint8_t *src = in + q;
    if (st) {
      if (kind == kChunkChar) {
        L = clen;
        nsp = lead_sp = (b == ' ') ? 1u : 0u;
        ends_sp = (b == ' ');
      } else if (kind == kChunkFffd) {
        L = 3;
      } else {
        if (kind == kChunkTarget) src = M.cm_targets + tgt;
        bool inlead = true;
        uint32_t lastch = 0;
        for (;;) {
          if (kind == kChunkVerbatim && L == clen) break;
          const uint32_t ch = src[L];
          if (kind == kChunkTarget && ch == 0) break;  // NUL-delimited, normalizer.cc:247-249
          if (ch == ' ') { ++nsp; if (inlead) ++lead_sp; } else { inlead = false; }
          lastch = ch;
          ++L;
        }
        ends_sp = L && lastch == ' ';
      }
    }
    // ---- is_prev_space before each chunk (normalizer.cc:130-162) ----
    // A chunk is E (empty: state unchanged), S (only spaces: state becomes true) or
    // T (has a non-space: state becomes "ends with space").
    const bool nonE = st && L > 0;
    const bool after_true = nonE && (nsp == L || ends_sp);
    const uint32_t m_nonE = T.ballot(nonE), m_true = T.ballot(after_true);
    bool p = prev_space;
    {
      const uint32_t below = m_nonE & T.below();
      if (below) p = (m_true >> (31 - __clz(below))) & 1u;
    }
    if (!rm) p = false;
    if (m_nonE) prev_space = rm && ((m_true >> (31 - __clz(m_nonE))) & 1u);
    // heading-space loop: chunks that are exactly " " before the first other chunk
    {
      const uint32_t m_other = T.ballot(st && !(L == 1 && nsp == 1));
      if (!seen && m_other) {
        seen = true;
        first_q = pos + (__ffs(m_other) - 1);
      }
    }
    // ---- emit ----
    const uint32_t strip = p ? lead_sp : 0u;
    const uint32_t emit = st ? (L - strip) + (w - 1u) * (nsp - strip) : 0u;
    const uint32_t incl = T.incl_scan(emit);
    const uint32_t total = T.shfl(incl, 31);
    if (emit) {
      uint32_t o = out + incl - emit;
      for (uint32_t k = strip; k < L; ++k) {
        const uint32_t ch = kind == kChunkFffd ? (k == 0 ? 0xEFu : (k == 1 ? 0xBFu : 0xBDu)) : src[k];
        if (ch == ' ' && esc) {
          if (o + 2 < ncap) {
            text[o] = 0xE2; text[o + 1] = 0x96; text[o + 2] = 0x81;
            if (SPANS) { tm.n2o[o] = q; tm.n2o[o + 1] = q; tm.n2o[o + 2] = q; }
          }
          o += 3;
        } else {
          if (o < ncap) { text[o] = static_cast<uint8_t>(ch); if (SPANS) tm.n2o[o] = q; }
          o += 1;
        }
      }
    }
    out += total;
  }
  // all chunks were heading spaces: "all chars are whitespace" (normalizer.cc:97-100)
  if (rm && !seen) return r;
  if (out > ncap) { r.n = out + w; return r; }  // does not fit: the caller defers the sentence
  if (SPANS && addp && !suffix && T.lane == 0)
    for (uint32_t k = 0; k < w; ++k) tm.n2o[k] = first_q;
  T.sync();
  uint32_t consumed = len;
  // trailing spaces (normalizer.cc:166-176) -- on the ESCAPED output
  if (rm) {
    if (esc) {
      while (out >= 3 && text[out - 3] == 0xE2 && text[out - 2] == 0x96 && text[out - 1] == 0x81) {
        out -= 3;
        if (SPANS) consumed = tm.n2o[out];
      }
    } else {
      while (out >= 1 && text[out - 1] == ' ') {
        out -= 1;
        if (SPANS) consumed = tm.n2o[out];
      }
    }
  }
  if (SPANS) T.sync();
  // dummy suffix (normalizer.cc:179)
  if (suffix && addp) {
    if (out + w > ncap) { r.n = out + w; return r; }
    if (T.lane == 0) {
      if (esc) { text[out] = 0xE2; text[out + 1] = 0x96; text[out + 2] = 0x81; } else { text[out] = ' '; }
      if (SPANS) for (uint32_t k = 0; k < w; ++k) tm.n2o[out + k] = consumed;
    }
    out += w;
  }
  if (SPANS && T.lane == 0) tm.n2o[out] = consumed;
  T.sync();
  r.n = out;
  r.consumed = consumed;
  return r;
}

// ---------------------------------------------------------- K2 viterbi ----

// unigram::Model::EncodeOptimized, src/unigram_model.cc:889-1020, for one tile.
// Phase A (parallel): every lane walks the piece trie from its own character start
// and buffers its matches.  Phase B (ordered): starts are folded into
// best_path_ends_at[] in increasing order, the matches of one start relaxed in
// parallel (they have distinct end positions).  This reproduces the reference's
// relaxation order exactly, including Q1 (double candidate vs float-rounded best)
// and Q2 (strict >, earliest start wins ties).
__device__ __forceinline__ void viterbi_tile(const KModel &M, const Tile &T, const HotTrie &H, const TileMem &tm,
                                             uint32_t n) {
  const uint8_t *text = tm.text;
  const uint32_t K = M.match_slots;
  for (uint32_t k = T.lane; k <= n; k += 32) tm.blen[k] = 0;
  if (T.lane == 0) tm.score[0] = 0.f;
  T.sync();
  const uint32_t root_link = H.link(0);
  uint32_t *mval = tm.mval + T.lane * K;
  uint32_t *midx = tm.midx + T.lane * K;
  uint16_t *mlen = tm.mlen + T.lane * K;
  for (uint32_t wnd = 0; wnd < n; wnd += 32) {
    const uint32_t s = wnd + T.lane;
    uint32_t cnt = 0;
    bool active = false;
    if (s < n) {
      const uint32_t lead = text[s];
      active = !is_trail(lead);  // normalized text is valid UTF-8: starts are the lead bytes
      if (active) {
        uint32_t mblen = one_char_len(lead);
        if (mblen > n - s) mblen = n - s;
        bool has_single = false;
        uint32_t l = root_link;
        for (uint32_t k = s; k < n; ++k) {  // trie_->traverse one byte at a time, :969-972
          const uint32_t c = text[k];
          const uint32_t v = (l >> kLinkBaseShift) ^ c;
          l = H.link(v);
          if ((l & kLinkLabelMask) != c) break;
          const uint32_t kind = (l >> kLinkKindShift) & 3u;
          if (kind == kKindNormal || kind == kKindUserDefined) {  // UNUSED pieces are skipped, :974
            const uint32_t plen = k + 1 - s;
            if (cnt < K) {
              mval[cnt] = kind == kKindNormal ? H.val(v) : kValUserDefined;
              midx[cnt] = v;
              mlen[cnt] = static_cast<uint16_t>(plen);
            }
            ++cnt;
            if (plen == mblen) has_single = true;  // :990-992
          }
        }
        if (!has_single) {  // UNK edge of one character, :995-1005
          if (cnt < K) { mval[cnt] = kValUnk; midx[cnt] = kIdxUnk; mlen[cnt] = static_cast<uint16_t>(mblen); }
          ++cnt;
        }
      }
    }
    T.sync();
    // ---- ordered fold ----
    uint32_t amask = T.ballot(active);
    while (amask) {
      const int j = __ffs(amask) - 1;
      amask &= amask - 1;
      const uint32_t sj = wnd + j;
      const uint32_t cntj = T.shfl(cnt, j);
      const float till_here = tm.score[sj];  // best_path_score_till_here, :963-964
      for (uint32_t m = T.lane; m < cntj; m += 32) {
        const uint32_t val = tm.mval[j * K + m];
        const uint32_t plen = tm.mlen[j * K + m];
        const uint32_t e = sj + plen;
        const float cur = tm.score[e];
        const bool unset = tm.blen[e] == 0;
        float ns;
        bool better;
        if (val == kValUnk) {
          ns = __fadd_rn(M.unk_score, till_here);  // float + float, :997-998
          better = unset || ns > cur;
        } else {
          // `score` is double (common type of double and float), :979-983
          const double sc = val == kValUserDefined
                                ? static_cast<double>(__fmul_rn(static_cast<float>(plen), M.max_score)) - 0.1
                                : static_cast<double>(__uint_as_float(val));
          const double cand = sc + static_cast<double>(till_here);
          better = unset || cand > static_cast<double>(cur);
          ns = static_cast<float>(cand);
        }
        if (better) {
          tm.score[e] = ns;
          tm.blen[e] = static_cast<uint16_t>(plen);
          tm.bidx[e] = tm.midx[j * K + m];
        }
      }
      T.sync();
    }
  }
}

// ------------------------------------------------------------ K4 finish ---

// Back-trace (unigram_model.cc:1010-1018) followed by the id path of
// PopulateSentencePieceText (sentencepiece_processor.cc:547-636): consecutive
// unknown pieces collapse into one id, or -- with byte fallback -- every byte of
// an unknown piece becomes its <0xXX> id.  Tokens are appended to the batch's
// temporary id buffer at a position claimed with one atomicAdd per sentence.
template <bool SPANS>
__device__ __forceinline__ void finish_tokens(const KModel &M, const KBatch &B, const Tile &T, const uint8_t *text,
                                              const uint32_t *tend, const int32_t *tid, uint32_t sent, uint32_t n_tok) {
  // tokens k = 0..n_tok-1: exclusive end offset tend[k] in the normalized text, vocab id tid[k]
  constexpr uint32_t slot0 = 0;
  const bool bf = M.flags & kFlagByteFallback;
  const int32_t unk = M.unk_id;
  // pass 1: count output tokens
  uint32_t count = 0;
  for (uint32_t k0 = 0; k0 < n_tok; k0 += 32) {
    const uint32_t k = k0 + T.lane;
    uint32_t c = 0;
    if (k < n_tok) {
      const bool isunk = tid[slot0 + k] == unk;
      if (bf) {
        c = isunk ? tend[slot0 + k] - (k ? tend[slot0 + k - 1] : 0u) : 1u;
      } else {
        const bool prevunk = k && tid[slot0 + k - 1] == unk;
        c = !(isunk && prevunk);
      }
    }
    count += T.red_add(c);
  }
  unsigned long long pos = 0;
  if (T.lane == 0) {
    pos = atomicAdd(B.cursor, static_cast<unsigned long long>(count));
    B.sent_start[sent] = pos;
    B.sent_count[sent] = count;
    if (pos + count > B.tmp_cap) atomicOr(B.status + 2, 1u);
  }
  pos = T.shfl(pos, 0);
  if (pos + count > B.tmp_cap) return;
  // pass 2: write
  uint32_t base = 0;
  for (uint32_t k0 = 0; k0 < n_tok; k0 += 32) {
    const uint32_t k = k0 + T.lane;
    uint32_t c = 0;
    bool isunk = false;
    uint32_t start = 0, end = 0;
    int32_t id = 0;
    if (k < n_tok) {
      id = tid[slot0 + k];
      isunk = id == unk;
      end = tend[slot0 + k];
      start = k ? tend[slot0 + k - 1] : 0u;
      if (bf) {
        c = isunk ? end - start : 1u;
      } else {
        const bool prevunk = k && tid[slot0 + k - 1] == unk;
        c = !(isunk && prevunk);
      }
    }
    const uint32_t incl = T.incl_scan(c);
    const uint32_t rank = base + incl - c;
    if (k < n_tok) {
      if (bf && isunk) {
        for (uint32_t i = 0; i < c; ++i) {
          B.tmp_ids[pos + rank + i] = __ldg(M.byte_to_id + text[start + i]);
          if (SPANS) B.tmp_tok_end[pos + rank + i] = start + i + 1;
        }
      } else {
        if (c) B.tmp_ids[pos + rank] = id;
        if (SPANS) {
          // the last piece of an unknown run carries the run's end offset
          const bool nextunk = (k + 1 < n_tok) && tid[slot0 + k + 1] == unk;
          if (bf || !(isunk && nextunk)) B.tmp_tok_end[pos + base + incl - 1] = end;
        }
      }
    }
    base += T.shfl(incl, 31);
  }
}

// Publishes the normalized text + alignment of one sentence (spans API).
__device__ __forceinline__ void publish_norm_tile(const KBatch &B, const Tile &T, const TileMem &tm, uint32_t sent,
                                                  uint32_t n, bool have_map) {
  unsigned long long pos = 0;
  if (T.lane == 0) {
    pos = atomicAdd(B.cursor + 1, static_cast<unsigned long long>(n) + 1ull);
    B.norm_start[sent] = pos;
    B.norm_len[sent] = n;
    if (pos + n + 1 > B.tmp_norm_cap) atomicOr(B.status + 2, 2u);
  }
  pos = T.shfl(pos, 0);
  if (pos + n + 1 > B.tmp_norm_cap) return;
  for (uint32_t k = T.lane; k < n; k += 32) B.tmp_norm[pos + k] = tm.text[k];
  if (have_map)
    for (uint32_t k = T.lane; k <= n; k += 32) B.tmp_n2o[pos + k] = tm.n2o[k];
}

// One sentence, unigram model: K1 -> K2 -> K4.  Returns false if the sentence does
// not fit the tile's scratch (the caller defers it to the long-sentence kernel).
template <bool SPANS>
__device__ __forceinline__ bool encode_unigram_sentence(const KModel &M, const KBatch &B, const Tile &T,
                                                        const HotTrie &H, const TileMem &tm, const uint8_t *in,
                                                        uint32_t len, uint32_t sent, uint32_t *need) {
  const NormResult nr = normalize_tile<SPANS>(M, T, in, len, tm);
  const uint32_t n = nr.n;
  if (n > tm.ncap) { *need = n; return false; }
  if (SPANS) publish_norm_tile(B, T, tm, sent, n, n > 0);
  if (n == 0) {
    if (T.lane == 0) { B.sent_start[sent] = 0; B.sent_count[sent] = 0; }
    return true;
  }
  viterbi_tile(M, T, H, tm, n);
  // back-trace by one lane; token records are packed in place at the top of the DP
  // arrays (slot n - t for the t-th token from the end: that slot is >= the current
  // position, whose entry has already been read).
  uint32_t n_tok = 0;
  if (T.lane == 0) {
    uint32_t e = n;
    uint32_t *tend = reinterpret_cast<uint32_t *>(tm.score);
    while (e > 0) {
      const uint32_t bl = tm.blen[e];
      const uint32_t ix = tm.bidx[e];
      if (bl == 0 || bl > e) { atomicOr(B.status + 1, 1u); break; }  // cannot happen: every start has an edge
      const uint32_t slot = n - n_tok;
      tm.bidx[slot] = ix;
      tend[slot] = e;
      e -= bl;
      ++n_tok;
    }
  }
  n_tok = T.shfl(n_tok, 0);
  T.sync();
  // resolve trie units to vocab ids (one L2 read per token)
  for (uint32_t k = T.lane; k < n_tok; k += 32) {
    const uint32_t slot = n - n_tok + 1 + k;
    const uint32_t ix = tm.bidx[slot];
    tm.bidx[slot] = static_cast<uint32_t>(ix == kIdxUnk ? M.unk_id : __ldg(M.trie_id + ix));
  }
  T.sync();
  finish_tokens<SPANS>(M, B, T, tm.text, reinterpret_cast<const uint32_t *>(tm.score) + (n - n_tok + 1),
                       reinterpret_cast<const int32_t *>(tm.bidx) + (n - n_tok + 1), sent, n_tok);
  return true;
}

// ------------------------------------------------------------ staging -----

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// Bulk (TMA, non-tensor) copy of the hot trie prefix global -> shared, completion
// signalled on an mbarrier; SASS: UBLKCP.
__device__ __forceinline__ void stage_hot_trie(const KModel &M, uint64_t *mbar, uint32_t *s_link, uint32_t *s_val) {
  const uint32_t bytes_link = M.hot_link * 4u, bytes_val = M.hot_val * 4u;
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(mbar)), "r"(1));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(mbar)),
                 "r"(bytes_link + bytes_val)
                 : "memory");
    if (bytes_link)
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                       smem_u32(s_link)),
                   "l"(M.trie_link), "r"(bytes_link), "r"(smem_u32(mbar))
                   : "memory");
    if (bytes_val)
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                       smem_u32(s_val)),
                   "l"(M.trie_val), "r"(bytes_val), "r"(smem_u32(mbar))
                   : "memory");
  }
  // every thread waits for phase 0 to complete
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(mbar)),
      "r"(0)
      : "memory");
}

// ------------------------------------------------------------- kernels ----

// Persistent kernel: every warp loops over sentences claimed one at a time from a
// global counter; inputs are staged into shared memory with aligned 16-byte loads.
template <bool SPANS>
__global__ void __launch_bounds__(512, 1) encode_unigram_kernel(const KModel M, const KBatch B) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t *mbar = reinterpret_cast<uint64_t *>(smem);
  uint32_t *s_link = reinterpret_cast<uint32_t *>(smem + 16);
  uint32_t *s_val = s_link + M.hot_link;
  uint8_t *tiles = reinterpret_cast<uint8_t *>(s_val + M.hot_val);
  stage_hot_trie(M, mbar, s_link, s_val);
  HotTrie H{s_link, s_val, M.trie_link, M.trie_val, M.hot_link, M.hot_val};

  const Tile T;
  const TileMem tm = carve_tile(tiles + static_cast<size_t>(threadIdx.x >> 5) * B.tile_bytes, B.ncap, M.match_slots, SPANS);

  for (;;) {
    uint32_t widx = 0;
    if (T.lane == 0) widx = atomicAdd(B.work_counter, 1u);
    widx = __shfl_sync(0xFFFFFFFFu, widx, 0);
    const uint32_t work_n = B.sub_list ? B.sub_n : B.n;
    if (widx >= work_n) break;
    const uint32_t sent = B.sub_list ? B.sub_list[2 * widx] : widx;
    const unsigned long long off = B.offsets[sent];
    const unsigned long long len64 = B.offsets[sent + 1] - off;
    bool fits = len64 + 32ull <= tm.stage_cap;
    uint32_t need = 0;
    if (fits) {
      const uint32_t len = static_cast<uint32_t>(len64);
      // coalesced, vectorised staging of the input bytes (16-byte aligned loads)
      const uint8_t *g = B.bytes + off;
      const uint32_t mis = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(g) & 15u);
      const uint4 *ga = reinterpret_cast<const uint4 *>(g - mis);
      const uint32_t nvec = (mis + len + 15u) >> 4;
      uint4 *sa = reinterpret_cast<uint4 *>(tm.stage);
      for (uint32_t v = T.lane; v < nvec; v += 32) sa[v] = __ldg(ga + v);
      T.sync();
      fits = encode_unigram_sentence<SPANS>(M, B, T, H, tm, tm.stage + mis, len, sent, &need);
    }
    if (!fits && T.lane == 0) {
      const uint32_t slot = atomicAdd(B.status, 1u);
      B.deferred[2 * slot] = sent;
      B.deferred[2 * slot + 1] = need;  // exact normalized length if known, else 0
    }
    __syncwarp();
  }
}

// Long sentences: one warp per sentence, scratch in a global slab sized for the
// sentence; input read straight from HBM/L2.
template <bool SPANS>
__global__ void __launch_bounds__(256) encode_unigram_long_kernel(const KModel M, const KBatch B) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t *mbar = reinterpret_cast<uint64_t *>(smem);
  uint32_t *s_link = reinterpret_cast<uint32_t *>(smem + 16);
  uint32_t *s_val = s_link + M.hot_link;
  stage_hot_trie(M, mbar, s_link, s_val);
  HotTrie H{s_link, s_val, M.trie_link, M.trie_val, M.hot_link, M.hot_val};
  const Tile T;
  const uint32_t warps_per_cta = blockDim.x >> 5;
  for (uint32_t w = blockIdx.x * warps_per_cta + (threadIdx.x >> 5); w < B.long_n; w += gridDim.x * warps_per_cta) {
    const uint32_t sent = B.long_list[2 * w];
    const unsigned long long so = B.long_scratch_off[w];
    const unsigned long long bytes = B.long_scratch_off[w + 1] - so;
    // invert tile_bytes_for(): the host sized the slab for ncap
    const uint32_t ncap = B.long_list[2 * w + 1];
    (void)bytes;
    const TileMem tm = carve_tile(B.long_scratch + so, ncap, M.match_slots, SPANS);
    const unsigned long long off = B.offsets[sent];
    const uint32_t len = static_cast<uint32_t>(B.offsets[sent + 1] - off);
    uint32_t need = 0;
    const bool ok = encode_unigram_sentence<SPANS>(M, B, T, H, tm, B.bytes + off, len, sent, &need);
    if (!ok && T.lane == 0) atomicOr(B.status + 1, 8u);  // slab sized from an upper bound too small: its own bit and message
    __syncwarp();
  }
}

// ------------------------------------------------- offsets + compaction ---

// Exclusive scan of per-sentence counts into 64-bit offsets, three small kernels
// (block sums, scan of block sums, block scan) -- pure streaming over 4-byte counts.
constexpr int kScanChunk = 2048;  // counts per block (256 threads x 8)

// FRAMED: id lists that get the encode frame (KFrame) -- each framed item counts np + ns more.
template <bool FRAMED = false>
__global__ void __launch_bounds__(256) scan_block_sums_kernel(const uint32_t *counts, uint32_t n,
                                                              unsigned long long *block_sums, uint32_t extra,
                                                              KFrame F = KFrame{}) {
  __shared__ unsigned long long warp_sums[8];
  const uint32_t base = blockIdx.x * kScanChunk;
  unsigned long long s = 0;
  for (uint32_t k = threadIdx.x; k < kScanChunk; k += 256) {
    const uint32_t i = base + k;
    if (i < n) s += counts[i] + extra + (FRAMED ? F.added(i) : 0u);
  }
  for (int d = 16; d > 0; d >>= 1) s += __shfl_down_sync(0xFFFFFFFFu, s, d);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int i = 0; i < 8; ++i) t += warp_sums[i];
    block_sums[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(1024) scan_block_prefix_kernel(unsigned long long *block_sums, uint32_t nb,
                                                                 unsigned long long *total_out) {
  __shared__ unsigned long long sh[1024];
  __shared__ unsigned long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < nb; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    const unsigned long long v = i < nb ? block_sums[i] : 0ull;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {
      const unsigned long long t = threadIdx.x >= d ? sh[threadIdx.x - d] : 0ull;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    if (i < nb) block_sums[i] = carry + sh[threadIdx.x] - v;  // exclusive
    __syncthreads();
    if (threadIdx.x == 1023) carry += sh[1023];
    __syncthreads();
  }
  if (threadIdx.x == 0) *total_out = carry;
}

// Block scan of counts -> offsets[i]; then every sentence's tokens are moved from
// completion order (tmp) to sentence order (out): coalesced 4-byte copies, 8 lanes
// per sentence.
// FRAMED (id lists only): the frame F is written around each framed item's ids, which are copied backwards when
// F.reverse.  A template flag rather than a run-time test, so that the text and norm_to_orig instantiations and the
// unframed id path keep their code as it was.
template <typename ElemT, bool FRAMED = false>
__global__ void __launch_bounds__(256) scan_write_gather_kernel(const uint32_t *counts, uint32_t n,
                                                                const unsigned long long *block_prefix,
                                                                unsigned long long *offsets,
                                                                const unsigned long long *src_start,
                                                                const ElemT *src, ElemT *dst,
                                                                const uint32_t *src2, uint32_t *dst2,
                                                                unsigned long long dst_cap, uint32_t extra,
                                                                unsigned long long off_base, KFrame F = KFrame{}) {
  static_assert(!FRAMED || sizeof(ElemT) == 4, "the frame applies to id lists");
  __shared__ unsigned long long sh_off[kScanChunk + 1];
  __shared__ unsigned long long warp_sums[8];
  const uint32_t base = blockIdx.x * kScanChunk;
  // each thread owns 8 consecutive counts
  uint32_t c[8];
  unsigned long long local = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint32_t i = base + threadIdx.x * 8 + k;
    c[k] = i < n ? counts[i] + extra + (FRAMED ? F.added(i) : 0u) : 0u;
    local += c[k];
  }
  unsigned long long incl = local;
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
    if ((threadIdx.x & 31) >= d) incl += t;
  }
  if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = incl;
  __syncthreads();
  unsigned long long wbase = block_prefix[blockIdx.x];
  for (int w = 0; w < (threadIdx.x >> 5); ++w) wbase += warp_sums[w];
  unsigned long long run = wbase + incl - local;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint32_t i = base + threadIdx.x * 8 + k;
    sh_off[threadIdx.x * 8 + k] = run;
    if (i < n) offsets[i] = run + off_base;  // off_base: ids of the batch's earlier chunks (pipelined host API)
    run += c[k];
    if (i + 1 == n) offsets[n] = run + off_base;
  }
  __syncthreads();
  if (dst == nullptr) return;
  // gather: 8 lanes per sentence
  const uint32_t lane8 = threadIdx.x & 7;
  if constexpr (FRAMED) {
    for (uint32_t k = threadIdx.x >> 3; k < kScanChunk; k += 32) {
      const uint32_t i = base + k;
      if (i >= n) break;
      const uint32_t body = counts[i];
      const uint32_t cnt = body + F.added(i);  // (an empty n-best slot has body 0 and no frame: nothing to write)
      const unsigned long long d0 = sh_off[k];
      if (d0 + cnt > dst_cap) continue;
      const ElemT *s = src + src_start[i];
      for (uint32_t t = lane8; t < cnt; t += 8)
        __stcs(dst + d0 + t, F.at(body, t, [&](uint32_t q) { return __ldcs(s + q); }));
    }
    return;
  }
  for (uint32_t k = threadIdx.x >> 3; k < kScanChunk; k += 32) {
    const uint32_t i = base + k;
    if (i >= n) break;
    const uint32_t cnt = counts[i] + extra;
    const unsigned long long d0 = sh_off[k];
    if (d0 + cnt > dst_cap) continue;
    const unsigned long long s0 = src_start[i];
    for (uint32_t t = lane8; t < cnt; t += 8) {  // streaming both ways
      __stcs(dst + d0 + t, __ldcs(src + s0 + t));
      if (dst2) __stcs(dst2 + d0 + t, __ldcs(src2 + s0 + t));
    }
  }
}

}  // namespace spm_b200
#endif
